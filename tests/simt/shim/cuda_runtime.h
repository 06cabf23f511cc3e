// tests/simt/shim/cuda_runtime.h — TEST INFRASTRUCTURE ONLY.  A host stand-in for <cuda_runtime.h> that lets g++ compile
// ray_tracing_b200/csrc/rt_api.cu (kernels included) into tests/simt/_build/librt_b200_simt.so, so that the CPU test suite
// can execute the kernels' own source — warp ballots, shuffles, reductions, shared-memory pools, persistent-CTA work queue,
// vote state machine — lane by lane, without a GPU, and compare the result with the oracle bit for bit.
//
// It is a SIMT *interpreter of the schedule*, not a second implementation of the path: every arithmetic expression that
// runs is the product's (rt_device.cuh / rt_devmath.cuh / rt_kernel_*.cuh, compiled with -ffp-contract=off, i.e. the same
// one-IEEE-operation-per-operator contract nvcc gets from -fmad=false).  The product never loads this library: the package
// (ray_tracing_b200/*.py), bench.py and __graft_entry__.py do not know it exists; only tests/test_simt_kernels.py builds and
// opens it.  It says nothing about speed.
//
// Execution model (simt_core.h): one CTA at a time per worker OS thread; the CTA's threads are fibers (hand-written x86-64
// context switch); a warp collective (__ballot_sync, __shfl_sync, __any_sync, __reduce_add_sync, __syncwarp) blocks a lane
// until every non-exited lane named in its mask has arrived; __syncthreads likewise for the CTA.  Divergent lanes really
// do run at different times, so a missing __syncwarp or a collective under divergent control flow shows up as a wrong
// result or a reported deadlock instead of passing by luck.
//
// Launches follow the H100's shared-memory rule: one above 48 KB of dynamic shared memory runs only if cudaFuncSetAttribute gave the
// kernel that much, and every launch that runs is logged as (kernel, bytes) for tests/test_simt_kernel_matrix.py.
#pragma once
#ifndef RT_SIMT_EMU
#error "tests/simt/shim/cuda_runtime.h is only for the RT_SIMT_EMU test build"
#endif

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <map>
#include <mutex>
#include <string>
#include <thread>
#include <vector>
#include <stdint.h>

// ---- qualifiers -----------------------------------------------------------------------------------------------------------
#define __device__
#define __host__
#define __global__
#define __forceinline__ inline __attribute__((always_inline))
#define __align__(n) __attribute__((aligned(n)))
#define __grid_constant__
#define __shared__ static thread_local      /* a static __shared__ array: one copy per worker thread = per resident CTA */
#define __launch_bounds__(...)

// ---- vector types -----------------------------------------------------------------------------------------------------------
struct __attribute__((aligned(16))) float4 { float x, y, z, w; };
struct __attribute__((aligned(16))) int4 { int x, y, z, w; };
struct __attribute__((aligned(16))) uint4 { unsigned int x, y, z, w; };
struct __attribute__((aligned(8))) int2 { int x, y; };
struct __attribute__((aligned(4))) uchar4 { unsigned char x, y, z, w; };
struct uint3 { unsigned int x, y, z; };
struct dim3
{
    unsigned int x, y, z;
    dim3(unsigned int x_ = 1, unsigned int y_ = 1, unsigned int z_ = 1) : x(x_), y(y_), z(z_) {}
};
static inline float4 make_float4(float x, float y, float z, float w) { float4 r; r.x = x; r.y = y; r.z = z; r.w = w; return r; }
static inline int4 make_int4(int x, int y, int z, int w) { int4 r; r.x = x; r.y = y; r.z = z; r.w = w; return r; }
static inline int2 make_int2(int x, int y) { int2 r; r.x = x; r.y = y; return r; }
static inline uchar4 make_uchar4(unsigned char x, unsigned char y, unsigned char z, unsigned char w) { uchar4 r; r.x = x; r.y = y; r.z = z; r.w = w; return r; }

#include "simt_core.h"
#include <cxxabi.h>

// ---- built-in variables (per fiber; refreshed by the scheduler at every switch) -------------------------------------------------
#define threadIdx (simt::tl_threadIdx)
#define blockIdx (simt::tl_blockIdx)
#define blockDim (simt::tl_blockDim)
#define gridDim (simt::tl_gridDim)

// ---- intrinsics -----------------------------------------------------------------------------------------------------------
// fminf / fmaxf as the GPU computes them (FMNMX): NaN-ignoring, and -0 ordered below +0.  libm's versions return their first argument
// for a pair of zeros, so the device code would see a different sign of zero here than on the GPU.
static inline float simt_fminf(float a, float b)
{
    if (a != a) return b;
    if (b != b) return a;
    if (a == b) { unsigned int u; memcpy(&u, &a, 4); return (u & 0x80000000u) ? a : b; }
    return a < b ? a : b;
}
static inline float simt_fmaxf(float a, float b)
{
    if (a != a) return b;
    if (b != b) return a;
    if (a == b) { unsigned int u; memcpy(&u, &a, 4); return (u & 0x80000000u) ? b : a; }
    return a > b ? a : b;
}
#define fminf simt_fminf
#define fmaxf simt_fmaxf
template <class T> static inline T __ldg(const T* p) { return *p; }
static inline int __popc(unsigned int v) { return __builtin_popcount(v); }
static inline int __ffs(unsigned int v) { return __builtin_ffs((int)v); }
static inline int __float_as_int(float f) { int i; memcpy(&i, &f, 4); return i; }
static inline float __int_as_float(int i) { float f; memcpy(&f, &i, 4); return f; }
static inline unsigned int __float_as_uint(float f) { unsigned int i; memcpy(&i, &f, 4); return i; }
static inline float __uint_as_float(unsigned int i) { float f; memcpy(&f, &i, 4); return f; }
static inline float __uint2float_rn(unsigned int u) { return (float)u; }            // default rounding mode = RNE
static inline float __int2float_rn(int i) { return (float)i; }
static inline unsigned int __float2uint_rz(float f)                                   // cvt.rzi.u32.f32 saturates; NaN -> 0
{
    if (!(f > 0.0f)) return 0u;
    if (f >= 4294967296.0f) return 0xffffffffu;
    return (unsigned int)f;
}

static inline unsigned int __activemask() { return simt::activemask(); }
static inline unsigned int __ballot_sync(unsigned int mask, int pred) { return (unsigned int)simt::collective(simt::OP_BALLOT, mask, pred ? 1u : 0u, 0); }
static inline int __any_sync(unsigned int mask, int pred) { return simt::collective(simt::OP_BALLOT, mask, pred ? 1u : 0u, 0) != 0; }
static inline unsigned int __reduce_add_sync(unsigned int mask, unsigned int v) { return (unsigned int)simt::collective(simt::OP_ADD, mask, v, 0); }
static inline void __syncwarp(unsigned int mask = 0xffffffffu) { simt::collective(simt::OP_SYNC, mask, 0, 0); }
static inline unsigned int __shfl_sync(unsigned int mask, unsigned int v, int srcLane) { return (unsigned int)simt::collective(simt::OP_SHFL, mask, v, srcLane); }
static inline int __shfl_sync(unsigned int mask, int v, int srcLane) { return (int)(unsigned int)simt::collective(simt::OP_SHFL, mask, (unsigned int)v, srcLane); }
static inline float __shfl_sync(unsigned int mask, float v, int srcLane) { return __uint_as_float((unsigned int)simt::collective(simt::OP_SHFL, mask, __float_as_uint(v), srcLane)); }
static inline unsigned int __shfl_down_sync(unsigned int mask, unsigned int v, unsigned int delta) { const unsigned int l = simt::lane_id(); return (unsigned int)simt::collective(simt::OP_SHFL, mask, v, l + delta < 32u ? (int)(l + delta) : (int)l); }
static inline int __shfl_down_sync(unsigned int mask, int v, unsigned int delta) { return (int)__shfl_down_sync(mask, (unsigned int)v, delta); }
static inline unsigned long long __shfl_down_sync(unsigned int mask, unsigned long long v, unsigned int delta)      // two 32-bit exchanges, as the hardware does
{
    const unsigned int lo = __shfl_down_sync(mask, (unsigned int)v, delta), hi = __shfl_down_sync(mask, (unsigned int)(v >> 32), delta);
    return ((unsigned long long)hi << 32) | lo;
}
static inline unsigned int __shfl_up_sync(unsigned int mask, unsigned int v, unsigned int delta) { const unsigned int l = simt::lane_id(); return (unsigned int)simt::collective(simt::OP_SHFL, mask, v, l >= delta ? (int)(l - delta) : (int)l); }
static inline int __shfl_up_sync(unsigned int mask, int v, unsigned int delta) { return (int)__shfl_up_sync(mask, (unsigned int)v, delta); }
static inline void __syncthreads() { simt::syncthreads(); }
static inline void __threadfence() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }

static inline unsigned int atomicAdd(unsigned int* p, unsigned int v) { return __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
static inline int atomicAdd(int* p, int v) { return __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
static inline unsigned int atomicMin(unsigned int* p, unsigned int v) { unsigned int old = __atomic_load_n(p, __ATOMIC_RELAXED); while (v < old && !__atomic_compare_exchange_n(p, &old, v, true, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) { } return old; }
static inline unsigned int atomicMax(unsigned int* p, unsigned int v) { unsigned int old = __atomic_load_n(p, __ATOMIC_RELAXED); while (v > old && !__atomic_compare_exchange_n(p, &old, v, true, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) { } return old; }
static inline unsigned long long atomicAdd(unsigned long long* p, unsigned long long v) { return __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
static inline unsigned long long atomicMin(unsigned long long* p, unsigned long long v) { unsigned long long old = __atomic_load_n(p, __ATOMIC_RELAXED); while (v < old && !__atomic_compare_exchange_n(p, &old, v, true, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) { } return old; }
static inline unsigned long long atomicMax(unsigned long long* p, unsigned long long v) { unsigned long long old = __atomic_load_n(p, __ATOMIC_RELAXED); while (v > old && !__atomic_compare_exchange_n(p, &old, v, true, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) { } return old; }

// ---- runtime API (the subset rt_api.cu / rt_repack.cuh call) ---------------------------------------------------------------------
typedef int cudaError_t;
enum : int { cudaSuccess = 0, cudaErrorInvalidValue = 1, cudaErrorMemoryAllocation = 2, cudaErrorInvalidConfiguration = 9, cudaErrorNotSupported = 801 };
enum cudaMemcpyKind { cudaMemcpyHostToHost = 0, cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2, cudaMemcpyDeviceToDevice = 3 };
enum : int { cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
enum : unsigned int { cudaStreamNonBlocking = 1, cudaIpcMemLazyEnablePeerAccess = 1 };
enum : unsigned long long { cudaEnableDefault = 0 };
enum cudaDriverEntryPointQueryResult { cudaDriverEntryPointSuccess = 0 };
struct simtStream; typedef simtStream* cudaStream_t;
struct simtEvent { std::chrono::steady_clock::time_point t; }; typedef simtEvent* cudaEvent_t;
struct cudaIpcMemHandle_t { char reserved[64]; };
struct cudaDeviceProp { int major, minor, multiProcessorCount; char name[64]; };

static inline const char* cudaGetErrorString(cudaError_t e)
{
    switch (e) { case 0: return "no error"; case 1: return "invalid value"; case 2: return "out of memory"; case 9: return "invalid configuration";
                 case 801: return "not supported by the SIMT test build"; default: return "error"; }
}
// The error a refused launch leaves pending for the launching host thread (per thread, as the runtime keeps it)
namespace simt { inline thread_local cudaError_t tl_lastError = cudaSuccess; }
static inline cudaError_t cudaGetLastError() { const cudaError_t e = simt::tl_lastError; simt::tl_lastError = cudaSuccess; return e; }
static inline cudaError_t cudaGetDeviceCount(int* n) { *n = 8; return cudaSuccess; }          // eight "devices" sharing the host's memory: lets rtCreateMulti groups run here
static inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
static inline cudaError_t cudaGetDeviceProperties(cudaDeviceProp* p, int)
{
    memset(p, 0, sizeof(*p)); p->major = 9; p->minor = 0; p->multiProcessorCount = simt::env_int("RT_SIMT_SMS", 2);
    snprintf(p->name, sizeof(p->name), "SIMT test interpreter"); return cudaSuccess;
}
static inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned int) { *s = nullptr; return cudaSuccess; }
static inline cudaError_t cudaStreamDestroy(cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }          // every call completes before it returns
template <class T> static inline cudaError_t cudaMalloc(T** p, size_t bytes)
{
    void* q = nullptr;
    if (posix_memalign(&q, 256, bytes ? bytes : 1) != 0) { *p = nullptr; return cudaErrorMemoryAllocation; }
    memset(q, 0xcd, bytes);                                                        // device memory is not zeroed: make a read of it visible
    *p = (T*)q; return cudaSuccess;
}
static inline cudaError_t cudaFree(void* p) { free(p); return cudaSuccess; }
static inline cudaError_t cudaMallocHost(void** p, size_t n) { *p = malloc(n ? n : 1); return *p ? cudaSuccess : cudaErrorMemoryAllocation; }
static inline cudaError_t cudaFreeHost(void* p) { free(p); return cudaSuccess; }
static inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) { memcpy(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t) { memcpy(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemset(void* d, int v, size_t n) { memset(d, v, n); return cudaSuccess; }
static inline cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t) { memset(d, v, n); return cudaSuccess; }
static inline cudaError_t cudaMemset2DAsync(void* d, size_t pitch, int v, size_t w, size_t h, cudaStream_t)
{
    for (size_t r = 0; r < h; r++) memset((char*)d + r * pitch, v, w);
    return cudaSuccess;
}
static inline cudaError_t cudaEventCreate(cudaEvent_t* e) { *e = new simtEvent(); return cudaSuccess; }
enum { cudaEventDisableTiming = 2 };
static inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned int) { *e = new simtEvent(); return cudaSuccess; }
static inline cudaError_t cudaEventDestroy(cudaEvent_t e) { delete e; return cudaSuccess; }
static inline cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t) { e->t = std::chrono::steady_clock::now(); return cudaSuccess; }
static inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
static inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned int) { return cudaSuccess; }
static inline cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t a, cudaEvent_t b)
{
    *ms = std::chrono::duration<float, std::milli>(b->t - a->t).count(); return cudaSuccess;
}
// cudaFuncAttributeMaxDynamicSharedMemorySize is recorded per function: simt::launch_kernel refuses a launch above 48 KB of dynamic
// shared memory that the function was not given, as the H100 does (the other attributes the product does not set)
namespace simt {
inline std::mutex attrMutex;
inline std::map<const void*, size_t> maxDynamicSmem;
}
template <class F> static inline cudaError_t cudaFuncSetAttribute(F f, int attr, int value)
{
    if (attr != cudaFuncAttributeMaxDynamicSharedMemorySize) return cudaErrorInvalidValue;
    if (value < 0 || value > 232448) return cudaErrorInvalidValue;
    std::lock_guard<std::mutex> lock(simt::attrMutex);
    simt::maxDynamicSmem[reinterpret_cast<const void*>(f)] = (size_t)value;
    return cudaSuccess;
}
template <class F> static inline cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessor(int* n, F, int, size_t) { *n = simt::env_int("RT_SIMT_CTAS_PER_SM", 2); return cudaSuccess; }
static inline cudaError_t cudaIpcGetMemHandle(cudaIpcMemHandle_t*, void*) { return cudaErrorNotSupported; }
static inline cudaError_t cudaIpcOpenMemHandle(void**, cudaIpcMemHandle_t, unsigned int) { return cudaErrorNotSupported; }
static inline cudaError_t cudaIpcCloseMemHandle(void*) { return cudaSuccess; }
static inline cudaError_t cudaGetDriverEntryPoint(const char*, void** fn, unsigned long long, cudaDriverEntryPointQueryResult*) { *fn = nullptr; return cudaErrorNotSupported; }

// ---- kernel launch ------------------------------------------------------------------------------------------------------------
#define RT_DYNAMIC_SMEM(name) unsigned char* const name = rtd::simtSmem
// A launch runs only when its dynamic shared memory is at most 48 KB or at most what cudaFuncSetAttribute gave the kernel; otherwise
// it leaves cudaErrorInvalidValue for cudaGetLastError, as the H100 does.  Every launch that runs is logged as (kernel's demangled
// symbol, dynamic shared-memory bytes) for the tests that check which instantiation a call chose (simtLaunchLog* below).
namespace simt {
constexpr size_t DEFAULT_DYNAMIC_SMEM = 48 * 1024;
struct LaunchRecord { std::string symbol; size_t smem; };
inline std::mutex logMutex;
inline std::vector<LaunchRecord> launchLog;

inline std::string kernel_symbol(const void* kern)
{
    Dl_info info; memset(&info, 0, sizeof(info));
    if (!dladdr(kern, &info) || !info.dli_sname || info.dli_saddr != kern) return "?";
    int status = 0;
    char* d = abi::__cxa_demangle(info.dli_sname, nullptr, nullptr, &status);
    std::string out = status == 0 && d ? d : info.dli_sname;
    free(d);
    return out;
}

inline void launch_kernel(const void* kern, dim3 grid, dim3 block, size_t smemBytes, const std::function<void()>& body)
{
    if (smemBytes > DEFAULT_DYNAMIC_SMEM)
    {
        std::lock_guard<std::mutex> lock(attrMutex);
        const auto it = maxDynamicSmem.find(kern);
        if (it == maxDynamicSmem.end() || smemBytes > it->second) { tl_lastError = cudaErrorInvalidValue; return; }
    }
    {
        LaunchRecord r{kernel_symbol(kern), smemBytes};
        std::lock_guard<std::mutex> lock(logMutex);
        launchLog.push_back(std::move(r));
    }
    launch(grid, block, smemBytes, body);
}
} // namespace simt

// The launch log, for the tests only (the product's ABI has no such calls): the number of records, record i's symbol and shared
// memory, and a reset
extern "C" __attribute__((visibility("default"))) size_t simtLaunchLogCount()
{
    std::lock_guard<std::mutex> lock(simt::logMutex);
    return simt::launchLog.size();
}
extern "C" __attribute__((visibility("default"))) size_t simtLaunchLogEntry(size_t i, char* symbol, size_t cap)
{
    std::lock_guard<std::mutex> lock(simt::logMutex);
    if (i >= simt::launchLog.size()) return 0;
    const simt::LaunchRecord& r = simt::launchLog[i];
    if (cap) { const size_t n = std::min(cap - 1, r.symbol.size()); memcpy(symbol, r.symbol.data(), n); symbol[n] = 0; }
    return r.smem;
}
extern "C" __attribute__((visibility("default"))) void simtLaunchLogReset()
{
    std::lock_guard<std::mutex> lock(simt::logMutex);
    simt::launchLog.clear();
}

#define RT_LAUNCH(grid, block, smem, stream, kern, ...) \
    simt::launch_kernel(reinterpret_cast<const void*>(kern), dim3(grid), dim3(block), (size_t)(smem), [&]() { kern(__VA_ARGS__); })

// ---- dynamic shared memory + the PTX helpers of rt_kernel_wave.cuh (mbarrier / TMA bulk copy), by their semantics ----------------
namespace rtd {
// the dynamic shared memory of the CTA a worker thread is running (RT_DYNAMIC_SMEM(name) in the kernels)
inline thread_local __attribute__((aligned(128))) unsigned char simtSmem[232448];
#define smemRaw simtSmem

static inline uint32_t smem_u32(const void* p) { return (uint32_t)((const unsigned char*)p - smemRaw); }
// mbarrier: 64-bit object {pending arrivals, pending transaction bytes, phase}
struct SimtMbar { int32_t arrivals; int32_t tx; };
static inline SimtMbar* simt_mbar(uint32_t off) { return reinterpret_cast<SimtMbar*>(smemRaw + off); }
static inline uint32_t& simt_mbar_phase(uint32_t off) { static thread_local std::map<uint32_t, uint32_t> ph; return ph[off]; }
static inline uint32_t& simt_mbar_count(uint32_t off) { static thread_local std::map<uint32_t, uint32_t> cn; return cn[off]; }
static inline void simt_mbar_check(uint32_t off)
{
    SimtMbar* m = simt_mbar(off);
    if (m->arrivals == 0 && m->tx == 0) { simt_mbar_phase(off) ^= 1u; m->arrivals = (int32_t)simt_mbar_count(off); }
}
static inline void mbar_init(uint32_t mbar, uint32_t count) { simt_mbar(mbar)->arrivals = (int32_t)count; simt_mbar(mbar)->tx = 0; simt_mbar_phase(mbar) = 0; simt_mbar_count(mbar) = count; }
static inline void mbar_fence_init() { }
static inline void mbar_expect_tx(uint32_t mbar, uint32_t bytes) { SimtMbar* m = simt_mbar(mbar); m->tx += (int32_t)bytes; m->arrivals -= 1; simt_mbar_check(mbar); }
static inline void tma_bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t mbar)
{
    if ((dst & 15u) || (bytes & 15u) || ((uintptr_t)src & 15u)) { fprintf(stderr, "simt: cp.async.bulk needs 16-byte aligned addresses and size\n"); abort(); }
    memcpy(smemRaw + dst, src, bytes);
    simt_mbar(mbar)->tx -= (int32_t)bytes; simt_mbar_check(mbar);
}
static inline bool mbar_try_wait(uint32_t mbar, uint32_t parity)
{
    if (simt_mbar_phase(mbar) != parity) return true;
    simt::yield();                                           // let the thread that issues the copy run
    return false;
}
#undef smemRaw
} // namespace rtd
