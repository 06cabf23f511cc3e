"""The kernel matrix of tests/test_gpu_kernel_matrix.py on the SIMT interpreter build (see tests/test_simt_kernels.py), plus what only the
CPU can check.  The interpreter's launch log (tests/simt/shim/cuda_runtime.h) records every launch as (kernel, dynamic shared memory), and
the interpreter refuses a launch above 48 KB of dynamic shared memory that cudaFuncSetAttribute did not allow, as the H100 does.  So:

  * completeness: the table's keys are exactly the __global__ functions of the nvcc build (cuobjdump -elf) and of the interpreter build;
  * reach: each row's call launches exactly its own kernel among the camera and query kernels (the single kernels: its own among
    others), the rows above 48 KB really are, and so are the kernel-2 rows;
  * parity: each row's buffers equal the oracle's bit for bit, and every call returns RT_OK (a refused launch would not)."""
import ctypes as C
import shutil
import subprocess

import pytest

from conftest import CUDA_LIB
import test_gpu_kernel_matrix as G
import test_simt_kernels as S

simt_lib = S.simt_lib

_libstdcxx = C.CDLL("libstdc++.so.6")
_libstdcxx.__cxa_demangle.restype = C.c_void_p
_libstdcxx.__cxa_demangle.argtypes = [C.c_char_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int)]
_libc = C.CDLL(None)
_libc.free.argtypes = [C.c_void_p]


def demangle(symbol: str) -> str:
    status = C.c_int(0)
    p = _libstdcxx.__cxa_demangle(symbol.encode(), None, None, C.byref(status))
    if status.value != 0 or not p:
        return symbol
    out = C.string_at(p).decode()
    _libc.free(p)
    return out


def kernel_name(demangled: str) -> str:
    """'void rtd::k_raytrace_pool<true, true, 96>(rtd::DevParams, ...)' -> 'k_raytrace_pool<true, true, 96>'"""
    name = demangled[5:] if demangled.startswith("void ") else demangled
    name = name.split("(", 1)[0]
    return name[5:] if name.startswith("rtd::") else name


def nvcc_kernels(lib=CUDA_LIB):
    """The __global__ functions of an nvcc build: one .text.<mangled name> section each in its sm_90a ELF."""
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    out = subprocess.run([tool, "-elf", lib], capture_output=True, text=True, check=True).stdout
    mangled = {tok[len(".text."):] for line in out.splitlines() for tok in line.split() if tok.startswith(".text._Z")}
    return {kernel_name(demangle(m)) for m in mangled}


def interpreter_kernels(lib):
    """The kernels of the interpreter build: its exported functions named rtd::k_* (the kernels' own names; __global__ means nothing there)."""
    out = subprocess.run(["nm", "-D", "--defined-only", lib], capture_output=True, text=True, check=True).stdout
    names = {kernel_name(demangle(line.split()[-1])) for line in out.splitlines() if len(line.split()) == 3}
    return {n for n in names if n.startswith("k_")}


class LaunchLog:
    def __init__(self, lib):
        self.L = C.CDLL(lib)
        self.L.simtLaunchLogCount.restype = C.c_size_t
        self.L.simtLaunchLogEntry.restype = C.c_size_t
        self.L.simtLaunchLogEntry.argtypes = [C.c_size_t, C.c_char_p, C.c_size_t]

    def reset(self):
        self.L.simtLaunchLogReset()

    def read(self):
        buf = C.create_string_buffer(4096)
        out = []
        for i in range(self.L.simtLaunchLogCount()):
            smem = self.L.simtLaunchLogEntry(i, buf, len(buf))
            out.append((kernel_name(buf.value.decode()), int(smem)))
        return out


@pytest.fixture(autouse=True)
def _point_matrix_at_the_interpreter(monkeypatch, simt_lib):
    monkeypatch.setattr(G, "CUDA_LIB", simt_lib)
    monkeypatch.setattr(G, "HOST_POINTERS", True)


@pytest.fixture(scope="module")
def launch_log(simt_lib):
    return LaunchLog(simt_lib)


# ---- completeness -------------------------------------------------------------------------------------------------------------------
def _same_sets(kernels, what):
    missing, stale = sorted(kernels - set(G.TABLE)), sorted(set(G.TABLE) - kernels)
    assert not missing and not stale, f"{what}: kernels without a row {missing}; rows without a kernel {stale}"


def test_simt_table_names_every_kernel_of_the_nvcc_build():
    _same_sets(nvcc_kernels(), "nvcc build")


def test_simt_table_names_every_kernel_of_the_interpreter_build(simt_lib):
    _same_sets(interpreter_kernels(simt_lib), "interpreter build")


def test_simt_every_kernel_1_instantiation_that_stages_tree_tops_has_a_row_above_48_kb():
    """Kernel 1's EXT and TLAS instantiations, read off their template arguments: <S, EXT, CHUNKED>, frames <S, EXT>, list <S, EXT, TLAS>."""
    staging = set()
    for k in G.TABLE:
        if k.startswith("k_raytrace_wave_tlas"):
            staging.add(k)
        elif k.startswith("k_raytrace_wave"):
            args = k.split("<", 1)[1].rstrip(">").split(", ")
            if "true" in (args[1:] if k.startswith("k_raytrace_wave_list") else args[1:2]):
                staging.add(k)
    assert set(G.SMEM_ROWS) == staging and len(staging) == 11, sorted(set(G.SMEM_ROWS) ^ staging)


# ---- reach and parity -----------------------------------------------------------------------------------------------------------------
CAMERA_AND_QUERY = {k for k, r in G.TABLE.items() if r.family != "single"}


def _run_and_check(simt_lib, launch_log, key, row, above_48_kb):
    launch_log.reset()
    got = G.run_row(simt_lib, row)
    log = launch_log.read()
    names = [n for n, _ in log]
    if row.family == "single":
        assert key in names, f"{key}: {row.entry} launched {sorted(set(names))}"
    else:
        assert set(names) & CAMERA_AND_QUERY == {key}, f"{key}: {row.entry} {row.options} launched {sorted(set(names) & CAMERA_AND_QUERY)}"
    if above_48_kb:
        smem = [s for n, s in log if n == key]
        assert smem and min(smem) > G.SMEM_DEFAULT, f"{key}: dynamic shared memory {smem} is not above 48 KB"
    G.assert_outputs_equal(got, G.oracle_outputs(row), f"{key} {row.entry} {row.options}")


@pytest.mark.parametrize("key", sorted(G.TABLE))
def test_simt_row_launches_its_kernel_and_equals_the_oracle(simt_lib, launch_log, key):
    row = G.TABLE[key]
    _run_and_check(simt_lib, launch_log, key, row, above_48_kb=row.family == "camera" and row.options["kernel"] == 2)


@pytest.mark.parametrize("key", sorted(G.SMEM_ROWS))
def test_simt_row_above_48_kb_launches_its_kernel_and_equals_the_oracle(simt_lib, launch_log, key):
    _run_and_check(simt_lib, launch_log, key, G.SMEM_ROWS[key], above_48_kb=True)

