"""In-tree build of the native code (no JIT cache: the built .so files travel with the repo snapshot).

    librt_b200.so  — CUDA kernels + C-ABI (include/rt_b200.h), sm_90a (H100) only, built with nvcc.
    librt_host.so  — C++ host side above the C-ABI: BVH builder + RayComputeManager mirror (g++).
    oracle/liboracle.so — the CPU oracle (test infrastructure; built here only so that tests / bench can
                     load it — building the checker is not using it).
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
REPO_DIR = os.path.dirname(PKG_DIR)
CSRC = os.path.join(PKG_DIR, "csrc")
HOST = os.path.join(PKG_DIR, "host")
INCLUDE = os.path.join(REPO_DIR, "include")
ORACLE = os.path.join(REPO_DIR, "oracle")
ORACLE_EXT = os.path.join(REPO_DIR, "tests", "oracle_ext")

LIB_CUDA = os.path.join(PKG_DIR, "librt_b200.so")
LIB_HOST = os.path.join(PKG_DIR, "librt_host.so")
LIB_ORACLE = os.path.join(ORACLE, "liboracle.so")

# -fmad=false: no FMA contraction — every FP32 op is a separate IEEE operation (the arithmetic contract,
# csrc/rt_devmath.cuh).  -prec-div / -prec-sqrt / -ftz=false are the nvcc defaults, spelled out.
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-fmad=false", "-prec-div=true", "-prec-sqrt=true", "-ftz=false",
    "-Xcompiler", "-fPIC,-ffp-contract=off,-fno-fast-math",
    "-Xlinker", "-Bsymbolic",
    "-shared",
]
GXX_FLAGS = ["-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-pthread", "-shared",
             "-Wl,-Bsymbolic"]


def _newer(target: str, sources: list[str]) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in sources if os.path.exists(s))


def _glob(d: str, exts: tuple[str, ...]) -> list[str]:
    return sorted(os.path.join(d, f) for f in os.listdir(d) if f.endswith(exts)) if os.path.isdir(d) else []


def _run(cmd: list[str]) -> None:
    print("[build]", " ".join(cmd), flush=True)
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("build failed: " + " ".join(cmd))
    if r.stderr.strip():
        print(r.stderr.strip(), flush=True)


def nvcc_path() -> str:
    p = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(p):
        raise RuntimeError("nvcc not found")
    return p


def build_cuda(force: bool = False, verbose_ptxas: bool = False, defines: tuple = (), out: str = "") -> str:
    """Builds librt_b200.so; `defines` / `out` build an experimental variant next to it (A/B measurements)."""
    srcs = _glob(CSRC, (".cu", ".cuh")) + _glob(INCLUDE, (".h",))
    target = out or LIB_CUDA
    if force or _newer(target, srcs):
        cmd = [nvcc_path()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose_ptxas else []) + [f"-D{d}" for d in defines] + \
              ["-I", INCLUDE, "-o", target, os.path.join(CSRC, "rt_api.cu")]
        _run(cmd)
    return target


def build_host(force: bool = False) -> str:
    srcs = _glob(HOST, (".cpp", ".h")) + _glob(INCLUDE, (".h",))
    cpps = _glob(HOST, (".cpp",))
    if not cpps:
        return ""
    if force or _newer(LIB_HOST, srcs):
        _run([os.environ.get("CXX", "g++")] + GXX_FLAGS + ["-I", INCLUDE, "-o", LIB_HOST] + cpps + ["-ldl"])
    return LIB_HOST


def build_oracle(force: bool = False) -> str:
    # the oracle (oracle/rt_oracle.cpp) with its per-pixel counters (PixelStats) around it: the extension includes the oracle's
    # source unchanged and wraps the entry points that reach the counters (tests/oracle_ext/rt_oracle_pixel_stats.cpp); rtDispatchFrames
    # is the loop over single-frame dispatches around that (tests/oracle_ext/rt_oracle_frames.cpp); rtTraceRays is CalculateRayCollision
    # per ray around that in turn (tests/oracle_ext/rt_oracle_trace_rays.cpp); rtTraceOcclusion is its tMax-bounded early-exit walk
    # around that (tests/oracle_ext/rt_oracle_occlusion.cpp); rtTracePaths is Shader::Trace per sample of a caller ray around that
    # (tests/oracle_ext/rt_oracle_paths.cpp); rtDispatchFeatures / rtCameraRays are its camera sample, CalculateRayCollision and
    # GetMaterialColour per pixel around that (tests/oracle_ext/rt_oracle_features.cpp); rtDenoise is the a-trous filter over those
    # images around that (tests/oracle_ext/rt_oracle_denoise.cpp); rtDenoiseTemporal is the reprojected, variance-guided filter with its
    # history around that (tests/oracle_ext/rt_oracle_temporal.cpp); rtDispatchAdaptive is the selection on its moments and Kernel_RayTrace
    # per active pixel around that (tests/oracle_ext/rt_oracle_adaptive.cpp); rtBakeProbes is Shader::Trace per probe sample, its SH
    # chunk sums and their padded tree around that (tests/oracle_ext/rt_oracle_probes.cpp); rtBakeCubemaps is Shader::Trace per texel
    # sample, its chunk sums and their padded tree around that (tests/oracle_ext/rt_oracle_cubemaps.cpp); rtBakeLightmap is Shader::Trace
    # per surface-texel sample and the same sums around that (tests/oracle_ext/rt_oracle_lightmaps.cpp, the translation unit built here)
    srcs = _glob(ORACLE, (".cpp", ".h")) + _glob(ORACLE_EXT, (".cpp",)) + _glob(INCLUDE, (".h",))
    if force or _newer(LIB_ORACLE, srcs):
        _run([os.environ.get("CXX", "g++")] + GXX_FLAGS + ["-I", INCLUDE, "-o", LIB_ORACLE, os.path.join(ORACLE_EXT, "rt_oracle_lightmaps.cpp")])
    return LIB_ORACLE


def build_all(force: bool = False) -> None:
    build_cuda(force)
    build_host(force)
    build_oracle(force)


if __name__ == "__main__":
    build_all(force="--force" in sys.argv)
    print("ok")
