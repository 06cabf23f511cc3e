"""TEST INFRASTRUCTURE ONLY.  Builds the primitive probe of the device arithmetic (rt_probe.cu in this directory):

    _build/librt_probe.so       nvcc, with the product's own NVCC_FLAGS (imported, so the two builds cannot drift apart)
    _build/librt_probe_simt.so  g++ against the SIMT interpreter of tests/simt (-DRT_SIMT_EMU): the same source on the CPU

The product (ray_tracing_b200/, bench.py) never builds or loads either library."""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
if REPO not in sys.path:
    sys.path.insert(0, REPO)

from ray_tracing_b200 import build as product_build   # noqa: E402


def _load(name: str, path: str):
    import importlib.util
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


simt_build = _load("simt_build", os.path.join(REPO, "tests", "simt", "build.py"))

SRC = os.path.join(HERE, "rt_probe.cu")
OUT_DIR = os.path.join(HERE, "_build")
LIB_PROBE = os.path.join(OUT_DIR, "librt_probe.so")
LIB_PROBE_SIMT = os.path.join(OUT_DIR, "librt_probe_simt.so")


def _sources() -> list[str]:
    csrc = os.path.join(REPO, "ray_tracing_b200", "csrc")
    inc = os.path.join(REPO, "include")
    return [SRC] + [os.path.join(csrc, f) for f in os.listdir(csrc)] + [os.path.join(inc, f) for f in os.listdir(inc)]


def _stale(target: str, extra: list[str] = ()) -> bool:
    return not os.path.exists(target) or any(os.path.getmtime(s) > os.path.getmtime(target) for s in _sources() + list(extra))


def _run(cmd: list[str]) -> None:
    print("[probe build]", " ".join(cmd), flush=True)
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("probe build failed")


def build_gpu(force: bool = False, flags: list[str] | None = None, out: str = "") -> str:
    """nvcc build for sm_90a.  `flags` / `out`: build a variant with other code-generation flags (e.g. -fmad=true) elsewhere."""
    target = out or LIB_PROBE
    os.makedirs(os.path.dirname(target), exist_ok=True)
    if force or out or _stale(target):
        _run([product_build.nvcc_path()] + (flags if flags is not None else product_build.NVCC_FLAGS) +
             ["-I", os.path.join(REPO, "include"), "-o", target, SRC])
    return target


def build_simt(force: bool = False) -> str:
    shim = simt_build.SHIM
    os.makedirs(OUT_DIR, exist_ok=True)
    if force or _stale(LIB_PROBE_SIMT, [os.path.join(shim, f) for f in os.listdir(shim)]):
        _run([os.environ.get("CXX", "g++")] + simt_build.FLAGS + ["-I", shim, "-I", os.path.join(REPO, "include"),
                                                                   "-x", "c++", SRC, "-o", LIB_PROBE_SIMT])
    return LIB_PROBE_SIMT


if __name__ == "__main__":
    print(build_simt(force=True))
    print(build_gpu(force=True))
