"""The randomised searches of tools/ against the real kernels (librt_b200.so on the H100): random scenes, random sessions of host calls and
random meshes for rtBuildBVH and the host builder, compared bit for bit with the oracle.  Sorts last, so that `pytest -x -m gpu` reaches it
after every hand-made case.  On the CPU the same searches run against the SIMT interpreter build (tests/test_fuzz_smoke.py)."""
import os
import subprocess
import sys

import pytest

from conftest import CUDA_LIB, REPO
from test_fuzz_smoke import run_switches

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("tool,args", [("simt_fuzz.py", ["--cases", "250", "--seed", "301", "--far", "0.03", "--spheres", "0.06", "--odd", "0.1"]),
                                       ("simt_fuzz_session.py", ["--cases", "50", "--seed", "302"]),
                                       ("simt_fuzz_bvh.py", ["--cases", "150", "--seed", "303"]),
                                       ("simt_fuzz_bvh.py", ["--cases", "60", "--seed", "304", "--large", "--odd", "0.5"])])
def test_randomised_search_on_the_gpu_finds_nothing(tool, args):
    r = subprocess.run([sys.executable, os.path.join(REPO, "tools", tool), "--lib", CUDA_LIB] + args, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
    assert r.stdout.strip().endswith("0 findings")


# every switch of the searches (tests/test_fuzz_smoke.py SWITCHES) against the real kernels, with seeds of their own; the session's
# device-form query steps go through torch CUDA tensors
GPU_SWITCHES = [("simt_fuzz.py", ["--cases", "100", "--seed", "311", "--pixel-stats", "--queries", "--occlusion", "--paths"],
                 [r"PixelStats compared in [1-9]\d* cases", r"query batches equal in 100 cases", r"occlusion batches equal in 100 cases", r"path batches equal in 100 cases"]),
                ("simt_fuzz.py", ["--cases", "12", "--seed", "312", "--far", "1.0", "--queries", "--occlusion", "--paths"],
                 [r"query batches equal in 12 cases", r"occlusion batches equal in 12 cases", r"path batches equal in 12 cases"]),
                ("simt_fuzz_session.py", ["--cases", "60", "--seed", "313", "--steps", "6", "--frames", "--pixel-stats", "--queries"],
                 [r"trace_rays [1-9]", r"trace_occlusion [1-9]", r"trace_paths [1-9]", r"manager [1-9]", r"context [1-9]", r"device [1-9]"])]


@pytest.mark.parametrize("tool,args,expect", GPU_SWITCHES)
def test_every_search_switch_on_the_gpu_finds_nothing(tool, args, expect):
    run_switches(tool, args, expect, lib_args=("--lib", CUDA_LIB), timeout=1200)
