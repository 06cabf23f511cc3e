"""What nvcc emits for the kernels, checked on the CPU (needs nvcc, no GPU): rt_api.cu compiled to PTX with the product's NVCC_FLAGS.

The arithmetic contract (DESIGN.md section 2) needs every FP32 operation to be a single IEEE operation, round to nearest even,
with subnormals kept.  In PTX that means: no fma (ptxas would keep it fused), no .ftz, no .approx, and an explicit .rn on every f32
mul / add / sub / div / sqrt / rcp — an un-annotated mul.f32 or add.f32 may be contracted into an FMA by ptxas.

saturate1 (fminf(fmaxf(a, 0), 1)) is lowered to max.f32 / min.f32 in most places and to cvt.sat.f32.f32 in a few; both lowerings are
checked against the contract on every input pattern by tests/test_gpu_arith_contract.py.  The set of functions that use cvt.sat is
pinned here: a change means a lowering changed and those results must be read again."""
import os
import re
import shutil
import subprocess

import pytest

from conftest import REPO
from ray_tracing_b200 import build as product_build

NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
CVT_SAT_FUNCTIONS = {"rtd::k_display", "rtd::GetEnvironmentLight"}     # DisplayEncode's clamp; the two smoothstep clamps of the sky


@pytest.fixture(scope="module")
def ptx(tmp_path_factory):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc is not installed")
    out = str(tmp_path_factory.mktemp("ptx") / "rt_api.ptx")
    flags = [f for f in product_build.NVCC_FLAGS if f not in ("-shared", "-Xlinker", "-Bsymbolic")]
    r = subprocess.run([NVCC] + flags + ["-ptx", "-I", os.path.join(REPO, "include"), "-o", out,
                        os.path.join(REPO, "ray_tracing_b200", "csrc", "rt_api.cu")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return open(out).read()


def _functions(text):
    """{mangled name: body} of every .entry / .func of a PTX module."""
    out, name = {}, None
    for line in text.splitlines():
        m = re.match(r"\s*(?:\.visible\s+|\.weak\s+|\.extern\s+)*\.(?:entry|func)\s+(?:\([^)]*\)\s*)?([\w$]+)", line)
        if m:
            name = m.group(1)
            out[name] = []
        elif name:
            out[name].append(line)
    return {k: "\n".join(v) for k, v in out.items()}


def test_no_contraction_flush_or_approximation(ptx):
    body = re.sub(r"//.*", "", ptx)
    assert not re.search(r"\bfma\.\w*\.?f32", body), "an FP32 fma in the PTX"
    assert ".ftz" not in body, "a flush-to-zero FP32 instruction in the PTX"
    assert ".approx" not in body, "an approximate FP32 instruction in the PTX"


def test_every_f32_arithmetic_instruction_is_round_to_nearest(ptx):
    ops = re.findall(r"^\s*(?:@!?%p\d+\s+)?((?:mul|add|sub|div|sqrt|rcp)(?:\.\w+)*\.f32)\b", ptx, flags=re.M)
    assert len(ops) > 1000
    bad = sorted({op for op in ops if ".rn." not in op})
    assert not bad, f"FP32 instructions without .rn (ptxas may contract or approximate them): {bad}"


def test_cvt_sat_appears_only_in_the_pinned_functions(ptx):
    funcs = _functions(ptx)
    users = [name for name, body in funcs.items() if "cvt.sat.f32.f32" in body]
    demangled = subprocess.run(["c++filt"], input="\n".join(users), capture_output=True, text=True).stdout.split("\n")[:len(users)]
    got = {re.sub(r"\(.*\)$", "", d) for d in demangled}
    assert got == CVT_SAT_FUNCTIONS, f"cvt.sat.f32.f32 now in {sorted(got)}; pinned {sorted(CVT_SAT_FUNCTIONS)}"
