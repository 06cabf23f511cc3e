"""The primitive-level arithmetic tests of tests/test_gpu_arith_contract.py on the CPU: the same probe source (tests/gpu_probe/rt_probe.cu)
compiled by g++ against the SIMT interpreter of tests/simt, over every 4,096th input pattern (at an odd offset, so mantissas are not
round) plus the full special-value sets, and 10^5 cases per primitive.  The arithmetic is the same by contract (-ffp-contract=off
here, -fmad=false there), so this proves the harness and catches a slip in the shared device source without a GPU; what nvcc makes
of that source is what the GPU run and tests/test_ptx_contract.py check."""
import pytest

import test_gpu_arith_contract as G

for _name in sorted(dir(G)):
    if _name.startswith("test_"):
        globals()["test_simt_" + _name[5:]] = getattr(G, _name)


@pytest.fixture(scope="module")
def libs():
    return G.P.Lib(G.probe_build.build_simt(), oracle=False), G.P.Lib(G.ORACLE_LIB, oracle=True)


@pytest.fixture(scope="module")
def scale():
    return dict(start=0x9E5, stride=4096, chunk=1 << 20, cases=10 ** 5, batch=10 ** 5, states=10 ** 5, pairs=10 ** 5)
