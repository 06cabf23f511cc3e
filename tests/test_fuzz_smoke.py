"""The randomised searches of tools/ (simt_fuzz.py: scenes against the oracle; simt_fuzz_session.py: sequences of host calls; simt_fuzz_bvh.py: rtBuildBVH and the host builder against the oracle's recursion) run
for a few dozen cases each, so that the tools keep working and a regression in what they once found shows up in the CPU suite.  The
long campaigns are run by hand (DESIGN.md 3b)."""
import os
import re
import subprocess
import sys

import pytest

from conftest import REPO


@pytest.mark.parametrize("tool,args", [("simt_fuzz.py", ["--cases", "40", "--seed", "1"]),
                                       ("simt_fuzz.py", ["--cases", "4", "--seed", "5", "--far", "1.0"]),
                                       ("simt_fuzz.py", ["--cases", "20", "--seed", "7", "--far", "0", "--odd", "1.0"]),
                                       ("simt_fuzz_session.py", ["--cases", "12", "--seed", "3", "--steps", "6"]),
                                       ("simt_fuzz_bvh.py", ["--cases", "30", "--seed", "11"]),
                                       # 16,383..150,000 triangles: the host builder's multi-threaded path against the oracle's recursion
                                       # (device builds of this size are left to the GPU suite: minutes each on the interpreter)
                                       ("simt_fuzz_bvh.py", ["--cases", "40", "--seed", "12", "--large", "--host-only", "--odd", "0.5"])])
def test_randomised_search_finds_nothing(tool, args):
    r = subprocess.run([sys.executable, os.path.join(REPO, "tools", tool)] + args, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert r.stdout.strip().endswith("0 findings")


# The switches of the searches (queries, occlusion, paths and PixelStats in simt_fuzz.py; frames, PixelStats and query steps in
# simt_fuzz_session.py), with seeds under which every switch is exercised: the last line must report no finding and a positive count
# for each comparison the switch adds (PixelStats only where a launch counts whole images, 3 of the 30 cases here).
SWITCHES = [("simt_fuzz.py", ["--cases", "30", "--seed", "41", "--pixel-stats", "--queries", "--occlusion", "--paths"],
             [r"PixelStats compared in [1-9]\d* cases", r"query batches equal in 30 cases", r"occlusion batches equal in 30 cases", r"path batches equal in 30 cases"]),
            ("simt_fuzz.py", ["--cases", "4", "--seed", "45", "--far", "1.0", "--queries", "--occlusion", "--paths"],
             [r"query batches equal in 4 cases", r"occlusion batches equal in 4 cases", r"path batches equal in 4 cases"]),
            ("simt_fuzz_session.py", ["--cases", "30", "--seed", "46", "--steps", "6", "--frames", "--pixel-stats", "--queries"],
             [r"trace_rays [1-9]", r"trace_occlusion [1-9]", r"trace_paths [1-9]", r"manager [1-9]", r"context [1-9]", r"device [1-9]"])]


def run_switches(tool, args, expect, lib_args=(), timeout=900):
    r = subprocess.run([sys.executable, os.path.join(REPO, "tools", tool)] + list(lib_args) + args, capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    last = r.stdout.strip().splitlines()[-1]
    assert re.match(r"\d+ cases, 0 findings", last), last
    for e in expect:
        assert re.search(e, last), f"{e!r} not in {last!r}"
    print(last)


@pytest.mark.parametrize("tool,args,expect", SWITCHES)
def test_every_search_switch_finds_nothing(tool, args, expect):
    run_switches(tool, args, expect)
