#!/usr/bin/env python
"""Counts the SASS instructions of each step kind of the pooled kernel's trace phase (no GPU needed).

    python tools/pool_sass_steps.py [--lib librt_b200.so] [--src rt_kernel_pool.cuh] [--kernel k_raytrace_poolILb0ELb0ELi64E]

Disassembles the kernel with its inline line info (`cuobjdump -xelf` + `nvdisasm -gi`; the library is built with -lineinfo) and
attributes every instruction to the line of `pool_body` it comes from, inlined callees included.  The step kinds are the source
blocks between the marker comments of the trace loop (census, fetch, vote, next model, inner nodes, leaf primitive).  These counts
are static: a block's cold paths (the ring spill, the sphere accelerator, the TLAS walk) are in it.  "inner visit" is the loop
body of one inner-node visit: from the head of the loop that contains the pair record's four LDG.E.128 to its back branch.  `--src` names the
rt_kernel_pool.cuh the library was built from (for a parent build, a copy taken with `git show`)."""
from __future__ import annotations

import argparse
import os
import re
import subprocess
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
SRC_DEFAULT = os.path.join(REPO, "ray_tracing_b200", "csrc", "rt_kernel_pool.cuh")
LIB_DEFAULT = os.path.join(REPO, "ray_tracing_b200", "librt_b200.so")

# (step kind, marker that starts it, marker that ends it): the first source line after pool_body's start containing each text
MARKERS = [
    ("census", "// ---- census:", "// ---- fetch:"),
    ("fetch", "// ---- fetch:", "// ---- vote:"),
    ("vote", "// ---- vote:", "// ---- advance to the next model"),
    ("next", "// ---- advance to the next model", "// ---- inner nodes:"),
    ("inner", "// ---- inner nodes:", "// ---- one leaf triangle:"),
    ("leaf", "// ---- one leaf triangle:", "// ---- counters"),
]
LOC_RE = re.compile(r'"([^"]+)", line (\d+)')
INST_RE = re.compile(r"/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;")
LABEL_RE = re.compile(r"^(\.L_x_\d+):")


def line_ranges(src: str) -> tuple[dict, tuple[int, int]]:
    lines = open(src).read().split("\n")

    def find(text: str, start: int = 0) -> int:
        for i in range(start, len(lines)):
            if text in lines[i]:
                return i + 1
        raise SystemExit(f"marker not found in {src}: {text!r}")

    body0 = find("RT_DI void pool_body(")
    body1 = find("// ---- counters", body0)
    ranges = {}
    for name, a, b in MARKERS:
        la = find(a, body0)
        ranges[name] = (la, find(b, la) - 1)
    return ranges, (body0, body1)


def disassemble(lib: str, kernel: str):
    """Instructions [(text, [(file basename, line), ...])] of the first function whose name contains `kernel`, and its labels
    {label: index of the instruction that follows}."""
    with tempfile.TemporaryDirectory() as d:
        subprocess.run(["cuobjdump", "-xelf", "all", os.path.abspath(lib)], cwd=d, check=True, capture_output=True)
        cubins = [f for f in os.listdir(d) if f.endswith(".cubin")]
        if not cubins:
            raise SystemExit("no cubin in " + lib)
        text = subprocess.run(["nvdisasm", "-gi", os.path.join(d, cubins[0])], check=True, capture_output=True, text=True).stdout
    insts, labels, inside, loc, in_block = [], {}, False, [], False
    for ln in text.split("\n"):
        if ln.startswith(".text."):
            if inside:
                break
            inside = kernel in ln
            continue
        if not inside:
            continue
        s = ln.strip()
        if s.startswith("//## File"):
            # one block of consecutive //## lines is one inline chain, innermost frame first
            frames = [(os.path.basename(f), int(n)) for f, n in LOC_RE.findall(s)]
            loc = (loc + frames) if in_block else frames
            in_block = True
            continue
        in_block = False
        m = LABEL_RE.match(s)
        if m:
            labels[m.group(1)] = len(insts)
            continue
        m = INST_RE.match(s)
        if m:
            insts.append((m.group(2), loc))
    if not insts:
        raise SystemExit(f"kernel {kernel!r} not found in {lib}")
    return insts, labels


def count(lib: str, src: str, kernel: str) -> dict:
    ranges, (b0, b1) = line_ranges(src)
    base = os.path.basename(src)
    insts, labels = disassemble(lib, kernel)
    counts = {k: 0 for k in ranges}
    counts["outside the trace loop"] = 0
    owner = []
    for text, loc in insts:
        body_lines = [n for f, n in loc if f == base and b0 <= n <= b1]
        kind = "outside the trace loop"
        if body_lines:
            n = body_lines[0]
            for k, (a, b) in ranges.items():
                if a <= n <= b:
                    kind = k
                    break
        counts[kind] += 1
        owner.append(kind)
    visit = None
    for i in range(len(insts) - 3):
        if owner[i] == "inner" and all(insts[i + j][0].startswith("LDG.E.128") for j in range(4)):
            for j in range(i + 4, len(insts)):
                m = re.search(r"\bBRA\b.*?(\.L_x_\d+)", insts[j][0])
                if m and labels.get(m.group(1), len(insts)) <= i:
                    visit = j - labels[m.group(1)] + 1          # from the loop head to the back branch
                    break
            break
    counts["total"] = len(insts)
    counts["inner visit (loop head .. back branch)"] = visit
    return counts


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=LIB_DEFAULT)
    ap.add_argument("--src", default=SRC_DEFAULT)
    ap.add_argument("--kernel", default="k_raytrace_poolILb0ELb0ELi64E")
    a = ap.parse_args()
    for k, v in count(a.lib, a.src, a.kernel).items():
        print(f"{k:44s} {v}")
