#!/usr/bin/env python
"""Randomised comparison of the BVH builders with the oracle's plain single-threaded restatement of the reference's recursion
(BvhCs::Builder in oracle/rt_oracle.cpp, after BVH.cs:26-318): Nodes and Triangles must be the same bytes.  Every case builds the mesh
with the device build (rtBuildBVH, csrc/rt_bvh_build.cuh, on the SIMT interpreter build or with --lib on the real kernels) and with the
host builder (host/BVH.cpp) at all threads and at 1 thread.  Random meshes with the things a level-synchronous or a multi-threaded
build can get wrong: duplicated and coincident triangles, degenerate ones, exact zeros of both signs, grids (many equal centres ->
equal split costs), tiny and huge coordinates, non-finite vertices, extents whose surface area overflows FP32 (empty leaves),
1..5 triangles, sorted / reversed / shuffled input orders, all three quality modes.  A mesh whose tree needs more than 2n + 1 nodes
must be refused by every builder.

--large draws 16,383 to 150,000 triangles instead of 1 to 9,000, so that the host builder's multi-threaded path (16,384 triangles and
up) meets every class.  --host-only leaves the device build out: a SIMT-interpreted device build of 150,000 triangles takes about a
minute, so the CPU suite runs --large with --host-only and the GPU suite runs --large against the real kernels.  --odd sets the share
of cases with non-finite vertices or overflowing extents (half each).

    python tools/simt_fuzz_bvh.py [--cases 300] [--seed 1] [--large] [--host-only] [--odd 0.12] [--lib librt_b200.so]
"""
import argparse
import os
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests", "simt"))
import build as simt_build                      # noqa: E402
import ray_tracing_b200 as rt                   # noqa: E402
from ray_tracing_b200 import build as rt_build, capi    # noqa: E402


def random_mesh(rng, large=False, odd_share=0.12):
    if large:                                       # both sides of the parallel threshold, and up to 150k triangles
        n = int(rng.choice([16383, 16384, 16385])) if rng.rand() < 0.3 else int(rng.randint(16386, 150001))
    else:
        n = int(rng.choice([1, 2, 3, 5, 17, 64, 300, 2000, 9000]))
    kind = int(rng.randint(0, 7))
    scale = float(rng.choice([1e-4, 1.0, 1.0, 1e4]))
    if kind == 0:                                   # soup
        c = rng.uniform(-1, 1, (n, 1, 3)); tri = c + rng.uniform(-0.05, 0.05, (n, 3, 3))
    elif kind == 1:                                 # regular grid of identical quads' halves: many equal centres and costs
        k = int(np.ceil(np.sqrt(n))); gx, gy = np.meshgrid(np.arange(k), np.arange(k)); g = np.stack([gx.ravel(), gy.ravel(), np.zeros(k * k)], 1)[:n]
        tri = g[:, None, :] + np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], dtype=np.float64)[None]
    elif kind == 2:                                 # every triangle the same
        tri = np.repeat(rng.uniform(-1, 1, (1, 3, 3)), n, axis=0)
    elif kind == 3:                                 # degenerate: points and segments mixed in
        c = rng.uniform(-1, 1, (n, 1, 3)); tri = c + rng.uniform(-0.05, 0.05, (n, 3, 3)); tri[::3, 1] = tri[::3, 0]; tri[::5, 2] = tri[::5, 0]
    elif kind == 4:                                 # exact zeros of both signs, axis-aligned planes
        tri = rng.choice([-1.0, -0.0, 0.0, 1.0, 0.5], (n, 3, 3))
    elif kind == 5:                                 # a line of triangles along one axis (two flat axes)
        tri = np.zeros((n, 3, 3)); tri[:, :, 0] = np.arange(n)[:, None] + rng.uniform(0, 0.9, (n, 3))
    else:                                           # clusters far apart
        c = rng.choice([-100.0, 0.0, 100.0], (n, 1, 3)) + rng.uniform(-1, 1, (n, 1, 3)); tri = c + rng.uniform(-0.2, 0.2, (n, 3, 3))
    tri = tri * scale
    odd = rng.rand()
    if odd < odd_share / 2:                         # non-finite vertices: the reference builds *something*; the device build must build the same
        for _ in range(int(rng.randint(1, 4))):
            tri[int(rng.randint(0, n)), int(rng.randint(0, 3)), int(rng.randint(0, 3))] = rng.choice([np.nan, np.inf, -np.inf])
    elif odd < odd_share:                           # extents whose surface area overflows FP32: every candidate costs inf, the reference
        tri = tri * (1e20 / scale)                  # then splits by "axis 0, position 0" (ChooseSplit's defaults)
    order = int(rng.randint(0, 4))
    if order == 1:
        tri = tri[::-1]
    elif order == 2:
        tri = tri[rng.permutation(n)]
    elif order == 3:
        tri = tri[np.argsort(tri[:, :, int(rng.randint(0, 3))].mean(1), kind="stable")]
    v = np.ascontiguousarray(tri.reshape(-1, 3), dtype=np.float32)
    nrm = np.ascontiguousarray(rng.uniform(-1, 1, v.shape), dtype=np.float32)
    return v, np.arange(3 * n, dtype=np.int32), nrm


def build_all(builders, v, idx, nrm, q):
    """{name: (triangles, nodes), or None where the builder refuses the mesh}"""
    out = {}
    for name, build in builders:
        try:
            out[name] = build(v, idx, nrm, q)
        except (ValueError, capi.RtError):          # more than 2n + 1 nodes (chains of empty children)
            out[name] = None
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", type=int, default=300)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--lib", default=None)
    ap.add_argument("--large", action="store_true", help="16,383 to 150,000 triangles per mesh")
    ap.add_argument("--host-only", action="store_true", help="compare the host builder only, no device build")
    ap.add_argument("--odd", type=float, default=0.12, help="share of meshes with non-finite vertices or overflowing extents")
    args = ap.parse_args()
    orc = capi.RtLib(rt_build.LIB_ORACLE).create(0)
    gpu = None if args.host_only else capi.RtLib(args.lib or simt_build.build()).create(0)

    def host(threads):
        def build(v, idx, nrm, q):
            rt.set_build_threads(threads)
            t, n, _ = rt.build_bvh(v, idx, nrm, q)
            return t, n
        return build

    builders = [("host, all threads", host(0)), ("host, 1 thread", host(1))] + ([("device", gpu.build_bvh)] if gpu else [])
    bad = refused = 0
    for case in range(args.cases):
        seed = args.seed * 100003 + case
        rng = np.random.RandomState(seed)
        v, idx, nrm = random_mesh(rng, args.large, args.odd)
        q = int(rng.choice([1, 1, 0, 2]))
        try:
            ref = orc.build_bvh(v, idx, nrm, q)
        except capi.RtError:
            ref = None
        refused += ref is None
        for name, got in build_all(builders, v, idx, nrm, q).items():
            if ref is None or got is None:
                if (ref is None) != (got is None):
                    bad += 1
                    print(f"case seed {seed}: {len(idx) // 3} triangles, quality {q}: {'the oracle' if ref is None else name} refuses "
                          f"(node capacity), {name if ref is None else 'the oracle'} does not", flush=True)
                continue
            (tg, ng), (to, no) = got, ref
            same_nodes = len(ng) == len(no) and np.array_equal(ng.view(np.uint8), no.view(np.uint8))
            if not (same_nodes and np.array_equal(tg.view(np.uint8), to.view(np.uint8))):
                bad += 1
                where = "node count" if len(ng) != len(no) else ("nodes" if not same_nodes else "triangle order")
                print(f"case seed {seed}: {len(idx) // 3} triangles, quality {q}: {name}: {where} differ from the oracle "
                      f"({len(no)} vs {len(ng)} nodes)", flush=True)
        if (case + 1) % 50 == 0:
            print(f"  {case + 1} cases, {bad} findings", flush=True)
    rt.set_build_threads(0)
    orc.destroy()
    if gpu:
        gpu.destroy()
    print(f"builders: {', '.join(n for n, _ in builders)}; the oracle refused {refused} meshes (node capacity)")
    print(f"{args.cases} cases, {bad} findings")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
