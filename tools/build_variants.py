#!/usr/bin/env python
"""Builds the compile-time A/B variants of librt_b200.so HERE (nvcc cross-compiles without a GPU) into ray_tracing_b200/variants/,
so that time on the GPU goes to measuring, not compiling.  The .so files are git-ignored.

    python tools/build_variants.py [name ...]        (no names: all)
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ray_tracing_b200 import build   # noqa: E402

VARIANTS = {
    "r1": ("RT_DEFAULTS_R1",),
    "pushpred": ("RT_PUSH_PREDICATED",),
    "stream": ("RT_STREAM_IMAGES",),
    "cold": ("RT_POOL_COLD_GLOBAL",),
    "cold_ring16": ("RT_POOL_COLD_GLOBAL", "RT_SMEM_STACK=16"),
    "mb7": ("RT_WAVE_MINBLOCKS=7",),
    "mb8": ("RT_WAVE_MINBLOCKS=8",),
    "sphleaf1": ("RT_SPHERE_LEAF=1", "RT_SPHERE_SAH_DEPTH=20"),
    "sphleaf2": ("RT_SPHERE_LEAF=2", "RT_SPHERE_SAH_DEPTH=18"),
    "sphleaf8": ("RT_SPHERE_LEAF=8",),
    "sphsah20": ("RT_SPHERE_SAH_DEPTH=20",),                                   # the round-1 default kernels
    # round 2, third call: on top of the promoted defaults
    "pw28_m32": ("RT_POOL_WARPS=28",),                            # run with poolSlots 32 (28 warps x 64 slots + the stack ring exceed 227 KB)
    "stack4": ("RT_SMEM_STACK=4",),
    "stack16": ("RT_SMEM_STACK=16",),
    "vote274": ("RT_VOTE_WI=2", "RT_VOTE_WL=7", "RT_VOTE_WN=4"),
    "leaf3": ("RT_LEAF_REPEAT=3",),
    "tri64": ("RT_TRI_PAD64",),
    "vote132": ("RT_VOTE_WL=3", "RT_VOTE_WN=2"),
    "vote142": ("RT_VOTE_WL=4", "RT_VOTE_WN=2"),
    "vote274": ("RT_VOTE_WI=2", "RT_VOTE_WL=7", "RT_VOTE_WN=4"),
    "vote163": ("RT_VOTE_WL=6", "RT_VOTE_WN=3"),
    "vote132_pfcur": ("RT_VOTE_WL=3", "RT_VOTE_WN=2", "RT_PREFETCH_CUR"),
    "vote132_pfcur_treelet": ("RT_VOTE_WL=3", "RT_VOTE_WN=2", "RT_PREFETCH_CUR", "RT_TREELET_PREFETCH"),
    "treelet": ("RT_TREELET_PREFETCH",),
    "treelet_stacktop": ("RT_TREELET_PREFETCH", "RT_STACK_TOP_REG"),
    "stacktop": ("RT_STACK_TOP_REG",),
    "tri_na": ("RT_TRI_LOAD_POLICY=1",),
    "tri_ef": ("RT_TRI_LOAD_POLICY=2",),
    "pf": ("RT_PREFETCH_NEXT_PAIR",),
    "pfcur": ("RT_PREFETCH_CUR",),
    "pfcur_ir1": ("RT_PREFETCH_CUR", "RT_INNER_REPEAT=1"),
    "pfcur_treelet": ("RT_PREFETCH_CUR", "RT_TREELET_PREFETCH"),
    "smemstack4": ("RT_SMEM_STACK=4",),
    "smemstack8": ("RT_SMEM_STACK=8",),
    "sphsah": ("RT_SPHERE_SAH_DEPTH=14",),
    "leaf2": ("RT_LEAF_REPEAT=2",),
    "ir1": ("RT_INNER_REPEAT=1",),
    "ir3": ("RT_INNER_REPEAT=3",),
    "rayinv": ("RT_CACHE_RAYINV",),
    "pw20": ("RT_POOL_WARPS=20",),
    "pw16": ("RT_POOL_WARPS=16",),
    "skipsqrt": ("RT_SPHERE_SKIP_SQRT",),
    "zerodefocus": ("RT_SKIP_ZERO_DEFOCUS",),
    "glassool": ("RT_GLASS_OUT_OF_LINE",),
    "cornell_all": ("RT_SKIP_ZERO_DEFOCUS", "RT_GLASS_OUT_OF_LINE", "RT_SPHERE_SKIP_SQRT"),
    "zerodefocus_skipsqrt": ("RT_SKIP_ZERO_DEFOCUS", "RT_SPHERE_SKIP_SQRT"),
    "mb5": ("RT_WAVE_MINBLOCKS=5",),
    # round 2: combinations of the first A/B round's winners on soup4k
    "c1": ("RT_VOTE_WL=3", "RT_VOTE_WN=2", "RT_SMEM_STACK=8"),
    "c2": ("RT_VOTE_WL=3", "RT_VOTE_WN=2", "RT_SMEM_STACK=8", "RT_LEAF_REPEAT=2"),
    "c3": ("RT_VOTE_WL=3", "RT_VOTE_WN=2", "RT_SMEM_STACK=8", "RT_LEAF_REPEAT=2", "RT_SPHERE_SAH_DEPTH=14"),
    "c5": ("RT_VOTE_WI=2", "RT_VOTE_WL=7", "RT_VOTE_WN=4", "RT_SMEM_STACK=8", "RT_LEAF_REPEAT=2", "RT_SPHERE_SAH_DEPTH=14"),
    "c6": ("RT_VOTE_WL=3", "RT_VOTE_WN=2", "RT_SMEM_STACK=16", "RT_LEAF_REPEAT=2", "RT_SPHERE_SAH_DEPTH=14"),
    "c7": ("RT_VOTE_WL=3", "RT_VOTE_WN=2", "RT_STACK_TOP_REG", "RT_LEAF_REPEAT=2", "RT_SPHERE_SAH_DEPTH=14"),
    "smemstack16": ("RT_SMEM_STACK=16",),
    "c8": ("RT_VOTE_WL=3", "RT_VOTE_WN=2", "RT_SMEM_STACK=8", "RT_BRANCHLESS_POP", "RT_LEAF_REPEAT=2", "RT_SPHERE_SAH_DEPTH=14"),
    "pw28": ("RT_POOL_WARPS=28",),
    "pw32": ("RT_POOL_WARPS=32",),
    "pw28_c": ("RT_POOL_WARPS=28", "RT_VOTE_WL=3", "RT_VOTE_WN=2", "RT_LEAF_REPEAT=2", "RT_SPHERE_SAH_DEPTH=14"),
    "pw32_c": ("RT_POOL_WARPS=32", "RT_VOTE_WL=3", "RT_VOTE_WN=2", "RT_LEAF_REPEAT=2", "RT_SPHERE_SAH_DEPTH=14"),
    "all_mesh": ("RT_TREELET_PREFETCH", "RT_STACK_TOP_REG", "RT_TRI_LOAD_POLICY=1", "RT_LEAF_REPEAT=2"),
    # the pooled kernel's cycle account per step kind (tools/pool_clocks.py)
    "clocks": ("RT_POOL_CLOCKS",),
    # rtDenoise with every tap loaded from global memory instead of the shared-memory sub-lattice tile (tools/denoise_bench.py --ab)
    "denoise_plain": ("RT_DENOISE_PLAIN",),
    # rtDenoiseTemporal's variance prefilter over the lattice neighbours at +-s from the staged tile instead of SVGF's immediate
    # neighbours, and its history tolerances (tools/temporal_denoise_bench.py --ab); none of these is bit-exact against the oracle
    "temporal_lattice": ("RT_TEMPORAL_LATTICE_PREFILTER",),
    "temporal_tauz02": ("RT_TEMPORAL_TAU_Z=0.02f",),
    "temporal_tauz10": ("RT_TEMPORAL_TAU_Z=0.1f",),
    "temporal_tauz20": ("RT_TEMPORAL_TAU_Z=0.2f",),
    "temporal_taun80": ("RT_TEMPORAL_TAU_N=0.8f",),
    "temporal_taun95": ("RT_TEMPORAL_TAU_N=0.95f",),
    "temporal_taun50": ("RT_TEMPORAL_TAU_N=0.5f",),
    # rtDispatchAdaptive's absolute floor for dark pixels, 2^-4 and 2^-12 against the default 2^-8 (tools/adaptive_bench.py --sweep)
    "adaptive_eps4": ("RT_ADAPTIVE_EPSILON=0.0625f",),
    "adaptive_eps12": ("RT_ADAPTIVE_EPSILON=0.000244140625f",),
}
OUT_DIR = os.path.join(build.PKG_DIR, "variants")


def path(name: str) -> str:
    return os.path.join(OUT_DIR, f"librt_b200_{name}.so")


if __name__ == "__main__":
    os.makedirs(OUT_DIR, exist_ok=True)
    names = sys.argv[1:] or list(VARIANTS)
    for n in names:
        build.build_cuda(force=True, defines=VARIANTS[n], out=path(n))
    print("built", len(names), "variants in", OUT_DIR)
