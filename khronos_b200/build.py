"""Builds the in-tree CUDA product library (sm_90a, H100) and, for tests, the CPU oracle."""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
SOURCES = ["kb_kernels.cu", "kb_motion_device.cu", "kb_objects_device.cu", "kb_tracks_device.cu", "kb_rays.cu", "kb_peer.cu", "kb_mesh.cu", "kb_api.cu", "kb_motion_host.cpp"]
HEADERS = ["kb_device.cuh", "kb_kernels.cuh", "kb_motion_device.cuh", "kb_objects_device.cuh", "kb_tracks_device.cuh", "kb_unionfind.cuh", "kb_mesh.cuh", "kb_mc_tables.h", "kb_motion_host.h", os.path.join(ROOT, "include", "khronos_b200.h")]
LIB = os.path.join(CSRC, "libkhronos_b200.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    # bit-parity with the fp32 reference arithmetic: no FMA contraction on device or host
    "-fmad=false", "-Xcompiler", "-fPIC,-ffp-contract=off,-fno-fast-math", "-shared",
]


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build_product(force=False, verbose=False):
    srcs = [os.path.join(CSRC, s) for s in SOURCES]
    deps = srcs + [h if os.path.isabs(h) else os.path.join(CSRC, h) for h in HEADERS]
    if not force and not _stale(LIB, deps):
        return LIB
    extra = [f"-DKB_FUSE_MIN_BLOCKS={os.environ['KB_FUSE_MIN_BLOCKS']}"] if os.environ.get("KB_FUSE_MIN_BLOCKS") else []
    cmd = ["nvcc"] + NVCC_FLAGS + extra + (["-Xptxas", "-v"] if verbose else []) + ["-o", LIB] + srcs
    print(" ".join(cmd), file=sys.stderr)
    subprocess.check_call(cmd, cwd=CSRC)
    return LIB


# Tuning builds for A/B measurements (never loaded unless KB_PRODUCT_LIB_VARIANT names them): same sources, other -D flags.
VARIANTS = {"mb12": ["-DKB_FUSE_MIN_BLOCKS=12"], "mb8": ["-DKB_FUSE_MIN_BLOCKS=8"]}


def build_variant(name):
    srcs = [os.path.join(CSRC, s) for s in SOURCES]
    out = os.path.join(CSRC, f"libkhronos_b200_{name}.so")
    cmd = ["nvcc"] + NVCC_FLAGS + VARIANTS[name] + ["-o", out] + srcs
    print(" ".join(cmd), file=sys.stderr)
    subprocess.check_call(cmd, cwd=CSRC)
    return out


def build_oracle():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle")])
    return os.path.join(ROOT, "oracle", "liboracle.so")


if __name__ == "__main__":
    build_product(force="--force" in sys.argv, verbose="-v" in sys.argv)
    build_oracle()
    for v in VARIANTS:
        if ("--variant=" + v) in sys.argv:
            build_variant(v)
