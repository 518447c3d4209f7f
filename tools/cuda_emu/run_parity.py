#!/usr/bin/env python
"""TEST TOOLING — NOT PRODUCT CODE. Runs the GPU parity tests (pytest -m gpu) against the CUDA-on-CPU build of the
product's own kernel sources (tools/cuda_emu/build_emu.py) instead of the real library, so kernel *logic* can be
checked against the oracle in a container without a GPU:

    python tools/cuda_emu/run_parity.py [pytest args / test files ...]
    KB_EMU_ORDER=reverse|shuffle [KB_EMU_SEED=n] ...            other thread schedules (see emu_runtime.cpp)
    KB_EMU_ASAN=1 LD_PRELOAD=$(g++ -print-file-name=libasan.so) ASAN_OPTIONS=detect_leaks=0:detect_stack_use_after_return=0 ...
                                                                 AddressSanitizer build: a memcheck of every kernel access

What this proves: the arithmetic, indexing, hashing, work distribution and synchronisation structure of the kernels
give the oracle's results when executed with CUDA's thread / warp / block semantics (one fiber per CUDA thread).
What it cannot prove: anything about real concurrency (races between warps or blocks), memory spaces, sm_90a code
generation or speed — the -m gpu run on an H100 remains the parity check. The emulated library is never shipped and
the product package never loads it (khronos_b200.lib() is monkeypatched in this process only)."""
import ctypes
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, HERE)


def main(argv):
    import build_emu
    lib = ctypes.CDLL(build_emu.build())
    import pytest
    import torch
    import khronos_b200 as kb
    from khronos_b200 import distributed as kd
    kb._LIB = lib                                    # khronos_b200.lib() -> the emulated library, this process only
    torch.set_num_threads(1)
    # "device" memory is host memory here: device tensors / pinned tensors of the tests become plain CPU tensors
    torch.Tensor.cuda = lambda self, *a, **k: self
    torch.Tensor.pin_memory = lambda self, *a, **k: self
    torch.cuda.synchronize = lambda *a, **k: None
    orig = kd.ShardedActiveWindow.__init__
    kd.ShardedActiveWindow.__init__ = lambda self, handles, comm, device="cpu": orig(self, handles, comm, device="cpu")
    orig_p, orig_l = kd.PeerShardedActiveWindow.__init__, kd.LocalPeers.__init__
    kd.PeerShardedActiveWindow.__init__ = lambda self, handles, peers, device="cpu": orig_p(self, handles, peers, device="cpu")
    kd.LocalPeers.__init__ = lambda self, n_shards, device="cpu": orig_l(self, n_shards, "cpu")
    args = list(argv) or [os.path.join(ROOT, "tests")]
    # tests that need a real device or a second process group are out of reach of the emulation
    deselect = ["-k", "not adaptor and not two_gpu"]
    return pytest.main(["-m", "gpu", "-q", "-p", "no:cacheprovider", "--tb=short"] + deselect + args)


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
