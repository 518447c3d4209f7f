"""Semantic likelihood rows of the fuse kernel against the oracle, bit for bit.

fuseKernel keeps each voxel's likelihood row in shared memory as [thread][S], S = the padded row length Lp rounded up to
an odd multiple of 4, and applies a frame's update as one scalar read of the label entry, a 16 B pass adding mle_off to
the whole row, and a scalar store of old + mle_diag into the label entry. Whether a frame has a label image or a dynamic
mask comes from per-batch bit words. These tests cover every rounding of Lp to S (S > Lp included), labels at and beyond
the edges (L-1, L, >= 64, negative, blocked), batches in which only some frames carry a label image or a mask, compact
(u8 label) batches and BINARY mode."""
import ctypes

import numpy as np
import pytest

from khronos_b200 import capi
import harness as hs
from test_parity_gpu import room_frames

pytestmark = pytest.mark.gpu

N_FRAMES = 33  # batch 32: one full batch and a single-frame one; batch 11: three batches
_FRAMES = {}


def scene(cam):
    if "room" not in _FRAMES:
        _FRAMES["room"] = room_frames(cam, N_FRAMES, laps=0.3)
    return _FRAMES["room"]


def map_config(vps):
    if vps == 16:
        return capi.default_map_config(voxel_size=0.05, vps=16, trunc=0.15, max_blocks=16384)
    return capi.default_map_config(voxel_size=0.1, vps=8, trunc=0.3, max_blocks=16384)


def blocked_labels(L):
    """One blocked label inside 0..L-1 and, where the configuration allows it, one beyond L."""
    out = [min(1, L - 1)]
    if L + 1 < 64:
        out.append(L + 1)
    return tuple(out)


def label_images(frames, L, seed):
    """The renderer's labels folded into 0..L-1, with edge values sprinkled in: L-1, L, 64, 100, negative, blocked."""
    rng = np.random.default_rng(seed)
    special = np.array([L - 1, L, 64, 100, -1, -7, *blocked_labels(L)], np.int32)
    out = []
    for _, l in frames:
        lab = (np.abs(l.astype(np.int64)) % L).astype(np.int32)
        pick = rng.random(lab.shape) < 0.15
        lab[pick] = rng.choice(special, size=int(pick.sum()))
        out.append(np.ascontiguousarray(lab))
    return out


def dynamic_masks(cam, n, seed):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        mk = np.zeros((cam.height, cam.width), np.int32)
        mk[30:80, 40:110] = rng.integers(0, 2, size=(50, 70))
        out.append(mk)
    return out


def has_label(i):
    return i % 4 != 1


def has_mask(i):
    return i % 3 == 0


def assert_maps_identical(o, g, what):
    bo, bg = o.export_blocks(), g.export_blocks()
    hs.assert_blocks_equal(bo, bg, exact_float=True, what=what)
    assert bo.semantic_likelihoods is not None and bg.semantic_likelihoods is not None
    np.testing.assert_array_equal(bo.semantic_likelihoods.view(np.uint32), bg.semantic_likelihoods.view(np.uint32),
                                  err_msg=f"{what} likelihood bits")
    assert o.map_checksum() == g.map_checksum(), what
    return bo


@pytest.mark.parametrize("vps", [16, 8])
@pytest.mark.parametrize("L", [2, 3, 4, 5, 8, 16, 20, 21, 24, 33, 64])
def test_mle_rows_bit_identical(oracle_lib, product_lib, L, vps):
    cam = hs.small_camera(4)
    frames, poses, stamps = scene(cam)
    labels = label_images(frames, L, seed=L)
    masks = dynamic_masks(cam, len(frames), seed=100 + L)
    lab = [labels[i] if has_label(i) else None for i in range(len(frames))]
    msk = [masks[i] if has_mask(i) else None for i in range(len(frames))]
    ic = capi.default_integrator_config(num_labels=L, blocked=blocked_labels(L), num_threads=hs.TEST_THREADS)
    o = hs.make_handle(oracle_lib, "ko_", cam=cam, map_cfg=map_config(vps), integ_cfg=ic)
    for i, ((d, _), T, st) in enumerate(zip(frames, poses, stamps)):
        o.integrate_frame(o.make_frame(d, T, st, label=lab[i], mask=msk[i]), want_stats=False)
    for batch in (32, 11):
        g = hs.make_handle(product_lib, "kb_", cam=cam, map_cfg=map_config(vps), integ_cfg=ic)
        for i in range(0, len(frames), batch):
            g.integrate_frames([g.make_frame(frames[j][0], poses[j], stamps[j], label=lab[j], mask=msk[j])
                                for j in range(i, min(i + batch, len(frames)))], want_stats=False)
        bo = assert_maps_identical(o, g, f"L{L} vps{vps} batch{batch}")
    assert (bo.semantic_empty == 0).sum() > 1000  # the semantic path did run


@pytest.mark.parametrize("L", [5, 20])
def test_compact_rows_bit_identical(oracle_lib, product_lib, L):
    """All-compact batches read u8 labels in place: the label flag word then follows label_u8."""
    cam = hs.small_camera(4)
    frames, poses, stamps = scene(cam)
    labels = label_images(frames, L, seed=7 + L)
    d16 = [np.round(d * 1000.0).astype(np.uint16) for d, _ in frames]
    l8 = [(labels[i] & 0xFF).astype(np.uint8) if has_label(i) else None for i in range(len(frames))]
    masks = dynamic_masks(cam, len(frames), seed=3)
    msk = [masks[i] if has_mask(i) else None for i in range(len(frames))]
    ic = capi.default_integrator_config(num_labels=L, blocked=blocked_labels(L), num_threads=hs.TEST_THREADS)
    o = hs.make_handle(oracle_lib, "ko_", cam=cam, map_cfg=map_config(16), integ_cfg=ic)
    g = hs.make_handle(product_lib, "kb_", cam=cam, map_cfg=map_config(16), integ_cfg=ic)
    for i in range(len(frames)):
        o.integrate_frame(o.make_frame(None, poses[i], stamps[i], depth_u16=d16[i], label_u8=l8[i], mask=msk[i]), want_stats=False)
    for i in range(0, len(frames), 11):
        g.integrate_frames([g.make_frame(None, poses[j], stamps[j], depth_u16=d16[j], label_u8=l8[j], mask=msk[j])
                            for j in range(i, min(i + 11, len(frames)))], want_stats=False)
    assert_maps_identical(o, g, f"compact L{L}")


@pytest.mark.parametrize("vps", [16, 8])
def test_binary_rows_bit_identical(oracle_lib, product_lib, vps):
    cam = hs.small_camera(4)
    frames, poses, stamps = scene(cam)
    target = int(np.bincount(np.abs(frames[0][1]).ravel()).argmax())
    obj = [l if has_label(i) else None for i, (_, l) in enumerate(frames)]
    masks = dynamic_masks(cam, len(frames), seed=5)
    msk = [masks[i] if has_mask(i) else None for i in range(len(frames))]
    ic = capi.default_integrator_config(semantic_mode=capi.SEM_BINARY, num_threads=hs.TEST_THREADS)
    o = hs.make_handle(oracle_lib, "ko_", cam=cam, map_cfg=map_config(vps), integ_cfg=ic)
    for i, ((d, _), T, st) in enumerate(zip(frames, poses, stamps)):
        o.integrate_frame(o.make_frame(d, T, st, object_image=obj[i], target_id=target, mask=msk[i]), want_stats=False)
    for batch in (32, 11):
        g = hs.make_handle(product_lib, "kb_", cam=cam, map_cfg=map_config(vps), integ_cfg=ic)
        for i in range(0, len(frames), batch):
            g.integrate_frames([g.make_frame(frames[j][0], poses[j], stamps[j], object_image=obj[j], target_id=target, mask=msk[j])
                                for j in range(i, min(i + batch, len(frames)))], want_stats=False)
        bo = assert_maps_identical(o, g, f"binary vps{vps} batch{batch}")
    assert (bo.semantic_label == 1).sum() > 100  # some voxels did take the target


def test_row_layout_keeps_occupancy(product_lib):
    """Resident fuse CTAs per SM (occupancy API). At L = 20 the padded row stride equals Lp, so the 10 KB of rows per CTA
    and the 10 CTAs/SM the kernel is compiled for (H100) are unchanged; at L = 64 the rows take 34 KB (stride 68) instead of
    32 KB, which still leaves 6 CTAs/SM."""
    fn = product_lib._ZN2kb15fuseBlocksPerSmEii
    fn.argtypes, fn.restype = [ctypes.c_int, ctypes.c_int], ctypes.c_int
    for vps in (16, 8):
        assert fn(vps, 20) == 10, vps
        assert fn(vps, 64) == 6, vps
