"""Fuse-kernel variants, selected by environment variables read in kb_create. Since round 2 KB_PIPELINE, KB_FUSE_ITEM_LIST,
KB_EVERFREE_V2 and KB_MOTION_SPARSE are ON by default (they won the A/B runs), so the rest of the suite runs
them and this file also runs the former defaults (=0); KB_FUSE_MLP and KB_H2D_NARROW_LABELS lost their A/Bs and stay off; KB_FUSE_COOP selects the CTA-cooperative two-phase fuse kernel:
  KB_FUSE_ITEM_LIST=1  items come from compacted heaviest-first lists instead of the dense box range
  KB_PIPELINE=1        the prologue (tile pyramid, K0, K0b) of batch i+1 runs on its own stream while the fuse kernel of
                       batch i is busy; work lists, pyramids and cursors are double-buffered by batch parity
  KB_H2D_NARROW_LABELS=1  host i32 label images with ids in 0..255 cross PCIe as u8 (narrowed by host threads, widened on the device)
  KB_FUSE_MLP=2|4      fuseKernelMlp: the frames of an item are processed in groups whose depth / label taps are issued
                       together (memory-level parallelism); nearest-pixel fallback selected from the four loaded taps
Only the processing order / instruction schedule changes: every result must stay bit-identical to the oracle."""
import os

import numpy as np
import pytest

from khronos_b200 import capi, synthetic as syn
import harness as hs
from test_parity_gpu import room_frames
import test_zzz_long_calls as tlc
from test_zzz_long_calls import hall_oracle  # noqa: F401  (fixture: the oracle's map of the long stream, once per session)

pytestmark = pytest.mark.gpu

# Settings equal to the defaults (KB_PIPELINE=1, KB_FUSE_ITEM_LIST=1, KB_FUSE_COOP=0) are what every other test file runs.
VARIANTS = [{"KB_FUSE_MLP": "2"}, {"KB_FUSE_MLP": "4", "KB_FUSE_ITEM_LIST": "1", "KB_FUSE_CTAS_PER_SM": "3"},
            {"KB_H2D_NARROW_LABELS": "1", "KB_H2D_THREADS": "3"},
            {"KB_PIPELINE": "0", "KB_FUSE_ITEM_LIST": "0"}, {"KB_PIPELINE": "0"}, {"KB_FUSE_ITEM_LIST": "0"},
            {"KB_FUSE_COOP": "1"}, {"KB_FUSE_COOP": "1", "KB_PIPELINE": "0"}]


@pytest.fixture(params=VARIANTS, ids=lambda v: "+".join(f"{k.replace('KB_', '').replace('FUSE_', '')}={x}" for k, x in v.items()))
def variant_env(request):
    os.environ.update(request.param)   # read by kb_create
    yield request.param
    for k in request.param:
        os.environ.pop(k, None)


@pytest.fixture(params=[{}] + VARIANTS + [{"KB_FUSE_CTAS_PER_SM": "1"}],
                ids=lambda v: "+".join(f"{k.replace('KB_', '').replace('FUSE_', '')}={x}" for k, x in v.items()) or "default")
def long_variant_env(request):
    """The defaults, every variant, and one fuse CTA per SM (longer fuse kernels widen the window the prologue overlaps)."""
    os.environ.update(request.param)   # read by kb_create
    yield request.param
    for k in request.param:
        os.environ.pop(k, None)


def batched(g, frames, poses, stamps, batch, masks=None, **kw):
    for i in range(0, len(frames), batch):
        fr = [g.make_frame(d, T, st, label=l, mask=None if masks is None else masks[i + j], **kw)
              for j, ((d, l), T, st) in enumerate(zip(frames[i:i + batch], poses[i:i + batch], stamps[i:i + batch]))]
        g.integrate_frames(fr)


@pytest.mark.parametrize("vps,batch", [(16, 32), (16, 11), (8, 32)])
def test_variant_hall_sweep_is_bit_identical(oracle_lib, product_lib, variant_env, vps, batch):
    cam = hs.small_camera(4)
    scene = syn.hall_scene(size=(20.0, 16.0, 6.0))
    poses, stamps = syn.sweep_trajectory(40, size=(20.0, 16.0), margin=4.0, lanes=2, yaw_turns=1.5)
    frames = hs.render_frames(scene, cam, poses, stamps)
    mc = capi.default_map_config(voxel_size=0.05 if vps == 16 else 0.1, vps=vps, trunc=0.15 if vps == 16 else 0.3, max_blocks=16384)
    o = hs.make_handle(oracle_lib, "ko_", cam=cam, map_cfg=mc)
    g = hs.make_handle(product_lib, "kb_", cam=cam, map_cfg=mc)
    so = hs.run_fusion(o, frames, poses, stamps)
    for i in range(0, len(frames), batch):
        fr = [g.make_frame(d, T, st, label=l) for (d, l), T, st in zip(frames[i:i + batch], poses[i:i + batch], stamps[i:i + batch])]
        s = g.integrate_frames(fr).as_dict()
        want = {k: sum(x[k] for x in so[i:i + batch]) for k in s}
        want["total_blocks"] = so[min(i + batch, len(so)) - 1]["total_blocks"]
        assert s == want, (i, s, want)
    hs.assert_blocks_equal(o.export_blocks(), g.export_blocks(), exact_float=True, what=f"{variant_env} vps{vps} batch{batch}")


@pytest.mark.parametrize("interp", [capi.INTERP_ADAPTIVE, capi.INTERP_NEAREST, capi.INTERP_BILINEAR])
def test_variant_masks_blocked_labels_interpolators_tracking(oracle_lib, product_lib, variant_env, interp):
    cam = hs.small_camera(4)
    frames, poses, stamps = room_frames(cam, 24, laps=0.3)
    rng = np.random.default_rng(4)
    masks = []
    for _ in frames:
        mk = np.zeros((cam.height, cam.width), np.int32)
        mk[20:70, 30:90] = rng.integers(0, 3, size=(50, 60))
        masks.append(mk)
    ic = capi.default_integrator_config(interpolation=interp, blocked=(4, 9), num_threads=4)
    o = hs.make_handle(oracle_lib, "ko_", cam=cam, integ_cfg=ic)
    g = hs.make_handle(product_lib, "kb_", cam=cam, integ_cfg=ic)
    g.set_culling(2)
    hs.run_fusion(o, frames[:12], poses[:12], stamps[:12], masks=masks[:12])
    o.update_tracking(stamps[11])
    hs.run_fusion(o, frames[12:], poses[12:], stamps[12:], masks=masks[12:])
    o.update_tracking(stamps[-1])
    batched(g, frames[:12], poses[:12], stamps[:12], 12, masks=masks[:12])
    g.update_tracking(stamps[11])
    batched(g, frames[12:], poses[12:], stamps[12:], 12, masks=masks[12:])
    g.update_tracking(stamps[-1])
    hs.assert_blocks_equal(o.export_blocks(), g.export_blocks(), exact_float=True, what=f"{variant_env} interp{interp}")


def test_variant_compact_frames_and_binary_extraction_map(oracle_lib, product_lib, variant_env):
    cam = hs.small_camera(4)
    frames, poses, stamps = room_frames(cam, 16, laps=0.2)
    d16 = [np.round(d * 1000.0).astype(np.uint16) for d, _ in frames]
    l8 = [l.astype(np.uint8) for _, l in frames]
    o = hs.make_handle(oracle_lib, "ko_", cam=cam)
    g = hs.make_handle(product_lib, "kb_", cam=cam)
    g.set_culling(2)
    for i in range(16):
        o.integrate_frame(o.make_frame(None, poses[i], stamps[i], depth_u16=d16[i], label_u8=l8[i]), want_stats=False)
    g.integrate_frames([g.make_frame(None, poses[i], stamps[i], depth_u16=d16[i], label_u8=l8[i]) for i in range(16)], want_stats=False)
    hs.assert_blocks_equal(o.export_blocks(), g.export_blocks(), exact_float=True, what=f"{variant_env} compact taps")
    # the extractor's private map: vps 8, binary semantics, no tracking, pre-allocated, 16 frames in one call
    mc = capi.default_map_config(voxel_size=0.04, vps=8, trunc=0.08, with_tracking=False, max_blocks=32768)
    ic = capi.default_integrator_config(semantic_mode=capi.SEM_BINARY)
    o2 = hs.make_handle(oracle_lib, "ko_", cam=cam, map_cfg=mc, integ_cfg=ic)
    g2 = hs.make_handle(product_lib, "kb_", cam=cam, map_cfg=mc, integ_cfg=ic)
    g2.set_culling(2)
    bs = 0.04 * 8
    lo, hi = np.floor(np.array([1.5, 1.5, -0.3]) / bs).astype(int), np.floor(np.array([3.5, 4.0, 1.7]) / bs).astype(int)
    for h in (o2, g2):
        h.allocate_box(lo, hi)
    for (d, l), T, st in zip(frames, poses, stamps):
        o2.integrate_frame(o2.make_frame(d, T, st, object_image=l, target_id=7), allocate_blocks=False, want_stats=False)
    g2.integrate_frames([g2.make_frame(d, T, st, object_image=l, target_id=7) for (d, l), T, st in zip(frames, poses, stamps)],
                        allocate_blocks=False, want_stats=False)
    hs.assert_blocks_equal(o2.export_blocks(), g2.export_blocks(), exact_float=True, what=f"{variant_env} binary vps8")


def test_narrowed_labels_fall_back_for_out_of_range_ids(oracle_lib, product_lib):
    """KB_H2D_NARROW_LABELS: frames whose label ids do not fit 8 bits (negative, >= 256) keep the i32 path, the others are
    narrowed; both kinds in one batch call, host and caller-kept (HOST_ASYNC) buffers."""
    os.environ["KB_H2D_NARROW_LABELS"] = "1"
    try:
        cam = hs.small_camera(4)
        frames, poses, stamps = room_frames(cam, 20, laps=0.3)
        rng = np.random.default_rng(9)
        out = []
        for i, (d, l) in enumerate(frames):
            l = l.copy()
            if i % 3 == 1:
                l[rng.random(l.shape) < 0.01] = rng.choice(np.array([-1, 256, 1000, 70000, -2 ** 31], np.int32))
            out.append((d, l))
        o = hs.make_handle(oracle_lib, "ko_", cam=cam)
        g = hs.make_handle(product_lib, "kb_", cam=cam)
        hs.run_fusion(o, out, poses, stamps)
        for i in range(4):
            g.integrate_frame(g.make_frame(out[i][0], poses[i], stamps[i], label=out[i][1]), want_stats=False)
        g.integrate_frames([g.make_frame(d, T, st, label=l) for (d, l), T, st in zip(out[4:12], poses[4:12], stamps[4:12])], want_stats=False)
        keep = [(np.ascontiguousarray(d), np.ascontiguousarray(l)) for d, l in out[12:]]
        g.integrate_frames([g.make_frame(d, T, st, label=l, memory=capi.MEM_HOST_ASYNC) for (d, l), T, st in zip(keep, poses[12:], stamps[12:])],
                           want_stats=False)
        g.synchronize()
        hs.assert_blocks_equal(o.export_blocks(), g.export_blocks(), exact_float=True, what="narrowed labels")
    finally:
        os.environ.pop("KB_H2D_NARROW_LABELS", None)


@pytest.mark.parametrize("sparse", ["1", "0"])
def test_motion_sparse_table_variant(oracle_lib, product_lib, sparse):
    """KB_MOTION_SPARSE=1: the clustering table is reset slot by slot after each frame instead of wholesale before it; the
    object detector (shared table memory) is interleaved on some frames to exercise the dirty -> full reset transition,
    including frames without seeds right after it."""
    os.environ["KB_MOTION_SPARSE"] = sparse
    try:
        import test_sharded_pipeline as tsp
        from test_object_detection_oracle import OBJECTS
        cam = hs.small_camera(4)
        frames, poses, stamps = tsp.dynamic_scenario(cam, 28)
        mot = capi.default_motion_config(min_cluster_size=5, min_separation_distance=2.0)
        o = hs.make_handle(oracle_lib, "ko_", cam=cam, mot_cfg=mot)
        g = hs.make_handle(product_lib, "kb_", cam=cam, mot_cfg=mot)
        cfg = capi.default_object_detector_config(OBJECTS, use_3d=True, min_cluster_size=10)
        dyn = 0
        for i, ((d, l), T, st) in enumerate(zip(frames, poses, stamps)):
            if i % 5 in (0, 1):  # object detection before the motion stage: leaves its entries in the shared table
                io_, no_ = o.detect_objects(cfg, o.make_frame(d, T, st, label=l))
                ig_, ng_ = g.detect_objects(cfg, g.make_frame(d, T, st, label=l))
                assert no_ == ng_
                np.testing.assert_array_equal(io_, ig_)
            io, so, co = o.spin_once(o.make_frame(d, T, st, label=l))
            ig, sg, cg = g.spin_once(g.make_frame(d, T, st, label=l))
            assert (so, co) == (sg, cg), f"frame {i}"
            np.testing.assert_array_equal(io, ig, err_msg=f"frame {i}")
            assert len(o.get_motion_clusters()) == len(g.get_motion_clusters())
            dyn += int((io > 0).sum())
        assert dyn > 100
        hs.assert_blocks_equal(o.export_blocks(), g.export_blocks(), exact_float=True, what="motion sparse")
    finally:
        os.environ.pop("KB_MOTION_SPARSE", None)


@pytest.mark.parametrize("v2", ["1", "0"])
def test_everfree_v2_variant(oracle_lib, product_lib, v2):
    """KB_EVERFREE_V2=1: vectorised halo fill of the ever-free pass; all three connectivities."""
    os.environ["KB_EVERFREE_V2"] = v2
    try:
        import test_sharded_pipeline as tsp
        cam = hs.small_camera(4)
        frames, poses, stamps = tsp.dynamic_scenario(cam, 24)
        for conn in (6, 18, 26):
            trk = capi.default_tracking_config(num_threads=4)
            trk.neighbor_connectivity = conn
            mot = capi.default_motion_config(min_cluster_size=5, min_separation_distance=2.0, num_threads=4)
            o = hs.make_handle(oracle_lib, "ko_", cam=cam, trk_cfg=trk, mot_cfg=mot)
            g = hs.make_handle(product_lib, "kb_", cam=cam, trk_cfg=trk, mot_cfg=mot)
            for i, ((d, l), T, st) in enumerate(zip(frames, poses, stamps)):
                io, so, co = o.spin_once(o.make_frame(d, T, st, label=l))
                ig, sg, cg = g.spin_once(g.make_frame(d, T, st, label=l))
                assert (so, co) == (sg, cg)
                np.testing.assert_array_equal(io, ig)
            bo = o.export_blocks()
            assert bo.ever_free.sum() > 1000
            hs.assert_blocks_equal(bo, g.export_blocks(), exact_float=True, what=f"everfree v2 conn {conn}")
    finally:
        os.environ.pop("KB_EVERFREE_V2", None)


@pytest.mark.gpu(slow=True)
def test_variant_long_pipelined_call_equals_oracle(product_lib, hall_oracle, long_variant_env):
    """The benchmark's call shape (test_zzz_long_calls: ~1000 hall640 frames in one call on a caller stream, then the
    revisit) under every fuse variant, against the oracle's map computed once for all of them."""
    g, sched = tlc.run_long_calls(product_lib, 19)
    sched.assert_covers()
    tlc.assert_matches_oracle(g, hall_oracle, f"long call {long_variant_env}")
