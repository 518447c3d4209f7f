"""The oracle (CPU) and the product (GPU) against the float64 model of K1 and the semantic update (tests/fusion_model.py,
ORACLE_SPEC §2-§6) on real geometry: rotated poses, depth edges, blocked labels, masks, all three interpolators, the
weight options and BINARY semantics. Everything else in the suite compares the product with the oracle bit for bit;
this pins both to the spec's arithmetic within fp32 rounding."""
import numpy as np
import pytest

from khronos_b200 import capi, synthetic as syn
import fusion_model as fm
import harness as hs

U24 = 2.0 ** -24   # fp32 unit roundoff
MAX_EXCLUDED = 0.01


def _frames(scene_frames, poses, stamps, masks=None, object_images=None, target_id=0):
    out = []
    for i, ((d, l), T, st) in enumerate(zip(scene_frames, poses, stamps)):
        out.append({"depth": d, "label": l, "pose": T, "stamp": st, "mask": None if masks is None else masks[i],
                    "object_image": None if object_images is None else object_images[i], "target_id": target_id})
    return out


def compare_to_model(blocks, sel, frames, cam, mc, ic, what, min_voxels=2000, allocate_blocks=True, min_clear=0.9):
    """Compares the exported blocks `sel` (indices into `blocks`) with the model; returns the model's result."""
    m = fm.fuse(blocks.block_index[sel], frames, cam, mc, ic, allocate_blocks=allocate_blocks)
    ex = m["excluded"]
    seen = m["updates"] > 0
    share = ex[seen].mean() if seen.any() else 0.0
    assert share < MAX_EXCLUDED, f"{what}: {share:.4f} of the updated voxels lie within fp32 error of a decision threshold"
    ok = ~ex
    assert int((ok & seen).sum()) >= min_voxels, f"{what}: only {int((ok & seen).sum())} voxels checked"
    got_d, got_w = blocks.distance[sel].astype(np.float64), blocks.weight[sel].astype(np.float64)
    if mc.with_tracking:
        np.testing.assert_array_equal(blocks.last_observed[sel][ok], m["last_observed"][ok], err_msg=f"{what} last_observed")
    upd = ok & seen
    n = m["updates"][upd]
    trunc = float(np.float32(mc.truncation_distance))
    # distance: the fp32 sdf of each frame is off by at most esdf (projection error times the local depth step, plus the
    # rounding of range and z); the fp32 running average adds a few roundings of values <= trunc per update
    tol_d = 2.0 * m["esdf"][upd] + n * 8.0 * U24 * trunc
    err_d = np.abs(got_d[upd] - m["distance"][upd])
    bad = err_d > tol_d
    assert not bad.any(), f"{what}: distance off in {int(bad.sum())} voxels, worst {err_d.max():.3g} (tol {tol_d[np.argmax(err_d)]:.3g})"
    # weight: the model bounds the fp32 error of each frame's weight (weight_error: z's error through 1/z^4, the roundings,
    # the sdf error through the drop-off factor); the running sum rounds once more per update
    err_w = np.abs(got_w[upd] - m["weight"][upd])
    tol_w = n * 2.0 * U24 * np.abs(m["weight"][upd]) + 2.0 * m["weight_error"][upd]
    bad = err_w > tol_w
    assert not bad.any(), f"{what}: weight off in {int(bad.sum())} voxels, worst {err_w.max():.3g} (tol {tol_w[np.argmax(err_w)]:.3g})"
    # the bounds above are worst cases (up to a few 1e-5 on distances next to depth edges); the errors themselves stay
    # inside the north star's 1e-4 for all but the voxels right at a depth edge or at the drop-off's tail, so the
    # tolerances cannot hide a wrong weight or interpolation formula (those move distances by millimetres and weights by
    # tens of per cent). Weights sit closer to it than distances: 30 m from the origin (hall640) z carries an fp32 error
    # of a few 1e-6 m, which 1/z^4 multiplies by four and the drop-off factor divides by (trunc + sdf).
    assert np.quantile(err_d, 0.99) < 1e-5 and np.quantile(err_w / m["weight"][upd], 0.99) < 1e-4, what
    if "likelihoods" in m:
        sem = ok & (m["band_updates"] > 0)
        np.testing.assert_array_equal(blocks.semantic_empty[sel][ok] == 0, m["band_updates"][ok] > 0, err_msg=f"{what} semantic_empty")
        lik_m, lik_g = m["likelihoods"][sem], blocks.semantic_likelihoods[sel][sem].astype(np.float64)
        # fp32 accumulation of one constant per band update: one rounding of a value <= |likelihood| per update
        tol_l = (m["band_updates"][sem][:, None] + 1) * U24 * (np.abs(lik_m) + 1.0) * 2.0
        assert (np.abs(lik_g - lik_m) <= tol_l).all(), f"{what}: likelihoods off"
        top2 = np.sort(lik_m, axis=1)[:, -2:]
        clear = (top2[:, 1] - top2[:, 0]) > 2.0 * tol_l.max(axis=1)
        np.testing.assert_array_equal(blocks.semantic_label[sel][sem][clear], m["semantic_label"][sem][clear], err_msg=f"{what} labels")
        assert clear.mean() > min_clear, what
    return m


def sample_blocks(blocks, k, seed):
    rng = np.random.default_rng(seed)
    return np.sort(rng.choice(blocks.n, size=min(k, blocks.n), replace=False))


def _masks(cam, n, seed):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        mk = np.zeros((cam.height, cam.width), np.int32)
        mk[20:70, 30:90] = rng.integers(0, 3, size=(50, 60))
        out.append(mk)
    return out


def _stream(kind, cam, n):
    if kind == "room":
        scene = syn.room_scene()
        poses, stamps = syn.orbit_trajectory(n, laps=0.3)
    else:
        scene = syn.hall_scene(size=(20.0, 16.0, 6.0))
        poses, stamps = syn.sweep_trajectory(n, size=(20.0, 16.0), margin=4.0, lanes=2, yaw_turns=1.0)
    return hs.render_frames(scene, cam, poses, stamps), poses, stamps


CASES = {
    # name: (scene, interpolation, integrator overrides, masks, blocked labels)
    "room-adaptive-masks-blocked": ("room", capi.INTERP_ADAPTIVE, {}, True, (4, 9)),
    "hall-adaptive": ("hall", capi.INTERP_ADAPTIVE, {}, False, ()),
    "hall-nearest-maxweight": ("hall", capi.INTERP_NEAREST, {"max_weight": 4.0}, False, (3,)),
    "room-bilinear-constweight": ("room", capi.INTERP_BILINEAR, {"use_constant_weight": 1, "max_weight": 30.0}, False, ()),
    "hall-adaptive-nodropoff": ("hall", capi.INTERP_ADAPTIVE, {"use_weight_dropoff": 0}, True, ()),
    "room-nearest-eps": ("room", capi.INTERP_NEAREST, {"weight_dropoff_epsilon": 0.03}, False, (1,)),
}


@pytest.mark.parametrize("case", list(CASES))
def test_oracle_matches_float64_model(oracle_lib, case):
    kind, interp, over, with_masks, blocked = CASES[case]
    cam = hs.small_camera(4)
    frames, poses, stamps = _stream(kind, cam, 16)
    ic = capi.default_integrator_config(interpolation=interp, blocked=blocked, num_threads=hs.TEST_THREADS)
    for k, v in over.items():
        setattr(ic, k, v)
    mc = capi.default_map_config(voxel_size=0.05, vps=16, trunc=0.15, max_blocks=16384)
    masks = _masks(cam, len(frames), 5) if with_masks else None
    o = hs.make_handle(oracle_lib, "ko_", cam=cam, map_cfg=mc, integ_cfg=ic)
    hs.run_fusion(o, frames, poses, stamps, masks=masks)
    b = o.export_blocks()
    sel = sample_blocks(b, 150, 11)
    compare_to_model(b, sel, _frames(frames, poses, stamps, masks), cam, mc, ic, case)


def test_oracle_binary_on_preallocated_box_matches_model(oracle_lib):
    cam = hs.small_camera(4)
    frames, poses, stamps = _stream("room", cam, 12)   # from (8.5, 5, 1.5) towards +x, turning left
    mc = capi.default_map_config(voxel_size=0.04, vps=8, trunc=0.08, with_tracking=False, max_blocks=32768)
    ic = capi.default_integrator_config(semantic_mode=capi.SEM_BINARY, num_threads=hs.TEST_THREADS)
    o = hs.make_handle(oracle_lib, "ko_", cam=cam, map_cfg=mc, integ_cfg=ic)
    bs = 0.04 * 8
    lo, hi = np.floor(np.array([8.5, 3.0, -0.3]) / bs).astype(int), np.floor(np.array([12.0, 8.0, 1.7]) / bs).astype(int)
    o.allocate_box(lo, hi)
    for (d, l), T, st in zip(frames, poses, stamps):
        o.integrate_frame(o.make_frame(d, T, st, object_image=l, target_id=9), allocate_blocks=False, want_stats=False)
    b = o.export_blocks()
    assert b.n == int(np.prod(hi - lo + 1))
    fr = _frames(frames, poses, stamps, object_images=[l for _, l in frames], target_id=9)   # the crate at (9..10.5, 6.5..8.5)
    for f in fr:
        f["label"] = None
    m = compare_to_model(b, np.arange(b.n), fr, cam, mc, ic, "binary box", min_voxels=500, allocate_blocks=False)
    sem = ~m["excluded"] & (m["band_updates"] > 0)
    assert (m["semantic_label"][sem] == 1).sum() > 50   # the target object really is in view


def _tie_frames(cam, n=6):
    """Depth terraces whose steps equal the adaptive threshold exactly (0.25 m, exact in fp32) and a label image that
    changes every column, seen from axis-aligned poses that put voxel centres on the optical axis planes, which project
    onto the exact half-pixel column / row (cx = 31.5, cy = 23.5) where two or four bilinear taps tie: the
    adaptive `<` and interpolateID's lowest-index tie rule decide many voxels here."""
    H, W = cam.height, cam.width
    u = np.arange(W)
    depth = np.broadcast_to(np.where((u // 5) % 2 == 0, 1.5, 1.75).astype(np.float32), (H, W)).copy()
    label = np.broadcast_to((u % 17).astype(np.int32), (H, W)).copy()
    label = (label + (np.arange(H) % 3)[:, None]).astype(np.int32)
    frames, poses, stamps = [], [], []
    for i in range(n):
        T = np.eye(4)
        T[:3, 3] = (0.03125 * (2 * i + 1), 0.03125 * (2 * i + 3), 0.0)   # voxel centres: p_C.x = 0 / p_C.y = 0 exactly
        frames.append((depth, label))
        poses.append(T)
        stamps.append(1_000_000_000 + i * 33_333_333)
    return frames, poses, stamps


@pytest.mark.parametrize("interp", [capi.INTERP_ADAPTIVE, capi.INTERP_BILINEAR])
def test_oracle_threshold_ties_match_model(oracle_lib, interp):
    cam = syn.make_camera(64, 48, 32.0, 32.0, max_range=3.0)   # cx = 31.5: p_C.x = 0 projects to u = 31.5 exactly
    frames, poses, stamps = _tie_frames(cam)
    mc = capi.default_map_config(voxel_size=0.0625, vps=8, trunc=0.1875, max_blocks=16384)
    ic = capi.default_integrator_config(interpolation=interp, num_threads=hs.TEST_THREADS)
    ic.adaptive_max_depth_difference = 0.25
    o = hs.make_handle(oracle_lib, "ko_", cam=cam, map_cfg=mc, integ_cfg=ic)
    hs.run_fusion(o, frames, poses, stamps)
    b = o.export_blocks()
    compare_to_model(b, np.arange(b.n), _frames(frames, poses, stamps), cam, mc, ic, f"ties interp{interp}", min_voxels=1000,
                     min_clear=0.2)   # a new label every column: many voxels see each label once


@pytest.mark.gpu(slow=True)   # about two minutes: deselect with -m "gpu and not gpu(slow=True)"
def test_product_matches_float64_model_hall640(product_lib):
    """The product at the benchmarked shape (hall640, 32-frame calls, culling on) against the model on 200 seeded blocks."""
    from test_bench_shape_parity import _hall_stream, _cfg
    n = 64
    cam, poses, stamps, d, l = _hall_stream(n, start=2400)
    mc, ic = _cfg()
    g = capi.MapHandle(product_lib, "kb_", mc, ic, capi.default_tracking_config(), None)
    g.set_camera(cam)
    for b0 in range(0, n, 32):
        g.integrate_frames([g.make_frame(d[i], poses[i], stamps[i], label=l[i]) for i in range(b0, b0 + 32)], want_stats=False)
    b = g.export_blocks()
    frames = [{"depth": d[i], "label": l[i], "pose": poses[i], "stamp": stamps[i]} for i in range(n)]
    compare_to_model(b, sample_blocks(b, 200, 3), frames, cam, mc, ic, "product hall640")
