"""The product's object detectors (kb_detect_objects 2D / 3D, kb_forward_instances) against the from-spec model
(object_model.py) and the oracle on the constructed frames of test_object_model.py; host, pinned, device and compact
inputs; both detectors and both modes on one handle, across a change of camera. Images, ids, semantic ids, counts,
pixel lists and box bits must be identical."""
import ctypes as C

import numpy as np
import pytest

from khronos_b200 import capi
import object_model as om
import test_object_model as tm

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", list(tm.DETECTOR_FRAMES))
def test_product_detect_objects_matches_model(oracle_lib, product_lib, name):
    fr, configs = tm.DETECTOR_FRAMES[name]()
    g = tm.handle(product_lib, "kb_", fr["cam"])
    o = tm.handle(oracle_lib, "ko_", fr["cam"])
    for c, check in configs:
        want = tm.model_detect(fr, c)
        assert check(want), f"{name} {c}: the frame does not produce its case"
        tm.assert_same_objects(want, tm.detect(g, fr, c), f"{name} {c} product")
        tm.assert_same_objects(want, tm.detect(o, fr, c), f"{name} {c} oracle")


@pytest.mark.parametrize("name", list(tm.INSTANCE_FRAMES))
def test_product_forward_instances_matches_model(oracle_lib, product_lib, name):
    fr, configs = tm.INSTANCE_FRAMES[name]()
    g = tm.handle(product_lib, "kb_", fr["cam"])
    o = tm.handle(oracle_lib, "ko_", fr["cam"])
    for kw, check in configs:
        want = tm.model_forward(fr, kw)
        assert check(want), f"{name} {kw}: the frame does not produce its case"
        tm.assert_same_instances(want, tm.forward(g, fr, kw), f"{name} {kw} product")
        tm.assert_same_instances(want, tm.forward(o, fr, kw), f"{name} {kw} oracle")


def test_product_rejects_out_of_range_instance_ids_then_recovers(product_lib):
    fr, _ = tm.i_ids_and_boxes()
    g = tm.handle(product_lib, "kb_", fr["cam"])
    for bad in (-1, 4096):
        lab = fr["label"].copy()
        lab[7, 9] = bad
        with pytest.raises(capi.KbError) as e:
            tm.forward(g, dict(fr, label=lab), {})
        assert e.value.status == capi.KB_ERR_INVALID
        tm.assert_same_instances(tm.model_forward(fr, {}), tm.forward(g, fr, {}), f"after rejecting {bad}")


def compact(fr, instance_ids, scale=0.25):
    """The frame with depth in u16 steps of `scale` and labels in u8, and its float / int32 equivalent (no vertex map:
    the detectors back-project the expanded depth)."""
    rng = np.random.default_rng(0)
    H, W = fr["label"].shape
    d16 = rng.integers(0, 12, (H, W)).astype(np.uint16)
    if instance_ids:
        l8 = (fr["label"] % 251).astype(np.uint8)
    else:
        l8 = np.where(np.isin(fr["label"], tm.OBJ), fr["label"], 0).astype(np.uint8)
        l8[rng.random((H, W)) < 0.05] = 200
    full = dict(fr, depth=d16.astype(np.float32) * np.float32(scale), label=l8.astype(np.int32), vertex=None)
    return d16, l8, full


def memory_kinds(torch, fr):
    """(name, make_frame kwargs) for host, pinned (synchronous and async) and device copies of one frame."""
    out = [("host", {})]
    pin = {k: torch.from_numpy(np.ascontiguousarray(fr[k])).pin_memory() for k in ("depth", "label", "vertex") if fr[k] is not None}
    dev = {k: v.cuda() for k, v in pin.items()}
    torch.cuda.synchronize()
    for name, bufs, mem in (("pinned", pin, capi.MEM_HOST), ("pinned_async", pin, capi.MEM_HOST_ASYNC), ("device", dev, capi.MEM_DEVICE)):
        out.append((name, dict(bufs=bufs, memory=mem)))
    return out


def frame_in(h, fr, bufs=None, memory=capi.MEM_HOST, **kw):
    if bufs is None:
        return tm.make_frame(h, fr, memory=memory, **kw)
    return h.make_frame(bufs["depth"], fr["pose"], 1_000_000_000, label=bufs["label"], vertex_world=bufs.get("vertex"), memory=memory)


@pytest.mark.parametrize("which", ["detect_2d", "detect_3d", "forward"])
def test_input_memory_and_compact_formats(product_lib, which):
    import torch
    fr = tm.f_faces_and_zeros()[0] if which != "forward" else tm.i_ids_and_boxes()[0]
    g = tm.handle(product_lib, "kb_", fr["cam"])
    c = tm.cfg3d(True) if which == "detect_3d" else tm.cfg2d(True)

    def run(f, ref):
        if which == "forward":
            img, cl = g.forward_instances(f, min_cluster_size=2)
            got = dict(image=img, ids=np.array([x["id"] for x in cl], np.int32), counts=np.array([len(x["pixels"]) for x in cl], np.int32),
                       pixels=np.concatenate([x["pixels"] for x in cl]), bbox=np.array([x["bbox"] for x in cl], np.float32))
            g.synchronize()
            tm.assert_same_instances(tm.model_forward(ref, dict(min_cluster_size=2)), got, which)
        else:
            img, n = g.detect_objects(tm.detector_config(c), f)
            got = tm.object_clusters(g)
            got["image"] = img
            g.synchronize()
            tm.assert_same_objects(tm.model_detect(ref, c), got, which)

    for name, kw in memory_kinds(torch, fr):
        run(frame_in(g, fr, **kw), fr)
    d16, l8, full = compact(fr, which == "forward")
    pd, pl = torch.from_numpy(d16).pin_memory(), torch.from_numpy(l8).pin_memory()
    dd, dl = pd.cuda(), pl.cuda()
    torch.cuda.synchronize()
    for mem, (a, b) in ((capi.MEM_HOST, (d16, l8)), (capi.MEM_HOST_ASYNC, (pd, pl)), (capi.MEM_DEVICE, (dd, dl))):
        run(g.make_frame(None, fr["pose"], 1_000_000_000, memory=mem, depth_u16=a, label_u8=b, depth_u16_scale=0.25), full)


def test_modes_alternate_on_one_handle_across_a_camera_change(product_lib):
    small = tm.f_exact_min_size()[0]
    specks = tm.f_many_specks()[0]
    big_ids = tm.i_full_frame()[0]
    small_ids = tm.i_thresholds()[0]
    g = tm.handle(product_lib, "kb_", small["cam"])
    steps = [(small, "2d"), (small, "3d"), (small_ids, "fwd"), (small, "2d"), (specks, "3d"), (specks, "2d"), (big_ids, "fwd"),
             (specks, "3d"), (small_ids, "fwd"), (small, "3d")]
    for i, (fr, kind) in enumerate(steps):
        g.set_camera(fr["cam"])
        if kind == "fwd":
            tm.assert_same_instances(tm.model_forward(fr, dict(min_cluster_size=3)), tm.forward(g, fr, dict(min_cluster_size=3)), f"step {i}")
        else:
            c = tm.cfg3d(True, min_size=20) if kind == "3d" else tm.cfg2d(False, min_size=1)
            tm.assert_same_objects(tm.model_detect(fr, c), tm.detect(g, fr, c), f"step {i} {kind}")


def instance_clusters_guarded(h, n_pixels_bound):
    """kb_get_instance_clusters into buffers far larger than the reported totals, each followed by a sentinel tail;
    the tails must stay intact."""
    f = h._fn("get_instance_clusters")
    n, tp = C.c_int32(0), C.c_int32(0)
    h._check(f(h._h, None, None, None, C.byref(n), C.byref(tp)))
    pad = 4096
    info = np.full(2 * (om.MAX_INSTANCE_IDS + pad), -7, np.int32)
    bbox = np.full(6 * (om.MAX_INSTANCE_IDS + pad), -7, np.float32)
    px = np.full(2 * (2 * n_pixels_bound + pad), -7, np.int32)
    h._check(f(h._h, C.c_void_p(info.ctypes.data), C.c_void_p(bbox.ctypes.data), C.c_void_p(px.ctypes.data), C.byref(n), C.byref(tp)))
    nc, t = n.value, tp.value
    assert (info[2 * nc:] == -7).all(), "cluster table written past its reported size"
    assert (bbox[6 * nc:].view(np.int32) == np.float32(-7).view(np.int32)).all(), "boxes written past their reported size"
    assert (px[2 * t:] == -7).all(), "pixel list written past its reported size"
    info = info[:2 * nc].reshape(-1, 2)
    return dict(ids=info[:, 0], counts=info[:, 1], pixels=px[:2 * t].reshape(-1, 2), bbox=bbox[:6 * nc].reshape(-1, 6))


def assert_instances_only(want, got, what):
    for k in ("ids", "counts", "pixels"):
        np.testing.assert_array_equal(got[k], want[k], err_msg=f"{what}: {k}")
    np.testing.assert_array_equal(got["bbox"].view(np.uint32), want["bbox"].view(np.uint32), err_msg=f"{what}: box bits")


def cross_frames():
    """A: 2D objects; B: instance ids whose pixels land on other ids than A's labels would give them."""
    H, W = 48, 64
    rng = np.random.default_rng(17)
    a = tm.f_random(W, H, 99, density=0.9)
    ids = rng.integers(0, 3000, (H, W)).astype(np.int32)
    ids[:, ::2] = 7                                   # a large cluster under labels that are small clusters in A
    b = tm.frame(W, H, ids, vertex=tm.instance_vertex(H, W, rng))
    return a, b


@pytest.mark.parametrize("mode", ["2d", "3d"])
def test_each_detector_keeps_its_own_result(product_lib, mode):
    a, b = cross_frames()
    c = tm.cfg2d(True) if mode == "2d" else tm.cfg3d(True, grid=1.0)
    a = dict(a, vertex=tm.instance_vertex(*a["label"].shape, np.random.default_rng(3)))
    want_a, want_b = tm.model_detect(a, c), tm.model_forward(b, {})
    g = tm.handle(product_lib, "kb_", a["cam"])
    # detect(A); forward(B); both getters
    tm.detect(g, a, c)
    tm.forward(g, b, {})
    got = tm.object_clusters(g)
    for k in ("ids", "semantic", "counts", "pixels"):
        np.testing.assert_array_equal(got[k], want_a[k], err_msg=f"object clusters after forward_instances: {k}")
    assert_instances_only(want_b, instance_clusters_guarded(g, b["label"].size), "instance clusters")
    # forward(B); detect(A); both getters
    tm.forward(g, b, {})
    tm.detect(g, a, c)
    assert_instances_only(want_b, instance_clusters_guarded(g, b["label"].size), "instance clusters after detect_objects")
    got = tm.object_clusters(g)
    for k in ("ids", "semantic", "counts", "pixels"):
        np.testing.assert_array_equal(got[k], want_a[k], err_msg=f"object clusters: {k}")


def test_getters_describe_the_image_they_came_from(product_lib):
    """The cluster getters after a set_camera to a larger image still return the last results, in their own pixels."""
    a, b = cross_frames()
    g = tm.handle(product_lib, "kb_", a["cam"])
    c = tm.cfg2d(False)
    want_a, want_b = tm.model_detect(a, c), tm.model_forward(b, {})
    tm.forward(g, b, {})
    tm.detect(g, a, c)
    g.set_camera(tm.camera(640, 480))
    assert_instances_only(want_b, instance_clusters_guarded(g, b["label"].size), "instance clusters after set_camera")
    got = tm.object_clusters(g)
    for k in ("ids", "semantic", "counts", "pixels"):
        np.testing.assert_array_equal(got[k], want_a[k], err_msg=f"object clusters after set_camera: {k}")
