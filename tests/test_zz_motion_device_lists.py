"""Motion clustering of frames that carry a caller vertex map stays on the device (min_separation_distance > 0), and
kb_get_motion_clusters builds the cluster lists there: which kernels and copies run, the lists, images and boxes
against tests/temporal_model.py and the oracle, the calls that may come between a detection and its list request, more
than 254 clusters, and the boxes of vertices at exactly -0 and +0."""
import json

import numpy as np
import pytest

from khronos_b200 import capi
import harness as hs
import temporal_model as tm
import test_temporal_model as ttm
import test_zz_temporal_model as zt

pytestmark = pytest.mark.gpu


def handles(oracle_lib, product_lib, sep, conn=26, sparse="1", cam=None):
    mot = capi.default_motion_config(num_threads=hs.TEST_THREADS, connectivity=conn, min_separation_distance=sep)
    o, mc, _, st = ttm.warm_handle(oracle_lib, "ko_", mot, cam=cam)
    with zt._env(KB_MOTION_SPARSE=sparse):
        g = ttm.warm_handle(product_lib, "kb_", mot, cam=cam)[0]
    return o, g, mot, mc, st


def model(o, depth, vertex, mot, mc, cam):
    return tm.detect_motion(depth, vertex, np.eye(4), cam, ttm.model_blocks(o), mot, mc.voxel_size, mc.voxels_per_side)


def gpu_trace(tmp_path, fn):
    """Runs fn under torch.profiler with CUDA activities; returns (kernel names, device-to-host copy sizes in bytes)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    path = tmp_path / "trace.json"
    prof.export_chrome_trace(str(path))
    events = json.loads(path.read_text())["traceEvents"]
    kernels = [e["name"] for e in events if e.get("cat") == "kernel"]
    d2h = [int(e["args"].get("bytes", 0)) for e in events
           if e.get("cat") == "gpu_memcpy" and "DtoH" in e["name"].replace(" ", "")]
    return kernels, d2h


def test_vertex_map_frames_take_the_device_path(oracle_lib, product_lib, tmp_path):
    """sep > 0: detect_motion + get_motion_clusters on a vertex-map frame launch the clustering and list kernels and never
    copy the per-pixel voxel keys (12 B per pixel) to the host. sep = 0 still clusters on the host, which copies them."""
    cam = ttm.motion_camera()
    key_bytes = 12 * cam.width * cam.height
    for sep in (2.5, 0.0):
        o, g, mot, mc, st = handles(oracle_lib, product_lib, sep)
        d, vx = ttm.border_vertex_map(cam, mc)
        want = model(o, d, vx, mot, mc, cam)
        got = {}

        def run():
            got["det"] = g.detect_motion(g.make_frame(d, np.eye(4), st, vertex_world=vx))
            got["lists"] = g.get_motion_clusters()

        kernels, d2h = gpu_trace(tmp_path, run)
        np.testing.assert_array_equal(got["det"][0], want[1])
        tm.assert_clusters_equal(got["lists"], want[2], f"sep {sep}")
        assert len(want[2]) > 0
        if sep > 0:
            for name in ("vtLinkKernel", "vtWriteImageKernel", "lsVoxelKernel", "lsPixelKernel"):
                assert any(name in k for k in kernels), (name, sorted(set(kernels)))
            assert key_bytes not in d2h, d2h
        else:
            assert not any("lsPixelKernel" in k for k in kernels)
            assert key_bytes in d2h, d2h


def frame_with_label(h, kind, depth, st, vertex, label):
    """zt.make_frames with a label image (kb_spin_once integrates the frame)."""
    if kind == "host":
        return h.make_frame(depth, np.eye(4), st, label=label, vertex_world=vertex), None
    import torch
    if kind == "pinned":
        bufs = [torch.from_numpy(np.ascontiguousarray(a)).pin_memory() for a in (depth, label, vertex)]
        mem = capi.MEM_HOST_ASYNC
    else:
        bufs = [zt.to_device(a) for a in (depth, label, vertex)]
        mem = capi.MEM_DEVICE
    return h.make_frame(bufs[0], np.eye(4), st, label=bufs[1], vertex_world=bufs[2], memory=mem), bufs


@pytest.mark.parametrize("sparse", ["1", "0"])
@pytest.mark.parametrize("kind", ["host", "pinned", "device"])
def test_detect_and_spin_once_with_vertex_maps_match_model_and_oracle(oracle_lib, product_lib, kind, sparse):
    """Boxes come from the vertex map, not from the depth (the depth back-projection gives other boxes here); kb_spin_once
    with a vertex map gives the model's image, counts and lists and the oracle's map bit for bit."""
    cam = ttm.motion_camera()
    for conn, sep in ((6, 2.5), (26, 1.0)):
        o, g, mot, mc, st = handles(oracle_lib, product_lib, sep, conn=conn, sparse=sparse)
        d, vx = ttm.border_vertex_map(cam, mc)
        want = model(o, d, vx, mot, mc, cam)
        from_depth = model(o, d, None, mot, mc, cam)
        assert any(a[2].tobytes() != b[2].tobytes() for a, b in zip(want[2], from_depth[2])) or len(want[2]) != len(from_depth[2])
        f, keep = zt.make_frames(g, kind, d, np.eye(4), st, vx)
        img, ns, nc = g.detect_motion(f)
        assert (ns, nc) == (want[0], len(want[2])) and nc > 0
        np.testing.assert_array_equal(img, want[1])
        tm.assert_clusters_equal(g.get_motion_clusters(), want[2], f"detect {kind} conn {conn} sep {sep}")
        l = np.full(d.shape, 3, np.int32)
        img_o, ns_o, nc_o = o.spin_once(o.make_frame(d, np.eye(4), st, label=l, vertex_world=vx))
        f, keep2 = frame_with_label(g, kind, d, st, vx, l)
        img_s, ns_s, nc_s = g.spin_once(f)
        assert (ns_s, nc_s) == (ns_o, nc_o) == (want[0], len(want[2]))
        np.testing.assert_array_equal(img_s, want[1])
        tm.assert_clusters_equal(g.get_motion_clusters(), want[2], f"spin_once {kind} conn {conn} sep {sep}")
        tm.assert_clusters_equal(o.get_motion_clusters(), want[2], f"oracle conn {conn} sep {sep}")
        hs.assert_blocks_equal(o.export_blocks(), g.export_blocks(), exact_float=True, what=f"spin_once {kind} conn {conn} sep {sep}")
        del keep, keep2


def test_lists_belong_to_the_last_detection(oracle_lib, product_lib):
    """detect_motion on frame A (device depth and vertex map), then the caller overwrites its buffers and object detection
    and track measurements run on frame B: the lists still are A's, and two list calls in a row agree."""
    import torch
    cam = ttm.motion_camera()
    o, g, mot, mc, st = handles(oracle_lib, product_lib, 2.5)
    d, vx = ttm.border_vertex_map(cam, mc)
    want = model(o, d, vx, mot, mc, cam)
    dd, vv = zt.to_device(d), zt.to_device(vx)
    img, ns, nc = g.detect_motion(g.make_frame(dd.data_ptr(), np.eye(4), st, vertex_world=vv.data_ptr(), memory=capi.MEM_DEVICE))
    assert nc == len(want[2]) > 0
    dd.fill_(1.5)
    vv.fill_(-7.0)
    torch.cuda.synchronize()
    mov = ttm.movers_frame(cam)
    vb = tm.vertex_map(mov, np.eye(4), cam) + np.float32(0.25)
    lb = np.full(mov.shape, 3, np.int32)
    fb = g.make_frame(mov, np.eye(4), st, label=lb, vertex_world=np.ascontiguousarray(vb))
    obj, n_obj = g.detect_objects(capi.default_object_detector_config((3,), use_3d=True), fb)
    g.track_measurements(fb, obj, max(n_obj, 1), mc.voxel_size)
    first = g.get_motion_clusters()
    tm.assert_clusters_equal(first, want[2], "after object detection and track measurements")
    second = g.get_motion_clusters()
    tm.assert_clusters_equal(second, want[2], "second call")
    for a, b in zip(first, second):
        np.testing.assert_array_equal(a["pixels"], b["pixels"])


def test_more_than_254_clusters_with_a_vertex_map(oracle_lib, product_lib):
    """The dust frame with a vertex map that is not the depth's back-projection: lists stay per cluster past the
    saturated image id 255."""
    cam = zt.overflow_camera()
    o, g, mot, mc, st = handles(oracle_lib, product_lib, 1.0, cam=cam)
    d = zt.overflow_dust(cam)
    vx = np.ascontiguousarray(tm.vertex_map(d, np.eye(4), cam) + np.array([0.0, 0.0, -0.01], np.float32))
    want = model(o, d, vx, mot, mc, cam)
    assert len(want[2]) > 254
    img, ns, nc = g.detect_motion(g.make_frame(d, np.eye(4), st, vertex_world=vx))
    assert (ns, nc) == (want[0], len(want[2]))
    np.testing.assert_array_equal(img, want[1])
    tm.assert_clusters_equal(g.get_motion_clusters(), want[2], "over 254 clusters")


def total_order_box(points):
    """IEEE 754-2019 minimum / maximum per axis: -0 counts as below +0."""
    bits = np.ascontiguousarray(points, np.float32).view(np.uint32)
    key = np.where(bits & 0x80000000, ~bits, bits | 0x80000000).astype(np.uint32)
    lo, hi = key.min(0), key.max(0)
    back = lambda k: np.where(k & 0x80000000, k & 0x7FFFFFFF, ~k).astype(np.uint32).view(np.float32)
    return np.concatenate([back(lo), back(hi)])


def test_box_orders_signed_zeros(oracle_lib, product_lib):
    """A mover whose vertices all have x = -0 or +0: the box's x range is [-0, +0] whatever order the pixels come in."""
    cam = ttm.motion_camera()
    o, g, mot, mc, st = handles(oracle_lib, product_lib, 2.0)
    d = np.full((cam.height, cam.width), ttm.WALL, np.float32)
    d[30:40, 42:54] = 2.05
    vx = tm.vertex_map(d, np.eye(4), cam)
    sel = d == np.float32(2.05)
    vx[..., 0] = np.where(sel, np.copysign(np.float32(0), vx[..., 0]), vx[..., 0])
    assert (np.signbit(vx[..., 0]) & sel).any() and (~np.signbit(vx[..., 0]) & sel).any()
    want = model(o, d, vx, mot, mc, cam)
    assert len(want[2]) == 1
    img, ns, nc = g.detect_motion(g.make_frame(d, np.eye(4), st, vertex_world=vx))
    np.testing.assert_array_equal(img, want[1])
    got = g.get_motion_clusters()
    uv = want[2][0][1]
    box = total_order_box(vx[uv[:, 1], uv[:, 0]])
    assert np.signbit(box[0]) and not np.signbit(box[3])
    np.testing.assert_array_equal(got[0]["bbox"].view(np.uint32), box.view(np.uint32))
    want[2][0] = (want[2][0][0], uv, box)
    tm.assert_clusters_equal(got, want[2], "signed zeros")
