"""The CPU oracle's two object detectors (ConnectedSemantics, InstanceForwarding) against the from-spec model in
object_model.py, on frames constructed to hit their edge cases: ids that carry across many scan tiles, diagonal-only
chains, scan-order neighbours that are not image neighbours, exact thresholds, voxel faces and signed zeros, non-finite
and out-of-range vertices, more than 4096 raw 3D components, and odd camera sizes. Each frame asserts that its case
really occurs. tests/test_zz_object_edge_cases.py runs the same frames through the product."""
import ctypes as C

import numpy as np
import pytest

from khronos_b200 import capi
import harness as hs
import object_model as om

OBJ = (7, 8, 9, 10, 11, 12, 19)
INT_MAX = 2**31 - 1
POSE = np.eye(4)


def camera(W, H, f=300.0):
    return capi.Camera(W, H, f, f, (W - 1) / 2.0, (H - 1) / 2.0, 0.1, 10.0)


def frame(W, H, label, depth=None, vertex=None, pose=POSE, f=300.0):
    label = np.ascontiguousarray(label, np.int32)
    depth = np.ones((H, W), np.float32) if depth is None else np.ascontiguousarray(depth, np.float32)
    if vertex is not None:
        vertex = np.ascontiguousarray(vertex, np.float32).reshape(H, W, 3)
    return dict(cam=camera(W, H, f), pose=np.asarray(pose, np.float64), depth=depth, label=label, vertex=vertex)


def cfg2d(full, min_size=0, max_size=-1, max_range=0.0):
    return dict(use_3d=False, use_full_connectivity=full, min_cluster_size=min_size, max_cluster_size=max_size, max_range=max_range)


def cfg3d(full, min_size=0, max_size=-1, max_range=0.0, grid=0.25):
    return dict(use_3d=True, use_full_connectivity=full, min_cluster_size=min_size, max_cluster_size=max_size,
                max_range=max_range, grid_size=grid)


# ---- ConnectedSemantics frames: name -> (frame, [(config, check(model result))]) ---------------------------------

def f_checkerboard():
    H, W = 480, 640
    v, u = np.mgrid[:H, :W]
    fr = frame(W, H, np.where((u + v) % 2 == 0, 7, 0))
    return fr, [(cfg2d(True), lambda r: len(r["ids"]) == 1),
                (cfg2d(False), lambda r: len(r["ids"]) == 153_600 and r["ids"][-1] == 153_600)]


def f_serpentine():
    """One 4-connected path over the whole image: full rows joined at alternating ends."""
    H, W = 480, 640
    lab = np.zeros((H, W), np.int32)
    lab[::2] = 9
    lab[1::4, W - 1] = 9
    lab[3::4, 0] = 9
    fr = frame(W, H, lab)
    n = int((lab == 9).sum())
    return fr, [(cfg2d(False), lambda r: len(r["ids"]) == 1 and r["counts"][0] == n),
                (cfg2d(True, min_size=n), lambda r: len(r["ids"]) == 1),
                (cfg2d(True, min_size=n + 1), lambda r: len(r["ids"]) == 0 and r["n_components"] == 1)]


def f_diagonals():
    """Anti-diagonal chains of 8 and diagonal chains of 10: connected only through corners."""
    H, W = 240, 320
    v, u = np.mgrid[:H, :W]
    lab = np.zeros((H, W), np.int32)
    lab[(u + v) % 5 == 0] = 8
    lab[(u - v) % 7 == 3] = 10
    fr = frame(W, H, lab)
    n = int((lab > 0).sum())
    return fr, [(cfg2d(False), lambda r: len(r["ids"]) == n),
                (cfg2d(True), lambda r: 10 < len(r["ids"]) < 3000)]


def f_column_seams():
    """The bottom of column u and the top of column u+1 carry the same label: neighbours in scan order, not in the
    image. Plus full-height stripes whose neighbours across the seam are of another label."""
    H, W = 97, 1031
    lab = np.zeros((H, W), np.int32)
    lab[H - 1, 0::2] = 11
    lab[0, 1::2] = 11
    lab[2:H - 2, 3::4] = 12
    fr = frame(W, H, lab)
    n11 = int((lab == 11).sum())
    return fr, [(cfg2d(False), lambda r: (r["semantic"] == 11).sum() == n11),
                (cfg2d(True), lambda r: (r["semantic"] == 11).sum() == n11 and (r["semantic"] == 12).sum() == len(range(3, W, 4)))]


def f_touching_labels_and_non_objects():
    """Blocks of different object labels touching each other, and non-object labels (-1, 64, 255, INT_MAX, 1) touching
    them; the non-objects must stay 0."""
    H, W = 60, 80
    lab = np.zeros((H, W), np.int32)
    vals = [7, 8, 9, -1, 64, 255, INT_MAX, 19, 1, 7]
    for i, val in enumerate(vals):
        lab[:, i * 8:(i + 1) * 8] = val
    lab[20:40, :] = np.where(np.arange(W) % 3 == 0, 8, INT_MAX)[None, :]
    fr = frame(W, H, lab)
    return fr, [(cfg2d(False), lambda r: set(r["semantic"]) == {7, 8, 9, 19}),
                (cfg2d(True, max_size=3), lambda r: r["counts"].max() > 3)]   # max_cluster_size does not apply in 2D


def f_exact_min_size():
    """Components of 5, 6 and 7 pixels; min_cluster_size equal to one of them and one more."""
    H, W = 16, 40
    lab = np.zeros((H, W), np.int32)
    for i, n in enumerate((5, 6, 7, 6, 5)):
        lab[2 + i % 2 * 8, i * 8:i * 8 + n] = 7 + i % 3
    fr = frame(W, H, lab)
    return fr, [(cfg2d(False, min_size=6), lambda r: sorted(r["counts"]) == [6, 6, 7] and set(r["ids"]) == {2, 3, 4}),
                (cfg2d(True, min_size=7), lambda r: list(r["counts"]) == [7] and list(r["ids"]) == [3])]


def f_random(W, H, seed, density=0.5):
    rng = np.random.default_rng(seed)
    lab = rng.choice(np.array([7, 8, 9, -1, 3], np.int32), size=(H, W))
    lab[rng.random((H, W)) > density] = 0
    return frame(W, H, lab)


def f_odd_cameras(W, H):
    def build():
        fr = f_random(W, H, W * 1000 + H)
        return fr, [(cfg2d(False), lambda r: len(r["ids"]) >= 1), (cfg2d(True, min_size=2), lambda r: True),
                    (cfg3d(True), lambda r: len(r["ids"]) >= 1)]
    return build


# 3D: supplied vertex maps on the 0.125 grid (grid_size 0.25: 1/0.25 = 4 exactly, so every cell index is exact)

def f_faces_and_zeros():
    """Vertices on voxel faces, at +-0, tiny negatives (cell -1) and in negative cells; random labels."""
    H, W = 48, 64
    rng = np.random.default_rng(5)
    vals = np.array([0.0, -0.0, 1e-30, -1e-30, -1e-45, 0.25, -0.25, 0.125, -0.125, 0.5, -0.5, -0.375, 0.75, -1.0, 1.0],
                    np.float32)
    vm = rng.choice(vals, size=(H, W, 3))
    lab = rng.choice(np.array([7, 8, 0], np.int32), size=(H, W))
    fr = frame(W, H, lab, vertex=vm)

    def check(r):
        cells = om.candidate_voxels(fr["cam"], fr["pose"], fr["depth"], lab, om_is_object(), 0.25, 0.0, vm)[1]
        return (cells == -1).any() and (cells == 0).any() and len(r["ids"]) >= 2
    return fr, [(cfg3d(False), check), (cfg3d(True, min_size=3), lambda r: True), (cfg3d(True, grid=0.5), lambda r: True)]


def f_edge_corner_chains():
    """Voxel chains that touch only by an edge (i, i, 0) or only by a corner (i, i, i): separate voxels under 6-, one
    cluster each under 26-connectivity. Clusters whose smallest voxels differ only in x, only in y, only in z."""
    H, W = 8, 40
    vm = np.full((H, W, 3), 40.0, np.float32)   # far away, label 0
    lab = np.zeros((H, W), np.int32)
    for i in range(W):
        vm[0, i] = (i * 0.25, i * 0.25, 0.0)              # edge chain, label 7
        vm[1, i] = (-i * 0.25, i * 0.25, -i * 0.25 - 5)   # corner chain, label 8
    lab[0], lab[1] = 7, 8
    base = np.array([10.0, 10.0, 10.0], np.float32)
    for row, d in ((2, (1.0, 0, 0)), (3, (0, 1.0, 0)), (4, (0, 0, 1.0))):   # single voxels: smallest keys differ in one axis
        vm[row, :2] = [base, base + np.float32(d)]
        lab[row, :2] = 9 + row
    fr = frame(W, H, lab, vertex=vm)
    return fr, [(cfg3d(False), lambda r: (r["semantic"] == 7).sum() == W and (r["semantic"] == 8).sum() == W),
                (cfg3d(True), lambda r: (r["semantic"] == 7).sum() == 1 and (r["semantic"] == 8).sum() == 1)]


def f_shared_voxels():
    """Two labels in the same voxels: clusters per label, ids by label first."""
    H, W = 20, 30
    rng = np.random.default_rng(9)
    vm = (rng.integers(-6, 6, (H, W, 3)) * 0.125).astype(np.float32)
    lab = np.where(rng.random((H, W)) < 0.5, 19, 7).astype(np.int32)
    fr = frame(W, H, lab, vertex=vm)
    return fr, [(cfg3d(True), lambda r: list(r["semantic"]) == [7, 19]), (cfg3d(False, grid=0.125), lambda r: len(r["ids"]) >= 2)]


def depth_frame(depth, lab):
    H, W = depth.shape
    pose = np.eye(4)
    pose[:3, 3] = (0.5, -0.25, 1.0)
    return frame(W, H, lab, depth=depth, pose=pose, f=4.0)


def f_depth_edges():
    """The back-projection path: depth 0, NaN, +-inf, and max_range equal to a pixel's range and just below it."""
    H, W = 12, 16
    rng = np.random.default_rng(3)
    depth = rng.choice(np.array([0.5, 1.0, 1.5, 2.0, 2.5], np.float32), size=(H, W))
    depth[0, :4] = [0.0, np.nan, np.inf, -np.inf]
    depth[5, 5:9] = [0.0, np.nan, np.inf, -np.inf]
    lab = rng.choice(np.array([7, 8, 0], np.int32), size=(H, W))
    lab[0, :4] = 7
    lab[5, 5:9] = 8
    fr = depth_frame(depth, lab)
    below = float(np.nextafter(np.float32(2.0), np.float32(0)))

    def sizes(r):
        return int(r["counts"].sum())
    n_at2 = int(((depth <= 2.0) & np.isin(lab, OBJ)).sum())
    return fr, [(cfg3d(True), lambda r: not r["candidates"][0, 1:4].any() and r["candidates"][0, 0]),
                # depth <= 2 keeps 0 and -inf; -inf and the NaN that passes the range test have no finite vertex
                (cfg3d(True, max_range=2.0), lambda r: sizes(r) == n_at2 - 3 + 1),
                (cfg3d(True, max_range=below), lambda r: sizes(r) < n_at2 - 2),
                (cfg3d(False, max_range=2.5), lambda r: True)]


def f_bad_vertices():
    """A supplied map with NaN and infinite entries and vertices just inside and just outside +-2^17 cells."""
    H, W = 10, 12
    vm = np.zeros((H, W, 3), np.float32)
    vm[..., 0] = np.arange(W, dtype=np.float32)[None, :] * 0.25
    vm[..., 1] = np.arange(H, dtype=np.float32)[:, None] * 0.25
    lim = np.float32(32768.0)   # 2^17 cells of 0.25
    vm[0, 0] = (np.nan, 0, 0)
    vm[0, 1] = (0, np.inf, 0)
    vm[0, 2] = (0, 0, -np.inf)
    vm[0, 3] = (lim, 0, 0)                              # cell 2^17: outside
    vm[0, 4] = (lim - np.float32(0.25), 0, 0)            # cell 2^17 - 1: inside
    vm[0, 5] = (0, -lim, 0)                             # cell -2^17: inside
    vm[0, 6] = (0, -lim - np.float32(0.25), 0)           # outside
    vm[0, 7] = (0, 0, np.float32(3e38))                  # finite vertex, cell overflows
    vm[1, 0] = (np.nan, np.nan, np.nan)
    lab = np.full((H, W), 7, np.int32)
    fr = frame(W, H, lab, vertex=vm)
    want = np.ones((H, W), bool)
    want[0, [0, 1, 2, 3, 6, 7]] = False
    want[1, 0] = False
    return fr, [(cfg3d(True), lambda r: (r["candidates"] == want).all() and (r["image"][0, [4, 5]] > 0).all()),
                (cfg3d(False, max_range=5.0), lambda r: True)]


def f_many_specks():
    """More than 4096 one-voxel specks and a few large clusters: with min_cluster_size 20 only the large ones get ids."""
    H, W = 480, 640
    v, u = np.mgrid[:H, :W]
    vm = np.stack([u * 0.5, v * 0.5, np.zeros_like(u, dtype=float)], -1).astype(np.float32)   # every pixel its own isolated voxel
    lab = np.zeros((H, W), np.int32)
    rng = np.random.default_rng(1)
    lab[rng.random((H, W)) < 0.02] = 7
    for k, (v0, u0) in enumerate(((10, 10), (200, 300), (400, 600))):
        lab[v0:v0 + 6, u0:u0 + 6] = 8 + k
        vm[v0:v0 + 6, u0:u0 + 6] = (u0 * 0.5, v0 * 0.5, 100.0)   # 36 pixels in one voxel
    fr = frame(W, H, lab, vertex=vm)
    return fr, [(cfg3d(True, min_size=20), lambda r: r["n_components"] > 4096 and list(r["semantic"]) == [8, 9, 10]),
                (cfg3d(False, min_size=20, max_size=36), lambda r: len(r["ids"]) == 3)]


DETECTOR_FRAMES = {
    "checkerboard": f_checkerboard, "serpentine": f_serpentine, "diagonals": f_diagonals, "column_seams": f_column_seams,
    "touching_and_non_objects": f_touching_labels_and_non_objects, "exact_min_size": f_exact_min_size,
    "cam_7x5": f_odd_cameras(7, 5), "cam_2x300": f_odd_cameras(2, 300), "cam_300x2": f_odd_cameras(300, 2),
    "cam_1000x3": f_odd_cameras(1000, 3), "cam_257x129": f_odd_cameras(257, 129),
    "faces_and_zeros": f_faces_and_zeros, "edge_corner_chains": f_edge_corner_chains, "shared_voxels": f_shared_voxels,
    "depth_edges": f_depth_edges, "bad_vertices": f_bad_vertices, "many_specks": f_many_specks,
}
CPU_ONLY_FRAMES = {"cam_1x50": f_odd_cameras(1, 50), "cam_50x1": f_odd_cameras(50, 1)}   # the product needs 2 x 2 or more


def om_is_object():
    flags = np.zeros(64, np.uint8)
    flags[list(OBJ)] = 1
    return flags


def model_detect(fr, c):
    if c["use_3d"]:
        return om.detect_3d(fr["cam"], fr["pose"], fr["depth"], fr["label"], om_is_object(), c["use_full_connectivity"],
                            c["grid_size"], c["min_cluster_size"], c["max_cluster_size"], c["max_range"], fr["vertex"])
    return om.detect_2d(fr["label"], om_is_object(), c["use_full_connectivity"], c["min_cluster_size"])


def detector_config(c):
    return capi.default_object_detector_config(OBJ, **c)


def handle(lib, prefix, cam):
    return hs.make_handle(lib, prefix, cam=cam)


def make_frame(h, fr, **kw):
    return h.make_frame(fr["depth"], fr["pose"], 1_000_000_000, label=fr["label"], vertex_world=fr["vertex"], **kw)


def object_clusters(h):
    """kb_get_object_clusters as flat arrays, pixels within a cluster sorted row-major (their order is unspecified)."""
    f = h._fn("get_object_clusters")
    nc, tp = C.c_int32(0), C.c_int32(0)
    h._check(f(h._h, None, None, C.byref(nc), C.byref(tp)))
    info = np.zeros((max(nc.value, 1), 3), np.int32)
    px = np.zeros((max(tp.value, 1), 2), np.int32)
    h._check(f(h._h, C.c_void_p(info.ctypes.data), C.c_void_p(px.ctypes.data), C.byref(nc), C.byref(tp)))
    info, px = info[:nc.value], px[:tp.value]
    which = np.repeat(np.arange(nc.value), info[:, 2])
    px = px[np.lexsort((px[:, 0], px[:, 1], which))]
    return dict(ids=info[:, 0], semantic=info[:, 1], counts=info[:, 2], pixels=px)


def detect(h, fr, c, **kw):
    img, n = h.detect_objects(detector_config(c), make_frame(h, fr, **kw))
    out = object_clusters(h)
    assert n == len(out["ids"])
    out["image"] = img
    return out


def assert_same_objects(want, got, what):
    np.testing.assert_array_equal(got["image"], want["image"], err_msg=f"{what}: object image")
    for k in ("ids", "semantic", "counts", "pixels"):
        np.testing.assert_array_equal(got[k], want[k], err_msg=f"{what}: {k}")


@pytest.mark.parametrize("name", list(DETECTOR_FRAMES) + list(CPU_ONLY_FRAMES))
def test_oracle_detect_objects_matches_model(oracle_lib, name):
    fr, configs = {**DETECTOR_FRAMES, **CPU_ONLY_FRAMES}[name]()
    o = handle(oracle_lib, "ko_", fr["cam"])
    for c, check in configs:
        want = model_detect(fr, c)
        assert check(want), f"{name} {c}: the frame does not produce its case"
        assert_same_objects(want, detect(o, fr, c), f"{name} {c}")


# ---- InstanceForwarding frames: name -> (frame, [(kwargs, check(model result))]) ---------------------------------

def instance_vertex(H, W, rng):
    return (rng.integers(-16, 16, (H, W, 3)) * 0.125).astype(np.float32)


def i_ids_and_boxes():
    """Ids 1 and 4095, signed zeros in both orders, NaN on one axis of a cluster, a cluster NaN on every pixel of
    one axis, infinite coordinates."""
    H, W = 24, 32
    rng = np.random.default_rng(21)
    ids = rng.choice(np.array([0, 1, 5, 4095, 300], np.int32), size=(H, W))
    vm = instance_vertex(H, W, rng)
    ids[0, :6] = 40                                   # x = -0 first, then +0: min -0, max +0
    vm[0, :6] = [(-0.0, 1, 1), (0.0, 1, 1), (-0.0, 2, 1), (0.0, 1, 2), (0.0, 1, 1), (-0.0, 1, 1)]
    ids[1, :3] = 41                                   # only zeros: +0 first
    vm[1, :3] = [(0.0, -0.0, 0.0), (-0.0, -0.0, 0.0), (0.0, -0.0, 0.0)]
    ids[2, :4] = 42                                   # NaN in some coordinates, a NaN-only z axis
    vm[2, :4] = [(np.nan, 1, np.nan), (1, np.nan, np.nan), (2, 3, np.nan), (-1, 0.5, np.nan)]
    ids[3, :4] = 43                                   # infinities
    vm[3, :4] = [(np.inf, 0, 0), (-np.inf, 1, 0), (0, np.inf, np.inf), (1, 2, -np.inf)]
    ids[4, :2] = 44                                   # every coordinate NaN
    vm[4, :2] = np.nan
    fr = frame(W, H, ids, vertex=vm)

    def check(r):
        by = {int(i): b for i, b in zip(r["ids"], r["bbox"])}
        return ({1, 4095, 40, 41, 42, 43, 44} <= set(by) and np.signbit(by[40][0]) and not np.signbit(by[40][3])
                and np.isnan(by[42][2]) and np.isnan(by[44]).all() and np.isinf(by[43]).any())
    return fr, [(dict(), check), (dict(min_object_volume=1e-9), lambda r: 44 in r["ids"] and 41 not in r["ids"])]


def i_thresholds():
    """Pixel counts hit min / max_cluster_size exactly; boxes of exactly 0.5 x 0.5 x 0.25 against min_object_volume;
    a flat cluster; background tables shorter than the largest id and longer than 4096; max_range on the range."""
    H, W = 30, 40
    rng = np.random.default_rng(4)
    ids = np.zeros((H, W), np.int32)
    vm = instance_vertex(H, W, rng)
    ids[0, :10] = 10                                  # 10 pixels
    ids[1, :12] = 12                                  # 12 pixels
    ids[2, :4] = 20                                   # box 0.5 x 0.5 x 0.25 = 0.0625
    vm[2, :4] = [(0, 0, 0), (0.5, 0, 0), (0, 0.5, 0), (0.25, 0.25, 0.25)]
    ids[3, :5] = 30                                   # flat: z all equal
    vm[3, :5, 2] = 1.0
    ids[10:, 10:] = rng.choice(np.array([0, 100, 2000, 4000], np.int32), size=(H - 10, W - 10))
    depth = rng.choice(np.array([1.0, 2.0, 3.0], np.float32), size=(H, W))
    fr = frame(W, H, ids, depth=depth, vertex=vm)
    bg_short = np.zeros(101, np.uint8)
    bg_short[100] = 1                                 # ids 2000, 4000 are past its end
    bg_long = np.zeros(5000, np.uint8)
    bg_long[[12, 2000, 4500]] = 1
    return fr, [(dict(min_cluster_size=10, max_cluster_size=12), lambda r: {10, 12} <= set(r["ids"])),
                (dict(min_cluster_size=11, max_cluster_size=11), lambda r: not {10, 12} & set(r["ids"])),
                (dict(min_object_volume=0.0625), lambda r: 20 in r["ids"] and 30 not in r["ids"]),
                (dict(min_object_volume=float(np.nextafter(0.0625, 1))), lambda r: 20 not in r["ids"]),
                (dict(max_object_volume=0.0625), lambda r: {20, 30} <= set(r["ids"])),
                (dict(background=bg_short), lambda r: 100 not in r["ids"] and 4000 in r["ids"]),
                (dict(background=bg_long), lambda r: not {12, 2000} & set(r["ids"]) and 4000 in r["ids"]),
                (dict(max_range=2.0), lambda r: len(r["ids"]) >= 3),
                (dict(max_range=float(np.nextafter(np.float32(2.0), np.float32(0)))), lambda r: True)]


def i_depth_path():
    """No vertex map: the back-projection of depth, with depth 0, NaN and inf in the clusters."""
    H, W = 16, 20
    rng = np.random.default_rng(8)
    depth = rng.choice(np.array([0.5, 1.0, 2.0], np.float32), size=(H, W))
    depth[0, :3] = [0.0, np.nan, np.inf]
    ids = rng.choice(np.array([0, 3, 4, 4095], np.int32), size=(H, W))
    ids[0, :3] = 3
    fr = depth_frame(depth, ids)
    return fr, [(dict(), lambda r: 3 in r["ids"]), (dict(max_range=1.0, min_cluster_size=2), lambda r: True)]


def i_full_frame():
    H, W = 480, 640
    rng = np.random.default_rng(2)
    ids = rng.integers(0, 4096, (H, W)).astype(np.int32)
    ids[rng.random((H, W)) < 0.3] = 0
    fr = frame(W, H, ids, vertex=instance_vertex(H, W, rng))
    return fr, [(dict(min_cluster_size=50, min_object_volume=0.5), lambda r: 100 < len(r["ids"]) < 4095)]


INSTANCE_FRAMES = {"ids_and_boxes": i_ids_and_boxes, "thresholds": i_thresholds, "depth_path": i_depth_path,
                   "full_frame": i_full_frame}


def model_forward(fr, kw):
    return om.forward_instances(fr["cam"], fr["pose"], fr["depth"], fr["label"], vertex=fr["vertex"], **kw)


def forward(h, fr, kw, **fkw):
    img, cl = h.forward_instances(make_frame(h, fr, **fkw), **kw)
    return dict(image=img, ids=np.array([c["id"] for c in cl], np.int32),
                counts=np.array([len(c["pixels"]) for c in cl], np.int32),
                pixels=np.concatenate([c["pixels"] for c in cl]) if cl else np.zeros((0, 2), np.int32),
                bbox=np.array([c["bbox"] for c in cl], np.float32).reshape(-1, 6))


def assert_same_instances(want, got, what):
    np.testing.assert_array_equal(got["image"], want["image"], err_msg=f"{what}: object image")
    for k in ("ids", "counts", "pixels"):
        np.testing.assert_array_equal(got[k], want[k], err_msg=f"{what}: {k}")
    np.testing.assert_array_equal(got["bbox"].view(np.uint32), want["bbox"].view(np.uint32), err_msg=f"{what}: box bits")


@pytest.mark.parametrize("name", list(INSTANCE_FRAMES))
def test_oracle_forward_instances_matches_model(oracle_lib, name):
    fr, configs = INSTANCE_FRAMES[name]()
    o = handle(oracle_lib, "ko_", fr["cam"])
    for kw, check in configs:
        want = model_forward(fr, kw)
        assert check(want), f"{name} {kw}: the frame does not produce its case"
        assert_same_instances(want, forward(o, fr, kw), f"{name} {kw}")


def test_oracle_rejects_out_of_range_instance_ids(oracle_lib):
    fr, _ = i_thresholds()
    o = handle(oracle_lib, "ko_", fr["cam"])
    for bad in (-1, 4096):
        lab = fr["label"].copy()
        lab[5, 5] = bad
        with pytest.raises(capi.KbError):
            forward(o, dict(fr, label=lab), {})
    assert_same_instances(model_forward(fr, {}), forward(o, fr, {}), "after a rejected call")


def test_model_matches_restated_scene_detector():
    """The model against the older restatement of §10 on the rendered room frame (3D, both connectivities)."""
    import test_object_detection_oracle as t
    cam, pose, d, l = t.scene_frame(noise_seed=7)
    for full in (True, False):
        img, kept = t.expected_3d(cam, pose, d, l, OBJ, full, 0.1, 5, 3000, 4.0)
        r = om.detect_3d(cam, pose, d, l, om_is_object(), full, 0.1, 5, 3000, 4.0)
        np.testing.assert_array_equal(r["image"], img)
        assert [tuple(x) for x in zip(r["ids"].tolist(), r["semantic"].tolist(), r["counts"].tolist())] == kept
