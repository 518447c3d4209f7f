"""The oracle's tracking pass and motion detector, and the product's host clustering (M2-M4, callable without a GPU),
against the restatement in tests/temporal_model.py across the configurations the defaults never reach: ever-free
connectivity 6/18/26, occupancy thresholds in voxels and in metres, windows and buffers whose float -> double promotion
is inexact, epoch-scale stamps (256 ns grain in double), stamps exactly on now - window / now - buffer, motion
connectivity, separation distances, size filters, range / height filters, caller vertex maps with points on block and
voxel borders, and more than 255 clusters."""
import ctypes as C

import numpy as np
import pytest

from khronos_b200 import capi, synthetic as syn
import harness as hs
import temporal_model as tm

EPOCH = 1_700_000_000_123_456_789
SMALL = 150_000_000


# ---- tracking schedules ----------------------------------------------------------------------------------------------

def tie_passes(ref_ns, w, after_ns, span=8192):
    """Pass stamps around ref + w: the last one with toSeconds(now) - w < toSeconds(ref), the first one with equality
    (if any) and the first one with >, all in double as the reference compares them; only stamps > after_ns."""
    r = tm.to_seconds(ref_ns)
    base = int(ref_ns) + int(round(w * 1e9))
    lo = eq = hi = None
    for now in range(base - span, base + span):
        val = tm.to_seconds(now) - w
        if val < r:
            lo = now
        elif val == r and eq is None:
            eq = now
        elif val > r and hi is None:
            hi = now
    return [p for p in (lo, eq, hi) if p is not None and p > after_ns]


class Schedule:
    """Events of one tracking case: ("frames", [stamp, ...]) or ("pass", stamp) or ("reset",) or ("inactive",)."""

    def __init__(self):
        self.events, self.last = [], 0

    def frames(self, stamps):
        stamps = [int(s) for s in stamps]
        assert stamps[0] >= self.last and all(b >= a for a, b in zip(stamps, stamps[1:]))
        self.events.append(("frames", stamps))
        self.last = stamps[-1]

    def passes(self, stamps, with_frames=False):
        """with_frames: a frame at each pass stamp first, so that every pass runs the ever-free sweep (it only visits
        blocks integrated since the previous pass)."""
        for s in stamps:
            if s > self.last:
                if with_frames:
                    self.frames([s])
                self.events.append(("pass", int(s)))
                self.last = int(s)

    def add(self, what):
        self.events.append((what,))

    def frame_stamps(self):
        return [s for e in self.events if e[0] == "frames" for s in e[1]]


def gaps_schedule(origin, window, buffer, epoch_pairs):
    """Irregular gaps between frames and passes, two silences longer than the window, removals, one finishMapping."""
    s = Schedule()
    s.last = int(origin)
    gaps = [0.05, 0.13, 0.3, 0.07, window + 0.4, 0.11, 0.2, buffer * 1.5, 0.04, window * 2.2, 0.09, 0.17]
    for k, g in enumerate(gaps):
        t = s.last + int(g * 1e9)
        fr = [t]
        if epoch_pairs and k % 3 == 1:
            fr.append(t + 100)   # distinct stamps 100 ns apart: one double at epoch scale
        if k % 4 == 2:
            fr.append(fr[-1] + int(0.02e9))
        s.frames(fr)
        s.passes([fr[-1] + (0 if k % 2 else int(buffer * 0.5e9))])
        if k in (4, 9):
            s.add("reset")
        if k == 7:
            s.add("inactive")
            s.add("reset")
    return s


def boundary_schedule(origin, window, buffer):
    """Passes placed so that stamps fall exactly on now - buffer (against 0 and against the previous pass) and on
    now - window (against 0 and against the last frame after a silence), with the pass one step before and after."""
    s, o = Schedule(), int(origin)
    step = int(buffer * 0.25e9)
    s.frames([o + k * step for k in range(1, 4)])
    s.passes(tie_passes(0, buffer, s.last), with_frames=True)
    for _ in range(2):
        p = s.last
        s.frames([s.last + k * step for k in range(1, 4)])
        s.passes(tie_passes(p, buffer, s.last), with_frames=True)
    s.passes(tie_passes(0, window, s.last))
    f = s.last
    s.passes(tie_passes(f, window, s.last))
    s.add("reset")
    s.frames([s.last + k * step for k in range(1, 4)])
    s.passes([s.last])
    s.passes(tie_passes(s.last, window, s.last))
    s.add("reset")
    return s


_RENDER = {}


def render(cam, stamps, vps):
    """A room with a cuboid moving through it, seen from a slowly turning camera; keyed by stamps (cached)."""
    key = (cam.width, tuple(stamps))
    if key not in _RENDER:
        scene = syn.room_scene()
        scene.mover = ((0.5, 0.5, 1.2), (7.6, 2.5, 0.9), (0.0, 1.5, 0.0), 1.6)
        out = []
        for i, st in enumerate(stamps):
            T = syn.look_pose((6.0, 5.0, 1.5), np.radians(3.0 * np.sin(0.7 * i)), np.radians(10.0))
            d, l = syn.render(scene, cam, T, ((st - stamps[0]) * 1e-9) % 4.0)
            out.append((d.numpy(), l.numpy(), T))
        _RENDER[key] = out
    return _RENDER[key]


TRACKING_CASES = {
    # name: (connectivity, tsdf_occupancy_threshold, (window, buffer), vps, origin, schedule)
    "c6_voxels_default_small_gaps": (6, -1.5, (3.0, 1.0), 16, SMALL, "gaps"),
    "c18_half_voxel_inexact_epoch_gaps": (18, -0.5, (1.7, 0.35), 8, EPOCH, "gaps"),
    "c26_metres_short_small_gaps": (26, 0.02, (0.5, 0.1), 16, SMALL, "gaps"),
    "c26_above_trunc_epoch_gaps": (26, 0.2, (3.0, 1.0), 16, EPOCH, "gaps"),
    "c6_boundary_small": (6, -1.5, (3.0, 1.0), 8, SMALL, "boundary"),
    "c18_boundary_epoch": (18, -1.5, (3.0, 1.0), 16, EPOCH, "boundary"),
    "c26_boundary_inexact_epoch": (26, -0.5, (1.7, 0.35), 16, EPOCH, "boundary"),
    "c18_boundary_short_small": (18, 0.02, (0.5, 0.1), 8, SMALL, "boundary"),
}


def case_setup(name):
    conn, thr, (window, buffer), vps, origin, kind = TRACKING_CASES[name]
    trk = capi.TrackingConfig(buffer, 1.0, thr, conn, window, hs.TEST_THREADS)
    w, b = tm.cfg_double(window), tm.cfg_double(buffer)
    sched = gaps_schedule(origin, w, b, origin == EPOCH) if kind == "gaps" else boundary_schedule(origin, w, b)
    vs, trunc = (0.05, 0.15) if vps == 16 else (0.1, 0.3)
    mc = capi.default_map_config(voxel_size=vs, vps=vps, trunc=trunc, max_blocks=8192)
    return trk, sched, mc


class TrackingCheck:
    """Drives one handle through a schedule and compares every pass, removal and finishMapping with the model."""

    def __init__(self, h, trk, mc, frames):
        self.h, self.trk, self.mc, self.frames = h, trk, mc, frames
        self.diag = {"ties_window": 0, "ties_buffer": 0, "collapsed": 0, "passes": 0, "removed": 0, "ever_free": 0}

    def run(self, sched, integrate):
        it = iter(self.frames)
        for e in sched.events:
            if e[0] == "frames":
                integrate(self.h, [(next(it), st) for st in e[1]])
            elif e[0] == "pass":
                self.tracking(e[1])
            elif e[0] == "reset":
                self.reset()
            else:
                self.h.mark_all_inactive()
                b = self.h.export_blocks(likelihoods=False)
                assert not (b.block_flags & capi.FLAG_HAS_ACTIVE_DATA).any()
        return self.diag

    def tracking(self, st):
        before = self.h.export_blocks(likelihoods=False)
        self.h.update_tracking(st)
        got = self.h.export_blocks(likelihoods=False)
        want = tm.tracking_pass(before, st, self.trk, self.mc.voxel_size, self.mc.voxels_per_side)
        tm.assert_tracking_equal(got, before, want, f"pass at {st}")
        for k in ("ties_window", "ties_buffer", "collapsed"):
            self.diag[k] += want[k]
        self.diag["passes"] += 1
        self.diag["ever_free"] = int(got.ever_free.sum())

    def reset(self):
        before = self.h.export_blocks(likelihoods=False)
        removed = self.h.reset_inactive()
        want = before.block_index[tm.reset_inactive(before)]
        np.testing.assert_array_equal(np.unique(removed, axis=0), np.unique(want.reshape(-1, 3), axis=0), err_msg="reset_inactive")
        after = self.h.export_blocks(likelihoods=False)
        assert after.n == before.n - len(want)
        self.diag["removed"] += len(want)


def integrate_one_by_one(h, items):
    for (d, l, T), st in items:
        h.integrate_frame(h.make_frame(d, T, st, label=l), want_stats=False)


def run_tracking_case(lib, prefix, name, integrate=integrate_one_by_one, cam=None, make_handle=hs.make_handle):
    """make_handle(lib, prefix, map_cfg=, cam=, trk_cfg=) builds what the schedule drives: a handle, or anything with
    the same integrate / update_tracking / reset_inactive / mark_all_inactive / export_blocks calls."""
    trk, sched, mc = case_setup(name)
    cam = cam or syn.make_camera(64, 48, 32.0, 32.0, max_range=3.0)
    frames = render(cam, sched.frame_stamps(), mc.voxels_per_side)
    h = make_handle(lib, prefix, map_cfg=mc, cam=cam, trk_cfg=trk)
    chk = TrackingCheck(h, trk, mc, frames)
    diag = chk.run(sched, integrate)
    assert_case_exercised(name, diag)
    return h, diag


def assert_case_exercised(name, diag):
    conn, thr, (window, buffer), vps, origin, kind = TRACKING_CASES[name]
    assert diag["passes"] >= 6, diag
    if kind == "boundary":
        assert diag["ties_window"] > 0, diag
        # below 2^53 ns the doubles are ~1e-16 s apart: a buffer like 0.1f (not a multiple of 1 ns) never ties there
        b = tm.cfg_double(buffer) * 1e9
        if origin == EPOCH or b == int(b):
            assert diag["ties_buffer"] > 0, diag
    if origin == EPOCH and kind == "gaps":
        assert diag["collapsed"] > 0, diag
    if kind == "gaps":
        assert diag["removed"] > 0, diag
    if thr > 0.15:   # above trunc: every observed voxel counts as occupied, ever-free cannot form
        assert diag["ever_free"] == 0, diag


@pytest.mark.parametrize("name", list(TRACKING_CASES))
def test_oracle_tracking_matches_model(oracle_lib, name):
    run_tracking_case(oracle_lib, "ko_", name)


def test_ever_free_differs_across_connectivity(oracle_lib):
    """The same stream with ever-free connectivity 6, 18 and 26: the model and the oracle agree and the three
    neighbourhoods give three different ever-free counts."""
    counts = {}
    for conn in (6, 18, 26):
        trk, sched, mc = case_setup("c6_voxels_default_small_gaps")
        trk.neighbor_connectivity = conn
        cam = syn.make_camera(64, 48, 32.0, 32.0, max_range=3.0)
        frames = render(cam, sched.frame_stamps(), mc.voxels_per_side)
        h = hs.make_handle(oracle_lib, "ko_", map_cfg=mc, cam=cam, trk_cfg=trk)
        TrackingCheck(h, trk, mc, frames).run(sched, integrate_one_by_one)
        counts[conn] = int(h.export_blocks(likelihoods=False).ever_free.sum())
    assert len(set(counts.values())) == 3 and min(counts.values()) > 100, counts


# ---- motion ----------------------------------------------------------------------------------------------------------

MCAM = dict(width=96, height=72, f=48.0)
WALL = 3.0


def motion_camera(max_range=5.0):
    return syn.make_camera(MCAM["width"], MCAM["height"], MCAM["f"], MCAM["f"], max_range=max_range)


def warm_handle(lib, prefix, mot, vps=8, trk=None, cam=None, make_handle=hs.make_handle):
    """A static wall at 3 m seen for 2.5 s: the space in front of it becomes ever-free."""
    cam = cam or motion_camera()
    vs, trunc = (0.1, 0.3) if vps == 8 else (0.05, 0.15)
    mc = capi.default_map_config(voxel_size=vs, vps=vps, trunc=trunc, max_blocks=16384)
    h = make_handle(lib, prefix, map_cfg=mc, cam=cam, mot_cfg=mot,
                       trk_cfg=trk or capi.default_tracking_config(num_threads=hs.TEST_THREADS),
                       integ_cfg=capi.default_integrator_config(interpolation=capi.INTERP_NEAREST, num_threads=hs.TEST_THREADS))
    d = np.full((cam.height, cam.width), WALL, np.float32)
    l = np.full((cam.height, cam.width), 3, np.int32)
    S = 1_000_000_000
    for k in range(6):
        st = S + k * S // 2
        h.integrate_frame(h.make_frame(d, np.eye(4), st, label=l), want_stats=False)
        h.update_tracking(st)
    return h, mc, cam, 4 * S


def place(depth, cam, u0, v0, w, h, z):
    depth[v0:v0 + h, u0:u0 + w] = z


def movers_frame(cam):
    """Movers at 2.05 m (voxel 20 of 0.1 m voxels) with pixel footprints chosen to give voxel gaps of 0 (touching), 1,
    2 (face), a diagonal gap and 3. At 2.05 m one 0.1 m voxel spans 48 * 0.1 / 2.05 = 2.3 pixels."""
    d = np.full((cam.height, cam.width), WALL, np.float32)
    z = 2.05
    # pairs side by side on rows; voxel columns are floor((u - cx) / f * z / 0.1)
    place(d, cam, 6, 6, 5, 5, z)
    place(d, cam, 11, 6, 5, 5, z)            # touching the previous one
    place(d, cam, 26, 6, 5, 5, z)
    place(d, cam, 33, 6, 5, 5, z)            # about one voxel of gap
    place(d, cam, 50, 6, 5, 5, z)
    place(d, cam, 60, 6, 5, 5, z)            # about two voxels of gap
    place(d, cam, 76, 6, 5, 5, z)
    place(d, cam, 87, 6, 6, 5, z)            # about three voxels of gap
    place(d, cam, 10, 30, 5, 5, z)
    place(d, cam, 17, 37, 5, 5, z)           # diagonal
    place(d, cam, 40, 30, 5, 5, z)
    place(d, cam, 47, 37, 5, 5, 2.25)        # diagonal in depth too
    place(d, cam, 66, 30, 3, 3, z)           # a small one for the size filter
    place(d, cam, 70, 44, 12, 12, 1.55)      # a large one, nearer
    return d


def model_blocks(h):
    return h.export_blocks(likelihoods=False)


def host_cluster(product_lib, cam, mot, pose, diag, depth):
    fn = product_lib.kb_host_cluster_motion
    fn.restype = C.c_int
    img = np.zeros((cam.height, cam.width), np.int32)
    ns, nc = C.c_int32(0), C.c_int32(0)
    Tm = (C.c_double * 16)(*np.asarray(pose, np.float64).reshape(16))
    gidx, seed = np.ascontiguousarray(diag["gidx"]), np.ascontiguousarray(diag["seed"])
    d = np.ascontiguousarray(depth, np.float32)
    assert fn(C.byref(cam), C.byref(mot), Tm, C.c_void_p(gidx.ctypes.data), C.c_void_p(seed.ctypes.data),
              C.c_void_p(d.ctypes.data), C.c_void_p(img.ctypes.data), C.byref(ns), C.byref(nc)) == 0
    return img, ns.value, nc.value


def check_motion(h, mc, cam, mot, depth, stamp, pose=np.eye(4), vertex=None, product_lib=None, frame=None):
    """detect_motion on the handle against the model (image, counts, clusters); the product's host clustering on the
    model's M1 output too. Returns the model's (n_seeds, image, clusters, diag)."""
    blocks = model_blocks(h)
    want = tm.detect_motion(depth, vertex, pose, cam, blocks, mot, mc.voxel_size, mc.voxels_per_side)
    ns_m, img_m, cl_m, diag = want
    f = frame if frame is not None else h.make_frame(depth, pose, stamp, vertex_world=vertex)
    img, ns, nc = h.detect_motion(f)
    assert (ns, nc) == (ns_m, len(cl_m)), (ns, nc, ns_m, len(cl_m))
    np.testing.assert_array_equal(img, img_m)
    tm.assert_clusters_equal(h.get_motion_clusters(), cl_m, "clusters")
    if product_lib is not None and vertex is None:
        img_h, ns_h, nc_h = host_cluster(product_lib, cam, mot, pose, diag, depth)
        assert (ns_h, nc_h) == (ns_m, len(cl_m))
        np.testing.assert_array_equal(img_h, img_m)
    return want


SEPARATIONS = [-1.0, 0.0, 0.5, 1.0, 1.5, 2.0, 2.5, 3.2]


@pytest.mark.parametrize("conn", [6, 18, 26])
def test_motion_separation_sweep_matches_model(oracle_lib, product_lib, conn):
    merged = set()
    d = movers_frame(motion_camera())
    for sep in SEPARATIONS:
        mot = capi.default_motion_config(num_threads=hs.TEST_THREADS, connectivity=conn, min_separation_distance=sep)
        h, mc, cam, st = warm_handle(oracle_lib, "ko_", mot)
        ns, img, cl, diag = check_motion(h, mc, cam, mot, d, st, product_lib=product_lib)
        assert ns > 0 and diag["raw"] >= 10
        merged.add(diag["merged"])
    assert len(merged) >= 3, merged


@pytest.mark.parametrize("vps", [8, 16])
def test_motion_filters_match_model(oracle_lib, product_lib, vps):
    """Size filters dropping a cluster on each side; max_range and min_z_coordinate cutting movers."""
    d = movers_frame(motion_camera())
    pose = np.eye(4)
    pose[:3, 3] = (0.013, -0.021, 0.037)   # the camera looks along world z: min_z_coordinate cuts by depth
    base = capi.default_motion_config(num_threads=hs.TEST_THREADS, min_separation_distance=1.0)
    h, mc, cam, st = warm_handle(oracle_lib, "ko_", base, vps)
    _, _, cl0, _ = check_motion(h, mc, cam, base, d, st, pose=pose, product_lib=product_lib)
    sizes = sorted(set(len(c[1]) for c in cl0))
    assert len(sizes) >= 4
    variants = [dict(min_cluster_size=sizes[0] + 1), dict(max_cluster_size=sizes[-1] - 1),
                dict(min_cluster_size=sizes[1], max_cluster_size=sizes[-2]),
                dict(max_range=2.1), dict(min_z_coordinate=1.9), dict(min_z_coordinate=2.1, max_range=2.9)]
    for v in variants:
        mot = capi.default_motion_config(num_threads=hs.TEST_THREADS, min_separation_distance=1.0)
        for k, x in v.items():
            setattr(mot, k, x)
        h, mc, cam, st = warm_handle(oracle_lib, "ko_", mot, vps)
        ns, img, cl, diag = check_motion(h, mc, cam, mot, d, st, pose=pose, product_lib=product_lib)
        assert 0 < len(cl) < len(cl0), (v, len(cl), len(cl0))


def border_vertex_map(cam, mc):
    """A caller vertex map unlike the back-projection: points at +-k * block_size, on voxel borders and one float below
    them, on both sides of the origin, at z inside the ever-free space; the rest of the frame is a wall at 3 m."""
    H, W = cam.height, cam.width
    d = np.full((H, W), WALL, np.float32)
    vx = tm.vertex_map(d, np.eye(4), cam)
    bs = np.float32(np.float32(mc.voxel_size) * np.float32(mc.voxels_per_side))
    vs = np.float32(mc.voxel_size)
    rng = np.random.default_rng(3)
    z_layers = [np.float32(2.0) * 1, bs * np.float32(2), np.float32(1.7)]
    n = 0
    for v in range(8, 40, 2):
        for u in range(8, 88, 2):
            k = int(rng.integers(-3, 4))
            base = [bs * np.float32(k), vs * np.float32(int(rng.integers(-9, 10)))][int(rng.integers(0, 2))]
            x = base if rng.random() < 0.5 else np.nextafter(base, np.float32(-np.inf))
            y = np.float32(k) * bs if rng.random() < 0.5 else np.nextafter(np.float32(-k) * bs, np.float32(np.inf))
            zz = z_layers[n % 3]
            zz = zz if rng.random() < 0.5 else np.nextafter(zz, np.float32(-np.inf))
            vx[v, u] = (x, y, zz)
            d[v, u] = zz
            n += 1
    return d, np.ascontiguousarray(vx)


@pytest.mark.parametrize("sep", [0.0, 1.0, 2.5])
def test_motion_caller_vertex_map_borders_match_model(oracle_lib, sep):
    mot = capi.default_motion_config(num_threads=hs.TEST_THREADS, min_separation_distance=sep)
    h, mc, cam, st = warm_handle(oracle_lib, "ko_", mot)
    d, vx = border_vertex_map(cam, mc)
    ns, img, cl, diag = check_motion(h, mc, cam, mot, d, st, vertex=vx)
    assert diag["dropped"] > 0 and ns > 0 and len(cl) > 0, diag["dropped"]


def dust_frame(cam, step=3, layers=(2.05,)):
    """Isolated one-pixel movers on a lattice `step` pixels apart (more than one voxel apart at these depths)."""
    d = np.full((cam.height, cam.width), WALL, np.float32)
    for k, z in enumerate(layers):
        d[2 + k::step * len(layers), 2::step] = z
    return d


def test_motion_dust_saturates_ids(oracle_lib, product_lib):
    mot = capi.default_motion_config(num_threads=hs.TEST_THREADS, min_separation_distance=1.0)
    cam = syn.make_camera(160, 120, 40.0, 40.0, max_range=5.0)
    h, mc, cam, st = warm_handle(oracle_lib, "ko_", mot, cam=cam)
    d = dust_frame(cam, step=4)   # at 2.05 m a voxel spans 1.95 pixels: lattice points lie 2.05 voxels apart
    ns, img, cl, diag = check_motion(h, mc, cam, mot, d, st, product_lib=product_lib)
    assert len(cl) > 255 and img.max() == 255, len(cl)
    # the exhaustive pairwise overlap and the neighbourhood search agree (on a corner: the former is quadratic)
    blocks = model_blocks(h)
    d[40:] = WALL
    d[:, 80:] = WALL
    for sep in (1.0, 2.5, 3.2):
        mot.min_separation_distance = sep
        a = tm.detect_motion(d, None, np.eye(4), cam, blocks, mot, mc.voxel_size, mc.voxels_per_side, exhaustive=True)
        b = tm.detect_motion(d, None, np.eye(4), cam, blocks, mot, mc.voxel_size, mc.voxels_per_side, exhaustive=False)
        np.testing.assert_array_equal(a[1], b[1])
        assert a[3]["merged"] == b[3]["merged"]
