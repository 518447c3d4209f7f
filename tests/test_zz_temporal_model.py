"""The product's tracking pass and motion detector against the restatement in tests/temporal_model.py and, bit for bit,
against the oracle, on the cases of test_temporal_model.py: both ever-free kernels, batched integration between passes,
the in-process sharded pass (2 and 3 shards, ever-free connectivity 6 and 26), the device and host clustering paths
with the sparse table on and off, host / pinned / device frames, device-resident caller vertex maps, kb_spin_once, and
a frame with more components than the device ranking used to hold, unsharded and through the sharded live path."""
import contextlib
import functools
import os

import numpy as np
import pytest

from khronos_b200 import capi, distributed as kd, synthetic as syn
import harness as hs
import temporal_model as tm
import test_temporal_model as ttm

pytestmark = pytest.mark.gpu


@contextlib.contextmanager
def _env(**kw):
    """Switches read by kb_create: set before the handle exists, restored to their earlier values afterwards."""
    old = {k: os.environ.get(k) for k in kw}
    os.environ.update(kw)
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def integrate_batched(h, items):
    h.integrate_frames([h.make_frame(d, T, st, label=l) for (d, l, T), st in items], want_stats=False)


@pytest.mark.parametrize("v2", ["1", "0"])
@pytest.mark.parametrize("name", list(ttm.TRACKING_CASES))
def test_product_tracking_matches_model_and_oracle(oracle_lib, product_lib, name, v2):
    with _env(KB_EVERFREE_V2=v2):
        g, dg = ttm.run_tracking_case(product_lib, "kb_", name, integrate=integrate_batched)
    o, do = ttm.run_tracking_case(oracle_lib, "ko_", name)
    assert dg == do
    hs.assert_blocks_equal(o.export_blocks(), g.export_blocks(), exact_float=True, what=f"{name} v2={v2}")


class ShardSet:
    """S block-hash shards of one map in this process, driven through the sharded per-frame pipeline
    (khronos_b200.distributed.ShardedActiveWindow: kb_tracking_begin / kb_tracking_pack_halo / kb_tracking_finish and
    kb_motion_lookup_local / kb_motion_cluster_global / kb_motion_result). It offers the handle calls the schedules
    use; exports are the union of the shards, in the handle's block order."""
    make_frame = staticmethod(capi.MapHandle.make_frame)

    def __init__(self, lib, prefix, nshards=2, **kw):
        self.shards = [hs.make_handle(lib, prefix, **kw) for _ in range(nshards)]
        for r, g in enumerate(self.shards):
            g.set_shard(r, nshards)
            g.set_shard_capacity(16384, 16384)
        self.win = kd.ShardedActiveWindow(self.shards, kd.LocalComm(), device="cuda" if prefix == "kb_" else "cpu")
        self._owner = getattr(lib, prefix + "block_owner")
        self.most_blocks = [0] * nshards   # per shard, over all exports (removals may empty a shard by the end)

    def integrate_frame(self, f, want_stats=False):
        for g in self.shards:
            g.integrate_frame(f, want_stats=False)

    def integrate_frames(self, fs, want_stats=False):
        for g in self.shards:
            g.integrate_frames(fs, want_stats=False)

    def update_tracking(self, st):
        self.win.update_tracking([st] * len(self.shards), with_motion_result=False)

    def spin_once(self, f):
        res = self.win.spin_once([f] * len(self.shards))
        for img, ns, nc in res[1:]:
            assert (ns, nc) == res[0][1:]
            np.testing.assert_array_equal(img, res[0][0])
        return res[0]

    def reset_inactive(self):
        rs = np.concatenate([g.reset_inactive() for g in self.shards]).reshape(-1, 3)
        return rs[np.lexsort(rs[:, ::-1].T)]

    def mark_all_inactive(self):
        for g in self.shards:
            g.mark_all_inactive()

    def export_blocks(self, likelihoods=True):
        parts = [g.export_blocks(likelihoods=likelihoods) for g in self.shards]
        self.most_blocks = [max(a, p.n) for a, p in zip(self.most_blocks, parts)]
        for r, p in enumerate(parts):   # every block lives on its owner
            assert all(self._owner(int(b[0]), int(b[1]), int(b[2]), len(parts)) == r for b in p.block_index)
        order = np.lexsort(np.concatenate([p.block_index for p in parts])[:, ::-1].T)
        cat = {}
        for name in ("block_index", "block_flags", "distance", "weight", "last_observed", "last_occupied", "ever_free", "active",
                     "to_remove", "semantic_label", "semantic_empty", "semantic_likelihoods", "color"):
            vals = [getattr(p, name) for p in parts]
            cat[name] = None if vals[0] is None else np.concatenate(vals)[order]
        return capi.Blocks(**cat)


SHARDED_CASES = ["c6_voxels_default_small_gaps", "c26_metres_short_small_gaps", "c6_boundary_small", "c26_boundary_inexact_epoch"]


@pytest.mark.parametrize("nshards", [2, 3])
@pytest.mark.parametrize("name", SHARDED_CASES)
def test_sharded_tracking_matches_model_and_oracle(oracle_lib, product_lib, name, nshards):
    """The sharded tracking pass (ghost masks of remote neighbour blocks) at ever-free connectivity 6 and 26: after every
    pass the union of the shards equals the model, and at the end the oracle bit for bit."""
    g, dg = ttm.run_tracking_case(product_lib, "kb_", name, integrate=integrate_batched,
                                  make_handle=functools.partial(ShardSet, nshards=nshards))
    o, do = ttm.run_tracking_case(oracle_lib, "ko_", name)
    assert dg == do
    assert min(g.most_blocks) > 0, g.most_blocks   # every shard held part of the map
    hs.assert_blocks_equal(o.export_blocks(), g.export_blocks(), exact_float=True, what=f"{name} {nshards} shards")


def to_device(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def make_frames(h, kind, depth, pose, st, vertex=None):
    """A frame of the given memory kind; returns (frame, keep-alive buffers)."""
    if kind == "host":
        return h.make_frame(depth, pose, st, vertex_world=vertex), None
    if kind == "pinned":
        import torch
        d = torch.from_numpy(depth).pin_memory()
        v = None if vertex is None else torch.from_numpy(np.ascontiguousarray(vertex)).pin_memory()
        return h.make_frame(d, pose, st, vertex_world=v, memory=capi.MEM_HOST_ASYNC), (d, v)
    d = to_device(depth)
    v = None if vertex is None else to_device(vertex)
    return h.make_frame(d, pose, st, vertex_world=v, memory=capi.MEM_DEVICE), (d, v)


@pytest.mark.parametrize("sparse", ["1", "0"])
@pytest.mark.parametrize("kind", ["host", "pinned", "device"])
def test_product_motion_paths_match_model(oracle_lib, product_lib, sparse, kind):
    """Device path (sep > 0) and host path (sep <= 0, and any frame with a vertex map); the movers frame under every
    connectivity and the caller vertex map with border points (device-resident for device frames: the bounding
    boxes must come from that map)."""
    cam = ttm.motion_camera()
    mov = ttm.movers_frame(cam)
    checked = 0
    for conn, sep in ((6, 2.5), (18, 1.5), (26, 3.2), (26, 0.0), (18, -1.0)):
        mot = capi.default_motion_config(num_threads=hs.TEST_THREADS, connectivity=conn, min_separation_distance=sep)
        o, mc, _, st = ttm.warm_handle(oracle_lib, "ko_", mot)
        with _env(KB_MOTION_SPARSE=sparse):
            g = ttm.warm_handle(product_lib, "kb_", mot)[0]
        for depth, vertex in ((mov, None), ttm.border_vertex_map(cam, mc)):
            want = tm.detect_motion(depth, vertex, np.eye(4), cam, ttm.model_blocks(o), mot, mc.voxel_size, mc.voxels_per_side)
            img_o, ns_o, nc_o = o.detect_motion(o.make_frame(depth, np.eye(4), st, vertex_world=vertex))
            f, keep = make_frames(g, kind, depth, np.eye(4), st, vertex)
            img_g, ns_g, nc_g = g.detect_motion(f)
            assert (ns_g, nc_g) == (ns_o, nc_o) == (want[0], len(want[2])), (conn, sep)
            np.testing.assert_array_equal(img_g, want[1])
            np.testing.assert_array_equal(img_o, want[1])
            tm.assert_clusters_equal(g.get_motion_clusters(), want[2], f"product conn {conn} sep {sep} {kind}")
            tm.assert_clusters_equal(o.get_motion_clusters(), want[2], f"oracle conn {conn} sep {sep}")
            checked += len(want[2])
            del keep
    assert checked > 20


def overflow_camera():
    # a wide field of view: at 2.05 m a 0.1 m voxel spans 3.9 pixels, so pixels 8 apart are 2.05 voxels apart; the range
    # reaches far enough sideways that most of the image lies in front of allocated, ever-free blocks
    return syn.make_camera(640, 480, 80.0, 80.0, max_range=10.0)


def overflow_dust(cam):
    """Two interleaved lattices of one-pixel movers 8 pixels apart, at 2.05 m and 2.45 m (four voxels apart in depth):
    within a layer neighbours are at least two voxels apart, so every mover is its own component."""
    d = np.full((cam.height, cam.width), ttm.WALL, np.float32)
    d[2::8, 2::8] = 2.05
    d[6::8, 6::8] = 2.45
    return d


@pytest.mark.parametrize("sparse", ["1", "0"])
def test_product_motion_over_4096_components(oracle_lib, product_lib, sparse):
    """A 640x480 dust frame with more than 4096 isolated components (nothing merges at sep 1): kb_detect_motion and
    kb_spin_once must give the oracle's image and counts, and after kb_spin_once the whole map must match."""
    cam = overflow_camera()
    mot = capi.default_motion_config(num_threads=hs.TEST_THREADS, min_separation_distance=1.0)
    o, mc, _, st = ttm.warm_handle(oracle_lib, "ko_", mot, cam=cam)
    with _env(KB_MOTION_SPARSE=sparse):
        g = ttm.warm_handle(product_lib, "kb_", mot, cam=cam)[0]
    d = overflow_dust(cam)
    want = tm.detect_motion(d, None, np.eye(4), cam, ttm.model_blocks(o), mot, mc.voxel_size, mc.voxels_per_side)
    assert want[3]["raw"] > 4096 and len(want[2]) > 4096, want[3]["raw"]
    img_g, ns_g, nc_g = g.detect_motion(g.make_frame(d, np.eye(4), st))
    assert (ns_g, nc_g) == (want[0], len(want[2]))
    np.testing.assert_array_equal(img_g, want[1])
    l = np.full(d.shape, 3, np.int32)
    img_o, ns_o, nc_o = o.spin_once(o.make_frame(d, np.eye(4), st, label=l))
    img_s, ns_s, nc_s = g.spin_once(g.make_frame(d, np.eye(4), st, label=l))
    assert (ns_s, nc_s) == (ns_o, nc_o) == (want[0], len(want[2]))
    np.testing.assert_array_equal(img_o, want[1])
    np.testing.assert_array_equal(img_s, img_o)
    hs.assert_blocks_equal(o.export_blocks(), g.export_blocks(), exact_float=True, what=f"spin_once over 4096 sparse={sparse}")


@pytest.mark.parametrize("nshards", [2, 3])
def test_sharded_motion_over_4096_components(oracle_lib, product_lib, nshards):
    """The overflow frame through the sharded live path (kb_motion_lookup_local, kb_motion_cluster_global after the
    flag reduction, kb_motion_result, then integration and the sharded tracking pass): every shard reports the oracle's
    image and counts, and the union of the shards equals the oracle's map."""
    cam = overflow_camera()
    mot = capi.default_motion_config(num_threads=hs.TEST_THREADS, min_separation_distance=1.0)
    o, mc, _, st = ttm.warm_handle(oracle_lib, "ko_", mot, cam=cam)
    g = ttm.warm_handle(product_lib, "kb_", mot, cam=cam, make_handle=functools.partial(ShardSet, nshards=nshards))[0]
    d = overflow_dust(cam)
    l = np.full(d.shape, 3, np.int32)
    img_o, ns_o, nc_o = o.spin_once(o.make_frame(d, np.eye(4), st, label=l))
    assert nc_o > 4096
    img_g, ns_g, nc_g = g.spin_once(g.make_frame(d, np.eye(4), st, label=l))
    assert (ns_g, nc_g) == (ns_o, nc_o)
    np.testing.assert_array_equal(img_g, img_o)
    hs.assert_blocks_equal(o.export_blocks(), g.export_blocks(), exact_float=True, what=f"sharded spin_once over 4096, {nshards} shards")


def test_product_spin_once_movers_match_oracle(oracle_lib, product_lib):
    """kb_spin_once on the movers frame at every separation of the sweep: image, counts and the map afterwards."""
    cam = ttm.motion_camera()
    d = ttm.movers_frame(cam)
    l = np.full(d.shape, 3, np.int32)
    for sep in ttm.SEPARATIONS:
        mot = capi.default_motion_config(num_threads=hs.TEST_THREADS, min_separation_distance=sep, connectivity=18)
        o, mc, _, st = ttm.warm_handle(oracle_lib, "ko_", mot)
        g = ttm.warm_handle(product_lib, "kb_", mot)[0]
        want = tm.detect_motion(d, None, np.eye(4), cam, ttm.model_blocks(o), mot, mc.voxel_size, mc.voxels_per_side)
        img_o, ns_o, nc_o = o.spin_once(o.make_frame(d, np.eye(4), st, label=l))
        img_g, ns_g, nc_g = g.spin_once(g.make_frame(d, np.eye(4), st, label=l))
        assert (ns_g, nc_g) == (ns_o, nc_o) == (want[0], len(want[2])), sep
        np.testing.assert_array_equal(img_g, want[1])
        np.testing.assert_array_equal(img_o, want[1])
        hs.assert_blocks_equal(o.export_blocks(), g.export_blocks(), exact_float=True, what=f"spin_once sep {sep}")
