"""Mesh extraction (docs/ORACLE_SPEC.md §13) on the oracle against the from-spec model in mesh_model.py, on maps built by
fusion so that they contain the cases where a marching-cubes kernel goes wrong.

The scenes use dyadic geometry so that the fused distances come out exact: voxels of 1/16 m, a pose that permutes the
world axes (the camera looks along world +x, and voxel centres lie at camera depths j/16 m), nearest interpolation so that
each voxel reads one pixel, and a camera whose fx = fy = 256 makes the weight of a voxel at depth 2 m exactly 16:
  tie        the surface lies midway between voxel centres, so edge crossings have sdf +-1/32 and t == 0.5 exactly;
  staircase  lateral neighbours at depth 2 m read depths 2 + kA*2^-22 and 2 - kB*2^-23, so |diff| = (2 kA + kB) * 2^-23 falls
             on both sides of 1e-6 (8 * 2^-23 < 1e-6 < 9 * 2^-23; the threshold itself is not on this grid);
  nan        a first frame puts voxels at sdf == -trunc (weight 0, distance 0/0), a second adds weight: NaN corners;
  holes      allocate_box over disjoint boxes, one block left out, fusion with allocate_blocks = False: cubes dropped for a
             missing face, edge and only-diagonal neighbour;
  removal    two depths fused 19 s apart, then update_tracking + reset_inactive: survivors border removed blocks;
  binary     the object extractor's map (BINARY semantics, allocate_box, scan_object_confidence);
  nosem      with_semantics = False;
  room_far   the room stream 5 cm / 16^3 fused ~2000 m from the origin, where positions do not come out exact.
The tie, staircase, nan and holes scenes also run translated to negative block indices and to ~2000 m from the origin.
Colour arrives only on the second frame of tie / holes (the colour layer appears mid-stream), and tie carries labels that
are not valid classes on some pixels, so some fused voxels stay semantically empty."""
import numpy as np
import pytest

from khronos_b200 import capi, synthetic as syn
import harness as hs
import mesh_model as mm
from test_mesh_oracle import TABLE

VS = 1.0 / 16
TRUNC = 0.25
W = H = 128
OFFSETS = {"origin": (0.0, 0.0, 0.0), "negative": (-4.0, -3.0, -2.0), "far": (2000.0, -1999.0, 1000.0)}
FLAG_SEQUENCE = [(True, True), (True, True), (True, False), (True, False), (False, False)]


def camera():
    return syn.make_camera(W, H, 256.0, 256.0, W / 2, H / 2, min_range=0.1, max_range=3.0)


def pose(off, lateral=(0.0, 0.0)):
    """Camera z = world +x, camera x = world +y, camera y = world +z; voxel centres at camera depths j/16."""
    T = np.eye(4)
    T[:3, :3] = [[0, 0, 1], [1, 0, 0], [0, 1, 0]]
    T[:3, 3] = (off[0] - VS / 2, off[1] + lateral[0], off[2] + lateral[1])
    return T


def voxel_bands():
    """Voxel column / row (relative to the camera axis) of every pixel at depth 2 m: 8 pixels per voxel."""
    u, v = np.meshgrid(np.arange(W), np.arange(H))
    return (u - W // 2) // 8, (v - H // 2) // 8


def labels_image(invalid=False):
    i, j = voxel_bands()
    lab = ((i + 2 * j) % 5 + 1).astype(np.int32)
    if invalid:
        lab[(i % 3 == 0) & (j % 2 == 0)] = 25  # not a class of the 20-label map: fused, but semantically empty
    return lab


def color_image():
    u, v = np.meshgrid(np.arange(W), np.arange(H))
    return np.ascontiguousarray(np.stack([(u * 7) % 256, (v * 11) % 256, ((u + v) * 3) % 256], -1).astype(np.uint8))


def flat(depth):
    return np.full((H, W), depth, np.float32)


def staircase_depth():
    i, j = voxel_bands()
    ka, kb = 1 + j % 4, 1 + (j // 4) % 4
    up = np.float32(2.0) + (ka * 2.0 ** -22).astype(np.float32)
    down = np.float32(2.0) - (kb * 2.0 ** -23).astype(np.float32)
    return np.ascontiguousarray(np.where(i % 2 == 0, up, down).astype(np.float32))


def stamp(k):
    return 1_000_000_000 + int(k * 1e9)


def map_config(vps, **kw):
    return capi.default_map_config(voxel_size=VS, vps=vps, trunc=TRUNC, max_blocks=kw.pop("max_blocks", 8192), **kw)


def integ_config(**kw):
    return capi.default_integrator_config(num_threads=hs.TEST_THREADS, interpolation=capi.INTERP_NEAREST, **kw)


def block_of(p, vps):
    bs = VS * vps
    return tuple(int(np.floor(x / bs)) for x in p)


def box_blocks(lo, hi, vps):
    a, b = block_of(lo, vps), block_of(hi, vps)
    return [(x, y, z) for x in range(a[0], b[0]) for y in range(a[1], b[1]) for z in range(a[2], b[2])]


# ---- scenes: each takes (lib, prefix, vps, offset) and returns (handle, info) ----------------------------------------------

def _handle(lib, prefix, vps, map_kw=None, integ_kw=None, cam=None):
    mc = map_config(vps, **(map_kw or {}))
    ic = integ_config(**(integ_kw or {}))
    return hs.make_handle(lib, prefix, map_cfg=mc, integ_cfg=ic, cam=cam or camera())


def scene_tie(lib, prefix, vps, off):
    h = _handle(lib, prefix, vps)
    d = flat(2.0 + VS / 2)
    lab = labels_image(invalid=True)
    h.integrate_frame(h.make_frame(d, pose(off), stamp(0), label=lab))
    h.integrate_frame(h.make_frame(d, pose(off, (0.25, 0.0)), stamp(1), label=lab, color=color_image()))
    return h, {}


def scene_staircase(lib, prefix, vps, off):
    h = _handle(lib, prefix, vps)
    h.integrate_frame(h.make_frame(staircase_depth(), pose(off), stamp(0), label=labels_image()))
    return h, {}


def scene_nan(lib, prefix, vps, off):
    h = _handle(lib, prefix, vps)
    h.integrate_frame(h.make_frame(flat(2.0 - TRUNC), pose(off), stamp(0), label=labels_image()))
    h.integrate_frame(h.make_frame(flat(2.0 + VS / 2), pose(off), stamp(1), label=labels_image()))
    return h, {}


def scene_holes(lib, prefix, vps, off):
    """Blocks of world [1, 3) x [-1, 1) x [-1, 1) m around the surface x = 2, without the block at (2, 0, 0) m."""
    h = _handle(lib, prefix, vps)
    o = np.array(off)
    gap = block_of(o + (2.0, 0.0, 0.0), vps)
    blocks = set(box_blocks(o + (1.0, -1.0, -1.0), o + (3.0, 1.0, 1.0), vps))
    # disjoint boxes: the slab below the gap in x, then the rest one block at a time
    x0 = min(b[0] for b in blocks)
    lo = (x0, min(b[1] for b in blocks), min(b[2] for b in blocks))
    hi = (gap[0] - 1, max(b[1] for b in blocks), max(b[2] for b in blocks))
    h.allocate_box(lo, hi)
    for b in sorted(blocks):
        if b[0] >= gap[0] and b != gap:
            h.allocate_box(b, b)
    d = flat(2.0 + VS / 2)
    h.integrate_frame(h.make_frame(d, pose(off), stamp(0), label=labels_image()), allocate_blocks=False)
    h.integrate_frame(h.make_frame(d, pose(off, (0.0, 0.25)), stamp(1), label=labels_image(), color=color_image()),
                      allocate_blocks=False)
    return h, {"gap": gap}


def pose_back(off):
    """Looking along world -x from x = 4 + 1/32 (camera x = world -y, camera y = world +z)."""
    T = np.eye(4)
    T[:3, :3] = [[0, 0, -1], [-1, 0, 0], [0, 1, 0]]
    T[:3, 3] = (off[0] + 4.0 + VS / 2, off[1], off[2])
    return T


def scene_removal(lib, prefix, vps, off):
    """At 1 s a camera looking along -x sees a surface at world x = 1.875 and fuses x >= 1.625; at 20 s the usual camera
    sees a surface at x = 1.5 and fuses x <= 1.75. The blocks beyond x = 2 were observed only at 1 s and are removed; the
    blocks before them stay, with the older voxels on their +x border."""
    h = _handle(lib, prefix, vps)
    h.integrate_frame(h.make_frame(flat(4.0 + VS / 2 - 1.875), pose_back(off), stamp(0), label=labels_image()))
    h.integrate_frame(h.make_frame(flat(1.5 + VS / 2), pose(off), stamp(19), label=labels_image()))
    h.update_tracking(stamp(19))
    removed = {tuple(b) for b in h.reset_inactive().tolist()}
    return h, {"removed": removed}


def scene_binary(lib, prefix, vps, off):
    h = _handle(lib, prefix, vps, map_kw={"with_tracking": False}, integ_kw={"semantic_mode": capi.SEM_BINARY})
    o = np.array(off)
    a, b = block_of(o + (1.0, -1.0, -1.0), vps), block_of(o + (2.9, 0.9, 0.9), vps)
    h.allocate_box(a, b)
    i, j = voxel_bands()
    obj = ((i + j) % 3).astype(np.int32)
    for k, dep in enumerate((2.0 + VS / 2, 2.0 + VS / 2, 2.0 - VS / 2)):
        h.integrate_frame(h.make_frame(flat(dep), pose(off, (0.0, 0.125 * k)), stamp(k), object_image=obj, target_id=1),
                          allocate_blocks=False)
    h.scan_object_confidence(0.5, 2)
    return h, {}


def scene_nosem(lib, prefix, vps, off):
    h = _handle(lib, prefix, vps, map_kw={"with_semantics": False})
    h.integrate_frame(h.make_frame(flat(2.0 + VS / 2), pose(off), stamp(0), label=labels_image()))
    h.integrate_frame(h.make_frame(staircase_depth(), pose(off, (0.125, 0.0)), stamp(1), color=color_image()))
    return h, {}


def scene_room_far(lib, prefix, vps, off):
    cam = hs.small_camera(8)
    frames, poses, stamps = room_frames_far(cam)
    mc = capi.default_map_config(vps=vps, max_blocks=8192)
    h = hs.make_handle(lib, prefix, map_cfg=mc, cam=cam)
    colors = [syn.colorize(l, d) for d, l in frames]
    hs.run_fusion(h, frames, poses, stamps, colors=[None] + colors[1:])
    return h, {}


_ROOM = {}


def room_frames_far(cam, shift=(1600.0, -1200.0, 800.0)):
    """Room frames rendered at the room's own poses and fused at poses ~2000 m away: the same images, a translated map."""
    if "frames" not in _ROOM:
        poses, stamps = syn.orbit_trajectory(3, laps=0.05)
        _ROOM["frames"] = (hs.render_frames(syn.room_scene(), cam, poses, stamps), poses, stamps)
    frames, poses, stamps = _ROOM["frames"]
    moved = []
    for T in poses:
        T = np.array(T, np.float64).copy()
        T[:3, 3] += shift
        moved.append(T)
    return frames, moved, stamps


SCENES = {"tie": scene_tie, "staircase": scene_staircase, "nan": scene_nan, "holes": scene_holes, "removal": scene_removal,
          "binary": scene_binary, "nosem": scene_nosem, "room_far": scene_room_far}
CASES = ([(s, o) for s in ("tie", "staircase", "nan", "holes") for o in OFFSETS] +
         [(s, "origin") for s in ("removal", "binary", "nosem")] + [("room_far", "origin")])


def voxel_size_of(name):
    return 0.05 if name == "room_far" else VS


# ---- checks ----------------------------------------------------------------------------------------------------------------

def assert_mesh_equals_model(got, model, what):
    bi, off, pts, col, lab = got
    np.testing.assert_array_equal(bi, model.block_index, err_msg=f"{what}: blocks")
    np.testing.assert_array_equal(off, model.offsets, err_msg=f"{what}: vertex offsets")
    np.testing.assert_array_equal(pts.view(np.uint32), model.points.view(np.uint32), err_msg=f"{what}: point bits")
    np.testing.assert_array_equal(col, model.colors, err_msg=f"{what}: colours")
    np.testing.assert_array_equal(lab, model.labels, err_msg=f"{what}: labels")


def min_weights(blocks):
    """1e-4, 0, -1, a weight that occurs in the map (so that >= and > differ), and one above every weight."""
    w = blocks.weight[np.isfinite(blocks.weight) & (blocks.weight > 0)]
    occurring = float(np.sort(w)[len(w) // 2])
    return [1e-4, 0.0, -1.0, occurring, float(w.max()) * 2.0]


def check_handle(h, voxel_size, vps, what, again=None):
    """Meshes the handle's map at every min_weight with (False, False), then runs the flag sequence; every mesh must equal
    the model on the handle's own export. Returns (meshes in call order, summed counters, union of missing blocks,
    weight_eq at the occurring weight)."""
    meshes, total, missing = [], dict.fromkeys(mm.COUNTERS, 0), set()

    def one(only, clear, mw, tag):
        before = h.export_blocks(likelihoods=False)
        model = mm.mesh(before, voxel_size, vps, TABLE, only_mesh_updated=only, min_weight=mw)
        got = h.generate_mesh(only, clear, mw)
        assert_mesh_equals_model(got, model, f"{what} {tag} min_weight={mw}")
        after = h.export_blocks(likelihoods=False)
        np.testing.assert_array_equal(after.block_flags, mm.flags_after(before, only, clear), err_msg=f"{what} {tag}: flags")
        for k, v in model.counts.items():
            total[k] += v
        missing.update(model.missing)
        meshes.append(got)
        return model

    blocks = h.export_blocks(likelihoods=False)
    mws = min_weights(blocks)
    eq = 0
    for mw in mws:
        m = one(False, False, mw, "all blocks")
        if mw == mws[3]:
            eq = m.counts["weight_eq"]
        if mw == mws[4]:
            assert len(m.points) == 0
    for k, (only, clear) in enumerate(FLAG_SEQUENCE):
        if k == 2 and again is not None:
            again(h)
        one(only, clear, 1e-4, f"call {k} ({only}, {clear})")
    return meshes, total, missing, eq


def again_fn(name, off):
    """A later frame for the flag sequence: it re-marks the blocks it touches as mesh_updated."""
    if name in ("room_far", "binary"):
        return None
    alloc = name != "holes"

    def f(h):
        h.integrate_frame(h.make_frame(flat(2.0 + VS / 2), pose(off, (-0.25, 0.0)), stamp(40), label=labels_image()),
                          allocate_blocks=alloc)
    return f


SCENE_TARGETS = {
    "tie": lambda c, info, miss: c["tie"] > 0,
    "staircase": lambda c, info, miss: c["midpoint_nonzero"] > 0 and c["near_threshold"] > 0,
    "nan": lambda c, info, miss: c["nan_corner"] > 0,
    "holes": lambda c, info, miss: c["drop_diag"] > 0 and c["drop_edge"] > 0 and c["drop_face"] > 0 and info["gap"] in miss,
    "removal": lambda c, info, miss: len(miss & info["removed"]) > 0 and c["tri_inside"] + c["tri_xplane"] > 0,
    "binary": lambda c, info, miss: c["processed"] > 0,
    "nosem": lambda c, info, miss: c["processed"] > 0,
    "room_far": lambda c, info, miss: c["tri_inside"] > 0,
}


def run_scene(lib, prefix, name, vps, offname):
    h, info = SCENES[name](lib, prefix, vps, OFFSETS[offname])
    meshes, counts, missing, eq = check_handle(h, voxel_size_of(name), vps, f"{prefix}{name}/{offname}/vps{vps}",
                                               again=again_fn(name, OFFSETS[offname]))
    assert SCENE_TARGETS[name](counts, info, missing), (name, counts, info, sorted(missing)[:8])
    assert eq > 0, "no corner weight equals the occurring min_weight"
    assert counts["tri_inside"] + counts["tri_xplane"] + counts["tri_yplane"] + counts["tri_zplane"] > 0
    return h, meshes, counts


@pytest.mark.parametrize("vps", [8, 16])
@pytest.mark.parametrize("name,offname", CASES)
def test_oracle_mesh_equals_model(oracle_lib, name, offname, vps):
    run_scene(oracle_lib, "ko_", name, vps, offname)


def test_scenes_reach_every_border_plane_and_attribute(oracle_lib):
    """Over the tie and staircase scenes at both block sizes, triangles come from the interior and all three border planes,
    and the vertex attributes include colours, labels and semantically empty (label 0) vertices."""
    planes = dict.fromkeys(("tri_inside", "tri_xplane", "tri_yplane", "tri_zplane"), 0)
    colours, labels = set(), set()
    for vps in (8, 16):
        for name in ("tie", "staircase"):
            h, meshes, counts = run_scene(oracle_lib, "ko_", name, vps, "negative")
            for k in planes:
                planes[k] += counts[k]
            for m in meshes:
                colours.update(map(tuple, m[3][:2000].tolist()))
                labels.update(np.unique(m[4]).tolist())
    assert all(v > 0 for v in planes.values()), planes
    assert (0, 0, 0) in colours and len(colours) > 10
    assert 0 in labels and len(labels) > 3
