"""Marching cubes (SURVEY.md §8f row 1, docs/ORACLE_SPEC.md §13): the case table and the oracle's mesher.
The reference's mesher lives in un-vendored Hydra (parity unpinned); what can be pinned is pinned here:
  * both copies of the 256-case table (product + oracle) are identical, every row uses exactly the cube edges whose end
    points differ in sign, and meshes of random sign fields are closed, 2-manifold and consistently oriented;
  * the oracle's mesh equals the from-spec model (mesh_model.py) on its own exported TSDF (bit-exact vertices, colours, labels);
  * geometry: the mesh of a fused flat wall lies on the wall, faces the camera side, and its area matches."""
import os
import re
from collections import Counter

import numpy as np
import pytest

from khronos_b200 import capi, synthetic as syn
import harness as hs
import mesh_model as mm

EDGES = [(0, 1), (1, 2), (2, 3), (3, 0), (4, 5), (5, 6), (6, 7), (7, 4), (0, 4), (1, 5), (2, 6), (3, 7)]
OFFS = [(0, 0, 0), (1, 0, 0), (1, 1, 0), (0, 1, 0), (0, 0, 1), (1, 0, 1), (1, 1, 1), (0, 1, 1)]


def _table(path):
    src = open(os.path.join(hs.ROOT, path)).read()
    body = src[src.index("[256][16] = {"):]
    body = body[:body.index("};")]
    rows = [[int(x) for x in re.findall(r"-?\d+", ln)] for ln in body.splitlines()[1:] if "{" in ln]
    t = np.array(rows)
    assert t.shape == (256, 16)
    return t


TABLE = _table("oracle/oracle_mc_tables.hpp")


def test_table_copies_identical_and_edge_sets_exact():
    np.testing.assert_array_equal(TABLE, _table("khronos_b200/csrc/kb_mc_tables.h"))
    for c in range(256):
        active = {e for e, (a, b) in enumerate(EDGES) if ((c >> a) & 1) != ((c >> b) & 1)}
        used = [e for e in TABLE[c] if e >= 0]
        assert set(used) == active and len(used) % 3 == 0, c
        k = len(used)
        assert all(e == -1 for e in TABLE[c][k:])


def test_table_meshes_are_closed_manifold_and_oriented():
    rng = np.random.default_rng(0)
    for p in (0.5, 0.3, 0.7):
        n = 10
        neg = np.zeros((n, n, n), bool)
        neg[1:-1, 1:-1, 1:-1] = rng.random((n - 2, n - 2, n - 2)) < p
        directed = Counter()
        for x in range(n - 1):
            for y in range(n - 1):
                for z in range(n - 1):
                    c = sum(1 << i for i, (dx, dy, dz) in enumerate(OFFS) if neg[x + dx, y + dy, z + dz])
                    row = TABLE[c]
                    k = 0
                    while k < 16 and row[k] >= 0:
                        vs = []
                        for e in (row[k + 2], row[k + 1], row[k]):
                            a, b = EDGES[e]
                            pa = (x + OFFS[a][0], y + OFFS[a][1], z + OFFS[a][2])
                            pb = (x + OFFS[b][0], y + OFFS[b][1], z + OFFS[b][2])
                            vs.append((min(pa, pb), max(pa, pb)))
                        for i in range(3):
                            directed[(vs[i], vs[(i + 1) % 3])] += 1
                        k += 3
        assert directed
        for (a, b), cnt in directed.items():
            assert cnt == 1 and directed.get((b, a), 0) == 1


def _room(n=5, scale=8):
    cam = hs.small_camera(scale)
    scene = syn.room_scene()
    poses, stamps = syn.orbit_trajectory(n, laps=0.1)
    return cam, hs.render_frames(scene, cam, poses, stamps), poses, stamps


def test_oracle_mesh_equals_numpy_restatement(oracle_lib):
    cam, frames, poses, stamps = _room()
    o = hs.make_handle(oracle_lib, "ko_", cam=cam)
    hs.run_fusion(o, frames, poses, stamps)
    bi, off, pts, col, lab = o.generate_mesh(only_mesh_updated=False, clear_updated_flag=False)
    ref = mm.mesh(o.export_blocks(), 0.05, 16, TABLE)
    assert len(ref.block_index) == len(bi) and off[-1] == len(pts) and len(pts) % 3 == 0 and len(pts) > 3000
    np.testing.assert_array_equal(bi, ref.block_index)
    np.testing.assert_array_equal(off, ref.offsets)
    np.testing.assert_array_equal(pts.view(np.uint32), ref.points.view(np.uint32))
    np.testing.assert_array_equal(col, ref.colors)
    np.testing.assert_array_equal(lab, ref.labels)


def test_mesh_updated_flag_semantics(oracle_lib):
    cam, frames, poses, stamps = _room(4)
    o = hs.make_handle(oracle_lib, "ko_", cam=cam)
    hs.run_fusion(o, frames[:2], poses[:2], stamps[:2])
    bi1, off1, *_ = o.generate_mesh(True, True)
    assert len(bi1) > 0
    bi2, off2, *_ = o.generate_mesh(True, True)
    assert len(bi2) == 0 and off2[-1] == 0          # flags cleared
    hs.run_fusion(o, frames[2:], poses[2:], stamps[2:])
    bi3, *_ = o.generate_mesh(True, False)
    bi4, *_ = o.generate_mesh(True, False)
    assert 0 < len(bi3) == len(bi4)                  # clear_updated_flag = false keeps them (extractor's call)
    flags = o.export_blocks().block_flags
    assert int(((flags & capi.FLAG_MESH_UPDATED) != 0).sum()) == len(bi3)


def test_flat_wall_mesh_geometry(oracle_lib):
    """Camera looks along +x at a wall x = 3: after fusing one frame the mesh is the plane x = 3 (vertex error well below
    a voxel), every triangle faces the camera (-x, the positive-sdf side), and the triangle areas tile the observed wall."""
    cam = hs.small_camera(4)
    T = syn.look_pose((0.0, 0.0, 1.0), 0.0, 0.0)
    d = np.zeros((cam.height, cam.width), np.float32)
    # z-depth of the plane x = 3 for a camera at the origin looking along +x is 3 everywhere
    d[:] = 3.0
    l = np.full((cam.height, cam.width), 3, np.int32)
    o = hs.make_handle(oracle_lib, "ko_", cam=cam)
    o.integrate_frame(o.make_frame(d, T, 1_000_000_000, label=l))
    bi, off, pts, col, lab = o.generate_mesh(False, False)
    assert len(pts) > 300
    assert np.abs(pts[:, 0] - 3.0).max() < 2e-3
    tri = pts.reshape(-1, 3, 3)
    nrm = np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0])
    assert (nrm[:, 0] < 0).all()
    area = 0.5 * np.linalg.norm(nrm, axis=1).sum()
    # the frustum at depth 3 spans (W-1)/fx*3 x (H-1)/fy*3 metres; the mesh covers it up to a voxel-wide rim
    full = (cam.width - 1) / cam.fx * 3.0 * (cam.height - 1) / cam.fy * 3.0
    assert 0.85 * full < area < 1.05 * full
    assert set(np.unique(lab)) == {3}
