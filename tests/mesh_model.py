"""Independent model of mesh extraction (docs/ORACLE_SPEC.md §13), written from the spec alone.

`mesh(blocks, voxel_size, vps, only_mesh_updated, min_weight)` runs marching cubes on an exported map (`capi.Blocks`) and
returns the mesh in the spec's order together with coverage counters. All arithmetic is numpy float32, one operation per
expression (numpy never contracts a multiply and an add), so vertex positions are bit-exact against any implementation
that follows the spec. The per-cube and per-edge work is vectorised over chunks of blocks.

Counters (`Mesh.counts`), so that a test can assert it reached the case it exists for:
  processed            blocks processed
  drop_face / drop_edge / drop_diag
                       cubes skipped for a missing neighbour block, and only for it (every corner that exists has
                       weight >= min_weight), classed by the nearest missing neighbour: a face (+x, +y or +z), an edge
                       (two offsets) or only the diagonal (+1, +1, +1)
  drop_weight          cubes whose 8 corners exist but at least one has weight < min_weight
  weight_eq            corners of cubes with all 8 corners present whose weight equals min_weight exactly
  nan_corner           emitted vertices whose edge has a NaN distance at either end
  midpoint             emitted vertices that took the |diff| < 1e-6 branch; midpoint_nonzero: of those, diff != 0
  near_threshold       emitted vertices interpolated with 1e-6 <= |diff| < 2e-6
  tie                  emitted vertices interpolated with t == 0.5 exactly (attributes from corner 1)
  tri_inside / tri_xplane / tri_yplane / tri_zplane
                       triangles from interior cubes and from the max-x, max-y and max-z border planes
`Mesh.missing` is the set of neighbour block indices whose absence dropped a cube (as counted above)."""
from dataclasses import dataclass, field

import numpy as np

f32 = np.float32
EDGES = np.array([(0, 1), (1, 2), (2, 3), (3, 0), (4, 5), (5, 6), (6, 7), (7, 4), (0, 4), (1, 5), (2, 6), (3, 7)])
OFFS = np.array([(0, 0, 0), (1, 0, 0), (1, 1, 0), (0, 1, 0), (0, 0, 1), (1, 0, 1), (1, 1, 1), (0, 1, 1)])
MIN_DIFF = f32(1e-6)
COUNTERS = ("processed", "drop_face", "drop_edge", "drop_diag", "drop_weight", "weight_eq", "nan_corner", "midpoint",
            "midpoint_nonzero", "near_threshold", "tie", "tri_inside", "tri_xplane", "tri_yplane", "tri_zplane")


@dataclass
class Mesh:
    block_index: np.ndarray   # (n, 3) int32, ascending (x, y, z)
    offsets: np.ndarray       # (n + 1,) int64 vertex offsets
    points: np.ndarray        # (nv, 3) float32
    colors: np.ndarray        # (nv, 3) uint8
    labels: np.ndarray        # (nv,) uint32
    counts: dict = field(default_factory=dict)
    missing: set = field(default_factory=set)


def cube_order(vps):
    """(x, y, z) of every cube of a block in emission order, and the region of each (0 inside, 1/2/3 max-x/y/z plane)."""
    m = vps - 1
    order = ([(x, y, z) for x in range(m) for y in range(m) for z in range(m)] +
             [(m, y, z) for z in range(vps) for y in range(vps)] +
             [(x, m, z) for z in range(vps) for x in range(m)] +
             [(x, y, m) for y in range(m) for x in range(m)])
    region = np.repeat([0, 1, 2, 3], [m ** 3, vps * vps, vps * m, m * m])
    assert len(order) == vps ** 3
    return np.array(order, np.int64), region


def _table_rows(table):
    """Per case: the edges of its vertices in emission order (each triple (e0, e1, e2) as (e2, e1, e0))."""
    rows = []
    for c in range(256):
        r = [int(e) for e in table[c] if e >= 0]
        rows.append([e for k in range(0, len(r), 3) for e in (r[k + 2], r[k + 1], r[k])])
    return rows


def mesh(blocks, voxel_size, vps, table, only_mesh_updated=False, min_weight=1e-4, flag_mesh_updated=2, chunk=256):
    V = vps ** 3
    vs = f32(voxel_size)
    bs = vs * f32(vps)
    mw = f32(min_weight)
    bidx = np.asarray(blocks.block_index, np.int64).reshape(-1, 3)
    row_of = {tuple(b): i for i, b in enumerate(bidx.tolist())}
    todo = [i for i in range(len(bidx)) if not only_mesh_updated or (int(blocks.block_flags[i]) & flag_mesh_updated)]
    todo.sort(key=lambda i: tuple(bidx[i]))
    dist = np.asarray(blocks.distance, f32).reshape(-1, vps, vps, vps).transpose(0, 3, 2, 1)  # [row, x, y, z]
    wgt = np.asarray(blocks.weight, f32).reshape(-1, vps, vps, vps).transpose(0, 3, 2, 1)
    label = np.where(np.asarray(blocks.semantic_empty).reshape(-1, V) != 0, 0,
                     np.asarray(blocks.semantic_label).reshape(-1, V)).astype(np.uint32)
    color = (np.zeros((len(bidx), V, 3), np.uint8) if blocks.color is None
             else np.asarray(blocks.color, np.uint8).reshape(-1, V, 3))
    order, region = cube_order(vps)
    rows = _table_rows(table)
    ntri = np.array([len(r) // 3 for r in rows])
    maxv = max(len(r) for r in rows)
    row_tab = np.full((256, maxv), -1, np.int64)
    for c, r in enumerate(rows):
        row_tab[c, :len(r)] = r
    # per corner: neighbour selector (bit0 +x, bit1 +y, bit2 +z) and local voxel of every cube in emission order
    cv = order[None, :, :] + OFFS[:, None, :]                    # (8, V, 3) padded voxel coords
    sel = ((cv == vps).astype(np.int64) * np.array([1, 2, 4])).sum(-1)   # (8, V)
    loc = cv % vps
    lin = loc[..., 0] + vps * (loc[..., 1] + vps * loc[..., 2])  # (8, V)
    pops = np.array([bin(s).count("1") for s in range(8)])

    counts = dict.fromkeys(COUNTERS, 0)
    counts["processed"] = len(todo)
    missing = set()
    out_pts, out_col, out_lab, per_block = [], [], [], []
    for c0 in range(0, len(todo), chunk):
        rows_c = np.array(todo[c0:c0 + chunk], np.int64)
        n = len(rows_c)
        nbr = np.full((n, 8), -1, np.int64)
        for k, b in enumerate(bidx[rows_c].tolist()):
            for s in range(8):
                nbr[k, s] = row_of.get((b[0] + (s & 1), b[1] + ((s >> 1) & 1), b[2] + ((s >> 2) & 1)), -1)
        # corner data per cube (n, 8, V): source row and voxel
        src = nbr[:, sel]                                       # (n, 8, V)
        present = src >= 0
        srow = np.where(present, src, 0)
        lx, ly, lz = loc[..., 0][None], loc[..., 1][None], loc[..., 2][None]
        D = dist[srow, lx, ly, lz]
        W = wgt[srow, lx, ly, lz]
        wok = W >= mw
        allp = present.all(1)
        # drops for a missing neighbour (only where every existing corner passes min_weight)
        only_missing = ~allp & (wok | ~present).all(1)
        kind = np.full((n, V), 9)
        for s in range(1, 8):
            miss_s = (~present & (sel[None] == s)).any(1)
            kind = np.where(miss_s, np.minimum(kind, pops[s]), kind)
            hit = only_missing & miss_s
            for k in np.nonzero(hit.any(1))[0]:
                b = bidx[rows_c[k]]
                missing.add((int(b[0] + (s & 1)), int(b[1] + ((s >> 1) & 1)), int(b[2] + ((s >> 2) & 1))))
        counts["drop_face"] += int((only_missing & (kind == 1)).sum())
        counts["drop_edge"] += int((only_missing & (kind == 2)).sum())
        counts["drop_diag"] += int((only_missing & (kind == 3)).sum())
        counts["drop_weight"] += int((allp & ~wok.all(1)).sum())
        counts["weight_eq"] += int(((W == mw) & allp[:, None, :]).sum())
        ok = allp & wok.all(1)
        case = ((D < 0).astype(np.int64) << np.arange(8)[None, :, None]).sum(1)
        case = np.where(ok & (case != 255), case, 0)             # (n, V)
        tri_per_cube = ntri[case]
        tri_block = tri_per_cube.sum(1)
        for r in range(4):
            counts[("tri_inside", "tri_xplane", "tri_yplane", "tri_zplane")[r]] += int(tri_per_cube[:, region == r].sum())
        per_block.extend((tri_block * 3).tolist())
        kb, kt = np.nonzero(tri_per_cube)                       # emitting cubes in (block, emission order)
        if len(kb) == 0:
            continue
        nvert = 3 * tri_per_cube[kb, kt]
        cube = np.repeat(np.arange(len(kb)), nvert)
        j = np.arange(len(cube)) - np.repeat(np.cumsum(nvert) - nvert, nvert)
        e = row_tab[case[kb, kt][cube], j]
        ca, cb = EDGES[e, 0], EDGES[e, 1]
        vb, vt = kb[cube], kt[cube]
        s0, s1 = D[vb, ca, vt], D[vb, cb, vt]

        def corner_pos(c):
            blk = bidx[rows_c[vb]] + (cv[c, vt] == vps)        # block of the corner
            return (blk.astype(f32) * bs + (loc[c, vt].astype(f32) + f32(0.5)) * vs).astype(f32)

        p0, p1 = corner_pos(ca), corner_pos(cb)
        diff = (s0 - s1).astype(f32)
        interp = np.abs(diff) >= MIN_DIFF
        with np.errstate(divide="ignore", invalid="ignore"):
            t = np.where(interp, s0 / np.where(interp, diff, f32(1)), f32(0.5)).astype(f32)
        v_int = (p0 + (t[:, None] * (p1 - p0)).astype(f32)).astype(f32)
        v_mid = (f32(0.5) * (p0 + p1).astype(f32)).astype(f32)
        pts = np.where(interp[:, None], v_int, v_mid).astype(f32)
        near = np.where(t < f32(0.5), ca, cb)
        nrow = src[vb, near, vt]
        nlin = lin[near, vt]
        out_pts.append(pts)
        out_col.append(color[nrow, nlin])
        out_lab.append(label[nrow, nlin])
        counts["nan_corner"] += int((np.isnan(s0) | np.isnan(s1)).sum())
        counts["midpoint"] += int((~interp).sum())
        counts["midpoint_nonzero"] += int((~interp & (diff != 0) & ~np.isnan(diff)).sum())
        counts["near_threshold"] += int((interp & (np.abs(diff) < f32(2e-6))).sum())
        counts["tie"] += int((interp & (t == f32(0.5))).sum())
    offsets = np.zeros(len(todo) + 1, np.int64)
    offsets[1:] = np.cumsum(per_block)
    cat = lambda xs, shape, dt: np.concatenate(xs) if xs else np.zeros(shape, dt)
    return Mesh(bidx[todo].astype(np.int32).reshape(-1, 3), offsets, cat(out_pts, (0, 3), f32), cat(out_col, (0, 3), np.uint8),
                cat(out_lab, (0,), np.uint32), counts, missing)


def flags_after(blocks, only_mesh_updated, clear_updated_flag, flag_mesh_updated=2):
    """The MESH_UPDATED flags the spec predicts after generateMesh: cleared on the processed blocks iff clear_updated_flag."""
    f = np.asarray(blocks.block_flags).astype(np.uint8).copy()
    if clear_updated_flag:
        done = np.ones(len(f), bool) if not only_mesh_updated else (f & flag_mesh_updated) != 0
        f[done] &= np.uint8(~flag_mesh_updated & 0xFF)
    return f
