"""A restatement of the tracking pass (K2/K3/K2r) and the free-space motion detector (M1-M4), written from the
reference's khronos/src/active_window/integration/tracking_integrator.cpp and
khronos/src/active_window/motion_detection/free_space_motion_detector.cpp and from docs/ORACLE_SPEC.md §1, §7 and §8
only; neither oracle/ nor the product's csrc/ was consulted.

The reference works in double seconds for time and in float for geometry; so does this model: stamps go through
`to_seconds(ns) = float(ns) / 1e9` (Python floats are doubles), config values are the float32 values promoted to
double, vertices and voxel indices are formed in numpy float32, op by op in the written order.

Two places keep the reference's structure on purpose instead of the product's:
  * the ever-free sweep writes `ever_free` in place, block after block, and reads neighbours' current state, as the
    reference's threads do. The order cannot matter: a voxel is only marked if it is free now, and a neighbour passes
    if it is "ever-free or free now", so a write never changes what another voxel reads (this is why ORACLE_SPEC §7
    calls the racy read benign, and why updating a whole block at once equals the reference's voxel-by-voxel loop).
    `tracking_pass` still runs the sweep in two block orders and asserts they agree, as a guard on the sweep's own
    indexing, not as evidence for the claim;
  * motion clustering keeps the point map keyed by (block, voxel index) with out-of-range voxel indices, the DFS with
    its closed set, the exhaustive pairwise overlap check with Eigen's truncating integer norm, the recursive
    connected-cluster search and the id saturation at 255."""
import math
import sys

import numpy as np

from khronos_b200 import capi

F32 = np.float32
FLAG_TRACKING_UPDATED, FLAG_HAS_ACTIVE_DATA = capi.FLAG_TRACKING_UPDATED, capi.FLAG_HAS_ACTIVE_DATA


def to_seconds(ns):
    """toSeconds: double(ns) / 1e9, elementwise for arrays (uint64 -> float64 rounds to nearest like C++)."""
    if isinstance(ns, np.ndarray):
        return ns.astype(np.float64) / 1e9
    return float(int(ns)) / 1e9


def cfg_double(x):
    """A float config field promoted to double."""
    return float(F32(x))


def neighbour_offsets(conn):
    out = []
    for dz in (-1, 0, 1):
        for dy in (-1, 0, 1):
            for dx in (-1, 0, 1):
                nnz = (dx != 0) + (dy != 0) + (dz != 0)
                if nnz == 0 or (conn == 6 and nnz > 1) or (conn == 18 and nnz > 2):
                    continue
                out.append((dx, dy, dz))
    assert len(out) == conn
    return out


# ---- tracking --------------------------------------------------------------------------------------------------------

def occupancy_threshold(trk_cfg, voxel_size):
    """updateBlockTracking: cfg < 0 is in voxels, the product with -voxel_size is formed in float."""
    t = F32(trk_cfg.tsdf_occupancy_threshold)
    return F32(t * F32(-F32(voxel_size))) if t < 0 else t


def _ever_free_sweep(blocks, free_now, upd, order, vps, conn):
    """updateBlockEverFree over the blocks `order` (indices into blocks), writing ever_free in place."""
    bi = blocks.block_index.astype(np.int64)
    lo = bi.min(axis=0) - 1
    dims = (bi.max(axis=0) - lo + 2) * vps
    # dense grid [z, y, x] with one missing block of padding on every side
    exists = np.zeros(dims[::-1], bool)
    ef = np.zeros(dims[::-1], bool)
    free = np.zeros(dims[::-1], bool)
    org = (bi - lo) * vps
    for k in range(blocks.n):
        x0, y0, z0 = org[k]
        sl = np.s_[z0:z0 + vps, y0:y0 + vps, x0:x0 + vps]
        exists[sl] = True
        ef[sl] = blocks.ever_free[k].reshape(vps, vps, vps) != 0
        free[sl] = free_now[k].reshape(vps, vps, vps)
    offs = neighbour_offsets(conn)
    for k in order:
        if not upd[k]:
            continue
        x0, y0, z0 = org[k]
        sl = np.s_[z0:z0 + vps, y0:y0 + vps, x0:x0 + vps]
        cand = ~ef[sl] & free[sl]
        if not cand.any():
            continue
        ok = np.ones((vps, vps, vps), bool)
        for dx, dy, dz in offs:
            nb = np.s_[z0 + dz:z0 + dz + vps, y0 + dy:y0 + dy + vps, x0 + dx:x0 + dx + vps]
            # a missing neighbour block blocks; an ever-free neighbour is fine; otherwise it must be free now
            ok &= exists[nb] & (ef[nb] | free[nb])
        ef[sl] |= cand & ok
    out = np.zeros_like(blocks.ever_free)
    for k in range(blocks.n):
        x0, y0, z0 = org[k]
        out[k] = ef[z0:z0 + vps, y0:y0 + vps, x0:x0 + vps].reshape(-1)
    return out


def tracking_pass(before: capi.Blocks, stamp_ns, trk_cfg, voxel_size, vps):
    """TrackingIntegrator::updateBlocks at `stamp_ns` on the exported state `before`. Returns a dict with the expected
    last_occupied, active, to_remove, ever_free, block_flags and diagnostics:
      ties_window / ties_buffer: voxels whose stamp compared exactly equal to now - window / now - buffer in double
      collapsed: distinct observed stamps that share one double-seconds value."""
    now = to_seconds(stamp_ns)
    window, buffer = cfg_double(trk_cfg.temporal_window), cfg_double(trk_cfg.temporal_buffer)
    thr = occupancy_threshold(trk_cfg, voxel_size)
    # updateBlockTracking / updateTrackingDuration over all blocks
    occupied = before.distance < thr
    last_occ = np.where(occupied, np.uint64(stamp_ns), before.last_occupied).astype(np.uint64)
    obs_s = to_seconds(before.last_observed)
    active = obs_s >= now - window
    to_remove = (before.to_remove != 0) | ((before.active != 0) & ~active)
    flags = before.block_flags.copy()
    upd = (flags & FLAG_TRACKING_UPDATED) != 0   # the ever-free sweep's block list is taken before the pass
    flags &= np.uint8(~FLAG_TRACKING_UPDATED & 0xFF)
    has_active = active.any(axis=1)
    flags = np.where(has_active, flags | FLAG_HAS_ACTIVE_DATA, flags & np.uint8(~FLAG_HAS_ACTIVE_DATA & 0xFF)).astype(np.uint8)
    # voxelIsFree with the new last_occupied
    occ_s = to_seconds(last_occ)
    free_now = (occ_s < now - buffer) & (before.last_observed != 0)
    if before.n:
        fwd = _ever_free_sweep(before, free_now, upd, range(before.n), vps, trk_cfg.neighbor_connectivity)
        rev = _ever_free_sweep(before, free_now, upd, range(before.n - 1, -1, -1), vps, trk_cfg.neighbor_connectivity)
        np.testing.assert_array_equal(fwd, rev, err_msg="the ever-free sweep depends on the block order")
    else:
        fwd = before.ever_free.copy()
    seen = np.unique(before.last_observed[before.last_observed != 0])
    return {"last_occupied": last_occ, "active": active.astype(np.uint8), "to_remove": to_remove.astype(np.uint8),
            "ever_free": fwd.astype(np.uint8), "block_flags": flags,
            "ties_window": int((obs_s == now - window).sum()), "ties_buffer": int((occ_s == now - buffer).sum()),
            "collapsed": int(len(seen) - len(np.unique(to_seconds(seen))))}


def reset_inactive(blocks: capi.Blocks):
    """TrackingIntegrator::resetInactive: indices (rows of block_index) of the blocks that are removed."""
    no_active = (blocks.block_flags & FLAG_HAS_ACTIVE_DATA) == 0
    all_remove = (blocks.to_remove != 0).all(axis=1)
    return np.nonzero(no_active | all_remove)[0]


def assert_tracking_equal(got: capi.Blocks, before: capi.Blocks, want, what=""):
    np.testing.assert_array_equal(got.block_index, before.block_index, err_msg=f"{what} block_index")
    for name in ("last_occupied", "active", "to_remove", "ever_free", "block_flags"):
        np.testing.assert_array_equal(getattr(got, name), want[name], err_msg=f"{what} {name}")
    np.testing.assert_array_equal(got.last_observed, before.last_observed, err_msg=f"{what} last_observed")


# ---- motion ----------------------------------------------------------------------------------------------------------

def vertex_map(depth, pose, cam):
    """ORACLE_SPEC §8: p_C = ((u-cx)/fx*d, (v-cy)/fy*d, d), p_W = R p_C + t, in float32 op by op. (H, W, 3)."""
    H, W = depth.shape
    T = np.asarray(pose, np.float64)
    R, t = T[:3, :3].astype(F32), T[:3, 3].astype(F32)
    u = np.broadcast_to(np.arange(W, dtype=F32)[None, :], (H, W))
    v = np.broadcast_to(np.arange(H, dtype=F32)[:, None], (H, W))
    d = depth.astype(F32)
    x = ((u - F32(cam.cx)) / F32(cam.fx) * d).astype(F32)
    y = ((v - F32(cam.cy)) / F32(cam.fy) * d).astype(F32)
    out = np.empty((H, W, 3), F32)
    for r in range(3):
        out[..., r] = (((R[r, 0] * x + R[r, 1] * y).astype(F32) + R[r, 2] * d).astype(F32) + t[r]).astype(F32)
    return out


def point_map(depth, vertex, pose, cam, blocks: capi.Blocks, mot_cfg, voxel_size, vps):
    """setUpPointMap(Part): returns (points, seeds, diag). points: {(block, voxel index): [pixel index, ...]} with
    out-of-range voxel indices kept; seeds: set of global voxel indices (tuples); the reference's filters are the
    range, the world z limit and the existence of the block."""
    H, W = depth.shape
    vx = vertex_map(depth, pose, cam) if vertex is None else np.asarray(vertex, F32).reshape(H, W, 3)
    T = np.asarray(pose, np.float64)
    min_z = F32(float(T[2, 3]) + cfg_double(mot_cfg.min_z_coordinate))   # double sum stored in a float member
    rng = depth.astype(F32)
    keep = (rng > 0) & ~(rng > F32(mot_cfg.max_range)) & ~(vx[..., 2] < min_z)
    bs = F32(F32(voxel_size) * F32(vps))
    bsi, vsi = F32(F32(1) / bs), F32(F32(1) / F32(voxel_size))
    b = np.floor((vx * bsi).astype(F32)).astype(np.int64)
    v = np.floor(((vx - (b.astype(F32) * bs).astype(F32)).astype(F32) * vsi).astype(F32)).astype(np.int64)
    lut = {tuple(ix): k for k, ix in enumerate(blocks.block_index.tolist())}
    points, seeds = {}, set()
    dropped = 0
    for vv, uu in zip(*np.nonzero(keep)):
        blk = tuple(int(a) for a in b[vv, uu])
        k = lut.get(blk)
        if k is None:
            continue
        vox = tuple(int(a) for a in v[vv, uu])
        points.setdefault((blk, vox), []).append(int(vv) * W + int(uu))
        if not all(0 <= a < vps for a in vox):
            dropped += 1   # appended under a key the clustering never looks up
            continue
        if blocks.ever_free[k, vox[0] + vps * (vox[1] + vps * vox[2])]:
            seeds.add(tuple(blk[a] * vps + vox[a] for a in range(3)))
    return points, seeds, vx, dropped


def _key(g, vps):
    """keyFromGlobalIndex: floor division."""
    blk = tuple(a // vps for a in g)
    return blk, tuple(a - bb * vps for a, bb in zip(g, blk))


def cluster_voxels(points, seeds, conn, vps):
    """clusterDynamicVoxels: DFS from every seed in ascending (z, y, x); returns [(voxel set, pixel list)]."""
    offs = neighbour_offsets(conn)
    closed = set()
    out = []
    for seed in sorted(seeds, key=lambda g: (g[2], g[1], g[0])):
        if seed in closed:
            continue
        stack = [seed]
        vox, pix = set(), []
        while stack:
            g = stack.pop()
            if g in closed:
                continue
            closed.add(g)
            px = points.get(_key(g, vps))
            if px is None:
                continue
            pix.extend(px)
            vox.add(g)
            for d in offs:
                n = (g[0] + d[0], g[1] + d[1], g[2] + d[2])
                if n in seeds:
                    stack.append(n)
                else:
                    npx = points.get(_key(n, vps))
                    if npx is not None:   # absorbed once per adjacent seed: no closed-set check here
                        pix.extend(npx)
                        vox.add(n)
                        closed.add(n)
        out.append((vox, pix))
    return out


def _near(s, sep):
    """(p1 - p2).norm() < min_separation_distance with Eigen's integer norm: int(sqrt(double(s))) compared in float."""
    return F32(int(math.sqrt(float(s)))) < F32(sep)


def overlap_matrix(clusters, sep, exhaustive=None):
    """checkClusterOverlap for every pair. The exhaustive pairwise loop is the reference's shape; above a few hundred
    clusters it is too slow in Python, so the same predicate is evaluated through a neighbourhood search instead: it
    depends on the squared distance s only and grows with s, so the pairs it accepts are those with s <= s_max."""
    C = len(clusters)
    arrs = [np.array(sorted(c[0]), np.int64).reshape(-1, 3) for c in clusters]
    ov = np.zeros((C, C), bool)
    if C < 2:
        return ov
    if exhaustive is None:
        exhaustive = C <= 400
    if not exhaustive:
        if not _near(0, sep):
            return ov
        s_max = 0
        while _near(s_max + 1, sep):
            s_max += 1
        r = int(math.isqrt(s_max))
        owners = {}
        for c, vox in enumerate(clusters):
            for g in vox[0]:
                owners.setdefault(g, []).append(c)
        offs = [(dx, dy, dz) for dx in range(-r, r + 1) for dy in range(-r, r + 1) for dz in range(-r, r + 1)
                if dx * dx + dy * dy + dz * dz <= s_max]
        for g, cs in owners.items():
            for dx, dy, dz in offs:
                for c2 in owners.get((g[0] + dx, g[1] + dy, g[2] + dz), ()):
                    for c1 in cs:
                        if c1 != c2:
                            ov[c1, c2] = ov[c2, c1] = True
        return ov
    # the predicate depends on s only, so evaluate it once per s value that occurs
    cache = {}
    for i in range(C):
        for j in range(i + 1, C):
            d = arrs[i][:, None, :] - arrs[j][None, :, :]
            s = np.unique((d * d).sum(-1))
            hit = False
            for x in s.tolist():
                r = cache.get(x)
                if r is None:
                    r = cache[x] = _near(x, sep)
                if r:
                    hit = True
                    break
            ov[i, j] = ov[j, i] = hit
    return ov


def connected_clusters(ov, merged, i):
    """getConnectedClusters: every not yet merged cluster reachable from i (marking them merged), without i."""
    result = set()
    for j in range(ov.shape[0]):
        if merged[j]:
            continue
        if ov[i, j]:
            merged[j] = True
            result.add(j)
            result |= connected_clusters(ov, merged, j)
    result.discard(i)
    return result


def merge_clusters(clusters, sep, exhaustive=None):
    ov = overlap_matrix(clusters, sep, exhaustive)
    C = len(clusters)
    merged = [False] * C
    keep = [False] * C
    vox = [set(c[0]) for c in clusters]
    pix = [list(c[1]) for c in clusters]
    for cur in range(C):
        if merged[cur]:
            continue
        for i in connected_clusters(ov, merged, cur):
            pix[cur].extend(pix[i])
            vox[cur] |= vox[i]
        keep[cur] = True
    return [(vox[c], pix[c]) for c in range(C) if keep[c]]


def detect_motion(depth, vertex, pose, cam, blocks: capi.Blocks, mot_cfg, voxel_size, vps, exhaustive=None):
    """FreeSpaceMotionDetector::processInput. Returns (n_seeds, dynamic image (H, W) int32, clusters, diag) with
    clusters = [(sorted voxel array (n, 3) in (z, y, x) order, sorted pixel (u, v) multiset (m, 2), bbox (6,) float32)]
    and diag = {raw, merged, dropped (pixels of out-of-range voxel indices), gidx (H, W, 3) int32 (x = INT32_MIN where
    the pixel has no voxel), seed (H, W) uint8} — the last two are the per-pixel M1 output the product's clustering
    consumes."""
    H, W = depth.shape
    points, seeds, vx, dropped = point_map(depth, vertex, pose, cam, blocks, mot_cfg, voxel_size, vps)
    gidx = np.zeros((H, W, 3), np.int32)
    gidx[..., 0] = np.iinfo(np.int32).min
    seed_img = np.zeros((H, W), np.uint8)
    for (blk, vox), pxs in points.items():
        if not all(0 <= a < vps for a in vox):
            continue
        g = tuple(blk[a] * vps + vox[a] for a in range(3))
        for p in pxs:
            gidx[p // W, p % W] = g
            seed_img[p // W, p % W] = g in seeds
    image = np.zeros((H, W), np.int32)
    diag = {"raw": 0, "merged": 0, "dropped": dropped, "gidx": gidx, "seed": seed_img}
    if not seeds:
        return 0, image, [], diag
    raw = cluster_voxels(points, seeds, mot_cfg.neighbor_connectivity, vps)
    old = sys.getrecursionlimit()
    sys.setrecursionlimit(max(old, 4 * len(raw) + 100))
    try:
        merged = merge_clusters(raw, mot_cfg.min_separation_distance, exhaustive)
    finally:
        sys.setrecursionlimit(old)
    diag["raw"], diag["merged"] = len(raw), len(merged)
    kept = [c for c in merged if mot_cfg.min_cluster_size <= len(c[1]) <= mot_cfg.max_cluster_size]
    out = []
    cid = 1
    flat = vx.reshape(-1, 3)
    for vox, pix in kept:
        p = np.array(pix, np.int64)
        image.reshape(-1)[p] = cid
        if cid < 255:
            cid += 1
        pts = flat[p]
        bbox = np.concatenate([pts.min(0), pts.max(0)]).astype(F32)
        uv = np.stack([p % W, p // W], axis=1)
        uv = uv[np.lexsort((uv[:, 1], uv[:, 0]))]
        va = np.array(sorted(vox, key=lambda g: (g[2], g[1], g[0])), np.int64).reshape(-1, 3)
        out.append((va, uv, bbox))
    return len(seeds), image, out, diag


def sorted_pixels(px):
    px = np.asarray(px, np.int64).reshape(-1, 2)
    return px[np.lexsort((px[:, 1], px[:, 0]))]


def assert_clusters_equal(got, want, what=""):
    """got: MapHandle.get_motion_clusters(); want: the model's clusters. Voxels exactly, pixels as sorted multisets,
    bounding boxes bit for bit."""
    assert len(got) == len(want), f"{what}: {len(got)} clusters vs {len(want)}"
    for c, (g, (va, uv, bbox)) in enumerate(zip(got, want)):
        np.testing.assert_array_equal(g["voxels"], va, err_msg=f"{what} cluster {c} voxels")
        np.testing.assert_array_equal(sorted_pixels(g["pixels"]), uv, err_msg=f"{what} cluster {c} pixels")
        np.testing.assert_array_equal(g["bbox"].view(np.uint32), bbox.view(np.uint32), err_msg=f"{what} cluster {c} bbox")
