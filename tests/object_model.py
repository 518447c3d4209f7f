"""The two object detectors written from the spec: ConnectedSemantics (docs/ORACLE_SPEC.md §10, 2D and 3D) and
InstanceForwarding (§14), read against connected_semantics.cpp and instance_forwarding.cpp. Vectorised with scipy so
that full 640x480 frames with ~10^5 components take seconds.

Results are flat arrays, clusters in id order:
  image      (H, W) int32 object image
  ids        (n,) cluster ids; semantic (n,) its label (detectors) ; counts (n,) pixels per cluster
  pixels     (sum(counts), 2) (u, v) of every cluster in turn, within a cluster in the order given per function
  bbox       (n, 6) float32 world box (instance forwarding only)
"""
import numpy as np
from scipy import ndimage, sparse
from scipy.sparse import csgraph

F32 = np.float32
CELL_LIMIT = 1 << 17        # voxels per axis on each side of the origin (§10)
MAX_INSTANCE_IDS = 4096     # KB_MAX_INSTANCE_IDS
NAN_BITS = 0x7FC00000       # the quiet NaN of an axis without a non-NaN coordinate


def object_labels(is_object):
    return np.array([lab for lab in range(64) if lab < len(is_object) and is_object[lab]], np.int64)


def is_object_image(label, objects):
    return np.isin(label.astype(np.int64), objects)


def vertex_map(cam, pose, depth, vertex=None):
    """(H, W, 3) fp32 world vertices: the caller's map, or R·((u-cx)/fx·d, (v-cy)/fy·d, d) + t evaluated in fp32 as
    ((R0·x + R1·y) + R2·z) + t with R, t the fp32 roundings of the pose."""
    if vertex is not None:
        return np.asarray(vertex, F32).reshape(depth.shape + (3,))
    H, W = depth.shape
    d = depth.astype(F32)
    u = np.arange(W, dtype=F32)[None, :]
    v = np.arange(H, dtype=F32)[:, None]
    x = (u - F32(cam.cx)) / F32(cam.fx) * d
    y = (v - F32(cam.cy)) / F32(cam.fy) * d
    T = np.asarray(pose, np.float64).reshape(4, 4)
    R, t = T[:3, :3].astype(F32), T[:3, 3].astype(F32)
    with np.errstate(invalid="ignore", over="ignore"):
        out = [((R[a, 0] * x + R[a, 1] * y) + R[a, 2] * d) + t[a] for a in range(3)]
    return np.stack(out, -1).astype(F32)


def _group_pixels(image_ids, order_key, n_ids):
    """Pixels of ids 1..n_ids grouped by id, within an id ascending in order_key (flat pixel -> key)."""
    flat = image_ids.ravel()
    sel = np.nonzero(flat)[0]
    o = np.lexsort((order_key.ravel()[sel], flat[sel]))
    pix = sel[o]
    W = image_ids.shape[1]
    counts = np.bincount(flat[sel], minlength=n_ids + 1)[1:]
    return np.stack([pix % W, pix // W], 1).astype(np.int32), counts


def detect_2d(label, is_object, full, min_cluster_size):
    """§10 2D mode. Components of equal object labels (4- / 8-connected); ids in the order of each component's first
    pixel in the column-major scan; components smaller than min_cluster_size are zeroed but keep their id slot;
    max_cluster_size and max_range do not apply. Pixels of a cluster are listed row-major."""
    label = np.asarray(label)
    H, W = label.shape
    objects = object_labels(is_object)
    structure = np.ones((3, 3), bool) if full else ndimage.generate_binary_structure(2, 1)
    comp = np.zeros((H, W), np.int64)
    sem = [0]
    n = 0
    for lab in objects:
        cc, k = ndimage.label(label == lab, structure=structure)
        if k == 0:
            continue
        comp[cc > 0] = cc[cc > 0] + n
        sem += [int(lab)] * k
        n += k
    sem = np.asarray(sem, np.int64)
    scan = comp.T.ravel()                                 # column-major scan order
    first = np.full(n + 1, scan.size, np.int64)
    np.minimum.at(first, scan, np.arange(scan.size))
    rank = np.empty(n + 1, np.int64)
    rank[0] = 0
    rank[1 + np.argsort(first[1:], kind="stable")] = np.arange(1, n + 1)   # creation order = id
    size = np.bincount(comp.ravel(), minlength=n + 1)
    keep = size >= min_cluster_size
    keep[0] = False
    image = np.where(keep[comp], rank[comp], 0).astype(np.int32)
    kept = np.nonzero(keep)[0]
    kept = kept[np.argsort(rank[kept])]
    ids = rank[kept].astype(np.int32)
    row_major = np.arange(H * W, dtype=np.int64).reshape(H, W)
    dense = np.zeros(n + 1, np.int64)
    dense[kept] = np.arange(1, kept.size + 1)
    pixels, counts = _group_pixels(dense[comp], row_major, kept.size)
    return dict(image=image, ids=ids, semantic=sem[kept].astype(np.int32), counts=counts.astype(np.int32), pixels=pixels,
                n_components=n)


def _neighbour_offsets(full):
    """Half of the 6 / 26 neighbourhood: every adjacent voxel pair is found once."""
    out = []
    for dz in (-1, 0, 1):
        for dy in (-1, 0, 1):
            for dx in (-1, 0, 1):
                nnz = (dx != 0) + (dy != 0) + (dz != 0)
                if nnz and (full or nnz == 1) and (dz, dy, dx) > (0, 0, 0):
                    out.append((dx, dy, dz))
    return out


def candidate_voxels(cam, pose, depth, label, is_object, grid_size, max_range, vertex=None):
    """§10 3D candidates: object-class pixels with !(max_range > 0 and range > max_range), a finite vertex and a voxel
    floor(p * (1/grid_size)) inside ±2^17 cells on every axis. Returns (candidate mask, (H, W, 3) int64 voxels)."""
    vm = vertex_map(cam, pose, depth, vertex)
    inv = F32(1.0) / F32(grid_size)
    with np.errstate(invalid="ignore", over="ignore"):
        cells = np.floor((vm * inv).astype(F32))
    cand = is_object_image(label, object_labels(is_object))
    if max_range > 0:
        cand &= ~(depth.astype(F32) > F32(max_range))
    cand &= np.isfinite(vm).all(-1)
    with np.errstate(invalid="ignore"):
        cand &= ((cells >= -CELL_LIMIT) & (cells < CELL_LIMIT)).all(-1)
    vox = np.where(cand[..., None], cells, 0).astype(np.int64)
    return cand, vox


def detect_3d(cam, pose, depth, label, is_object, full, grid_size, min_cluster_size, max_cluster_size, max_range,
              vertex=None):
    """§10 3D mode. Voxels of candidate pixels per semantic id; components of the same-label voxel graph; components
    outside [min_cluster_size, max_cluster_size (if > 0)] pixels are dropped before ids are given; ids 1..n ordered by
    label, then by the component's smallest (z, y, x) voxel. Pixels of a cluster are listed row-major."""
    label = np.asarray(label)
    H, W = label.shape
    cand, vox = candidate_voxels(cam, pose, depth, label, is_object, grid_size, max_range, vertex)
    pix = np.nonzero(cand.ravel())[0]
    lab = label.ravel()[pix].astype(np.int64)
    xyz = vox.reshape(-1, 3)[pix]
    B = 2 * CELL_LIMIT

    def key(l, x, y, z):  # ascending in (label, z, y, x)
        return ((l * B + (z + CELL_LIMIT)) * B + (y + CELL_LIMIT)) * B + (x + CELL_LIMIT)

    keys, voxel_of_pixel = np.unique(key(lab, xyz[:, 0], xyz[:, 1], xyz[:, 2]), return_inverse=True)
    nv = keys.size
    first_pixel = np.zeros(nv, np.int64)
    first_pixel[voxel_of_pixel[::-1]] = np.arange(pix.size)[::-1]
    vl, vxyz = lab[first_pixel], xyz[first_pixel]
    rows, cols = [np.zeros(0, np.int64)], [np.zeros(0, np.int64)]
    for dx, dy, dz in _neighbour_offsets(full) if nv else ():
        n = vxyz + np.array([dx, dy, dz])
        inside = ((n >= -CELL_LIMIT) & (n < CELL_LIMIT)).all(1)
        k = key(vl, n[:, 0], n[:, 1], n[:, 2])
        j = np.minimum(np.searchsorted(keys, k), nv - 1)
        hit = inside & (keys[j] == k)
        rows.append(np.nonzero(hit)[0])
        cols.append(j[hit])
    rows, cols = np.concatenate(rows), np.concatenate(cols)
    graph = sparse.coo_matrix((np.ones(rows.size, np.int8), (rows, cols)), shape=(nv, nv))
    n_comp, comp_of_voxel = csgraph.connected_components(graph, directed=False)
    comp_of_pixel = comp_of_voxel[voxel_of_pixel]
    size = np.bincount(comp_of_pixel, minlength=n_comp)
    keep = size >= max(min_cluster_size, 0)
    if max_cluster_size > 0:
        keep &= size <= max_cluster_size
    smallest = np.full(n_comp, np.iinfo(np.int64).max)
    np.minimum.at(smallest, comp_of_voxel, keys)
    kept = np.nonzero(keep)[0]
    kept = kept[np.argsort(smallest[kept])]
    id_of_comp = np.zeros(n_comp, np.int64)
    id_of_comp[kept] = np.arange(1, kept.size + 1)
    image = np.zeros(H * W, np.int32)
    image[pix] = id_of_comp[comp_of_pixel]
    image = image.reshape(H, W)
    pixels, counts = _group_pixels(image, np.arange(H * W, dtype=np.int64).reshape(H, W), kept.size)
    semantic = (smallest[kept] // B ** 3).astype(np.int32)  # the label is the key's leading digit
    return dict(image=image, ids=np.arange(1, kept.size + 1, dtype=np.int32), semantic=semantic,
                counts=counts.astype(np.int32), pixels=pixels, n_components=int(n_comp), candidates=cand)


def ieee_min_max(values, groups, n_groups):
    """Per group the IEEE 754-2019 minimum and maximum over the non-NaN values (-0 below +0); a group without a non-NaN
    value gets NaN at both ends. values float32, groups in 0..n_groups-1."""
    ok = ~np.isnan(values)
    v, g = values[ok].astype(np.float64), groups[ok]
    lo = np.full(n_groups, np.inf)
    hi = np.full(n_groups, -np.inf)
    np.minimum.at(lo, g, v)
    np.maximum.at(hi, g, v)
    has = np.bincount(g, minlength=n_groups) > 0
    neg_zero = np.bincount(g, weights=(v == 0) & np.signbit(v), minlength=n_groups) > 0
    pos_zero = np.bincount(g, weights=(v == 0) & ~np.signbit(v), minlength=n_groups) > 0
    lo, hi = lo.astype(F32), hi.astype(F32)
    lo[(lo == 0) & neg_zero] = F32(-0.0)
    lo[(lo == 0) & ~neg_zero] = F32(0.0)
    hi[(hi == 0) & pos_zero] = F32(0.0)
    hi[(hi == 0) & ~pos_zero] = F32(-0.0)
    nan = np.array([NAN_BITS], np.uint32).view(F32)[0]
    lo[~has] = nan
    hi[~has] = nan
    return lo, hi


def forward_instances(cam, pose, depth, ids, max_range=0.0, min_cluster_size=0, max_cluster_size=-1,
                      min_object_volume=0.0, max_object_volume=-1.0, background=None, vertex=None):
    """§14. The object image is the label image. A pixel joins its id's cluster unless the id is 0, the id is marked in
    the background table (ids past its end are not), or max_range > 0 and range > max_range. Clusters ascending by id;
    dropped by pixel count, then, if min_object_volume > 0 or max_object_volume > 0, by the fp32 volume of the box
    (per axis the IEEE minimum / maximum of the non-NaN vertex coordinates). Pixels column-major within a cluster."""
    ids = np.asarray(ids)
    assert ids.min() >= 0 and ids.max() < MAX_INSTANCE_IDS, "ids outside 0..4095 are rejected"
    H, W = ids.shape
    sel = ids != 0
    if background is not None and len(background):
        table = np.zeros(MAX_INSTANCE_IDS, bool)
        n = min(len(background), MAX_INSTANCE_IDS)
        table[:n] = np.asarray(background[:n]) != 0
        sel &= ~table[ids]
    if max_range > 0:
        sel &= ~(depth.astype(F32) > F32(max_range))
    member = np.where(sel, ids, 0).astype(np.int64)
    counts = np.bincount(member.ravel(), minlength=MAX_INSTANCE_IDS)
    counts[0] = 0
    vm = vertex_map(cam, pose, depth, vertex).reshape(-1, 3)
    flat = member.ravel()
    m = flat > 0
    box = np.stack([ieee_min_max(vm[m, a], flat[m], MAX_INSTANCE_IDS) for a in range(3)], 0)  # (3, 2, ids)
    bbox = np.concatenate([box[:, 0].T, box[:, 1].T], 1)
    keep = counts > 0
    keep &= counts >= min_cluster_size
    if max_cluster_size > 0:
        keep &= counts <= max_cluster_size
    if min_object_volume > 0 or max_object_volume > 0:
        with np.errstate(invalid="ignore", over="ignore"):
            vol = ((bbox[:, 3] - bbox[:, 0]) * (bbox[:, 4] - bbox[:, 1]) * (bbox[:, 5] - bbox[:, 2])).astype(F32)
            vol = vol.astype(np.float64)
            drop = vol < min_object_volume
            if max_object_volume > 0:
                drop |= vol > max_object_volume
        keep &= ~drop
    kept = np.nonzero(keep)[0]
    dense = np.zeros(MAX_INSTANCE_IDS, np.int64)
    dense[kept] = np.arange(1, kept.size + 1)
    scan = (np.arange(W, dtype=np.int64)[None, :] * H + np.arange(H, dtype=np.int64)[:, None])
    pixels, c = _group_pixels(dense[member], scan, kept.size)
    return dict(image=ids.astype(np.int32).copy(), ids=kept.astype(np.int32), counts=c.astype(np.int32), pixels=pixels,
                bbox=bbox[kept].astype(F32))
