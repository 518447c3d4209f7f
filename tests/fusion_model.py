"""An independent float64 model of K1 (per-voxel fusion) and the semantic update, written from docs/ORACLE_SPEC.md
§2-§6 only. Given a list of blocks (K0 is pinned separately) and a frame sequence, `fuse` returns the voxel state the
spec prescribes, vectorised over voxels and looping over frames.

The product and the oracle evaluate the spec in fp32; this model evaluates it in float64, except where the spec itself
prescribes a rounding to float (§1 voxel centres, §2 the pose inverse, §6 the MLE constants, config values). fp32 and
float64 may take different branches where a value lies next to a decision threshold, so every (voxel, frame) records
whether one of its decisions is within the fp32 error `delta` of its threshold:
  * z > 0 and the image bounds (projection validity);
  * the round() half-points and floor() integer points of u and v, and near-ties of the largest bilinear tap weight
    (interpolateID): these are found by re-evaluating the taps at u +- du, v +- dv, with (du, dv) the fp32 error bound
    of the projection; a decision counts as near only if the perturbed point takes a different branch (another nearest
    depth, another label or mask value at the ID pixel, bilinear <-> nearest, valid <-> invalid);
  * the adaptive depth-difference threshold: max - min of two fp32 depths is exact in float64, and fp32 rounds it to
    nearest, so the branches can differ only for a difference strictly inside (thr - ulp(thr), thr);
  * sdf against -trunc (skip), +-trunc (band) and -eps (drop-off).
A voxel with any near decision in any frame is `excluded`; callers assert that the excluded share stays small."""
import numpy as np

from khronos_b200 import capi

F32 = np.float32
U24 = 2.0 ** -24   # fp32 unit roundoff


def voxel_centres(block_index, voxel_size, vps):
    """§1 in fp32 (the spec's index math), returned as float64 (n, V, 3)."""
    vs = F32(voxel_size)
    bs = F32(vs * F32(vps))
    lin = np.arange(vps ** 3)
    v = np.stack([lin % vps, (lin // vps) % vps, lin // (vps * vps)], axis=-1).astype(F32)
    o = np.asarray(block_index, np.int64).astype(F32)[:, None, :] * bs
    return (o + (v[None] + F32(0.5)) * vs).astype(np.float64)


def mle_constants(num_labels, confidence):
    """§6: formed in double, rounded once to float."""
    a = float(F32(np.log(float(F32(confidence)))))
    b = float(F32(np.log((1.0 - float(F32(confidence))) / (num_labels - 1))))
    init = float(F32(np.log(1.0 / num_labels)))
    return a, b, init


class _Taps:
    """Interpolation of §5.1 for a set of projected points (float64 u, v)."""

    def __init__(self, cam, depth, interp, adaptive_thr, u, v):
        W, H = cam.width, cam.height
        self.W = W
        inside = (u >= 0) & (u <= W - 1) & (v >= 0) & (v <= H - 1)
        ur, vr = np.floor(u + 0.5), np.floor(v + 0.5)  # round half away from zero (u, v >= 0 where it matters)
        un = np.clip(ur, 0, W - 1).astype(np.int64)
        vn = np.clip(vr, 0, H - 1).astype(np.int64)
        d_flat = depth.reshape(-1).astype(np.float64)
        near_px = vn * W + un
        near_ok = inside & (d_flat[near_px] > 0)
        u0f, v0f = np.floor(u), np.floor(v)
        foot = inside & (u0f + 1 < W) & (v0f + 1 < H)
        u0 = np.clip(u0f, 0, W - 2).astype(np.int64)
        v0 = np.clip(v0f, 0, H - 2).astype(np.int64)
        du, dv = u - u0f, v - v0f
        px = np.stack([v0 * W + u0, (v0 + 1) * W + u0, v0 * W + u0 + 1, (v0 + 1) * W + u0 + 1], axis=-1)
        r = d_flat[px]
        wts = np.stack([(1 - du) * (1 - dv), (1 - du) * dv, du * (1 - dv), du * dv], axis=-1)
        bil_ok = foot & (r > 0).all(axis=-1)
        spread = r.max(axis=-1) - r.min(axis=-1)   # exact: difference of two fp32 values
        if interp == capi.INTERP_NEAREST:
            use_bil = np.zeros_like(inside)
        elif interp == capi.INTERP_BILINEAR:
            use_bil = np.ones_like(inside)
        else:
            use_bil = bil_ok & (spread < adaptive_thr)
        self.spread = np.where(bil_ok, spread, 0.0)
        self.valid = np.where(use_bil, bil_ok, near_ok)
        self.use_bil = use_bil
        self.range = np.where(use_bil, (((wts[:, 0] * r[:, 0] + wts[:, 1] * r[:, 1]) + wts[:, 2] * r[:, 2]) + wts[:, 3] * r[:, 3]),
                              d_flat[near_px])
        k = np.argmax(wts, axis=-1)  # first maximum = lowest tap index on ties
        self.id_px = np.where(use_bil, np.take_along_axis(px, k[:, None], axis=-1)[:, 0], near_px)
        # adaptive decisions whose fp32 rounding of (max - min) could land on the other side of the threshold
        ulp = float(np.spacing(F32(adaptive_thr)))
        self.adaptive_near = (interp == capi.INTERP_ADAPTIVE) & bil_ok & (spread < adaptive_thr) & (spread > adaptive_thr - ulp)


def block_in_frustum(cam, mc, block_index, pose):
    """§4 K0 (allocate_blocks = true) for the given blocks: the block centre passes the §3 frustum test with
    infl = block_size * 0.8660254. Returns (selected, near) with `near` = within fp32 error of one of the planes."""
    bs = F32(F32(mc.voxel_size) * F32(mc.voxels_per_side))
    infl = float(F32(bs * F32(0.8660254)))
    c = ((np.asarray(block_index, np.int64).astype(F32) + F32(0.5)) * bs).astype(np.float64)
    T = np.asarray(pose, np.float64).reshape(4, 4)
    Ri = (T[:3, :3].T).astype(F32).astype(np.float64)
    ti = (-(T[:3, :3].T @ T[:3, 3])).astype(F32).astype(np.float64)
    p = c @ Ri.T + ti
    ep = 8.0 * U24 * (np.abs(c) @ np.abs(Ri).T + np.abs(ti)).max(axis=1)
    fx, fy, cx, cy = float(F32(cam.fx)), float(F32(cam.fy)), float(F32(cam.cx)), float(F32(cam.cy))
    xl, xr = (0 - cx) / fx, (cam.width - 1 - cx) / fx
    yt, yb = (0 - cy) / fy, (cam.height - 1 - cy) / fy
    r = np.sqrt((p ** 2).sum(axis=1))
    tests = [p[:, 2] + infl, r - (float(F32(cam.min_range)) - infl), (float(F32(cam.max_range)) + infl) - r,
             (p[:, 0] - xl * p[:, 2]) / np.sqrt(1 + xl * xl) + infl, (-p[:, 0] + xr * p[:, 2]) / np.sqrt(1 + xr * xr) + infl,
             (p[:, 1] - yt * p[:, 2]) / np.sqrt(1 + yt * yt) + infl, (-p[:, 1] + yb * p[:, 2]) / np.sqrt(1 + yb * yb) + infl]
    sel = np.ones(len(c), bool)
    near = np.zeros(len(c), bool)
    for t in tests:
        sel &= ~(t < 0)
        near |= np.abs(t) < ep
    return sel, near


def _frame_update(cam, mc, ic, P, fr, delta_scale=1.0):
    """One frame over the points P (m, 3) float64. Returns a dict of per-point measurement fields."""
    T = np.asarray(fr["pose"], np.float64).reshape(4, 4)
    R, t = T[:3, :3], T[:3, 3]
    Ri = (R.T).astype(F32).astype(np.float64)              # §2: sensor_T_world formed in double, rounded once to float
    ti = (-(R.T @ t)).astype(F32).astype(np.float64)
    pc = P @ Ri.T + ti
    x, y, z = pc[:, 0], pc[:, 1], pc[:, 2]
    fx, fy, cx, cy = float(F32(cam.fx)), float(F32(cam.fy)), float(F32(cam.cx)), float(F32(cam.cy))
    # fp32 error bound of p_C per axis: ((a + b) + c) + t rounds four times, each by at most u of a partial sum bounded by
    # the sum of the magnitudes of the terms; u/v add a product, a quotient and a sum
    ep = 4.0 * U24 * (np.abs(P) @ np.abs(Ri).T + np.abs(ti)) * delta_scale
    zpos = z > 0
    with np.errstate(divide="ignore", invalid="ignore"):
        zs = np.where(zpos, z, 1.0)
        u = fx * x / zs + cx
        v = fy * y / zs + cy
        du = fx * (ep[:, 0] + np.abs(x / zs) * ep[:, 2]) / zs + 3.0 * U24 * (np.abs(u) + cx) * delta_scale
        dv = fy * (ep[:, 1] + np.abs(y / zs) * ep[:, 2]) / zs + 3.0 * U24 * (np.abs(v) + cy) * delta_scale
    # where the fp32 evaluation in the spec's operation order is exact (axis-aligned poses, dyadic coordinates), the
    # error is zero and exact ties stay decided the same way in both precisions
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        P32, R32, t32 = P.astype(F32), Ri.astype(F32), ti.astype(F32)
        pc32 = np.stack([((R32[i, 0] * P32[:, 0] + R32[i, 1] * P32[:, 1]) + R32[i, 2] * P32[:, 2]) + t32[i] for i in range(3)], axis=1)
        exact = (pc32.astype(np.float64) == pc).all(axis=1)
        zs32 = np.where(zpos, pc32[:, 2], F32(1))
        u32 = F32(fx) * pc32[:, 0] / zs32 + F32(cx)
        v32 = F32(fy) * pc32[:, 1] / zs32 + F32(cy)
    du = np.where(exact & (u32.astype(np.float64) == u), 0.0, du)
    dv = np.where(exact & (v32.astype(np.float64) == v), 0.0, dv)
    ep = np.where(exact, 0.0, ep[:, 2])
    interp, thr = ic.interpolation_method, float(F32(ic.adaptive_max_depth_difference))
    tp = _Taps(cam, fr["depth"], interp, thr, u, v)
    valid = zpos & tp.valid
    # what the ID pixel selects: the label (or the BINARY object test) and the mask; another ID pixel with the same
    # values takes the same branch
    idkey = np.zeros(cam.width * cam.height, np.int64)
    if ic.semantic_mode == capi.SEM_MLE and fr.get("label") is not None:
        idkey = idkey + fr["label"].reshape(-1).astype(np.int64)
    elif ic.semantic_mode == capi.SEM_BINARY:
        idkey = idkey + (fr["object_image"].reshape(-1) == fr["target_id"])
    if fr.get("mask") is not None:
        idkey = idkey * 2 + (fr["mask"].reshape(-1) != 0)
    # perturbation: does a shift of the projection within the fp32 error change a branch?
    unstable = np.zeros_like(valid)
    for su, sv in ((-1, -1), (-1, 1), (1, -1), (1, 1)):
        q = _Taps(cam, fr["depth"], interp, thr, u + su * du, v + sv * dv)
        unstable |= (q.valid != tp.valid) | ((q.use_bil != tp.use_bil) & tp.valid) | ((idkey[q.id_px] != idkey[tp.id_px]) & tp.valid)
        unstable |= tp.valid & ~tp.use_bil & q.valid & (q.range != tp.range)   # another nearest pixel
    unstable &= zpos
    near = (np.abs(z) < ep) | (zpos & unstable) | (zpos & tp.adaptive_near)

    trunc = float(F32(mc.truncation_distance))
    vs = float(F32(mc.voxel_size))
    sdf = tp.range - z
    # fp32 error of sdf: the interpolated range (weights carry the projection error times the depth step) and z
    # (the bilinear range moves by at most the 2x2 depth spread per pixel of shift)
    esdf = (du + dv) * np.where(tp.use_bil, tp.spread, 0.0) + 4.0 * U24 * (np.abs(tp.range) + np.abs(z)) + ep
    keep = valid & ~(sdf < -trunc)
    near |= valid & (np.abs(sdf + trunc) < esdf)
    band = keep & (np.abs(sdf) < trunc)
    near |= keep & (np.abs(np.abs(sdf) - trunc) < esdf)
    idp = tp.id_px
    if fr.get("mask") is not None:
        keep &= ~(band & (fr["mask"].reshape(-1)[idp] != 0))
    label = None
    if ic.semantic_mode == capi.SEM_MLE and fr.get("label") is not None:
        label = fr["label"].reshape(-1)[idp].astype(np.int64)
        blocked = np.asarray(ic.label_blocked, np.uint8)
        lab_c = np.clip(label, 0, len(blocked) - 1)
        keep &= ~(band & (label >= 0) & (label < len(blocked)) & (blocked[lab_c] != 0))
    elif ic.semantic_mode == capi.SEM_BINARY:
        label = (fr["object_image"].reshape(-1)[idp] == fr["target_id"]).astype(np.int64)
    band &= keep
    w = (fx * fy) * (vs * vs) / (zs * zs)
    if not ic.use_constant_weight:
        w = w / (zs * zs)
    # weight error: 1/z^4 (1/z^2 with constant weight) inherits the relative error of z four (two) times, plus ~8 fp32
    # roundings; the drop-off factor inherits the sdf error
    ew = w * ((2.0 if ic.use_constant_weight else 4.0) * ep / zs + 8.0 * U24)
    if ic.use_weight_dropoff:
        e = float(F32(ic.weight_dropoff_epsilon))
        eps = e if e > 0 else -e * vs
        drop = sdf < -eps
        near |= keep & (np.abs(sdf + eps) < esdf)
        fac = (trunc + sdf) / (trunc - eps)
        ew = np.where(drop, ew * np.maximum(fac, 0.0) + w * esdf / (trunc - eps), ew)
        w = np.where(drop, np.maximum(w * fac, 0.0), w)
    return {"ew": ew, "keep": keep, "band": band, "sdf": np.clip(sdf, -trunc, trunc), "w": w, "label": label, "near": near, "esdf": esdf}


def fuse(block_index, frames, cam, mc, ic, allocate_blocks=True, delta_scale=1.0):
    """Voxel state after fusing `frames` (dicts: depth, pose, stamp, optional label / mask / object_image + target_id)
    into the blocks `block_index` (all initially empty); with `allocate_blocks` a block takes part in a frame only if
    it passes that frame's frustum test (§4), otherwise every block is processed. Returns a dict of (n, V[, L]) arrays: distance, weight,
    last_observed, updates, band_updates, likelihoods, semantic_label, semantic_empty, excluded, the per-voxel fp32
    error bound of the measured sdf (max over frames) and the weight error the drop-off factor inherits from it."""
    n, V = len(block_index), mc.voxels_per_side ** 3
    P = voxel_centres(block_index, mc.voxel_size, mc.voxels_per_side).reshape(-1, 3)
    m = len(P)
    L = {capi.SEM_MLE: ic.num_labels, capi.SEM_BINARY: 2}.get(ic.semantic_mode, 0) if mc.with_semantics else 0
    dist, wt = np.zeros(m), np.zeros(m)
    last = np.zeros(m, np.uint64)
    ups, bups = np.zeros(m, np.int64), np.zeros(m, np.int64)
    lik = np.zeros((m, max(L, 1)))
    empty = np.ones(m, bool)
    excl = np.zeros(m, bool)
    esdf_max = np.zeros(m)
    werr = np.zeros(m)
    maxw = float(F32(ic.max_weight))
    if ic.semantic_mode == capi.SEM_MLE and L:
        a, b, init = mle_constants(L, ic.label_confidence)
    for fr in frames:
        r = _frame_update(cam, mc, ic, P, fr, delta_scale)
        k = r["keep"]
        near = r["near"]
        if allocate_blocks:
            bsel, bnear = block_in_frustum(cam, mc, block_index, fr["pose"])
            bsel, bnear = np.repeat(bsel, V), np.repeat(bnear, V)
            near = (near & bsel) | (bnear & (r["keep"] | near))
            k &= bsel
            r["band"] &= bsel
        excl |= near
        esdf_max = np.maximum(esdf_max, np.where(k, r["esdf"], 0.0))
        werr += np.where(k, r["ew"], 0.0)
        with np.errstate(divide="ignore", invalid="ignore"):
            nd = (dist * wt + r["sdf"] * r["w"]) / (wt + r["w"])
        dist = np.where(k, nd, dist)
        wt = np.where(k, np.minimum(wt + r["w"], maxw), wt)
        last = np.where(k, np.uint64(fr["stamp"]), last)
        ups += k
        if L and r["label"] is not None:
            sem = r["band"] & (r["label"] >= 0) & (r["label"] < L)
            bups += sem
            idx = np.nonzero(sem)[0]
            first = idx[empty[idx]]
            if ic.semantic_mode == capi.SEM_MLE:
                lik[first] = init
                onehot = np.arange(L)[None, :] == r["label"][idx][:, None]
                lik[idx] += np.where(onehot, a, b)
            else:
                lik[first] = 0.0
                lik[idx, r["label"][idx]] += 1.0
            empty[idx] = False
    out = {"distance": dist, "weight": wt, "last_observed": last, "updates": ups, "band_updates": bups,
           "excluded": excl, "esdf": esdf_max, "weight_error": werr, "semantic_empty": empty}
    if L:
        out["likelihoods"] = lik[:, :L]
        if ic.semantic_mode == capi.SEM_MLE:
            out["semantic_label"] = np.argmax(lik[:, :L], axis=1)
        else:
            out["semantic_label"] = (lik[:, 1] > lik[:, 0]).astype(np.int64)
    return {k: (x.reshape(n, V, -1) if x.ndim == 2 else x.reshape(n, V)) for k, x in out.items()}
