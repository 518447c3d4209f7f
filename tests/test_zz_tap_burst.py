"""The fuse kernel's image taps against the oracle, bit for bit, on scenes built around the pixel choices of its taps.

fuseKernel loads a frame's four depth taps together at clamped addresses and restates computeTaps on them: the nearest
pixel (the nearest interpolator, the adaptive fallback, the last column and row) is selected from the four registers
instead of being loaded again. The label / mask pixel (interpolateID) is the dominant bilinear tap (ties -> the lowest
tap index) when bilinear interpolation is used, else the nearest pixel; the two differ where the weights tie, so a
kernel that read the label at the dominant tap after the adaptive fallback to nearest fails here.

The scenes: voxels of 1/16 m seen from axis-aligned poses, so that the voxel centres on the camera's optical-axis planes
and on the plane z = 2 m project exactly onto half-pixel columns and rows (cx = 31.5, cy = 23.5, f = 32), where two or
four bilinear weights tie; other poses put the centres at z = 2 m on whole pixels, up to the last column and row. The
depth image is a checkerboard of terraces whose step equals the adaptive threshold, so quads across a step fall back to
nearest and flat ones stay bilinear; labels, object ids and the dynamic mask change across every pixel line."""
import numpy as np
import pytest

from khronos_b200 import capi, synthetic as syn
import fusion_model as fm
import harness as hs

pytestmark = pytest.mark.gpu

F32 = np.float32
W, H = 64, 48
NEAR_MM, FAR_MM = 1875, 2125  # terraces at 1.875 m and 2.125 m: the step is the adaptive threshold, 0.25 m
N_FRAMES = 8
TARGET = 0


def camera():
    return syn.make_camera(W, H, 32.0, 32.0, max_range=5.0)  # cx = 31.5, cy = 23.5


def images():
    u, v = np.meshgrid(np.arange(W), np.arange(H))
    depth_mm = np.where(((u // 3) + (v // 4)) % 2 == 0, NEAR_MM, FAR_MM).astype(np.uint16)
    depth_mm[(u % 13 == 7) & (v % 11 == 5)] = 0  # holes: invalid quads and invalid nearest pixels
    label = ((3 * u + 5 * v) % 20).astype(np.int32)  # differs between any two pixels of a quad
    obj = ((u + v) % 3).astype(np.int32)  # the BINARY object test differs across most pixel lines
    mask = (u % 2).astype(np.int32)
    color = np.stack([(7 * u) % 256, (11 * v) % 256, (u * v) % 256], axis=-1).astype(np.uint8)
    return depth_mm, label, obj, mask, color


def poses():
    out = []
    for i in range(N_FRAMES):
        T = np.eye(4)
        if i % 2 == 0:
            # p_C.x, p_C.y: multiples of the voxel size; half-pixel columns / rows on the axis planes and at z = 2 m
            T[:3, 3] = (0.03125 * (2 * i + 1), 0.03125 * (2 * i + 3), -0.03125 - 0.0625 * (i // 2 % 2))
        else:
            # p_C.x, p_C.y: odd multiples of half a voxel; whole pixels at z = 2 m, up to column W - 1 and row H - 1
            T[:3, 3] = (0.0625 * i, 0.0625 * (i + 1), -0.03125)
        out.append(T)
    return out


def has_mask(i):
    return i % 3 != 1


def config(kind, interp, vps):
    # trunc is not a multiple of 1/16: no sdf of these dyadic scenes equals -trunc, where the weight drop-off makes a first
    # update 0 / 0 (the NaN payloads of the oracle and the product differ)
    mc = capi.default_map_config(voxel_size=0.0625, vps=vps, trunc=0.2, max_blocks=16384)
    mode = capi.SEM_BINARY if kind == "binary" else capi.SEM_MLE
    ic = capi.default_integrator_config(semantic_mode=mode, interpolation=interp, num_threads=hs.TEST_THREADS)
    scale = F32(0.001)
    # the fp32 depth step exactly (Sterbenz), so that `max - min < threshold` is decided by an exact equality
    ic.adaptive_max_depth_difference = float(F32(FAR_MM) * scale - F32(NEAR_MM) * scale) if kind == "compact" else 0.25
    return mc, ic


def frames(kind):
    depth_mm, label, obj, mask, color = images()
    depth = depth_mm.astype(np.float32) / F32(1000.0)  # 1.875, 2.125 and 0: exact
    out = []
    for i, T in enumerate(poses()):
        fr = {"pose": T, "stamp": 1_000_000_000 + i * 33_333_333, "mask": mask if has_mask(i) else None,
              "depth": depth, "label": None, "object_image": None, "color": None, "target_id": TARGET}
        if kind == "binary":
            fr["object_image"] = obj
        else:
            fr["label"] = label
        if kind == "mle_color":
            fr["color"] = color
        if kind == "compact":
            fr["depth"] = depth_mm.astype(np.float32) * F32(0.001)  # what the kernel reads from the u16 image
            fr["depth_u16"], fr["label_u8"] = depth_mm, label.astype(np.uint8)
        out.append(fr)
    return out


def make_frame(h, fr):
    if "depth_u16" in fr:
        return h.make_frame(None, fr["pose"], fr["stamp"], depth_u16=fr["depth_u16"], label_u8=fr["label_u8"], mask=fr["mask"])
    return h.make_frame(fr["depth"], fr["pose"], fr["stamp"], label=fr["label"], mask=fr["mask"], color=fr["color"],
                        object_image=fr["object_image"], target_id=fr["target_id"])


def tap_counts(blocks, frs, cam, mc, ic):
    """The kernel's per-frame decisions restated in fp32 over the map's voxels. Returns the number of in-band (voxel,
    frame) pairs whose interpolateID pixel is not the dominant bilinear tap of an in-image quad and carries another
    label or mask value, and the number of pairs next to the surface that project onto the last column or row."""
    P = fm.voxel_centres(blocks.block_index, mc.voxel_size, mc.voxels_per_side).reshape(-1, 3).astype(F32)
    V = mc.voxels_per_side ** 3
    fx, fy, cx, cy = F32(cam.fx), F32(cam.fy), F32(cam.cx), F32(cam.cy)
    trunc, thr = F32(mc.truncation_distance), F32(ic.adaptive_max_depth_difference)
    split = border = 0
    for fr in frs:
        T = np.asarray(fr["pose"], np.float64)
        R, t = (T[:3, :3].T).astype(F32), (-(T[:3, :3].T @ T[:3, 3])).astype(F32)
        pc = [((R[i, 0] * P[:, 0] + R[i, 1] * P[:, 1]) + R[i, 2] * P[:, 2]) + t[i] for i in range(3)]
        x, y, z = pc
        sel = np.repeat(fm.block_in_frustum(cam, mc, blocks.block_index, fr["pose"])[0], V) & (z > 0)
        zs = np.where(z > 0, z, F32(1))
        u, v = fx * x / zs + cx, fy * y / zs + cy
        sel &= (u >= 0) & (u <= F32(W - 1)) & (v >= 0) & (v <= F32(H - 1))
        uc, vc = np.clip(u, 0, W - 1), np.clip(v, 0, H - 1)
        u0, v0 = np.floor(uc).astype(np.int64), np.floor(vc).astype(np.int64)
        du, dv = uc - u0.astype(F32), vc - v0.astype(F32)
        i0 = v0 * W + u0
        su, sv = (u0 + 1 < W).astype(np.int64), np.where(v0 + 1 < H, W, 0)
        d = fr["depth"].reshape(-1)
        r = np.stack([d[i0], d[i0 + sv], d[i0 + su], d[i0 + sv + su]], axis=-1)
        inside = (su != 0) & (sv != 0)
        near_px = i0 + (du >= F32(0.5)) + np.where(dv >= F32(0.5), W, 0)
        one = F32(1)
        wts = np.stack([(one - du) * (one - dv), (one - du) * dv, du * (one - dv), du * dv], axis=-1)
        k = np.argmax(wts, axis=-1)  # first maximum: the lowest tap index on ties
        dom_px = i0 + (k >> 1) + np.where(k & 1, W, 0)
        border += int((sel & (np.abs(d[near_px] - z) < trunc) & ((u0 == W - 1) | (v0 == H - 1))).sum())
        all_valid = (r > 0).all(axis=-1)
        interp = ic.interpolation_method
        if interp == capi.INTERP_NEAREST:
            bil = np.zeros_like(inside)
        elif interp == capi.INTERP_BILINEAR:
            bil = inside & all_valid
            sel &= bil
        else:
            bil = inside & all_valid & ((r.max(axis=-1) - r.min(axis=-1)) < thr)
        rng = np.where(bil, ((wts[:, 0] * r[:, 0] + wts[:, 1] * r[:, 1]) + wts[:, 2] * r[:, 2]) + wts[:, 3] * r[:, 3], d[near_px])
        sel &= bil | (d[near_px] > 0)
        band = sel & (np.abs(rng - z) < trunc)
        quad_px = np.where(inside & (interp != capi.INTERP_NEAREST), dom_px, near_px)  # the dominant tap of a quad
        id_px = np.where(bil, dom_px, near_px)
        key = np.zeros(W * H, np.int64)
        if fr["label"] is not None:
            key += fr["label"].reshape(-1)
        if fr["object_image"] is not None:
            key += fr["object_image"].reshape(-1) == fr["target_id"]
        if fr["mask"] is not None:
            key = key * 2 + (fr["mask"].reshape(-1) != 0)
        split += int((band & (quad_px != id_px) & (key[quad_px] != key[id_px])).sum())
    return split, border


KINDS = ["mle", "mle_color", "compact", "binary"]
INTERPS = {"nearest": capi.INTERP_NEAREST, "bilinear": capi.INTERP_BILINEAR, "adaptive": capi.INTERP_ADAPTIVE}


@pytest.mark.parametrize("vps", [8, 16])
@pytest.mark.parametrize("interp", list(INTERPS))
@pytest.mark.parametrize("kind", KINDS)
def test_depth_quad_taps_bit_identical(oracle_lib, product_lib, kind, interp, vps):
    cam = camera()
    mc, ic = config(kind, INTERPS[interp], vps)
    frs = frames(kind)
    o = hs.make_handle(oracle_lib, "ko_", cam=cam, map_cfg=mc, integ_cfg=ic)
    g = hs.make_handle(product_lib, "kb_", cam=cam, map_cfg=mc, integ_cfg=ic)
    for fr in frs:
        o.integrate_frame(make_frame(o, fr), want_stats=False)
    g.integrate_frames([make_frame(g, fr) for fr in frs], want_stats=False)
    what = f"{kind} {interp} vps{vps}"
    bo, bg = o.export_blocks(), g.export_blocks()
    hs.assert_blocks_equal(bo, bg, exact_float=True, what=what)
    np.testing.assert_array_equal(bo.semantic_likelihoods.view(np.uint32), bg.semantic_likelihoods.view(np.uint32),
                                  err_msg=f"{what} likelihood bits")
    assert o.map_checksum() == g.map_checksum(), what
    assert (bo.semantic_empty == 0).sum() > 500, what  # the semantic path did run
    split, border = tap_counts(bo, frs, cam, mc, ic)
    assert border > 0, what  # voxels on the last column / row are in the scene
    if interp == "adaptive":
        assert split > 0, what  # the fallback to nearest moves the label / mask pixel off the dominant tap
