"""ctypes binding of the C ABI declared in include/khronos_b200.h.

`MapHandle` is a thin, 1:1 wrapper over the C entry points (prefix ``kb_``). The struct layouts
here must match the header exactly. The same class can drive any library exporting the same
entry points under another prefix (the tests use this to drive the CPU oracle with ``ko_``);
the product itself only ever loads ``libkhronos_b200.so``.
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass, field
from typing import Optional

import numpy as np

KB_MAX_LABELS = 64
KB_OK = 0
KB_ERR_NO_DEVICE = 4
KB_ERR_INVALID, KB_ERR_CUDA, KB_ERR_CAPACITY, KB_ERR_STATE = 1, 2, 3, 5
INTERP_NEAREST, INTERP_BILINEAR, INTERP_ADAPTIVE = 0, 1, 2
SEM_NONE, SEM_MLE, SEM_BINARY = 0, 1, 2
MEM_HOST, MEM_DEVICE, MEM_HOST_ASYNC = 0, 1, 2
MASK_LAST_DETECTION = 1  # kb_frame.mask sentinel: reuse the device-resident dynamic image of the last detection
EXPORT_ALL, EXPORT_UPDATED = 0, 1
FLAG_UPDATED, FLAG_MESH_UPDATED, FLAG_ESDF_UPDATED, FLAG_TRACKING_UPDATED, FLAG_HAS_ACTIVE_DATA = 1, 2, 4, 8, 16


class MapConfig(C.Structure):
    _fields_ = [("voxel_size", C.c_float), ("voxels_per_side", C.c_int32),
                ("truncation_distance", C.c_float), ("with_semantics", C.c_int32),
                ("with_tracking", C.c_int32), ("max_blocks", C.c_int32),
                ("max_semantic_blocks", C.c_int32)]


class IntegratorConfig(C.Structure):
    _fields_ = [("use_weight_dropoff", C.c_int32), ("weight_dropoff_epsilon", C.c_float),
                ("use_constant_weight", C.c_int32), ("max_weight", C.c_float),
                ("interpolation_method", C.c_int32), ("adaptive_max_depth_difference", C.c_float),
                ("semantic_mode", C.c_int32), ("num_labels", C.c_int32),
                ("label_confidence", C.c_float), ("label_blocked", C.c_uint8 * KB_MAX_LABELS),
                ("num_threads", C.c_int32)]


class TrackingConfig(C.Structure):
    _fields_ = [("temporal_buffer", C.c_float), ("burn_in_period", C.c_float),
                ("tsdf_occupancy_threshold", C.c_float), ("neighbor_connectivity", C.c_int32),
                ("temporal_window", C.c_float), ("num_threads", C.c_int32)]


class MotionConfig(C.Structure):
    _fields_ = [("neighbor_connectivity", C.c_int32), ("min_cluster_size", C.c_int32),
                ("max_cluster_size", C.c_int32), ("min_separation_distance", C.c_float),
                ("max_range", C.c_float), ("min_z_coordinate", C.c_float),
                ("num_threads", C.c_int32)]


class ObjectDetectorConfig(C.Structure):
    _fields_ = [("use_full_connectivity", C.c_int32), ("min_cluster_size", C.c_int32),
                ("max_cluster_size", C.c_int32), ("use_3d", C.c_int32), ("grid_size", C.c_float),
                ("max_range", C.c_float), ("is_object", C.c_uint8 * KB_MAX_LABELS)]


class InstanceForwardingConfig(C.Structure):
    _fields_ = [("max_range", C.c_float), ("min_cluster_size", C.c_int32), ("max_cluster_size", C.c_int32),
                ("min_object_volume", C.c_double), ("max_object_volume", C.c_double)]


class ShardLayout(C.Structure):
    _fields_ = [("nranks", C.c_int32), ("cell_blocks", C.c_int32), ("grid_x", C.c_int32), ("grid_y", C.c_int32),
                ("table_origin_cx", C.c_int32), ("table_origin_cy", C.c_int32), ("table_width", C.c_int32),
                ("table_height", C.c_int32), ("table", C.c_void_p)]


def frame_owners_host(lib, prefix, cam, voxel_size, vps, frames, nranks, cell_blocks=0, grid=(1, 1), origin=(0, 0), table=None):
    """kb_frame_owners_host / ko_frame_owners_host: owner masks without a handle (no GPU needed)."""
    arr = frames if isinstance(frames, C.Array) else (Frame * len(frames))(*frames)
    t = None if table is None else np.ascontiguousarray(table, np.uint8)
    lay = ShardLayout(nranks, cell_blocks, grid[0], grid[1], int(origin[0]), int(origin[1]), 0 if t is None else t.shape[1],
                      0 if t is None else t.shape[0], None if t is None else t.ctypes.data)
    out = np.zeros(len(arr), np.uint32)
    st = getattr(lib, prefix + "frame_owners_host")(C.byref(cam), C.c_float(voxel_size), vps, C.byref(lay), arr, len(arr), C.c_void_p(out.ctypes.data))
    if st != KB_OK:
        raise KbError(st, "frame_owners_host failed")
    return out


def frame_cells_host(lib, prefix, cam, voxel_size, vps, frames, cell_blocks, origin, width, height):
    """kb_frame_cells_host / ko_frame_cells_host: (n, height, width) touched cells without a handle."""
    arr = frames if isinstance(frames, C.Array) else (Frame * len(frames))(*frames)
    out = np.zeros((len(arr), height, width), np.uint8)
    st = getattr(lib, prefix + "frame_cells_host")(C.byref(cam), C.c_float(voxel_size), vps, arr, len(arr), cell_blocks, int(origin[0]), int(origin[1]),
                                                   width, height, C.c_void_p(out.ctypes.data))
    if st != KB_OK:
        raise KbError(st, "frame_cells_host failed")
    return out


class Camera(C.Structure):
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("fx", C.c_float), ("fy", C.c_float),
                ("cx", C.c_float), ("cy", C.c_float), ("min_range", C.c_float),
                ("max_range", C.c_float)]


class Frame(C.Structure):
    _fields_ = [("depth", C.c_void_p), ("label", C.c_void_p), ("mask", C.c_void_p),
                ("object_image", C.c_void_p), ("color", C.c_void_p), ("vertex_world", C.c_void_p),
                ("world_T_sensor", C.c_double * 16), ("stamp_ns", C.c_uint64),
                ("object_target_id", C.c_int32), ("memory", C.c_int32),
                ("depth_u16", C.c_void_p), ("label_u8", C.c_void_p), ("depth_u16_scale", C.c_float),
                ("reserved_", C.c_int32)]


class FrameStats(C.Structure):
    _fields_ = [(n, C.c_int32) for n in
                ("blocks_in_frustum", "blocks_allocated", "blocks_updated", "voxels_updated",
                 "voxels_in_band", "voxels_semantic", "total_blocks", "capacity_exceeded")]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


class Totals64(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in
                ("blocks_in_frustum", "blocks_allocated", "blocks_updated", "voxels_updated", "voxels_in_band",
                 "voxels_semantic", "block_frame_pairs", "total_blocks", "capacity_exceeded", "frames")]

    def as_dict(self):
        return {n: int(getattr(self, n)) for n, _ in self._fields_}


class BlockExport(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in
                ("block_index", "block_flags", "distance", "weight", "color", "last_observed",
                 "last_occupied", "ever_free", "active", "to_remove", "semantic_label",
                 "semantic_empty", "semantic_likelihoods")]


# ---- defaults mirroring the reference configs ------------------------------------------------------

def default_map_config(voxel_size=0.05, vps=16, trunc=0.15, with_semantics=True, with_tracking=True,
                       max_blocks=4096, max_semantic_blocks=0) -> MapConfig:
    """hydra::VolumetricMap::Config; values of khronos_ros/config/mapper/ground_truth.yaml:63-67."""
    return MapConfig(voxel_size, vps, trunc, int(with_semantics), int(with_tracking), max_blocks,
                     max_semantic_blocks)


def default_integrator_config(semantic_mode=SEM_MLE, num_labels=20, blocked=(), num_threads=-1,
                              interpolation=INTERP_ADAPTIVE) -> IntegratorConfig:
    """hydra::ProjectiveIntegrator::Config defaults (SURVEY.md Appendix A.4)."""
    c = IntegratorConfig()
    c.use_weight_dropoff = 1
    c.weight_dropoff_epsilon = -1.0
    c.use_constant_weight = 0
    c.max_weight = 1e5
    c.interpolation_method = interpolation
    c.adaptive_max_depth_difference = 0.2
    c.semantic_mode = semantic_mode
    c.num_labels = num_labels if semantic_mode == SEM_MLE else (2 if semantic_mode == SEM_BINARY else 0)
    c.label_confidence = 0.9
    for b in blocked:
        c.label_blocked[b] = 1
    c.num_threads = num_threads
    return c


def default_tracking_config(num_threads=-1) -> TrackingConfig:
    """khronos::TrackingIntegrator::Config defaults (tracking_integrator.h:59-83)."""
    return TrackingConfig(1.0, 1.0, -1.5, 18, 3.0, num_threads)


def default_motion_config(num_threads=-1, min_cluster_size=0, max_cluster_size=1000000,
                          min_separation_distance=1.0, connectivity=26) -> MotionConfig:
    """khronos::FreeSpaceMotionDetector::Config defaults (free_space_motion_detector.h:70-95)."""
    return MotionConfig(connectivity, min_cluster_size, max_cluster_size, min_separation_distance,
                        10000.0, -10000.0, num_threads)


def default_object_detector_config(object_labels=(), use_3d=True, min_cluster_size=0, max_cluster_size=-1,
                                   use_full_connectivity=True, grid_size=0.1, max_range=0.0) -> ObjectDetectorConfig:
    """khronos::ConnectedSemantics::Config defaults (object_detection/connected_semantics.h:64-84)."""
    c = ObjectDetectorConfig(int(use_full_connectivity), min_cluster_size, max_cluster_size, int(use_3d), grid_size, max_range)
    for l in object_labels:
        c.is_object[l] = 1
    return c


class KbError(RuntimeError):
    def __init__(self, status, msg):
        super().__init__(f"status {status}: {msg}")
        self.status = status


def _ptr(a) -> Optional[int]:
    """Address of a numpy array (host) / torch tensor (device or host) / raw int, or None."""
    if a is None:
        return None
    if isinstance(a, int):
        return a
    if isinstance(a, np.ndarray):
        assert a.flags["C_CONTIGUOUS"]
        return a.ctypes.data
    if hasattr(a, "data_ptr"):
        assert a.is_contiguous()
        return a.data_ptr()
    raise TypeError(type(a))


@dataclass
class Blocks:
    """Host copy of exported blocks (sorted by block index x,y,z)."""
    block_index: np.ndarray
    block_flags: np.ndarray
    distance: np.ndarray
    weight: np.ndarray
    last_observed: np.ndarray
    last_occupied: np.ndarray
    ever_free: np.ndarray
    active: np.ndarray
    to_remove: np.ndarray
    semantic_label: np.ndarray
    semantic_empty: np.ndarray
    semantic_likelihoods: Optional[np.ndarray] = None
    color: Optional[np.ndarray] = None  # (n, V, 3) u8 TsdfVoxel::color (rgb)
    extra: dict = field(default_factory=dict)

    @property
    def n(self):
        return int(self.block_index.shape[0])


class MapHandle:
    """One volumetric map + integrators behind the C ABI (see include/khronos_b200.h)."""

    def __init__(self, lib: C.CDLL, prefix: str, map_cfg: MapConfig, integ_cfg: IntegratorConfig,
                 tracking_cfg: Optional[TrackingConfig] = None,
                 motion_cfg: Optional[MotionConfig] = None, device: int = 0):
        self._lib, self._p = lib, prefix
        self.map_cfg, self.integ_cfg = map_cfg, integ_cfg
        self.V = map_cfg.voxels_per_side ** 3
        self.L = 0
        if map_cfg.with_semantics:
            self.L = {SEM_MLE: integ_cfg.num_labels, SEM_BINARY: 2}.get(integ_cfg.semantic_mode, 0)
        self._h = C.c_void_p()
        self._camera = None
        st = self._fn("create")(C.byref(map_cfg), C.byref(integ_cfg),
                                C.byref(tracking_cfg) if tracking_cfg else None,
                                C.byref(motion_cfg) if motion_cfg else None, device, C.byref(self._h))
        if st != KB_OK:
            self._h = C.c_void_p()
            raise KbError(st, "create failed (no CUDA device?)" if st == KB_ERR_NO_DEVICE else "create failed")

    def _fn(self, name):
        f = getattr(self._lib, self._p + name)
        f.restype = C.c_int
        return f

    def _check(self, st):
        if st != KB_OK:
            e = getattr(self._lib, self._p + "last_error")
            e.restype = C.c_char_p
            raise KbError(st, (e(self._h) or b"").decode())

    def close(self):
        if self._h:
            self._fn("destroy")(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- configuration
    def set_camera(self, cam: Camera):
        self._camera = cam
        self._check(self._fn("set_camera")(self._h, C.byref(cam)))

    def set_stream(self, cuda_stream: int):
        self._check(self._fn("set_stream")(self._h, C.c_void_p(cuda_stream)))

    def synchronize(self):
        self._check(self._fn("synchronize")(self._h))

    def set_shard(self, rank: int, nranks: int):
        self._check(self._fn("set_shard")(self._h, rank, nranks))

    # ---- hot path
    def set_shard_cells(self, rank: int, nranks: int, cell_blocks: int, grid_x: int, grid_y: int):
        self._check(self._fn("set_shard_cells")(self._h, rank, nranks, cell_blocks, grid_x, grid_y))

    def set_shard_table(self, rank: int, nranks: int, cell_blocks: int, origin, table: np.ndarray):
        """kb_set_shard_table: table[cy, cx] (uint8, shape (height, width)) = rank of cell (origin[0] + cx, origin[1] + cy)."""
        t = np.ascontiguousarray(table, np.uint8)
        self._check(self._fn("set_shard_table")(self._h, rank, nranks, cell_blocks, int(origin[0]), int(origin[1]), int(t.shape[1]), int(t.shape[0]),
                                                C.c_void_p(t.ctypes.data)))

    def frame_cells(self, frames, cell_blocks: int, origin, width: int, height: int) -> np.ndarray:
        """kb_frame_cells: (n_frames, height, width) uint8, 1 where the frame's frustum selection touches the cell."""
        arr = frames if isinstance(frames, C.Array) else (Frame * len(frames))(*frames)
        out = np.zeros((len(arr), height, width), np.uint8)
        self._check(self._fn("frame_cells")(self._h, arr, len(arr), cell_blocks, int(origin[0]), int(origin[1]), width, height, C.c_void_p(out.ctypes.data)))
        return out

    def frame_owners(self, frames) -> np.ndarray:
        """Bit mask of the ranks that need each frame (kb_frame_owners)."""
        arr = frames if isinstance(frames, C.Array) else (Frame * len(frames))(*frames)
        out = np.zeros(len(arr), np.uint32)
        self._check(self._fn("frame_owners")(self._h, arr, len(arr), C.c_void_p(out.ctypes.data)))
        return out

    @staticmethod
    def make_frame(depth, pose, stamp_ns, label=None, mask=None, object_image=None, color=None,
                   vertex_world=None, target_id=0, memory=MEM_HOST, depth_u16=None, label_u8=None,
                   depth_u16_scale=0.001) -> Frame:
        f = Frame()
        f.depth, f.label, f.mask = _ptr(depth), _ptr(label), _ptr(mask)
        f.depth_u16, f.label_u8, f.depth_u16_scale = _ptr(depth_u16), _ptr(label_u8), depth_u16_scale
        f.object_image, f.color, f.vertex_world = _ptr(object_image), _ptr(color), _ptr(vertex_world)
        T = np.asarray(pose, dtype=np.float64).reshape(16)
        for i in range(16):
            f.world_T_sensor[i] = float(T[i])
        f.stamp_ns = int(stamp_ns)
        f.object_target_id = int(target_id)
        f.memory = memory
        f._keep = (depth, label, mask, object_image, color, vertex_world, depth_u16, label_u8)  # keep buffers alive
        return f

    def integrate_frame(self, frame: Frame, allocate_blocks=True, want_stats=True):
        stats = FrameStats()
        self._check(self._fn("integrate_frame")(self._h, C.byref(frame), int(allocate_blocks),
                                                C.byref(stats) if want_stats else None))
        return stats if want_stats else None

    def integrate_frames(self, frames, allocate_blocks=True, want_stats=True):
        """kb_integrate_frames: identical to integrating the frames one by one, fused on the GPU."""
        arr = (Frame * len(frames))(*frames)
        arr._keep = frames
        stats = FrameStats()
        self._check(self._fn("integrate_frames")(self._h, arr, len(frames), int(allocate_blocks),
                                                 C.byref(stats) if want_stats else None))
        return stats if want_stats else None

    def get_debug_counters(self, n=24) -> np.ndarray:
        out = np.zeros(n, np.int32)
        self._check(self._fn("get_debug_counters")(self._h, C.c_void_p(out.ctypes.data), n))
        return out

    def set_culling(self, enabled):
        """0 = off, 1/True = default (calls with >= 4 frames), 2 = always."""
        self._check(self._fn("set_culling")(self._h, int(enabled)))

    def get_totals(self) -> FrameStats:
        t = FrameStats()
        self._check(self._fn("get_totals")(self._h, C.byref(t)))
        return t

    def get_totals64(self) -> Totals64:
        """Cumulative counters since creation in 64 bits (never wrap)."""
        t = Totals64()
        self._check(self._fn("get_totals64")(self._h, C.byref(t)))
        return t

    def map_checksum(self):
        """(sum, xor, blocks, observed voxels): order-independent checksum of the whole map (kb_map_checksum)."""
        out = (C.c_uint64 * 4)()
        self._check(self._fn("map_checksum")(self._h, out))
        return tuple(int(x) for x in out)

    def update_tracking(self, stamp_ns: int):
        self._check(self._fn("update_tracking")(self._h, C.c_uint64(int(stamp_ns))))

    def reset_inactive(self, max_removed=1 << 20) -> np.ndarray:
        n = C.c_int32(0)
        buf = np.zeros((max_removed, 3), np.int32)
        self._check(self._fn("reset_inactive")(self._h, C.c_void_p(buf.ctypes.data), max_removed, C.byref(n)))
        return buf[: n.value].copy()

    def mark_all_inactive(self):
        self._check(self._fn("mark_all_inactive")(self._h))

    def clear_updated(self):
        self._check(self._fn("clear_updated")(self._h))

    def detect_motion(self, frame: Frame):
        H, W = self._camera.height, self._camera.width
        img = np.zeros((H, W), np.int32)
        ns, nc = C.c_int32(0), C.c_int32(0)
        self._check(self._fn("detect_motion")(self._h, C.byref(frame), C.c_void_p(img.ctypes.data),
                                              C.byref(ns), C.byref(nc)))
        self._last_nc = nc.value
        return img, ns.value, nc.value

    def spin_once(self, frame: Frame, want_image=True):
        """kb_spin_once: detect -> integrate(mask) -> track with one host round trip."""
        H, W = self._camera.height, self._camera.width
        img = np.zeros((H, W), np.int32) if want_image else None
        ns, nc = C.c_int32(0), C.c_int32(0)
        self._check(self._fn("spin_once")(self._h, C.byref(frame), C.c_void_p(img.ctypes.data) if want_image else None,
                                          C.byref(ns), C.byref(nc)))
        self._last_nc = nc.value
        return img, ns.value, nc.value

    # ---- sharded per-frame pipeline (include/khronos_b200.h "sharded per-frame pipeline"); buffers are torch
    # tensors / raw pointers in the library's memory space (device for the product)
    def set_shard_capacity(self, pending_capacity: int, halo_capacity: int):
        self._check(self._fn("set_shard_capacity")(self._h, int(pending_capacity), int(halo_capacity)))

    def shard_buffer_sizes(self):
        a, b, c = C.c_int64(0), C.c_int64(0), C.c_int64(0)
        self._check(self._fn("shard_buffer_sizes")(self._h, C.byref(a), C.byref(b), C.byref(c)))
        return a.value, b.value, c.value

    def tracking_begin(self, stamp_ns: int, pending_out):
        self._check(self._fn("tracking_begin")(self._h, C.c_uint64(int(stamp_ns)), C.c_void_p(_ptr(pending_out))))

    def tracking_pack_halo(self, all_pending, halo_out):
        self._check(self._fn("tracking_pack_halo")(self._h, C.c_void_p(_ptr(all_pending)), C.c_void_p(_ptr(halo_out))))

    def tracking_finish(self, all_pending, all_halo):
        self._check(self._fn("tracking_finish")(self._h, C.c_void_p(_ptr(all_pending)), C.c_void_p(_ptr(all_halo))))

    @staticmethod
    def _ptr_array(bufs):
        arr = (C.c_void_p * len(bufs))(*[_ptr(b) for b in bufs])
        return arr

    def tracking_begin_peers(self, stamp_ns: int, peer_all_pending):
        arr = self._ptr_array(peer_all_pending)
        self._check(self._fn("tracking_begin_peers")(self._h, C.c_uint64(int(stamp_ns)), arr, len(peer_all_pending)))

    def tracking_pack_halo_peers(self, all_pending, peer_all_halo):
        arr = self._ptr_array(peer_all_halo)
        self._check(self._fn("tracking_pack_halo_peers")(self._h, C.c_void_p(_ptr(all_pending)), arr, len(peer_all_halo)))

    def motion_lookup_peers(self, frame: Frame, peer_flags):
        arr = self._ptr_array(peer_flags)
        self._check(self._fn("motion_lookup_peers")(self._h, C.byref(frame), arr, len(peer_flags)))

    def motion_lookup_local(self, frame: Frame, pixel_flags):
        self._check(self._fn("motion_lookup_local")(self._h, C.byref(frame), C.c_void_p(_ptr(pixel_flags))))

    def motion_cluster_global(self, pixel_flags):
        self._check(self._fn("motion_cluster_global")(self._h, C.c_void_p(_ptr(pixel_flags))))

    def motion_result(self, want_image=True):
        H, W = self._camera.height, self._camera.width
        img = np.zeros((H, W), np.int32) if want_image else None
        ns, nc = C.c_int32(0), C.c_int32(0)
        self._check(self._fn("motion_result")(self._h, C.c_void_p(img.ctypes.data) if want_image else None,
                                              C.byref(ns), C.byref(nc)))
        self._last_nc = nc.value
        return img, ns.value, nc.value

    def get_motion_clusters(self):
        tp, tv = C.c_int32(0), C.c_int32(0)
        f = self._fn("get_motion_clusters")
        self._check(f(self._h, None, None, None, None, C.byref(tp), C.byref(tv)))
        nc = getattr(self, "_last_nc", 0)
        counts = np.zeros((max(nc, 1), 2), np.int32)
        px = np.zeros((max(tp.value, 1), 2), np.int32)
        vx = np.zeros((max(tv.value, 1), 3), np.int64)
        bb = np.zeros((counts.shape[0], 6), np.float32)
        self._check(f(self._h, C.c_void_p(counts.ctypes.data), C.c_void_p(px.ctypes.data),
                      C.c_void_p(vx.ctypes.data), C.c_void_p(bb.ctypes.data), C.byref(tp), C.byref(tv)))
        out, po, vo = [], 0, 0
        for c in range(nc):
            npx, nvx = int(counts[c, 0]), int(counts[c, 1])
            out.append({"pixels": px[po:po + npx].copy(), "voxels": vx[vo:vo + nvx].copy(),
                        "bbox": bb[c].copy()})
            po += npx
            vo += nvx
        return out

    def detect_objects(self, cfg: ObjectDetectorConfig, frame: Frame):
        """kb_detect_objects: returns (object image H x W int32, number of clusters)."""
        H, W = self._camera.height, self._camera.width
        img = np.zeros((H, W), np.int32)
        nc = C.c_int32(0)
        self._check(self._fn("detect_objects")(self._h, C.byref(cfg), C.byref(frame), C.c_void_p(img.ctypes.data), C.byref(nc)))
        return img, nc.value

    def forward_instances(self, frame: Frame, max_range=0.0, min_cluster_size=0, max_cluster_size=-1, min_object_volume=0.0,
                          max_object_volume=-1.0, background=None):
        """kb_forward_instances (khronos::InstanceForwarding): returns (object image, clusters) with clusters =
        [{"id", "pixels" (n, 2) in the reference's scan order, "bbox" (6,)}], ascending id."""
        H, W = self._camera.height, self._camera.width
        cfg = InstanceForwardingConfig(max_range, min_cluster_size, max_cluster_size, min_object_volume, max_object_volume)
        img = np.zeros((H, W), np.int32)
        nc = C.c_int32(0)
        bg = None if background is None else np.ascontiguousarray(background, np.uint8)
        self._check(self._fn("forward_instances")(self._h, C.byref(cfg), C.byref(frame), None if bg is None else C.c_void_p(bg.ctypes.data),
                                                  0 if bg is None else int(bg.size), C.c_void_p(img.ctypes.data), C.byref(nc)))
        n, tp = C.c_int32(0), C.c_int32(0)
        f = self._fn("get_instance_clusters")
        self._check(f(self._h, None, None, None, C.byref(n), C.byref(tp)))
        info = np.zeros((max(n.value, 1), 2), np.int32)
        bbox = np.zeros((max(n.value, 1), 6), np.float32)
        px = np.zeros((max(tp.value, 1), 2), np.int32)
        self._check(f(self._h, C.c_void_p(info.ctypes.data), C.c_void_p(bbox.ctypes.data), C.c_void_p(px.ctypes.data), C.byref(n), C.byref(tp)))
        out, po = [], 0
        for c in range(n.value):
            k = int(info[c, 1])
            out.append({"id": int(info[c, 0]), "pixels": px[po:po + k].copy(), "bbox": bbox[c].copy()})
            po += k
        return img, out

    def get_object_clusters(self):
        f = self._fn("get_object_clusters")
        nc, tp = C.c_int32(0), C.c_int32(0)
        self._check(f(self._h, None, None, C.byref(nc), C.byref(tp)))
        info = np.zeros((max(nc.value, 1), 3), np.int32)
        px = np.zeros((max(tp.value, 1), 2), np.int32)
        self._check(f(self._h, C.c_void_p(info.ctypes.data), C.c_void_p(px.ctypes.data), C.byref(nc), C.byref(tp)))
        out, po = [], 0
        for c in range(nc.value):
            n = int(info[c, 2])
            out.append({"id": int(info[c, 0]), "semantic_id": int(info[c, 1]), "pixels": px[po:po + n].copy()})
            po += n
        return out

    def compute_vertex_map(self, frame: Frame, out_ptr=None):
        """kb_compute_vertex_map: (H, W, 3) float32 world-frame vertex map (host frames), or written to the device pointer
        out_ptr for MEM_DEVICE frames."""
        if out_ptr is not None:
            self._check(self._fn("compute_vertex_map")(self._h, C.byref(frame), C.c_void_p(out_ptr)))
            return None
        out = np.zeros((self._camera.height, self._camera.width, 3), np.float32)
        self._check(self._fn("compute_vertex_map")(self._h, C.byref(frame), C.c_void_p(out.ctypes.data)))
        return out

    def track_measurements(self, frame: Frame, id_image, clusters, voxel_size: float = 0.1, tracks=()):
        """kb_track_measurements (MaxIoUTracker, track_by = voxels). id_image: H x W int32 host array for host frames, or a device pointer (int) for
        MEM_DEVICE frames. clusters: n (pixel values 1..n) or an ascending list of pixel values. tracks: sequence of
        (n_i, 3) int64 arrays (Track::last_voxels). Returns a dict with voxel_counts [n], voxel_sums [n, 3],
        intersections / iou [n, n_tracks]."""
        if isinstance(id_image, int):  # raw pointer (device image of a MEM_DEVICE frame)
            ids_ptr = C.c_void_p(id_image)
        else:
            ids = np.ascontiguousarray(id_image, np.int32)
            ids_ptr = C.c_void_p(ids.ctypes.data)
        if isinstance(clusters, (int, np.integer)):   # pixel values 1..clusters
            max_id, cid_ptr = int(clusters), None
        else:                                          # ascending list of pixel values
            cids = np.ascontiguousarray(clusters, np.int32)
            max_id, cid_ptr = len(cids), C.c_void_p(cids.ctypes.data)
        tracks = [np.ascontiguousarray(t, np.int64).reshape(-1, 3) for t in tracks]
        nt = len(tracks)
        offsets = np.zeros(nt + 1, np.int32)
        for i, t in enumerate(tracks):
            offsets[i + 1] = offsets[i] + len(t)
        flat = np.concatenate(tracks) if nt and offsets[-1] > 0 else np.zeros((1, 3), np.int64)
        flat = np.ascontiguousarray(flat)
        counts = np.zeros(max_id, np.int32)
        sums = np.zeros((max_id, 3), np.int64)
        inter = np.zeros((max_id, max(nt, 1)), np.int32)
        iou = np.zeros((max_id, max(nt, 1)), np.float32)
        self._check(self._fn("track_measurements")(
            self._h, C.byref(frame), ids_ptr, C.c_int32(max_id), cid_ptr, C.c_float(voxel_size), C.c_int32(nt),
            C.c_void_p(offsets.ctypes.data) if nt else None, C.c_void_p(flat.ctypes.data) if nt else None,
            C.c_void_p(counts.ctypes.data), C.c_void_p(sums.ctypes.data),
            C.c_void_p(inter.ctypes.data) if nt else None, C.c_void_p(iou.ctypes.data) if nt else None))
        return {"voxel_counts": counts, "voxel_sums": sums, "intersections": inter[:, :nt], "iou": iou[:, :nt]}

    def get_cluster_voxels(self, max_id: int):
        """kb_get_cluster_voxels: list of (n_c, 3) int64 arrays, one per id 1..max_id of the last track_measurements
        call, voxels ascending in (z, y, x)."""
        f = self._fn("get_cluster_voxels")
        total = C.c_int32(0)
        offsets = np.zeros(max_id + 1, np.int32)
        self._check(f(self._h, C.c_void_p(offsets.ctypes.data), None, 0, C.byref(total)))
        vox = np.zeros((max(total.value, 1), 3), np.int64)
        self._check(f(self._h, C.c_void_p(offsets.ctypes.data), C.c_void_p(vox.ctypes.data), C.c_int32(total.value), C.byref(total)))
        return [vox[offsets[i]:offsets[i + 1]].copy() for i in range(max_id)]

    def generate_mesh(self, only_mesh_updated=True, clear_updated_flag=True, min_weight=1e-4):
        """hydra::MeshIntegrator::generateMesh on the map; returns (block_index (n,3), vertex offsets (n+1,), points (nv,3) f32,
        colors (nv,3) u8, labels (nv,) u32); triangle k = vertices 3k..3k+2."""
        nb, nv = C.c_int32(0), C.c_int64(0)
        self._check(self._fn("generate_mesh")(self._h, int(only_mesh_updated), int(clear_updated_flag), C.c_float(min_weight),
                                              C.byref(nb), C.byref(nv)))
        n, v = nb.value, nv.value
        bi = np.zeros((n, 3), np.int32)
        off = np.zeros(n + 1, np.int64)
        pts = np.zeros((v, 3), np.float32)
        col = np.zeros((v, 3), np.uint8)
        lab = np.zeros(v, np.uint32)
        self._check(self._fn("get_mesh")(self._h, C.c_void_p(bi.ctypes.data), C.c_void_p(off.ctypes.data), C.c_void_p(pts.ctypes.data),
                                         C.c_void_p(col.ctypes.data), C.c_void_p(lab.ctypes.data), C.c_int64(v)))
        return bi, off, pts, col, lab

    def allocate_box(self, mn, mx):
        a = (C.c_int32 * 3)(*[int(v) for v in mn])
        b = (C.c_int32 * 3)(*[int(v) for v in mx])
        self._check(self._fn("allocate_box")(self._h, a, b))

    def scan_object_confidence(self, min_confidence=0.5, min_observations=10) -> int:
        n = C.c_int32(0)
        self._check(self._fn("scan_object_confidence")(self._h, C.c_float(min_confidence),
                                                       int(min_observations), C.byref(n)))
        return n.value

    # ---- export
    def num_blocks(self, which=EXPORT_ALL) -> int:
        n = C.c_int32(0)
        self._check(self._fn("num_blocks")(self._h, which, C.byref(n)))
        return n.value

    def export_blocks(self, which=EXPORT_ALL, likelihoods=True) -> Blocks:
        n, V, L = self.num_blocks(which), self.V, self.L
        b = Blocks(
            block_index=np.zeros((n, 3), np.int32), block_flags=np.zeros(n, np.uint8),
            distance=np.zeros((n, V), np.float32), weight=np.zeros((n, V), np.float32),
            last_observed=np.zeros((n, V), np.uint64), last_occupied=np.zeros((n, V), np.uint64),
            ever_free=np.zeros((n, V), np.uint8), active=np.zeros((n, V), np.uint8),
            to_remove=np.zeros((n, V), np.uint8), semantic_label=np.zeros((n, V), np.uint32),
            semantic_empty=np.ones((n, V), np.uint8),
            semantic_likelihoods=np.zeros((n, V, L), np.float32) if (likelihoods and L > 0) else None,
            color=np.zeros((n, V, 3), np.uint8))
        ex = BlockExport()
        for name, _ in BlockExport._fields_:
            arr = getattr(b, name, None)
            setattr(ex, name, arr.ctypes.data if isinstance(arr, np.ndarray) and arr.size else None)
        nw = C.c_int32(0)
        if n:
            self._check(self._fn("export_blocks")(self._h, which, n, C.byref(ex), C.byref(nw)))
            assert nw.value == n
        return b


def load_product_library() -> C.CDLL:
    """Load the in-tree CUDA product library. Fails loudly if it is missing: there is no fallback."""
    here = os.path.dirname(os.path.abspath(__file__))
    variant = os.environ.get("KB_PRODUCT_LIB_VARIANT")  # tuning builds (khronos_b200/build.py VARIANTS), A/B runs only
    path = os.path.join(here, "csrc", f"libkhronos_b200_{variant}.so" if variant else "libkhronos_b200.so")
    if not os.path.exists(path):
        raise ImportError(
            f"{path} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). khronos_b200 has no CPU fallback.")
    return C.CDLL(path, mode=C.RTLD_GLOBAL)


# ---- ray index (khronos::RayVerificator; include/khronos_b200.h "ray index") --------------------------------------------
class RayConfig(C.Structure):
    _fields_ = [("block_size", C.c_float), ("radial_tolerance", C.c_float), ("depth_tolerance", C.c_float)]


def default_ray_config(block_size=1.0, radial_tolerance=0.1, depth_tolerance=0.1) -> RayConfig:
    """RayVerificator::Config defaults (ray_verificator.h:68-100)."""
    return RayConfig(block_size, radial_tolerance, depth_tolerance)


RAYS_FIRST, RAYS_LAST, RAYS_FIRST_AND_LAST, RAYS_MIDDLE, RAYS_ALL = range(5)


class RayIndex:
    """kb_rays_* (product, prefix "kb_") or ko_rays_* (oracle, prefix "ko_") through ctypes."""

    def __init__(self, lib, prefix, cfg: RayConfig, device=0):
        self._lib, self._p, self._h = lib, prefix, C.c_void_p()
        st = self._fn("create")(C.byref(cfg), device, C.byref(self._h))
        if st != KB_OK:
            self._h = C.c_void_p()
            raise KbError(st, "rays_create failed (no CUDA device?)" if st == KB_ERR_NO_DEVICE else "rays_create failed")

    def _fn(self, name):
        f = getattr(self._lib, self._p + "rays_" + name)
        f.restype = C.c_int
        return f

    def _check(self, st):
        if st != KB_OK:
            e = getattr(self._lib, self._p + "rays_last_error")
            e.restype = C.c_char_p
            raise KbError(st, (e(self._h) or b"").decode())

    def close(self):
        if self._h:
            self._fn("destroy")(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def clear(self):
        self._check(self._fn("clear")(self._h))

    def size(self):
        n, e = C.c_int32(0), C.c_int64(0)
        self._check(self._fn("size")(self._h, C.byref(n), C.byref(e)))
        return n.value, e.value

    def add(self, sources, targets, stamps, want_observed=True):
        """Adds rays; returns the (k, 3) int32 array of blocks the new rays pass through (ascending z, y, x)."""
        s = np.ascontiguousarray(sources, np.float32).reshape(-1, 3)
        t = np.ascontiguousarray(targets, np.float32).reshape(-1, 3)
        ts = np.ascontiguousarray(stamps, np.uint64)
        n = len(s)
        f = self._fn("add")
        if not want_observed:
            self._check(f(self._h, n, C.c_void_p(s.ctypes.data), C.c_void_p(t.ctypes.data), C.c_void_p(ts.ctypes.data), None, 0, None))
            return None
        cap, nobs = 64, C.c_int32(0)
        while True:
            obs = np.zeros((cap, 3), np.int32)
            st = f(self._h, n, C.c_void_p(s.ctypes.data), C.c_void_p(t.ctypes.data), C.c_void_p(ts.ctypes.data),
                   C.c_void_p(obs.ctypes.data), cap, C.byref(nobs))
            if st == KB_ERR_CAPACITY and nobs.value > cap:
                cap = nobs.value
                continue
            self._check(st)
            return obs[:nobs.value].copy()

    def add_vertices(self, policy, pose_stamps, pose_positions, vertices, first_seen, last_seen, vertex_index_base=0,
                     active_window_duration=0.0):
        """kb_rays_add_vertices; returns (observed blocks (k, 3), number of rays added)."""
        ps = np.ascontiguousarray(pose_stamps, np.uint64)
        pp = np.ascontiguousarray(pose_positions, np.float32).reshape(-1, 3)
        vx = np.ascontiguousarray(vertices, np.float32).reshape(-1, 3)
        fs, ls = np.ascontiguousarray(first_seen, np.uint64), np.ascontiguousarray(last_seen, np.uint64)
        f = self._fn("add_vertices")
        cap, nobs, nadd = 256, C.c_int32(0), C.c_int32(0)
        while True:
            obs = np.zeros((cap, 3), np.int32)
            st = f(self._h, int(policy), C.c_float(active_window_duration), len(ps), C.c_void_p(ps.ctypes.data), C.c_void_p(pp.ctypes.data),
                   len(vx), int(vertex_index_base), C.c_void_p(vx.ctypes.data), C.c_void_p(fs.ctypes.data), C.c_void_p(ls.ctypes.data),
                   C.c_void_p(obs.ctypes.data), cap, C.byref(nobs), C.byref(nadd))
            if st == KB_ERR_CAPACITY and nobs.value > cap:
                cap = nobs.value
                continue
            self._check(st)
            return obs[:nobs.value].copy(), nadd.value

    def ray_ids(self):
        n, _ = self.size()
        pose, vert, ts = np.zeros(max(n, 1), np.int32), np.zeros(max(n, 1), np.int32), np.zeros(max(n, 1), np.uint64)
        self._check(self._fn("get_ray_ids")(self._h, C.c_void_p(pose.ctypes.data), C.c_void_p(vert.ctypes.data), C.c_void_p(ts.ctypes.data), n))
        return pose[:n], vert[:n], ts[:n]

    def set_endpoints(self, sources, targets):
        s = np.ascontiguousarray(sources, np.float32).reshape(-1, 3)
        t = np.ascontiguousarray(targets, np.float32).reshape(-1, 3)
        self._check(self._fn("set_endpoints")(self._h, len(s), C.c_void_p(s.ctypes.data), C.c_void_p(t.ctypes.data)))

    def rehash(self):
        self._check(self._fn("rehash")(self._h))

    def check(self, points, earliest=0, latest=2**64 - 1):
        """Returns (counts (n, 2) int32 [absent, present], list of (absent stamps, present stamps) per point)."""
        p = np.ascontiguousarray(points, np.float32).reshape(-1, 3)
        n = len(p)
        lo = np.ascontiguousarray(np.broadcast_to(np.asarray(earliest, np.uint64), (n,)))
        hi = np.ascontiguousarray(np.broadcast_to(np.asarray(latest, np.uint64), (n,)))
        counts = np.zeros((max(n, 1), 2), np.int32)
        total = C.c_int64(0)
        self._check(self._fn("check")(self._h, n, C.c_void_p(p.ctypes.data), C.c_void_p(lo.ctypes.data), C.c_void_p(hi.ctypes.data),
                                      C.c_void_p(counts.ctypes.data), C.byref(total)))
        stamps = np.zeros(max(total.value, 1), np.uint64)
        self._check(self._fn("get_stamps")(self._h, C.c_void_p(stamps.ctypes.data), C.c_int64(total.value)))
        out, o = [], 0
        for i in range(n):
            a, b = int(counts[i, 0]), int(counts[i, 1])
            out.append((stamps[o:o + a].copy(), stamps[o + a:o + a + b].copy()))
            o += a + b
        return counts[:n], out
