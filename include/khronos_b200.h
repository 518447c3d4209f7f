/*
 * khronos_b200.h — C ABI of the H100-native active-window volumetric integrator.
 *
 * This is the drop-in boundary for Khronos' per-frame active-window fusion hot path. Every entry
 * point cites the reference interface it replaces (paths relative to the Khronos checkout;
 * "UP" = upstream MIT-SPARK/Hydra, which Khronos only calls / subclasses).
 *
 * Conventions
 *   - extern "C", plain pointers and sizes, no C++/torch types. Every function returns a kb_status
 *     (0 = ok) and never throws across the ABI; kb_last_error() gives a message for the handle.
 *   - A handle owns all device memory of one volumetric map (TSDF + tracking + semantic layers over
 *     an open-addressed GPU block hash) and one CUDA stream. Calls on one handle are serialised by
 *     the caller (the reference holds mutex_, khronos/src/active_window/active_window.cpp:119);
 *     different handles are fully concurrent (extraction workers own private maps,
 *     khronos/src/active_window/object_extraction/object_worker_pool.cpp:130).
 *   - Input pointers are borrowed for the duration of the call. kb_frame.memory says whether image
 *     pointers are host (pageable or pinned) or device pointers. Outputs are caller-allocated.
 *   - Images are row-major H x W like cv::Mat (depth CV_32FC1, label/mask/object CV_32SC1,
 *     vertex CV_32FC3, color CV_8UC3).
 *   - There is NO CPU fallback: kb_create fails with KB_ERR_NO_DEVICE if no CUDA device exists.
 */
#ifndef KHRONOS_B200_H_
#define KHRONOS_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define KB_ABI_VERSION 8

typedef enum kb_status {
  KB_OK = 0,
  KB_ERR_INVALID = 1,    /* invalid argument / configuration (reference: config::checkValid aborts) */
  KB_ERR_CUDA = 2,       /* CUDA runtime error */
  KB_ERR_CAPACITY = 3,   /* block pool / hash table / semantic pool exhausted */
  KB_ERR_NO_DEVICE = 4,  /* no usable CUDA device: the product path refuses to run */
  KB_ERR_STATE = 5       /* call order violated (e.g. non-monotonic stamps) */
} kb_status;

typedef struct kb_handle kb_handle;

/* hydra::VolumetricMap::Config (UP; fields as used at
 * khronos/src/active_window/object_extraction/mesh_object_extractor.cpp:201-211) + pool sizing. */
typedef struct kb_map_config {
  float voxel_size;           /* metres */
  int32_t voxels_per_side;    /* 8 or 16 */
  float truncation_distance;  /* metres */
  int32_t with_semantics;
  int32_t with_tracking;
  int32_t max_blocks;           /* capacity of the device block pool */
  int32_t max_semantic_blocks;  /* capacity of the lazily assigned semantic pool (0 => max_blocks) */
} kb_map_config;

enum { KB_INTERP_NEAREST = 0, KB_INTERP_BILINEAR = 1, KB_INTERP_ADAPTIVE = 2 };
enum { KB_SEMANTICS_NONE = 0, KB_SEMANTICS_MLE = 1, KB_SEMANTICS_BINARY = 2 };
#define KB_MAX_LABELS 64

/* hydra::ProjectiveIntegrator::Config (UP; Khronos only sets num_threads,
 * khronos_ros/config/mapper/uHumans2.yaml:80-81) + the semantic integrator choice
 * (khronos/src/active_window/integration/object_integrator.cpp:44-48 forces BINARY). */
typedef struct kb_integrator_config {
  int32_t use_weight_dropoff;     /* default 1 */
  float weight_dropoff_epsilon;   /* default -1 (negative => multiple of voxel size) */
  int32_t use_constant_weight;    /* default 0 */
  float max_weight;               /* default 1e5 */
  int32_t interpolation_method;   /* default KB_INTERP_ADAPTIVE */
  float adaptive_max_depth_difference; /* bilinear only if max-min of the 4 taps < this; default 0.2 */
  int32_t semantic_mode;          /* KB_SEMANTICS_* */
  int32_t num_labels;             /* MLE: total labels N (<= KB_MAX_LABELS) */
  float label_confidence;         /* MLE: default 0.9 */
  uint8_t label_blocked[KB_MAX_LABELS]; /* MLE: 1 => label is dynamic/invalid: canIntegrate false */
  int32_t num_threads;            /* CPU oracle only; ignored by the GPU product */
} kb_integrator_config;

/* khronos::TrackingIntegrator::Config,
 * khronos/include/khronos/active_window/integration/tracking_integrator.h:59-83 */
typedef struct kb_tracking_config {
  float temporal_buffer;           /* s, default 1 */
  float burn_in_period;            /* s, default 1 (declared but unused by the reference) */
  float tsdf_occupancy_threshold;  /* m; negative => multiple of voxel size; default -1.5 */
  int32_t neighbor_connectivity;   /* 6 | 18 | 26, default 18 */
  float temporal_window;           /* s, default 3 */
  int32_t num_threads;             /* CPU oracle only */
} kb_tracking_config;

/* khronos::FreeSpaceMotionDetector::Config,
 * khronos/include/khronos/active_window/motion_detection/free_space_motion_detector.h:70-95 */
typedef struct kb_motion_config {
  int32_t neighbor_connectivity;   /* 6 | 18 | 26, default 26 */
  int32_t min_cluster_size;        /* default 0 */
  int32_t max_cluster_size;        /* default 1000000 */
  float min_separation_distance;   /* voxels, default 1 */
  float max_range;                 /* m, default 10000 */
  float min_z_coordinate;          /* m (sensor frame offset), default -10000 */
  int32_t num_threads;             /* CPU oracle only */
} kb_motion_config;

/* Pinhole hydra::Camera (UP) + range limits from InputData. */
typedef struct kb_camera {
  int32_t width, height;
  float fx, fy, cx, cy;
  float min_range, max_range;
} kb_camera;

/* KB_MEM_HOST: host images, borrowed until the call returns. KB_MEM_DEVICE: device pointers, used in place.
 * KB_MEM_HOST_ASYNC: pinned host images the caller keeps valid and unmodified until kb_synchronize() (or
 * a later call that returns stats) — the H2D copies of consecutive calls then run back to back. */
enum { KB_MEM_HOST = 0, KB_MEM_DEVICE = 1, KB_MEM_HOST_ASYNC = 2 };

/* Pass as kb_frame.mask to integrate with the dynamic image of the most recent kb_detect_motion call, which is
 * still resident on the device (saves the H2D copy of the mask in the per-frame pipeline
 * detect -> integrate -> track, active_window.cpp:127,209-210). */
#define KB_MASK_LAST_DETECTION ((const int32_t*)(uintptr_t)1)

/* khronos::FrameData (khronos/include/khronos/active_window/data/frame_data.h:59-83) wrapping
 * hydra::InputData (UP). */
typedef struct kb_frame {
  const float* depth;          /* H*W z-depth == range image for cameras; <= 0 invalid */
  const int32_t* label;        /* H*W semantic labels, may be NULL */
  const int32_t* mask;         /* H*W dynamic_image; non-zero pixels are not integrated near the
                                  surface (hydra::maskNonZero, active_window.cpp:209); may be NULL */
  const int32_t* object_image; /* H*W, BINARY mode label source (object_integrator.cpp:76-79) */
  const uint8_t* color;        /* H*W*3 RGB, may be NULL */
  const float* vertex_world;   /* H*W*3 world-frame vertex map; NULL => computed from depth+pose */
  double world_T_sensor[16];   /* row-major 4x4, InputData::getSensorPose() */
  uint64_t stamp_ns;           /* must be > 0 (0 is the reference's "never observed" sentinel) */
  int32_t object_target_id;    /* BINARY mode: ObjectIntegrator::setFrameData target id */
  int32_t memory;              /* KB_MEM_HOST | KB_MEM_DEVICE | KB_MEM_HOST_ASYNC for the image pointers */
  /* Compact sensor formats (optional; `depth` / `label` must then be NULL). They are the raw inputs of hydra's
   * input conversion (parseInputPacket, call site active_window.cpp:275: 16UC1 depth in millimetres -> 32FC1
   * metres, 8-bit class ids -> 32SC1) and are expanded on the device: depth = float(depth_u16) * depth_u16_scale
   * (0 stays invalid), label = int32(label_u8). 3 instead of 8 bytes per pixel cross PCIe / NVLink. */
  const uint16_t* depth_u16;
  const uint8_t* label_u8;
  float depth_u16_scale;       /* metres per count, e.g. 0.001f */
  int32_t reserved_;
} kb_frame;

typedef struct kb_frame_stats {
  int32_t blocks_in_frustum;   /* blocks selected by the frustum test (or all allocated blocks) */
  int32_t blocks_allocated;    /* new blocks allocated by this call */
  int32_t blocks_updated;      /* blocks with at least one integrated voxel */
  int32_t voxels_updated;      /* Nv: voxels with a valid measurement */
  int32_t voxels_in_band;      /* Nb: of those, |sdf| < truncation */
  int32_t voxels_semantic;     /* band voxels whose semantic state was updated */
  int32_t total_blocks;        /* blocks allocated in the map after the call */
  int32_t capacity_exceeded;   /* non-zero if a pool ran out (results incomplete) */
} kb_frame_stats;

/* ---- lifecycle -------------------------------------------------------------------------------- */

/* Replaces VolumetricMap construction + ProjectiveIntegrator / TrackingIntegrator /
 * FreeSpaceMotionDetector construction (active_window.cpp:75-98). tracking/motion may be NULL. */
int kb_create(const kb_map_config* map, const kb_integrator_config* integrator,
              const kb_tracking_config* tracking, const kb_motion_config* motion, int device,
              kb_handle** out);
int kb_destroy(kb_handle* h);
const char* kb_last_error(const kb_handle* h);
int kb_abi_version(void);

/* Use an externally owned cudaStream_t (e.g. torch's current stream) for all work of this handle. Stream order is honoured
 * at CALL boundaries: work the caller enqueued on the stream before a call precedes everything the call does, and
 * everything a call does precedes what the caller enqueues afterwards. Inside one kb_integrate_frames call the batches of
 * 32 frames are pipelined over an internal stream (the block selection of batch i+1 overlaps the fusion of batch i), so
 * hand a stream's frames over in large calls (a whole replay step), not 32 at a time. */
int kb_set_stream(kb_handle* h, void* cuda_stream);
int kb_synchronize(kb_handle* h);

int kb_set_camera(kb_handle* h, const kb_camera* camera);

/* Spatial block-hash sharding across the GPUs of one box (new in this build, SURVEY.md §8e): this
 * handle only allocates/integrates blocks with owner(block) == rank. rank=0,nranks=1 = unsharded. */
int kb_set_shard(kb_handle* h, int rank, int nranks);
/* Owner rank of a block index under the shard hash (pure function; usable without a device). */
int kb_block_owner(int32_t bx, int32_t by, int32_t bz, int nranks);

/* Spatial CELL sharding (new in this build): blocks are grouped into square cells of cell_blocks x cell_blocks blocks in
 * x/y (all z); cell (cx, cy) belongs to rank ((cx mod grid_x) + grid_x * (cy mod grid_y)) mod nranks, a periodic tiling,
 * so a camera frustum (a few metres across) touches 1-4 ranks instead of all of them and each rank needs only the frames
 * that touch its cells. cell_blocks == 0 restores the per-block hash of kb_set_shard. Every sharded entry point (fusion,
 * box allocation, the tracking / motion exchanges) uses the layout set last. grid_x * grid_y should be a multiple of
 * nranks (e.g. 4 x 2 for 8 ranks). */
int kb_set_shard_cells(kb_handle* h, int rank, int nranks, int cell_blocks, int grid_x, int grid_y);
/* The same cell sharding with an explicit cell -> rank table instead of the periodic tiling: owners[cy * width + cx] is the
 * rank of cell (origin_cx + cx, origin_cy + cy) (cell index = floor(block index / cell_blocks)); cells outside the table
 * fall back to the tiling. Lets a replay scheduler fit the layout to the trajectory (khronos_b200/replay.py::bisect_layout:
 * contiguous regions with equal numbers of frames touching each). */
int kb_set_shard_table(kb_handle* h, int rank, int nranks, int cell_blocks, int32_t origin_cx, int32_t origin_cy,
                       int32_t width, int32_t height, const uint8_t* owners);
/* touched[i * width * height + cy * width + cx] = 1 iff some block that K0 would select for frames[i] lies in cell
 * (origin_cx + cx, origin_cy + cy): the per-cell counterpart of kb_frame_owners (host arithmetic on the poses only). */
int kb_frame_cells(kb_handle* h, const kb_frame* frames, int32_t n_frames, int cell_blocks, int32_t origin_cx,
                   int32_t origin_cy, int32_t width, int32_t height, uint8_t* touched);
/* Handle-free variants of kb_frame_owners / kb_frame_cells (need no GPU): the scheduler of a sharded replay may run on a host
 * without a device. The layout is passed explicitly: cell_blocks == 0 = per-block hash (kb_set_shard); table == NULL = periodic
 * tiling (kb_set_shard_cells); otherwise the table of kb_set_shard_table. Same arithmetic as the handle-based calls. */
typedef struct kb_shard_layout {
  int32_t nranks, cell_blocks, grid_x, grid_y;
  int32_t table_origin_cx, table_origin_cy, table_width, table_height;
  const uint8_t* table;
} kb_shard_layout;
int kb_frame_owners_host(const kb_camera* camera, float voxel_size, int32_t voxels_per_side, const kb_shard_layout* layout,
                         const kb_frame* frames, int32_t n_frames, uint32_t* owner_mask);
int kb_frame_cells_host(const kb_camera* camera, float voxel_size, int32_t voxels_per_side, const kb_frame* frames,
                        int32_t n_frames, int cell_blocks, int32_t origin_cx, int32_t origin_cy, int32_t width, int32_t height,
                        uint8_t* touched);
/* Owner of a block under the cell layout (pure function; usable without a device). */
int kb_cell_owner(int32_t bx, int32_t by, int cell_blocks, int grid_x, int grid_y, int nranks);
/* Which ranks need a frame: bit r of owner_mask[i] is set iff some block that hydra's findBlocksInViewFrustum would select
 * for frames[i] (the candidates of K0: block centre inside the inflated view frustum, upstream ProjectiveIntegrator::
 * updateMap; call site active_window.cpp:210) is owned by rank r under this handle's shard layout. Host arithmetic only
 * (poses, camera, layout; the images are not touched): the scheduler of a sharded replay uses it to send each frame
 * only where it is needed. Evaluated with a 1 mm larger inflation than K0, so the mask is a superset of the ranks on which
 * the device finds work (an extra frame on a rank is a no-op). nranks <= 32. */
int kb_frame_owners(kb_handle* h, const kb_frame* frames, int32_t n_frames, uint32_t* owner_mask);

/* ---- peer-memory frame exchange (new in this build; csrc/kb_peer.cu) -----------------------------------------------
 * The sharded replay keeps the stream striped over the GPUs' frame pools and every rank pulls the frames it needs out
 * of its peers' pools over NVLink. Pools are plain device allocations shared through CUDA IPC: kb_peer_alloc +
 * kb_peer_export on the owner, kb_peer_open (-> a pointer valid on `device`) on the readers. No handle, no collective:
 * the pools are read-only while frames are being pulled. Errors: kb_peer_last_error() (thread-local). */
int kb_peer_alloc(int device, size_t bytes, void** ptr);
int kb_peer_free(int device, void* ptr);
int kb_peer_export(int device, void* ptr, uint8_t handle[64]);
int kb_peer_open(int device, const uint8_t handle[64], void** mapped);
int kb_peer_close(int device, void* mapped);
int kb_peer_enable_access(int device, int peer_device);  /* same-process multi-device use (tests) */
const char* kb_peer_last_error(void);
/* A gather plan = n contiguous ranges (src[i] -> dst[i], bytes[i]; 16-byte aligned and sized; src may be a peer
 * mapping), uploaded once and run many times. Transports: */
enum { KB_GATHER_CE = 0,    /* cudaMemcpyAsync per range (copy engines, no SM time) */
       KB_GATHER_SM = 1,    /* persistent CTAs, 16 B loads / stores */
       KB_GATHER_BULK = 2   /* single-warp CTAs driving a cp.async.bulk + mbarrier pipeline (TMA unit) */ };
typedef struct kb_gather_plan kb_gather_plan;
int kb_gather_plan_create(int device, int32_t n, const void* const* src, void* const* dst, const uint64_t* bytes,
                          kb_gather_plan** out);
int kb_gather_plan_destroy(kb_gather_plan* plan);
uint64_t kb_gather_plan_bytes(const kb_gather_plan* plan);
/* Enqueues the plan's copies on cuda_stream (max_ctas bounds the grid of the two kernel transports). */
int kb_gather_run(kb_gather_plan* plan, int mode, int max_ctas, void* cuda_stream);

/* ---- the hot path ----------------------------------------------------------------------------- */

/* K0+K1. Replaces hydra::ProjectiveIntegrator::updateMap(data, map, allocate_blocks, mask)
 * (call sites active_window.cpp:210, mesh_object_extractor.cpp:242) incl. the computeLabel hook
 * (object_integrator.cpp:58-81). stats may be NULL (then no device->host sync happens). */
int kb_integrate_frame(kb_handle* h, const kb_frame* frame, int allocate_blocks,
                       kb_frame_stats* stats);

/* Batched K0+K1 for streams that are available ahead of time — replay / benchmarking and the object
 * extractor's loop "for each semantic frame: integrator.updateMap(...)" (mesh_object_extractor.cpp
 * :239-243). Results are identical to calling kb_integrate_frame on each frame in order; internally up
 * to 32 frames are fused per kernel launch with the voxel state held in registers. stats (optional)
 * receives the sums over the n frames. */
int kb_integrate_frames(kb_handle* h, const kb_frame* frames, int32_t n_frames, int allocate_blocks,
                        kb_frame_stats* stats);

/* Raw cumulative device counters (diagnostics; layout = enum Counter in csrc/kb_device.cuh). Writes
 * min(n, available) values. Index 17 = (block, frame) pairs that survived K0 culling. */
int kb_get_debug_counters(kb_handle* h, int32_t* out, int32_t n);

/* 1 (default): conservative per-(block, frame) depth culling for calls with >= 4 frames; 0: never; 2: always.
 * Results do not depend on this switch; it exists so tests can prove that. */
int kb_set_culling(kb_handle* h, int enabled);

/* Cumulative counters since kb_create (same fields as kb_frame_stats, summed over all frames;
 * total_blocks = live blocks now; the 32-bit sums wrap modulo 2^32 — difference them as uint32).
 * One 64 B device->host read + stream sync. Used for metrics
 * (SURVEY.md §5 "C-ABI returns counters") and for the bench's byte model. */
int kb_get_totals(kb_handle* h, kb_frame_stats* totals);

/* The same cumulative counters in 64 bits (the hydra::timing-style metrics a long run logs, SURVEY.md §5): they never
 * wrap (voxels_updated passes 2^32 after ~36 k frames of a 640x480 stream). frames = distinct stamps seen so far;
 * block_frame_pairs = (block, frame) pairs that survived the block-level culling. One device->host read + stream sync. */
typedef struct kb_totals64 {
  uint64_t blocks_in_frustum, blocks_allocated, blocks_updated;
  uint64_t voxels_updated, voxels_in_band, voxels_semantic;
  uint64_t block_frame_pairs, total_blocks, capacity_exceeded, frames;
} kb_totals64;
int kb_get_totals64(kb_handle* h, kb_totals64* totals);

/* Order-independent checksum of the whole map, computed on the device (for self-verifying benchmarks and shard-count
 * invariance: the sums of the shards of a sharded map add up to the unsharded map's). Every voxel of every allocated
 * block contributes v = mix64(mix64(mix64(mix64(key ^ mix64(lin + 1)) ^ (distance bits | weight bits << 32)) ^ label) ^
 * last_observed_ns), key = the 63-bit packed block index ((x + 2^20) | (y + 2^20) << 21 | (z + 2^20) << 42), lin = linear
 * voxel index, label = semantic_label or 0xFFFFFFFF when empty, mix64 = the murmur3 finaliser:
 * out[0] = sum of v mod 2^64, out[1] = xor of v, out[2] = allocated blocks, out[3] = voxels observed at least once.
 * tests/harness.py::map_checksum is the same function over a kb_block_export (product or oracle). */
int kb_map_checksum(kb_handle* h, uint64_t out[4]);

/* K2+K3. Replaces TrackingIntegrator::updateBlocks (tracking_integrator.cpp:71-104). */
int kb_update_tracking(kb_handle* h, uint64_t stamp_ns);

/* K2r. Replaces TrackingIntegrator::resetInactive (tracking_integrator.cpp:106-131). Removed block
 * indices (x,y,z triples, ascending) are written to removed_xyz (capacity max_removed triples). */
int kb_reset_inactive(kb_handle* h, int32_t* removed_xyz, int32_t max_removed, int32_t* n_removed);

/* ActiveWindow::finishMapping (active_window.cpp:181-183): has_active_data=false on all blocks. */
int kb_mark_all_inactive(kb_handle* h);

/* Clears the `updated` flag of all blocks (active_window.cpp:169-171). */
int kb_clear_updated(kb_handle* h);

/* M1-M4. Replaces FreeSpaceMotionDetector::processInput (free_space_motion_detector.cpp:73-103).
 * dynamic_image_out: H*W int32 (host), 0 = static, cluster ids 1..255. n_seeds/n_clusters optional.
 * Where it runs: M1 always on the device. M2-M4 on the device when min_separation_distance > 0, with or without
 * frame->vertex_world (host, pinned or device; the map is copied, so the caller may reuse its buffer after the call);
 * on the host when min_separation_distance <= 0 (one voxel may then belong to several clusters). */
int kb_detect_motion(kb_handle* h, const kb_frame* frame, int32_t* dynamic_image_out,
                     int32_t* n_seeds, int32_t* n_clusters);
/* One frame of the active-window loop in a single call: motion detection (active_window.cpp:127), integration
 * with the resulting dynamic image as mask (:209-210) and the tracking update (:214), enqueued back to back with
 * ONE device->host round trip at the end (image + counters). Same results as kb_detect_motion +
 * kb_integrate_frame(mask = dynamic image) + kb_update_tracking(frame->stamp_ns). dynamic_image_out (host; pinned
 * memory avoids a staging copy) may be NULL when only the counts are needed. */
int kb_spin_once(kb_handle* h, const kb_frame* frame, int32_t* dynamic_image_out, int32_t* n_seeds,
                 int32_t* n_clusters);

/* Clusters of the last kb_detect_motion call (MeasurementCluster, measurement_clusters.h:63-81):
 * counts[c*2+0]=#pixels, counts[c*2+1]=#voxels; then flat pixel (u,v) pairs (order within a cluster
 * unspecified, duplicates preserved as in the reference) and voxel (x,y,z) global indices (ascending
 * z,y,x) in cluster order; bbox_min_max[c*6..] = world AABB of the cluster's vertices
 * (writeClustersToData, free_space_motion_detector.cpp:396-397): of frame->vertex_world when the frame had one, else of
 * the back-projected depth. NULL pointers are skipped. Also valid after kb_spin_once and kb_motion_result, and unaffected
 * by calls other than motion detections in between. After a device clustering (min_separation_distance > 0) the first
 * call builds the lists on the device and copies only them back; later calls for the same detection reuse them. There
 * the boxes order -0 below +0 (IEEE 754-2019 minimum / maximum), as the pixel order they would otherwise depend on is
 * unspecified. */
int kb_get_motion_clusters(kb_handle* h, int32_t* counts, int32_t* pixels_uv, int64_t* voxels_xyz,
                           float* bbox_min_max, int32_t* total_pixels, int32_t* total_voxels);

/* Host-only entry point (needs no GPU, no handle): the M2-M4 host path on caller-supplied per-pixel voxel keys
 * (3 ints per pixel, x == INT32_MIN for dropped pixels) and seed flags — what the M1 kernel produces. Used by the
 * CPU test-suite to check the product's host clustering against the oracle; writes cluster ids into
 * dynamic_image_out and returns the number of seed voxels / clusters. */
int kb_host_cluster_motion(const kb_camera* camera, const kb_motion_config* motion, const double world_T_sensor[16],
                           const int32_t* pixel_voxel_xyz, const uint8_t* pixel_seed, const float* depth,
                           int32_t* dynamic_image_out, int32_t* n_seeds, int32_t* n_clusters);

/* E0. Replaces the dense allocation loop of MeshObjectExtractor::extractStaticObject
 * (mesh_object_extractor.cpp:220-228): allocates all blocks in [min,max] (inclusive). */
int kb_allocate_box(kb_handle* h, const int32_t min_block[3], const int32_t max_block[3]);

/* K4. Replaces the low-confidence erase loop (mesh_object_extractor.cpp:246-264) with
 * computeConfidence (:342-356): voxels with distance <= 0 and confidence < min_confidence get
 * distance = +truncation. */
int kb_scan_object_confidence(kb_handle* h, float min_confidence, int32_t min_observations,
                              int32_t* n_erased);

/* ---- semantic object detection (the step before the path; SURVEY.md §8f row 2) ----------------------------------
 * khronos::ConnectedSemantics::Config (khronos/include/khronos/active_window/object_detection/connected_semantics.h
 * :64-84) + the object classes of hydra's label space (GlobalInfo::getLabelSpaceConfig().isObject, call sites
 * connected_semantics.cpp:134,164). */
typedef struct kb_object_detector_config {
  int32_t use_full_connectivity;  /* 26 / 8 neighbours if non-zero, else 6 / 4; default 1 */
  int32_t min_cluster_size;       /* pixels; default 0 */
  int32_t max_cluster_size;       /* pixels; <= 0 disables (3D mode only, as in the reference); default -1 */
  int32_t use_3d;                 /* 1: cluster in a voxel grid (semanticClustering3D), 0: in image space; default 1 */
  float grid_size;                /* m, 3D mode; default 0.1 */
  float max_range;                /* m, 3D mode; 0 = infinite; default 0 */
  uint8_t is_object[KB_MAX_LABELS]; /* 1 => the label is an object class */
} kb_object_detector_config;

/* Replaces ConnectedSemantics::processInput (connected_semantics.cpp:60-69 -> semanticClustering3D :71-122 with
 * computeCandidateVoxels :124-146, or semanticClustering2D :148-198 + filterClusters :200-217): connected components
 * of the object-class pixels (per semantic id) in a voxel grid of the world-frame vertex map or in image space.
 * object_image_out: H*W int32 (host), 0 = no object, else the cluster id (FrameData::object_image, the label source
 * of the ObjectIntegrator, object_integrator.cpp:76-79). The frame needs depth (+ pose, or vertex_world) and label.
 * Cluster ids: 2D mode exactly as the reference (creation order of the column-major scan, ids of filtered clusters
 * are not reused); 3D mode: semantic ids ascending (std::map, connected_semantics.h:88), clusters of one id ordered
 * by their smallest voxel in (z, y, x) order — a determinisation of the reference's unordered_map iteration. 3D mode
 * skips pixels whose vertex has a non-finite coordinate or whose voxel lies outside +-2^17 cells (docs/ORACLE_SPEC.md
 * §10); the size filter runs before the ranking, and KB_ERR_CAPACITY means more than 4096 clusters passed it. */
int kb_detect_objects(kb_handle* h, const kb_object_detector_config* config, const kb_frame* frame,
                      int32_t* object_image_out, int32_t* n_clusters);
/* Clusters of the last kb_detect_objects call (MeasurementCluster id / semantics.category_id / pixels,
 * measurement_clusters.h:63-81), ascending id: id_semantic_count[c*3+0..2] = id, semantic id, #pixels; then the
 * flat (u, v) pixel list in cluster order (order within a cluster unspecified). NULL pointers are skipped. Unaffected by
 * kb_forward_instances and kb_set_camera: (u, v) are pixels of the image that was detected. */
int kb_get_object_clusters(kb_handle* h, int32_t* id_semantic_count, int32_t* pixels_uv, int32_t* n_clusters,
                           int32_t* total_pixels);

/* khronos::InstanceForwarding (khronos/include/khronos/active_window/object_detection/instance_forwarding.h:62-86): the
 * other shipped ObjectDetector — forwards the instance ids of an upstream segmenter instead of clustering class labels. */
#define KB_MAX_INSTANCE_IDS 4096
typedef struct kb_instance_forwarding_config {
  float max_range;            /* m; 0 = infinite */
  int32_t min_cluster_size;   /* pixels */
  int32_t max_cluster_size;   /* pixels; <= 0 disables */
  double min_object_volume;   /* m^3 of the cluster's world AABB; the volume filter runs if min > 0 or max > 0 (:68) */
  double max_object_volume;   /* <= 0 disables the upper bound */
} kb_instance_forwarding_config;
/* Replaces InstanceForwarding::processInput / extractSemanticClusters (instance_forwarding.cpp:73-149). label = instance id
 * image (ids 1 .. KB_MAX_INSTANCE_IDS - 1, 0 = none). id_is_background[id] != 0 (host, n_background entries, may be NULL)
 * is the caller's per-id open-set decision "best background score > max_background_score" (:96-104: embeddings and prompts
 * stay on the host; the decision only depends on the id). object_image_out (host, H*W) = the label image, as in the
 * reference, where object_image shares the label image's buffer (:83) so that filtered pixels keep their id. A pixel
 * belongs to its id's cluster if the id is not background and range <= max_range; clusters are then filtered by pixel
 * count and by the volume of the world-frame bounding box of their vertices (:118-135). Cluster order: ascending id (a
 * determinisation of the reference's unordered_map iteration). */
int kb_forward_instances(kb_handle* h, const kb_instance_forwarding_config* config, const kb_frame* frame,
                         const uint8_t* id_is_background, int32_t n_background, int32_t* object_image_out,
                         int32_t* n_clusters);
/* Clusters of the last kb_forward_instances: id_count[c*2+0..1] = id, #pixels; bbox_min_max[c*6..] = world AABB (min xyz,
 * max xyz; per axis the minimum / maximum over the non-NaN coordinates with -0 < +0, NaN if there is none); pixels_uv = flat
 * (u, v) lists in cluster order, pixels within a cluster in the reference's column-major scan order (u outer, v inner);
 * pixels_uv needs total_pixels entries, id_count / bbox_min_max n_clusters. NULL pointers are skipped. Unaffected by
 * kb_detect_objects and kb_set_camera. */
int kb_get_instance_clusters(kb_handle* h, int32_t* id_count, float* bbox_min_max, int32_t* pixels_uv, int32_t* n_clusters,
                             int32_t* total_pixels);

/* Input conversion (SURVEY.md §8f row 2, first half): the world-frame vertex map that upstream parseInputPacket builds for
 * FrameData (call site active_window.cpp:275; InputData::vertex_map, read e.g. at free_space_motion_detector.cpp:174-175,
 * max_iou_tracker.cpp:456): p_W = R * ((u-cx)/fx*d, (v-cy)/fy*d, d) + t in fp32 for every pixel (no validity test; d = 0
 * gives the sensor position). vertex_world_out: H*W*3 floats in frame->memory space. The entry points of this library
 * compute these points themselves; this is for host code that still wants the map. */
int kb_compute_vertex_map(kb_handle* h, const kb_frame* frame, float* vertex_world_out);

/* ---- track measurements (the step after the path; SURVEY.md §8f row 4) -------------------------------------------
 * khronos::MaxIoUTracker in its shipped mode track_by = "voxels" (khronos_ros/config/mapper/uHumans2.yaml:72). The
 * association itself (max_iou_tracker.cpp:216-448) is list bookkeeping and stays with the caller; this entry replaces
 * what it loops over pixels and voxel sets for, for all clusters of one id image at once:
 *   setupTrackMeasurementVoxels (max_iou_tracker.cpp:450-459)  cluster.voxels = { grid.toIndex(vertex_map(pixel)) } at
 *                                                              Config::voxel_size (max_iou_tracker.h:95, default 0.1)
 *   computeCentroid, voxel mode (:534-539)                     centroid = (voxel_sums / voxel_counts + 0.5) * voxel_size
 *                                                              (the reference adds float voxel centres in the iteration
 *                                                              order of an unordered_set; the integer sums are order free)
 *   computeIoUVoxels (:551-562)                                intersections / iou against every track's last_voxels
 * frame: depth (+ pose) or vertex_world, as for kb_detect_objects. id_image: H*W int32 in frame->memory space —
 * FrameData::dynamic_image or object_image. Clusters: n_clusters <= 1022 rows; cluster_ids (host, strictly ascending
 * pixel values, e.g. the ids of kb_get_object_clusters — the 2D detector keeps creation-order ids, which can be large)
 * or NULL for the pixel values 1..n_clusters (dynamic images, 3D object images). Pixels with any other value belong
 * to no cluster. Tracks: n_tracks lists of global voxel indices (x, y, z int64; Track::last_voxels, unique within a
 * track), track t = track_voxels_xyz[3*track_offsets[t] .. 3*track_offsets[t+1]).
 * Outputs (host, NULL = skipped): voxel_counts[n_clusters], voxel_sums[n_clusters*3], intersections[n_clusters*n_tracks]
 * and iou[n_clusters*n_tracks] (row = position in cluster_ids, or id - 1), iou formed exactly like :562 (float inter /
 * (float(size + size) - inter), so an empty cluster against an empty track is NaN as in the reference). Voxels further
 * than 2^17 tracker voxels from the origin are dropped (13 km at 0.1 m).
 * Precondition: the clusters are disjoint in the id image (one id per pixel). The reference's MeasurementCluster.pixels can
 * put one pixel into two dynamic clusters when min_separation_distance == 0 (clusterDynamicVoxels has no closed-set check on
 * absorbed neighbours) and its ids saturate at 255 (writeClustersToData); the image then keeps only the last id and the
 * per-cluster rows differ from MaxIoUTracker's. With min_separation_distance > 0 (shipped: 2) and <= 254 dynamic clusters the
 * image is exact. */
int kb_track_measurements(kb_handle* h, const kb_frame* frame, const int32_t* id_image, int32_t n_clusters,
                          const int32_t* cluster_ids, float voxel_size, int32_t n_tracks, const int32_t* track_offsets,
                          const int64_t* track_voxels_xyz, int32_t* voxel_counts, int64_t* voxel_sums,
                          int32_t* intersections, float* iou);
/* Voxel sets of the last kb_track_measurements call (what updateTrack stores as Track::last_voxels, :487-489):
 * offsets[n_clusters + 1] and the flat (x, y, z) list, clusters in row order, voxels ascending in (z, y, x). Valid until the
 * handle's next motion / object detection or track measurement. NULL pointers are skipped. */
int kb_get_cluster_voxels(kb_handle* h, int32_t* offsets, int64_t* voxels_xyz, int32_t capacity, int32_t* total);

/* ---- ray index (SURVEY.md §8f row 3) -------------------------------------------------------------------------------
 * khronos::RayVerificator (khronos/include/khronos/backend/change_detection/ray_verificator.h:58-258,
 * khronos/src/backend/change_detection/ray_verificator.cpp): the measurement rays of the scene graph (sensor position at
 * a pose-graph node -> mesh vertex, with the stamp of the node) hashed into the coarse blocks they pass through, and the
 * per-point query "which rays through this block saw the point / saw through it". Its own handle: it lives in the
 * backend, independent of the active-window map. The scene-graph side (which vertex gets rays from which pose nodes,
 * computeVertexSources :278-330, RayLookup) stays with the caller, who passes endpoints and stamps as arrays. */
typedef struct kb_ray_index kb_ray_index;
typedef struct kb_ray_config {   /* RayVerificator::Config (ray_verificator.h:68-100) */
  float block_size;              /* m, default 1.0 */
  float radial_tolerance;        /* m, default 0.1 */
  float depth_tolerance;         /* m, default 0.1 */
} kb_ray_config;
int kb_rays_create(const kb_ray_config* config, int device, kb_ray_index** out);  /* all three must be > 0 (:56-61) */
int kb_rays_destroy(kb_ray_index* h);
const char* kb_rays_last_error(const kb_ray_index* h);
int kb_rays_clear(kb_ray_index* h);                                               /* setDsg's reset (:150-166) */
int kb_rays_size(kb_ray_index* h, int32_t* n_rays, int64_t* n_block_entries);
/* addVertices' ray loop + addRayToHash (:264-273, :326-350) for n new rays (indices continue from the rays already
 * held): sources / targets = lookup.getSource / getTarget (x, y, z float), timestamps = Ray::timestamp. Marches each
 * ray in steps of block_size / 4 and adds it to every block entered. observed_blocks_xyz (optional, capacity
 * max_observed blocks) receives the distinct blocks the NEW rays pass through (addVertices' return value, what
 * updateDsg intersects with vertices_in_block_ / objects_in_block_ :176-189), ascending in (z, y, x); if it is too
 * small the call fails with KB_ERR_CAPACITY, *n_observed holds the needed size and no ray is added. */
int kb_rays_add(kb_ray_index* h, int32_t n, const float* sources_xyz, const float* targets_xyz, const uint64_t* timestamps,
                int32_t* observed_blocks_xyz, int32_t max_observed, int32_t* n_observed);
/* RayVerificator::Config::RayPolicy (ray_verificator.h:84-92); kRandom / kRandom3 draw from rand_r and are not offered. */
enum { KB_RAYS_FIRST = 0, KB_RAYS_LAST = 1, KB_RAYS_FIRST_AND_LAST = 2, KB_RAYS_MIDDLE = 3, KB_RAYS_ALL = 4 };
/* addVertices (:222-276) for n_vertices new mesh vertices (global indices vertex_index_base + i): per vertex the pose
 * nodes chosen by computeVertexSources (:278-330) from the ascending pose stamps (timestamps_) — upper_bound(first_seen),
 * lower_bound(last_seen - active_window_duration), lower_bound of their mean, or all poses in between — each giving one
 * ray pose position -> vertex with the pose's stamp; then kb_rays_add. The selection (binary searches) runs on the
 * host, the march on the device. Rays are appended vertex by vertex, pose indices ascending within a vertex. */
int kb_rays_add_vertices(kb_ray_index* h, int32_t policy, float active_window_duration, int32_t n_poses, const uint64_t* pose_stamps,
                         const float* pose_positions_xyz, int32_t n_vertices, int32_t vertex_index_base, const float* vertices_xyz,
                         const uint64_t* first_seen, const uint64_t* last_seen, int32_t* observed_blocks_xyz, int32_t max_observed,
                         int32_t* n_observed, int32_t* n_rays_added);
/* Ray::source_node (as index into the pose arrays), Ray::target_index and Ray::timestamp of all rays (-1 ids for rays
 * added through kb_rays_add): what the caller gathers new endpoints with after a deformation. NULL pointers are skipped. */
int kb_rays_get_ray_ids(kb_ray_index* h, int32_t* pose_index, int32_t* vertex_index, uint64_t* timestamps, int32_t capacity);
/* The rays are deformable: check() reads their endpoints from the current scene graph (:88-100) while the hash keeps
 * the blocks computed when they were added. Replaces the endpoints of ALL rays (n_rays must match). */
int kb_rays_set_endpoints(kb_ray_index* h, int32_t n_rays, const float* sources_xyz, const float* targets_xyz);
int kb_rays_rehash(kb_ray_index* h);                                              /* recomputeHash (:314-324) */
/* check (:66-146) for n_points points, each with its own [earliest, latest] stamp window: counts[2*i] = rays that saw
 * through point i (CheckResult::absent), counts[2*i+1] = rays that ended at it (present); rays outside the window,
 * further than radial_tolerance from the point or occluded before it count for neither. *total_stamps = sum of counts. */
int kb_rays_check(kb_ray_index* h, int32_t n_points, const float* points_xyz, const uint64_t* earliest, const uint64_t* latest,
                  int32_t* counts, int64_t* total_stamps);
/* The stamps of the last kb_rays_check: for every point its absent stamps, then its present stamps, each ascending (the
 * reference returns them in unordered_set iteration order; the consumers bucket them, ray_change_detector.cpp:72-81). */
int kb_rays_get_stamps(kb_ray_index* h, uint64_t* stamps, int64_t capacity);

/* ---- sharded per-frame pipeline (new in this build; SURVEY.md §8e exchange steps 1 and 2) -----------------------
 * With kb_set_shard(rank, nranks > 1) a handle holds only the blocks it owns. Fusion (K0/K1/K1b), K2, K2r and K4 are
 * independent per block and need nothing else. Two steps of ActiveWindow::spinOnce look across blocks:
 *   M1 (free_space_motion_detector.cpp:158-203) asks the block of every pixel's endpoint whether that voxel is
 *      ever-free: only the owner knows  ->  per-pixel flag bytes, MAX-all-reduced over the ranks;
 *   K3 (tracking_integrator.cpp:168-222) reads the 6/18/26 neighbours of every voxel of an updated block, across
 *      block borders  ->  the owners publish 1 bit per voxel ("ever_free || voxelIsFree at this pass", exactly the
 *      predicate K3 evaluates on neighbours) for the blocks that neighbour another rank's updated blocks.
 * The collectives themselves (2 all-gathers, 1 all-reduce per frame) are issued by the host program between these
 * calls (khronos_b200/distributed.py uses torch.distributed / NCCL) on buffers of the sizes kb_shard_buffer_sizes
 * reports; all buffer arguments are DEVICE pointers on the handle's stream (make it the stream the collectives
 * are ordered with via kb_set_stream). Buffer layouts: struct ShardExchange in csrc/kb_kernels.cuh. Lists that
 * do not fit raise capacity_exceeded (reported by the next stats / totals read). */
int kb_set_shard_capacity(kb_handle* h, int32_t pending_capacity, int32_t halo_capacity); /* blocks per rank and pass; default 1024 / 2048 */
int kb_shard_buffer_sizes(kb_handle* h, int64_t* pending_bytes, int64_t* halo_bytes, int64_t* pixel_flag_bytes);
/* K2 on the local shard (TrackingIntegrator::updateBlockTracking, tracking_integrator.cpp:133-166) + export of this
 * rank's ever-free work list (the tracking_updated blocks, :75-77) into pending_out. */
int kb_tracking_begin(kb_handle* h, uint64_t stamp_ns, void* pending_out);
/* all_pending = the nranks pending buffers concatenated in rank order (all-gather). Writes the free masks of the
 * locally owned blocks that neighbour another rank's pending block into halo_out. */
int kb_tracking_pack_halo(kb_handle* h, const void* all_pending, void* halo_out);
/* all_halo = the nranks halo buffers concatenated. K3 (updateBlockEverFree, :168-222) on the local pending blocks;
 * must stay valid until the stream has run the pass. Completes the pass kb_tracking_begin opened. */
int kb_tracking_finish(kb_handle* h, const void* all_pending, const void* all_halo);
/* M1 on the local shard: pixel_flags[H*W] (device) gets bit0 = the pixel is in this rank's point map (its block
 * exists here and the voxel index is valid), bit1 = that voxel is ever-free (a seed). */
int kb_motion_lookup_local(kb_handle* h, const kb_frame* frame, uint8_t* pixel_flags);
/* pixel_flags after the MAX all-reduce: M2-M4 run replicated (and deterministically) on every rank; the dynamic
 * image stays on the device for KB_MASK_LAST_DETECTION. Enqueue only. */
int kb_motion_cluster_global(kb_handle* h, const uint8_t* pixel_flags);
/* Synchronises the handle's stream and returns the last detection's counts (+ the dynamic image to host memory if
 * dynamic_image_out != NULL). */
int kb_motion_result(kb_handle* h, int32_t* dynamic_image_out, int32_t* n_seeds, int32_t* n_clusters);

/* Peer-memory variants of the three exchanges: instead of filling a local buffer for a collective, the producing kernels
 * store this rank's part directly into every rank's buffer (peer_*[q] = base address of rank q's buffer as mapped on
 * this device, e.g. torch.distributed._symmetric_memory buffer_ptrs; peer_*[rank] is the local one; n_peers = nranks
 * <= 16). all_pending / all_halo buffers have the all-gather layout (nranks slots); the flag images are H*W bytes
 * and must be zero before the peers write (the consumer zeroes its own image after kb_motion_cluster_global). The
 * host places one barrier between each producer call and the matching consumer call (kb_tracking_pack_halo[_peers]
 * reads all_pending, kb_tracking_finish reads all_halo, kb_motion_cluster_global reads the flag image). */
int kb_tracking_begin_peers(kb_handle* h, uint64_t stamp_ns, void* const* peer_all_pending, int32_t n_peers);
int kb_tracking_pack_halo_peers(kb_handle* h, const void* all_pending, void* const* peer_all_halo, int32_t n_peers);
int kb_motion_lookup_peers(kb_handle* h, const kb_frame* frame, uint8_t* const* peer_flags, int32_t n_peers);

/* NVLS frame broadcast for the sharded map (no handle needed): copies `bytes` (multiple of 16, both pointers 16 B
 * aligned) from local device memory to the MULTICAST address of a symmetric buffer (e.g. _SymmetricMemory.multicast_ptr
 * + offset), on the given stream: NVSwitch delivers every store to all ranks of the multicast group. The caller orders
 * it against the consumers with a barrier (e.g. _SymmetricMemory.barrier()). Untested on hardware in round 1. */
int kb_multicast_copy(void* multicast_dst, const void* src, size_t bytes, void* cuda_stream);

/* ---- mesh extraction (SURVEY.md §8f row 1) ------------------------------------------------------------------------
 * Replaces hydra::MeshIntegrator::generateMesh(map, only_mesh_updated_blocks, clear_updated_flag) (UPSTREAM; call sites
 * active_window.cpp:223 with (true, true), mesh_object_extractor.cpp:267 with (true, false)): marching cubes over the
 * TSDF of the blocks whose mesh_updated flag is set (or all blocks), on the device, so that an output tick moves the
 * triangles to the host instead of every updated voxel block. Per block: the cubes inside the block (x-major), then
 * the cubes on its max-x / max-y / max-z faces, which read the +x/+y/+z neighbour blocks (skipped when a neighbour is
 * missing); a cube is meshed only if all 8 corner voxels have weight >= min_weight (hydra's MeshIntegratorConfig,
 * default 1e-4); vertices are interpolated along the cube edges with a sign change; vertex colour / label are those of
 * the nearer corner voxel. Vertices are not shared: triangle k is vertices (3k, 3k+1, 3k+2), so the face list of
 * utils::combineMeshLayer (khronos/src/utils/geometry_utils.cpp:61-86) is the identity. Results stay on the device
 * until kb_get_mesh. On a sharded map the cubes on a shard border miss their remote neighbour blocks (seams). */
int kb_generate_mesh(kb_handle* h, int only_mesh_updated_blocks, int clear_updated_flag, float min_weight,
                     int32_t* n_blocks, int64_t* n_vertices);
/* Mesh of the last kb_generate_mesh: the processed blocks ascending in (x, y, z) (one hydra MeshBlock each, empty ones
 * included), block_vertex_offsets[n_blocks + 1] into the concatenated vertex arrays (= combineMeshLayer's output plus
 * the block boundaries), points in the world frame. NULL pointers are skipped; capacity_vertices must be >= n_vertices. */
int kb_get_mesh(kb_handle* h, int32_t* block_index_xyz, int64_t* block_vertex_offsets, float* points_xyz,
                uint8_t* colors_rgb, uint32_t* labels, int64_t capacity_vertices);

/* ---- mirror-back / parity export ---------------------------------------------------------------- */

enum { KB_EXPORT_ALL = 0, KB_EXPORT_UPDATED = 1 };

/* Block flags bits (hydra::TsdfBlock flags + TrackingBlock::has_active_data). */
enum {
  KB_FLAG_UPDATED = 1, KB_FLAG_MESH_UPDATED = 2, KB_FLAG_ESDF_UPDATED = 4,
  KB_FLAG_TRACKING_UPDATED = 8, KB_FLAG_HAS_ACTIVE_DATA = 16
};

/* Caller-allocated arrays for n blocks of V = voxels_per_side^3 voxels, blocks sorted ascending by
 * (x, y, z). Any pointer may be NULL to skip that field. This is what repopulates
 * hydra::VolumetricMap for MeshIntegrator / cloneUpdated (active_window.cpp:223,229). */
typedef struct kb_block_export {
  int32_t* block_index;     /* n*3 */
  uint8_t* block_flags;     /* n */
  float* distance;          /* n*V  TsdfVoxel::distance */
  float* weight;            /* n*V  TsdfVoxel::weight */
  uint8_t* color;           /* n*V*3 */
  uint64_t* last_observed;  /* n*V  TrackingVoxel */
  uint64_t* last_occupied;  /* n*V */
  uint8_t* ever_free;       /* n*V */
  uint8_t* active;          /* n*V */
  uint8_t* to_remove;       /* n*V */
  uint32_t* semantic_label; /* n*V  SemanticVoxel */
  uint8_t* semantic_empty;  /* n*V */
  float* semantic_likelihoods; /* n*V*L (L = num_labels for MLE, 2 for BINARY) */
} kb_block_export;

int kb_num_blocks(kb_handle* h, int which, int32_t* n);
int kb_export_blocks(kb_handle* h, int which, int32_t max_blocks, kb_block_export* out,
                     int32_t* n_written);

#ifdef __cplusplus
}
#endif
#endif  /* KHRONOS_B200_H_ */
