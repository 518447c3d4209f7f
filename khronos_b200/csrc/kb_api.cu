// C ABI (include/khronos_b200.h) over the sm_90a kernels: handle lifetime, device memory, frame
// staging, stamp <-> frame-index bookkeeping, export. Host code only; no CPU compute fallback exists:
// every entry point that touches voxels launches a kernel, and kb_create refuses to run without a GPU.
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <thread>
#include <type_traits>
#include <vector>

#include "../../include/khronos_b200.h"
#include "kb_kernels.cuh"
#include "kb_mesh.cuh"
#include "kb_motion_device.cuh"
#include "kb_objects_device.cuh"
#include "kb_tracks_device.cuh"
#include "kb_motion_host.h"

using namespace kb;

struct kb_handle {
  kb_map_config map{};
  kb_integrator_config integ{};
  kb_tracking_config trk{};
  kb_motion_config mot{};
  kb_camera cam{};
  bool has_trk = false, has_mot = false, has_cam = false;
  int device = 0;
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  int rank = 0, nranks = 1;
  DeviceMap dm{};
  int L = 0;
  float block_size = 0, mle_diag = 0, mle_off = 0, mle_init = 0;
  unsigned long long blocked_mask = 0;
  std::vector<uint64_t> stamps;  // frame index -> stamp; [0] = 0 ("never")
  // host frame staging: 2 sets x kMaxBatch frames (device copies of host images), filled on the copy
  // stream so that the H2D of batch i+1 overlaps the kernels of batch i
  float* stg_depth = nullptr;
  int* stg_label = nullptr;
  int* stg_mask = nullptr;
  int* stg_object = nullptr;
  uint16_t* stg_depth16 = nullptr;  // compact inputs (2 sets x kMaxBatch frames)
  uint8_t* stg_label8 = nullptr;
  uint8_t* stg_color = nullptr;     // RGB staging (3 B/pixel), allocated with the first host colour image
  size_t stg_color_pixels = 0;
  uint16_t* mot_depth16 = nullptr;
  float* stg_vertex = nullptr;
  float* mot_depth = nullptr;
  float* mot_vertex = nullptr;  // vertex map of the last motion detection, when its frame carried one
  size_t stg_pixels = 0, mot_pixels = 0;
  int stg_set = 0;
  cudaStream_t copy_stream = nullptr;
  cudaEvent_t stg_ready[2] = {nullptr, nullptr}, stg_consumed[2] = {nullptr, nullptr};
  // batched integration
  BatchParams batch{};
  float* tile_max = nullptr;
  size_t tile_stride = 0;
  int* work_slots = nullptr;
  uint32_t* work_masks = nullptr;
  uint32_t* work_upd = nullptr;
  uint32_t* item_fmask = nullptr;
  int* item_list = nullptr;    // KB_FUSE_ITEM_LIST experiment: compacted heaviest-first item lists (3 x item_list_cap)
  int item_list_cap = 0;
  bool use_item_list = true;   // default since round 2 (won its A/B); KB_FUSE_ITEM_LIST=0 disables
  // KB_PIPELINE experiment: the prologue (tile pyramid, K0, K0b[, compaction]) of batch i+1 runs on its own stream while
  // the fuse kernel of batch i is still busy; work lists, tile pyramids and cursors exist twice (index = batch parity)
  bool pipelined = true;       // default since round 2 (won its A/B); KB_PIPELINE=0 disables
  cudaStream_t pre_stream = nullptr;
  cudaEvent_t pre_done[2] = {nullptr, nullptr}, fuse_done[2] = {nullptr, nullptr}, main_front = nullptr;
  bool main_dirty = true;      // main-stream work other than fuse kernels was enqueued since the last prologue
  int* work_slots2 = nullptr;
  uint32_t* work_masks2 = nullptr;
  uint32_t* work_upd2 = nullptr;
  uint32_t* item_fmask2 = nullptr;
  // KB_H2D_NARROW_LABELS experiment: host i32 label images whose ids fit 8 bits are narrowed on the host (worker threads)
  // into a pinned buffer, cross PCIe as 1 B/pixel and are widened again by expandFramesKernel: 5 instead of 8 B/pixel of
  // H2D traffic for hydra::InputData frames, bit-identical results (frames with ids outside 0..255 take the i32 path)
  bool narrow_labels = false;
  int narrow_threads = 8;
  uint8_t* pin_label8 = nullptr;
  size_t pin_label8_pixels = 0;
  int fuse_coop = 0;           // KB_FUSE_COOP: two-phase CTA-cooperative fuse kernel
  int mlp_group = 0;           // KB_FUSE_MLP experiment: 0 (off), 2 or 4 frames per memory-level-parallel group
  int cull_grid = 0;
  int parity = 0;
  // lazy tracking
  TrackEval pass{};           // state of the last tracking pass
  float trk_cfg_thr = 0.f;    // occupancy threshold in metres
  uint64_t last_pass_stamp = 0;
  int* pending = nullptr;     // ever-free work list
  int everfree_grid = 0;
  bool cull = true;
  bool cull_forced = false;  // kb_set_culling(2): cull even single frames (tests)
  int fuse_grid = 0;
  bool hwm_dirty = true;
  size_t tombstones_ub = 0;      // upper bound on the tombstones in the block hash (removed blocks since the last rebuild)
  size_t rehash_threshold = 0;   // rebuild the hash when the bound exceeds this (default: a quarter of the table)
  int hwm_cached = 0;
  // counters
  int* h_ctr = nullptr;  // pinned mirror
  int prev_ctr[kNumCounters] = {0};
  bool ctr_dirty = false;  // launches happened since prev_ctr was refreshed
  // motion detection scratch + result
  int3* d_pixel_gidx = nullptr;
  uint8_t* d_pixel_seed = nullptr;
  std::vector<int32_t> h_pixel_gidx;
  std::vector<uint8_t> h_pixel_seed;
  std::vector<float> h_depth;
  std::vector<float> h_vertex;  // host copy of the kept vertex map (host clustering of device frames)
  MotionResult motion;
  MotionTable mt{};            // device clustering table (M2-M4)
  bool motion_vertex = false;  // the last detection's frame carried a vertex map (kept in mot_vertex)
  // cluster lists of the last detection (kb_get_motion_clusters), flat in cluster order
  std::vector<int32_t> mcl_counts;  // (pixels, voxels) per cluster
  std::vector<int32_t> mcl_pixels;  // (u, v)
  std::vector<int64_t> mcl_voxels;  // (x, y, z)
  std::vector<float> mcl_bbox;      // min xyz, max xyz per cluster
  // Device-built lists cluster again in a table of their own: the detection's table is reset after use (sparse) or
  // taken over by kb_detect_objects / kb_track_measurements before the lists are asked for.
  MotionTable lt{};
  MotionLists ml{};
  int* ml_gate = nullptr;     // device 1: the list table's stages always run
  size_t ml_clusters = 0, ml_pixels = 0, ml_voxels = 0, ml_sort_bytes = 0;
  void* ml_sort_tmp = nullptr;
  int32_t* d_dynamic = nullptr;  // device copy of the last dynamic image (usable as KB_MASK_LAST_DETECTION)
  int* h_mscal = nullptr;      // pinned mirror of the clustering scalars
  bool motion_stale = false;   // cluster lists of the last device detection not built yet
  MotionHostParams motion_hp{};
  bool motion_have_image = false;
  bool everfree_v2 = true;     // vectorised halo fill of the ever-free pass (default since round 2; KB_EVERFREE_V2=0 disables)
  bool motion_sparse = true;   // slot-wise reset of the clustering table (default since round 2; KB_MOTION_SPARSE=0 disables)
  bool mt_dirty = false;       // the shared table holds entries of another user (object detection / dense clustering)
  int3* d_removed = nullptr;
  int max_removed = 0;
  // semantic object detection (kb_detect_objects): inputs staged here, result image on the device + host copies
  float* obj_depth = nullptr;
  int* obj_label = nullptr;
  int32_t* d_object = nullptr;
  int* h_oscal = nullptr;       // pinned mirror of the clustering scalars
  size_t obj_pixels = 0;
  std::vector<int32_t> obj_image_host, obj_label_host;
  bool obj_have = false;
  // track measurements (kb_track_measurements): staged id image, per-id accumulators, packed track voxels, results
  int32_t* trk_ids = nullptr;
  unsigned long long* trk_export = nullptr;
  size_t trk_pixels = 0;
  int* trk_counts = nullptr;
  unsigned long long* trk_sums = nullptr;
  int* trk_present = nullptr;
  int* trk_idlist = nullptr;
  unsigned long long* trk_keys = nullptr;
  int* trk_of = nullptr;
  size_t trk_voxel_cap = 0;
  int* trk_inter = nullptr;
  size_t trk_inter_cap = 0;
  std::vector<int32_t> trk_counts_host;
  bool trk_have = false;
  // sharded per-frame pipeline (kb_tracking_begin / pack_halo / finish, kb_motion_lookup_local / cluster_global)
  ShardExchange xch{};
  int cap_pending = 1024, cap_halo = 2048;
  uint8_t* d_flags_local = nullptr;  // peer-memory M1 exchange: this rank's flag bytes before they are scattered
  size_t flags_local_pixels = 0;
  TrackingParams open_pass{};   // parameters of the pass between kb_tracking_begin and kb_tracking_finish
  uint64_t open_pass_stamp = 0;
  int open_pass_state = 0;      // 0 none, 1 begun, 2 halo packed
  std::vector<uint8_t> shard_table_host;  // kb_set_shard_table: host copy (kb_frame_owners), device copy in dm.shard_table
  uint8_t* shard_table_dev = nullptr;
  // InstanceForwarding (kb_forward_instances): per-id accumulators on the device, kept clusters + keep mask on the host
  int* inst_counts = nullptr;
  unsigned int* inst_bbox = nullptr;
  uint8_t* inst_background = nullptr;
  uint8_t* inst_keep = nullptr;
  int* inst_bad = nullptr;
  size_t inst_pixels = 0;
  struct InstCluster { int id, count; float bbox[6]; };
  std::vector<InstCluster> inst_clusters;
  std::vector<uint8_t> inst_keep_host;
  bool inst_have = false;
  // marching cubes (kb_generate_mesh): device results of the last call + host copies of the block list
  int* mesh_slots = nullptr;
  unsigned char* mesh_cases = nullptr;
  int* mesh_tri_count = nullptr;
  long long* mesh_tri_base = nullptr;
  size_t mesh_block_cap = 0;
  float* mesh_points = nullptr;
  unsigned char* mesh_colors = nullptr;
  unsigned int* mesh_labels = nullptr;
  size_t mesh_tri_cap = 0;
  std::vector<int3> mesh_index;
  std::vector<long long> mesh_base;  // [n_blocks + 1] triangle offsets
  bool mesh_have = false;
  std::string err;
};

namespace {

#define KB_CUDA(h, call)                                                                       \
  do {                                                                                         \
    cudaError_t e_ = (call);                                                                   \
    if (e_ != cudaSuccess) {                                                                   \
      (h)->err = std::string(#call) + ": " + cudaGetErrorString(e_);                           \
      return KB_ERR_CUDA;                                                                      \
    }                                                                                          \
  } while (0)

int fail(kb_handle* h, int code, const char* msg) {
  if (h) h->err = msg;
  return code;
}

inline double toSeconds(uint64_t ns) { return static_cast<double>(ns) / 1e9; }

template <typename T>
cudaError_t devAlloc(T** p, size_t n, int fill_byte) {
  cudaError_t e = cudaMalloc(reinterpret_cast<void**>(p), std::max<size_t>(n, 1) * sizeof(T));
  if (e != cudaSuccess) return e;
  return cudaMemset(*p, fill_byte, std::max<size_t>(n, 1) * sizeof(T));
}

int ensureStaging(kb_handle* h, size_t pixels) {
  if (h->stg_pixels >= pixels) return KB_OK;
  cudaFree(h->stg_depth); cudaFree(h->stg_label); cudaFree(h->stg_mask); cudaFree(h->stg_object);
  const size_t n = pixels * kMaxBatch * 2;
  KB_CUDA(h, devAlloc(&h->stg_depth, n, 0));
  KB_CUDA(h, devAlloc(&h->stg_label, n, 0));
  KB_CUDA(h, devAlloc(&h->stg_mask, n, 0));
  KB_CUDA(h, devAlloc(&h->stg_object, n, 0));
  cudaFree(h->stg_depth16); cudaFree(h->stg_label8);
  KB_CUDA(h, devAlloc(&h->stg_depth16, n, 0));
  KB_CUDA(h, devAlloc(&h->stg_label8, n, 0));
  h->stg_pixels = pixels;
  return KB_OK;
}

// TsdfVoxel::color lives in its own array that is only allocated once a frame carries a colour image
// (the BASELINE workloads are colour-less and pay nothing for it).
int ensureColorLayer(kb_handle* h) {
  DeviceMap& m = h->dm;
  if (m.color) return KB_OK;
  const size_t n = static_cast<size_t>(m.max_blocks) * m.V;
  KB_CUDA(h, cudaMalloc(reinterpret_cast<void**>(&m.color), n * sizeof(uchar4)));
  KB_CUDA(h, cudaMemsetAsync(m.color, 0, n * sizeof(uchar4), h->stream));
  return KB_OK;
}

int ensureColorStaging(kb_handle* h, size_t pixels) {
  if (h->stg_color_pixels >= pixels) return KB_OK;
  KB_CUDA(h, cudaStreamSynchronize(h->stream));
  KB_CUDA(h, cudaStreamSynchronize(h->copy_stream));
  cudaFree(h->stg_color);
  h->stg_color = nullptr;
  KB_CUDA(h, devAlloc(&h->stg_color, pixels * 3 * kMaxBatch * 2, 0));
  h->stg_color_pixels = pixels;
  return KB_OK;
}

int ensureObjectBuffers(kb_handle* h, size_t pixels) {
  if (h->obj_pixels >= pixels) return KB_OK;
  cudaFree(h->obj_depth); cudaFree(h->obj_label); cudaFree(h->d_object);
  KB_CUDA(h, devAlloc(&h->obj_depth, pixels, 0));
  KB_CUDA(h, devAlloc(&h->obj_label, pixels, 0));
  KB_CUDA(h, devAlloc(&h->d_object, pixels, 0));
  if (!h->h_oscal) KB_CUDA(h, cudaMallocHost(reinterpret_cast<void**>(&h->h_oscal), sizeof(int) * kMsCount));
  h->obj_pixels = pixels;
  return KB_OK;
}

int ensureTrackBuffers(kb_handle* h, size_t pixels, size_t track_voxels, size_t inter) {
  if (h->trk_pixels < pixels) {
    cudaFree(h->trk_ids); cudaFree(h->trk_export);
    KB_CUDA(h, devAlloc(&h->trk_ids, pixels, 0));
    KB_CUDA(h, devAlloc(&h->trk_export, pixels, 0));
    h->trk_pixels = pixels;
  }
  if (!h->trk_counts) {
    KB_CUDA(h, devAlloc(&h->trk_counts, static_cast<size_t>(kTrackMaxIds), 0));
    KB_CUDA(h, devAlloc(&h->trk_sums, static_cast<size_t>(kTrackMaxIds) * 3, 0));
    KB_CUDA(h, devAlloc(&h->trk_present, static_cast<size_t>(kTrackMaxIds), 0));
    KB_CUDA(h, devAlloc(&h->trk_idlist, static_cast<size_t>(kTrackMaxIds), 0));
  }
  if (h->trk_voxel_cap < track_voxels) {
    cudaFree(h->trk_keys); cudaFree(h->trk_of);
    KB_CUDA(h, devAlloc(&h->trk_keys, track_voxels * 2, 0));
    KB_CUDA(h, devAlloc(&h->trk_of, track_voxels * 2, 0));
    h->trk_voxel_cap = track_voxels * 2;
  }
  if (h->trk_inter_cap < inter) {
    cudaFree(h->trk_inter);
    KB_CUDA(h, devAlloc(&h->trk_inter, inter * 2, 0));
    h->trk_inter_cap = inter * 2;
  }
  return KB_OK;
}

int ensureShardBuffers(kb_handle* h) {
  ShardExchange& x = h->xch;
  if (x.halo_mark && x.nranks == h->nranks && x.cap_pending == h->cap_pending && x.cap_halo == h->cap_halo) {
    x.rank = h->rank;
    return KB_OK;
  }
  KB_CUDA(h, cudaStreamSynchronize(h->stream));
  cudaFree(x.halo_mark); cudaFree(x.publish); cudaFree(x.ghost_keys); cudaFree(x.ghost_vals);
  x = ShardExchange{};
  x.rank = h->rank; x.nranks = h->nranks;
  x.cap_pending = h->cap_pending; x.cap_halo = h->cap_halo;
  x.mask_words = h->dm.V / 32;
  uint32_t cap = 1024;
  while (cap < 2u * static_cast<uint32_t>(x.nranks) * static_cast<uint32_t>(x.cap_halo)) cap <<= 1;
  x.ghost_mask = cap - 1;
  KB_CUDA(h, devAlloc(&x.halo_mark, static_cast<size_t>(h->dm.max_blocks), 0));
  KB_CUDA(h, devAlloc(&x.publish, static_cast<size_t>(x.cap_halo), 0));
  KB_CUDA(h, devAlloc(&x.ghost_keys, static_cast<size_t>(cap), 0xFF));
  KB_CUDA(h, devAlloc(&x.ghost_vals, static_cast<size_t>(cap), 0));
  return KB_OK;
}

void freeMotionTable(MotionTable& t) {
  cudaFree(t.keys); cudaFree(t.count); cudaFree(t.flags); cudaFree(t.deg); cudaFree(t.parent); cudaFree(t.pix_total);
  cudaFree(t.min_seed); cudaFree(t.cluster_id); cudaFree(t.roots); cudaFree(t.scalars); cudaFree(t.pix_slot);
  cudaFree(t.occupied);
  t = MotionTable{};
}

// A clean clustering table for `pixels` pixels (gate left to the caller).
int allocMotionTable(kb_handle* h, MotionTable& t, size_t pixels) {
  freeMotionTable(t);
  uint32_t cap = 1024;
  while (cap < 2 * pixels) cap <<= 1;
  t.mask = cap - 1;
  // every root is an occupied slot and at most one slot per pixel is occupied, so the root list never overflows
  t.max_roots = static_cast<int>(pixels);
  KB_CUDA(h, devAlloc(&t.keys, cap, 0xFF));
  KB_CUDA(h, devAlloc(&t.count, cap, 0));
  KB_CUDA(h, devAlloc(&t.flags, cap, 0));
  KB_CUDA(h, devAlloc(&t.deg, cap, 0));
  KB_CUDA(h, devAlloc(&t.parent, cap, 0));
  KB_CUDA(h, devAlloc(&t.pix_total, cap, 0));
  KB_CUDA(h, devAlloc(&t.min_seed, cap, 0xFF));
  KB_CUDA(h, devAlloc(&t.cluster_id, cap, 0));
  KB_CUDA(h, devAlloc(&t.roots, static_cast<size_t>(t.max_roots), 0));
  KB_CUDA(h, devAlloc(&t.occupied, pixels, 0));
  KB_CUDA(h, devAlloc(&t.scalars, static_cast<size_t>(kMsCount), 0));
  KB_CUDA(h, devAlloc(&t.pix_slot, pixels, 0xFF));
  return KB_OK;
}

int ensureMotionBuffers(kb_handle* h, size_t pixels) {
  if (h->mot_pixels >= pixels) return KB_OK;
  cudaFree(h->mot_depth); cudaFree(h->mot_vertex); cudaFree(h->stg_vertex); cudaFree(h->d_pixel_gidx); cudaFree(h->d_pixel_seed);
  cudaFree(h->d_dynamic);
  cudaFree(h->mot_depth16);
  KB_CUDA(h, devAlloc(&h->mot_depth16, pixels, 0));
  KB_CUDA(h, devAlloc(&h->mot_depth, pixels, 0));
  KB_CUDA(h, devAlloc(&h->mot_vertex, pixels * 3, 0));
  KB_CUDA(h, devAlloc(&h->stg_vertex, pixels * 3, 0));
  KB_CUDA(h, devAlloc(&h->d_pixel_gidx, pixels, 0));
  KB_CUDA(h, devAlloc(&h->d_pixel_seed, pixels, 0));
  KB_CUDA(h, devAlloc(&h->d_dynamic, pixels, 0));
  int st = allocMotionTable(h, h->mt, pixels);
  if (st != KB_OK) return st;
  h->mt.gate = h->dm.counters + kCtrSeeds;
  if (!h->h_mscal) KB_CUDA(h, cudaMallocHost(reinterpret_cast<void**>(&h->h_mscal), sizeof(int) * kMsCount));
  h->mot_pixels = pixels;
  return KB_OK;
}

// Resolves one image pointer of a frame to a device pointer (copying host images to staging).
template <typename T>
int stage(kb_handle* h, const T* src, T* staging, size_t count, int memory, const T** out) {
  *out = nullptr;
  if (!src) return KB_OK;
  if (memory == KB_MEM_DEVICE) { *out = src; return KB_OK; }
  KB_CUDA(h, cudaMemcpyAsync(staging, src, count * sizeof(T), cudaMemcpyHostToDevice, h->stream));
  *out = staging;
  return KB_OK;
}

void poseToFloat(const double T[16], float R[9], float t[3], float Rw[9], float tw[3]) {
  // sensor_T_world = world_T_sensor^-1 (rigid), formed in double and rounded once to float.
  double Rd[9], td[3];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) Rd[r * 3 + c] = T[c * 4 + r];
  for (int r = 0; r < 3; ++r) td[r] = -(Rd[r * 3 + 0] * T[3] + Rd[r * 3 + 1] * T[7] + Rd[r * 3 + 2] * T[11]);
  for (int i = 0; i < 9; ++i) R[i] = static_cast<float>(Rd[i]);
  for (int i = 0; i < 3; ++i) t[i] = static_cast<float>(td[i]);
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) Rw[r * 3 + c] = static_cast<float>(T[r * 4 + c]);
    tw[r] = static_cast<float>(T[r * 4 + 3]);
  }
}

// Frame index of a stamp (appends new stamps; stamps must not decrease while tracking is on).
int frameIndex(kb_handle* h, uint64_t stamp, uint32_t* idx) {
  if (stamp == 0) return fail(h, KB_ERR_INVALID, "stamp_ns must be > 0");
  if (stamp == h->stamps.back()) { *idx = static_cast<uint32_t>(h->stamps.size() - 1); return KB_OK; }
  if (stamp < h->stamps.back()) {
    if (h->map.with_tracking) return fail(h, KB_ERR_STATE, "stamps must be non-decreasing when tracking is enabled");
    *idx = static_cast<uint32_t>(h->stamps.size() - 1);
    return KB_OK;
  }
  h->stamps.push_back(stamp);
  *idx = static_cast<uint32_t>(h->stamps.size() - 1);
  DeviceMap& m = h->dm;
  if (m.next_pass && static_cast<int>(h->stamps.size()) + 2 > m.frame_capacity) {
    // grow the per-frame-index tables of the lazy tracking
    const int cap = m.frame_capacity * 2;
    uint32_t *np = nullptr, *am = nullptr;
    KB_CUDA(h, cudaStreamSynchronize(h->stream));
    KB_CUDA(h, devAlloc(&np, static_cast<size_t>(cap), 0));
    KB_CUDA(h, devAlloc(&am, static_cast<size_t>(cap), 0));
    KB_CUDA(h, cudaMemcpy(np, m.next_pass, sizeof(uint32_t) * m.frame_capacity, cudaMemcpyDeviceToDevice));
    KB_CUDA(h, cudaMemcpy(am, m.act_min, sizeof(uint32_t) * m.frame_capacity, cudaMemcpyDeviceToDevice));
    cudaFree(m.next_pass); cudaFree(m.act_min);
    m.next_pass = np; m.act_min = am; m.frame_capacity = cap;
  }
  return KB_OK;
}

int readCounters(kb_handle* h) {
  KB_CUDA(h, cudaMemcpyAsync(h->h_ctr, h->dm.counters, sizeof(int) * kCounterInts, cudaMemcpyDeviceToHost, h->stream));
  KB_CUDA(h, cudaStreamSynchronize(h->stream));
  return KB_OK;
}

int slotHwm(kb_handle* h, int* n) {
  // Upper bound on live slots without a sync: the pool capacity would do, but launching one CTA per
  // potential slot is wasteful, so we read the high-water mark (4 B, one sync).
  int st = readCounters(h);
  if (st != KB_OK) return st;
  *n = std::min(h->h_ctr[kCtrPoolHwm], h->dm.max_blocks);
  return KB_OK;
}

// Host M2-M4 on the per-pixel voxel keys of the last M1 launch (min_separation_distance <= 0, where one voxel can belong
// to several clusters). The bounding boxes come from the frame's vertex map when it has one (:396-397): host_vertex
// for host frames, else the copy kept on the device.
int buildMotionClustersOnHost(kb_handle* h, const float* host_vertex, int32_t* image_out) {
  const size_t px = static_cast<size_t>(h->cam.width) * h->cam.height;
  h->h_pixel_gidx.resize(px * 3);
  h->h_pixel_seed.resize(px);
  h->h_depth.resize(px);
  KB_CUDA(h, cudaMemcpyAsync(h->h_pixel_gidx.data(), h->d_pixel_gidx, sizeof(int3) * px, cudaMemcpyDeviceToHost, h->stream));
  KB_CUDA(h, cudaMemcpyAsync(h->h_pixel_seed.data(), h->d_pixel_seed, px, cudaMemcpyDeviceToHost, h->stream));
  KB_CUDA(h, cudaMemcpyAsync(h->h_depth.data(), h->mot_depth, sizeof(float) * px, cudaMemcpyDeviceToHost, h->stream));
  if (!host_vertex && h->motion_vertex) {
    h->h_vertex.resize(px * 3);
    KB_CUDA(h, cudaMemcpyAsync(h->h_vertex.data(), h->mot_vertex, sizeof(float) * 3 * px, cudaMemcpyDeviceToHost, h->stream));
    host_vertex = h->h_vertex.data();
  }
  KB_CUDA(h, cudaStreamSynchronize(h->stream));
  clusterMotion(h->motion_hp, h->h_pixel_gidx.data(), h->h_pixel_seed.data(), h->h_depth.data(), host_vertex,
                image_out, &h->motion);
  const auto& cl = h->motion.clusters;
  for (const MotionCluster& c : cl) {
    h->mcl_counts.push_back(static_cast<int32_t>(c.pixels.size() / 2));
    h->mcl_counts.push_back(static_cast<int32_t>(c.voxels.size() / 3));
    h->mcl_pixels.insert(h->mcl_pixels.end(), c.pixels.begin(), c.pixels.end());
    h->mcl_voxels.insert(h->mcl_voxels.end(), c.voxels.begin(), c.voxels.end());
    h->mcl_bbox.insert(h->mcl_bbox.end(), c.bbox, c.bbox + 6);
  }
  return KB_OK;
}

void freeMotionLists(kb_handle* h) {
  MotionLists& l = h->ml;
  cudaFree(l.pix_count); cudaFree(l.vox_count); cudaFree(l.pix_off); cudaFree(l.vox_off); cudaFree(l.pix_fill);
  cudaFree(l.vox_fill); cudaFree(l.box_min); cudaFree(l.box_max); cudaFree(l.bbox); cudaFree(l.vox_next);
  cudaFree(l.pixels_uv); cudaFree(l.vox_keys); cudaFree(l.vox_sorted); cudaFree(l.voxels_xyz);
  cudaFree(h->ml_gate); cudaFree(h->ml_sort_tmp);
  freeMotionTable(h->lt);
  l = MotionLists{};
  h->ml_gate = nullptr;
  h->ml_sort_tmp = nullptr;
  h->ml_clusters = h->ml_pixels = h->ml_voxels = h->ml_sort_bytes = 0;
}

// Cluster lists of the last device detection, built on the device from what the detection kept: its M1 output
// (d_pixel_gidx / d_pixel_seed, written only by the motion calls) and its vertex map or depth. Only the lists cross
// to the host.
int buildMotionListsOnDevice(kb_handle* h) {
  const size_t px = static_cast<size_t>(h->cam.width) * h->cam.height;
  const int K = h->h_mscal[kMsClusters];
  MotionLists& l = h->ml;
  MotionTable& t = h->lt;
  if (!t.keys || t.max_roots < static_cast<int>(px)) {  // first call, or the camera grew
    KB_CUDA(h, cudaStreamSynchronize(h->stream));
    freeMotionLists(h);
    int st = allocMotionTable(h, t, px);
    if (st != KB_OK) return st;
    const int one = 1;
    KB_CUDA(h, cudaMalloc(reinterpret_cast<void**>(&h->ml_gate), sizeof(int)));
    KB_CUDA(h, cudaMemcpy(h->ml_gate, &one, sizeof(int), cudaMemcpyHostToDevice));
    t.gate = h->ml_gate;
    KB_CUDA(h, cudaMalloc(reinterpret_cast<void**>(&l.vox_next), sizeof(int) * (static_cast<size_t>(t.mask) + 1)));
  }
  if (h->ml_clusters < static_cast<size_t>(K)) {
    KB_CUDA(h, cudaStreamSynchronize(h->stream));
    cudaFree(l.pix_count); cudaFree(l.vox_count); cudaFree(l.pix_off); cudaFree(l.vox_off); cudaFree(l.pix_fill);
    cudaFree(l.vox_fill); cudaFree(l.box_min); cudaFree(l.box_max); cudaFree(l.bbox);
    const size_t n = static_cast<size_t>(K);
    h->ml_clusters = 0;
    KB_CUDA(h, cudaMalloc(reinterpret_cast<void**>(&l.pix_count), sizeof(int) * n));
    KB_CUDA(h, cudaMalloc(reinterpret_cast<void**>(&l.vox_count), sizeof(int) * n));
    KB_CUDA(h, cudaMalloc(reinterpret_cast<void**>(&l.pix_off), sizeof(int) * (n + 1)));
    KB_CUDA(h, cudaMalloc(reinterpret_cast<void**>(&l.vox_off), sizeof(int) * (n + 1)));
    KB_CUDA(h, cudaMalloc(reinterpret_cast<void**>(&l.pix_fill), sizeof(int) * n));
    KB_CUDA(h, cudaMalloc(reinterpret_cast<void**>(&l.vox_fill), sizeof(int) * n));
    KB_CUDA(h, cudaMalloc(reinterpret_cast<void**>(&l.box_min), sizeof(unsigned int) * 3 * n));
    KB_CUDA(h, cudaMalloc(reinterpret_cast<void**>(&l.box_max), sizeof(unsigned int) * 3 * n));
    KB_CUDA(h, cudaMalloc(reinterpret_cast<void**>(&l.bbox), sizeof(float) * 6 * n));
    h->ml_clusters = n;
  }
  const int P = static_cast<int>(px);
  const int D = static_cast<int>(std::ceil(h->mot.min_separation_distance));
  launchMotionListCounts(t, l, h->d_pixel_gidx, h->d_pixel_seed, P, h->mot.neighbor_connectivity, D, h->mot.min_cluster_size,
                         h->mot.max_cluster_size, K, h->stream);
  KB_CUDA(h, cudaGetLastError());
  std::vector<int32_t> npix(K), nvox(K);
  int scal[kMsCount];
  KB_CUDA(h, cudaMemcpyAsync(npix.data(), l.pix_count, sizeof(int) * K, cudaMemcpyDeviceToHost, h->stream));
  KB_CUDA(h, cudaMemcpyAsync(nvox.data(), l.vox_count, sizeof(int) * K, cudaMemcpyDeviceToHost, h->stream));
  KB_CUDA(h, cudaMemcpyAsync(scal, t.scalars, sizeof(scal), cudaMemcpyDeviceToHost, h->stream));
  KB_CUDA(h, cudaStreamSynchronize(h->stream));
  if (scal[kMsClusters] != K) return fail(h, KB_ERR_STATE, "the cluster lists disagree with the detection");
  std::vector<int32_t> off(2 * (static_cast<size_t>(K) + 1));  // pixel offsets, then voxel offsets
  int32_t* poff = off.data();
  int32_t* voff = off.data() + K + 1;
  int64_t tp = 0, tv = 0;
  for (int c = 0; c < K; ++c) {
    poff[c] = static_cast<int32_t>(tp);
    voff[c] = static_cast<int32_t>(tv);
    tp += npix[c];
    tv += nvox[c];
    if (tp > INT32_MAX) return fail(h, KB_ERR_CAPACITY, "more than 2^31 cluster pixels");
  }
  poff[K] = static_cast<int32_t>(tp);
  voff[K] = static_cast<int32_t>(tv);
  if (h->ml_pixels < static_cast<size_t>(tp)) {
    cudaFree(l.pixels_uv);
    h->ml_pixels = 0;
    KB_CUDA(h, cudaMalloc(reinterpret_cast<void**>(&l.pixels_uv), sizeof(int32_t) * 2 * tp));
    h->ml_pixels = static_cast<size_t>(tp);
  }
  if (h->ml_voxels < static_cast<size_t>(tv)) {
    cudaFree(l.vox_keys); cudaFree(l.vox_sorted); cudaFree(l.voxels_xyz);
    h->ml_voxels = 0;
    KB_CUDA(h, cudaMalloc(reinterpret_cast<void**>(&l.vox_keys), sizeof(unsigned long long) * tv));
    KB_CUDA(h, cudaMalloc(reinterpret_cast<void**>(&l.vox_sorted), sizeof(unsigned long long) * tv));
    KB_CUDA(h, cudaMalloc(reinterpret_cast<void**>(&l.voxels_xyz), sizeof(int64_t) * 3 * tv));
    h->ml_voxels = static_cast<size_t>(tv);
  }
  KB_CUDA(h, cudaMemcpyAsync(l.pix_off, poff, sizeof(int32_t) * (K + 1), cudaMemcpyHostToDevice, h->stream));
  KB_CUDA(h, cudaMemcpyAsync(l.vox_off, voff, sizeof(int32_t) * (K + 1), cudaMemcpyHostToDevice, h->stream));
  MotionBoxParams b{};
  const MotionHostParams& mp = h->motion_hp;
  b.vertex = h->motion_vertex ? h->mot_vertex : nullptr;
  b.depth = h->mot_depth;
  b.W = mp.W; b.fx = mp.fx; b.fy = mp.fy; b.cx = mp.cx; b.cy = mp.cy;
  std::memcpy(b.Rw, mp.Rw, sizeof(b.Rw));
  std::memcpy(b.tw, mp.tw, sizeof(b.tw));
  size_t bytes = 0;
  KB_CUDA(h, launchMotionListFill(t, l, b, P, K, static_cast<int>(tv), nullptr, &bytes, h->stream));
  if (h->ml_sort_bytes < bytes) {
    cudaFree(h->ml_sort_tmp);
    h->ml_sort_bytes = 0;
    KB_CUDA(h, cudaMalloc(&h->ml_sort_tmp, bytes));
    h->ml_sort_bytes = bytes;
  }
  KB_CUDA(h, launchMotionListFill(t, l, b, P, K, static_cast<int>(tv), h->ml_sort_tmp, &bytes, h->stream));
  h->mcl_counts.resize(2 * static_cast<size_t>(K));
  for (int c = 0; c < K; ++c) { h->mcl_counts[2 * c] = npix[c]; h->mcl_counts[2 * c + 1] = nvox[c]; }
  h->mcl_pixels.resize(static_cast<size_t>(2 * tp));
  h->mcl_voxels.resize(static_cast<size_t>(3 * tv));
  h->mcl_bbox.resize(6 * static_cast<size_t>(K));
  KB_CUDA(h, cudaMemcpyAsync(h->mcl_pixels.data(), l.pixels_uv, sizeof(int32_t) * 2 * tp, cudaMemcpyDeviceToHost, h->stream));
  KB_CUDA(h, cudaMemcpyAsync(h->mcl_voxels.data(), l.voxels_xyz, sizeof(int64_t) * 3 * tv, cudaMemcpyDeviceToHost, h->stream));
  KB_CUDA(h, cudaMemcpyAsync(h->mcl_bbox.data(), l.bbox, sizeof(float) * 6 * K, cudaMemcpyDeviceToHost, h->stream));
  KB_CUDA(h, cudaStreamSynchronize(h->stream));
  h->motion_stale = false;
  return KB_OK;
}

}  // namespace

extern "C" {

int kb_abi_version(void) { return KB_ABI_VERSION; }

const char* kb_last_error(const kb_handle* h) { return h ? h->err.c_str() : "null handle"; }

int kb_block_owner(int32_t bx, int32_t by, int32_t bz, int nranks) {
  return nranks <= 1 ? 0 : blockOwner(bx, by, bz, nranks);
}

int kb_create(const kb_map_config* map, const kb_integrator_config* integ, const kb_tracking_config* trk,
              const kb_motion_config* mot, int device, kb_handle** out) {
  if (!map || !integ || !out) return KB_ERR_INVALID;
  *out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || device < 0 || device >= ndev) {
    cudaGetLastError();
    return KB_ERR_NO_DEVICE;  // the product path refuses to run without a GPU
  }
  if ((map->voxels_per_side != 8 && map->voxels_per_side != 16) || !(map->voxel_size > 0.f) ||
      !(map->truncation_distance > 0.f) || map->max_blocks <= 0)
    return KB_ERR_INVALID;
  if (integ->semantic_mode == KB_SEMANTICS_MLE && (integ->num_labels < 2 || integ->num_labels > KB_MAX_LABELS))
    return KB_ERR_INVALID;
  if (trk && (trk->neighbor_connectivity != 6 && trk->neighbor_connectivity != 18 && trk->neighbor_connectivity != 26))
    return KB_ERR_INVALID;
  if (trk && (!(trk->temporal_buffer > 0.f) || !(trk->temporal_window > 0.f) || trk->tsdf_occupancy_threshold == 0.f))
    return KB_ERR_INVALID;  // tracking_integrator.cpp:61-65
  if (mot && (mot->neighbor_connectivity != 6 && mot->neighbor_connectivity != 18 && mot->neighbor_connectivity != 26))
    return KB_ERR_INVALID;
  if (mot && (mot->max_cluster_size < mot->min_cluster_size || !(mot->max_range > 0.f)))
    return KB_ERR_INVALID;  // free_space_motion_detector.cpp:61-66

  auto* h = new kb_handle();
  h->map = *map;
  h->integ = *integ;
  if (trk) { h->trk = *trk; h->has_trk = true; }
  {
    const float cfg = trk ? trk->tsdf_occupancy_threshold : -1.5f;  // tracking_integrator.h:72
    h->trk_cfg_thr = cfg < 0 ? cfg * -map->voxel_size : cfg;        // tracking_integrator.cpp:136-138
  }
  if (mot) { h->mot = *mot; h->has_mot = true; }
  h->device = device;
  h->stamps.push_back(0);
  h->block_size = map->voxel_size * static_cast<float>(map->voxels_per_side);
  h->L = !map->with_semantics ? 0
         : integ->semantic_mode == KB_SEMANTICS_MLE ? integ->num_labels
         : integ->semantic_mode == KB_SEMANTICS_BINARY ? 2 : 0;
  if (integ->semantic_mode == KB_SEMANTICS_MLE) {
    // MLESemanticIntegrator constants (UP, SURVEY App. A.8), formed in double, rounded once.
    const double c = static_cast<double>(integ->label_confidence), N = static_cast<double>(integ->num_labels);
    h->mle_diag = static_cast<float>(std::log(c));
    h->mle_off = static_cast<float>(std::log((1.0 - c) / (N - 1.0)));
    h->mle_init = static_cast<float>(std::log(1.0 / N));
    for (int i = 0; i < KB_MAX_LABELS; ++i)
      if (integ->label_blocked[i]) h->blocked_mask |= 1ull << i;
  }

  DeviceMap& m = h->dm;
  m.vps = map->voxels_per_side;
  m.V = m.vps * m.vps * m.vps;
  m.max_blocks = map->max_blocks;
  m.max_sem = h->L > 0 ? (map->max_semantic_blocks > 0 ? map->max_semantic_blocks : map->max_blocks) : 0;
  m.Lp = h->L == 0 ? 0 : (integ->semantic_mode == KB_SEMANTICS_BINARY ? 2 : ((h->L + 3) / 4) * 4);
  uint32_t cap = 1024;
  while (cap < static_cast<uint32_t>(m.max_blocks) * 2u) cap <<= 1;
  m.hash_mask = cap - 1;

  int st = KB_OK;
  auto run = [&]() -> int {
    KB_CUDA(h, cudaSetDevice(device));
    KB_CUDA(h, cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
    h->own_stream = true;
    const size_t S = m.max_blocks, V = m.V;
    KB_CUDA(h, devAlloc(&m.hash_keys, cap, 0xFF));
    KB_CUDA(h, devAlloc(&m.hash_vals, cap, 0xFF));
    KB_CUDA(h, devAlloc(&m.counters, kCounterInts, 0));
    KB_CUDA(h, devAlloc(&m.free_list, S, 0));
    KB_CUDA(h, devAlloc(&m.block_index, S, 0));
    KB_CUDA(h, devAlloc(&m.block_flags, S, 0));
    KB_CUDA(h, devAlloc(&m.block_sem, S, 0xFF));
    KB_CUDA(h, devAlloc(&m.tsdf, S * V, 0));
    if (map->with_tracking) {
      KB_CUDA(h, devAlloc(&m.last_obs, S * V, 0));
      KB_CUDA(h, devAlloc(&m.last_occ, S * V, 0));
      KB_CUDA(h, devAlloc(&m.vflags, S * V, 0));
      KB_CUDA(h, devAlloc(&m.born_frame, S, 0));
      m.frame_capacity = 1 << 20;
      KB_CUDA(h, devAlloc(&m.next_pass, static_cast<size_t>(m.frame_capacity), 0));
      KB_CUDA(h, devAlloc(&m.act_min, static_cast<size_t>(m.frame_capacity), 0));
      KB_CUDA(h, devAlloc(&h->pending, S, 0));
    }
    if (h->L > 0) {
      const size_t Q = m.max_sem;
      KB_CUDA(h, devAlloc(&m.sem_free_list, Q, 0));
      KB_CUDA(h, devAlloc(&m.sem_label, Q * V, 0xFF));
      KB_CUDA(h, devAlloc(&m.sem_lik, Q * V * m.Lp, 0));
    }
    KB_CUDA(h, cudaMallocHost(reinterpret_cast<void**>(&h->h_ctr), sizeof(int) * kCounterInts));
    std::memset(h->h_ctr, 0, sizeof(int) * kCounterInts);
    KB_CUDA(h, cudaStreamCreateWithFlags(&h->copy_stream, cudaStreamNonBlocking));
    for (int i = 0; i < 2; ++i) {
      KB_CUDA(h, cudaEventCreateWithFlags(&h->stg_ready[i], cudaEventDisableTiming));
      KB_CUDA(h, cudaEventCreateWithFlags(&h->stg_consumed[i], cudaEventDisableTiming));
    }
    KB_CUDA(h, devAlloc(&h->work_slots, S, 0));
    KB_CUDA(h, devAlloc(&h->work_masks, S, 0));
    KB_CUDA(h, devAlloc(&h->work_upd, S, 0));
    h->batch.items_per_block = m.V / 128;
    KB_CUDA(h, devAlloc(&h->item_fmask, S * h->batch.items_per_block, 0));
    if (const char* e = std::getenv("KB_FUSE_ITEM_LIST")) h->use_item_list = e[0] == '1';
    h->rehash_threshold = (static_cast<size_t>(cap)) / 4;
    if (const char* e = std::getenv("KB_REHASH_TOMBSTONES")) h->rehash_threshold = static_cast<size_t>(std::max(1, std::atoi(e)));  // tests
    if (const char* e = std::getenv("KB_EVERFREE_V2")) h->everfree_v2 = e[0] == '1';
    if (const char* e = std::getenv("KB_MOTION_SPARSE")) h->motion_sparse = e[0] == '1';
    if (const char* e = std::getenv("KB_H2D_NARROW_LABELS")) h->narrow_labels = e[0] == '1';
    if (const char* e = std::getenv("KB_H2D_THREADS")) h->narrow_threads = std::max(1, std::atoi(e));
    if (const char* e = std::getenv("KB_PIPELINE")) h->pipelined = e[0] == '1';
    if (h->pipelined) {
      KB_CUDA(h, cudaStreamCreateWithFlags(&h->pre_stream, cudaStreamNonBlocking));
      for (int i = 0; i < 2; ++i) {
        KB_CUDA(h, cudaEventCreateWithFlags(&h->pre_done[i], cudaEventDisableTiming));
        KB_CUDA(h, cudaEventCreateWithFlags(&h->fuse_done[i], cudaEventDisableTiming));
      }
      KB_CUDA(h, cudaEventCreateWithFlags(&h->main_front, cudaEventDisableTiming));
      KB_CUDA(h, devAlloc(&h->work_slots2, S, 0));
      KB_CUDA(h, devAlloc(&h->work_masks2, S, 0));
      KB_CUDA(h, devAlloc(&h->work_upd2, S, 0));
      KB_CUDA(h, devAlloc(&h->item_fmask2, S * h->batch.items_per_block, 0));
    }
    if (const char* e = std::getenv("KB_FUSE_COOP")) h->fuse_coop = e[0] == '1' ? 1 : 0;
    if (const char* e = std::getenv("KB_FUSE_MLP")) h->mlp_group = e[0] == '2' ? 2 : (e[0] == '4' ? 4 : 0);
    if (h->use_item_list) {  // experiment, off by default (results are identical either way: only the item order changes)
      h->item_list_cap = static_cast<int>(std::min<size_t>(S * h->batch.items_per_block, size_t(1) << 28));
      KB_CUDA(h, devAlloc(&h->item_list, static_cast<size_t>(2 * kItemClasses) * h->item_list_cap, 0));  // 2 parities x classes
    }
    {
      cudaDeviceProp prop{};
      KB_CUDA(h, cudaGetDeviceProperties(&prop, device));
      h->everfree_grid = prop.multiProcessorCount * 4;
      h->cull_grid = prop.multiProcessorCount * 8;
      h->fuse_grid = prop.multiProcessorCount * fuseBlocksPerSm(m.vps, m.Lp);  // persistent CTAs of independent warps
      if (const char* e = std::getenv("KB_FUSE_CTAS_PER_SM")) {  // tuning knob (e.g. leave SM room for KB_PIPELINE's prologue)
        const int n = std::atoi(e);
        if (n > 0) h->fuse_grid = prop.multiProcessorCount * n;
      }
    }
    h->max_removed = m.max_blocks;
    KB_CUDA(h, devAlloc(&h->d_removed, static_cast<size_t>(h->max_removed), 0));
    KB_CUDA(h, cudaDeviceSynchronize());
    return KB_OK;
  };
  st = run();
  if (st != KB_OK) {
    std::fprintf(stderr, "kb_create: %s\n", h->err.c_str());
    kb_destroy(h);
    return st;
  }
  *out = h;
  return KB_OK;
}

int kb_destroy(kb_handle* h) {
  if (!h) return KB_OK;
  cudaSetDevice(h->device);
  if (h->stream) cudaStreamSynchronize(h->stream);
  DeviceMap& m = h->dm;
  cudaFree(m.hash_keys); cudaFree(m.hash_vals); cudaFree(m.counters); cudaFree(m.free_list);
  cudaFree(m.sem_free_list); cudaFree(m.block_index); cudaFree(m.block_flags); cudaFree(m.block_sem);
  cudaFree(m.tsdf); cudaFree(m.last_obs); cudaFree(m.last_occ); cudaFree(m.vflags);
  cudaFree(m.born_frame); cudaFree(m.next_pass); cudaFree(m.act_min); cudaFree(h->pending);
  cudaFree(m.sem_label); cudaFree(m.sem_lik); cudaFree(m.color); cudaFree(h->stg_color);
  cudaFree(h->xch.halo_mark); cudaFree(h->xch.publish); cudaFree(h->xch.ghost_keys); cudaFree(h->xch.ghost_vals);
  cudaFree(h->obj_depth); cudaFree(h->obj_label); cudaFree(h->d_object); cudaFree(h->d_flags_local);
  if (h->h_oscal) cudaFreeHost(h->h_oscal);
  cudaFree(h->trk_ids); cudaFree(h->trk_export); cudaFree(h->trk_counts); cudaFree(h->trk_sums); cudaFree(h->trk_present); cudaFree(h->trk_idlist);
  cudaFree(h->trk_keys); cudaFree(h->trk_of); cudaFree(h->trk_inter);
  cudaFree(h->stg_depth); cudaFree(h->stg_label); cudaFree(h->stg_mask); cudaFree(h->stg_object);
  cudaFree(h->stg_vertex); cudaFree(h->d_pixel_gidx); cudaFree(h->d_pixel_seed); cudaFree(h->d_removed);
  cudaFree(h->d_dynamic);
  freeMotionTable(h->mt);
  freeMotionLists(h);
  cudaFree(h->mot_vertex);
  if (h->h_mscal) cudaFreeHost(h->h_mscal);
  cudaFree(h->stg_depth16); cudaFree(h->stg_label8); cudaFree(h->mot_depth16);
  cudaFree(h->mot_depth); cudaFree(h->tile_max); cudaFree(h->work_slots); cudaFree(h->work_masks); cudaFree(h->work_upd); cudaFree(h->item_fmask); cudaFree(h->item_list);
  for (int i = 0; i < 2; ++i) {
    if (h->stg_ready[i]) cudaEventDestroy(h->stg_ready[i]);
    if (h->stg_consumed[i]) cudaEventDestroy(h->stg_consumed[i]);
  }
  if (h->copy_stream) { cudaStreamSynchronize(h->copy_stream); cudaStreamDestroy(h->copy_stream); }
  if (h->pin_label8) cudaFreeHost(h->pin_label8);
  if (h->pre_stream) { cudaStreamSynchronize(h->pre_stream); cudaStreamDestroy(h->pre_stream); }
  for (int i = 0; i < 2; ++i) {
    if (h->pre_done[i]) cudaEventDestroy(h->pre_done[i]);
    if (h->fuse_done[i]) cudaEventDestroy(h->fuse_done[i]);
  }
  if (h->main_front) cudaEventDestroy(h->main_front);
  cudaFree(h->work_slots2); cudaFree(h->work_masks2); cudaFree(h->work_upd2); cudaFree(h->item_fmask2);
  cudaFree(h->shard_table_dev);
  cudaFree(h->inst_counts); cudaFree(h->inst_bbox); cudaFree(h->inst_background); cudaFree(h->inst_keep); cudaFree(h->inst_bad);
  cudaFree(h->mesh_slots); cudaFree(h->mesh_cases); cudaFree(h->mesh_tri_count); cudaFree(h->mesh_tri_base);
  cudaFree(h->mesh_points); cudaFree(h->mesh_colors); cudaFree(h->mesh_labels);
  if (h->h_ctr) cudaFreeHost(h->h_ctr);
  if (h->own_stream && h->stream) cudaStreamDestroy(h->stream);
  delete h;
  return KB_OK;
}

int kb_set_stream(kb_handle* h, void* cuda_stream) {
  if (h) h->main_dirty = true;  // KB_PIPELINE: the next prologue must wait for this main-stream work
  if (!h) return KB_ERR_INVALID;
  KB_CUDA(h, cudaSetDevice(h->device));
  KB_CUDA(h, cudaStreamSynchronize(h->stream));
  if (h->own_stream) cudaStreamDestroy(h->stream);
  h->stream = static_cast<cudaStream_t>(cuda_stream);
  h->own_stream = false;
  return KB_OK;
}

int kb_synchronize(kb_handle* h) {
  if (!h) return KB_ERR_INVALID;
  KB_CUDA(h, cudaStreamSynchronize(h->copy_stream));
  KB_CUDA(h, cudaStreamSynchronize(h->stream));
  return KB_OK;
}

int kb_set_camera(kb_handle* h, const kb_camera* cam) {
  if (!h || !cam || cam->width <= 1 || cam->height <= 1 || !(cam->fx > 0.f) || !(cam->fy > 0.f))
    return fail(h, KB_ERR_INVALID, "invalid camera");
  KB_CUDA(h, cudaSetDevice(h->device));
  const bool same = h->has_cam && std::memcmp(&h->cam, cam, sizeof(kb_camera)) == 0;
  h->cam = *cam;
  h->has_cam = true;
  if (same) return KB_OK;
  const kb_camera& c = h->cam;
  BatchParams& p = h->batch;
  p.W = c.width; p.H = c.height;
  p.fx = c.fx; p.fy = c.fy; p.cx = c.cx; p.cy = c.cy;
  p.min_range = c.min_range; p.max_range = c.max_range;
  {
    // Inward unit normals of the four frustum side planes (same float expressions as the oracle).
    const float xl = (0.f - c.cx) / c.fx, xr = (static_cast<float>(c.width - 1) - c.cx) / c.fx;
    const float yt = (0.f - c.cy) / c.fy, yb = (static_cast<float>(c.height - 1) - c.cy) / c.fy;
    const float il = 1.f / std::sqrt(1.f + xl * xl), ir = 1.f / std::sqrt(1.f + xr * xr);
    const float it = 1.f / std::sqrt(1.f + yt * yt), ib = 1.f / std::sqrt(1.f + yb * yb);
    p.pl[0][0] = il;  p.pl[0][1] = -xl * il;
    p.pl[1][0] = -ir; p.pl[1][1] = xr * ir;
    p.pl[2][0] = it;  p.pl[2][1] = -yt * it;
    p.pl[3][0] = -ib; p.pl[3][1] = yb * ib;
  }
  p.voxel_size = h->map.voxel_size;
  p.block_size = h->block_size;
  p.trunc = h->map.truncation_distance;
  p.infl = h->block_size * 0.8660254f;
  p.use_dropoff = h->integ.use_weight_dropoff;
  p.dropoff_eps = h->integ.weight_dropoff_epsilon > 0.f ? h->integ.weight_dropoff_epsilon
                                                       : h->integ.weight_dropoff_epsilon * -h->map.voxel_size;
  p.constant_weight = h->integ.use_constant_weight;
  p.max_weight = h->integ.max_weight;
  p.interp = h->integ.interpolation_method;
  p.adaptive_thr = h->integ.adaptive_max_depth_difference;
  p.sem_mode = h->L > 0 ? h->integ.semantic_mode : KB_SEMANTICS_NONE;
  p.L = h->L;
  p.mle_diag = h->mle_diag; p.mle_off = h->mle_off; p.mle_init = h->mle_init;
  p.blocked_mask = h->blocked_mask;
  p.with_tracking = h->map.with_tracking;
  p.occ_thr = h->trk_cfg_thr;
  h->tile_stride = 0;
  for (int l = 0; l < kTileLevels; ++l) {
    p.lvl_tx[l] = l == 0 ? (c.width + 7) / 8 : (p.lvl_tx[l - 1] + 1) / 2;
    p.lvl_ty[l] = l == 0 ? (c.height + 7) / 8 : (p.lvl_ty[l - 1] + 1) / 2;
    p.lvl_off[l] = static_cast<int>(h->tile_stride);
    h->tile_stride += static_cast<size_t>(p.lvl_tx[l]) * p.lvl_ty[l];
  }
  p.work_slots = h->work_slots;
  p.work_masks = h->work_masks;
  p.work_upd = h->work_upd;
  p.item_fmask = h->item_fmask;
  p.max_work = h->dm.max_blocks;
  cudaFree(h->tile_max);
  h->tile_max = nullptr;
  KB_CUDA(h, devAlloc(&h->tile_max, h->tile_stride * kMaxBatch * 2, 0));  // two sets (KB_PIPELINE uses one per batch parity)
  return ensureMotionBuffers(h, static_cast<size_t>(c.width) * c.height);
}

int kb_get_debug_counters(kb_handle* h, int32_t* out, int32_t n) {
  if (!h || !out) return KB_ERR_INVALID;
  KB_CUDA(h, cudaSetDevice(h->device));
  int st = readCounters(h);
  if (st != KB_OK) return st;
  for (int i = 0; i < std::min<int>(n, kNumCounters); ++i) out[i] = h->h_ctr[i];
  return KB_OK;
}

int kb_set_culling(kb_handle* h, int enabled) {
  if (!h) return KB_ERR_INVALID;
  h->cull = enabled != 0;
  h->cull_forced = enabled == 2;
  return KB_OK;
}

int kb_set_shard(kb_handle* h, int rank, int nranks) {
  if (h) h->main_dirty = true;  // KB_PIPELINE: the next prologue must wait for this main-stream work
  if (!h || nranks < 1 || rank < 0 || rank >= nranks) return fail(h, KB_ERR_INVALID, "invalid shard");
  h->rank = rank;
  h->nranks = nranks;
  h->dm.shard_cell = 0;
  h->dm.shard_gx = h->dm.shard_gy = 1;
  h->dm.shard_table = nullptr;
  h->shard_table_host.clear();
  return KB_OK;
}

int kb_set_shard_cells(kb_handle* h, int rank, int nranks, int cell_blocks, int grid_x, int grid_y) {
  if (h) h->main_dirty = true;
  if (!h || nranks < 1 || rank < 0 || rank >= nranks || cell_blocks < 0 || (cell_blocks > 0 && (grid_x < 1 || grid_y < 1)))
    return fail(h, KB_ERR_INVALID, "invalid cell shard layout");
  h->rank = rank;
  h->nranks = nranks;
  h->dm.shard_cell = cell_blocks;
  h->dm.shard_gx = cell_blocks > 0 ? grid_x : 1;
  h->dm.shard_gy = cell_blocks > 0 ? grid_y : 1;
  h->dm.shard_table = nullptr;
  h->shard_table_host.clear();
  return KB_OK;
}

int kb_set_shard_table(kb_handle* h, int rank, int nranks, int cell_blocks, int32_t origin_cx, int32_t origin_cy, int32_t width,
                       int32_t height, const uint8_t* owners) {
  if (h) h->main_dirty = true;
  if (!h || nranks < 1 || nranks > 255 || rank < 0 || rank >= nranks || cell_blocks < 1 || width < 1 || height < 1 || !owners ||
      static_cast<long long>(width) * height > (1 << 24))
    return fail(h, KB_ERR_INVALID, "invalid cell table");
  KB_CUDA(h, cudaSetDevice(h->device));
  const size_t n = static_cast<size_t>(width) * height;
  for (size_t i = 0; i < n; ++i)
    if (owners[i] >= nranks) return fail(h, KB_ERR_INVALID, "cell table entry >= nranks");
  KB_CUDA(h, cudaStreamSynchronize(h->stream));
  cudaFree(h->shard_table_dev);
  h->shard_table_dev = nullptr;
  KB_CUDA(h, cudaMalloc(reinterpret_cast<void**>(&h->shard_table_dev), n));
  KB_CUDA(h, cudaMemcpy(h->shard_table_dev, owners, n, cudaMemcpyHostToDevice));
  h->shard_table_host.assign(owners, owners + n);
  h->rank = rank;
  h->nranks = nranks;
  h->dm.shard_cell = cell_blocks;
  // cells outside the table fall back to a periodic tiling of the ranks
  int gy = static_cast<int>(std::floor(std::sqrt(static_cast<double>(nranks))));
  while (nranks % gy) --gy;
  h->dm.shard_gx = nranks / gy;
  h->dm.shard_gy = gy;
  h->dm.shard_table = h->shard_table_dev;
  h->dm.tab_ox = origin_cx; h->dm.tab_oy = origin_cy; h->dm.tab_w = width; h->dm.tab_h = height;
  return KB_OK;
}

int kb_cell_owner(int32_t bx, int32_t by, int cell_blocks, int grid_x, int grid_y, int nranks) {
  if (nranks <= 1 || cell_blocks < 1 || grid_x < 1 || grid_y < 1) return 0;
  return cellOwner(bx, by, cell_blocks, grid_x, grid_y, nranks);
}

// ---- host-side frame scheduling arithmetic (kb_frame_owners / kb_frame_cells and their handle-free _host variants) --------
// A restatement of K0's candidate test (selectBlocksKernel: xform + inFrustum, same fp32 expressions; this translation unit is
// compiled without FMA contraction like the device code), evaluated with a 1 mm larger inflation so that the result is a
// superset of the device's selection.
namespace {
struct HostFrustum { float pl[4][2]; float infl, min_range, max_range, block_size; };
struct HostLayout { int nranks, cell, gx, gy; const uint8_t* table; int ox, oy, w, h; };

// The frustum side planes / inflation of a camera: the expressions of kb_set_camera.
void hostFrustum(const kb_camera& c, float block_size, HostFrustum* f) {
  const float xl = (0.f - c.cx) / c.fx, xr = (static_cast<float>(c.width - 1) - c.cx) / c.fx;
  const float yt = (0.f - c.cy) / c.fy, yb = (static_cast<float>(c.height - 1) - c.cy) / c.fy;
  const float il = 1.f / std::sqrt(1.f + xl * xl), ir = 1.f / std::sqrt(1.f + xr * xr);
  const float it = 1.f / std::sqrt(1.f + yt * yt), ib = 1.f / std::sqrt(1.f + yb * yb);
  f->pl[0][0] = il;  f->pl[0][1] = -xl * il;
  f->pl[1][0] = -ir; f->pl[1][1] = xr * ir;
  f->pl[2][0] = it;  f->pl[2][1] = -yt * it;
  f->pl[3][0] = -ib; f->pl[3][1] = yb * ib;
  f->infl = block_size * 0.8660254f;
  f->min_range = c.min_range;
  f->max_range = c.max_range;
  f->block_size = block_size;
}

void handleFrustum(const kb_handle* h, HostFrustum* f) {  // the values the kernels use
  const BatchParams& p = h->batch;
  std::memcpy(f->pl, p.pl, sizeof(f->pl));
  f->infl = p.infl; f->min_range = p.min_range; f->max_range = p.max_range; f->block_size = p.block_size;
}

int layoutOwner(const HostLayout& L, int x, int y, int z) {
  if (L.cell <= 0) return blockOwner(x, y, z, L.nranks);
  if (L.table) return tableOwner(L.table, L.ox, L.oy, L.w, L.h, L.cell, L.gx, L.gy, x, y, L.nranks);
  return cellOwner(x, y, L.cell, L.gx, L.gy, L.nranks);
}

inline bool candidateSelected(const HostFrustum& f, float infl, const float R[9], const float t[3], int bx, int by, int bz) {
  const float cx = (static_cast<float>(bx) + 0.5f) * f.block_size;
  const float cy = (static_cast<float>(by) + 0.5f) * f.block_size;
  const float cz = (static_cast<float>(bz) + 0.5f) * f.block_size;
  const float x = ((R[0] * cx + R[1] * cy) + R[2] * cz) + t[0];
  const float y = ((R[3] * cx + R[4] * cy) + R[5] * cz) + t[1];
  const float z = ((R[6] * cx + R[7] * cy) + R[8] * cz) + t[2];
  if (z < -infl) return false;
  const float r = std::sqrt((x * x + y * y) + z * z);
  if (r < f.min_range - infl || r > f.max_range + infl) return false;
  if (f.pl[0][0] * x + f.pl[0][1] * z < -infl) return false;
  if (f.pl[1][0] * x + f.pl[1][1] * z < -infl) return false;
  if (f.pl[2][0] * y + f.pl[2][1] * z < -infl) return false;
  if (f.pl[3][0] * y + f.pl[3][1] * z < -infl) return false;
  return true;
}

// returns false on a non-finite pose
bool frameBox(const HostFrustum& f, float infl, const kb_frame& fr, float R[9], float t[3], int lo[3], int hi[3]) {
  float Rw[9], tw[3];
  for (int k = 0; k < 16; ++k)
    if (!std::isfinite(fr.world_T_sensor[k])) return false;
  poseToFloat(fr.world_T_sensor, R, t, Rw, tw);
  const float reach = f.max_range + infl;
  const float inv = 1.f / f.block_size;
  for (int a = 0; a < 3; ++a) {
    lo[a] = static_cast<int>(std::floor((tw[a] - reach) * inv));
    hi[a] = static_cast<int>(std::floor((tw[a] + reach) * inv));
  }
  return true;
}

int frameOwnersImpl(const HostFrustum& f, const HostLayout& L, const kb_frame* frames, int32_t n_frames, uint32_t* owner_mask) {
  const uint32_t all = L.nranks >= 32 ? 0xffffffffu : ((1u << L.nranks) - 1u);
  const float infl = f.infl + 1e-3f;  // superset of the device's selection
  for (int i = 0; i < n_frames; ++i) {
    float R[9], t[3];
    int lo[3], hi[3];
    if (!frameBox(f, infl, frames[i], R, t, lo, hi)) return KB_ERR_INVALID;
    if (L.nranks == 1) { owner_mask[i] = 1u; continue; }
    uint32_t mask = 0;
    for (int bz = lo[2]; bz <= hi[2] && mask != all; ++bz)
      for (int by = lo[1]; by <= hi[1] && mask != all; ++by)
        for (int bx = lo[0]; bx <= hi[0]; ++bx) {
          const int owner = layoutOwner(L, bx, by, bz);
          if ((mask >> owner) & 1u) continue;
          if (!candidateSelected(f, infl, R, t, bx, by, bz)) continue;
          mask |= 1u << owner;
          if (mask == all) break;
        }
    owner_mask[i] = mask;
  }
  return KB_OK;
}

int frameCellsImpl(const HostFrustum& f, const kb_frame* frames, int32_t n_frames, int cell_blocks, int32_t origin_cx, int32_t origin_cy,
                   int32_t width, int32_t height, uint8_t* touched) {
  const float infl = f.infl + 1e-3f;
  const size_t cells = static_cast<size_t>(width) * height;
  std::memset(touched, 0, cells * static_cast<size_t>(n_frames));
  for (int i = 0; i < n_frames; ++i) {
    float R[9], t[3];
    int lo[3], hi[3];
    if (!frameBox(f, infl, frames[i], R, t, lo, hi)) return KB_ERR_INVALID;
    uint8_t* row = touched + cells * static_cast<size_t>(i);
    for (int by = lo[1]; by <= hi[1]; ++by) {
      const int cy = floorDiv(by, cell_blocks) - origin_cy;
      if (cy < 0 || cy >= height) continue;
      for (int bx = lo[0]; bx <= hi[0]; ++bx) {
        const int cx = floorDiv(bx, cell_blocks) - origin_cx;
        if (cx < 0 || cx >= width || row[cy * width + cx]) continue;
        for (int bz = lo[2]; bz <= hi[2]; ++bz)
          if (candidateSelected(f, infl, R, t, bx, by, bz)) { row[cy * width + cx] = 1; break; }
      }
    }
  }
  return KB_OK;
}

HostLayout handleLayout(const kb_handle* h) {
  const DeviceMap& m = h->dm;
  return HostLayout{h->nranks, m.shard_cell, m.shard_gx, m.shard_gy, h->shard_table_host.empty() ? nullptr : h->shard_table_host.data(),
                    m.tab_ox, m.tab_oy, m.tab_w, m.tab_h};
}
}  // namespace

int kb_frame_owners(kb_handle* h, const kb_frame* frames, int32_t n_frames, uint32_t* owner_mask) {
  if (!h || !frames || !owner_mask || n_frames < 0) return fail(h, KB_ERR_INVALID, "null argument");
  if (!h->has_cam) return fail(h, KB_ERR_STATE, "kb_set_camera must be called first");
  if (h->nranks > 32) return fail(h, KB_ERR_INVALID, "kb_frame_owners supports at most 32 ranks");
  HostFrustum f;
  handleFrustum(h, &f);
  const int st = frameOwnersImpl(f, handleLayout(h), frames, n_frames, owner_mask);
  return st == KB_OK ? KB_OK : fail(h, st, "non-finite sensor pose");
}

int kb_frame_cells(kb_handle* h, const kb_frame* frames, int32_t n_frames, int cell_blocks, int32_t origin_cx, int32_t origin_cy,
                   int32_t width, int32_t height, uint8_t* touched) {
  if (!h || !frames || !touched || n_frames < 0 || cell_blocks < 1 || width < 1 || height < 1) return fail(h, KB_ERR_INVALID, "invalid argument");
  if (!h->has_cam) return fail(h, KB_ERR_STATE, "kb_set_camera must be called first");
  HostFrustum f;
  handleFrustum(h, &f);
  const int st = frameCellsImpl(f, frames, n_frames, cell_blocks, origin_cx, origin_cy, width, height, touched);
  return st == KB_OK ? KB_OK : fail(h, st, "non-finite sensor pose");
}

// Handle-free variants (need no GPU): the scheduler of a sharded replay can run on a host without a device.
int kb_frame_owners_host(const kb_camera* camera, float voxel_size, int32_t voxels_per_side, const kb_shard_layout* layout,
                         const kb_frame* frames, int32_t n_frames, uint32_t* owner_mask) {
  if (!camera || !layout || !frames || !owner_mask || n_frames < 0 || !(voxel_size > 0.f) || voxels_per_side < 1 || layout->nranks < 1 ||
      layout->nranks > 32 || layout->cell_blocks < 0 || (layout->cell_blocks > 0 && (layout->grid_x < 1 || layout->grid_y < 1)))
    return KB_ERR_INVALID;
  HostFrustum f;
  hostFrustum(*camera, voxel_size * static_cast<float>(voxels_per_side), &f);
  const HostLayout L{layout->nranks, layout->cell_blocks, layout->grid_x, layout->grid_y, layout->table, layout->table_origin_cx,
                     layout->table_origin_cy, layout->table_width, layout->table_height};
  return frameOwnersImpl(f, L, frames, n_frames, owner_mask);
}

int kb_frame_cells_host(const kb_camera* camera, float voxel_size, int32_t voxels_per_side, const kb_frame* frames, int32_t n_frames,
                        int cell_blocks, int32_t origin_cx, int32_t origin_cy, int32_t width, int32_t height, uint8_t* touched) {
  if (!camera || !frames || !touched || n_frames < 0 || !(voxel_size > 0.f) || voxels_per_side < 1 || cell_blocks < 1 || width < 1 || height < 1)
    return KB_ERR_INVALID;
  HostFrustum f;
  hostFrustum(*camera, voxel_size * static_cast<float>(voxels_per_side), &f);
  return frameCellsImpl(f, frames, n_frames, cell_blocks, origin_cx, origin_cy, width, height, touched);
}

// Fuses up to kMaxBatch frames with one K0 + one K1 launch (plus one tile-max launch when culling).
static int integrateBatch(kb_handle* h, const kb_frame* frames, int n, int allocate_blocks) {
  const kb_camera& c = h->cam;
  const size_t px = static_cast<size_t>(c.width) * c.height;
  BatchParams& p = h->batch;  // persistent: camera / integrator fields are filled by kb_set_camera
  if (allocate_blocks && n > 1) {
    // K0 enumerates the union AABB of the batch's frusta, which assumes the frames are neighbours in space. Frames far
    // apart (a jump in the stream, an extractor batch spanning a long track) would blow that box up: split such batches
    // (results do not depend on how a frame sequence is cut into batches).
    const double reach = static_cast<double>(c.max_range) + static_cast<double>(h->block_size) * 0.8660254;
    const double inv = 1.0 / static_cast<double>(h->block_size);
    double lo[3] = {1e300, 1e300, 1e300}, hi[3] = {-1e300, -1e300, -1e300};
    for (int b = 0; b < n; ++b)
      for (int a = 0; a < 3; ++a) {
        const double t = frames[b].world_T_sensor[a * 4 + 3];
        lo[a] = std::min(lo[a], std::floor((t - reach) * inv));
        hi[a] = std::max(hi[a], std::floor((t + reach) * inv));
      }
    const double single = std::pow(2.0 * reach * inv + 2.0, 3.0);
    const double cells = (hi[0] - lo[0] + 1.0) * (hi[1] - lo[1] + 1.0) * (hi[2] - lo[2] + 1.0);
    if (!(cells <= 8.0 * single)) {  // also catches NaN poses: they end up alone and fail the frustum test
      int st = integrateBatch(h, frames, n / 2, allocate_blocks);
      if (st != KB_OK) return st;
      return integrateBatch(h, frames + n / 2, n - n / 2, allocate_blocks);
    }
  }
  p.n_frames = n;
  p.allocate = allocate_blocks ? 1 : 0;
  p.rank = h->rank;
  p.nranks = h->nranks;
  p.parity = h->parity;
  h->parity ^= 1;
  const int par = p.parity;
  // Short calls (the per-frame pipeline: detect -> integrate -> track) gain nothing from a second stream: their prologue
  // depends on the main-stream work right before it. They run entirely on the main stream with the first buffer set.
  const bool pipe = h->pipelined && n >= 4;
  if (!pipe) h->main_dirty = true;  // a later pipelined prologue must wait for this batch's main-stream kernels
  p.pipelined = pipe ? 1 : 0;
  p.fetch_ctr = (pipe && par) ? kCtrFetchB : kCtrFetch;
  p.items_ctr = (pipe && par) ? kCtrItemsB0 : kCtrItems0;
  p.work_slots = (pipe && par) ? h->work_slots2 : h->work_slots;
  p.work_masks = (pipe && par) ? h->work_masks2 : h->work_masks;
  p.work_upd = (pipe && par) ? h->work_upd2 : h->work_upd;
  p.item_fmask = (pipe && par) ? h->item_fmask2 : h->item_fmask;
  const size_t tile_set = (pipe && par) ? h->tile_stride * kMaxBatch : 0;
  // the culling stages cost ~3 extra launches: they pay off once a few frames share them
  p.cull = (h->cull && (n >= 4 || h->cull_forced)) ? 1 : 0;
  p.layers_per_item = n >= 8 ? 1 : 4;
  p.trk = h->pass;

  // ---- stage host images (double-buffered, on the copy stream so they overlap the previous batch)
  bool any_host = false, any_compact = false, any_color = false, any_host_color = false;
  for (int b = 0; b < n; ++b) {
    any_host |= frames[b].memory != KB_MEM_DEVICE;
    any_compact |= frames[b].depth_u16 != nullptr || frames[b].label_u8 != nullptr;
    any_color |= frames[b].color != nullptr;
    any_host_color |= frames[b].color != nullptr && frames[b].memory != KB_MEM_DEVICE;
  }
  p.has_color = any_color ? 1 : 0;
  // the compacted item lists pay for their extra launch only where items are many and uneven: long culled batches
  p.item_list = (h->use_item_list && p.cull && n >= 8 && !any_color)
                    ? h->item_list + ((pipe && par) ? static_cast<size_t>(kItemClasses) * h->item_list_cap : 0) : nullptr;
  p.item_list_cap = h->item_list_cap;
  p.mlp_group = h->mlp_group;
  p.coop = h->fuse_coop;
  if (any_color) {
    int st = ensureColorLayer(h);
    if (st == KB_OK && any_host_color) st = ensureColorStaging(h, px);
    if (st != KB_OK) return st;
  }
  const int set = h->stg_set;
  const bool use_staging = any_host || any_compact;
  if (use_staging) {
    int st = ensureStaging(h, px);
    if (st != KB_OK) return st;
    h->stg_set ^= 1;
    // wait until the kernels that last read this staging set are done
    KB_CUDA(h, cudaStreamWaitEvent(h->copy_stream, h->stg_consumed[set], 0));
  }
  // ---- optional host-side narrowing of i32 label images (KB_H2D_NARROW_LABELS)
  bool narrowed[kMaxBatch] = {false};
  bool any_narrowed = false;
  if (h->narrow_labels && any_host) {
    int cand[kMaxBatch], nc = 0;
    for (int b = 0; b < n; ++b)
      if (frames[b].memory != KB_MEM_DEVICE && frames[b].label && !frames[b].label_u8) cand[nc++] = b;
    if (nc > 0) {
      if (h->pin_label8_pixels < px) {
        KB_CUDA(h, cudaStreamSynchronize(h->copy_stream));
        if (h->pin_label8) cudaFreeHost(h->pin_label8);
        h->pin_label8 = nullptr;
        KB_CUDA(h, cudaMallocHost(reinterpret_cast<void**>(&h->pin_label8), px * kMaxBatch * 2));
        h->pin_label8_pixels = px;
      }
      // the H2D copies that last read this half of the pinned buffer (two batches ago) must be done; the copies of the
      // previous batch (other half) keep running while this batch is narrowed
      KB_CUDA(h, cudaEventSynchronize(h->stg_ready[set]));
      uint8_t* base8 = h->pin_label8 + static_cast<size_t>(set) * kMaxBatch * px;
      auto work = [&](int t, int T) {
        for (int k = t; k < nc; k += T) {
          const int b = cand[k];
          const int32_t* __restrict__ src = frames[b].label;
          uint8_t* __restrict__ dst = base8 + static_cast<size_t>(b) * px;
          int32_t acc = 0;
          for (size_t i = 0; i < px; ++i) { acc |= src[i]; dst[i] = static_cast<uint8_t>(src[i]); }
          narrowed[b] = (acc & ~0xFF) == 0;  // every id in 0..255 (negative ids set the high bits)
        }
      };
      const int T = std::max(1, std::min(h->narrow_threads, nc));
      if (T == 1) {
        work(0, 1);
      } else {
        std::vector<std::thread> pool;
        for (int t = 0; t < T; ++t) pool.emplace_back(work, t, T);
        for (auto& th : pool) th.join();
      }
      for (int b = 0; b < n; ++b) any_narrowed |= narrowed[b];
    }
  }
  int lo[3] = {INT32_MAX, INT32_MAX, INT32_MAX}, hi[3] = {INT32_MIN, INT32_MIN, INT32_MIN};
  for (int b = 0; b < n; ++b) {
    const kb_frame& f = frames[b];
    FrameView& v = p.f[b];
    float Rw[9], tw[3];
    poseToFloat(f.world_T_sensor, v.R, v.t, Rw, tw);
    if (h->map.with_tracking && f.stamp_ns <= h->last_pass_stamp)
      return fail(h, KB_ERR_STATE, "frames must be newer than the last kb_update_tracking stamp");
    uint32_t fidx = 0;
    int st = frameIndex(h, f.stamp_ns, &fidx);
    if (st != KB_OK) return st;
    v.frame_idx = fidx;
    v.target_id = f.object_target_id;
    const size_t off = (static_cast<size_t>(set) * kMaxBatch + b) * px;
    if (f.memory == KB_MEM_DEVICE) {
      v.depth = f.depth; v.label = f.label; v.mask = f.mask; v.object_image = f.object_image;
      v.depth16 = f.depth_u16; v.label8 = f.label_u8;
      v.color = f.color;
    } else {
      v.color = f.color ? h->stg_color + off * 3 : nullptr;
      v.depth = f.depth ? h->stg_depth + off : nullptr;
      v.label = f.label ? h->stg_label + off : nullptr;
      v.mask = f.mask ? h->stg_mask + off : nullptr;
      v.object_image = f.object_image ? h->stg_object + off : nullptr;
      v.depth16 = f.depth_u16 ? h->stg_depth16 + off : nullptr;
      v.label8 = (f.label_u8 || narrowed[b]) ? h->stg_label8 + off : nullptr;
    }
    v.depth_scale = f.depth_u16_scale;
    if (v.depth16) v.depth = h->stg_depth + off;   // expandFramesKernel fills these staging slots
    if (v.label8) v.label = h->stg_label + off;
    if (!v.depth) return fail(h, KB_ERR_INVALID, "frame without depth image");
    if (f.mask == KB_MASK_LAST_DETECTION)  // dynamic image of the last kb_detect_motion, still on the device
      v.mask = h->motion_have_image ? h->d_dynamic : nullptr;
    v.tiles = h->tile_max + tile_set + static_cast<size_t>(b) * h->tile_stride;
    if (allocate_blocks) {
      const float reach = c.max_range + p.infl;
      const float inv = 1.f / h->block_size;
      for (int a = 0; a < 3; ++a) {
        lo[a] = std::min(lo[a], static_cast<int>(std::floor((tw[a] - reach) * inv)));
        hi[a] = std::max(hi[a], static_cast<int>(std::floor((tw[a] + reach) * inv)));
      }
    }
  }
  if (any_host) {
    // H2D staging. Runs of frames whose host images are contiguous in memory (a ring buffer / video
    // tensor) are coalesced into one copy per image kind; separate cv::Mat buffers copy one by one.
    auto copyKind = [&](auto member, auto* staging, size_t per = 1) -> int {  // per: elements per pixel
      using T = std::remove_pointer_t<decltype(staging)>;
      const size_t img = px * per;
      int b = 0;
      while (b < n) {
        const T* src = (frames[b].memory == KB_MEM_DEVICE) ? nullptr : static_cast<const T*>(frames[b].*member);
        if (!src || static_cast<const void*>(src) == static_cast<const void*>(KB_MASK_LAST_DETECTION)) { ++b; continue; }
        int e = b + 1;
        while (e < n && frames[e].memory != KB_MEM_DEVICE && static_cast<const T*>(frames[e].*member) == src + static_cast<size_t>(e - b) * img) ++e;  // contiguous run
        T* dst = staging + (static_cast<size_t>(set) * kMaxBatch + b) * img;
        KB_CUDA(h, cudaMemcpyAsync(dst, src, static_cast<size_t>(e - b) * img * sizeof(T), cudaMemcpyHostToDevice, h->copy_stream));
        b = e;
      }
      return KB_OK;
    };
    int cst;
    if ((cst = copyKind(&kb_frame::depth, h->stg_depth)) != KB_OK) return cst;
    if (!any_narrowed) {
      if ((cst = copyKind(&kb_frame::label, h->stg_label)) != KB_OK) return cst;
    } else {
      // narrowed frames ship their pinned 8-bit copy (runs of consecutive frames in one transfer), the others their i32 image
      for (int b = 0; b < n;) {
        if (narrowed[b]) {
          int e = b + 1;
          while (e < n && narrowed[e]) ++e;
          const size_t o = (static_cast<size_t>(set) * kMaxBatch + b) * px;
          KB_CUDA(h, cudaMemcpyAsync(h->stg_label8 + o, h->pin_label8 + o, static_cast<size_t>(e - b) * px, cudaMemcpyHostToDevice, h->copy_stream));
          b = e;
        } else {
          if (frames[b].memory != KB_MEM_DEVICE && frames[b].label) {
            const size_t o = (static_cast<size_t>(set) * kMaxBatch + b) * px;
            KB_CUDA(h, cudaMemcpyAsync(h->stg_label + o, frames[b].label, px * sizeof(int32_t), cudaMemcpyHostToDevice, h->copy_stream));
          }
          ++b;
        }
      }
    }
    if ((cst = copyKind(&kb_frame::mask, h->stg_mask)) != KB_OK) return cst;
    if ((cst = copyKind(&kb_frame::object_image, h->stg_object)) != KB_OK) return cst;
    if ((cst = copyKind(&kb_frame::depth_u16, h->stg_depth16)) != KB_OK) return cst;
    if ((cst = copyKind(&kb_frame::label_u8, h->stg_label8)) != KB_OK) return cst;
    if (any_host_color && (cst = copyKind(&kb_frame::color, h->stg_color, 3)) != KB_OK) return cst;
    KB_CUDA(h, cudaEventRecord(h->stg_ready[set], h->copy_stream));
    KB_CUDA(h, cudaStreamWaitEvent(h->stream, h->stg_ready[set], 0));
  }
  if (allocate_blocks) {
    for (int a = 0; a < 3; ++a) { p.lo[a] = lo[a]; p.dims[a] = hi[a] - lo[a] + 1; }
    h->hwm_dirty = true;
  } else {
    if (h->hwm_dirty) {
      int st, nslots = 0;
      if ((st = slotHwm(h, &nslots)) != KB_OK) return st;
      h->hwm_cached = nslots;
      h->hwm_dirty = false;
    }
    p.n_slots = h->hwm_cached;
  }
  // All-compact batches are read in place (conversion per tap); mixed batches expand the compact frames first.
  any_compact = any_compact || any_narrowed;  // narrowed labels are widened by expandFramesKernel like label_u8 inputs
  bool all_compact = any_compact;
  for (int b = 0; b < n; ++b) all_compact = all_compact && frames[b].depth_u16 != nullptr && frames[b].label == nullptr;
  p.compact_taps = all_compact ? 1 : 0;
  // Per-frame image presence as bit words, so the fuse kernel's frame loop tests one bit instead of loading pointers. The
  // label image a frame is read through: the object image in BINARY mode, else the u8 labels of an all-compact batch
  // (read in place) or the i32 ones (caller's, staged, or expanded from u8).
  p.label_frames = 0;
  p.mask_frames = 0;
  for (int b = 0; b < n; ++b) {
    const FrameView& v = p.f[b];
    const void* lab = p.sem_mode == KB_SEMANTICS_BINARY ? static_cast<const void*>(v.object_image)
                      : all_compact                     ? static_cast<const void*>(v.label8)
                                                        : static_cast<const void*>(v.label);
    if (p.L > 0 && lab != nullptr) p.label_frames |= 1u << b;
    if (v.mask != nullptr) p.mask_frames |= 1u << b;
  }
  cudaStream_t ps = h->stream;
  if (pipe) {
    // The prologue of this batch goes to its own stream: it may run while the previous batch's fuse kernel is still
    // busy (that kernel only reads the other parity's lists). It has to wait for (a) the staged frames, (b) the fuse
    // kernel that last used this parity's buffers, (c) any other main-stream work enqueued since the last prologue
    // (tracking pass, block removal, box allocation ...: K0 reads what they write).
    ps = h->pre_stream;
    if (any_host) KB_CUDA(h, cudaStreamWaitEvent(ps, h->stg_ready[set], 0));
    KB_CUDA(h, cudaStreamWaitEvent(ps, h->fuse_done[par], 0));
    if (h->main_dirty) {
      KB_CUDA(h, cudaEventRecord(h->main_front, h->stream));
      KB_CUDA(h, cudaStreamWaitEvent(ps, h->main_front, 0));
      h->main_dirty = false;
    }
    KB_CUDA(h, cudaMemsetAsync(h->dm.counters + kCtrWork0 + par, 0, sizeof(int), ps));
    KB_CUDA(h, cudaMemsetAsync(h->dm.counters + p.fetch_ctr, 0, sizeof(int), ps));
  }
  if (!pipe && h->pipelined) {
    // Short batch between pipelined ones: the classic protocol expects the PREVIOUS batch's K0 to have zeroed this batch's
    // work counter, which pipelined batches (whose counters the host resets) do not do.
    KB_CUDA(h, cudaMemsetAsync(h->dm.counters + kCtrWork0 + par, 0, sizeof(int), ps));
  }
  if (any_compact && !all_compact) launchExpandFrames(p, ps);
  if (p.cull) launchTileMax(p, ps);
  launchSelectBlocks(h->dm, p, h->cull_grid, ps);
  if (pipe) {
    KB_CUDA(h, cudaEventRecord(h->pre_done[par], ps));
    KB_CUDA(h, cudaStreamWaitEvent(h->stream, h->pre_done[par], 0));
  }
  launchFuse(h->dm, p, h->fuse_grid, h->stream);
  if (pipe) KB_CUDA(h, cudaEventRecord(h->fuse_done[par], h->stream));
  KB_CUDA(h, cudaGetLastError());
  if (use_staging) KB_CUDA(h, cudaEventRecord(h->stg_consumed[set], h->stream));
  if (any_host) {
    // KB_MEM_HOST buffers are borrowed only for the duration of the call: wait for the copies (the
    // kernels keep running asynchronously and overlap the next call's copies). KB_MEM_HOST_ASYNC
    // callers keep their (pinned) buffers valid until kb_synchronize, so the copy engine never idles.
    bool must_wait = false;
    for (int b = 0; b < n; ++b) must_wait |= frames[b].memory == KB_MEM_HOST;
    if (must_wait) KB_CUDA(h, cudaStreamSynchronize(h->copy_stream));
  }
  h->ctr_dirty = true;
  return KB_OK;
}

int kb_integrate_frames(kb_handle* h, const kb_frame* frames, int32_t n_frames, int allocate_blocks,
                        kb_frame_stats* stats) {
  if (!h || !frames || n_frames < 0) return fail(h, KB_ERR_INVALID, "null frames");
  if (!h->has_cam) return fail(h, KB_ERR_STATE, "kb_set_camera must be called first");
  for (int i = 0; i < n_frames; ++i) {
    if (!frames[i].depth && !frames[i].depth_u16) return fail(h, KB_ERR_INVALID, "frame without depth image");
    for (int k = 0; k < 16; ++k)
      if (!std::isfinite(frames[i].world_T_sensor[k])) return fail(h, KB_ERR_INVALID, "non-finite sensor pose");
  }
  KB_CUDA(h, cudaSetDevice(h->device));
  int st;
  if (stats && h->ctr_dirty) {
    if ((st = readCounters(h)) != KB_OK) return st;
    std::memcpy(h->prev_ctr, h->h_ctr, sizeof(h->prev_ctr));
    h->ctr_dirty = false;
  }
  // Caller-owned stream (kb_set_stream): whatever the caller enqueued on it before this call (e.g. the copy / kernel that
  // produces device-resident frames) must precede the call's work. The prologue of a pipelined batch runs on an internal
  // stream, so the first batch of every call orders itself behind the caller's stream; the batches inside the call pipeline.
  if (!h->own_stream) h->main_dirty = true;
  for (int i = 0; i < n_frames; i += kMaxBatch) {
    if ((st = integrateBatch(h, frames + i, std::min(kMaxBatch, n_frames - i), allocate_blocks)) != KB_OK) return st;
  }
  if (stats) {
    if ((st = readCounters(h)) != KB_OK) return st;
    const int* c1 = h->h_ctr;
    const int* c0 = h->prev_ctr;
    auto d = [&](int k) { return static_cast<int32_t>(static_cast<uint32_t>(c1[k]) - static_cast<uint32_t>(c0[k])); };
    stats->blocks_in_frustum = d(kCtrFrustum);
    stats->blocks_allocated = d(kCtrAllocated);
    stats->blocks_updated = d(kCtrBlocksUpdated);
    stats->voxels_updated = d(kCtrVoxelsUpdated);
    stats->voxels_in_band = d(kCtrVoxelsBand);
    stats->voxels_semantic = d(kCtrVoxelsSemantic);
    stats->total_blocks = c1[kCtrLiveBlocks];
    stats->capacity_exceeded = c1[kCtrCapacityExceeded];
    std::memcpy(h->prev_ctr, h->h_ctr, sizeof(h->prev_ctr));
    h->ctr_dirty = false;
    if (c1[kCtrCapacityExceeded]) return fail(h, KB_ERR_CAPACITY, "block / semantic pool exhausted");
  }
  return KB_OK;
}

int kb_integrate_frame(kb_handle* h, const kb_frame* f, int allocate_blocks, kb_frame_stats* stats) {
  return kb_integrate_frames(h, f, f ? 1 : 0, allocate_blocks, stats);
}

int kb_get_totals(kb_handle* h, kb_frame_stats* t) {
  if (!h || !t) return KB_ERR_INVALID;
  KB_CUDA(h, cudaSetDevice(h->device));
  int st = readCounters(h);
  if (st != KB_OK) return st;
  const int* c = h->h_ctr;
  t->blocks_in_frustum = c[kCtrFrustum];
  t->blocks_allocated = c[kCtrAllocated];
  t->blocks_updated = c[kCtrBlocksUpdated];
  t->voxels_updated = c[kCtrVoxelsUpdated];
  t->voxels_in_band = c[kCtrVoxelsBand];
  t->voxels_semantic = c[kCtrVoxelsSemantic];
  t->total_blocks = c[kCtrLiveBlocks];
  t->capacity_exceeded = c[kCtrCapacityExceeded];
  return KB_OK;
}

int kb_get_totals64(kb_handle* h, kb_totals64* t) {
  if (!h || !t) return KB_ERR_INVALID;
  KB_CUDA(h, cudaSetDevice(h->device));
  int st = readCounters(h);
  if (st != KB_OK) return st;
  const unsigned long long* c = totals64(h->h_ctr);
  t->blocks_in_frustum = c[kTotFrustum];
  t->blocks_allocated = c[kTotAllocated];
  t->blocks_updated = c[kTotBlocksUpdated];
  t->voxels_updated = c[kTotVoxelsUpdated];
  t->voxels_in_band = c[kTotVoxelsBand];
  t->voxels_semantic = c[kTotVoxelsSemantic];
  t->block_frame_pairs = c[kTotPairs];
  t->total_blocks = static_cast<uint64_t>(std::max(h->h_ctr[kCtrLiveBlocks], 0));
  t->capacity_exceeded = static_cast<uint64_t>(h->h_ctr[kCtrCapacityExceeded]);
  t->frames = static_cast<uint64_t>(h->stamps.size() - 1);
  return KB_OK;
}

int kb_map_checksum(kb_handle* h, uint64_t out[4]) {
  if (!h || !out) return KB_ERR_INVALID;
  KB_CUDA(h, cudaSetDevice(h->device));
  int st, n = 0;
  if ((st = slotHwm(h, &n)) != KB_OK) return st;
  unsigned long long *d_stamps = nullptr, *d_out = nullptr;
  auto body = [&]() -> int {
    KB_CUDA(h, cudaMalloc(&d_stamps, sizeof(uint64_t) * h->stamps.size()));
    KB_CUDA(h, cudaMalloc(&d_out, sizeof(uint64_t) * 4));
    KB_CUDA(h, cudaMemcpyAsync(d_stamps, h->stamps.data(), sizeof(uint64_t) * h->stamps.size(), cudaMemcpyHostToDevice, h->stream));
    KB_CUDA(h, cudaMemsetAsync(d_out, 0, sizeof(uint64_t) * 4, h->stream));
    launchChecksum(h->dm, n, d_stamps, d_out, h->stream);
    KB_CUDA(h, cudaGetLastError());
    KB_CUDA(h, cudaMemcpyAsync(out, d_out, sizeof(uint64_t) * 4, cudaMemcpyDeviceToHost, h->stream));
    KB_CUDA(h, cudaStreamSynchronize(h->stream));
    return KB_OK;
  };
  st = body();
  cudaFree(d_stamps);
  cudaFree(d_out);
  h->main_dirty = true;
  return st;
}

// Parameters of the tracking pass at `stamp_ns` (no launch, no state change besides the stamp table).
static int trackingParams(kb_handle* h, uint64_t stamp_ns, TrackingParams* out) {
  if (stamp_ns <= h->last_pass_stamp) return fail(h, KB_ERR_STATE, "tracking stamps must increase");
  uint32_t fidx = 0;
  int st = frameIndex(h, stamp_ns, &fidx);
  if (st != KB_OK) return st;
  // The reference compares stamps in double seconds (tracking_integrator.cpp:238,250). Stamps are
  // strictly increasing in the frame-index table, so each predicate is a threshold on the index.
  const double now = toSeconds(stamp_ns);
  const double t_active = now - h->trk.temporal_window;
  const double t_free = now - h->trk.temporal_buffer;
  auto firstAtLeast = [&](double thr) {  // first frame index (>= 1) with toSeconds(stamp) >= thr
    auto it = std::partition_point(h->stamps.begin() + 1, h->stamps.end(),
                                   [&](uint64_t s) { return toSeconds(s) < thr; });
    return static_cast<uint32_t>(it - h->stamps.begin());
  };
  TrackingParams p{};
  p.prev_pass = h->pass.k_last;
  p.ev.k_last = fidx;
  p.ev.act_min = firstAtLeast(t_active);  // last_obs >= act_min <=> toSeconds(last_obs) >= now - window
  // a never-observed voxel (stamp 0) is "active" at pass k iff 0.0 >= toSeconds(stamp_k) - window; the
  // passes for which that holds are a prefix of the (increasing) stamp table
  {
    auto it = std::partition_point(h->stamps.begin() + 1, h->stamps.end(), [&](uint64_t s) {
      return 0.0 >= toSeconds(s) - h->trk.temporal_window;
    });
    p.ev.zero_max = static_cast<uint32_t>(it - h->stamps.begin()) - 1;
  }
  p.ev.free_max = firstAtLeast(t_free);   // last_occ < free_max <=> toSeconds(last_occ) < now - buffer
  p.ev.zero_free = 0.0 < t_free;
  p.connectivity = h->trk.neighbor_connectivity;
  p.n_slots = h->dm.max_blocks;
  p.pending = h->pending;
  p.rank = h->rank;
  p.nranks = h->nranks;
  p.everfree_v2 = h->everfree_v2 ? 1 : 0;
  *out = p;
  return KB_OK;
}

static int updateTrackingImpl(kb_handle* h, uint64_t stamp_ns) {
  if (h) h->main_dirty = true;  // KB_PIPELINE: the next prologue must wait for this main-stream work
  if (h->open_pass_state != 0) return fail(h, KB_ERR_STATE, "a sharded tracking pass is open (kb_tracking_finish missing)");
  TrackingParams p{};
  int st = trackingParams(h, stamp_ns, &p);
  if (st != KB_OK) return st;
  launchTrackingPass(h->dm, p, h->everfree_grid, h->stream);
  KB_CUDA(h, cudaGetLastError());
  h->pass = p.ev;
  h->last_pass_stamp = stamp_ns;
  return KB_OK;
}

int kb_update_tracking(kb_handle* h, uint64_t stamp_ns) {
  if (!h) return KB_ERR_INVALID;
  if (!h->has_trk || !h->map.with_tracking) return fail(h, KB_ERR_STATE, "tracking not configured");
  KB_CUDA(h, cudaSetDevice(h->device));
  return updateTrackingImpl(h, stamp_ns);
}

int kb_set_shard_capacity(kb_handle* h, int32_t pending_capacity, int32_t halo_capacity) {
  if (!h || pending_capacity <= 0 || halo_capacity <= 0) return fail(h, KB_ERR_INVALID, "invalid shard capacity");
  if (h->open_pass_state != 0) return fail(h, KB_ERR_STATE, "a sharded tracking pass is open");
  h->cap_pending = pending_capacity;
  h->cap_halo = halo_capacity;
  return KB_OK;
}

int kb_shard_buffer_sizes(kb_handle* h, int64_t* pending_bytes, int64_t* halo_bytes, int64_t* pixel_flag_bytes) {
  if (!h) return KB_ERR_INVALID;
  ShardExchange x{};
  x.cap_pending = h->cap_pending; x.cap_halo = h->cap_halo; x.mask_words = h->dm.V / 32;
  if (pending_bytes) *pending_bytes = static_cast<int64_t>(x.pending_stride()) * 4;
  if (halo_bytes) *halo_bytes = static_cast<int64_t>(x.halo_stride()) * 4;
  if (pixel_flag_bytes) *pixel_flag_bytes = h->has_cam ? static_cast<int64_t>(h->cam.width) * h->cam.height : 0;
  return KB_OK;
}

int kb_tracking_begin(kb_handle* h, uint64_t stamp_ns, void* pending_out) {
  if (h) h->main_dirty = true;  // KB_PIPELINE: the next prologue must wait for this main-stream work
  if (!h || !pending_out) return fail(h, KB_ERR_INVALID, "null argument");
  if (!h->has_trk || !h->map.with_tracking) return fail(h, KB_ERR_STATE, "tracking not configured");
  if (h->open_pass_state != 0) return fail(h, KB_ERR_STATE, "kb_tracking_begin: the previous pass was not finished");
  KB_CUDA(h, cudaSetDevice(h->device));
  int st = ensureShardBuffers(h);
  if (st != KB_OK) return st;
  TrackingParams p{};
  if ((st = trackingParams(h, stamp_ns, &p)) != KB_OK) return st;
  launchTrackingBegin(h->dm, p, h->xch, static_cast<int32_t*>(pending_out), h->stream);
  KB_CUDA(h, cudaGetLastError());
  h->open_pass = p;
  h->open_pass_stamp = stamp_ns;
  h->open_pass_state = 1;
  return KB_OK;
}

static int makePeers(kb_handle* h, void* const* ptrs, int32_t n, PeerBuffers* out) {
  if (!ptrs || n != h->nranks || n > kMaxPeers) return fail(h, KB_ERR_INVALID, "peer buffer list must have one entry per rank (<= 16)");
  out->n = n;
  for (int i = 0; i < kMaxPeers; ++i) out->p[i] = i < n ? ptrs[i] : nullptr;
  for (int i = 0; i < n; ++i)
    if (!ptrs[i]) return fail(h, KB_ERR_INVALID, "null peer buffer");
  return KB_OK;
}

int kb_tracking_begin_peers(kb_handle* h, uint64_t stamp_ns, void* const* peer_all_pending, int32_t n_peers) {
  if (!h) return KB_ERR_INVALID;
  if (!h->has_trk || !h->map.with_tracking) return fail(h, KB_ERR_STATE, "tracking not configured");
  if (h->open_pass_state != 0) return fail(h, KB_ERR_STATE, "kb_tracking_begin: the previous pass was not finished");
  h->main_dirty = true;
  KB_CUDA(h, cudaSetDevice(h->device));
  int st = ensureShardBuffers(h);
  if (st != KB_OK) return st;
  PeerBuffers peers{};
  if ((st = makePeers(h, peer_all_pending, n_peers, &peers)) != KB_OK) return st;
  TrackingParams p{};
  if ((st = trackingParams(h, stamp_ns, &p)) != KB_OK) return st;
  launchTrackingBeginPeers(h->dm, p, h->xch, peers, h->stream);
  KB_CUDA(h, cudaGetLastError());
  h->open_pass = p;
  h->open_pass_stamp = stamp_ns;
  h->open_pass_state = 1;
  return KB_OK;
}

int kb_tracking_pack_halo_peers(kb_handle* h, const void* all_pending, void* const* peer_all_halo, int32_t n_peers) {
  if (!h || !all_pending) return fail(h, KB_ERR_INVALID, "null argument");
  if (h->open_pass_state != 1) return fail(h, KB_ERR_STATE, "kb_tracking_pack_halo needs kb_tracking_begin first");
  h->main_dirty = true;
  KB_CUDA(h, cudaSetDevice(h->device));
  PeerBuffers peers{};
  int st = makePeers(h, peer_all_halo, n_peers, &peers);
  if (st != KB_OK) return st;
  launchHaloPackPeers(h->dm, h->open_pass, h->xch, static_cast<const int32_t*>(all_pending), peers, h->stream);
  KB_CUDA(h, cudaGetLastError());
  h->open_pass_state = 2;
  return KB_OK;
}

int kb_tracking_pack_halo(kb_handle* h, const void* all_pending, void* halo_out) {
  if (h) h->main_dirty = true;  // KB_PIPELINE: the next prologue must wait for this main-stream work
  if (!h || !all_pending || !halo_out) return fail(h, KB_ERR_INVALID, "null argument");
  if (h->open_pass_state != 1) return fail(h, KB_ERR_STATE, "kb_tracking_pack_halo needs kb_tracking_begin first");
  KB_CUDA(h, cudaSetDevice(h->device));
  launchHaloPack(h->dm, h->open_pass, h->xch, static_cast<const int32_t*>(all_pending), static_cast<int32_t*>(halo_out), h->stream);
  KB_CUDA(h, cudaGetLastError());
  h->open_pass_state = 2;
  return KB_OK;
}

int kb_tracking_finish(kb_handle* h, const void* all_pending, const void* all_halo) {
  if (h) h->main_dirty = true;  // KB_PIPELINE: the next prologue must wait for this main-stream work
  if (!h || !all_pending || !all_halo) return fail(h, KB_ERR_INVALID, "null argument");
  if (h->open_pass_state != 2) return fail(h, KB_ERR_STATE, "kb_tracking_finish needs kb_tracking_pack_halo first");
  KB_CUDA(h, cudaSetDevice(h->device));
  TrackingParams p = h->open_pass;
  p.ghost_bits = static_cast<const int32_t*>(all_halo);
  p.ghost_keys = h->xch.ghost_keys;
  p.ghost_vals = h->xch.ghost_vals;
  p.ghost_mask = h->xch.ghost_mask;
  launchTrackingFinish(h->dm, p, h->xch, static_cast<const int32_t*>(all_pending), static_cast<const int32_t*>(all_halo),
                       h->everfree_grid, h->stream);
  KB_CUDA(h, cudaGetLastError());
  h->pass = p.ev;
  h->last_pass_stamp = h->open_pass_stamp;
  h->open_pass_state = 0;
  h->ctr_dirty = true;
  return KB_OK;
}

int kb_reset_inactive(kb_handle* h, int32_t* removed_xyz, int32_t max_removed, int32_t* n_removed) {
  if (h) h->main_dirty = true;  // KB_PIPELINE: the next prologue must wait for this main-stream work
  if (!h) return KB_ERR_INVALID;
  if (!h->map.with_tracking) { if (n_removed) *n_removed = 0; return KB_OK; }  // no tracking blocks
  KB_CUDA(h, cudaSetDevice(h->device));
  int st, nslots = 0;
  if ((st = slotHwm(h, &nslots)) != KB_OK) return st;
  KB_CUDA(h, cudaMemsetAsync(h->dm.counters + kCtrRemoved, 0, sizeof(int), h->stream));
  launchResetInactive(h->dm, h->pass, nslots, h->d_removed, h->max_removed, h->stream);
  KB_CUDA(h, cudaGetLastError());
  if ((st = readCounters(h)) != KB_OK) return st;
  const int n = std::min(h->h_ctr[kCtrRemoved], h->max_removed);
  std::vector<int3> host(static_cast<size_t>(std::max(n, 0)));
  if (n > 0) KB_CUDA(h, cudaMemcpy(host.data(), h->d_removed, sizeof(int3) * n, cudaMemcpyDeviceToHost));
  std::sort(host.begin(), host.end(), [](const int3& a, const int3& b) {
    return a.x != b.x ? a.x < b.x : (a.y != b.y ? a.y < b.y : a.z < b.z);
  });
  h->hwm_dirty = true;
  // every removal leaves a tombstone; rebuild the table before they crowd out its empty entries
  h->tombstones_ub += static_cast<size_t>(std::max(h->h_ctr[kCtrRemoved], 0));
  if (h->tombstones_ub >= h->rehash_threshold) {
    launchRehash(h->dm, nslots, h->stream);
    KB_CUDA(h, cudaGetLastError());
    h->tombstones_ub = 0;
  }
  if (n_removed) *n_removed = static_cast<int32_t>(host.size());
  if (removed_xyz)
    for (int i = 0; i < std::min<int>(max_removed, host.size()); ++i) {
      removed_xyz[i * 3 + 0] = host[i].x; removed_xyz[i * 3 + 1] = host[i].y; removed_xyz[i * 3 + 2] = host[i].z;
    }
  return KB_OK;
}

int kb_mark_all_inactive(kb_handle* h) {
  if (h) h->main_dirty = true;  // KB_PIPELINE: the next prologue must wait for this main-stream work
  if (!h) return KB_ERR_INVALID;
  KB_CUDA(h, cudaSetDevice(h->device));
  int st, n = 0;
  if ((st = slotHwm(h, &n)) != KB_OK) return st;
  launchMarkAllInactive(h->dm, n, h->stream);
  KB_CUDA(h, cudaGetLastError());
  return KB_OK;
}

int kb_clear_updated(kb_handle* h) {
  if (h) h->main_dirty = true;  // KB_PIPELINE: the next prologue must wait for this main-stream work
  if (!h) return KB_ERR_INVALID;
  KB_CUDA(h, cudaSetDevice(h->device));
  int st, n = 0;
  if ((st = slotHwm(h, &n)) != KB_OK) return st;
  launchClearUpdated(h->dm, n, h->stream);
  KB_CUDA(h, cudaGetLastError());
  return KB_OK;
}

int kb_allocate_box(kb_handle* h, const int32_t mn[3], const int32_t mx[3]) {
  if (h) h->main_dirty = true;  // KB_PIPELINE: the next prologue must wait for this main-stream work
  if (!h || !mn || !mx) return KB_ERR_INVALID;
  KB_CUDA(h, cudaSetDevice(h->device));
  const int3 lo = make_int3(mn[0], mn[1], mn[2]);
  const int3 dims = make_int3(mx[0] - mn[0] + 1, mx[1] - mn[1] + 1, mx[2] - mn[2] + 1);
  if (dims.x <= 0 || dims.y <= 0 || dims.z <= 0) return KB_OK;
  if (static_cast<double>(dims.x) * dims.y * dims.z > static_cast<double>(h->dm.max_blocks) * (h->nranks > 1 ? 2.0 * h->nranks : 1.0))
    return fail(h, KB_ERR_CAPACITY, "kb_allocate_box: the box holds more blocks than the pool");
  // blocks allocated now are seen by tracking passes with a frame index >= born
  const uint32_t last_idx = static_cast<uint32_t>(h->stamps.size() - 1);
  const uint32_t born = std::max(last_idx, h->pass.k_last + 1);
  launchAllocateBox(h->dm, lo, dims, h->rank, h->nranks, born, h->stream);
  h->hwm_dirty = true;
  KB_CUDA(h, cudaGetLastError());
  int st = readCounters(h);
  if (st != KB_OK) return st;
  if (h->h_ctr[kCtrCapacityExceeded]) return fail(h, KB_ERR_CAPACITY, "block pool exhausted");
  return KB_OK;
}

int kb_scan_object_confidence(kb_handle* h, float min_confidence, int32_t min_observations, int32_t* n_erased) {
  if (h) h->main_dirty = true;  // KB_PIPELINE: the next prologue must wait for this main-stream work
  if (!h) return KB_ERR_INVALID;
  if (h->L != 2 || h->integ.semantic_mode != KB_SEMANTICS_BINARY)
    return fail(h, KB_ERR_STATE, "kb_scan_object_confidence needs binary semantics");
  if (h->map.with_tracking)
    return fail(h, KB_ERR_STATE, "kb_scan_object_confidence is for tracking-less extraction maps (mesh_object_extractor.cpp:210)");
  KB_CUDA(h, cudaSetDevice(h->device));
  int st, n = 0;
  if ((st = slotHwm(h, &n)) != KB_OK) return st;
  const int before = h->h_ctr[kCtrErased];
  launchScanConfidence(h->dm, min_confidence, static_cast<float>(min_observations), h->map.truncation_distance, n, h->stream);
  KB_CUDA(h, cudaGetLastError());
  if ((st = readCounters(h)) != KB_OK) return st;
  if (n_erased) *n_erased = h->h_ctr[kCtrErased] - before;
  return KB_OK;
}

// M1 launch shared by kb_detect_motion and kb_spin_once: stages depth / vertex map, resets the seed counter,
// enqueues the per-pixel lookup and records what lazily built cluster lists need (depth, vertex map, parameters).
static int enqueueMotionLookup(kb_handle* h, const kb_frame* f, uint8_t* shard_flags = nullptr) {
  if (h) h->main_dirty = true;  // KB_PIPELINE: the next prologue must wait for this main-stream work
  const kb_camera& c = h->cam;
  const size_t px = static_cast<size_t>(c.width) * c.height;
  MotionParams p{};
  float R[9], t[3];
  poseToFloat(f->world_T_sensor, R, t, p.Rw, p.tw);
  p.W = c.width; p.H = c.height; p.fx = c.fx; p.fy = c.fy; p.cx = c.cx; p.cy = c.cy;
  p.max_range = h->mot.max_range;
  p.min_z_world = p.tw[2] + h->mot.min_z_coordinate;  // free_space_motion_detector.cpp:80
  p.block_size = h->block_size;
  p.block_size_inv = 1.f / h->block_size;
  p.voxel_size_inv = 1.f / h->map.voxel_size;
  int st;
  if (f->depth_u16) {  // compact depth: expand on the device
    const uint16_t* d16 = nullptr;
    if ((st = stage(h, f->depth_u16, h->mot_depth16, px, f->memory, &d16)) != KB_OK) return st;
    launchExpandDepth(d16, f->depth_u16_scale, h->mot_depth, static_cast<int>(px), h->stream);
    p.depth = h->mot_depth;
  } else if ((st = stage(h, f->depth, h->mot_depth, px, f->memory, &p.depth)) != KB_OK) {
    return st;
  }
  h->motion_vertex = f->vertex_world != nullptr;
  if (f->vertex_world) {  // kept for the cluster lists' boxes: a device map is only borrowed for the call
    KB_CUDA(h, cudaMemcpyAsync(h->mot_vertex, f->vertex_world, sizeof(float) * 3 * px,
                               f->memory == KB_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, h->stream));
    p.vertex = h->mot_vertex;
  }
  p.pixel_gidx = h->d_pixel_gidx;
  p.pixel_seed = h->d_pixel_seed;
  p.pixel_flags = shard_flags;
  KB_CUDA(h, cudaMemsetAsync(h->dm.counters + kCtrSeeds, 0, sizeof(int), h->stream));
  if (shard_flags) launchMotionLookupLocal(h->dm, p, h->stream);  // seeds are counted after the cross-rank reduce
  else launchMotionLookup(h->dm, p, h->stream);
  KB_CUDA(h, cudaGetLastError());
  // keep the depth image on the device for lazily built cluster lists (bounding boxes)
  if (f->memory == KB_MEM_DEVICE && p.depth != h->mot_depth)
    KB_CUDA(h, cudaMemcpyAsync(h->mot_depth, p.depth, sizeof(float) * px, cudaMemcpyDeviceToDevice, h->stream));
  MotionHostParams& mp = h->motion_hp;
  mp.W = c.width; mp.H = c.height; mp.fx = c.fx; mp.fy = c.fy; mp.cx = c.cx; mp.cy = c.cy;
  std::memcpy(mp.Rw, p.Rw, sizeof(mp.Rw));
  std::memcpy(mp.tw, p.tw, sizeof(mp.tw));
  mp.connectivity = h->mot.neighbor_connectivity;
  mp.min_cluster_size = h->mot.min_cluster_size;
  mp.max_cluster_size = h->mot.max_cluster_size;
  mp.min_separation_distance = h->mot.min_separation_distance;
  h->motion.clusters.clear();
  h->motion.n_seeds = 0;
  h->mcl_counts.clear(); h->mcl_pixels.clear(); h->mcl_voxels.clear(); h->mcl_bbox.clear();
  h->motion_stale = false;
  h->motion_have_image = false;
  return KB_OK;
}

// M2-M4 on the device (connected components over the voxels that contain points) for min_separation_distance > 0, with
// or without a caller vertex map; every stage is gated by the device-side seed counter, so this can be enqueued without
// knowing whether M1 found seeds. The cluster lists are built only when asked for (buildMotionListsOnDevice).
static int enqueueDeviceClustering(kb_handle* h) {
  const size_t px = static_cast<size_t>(h->cam.width) * h->cam.height;
  const int D = static_cast<int>(std::ceil(h->mot.min_separation_distance));
  h->trk_have = false;  // the shared table is reused
  if (h->motion_sparse) {
    launchMotionClusteringSparse(h->mt, h->d_pixel_gidx, h->d_pixel_seed, static_cast<int>(px), h->mot.neighbor_connectivity, D,
                                 h->mot.min_cluster_size, h->mot.max_cluster_size, h->d_dynamic, h->mt_dirty, h->stream);
    h->mt_dirty = false;
  } else {
    launchMotionClustering(h->mt, h->d_pixel_gidx, h->d_pixel_seed, static_cast<int>(px), h->mot.neighbor_connectivity, D,
                           h->mot.min_cluster_size, h->mot.max_cluster_size, h->d_dynamic, h->stream);
    h->mt_dirty = true;  // the dense path leaves its entries in the table
  }
  KB_CUDA(h, cudaGetLastError());
  KB_CUDA(h, cudaMemcpyAsync(h->h_mscal, h->mt.scalars, sizeof(int) * kMsCount, cudaMemcpyDeviceToHost, h->stream));
  return KB_OK;
}

int kb_detect_motion(kb_handle* h, const kb_frame* f, int32_t* dynamic_image_out, int32_t* n_seeds, int32_t* n_clusters) {
  if (!h || !f || (!f->depth && !f->depth_u16) || !dynamic_image_out) return fail(h, KB_ERR_INVALID, "null argument");
  if (!h->has_mot || !h->map.with_tracking) return fail(h, KB_ERR_STATE, "motion detector not configured");
  if (!h->has_cam) return fail(h, KB_ERR_STATE, "kb_set_camera must be called first");
  KB_CUDA(h, cudaSetDevice(h->device));
  const size_t px = static_cast<size_t>(h->cam.width) * h->cam.height;
  int st;
  if ((st = enqueueMotionLookup(h, f)) != KB_OK) return st;
  if ((st = readCounters(h)) != KB_OK) return st;  // one 4 B round trip: are there any seeds at all?
  const int seed_pixels = h->h_ctr[kCtrSeeds];
  int n_clusters_out = 0;
  if (seed_pixels == 0) {
    std::memset(dynamic_image_out, 0, sizeof(int32_t) * px);
  } else {
    if (h->mot.min_separation_distance > 0.f) {
      if ((st = enqueueDeviceClustering(h)) != KB_OK) return st;
      KB_CUDA(h, cudaMemcpyAsync(dynamic_image_out, h->d_dynamic, sizeof(int32_t) * px, cudaMemcpyDeviceToHost, h->stream));
      KB_CUDA(h, cudaStreamSynchronize(h->stream));
      h->motion.n_seeds = h->h_mscal[kMsSeeds];
      n_clusters_out = h->h_mscal[kMsClusters];
      h->motion_stale = n_clusters_out > 0;  // cluster lists are built on demand (kb_get_motion_clusters)
      h->motion_have_image = true;
    } else {
      std::memset(dynamic_image_out, 0, sizeof(int32_t) * px);
      const float* host_vertex = f->memory == KB_MEM_DEVICE ? nullptr : f->vertex_world;
      if ((st = buildMotionClustersOnHost(h, host_vertex, dynamic_image_out)) != KB_OK) return st;
      n_clusters_out = static_cast<int>(h->motion.clusters.size());
      KB_CUDA(h, cudaMemcpyAsync(h->d_dynamic, dynamic_image_out, sizeof(int32_t) * px, cudaMemcpyHostToDevice, h->stream));
      h->motion_have_image = true;
    }
  }
  if (n_seeds) *n_seeds = h->motion.n_seeds;
  if (n_clusters) *n_clusters = n_clusters_out;
  return KB_OK;
}

int kb_spin_once(kb_handle* h, const kb_frame* f, int32_t* dynamic_image_out, int32_t* n_seeds, int32_t* n_clusters) {
  if (!h || !f || (!f->depth && !f->depth_u16)) return fail(h, KB_ERR_INVALID, "null argument");
  if (!h->has_mot || !h->has_trk || !h->map.with_tracking) return fail(h, KB_ERR_STATE, "motion detector / tracking not configured");
  if (!h->has_cam) return fail(h, KB_ERR_STATE, "kb_set_camera must be called first");
  KB_CUDA(h, cudaSetDevice(h->device));
  const size_t px = static_cast<size_t>(h->cam.width) * h->cam.height;
  int st;
  if (!(h->mot.min_separation_distance > 0.f)) {
    // the host clustering (one voxel may belong to several clusters): run the three steps one after the other
    std::vector<int32_t> tmp;
    int32_t* img = dynamic_image_out;
    if (!img) { tmp.assign(px, 0); img = tmp.data(); }
    if ((st = kb_detect_motion(h, f, img, n_seeds, n_clusters)) != KB_OK) return st;
    kb_frame g = *f;
    g.mask = KB_MASK_LAST_DETECTION;
    if ((st = kb_integrate_frames(h, &g, 1, 1, nullptr)) != KB_OK) return st;
    return updateTrackingImpl(h, f->stamp_ns);
  }
  // Everything is enqueued back to back; the device decides (seed counter) whether the clustering stages do
  // anything, and the host reads image + counters once at the end.
  if ((st = enqueueMotionLookup(h, f)) != KB_OK) return st;
  if ((st = enqueueDeviceClustering(h)) != KB_OK) return st;
  if (dynamic_image_out)
    KB_CUDA(h, cudaMemcpyAsync(dynamic_image_out, h->d_dynamic, sizeof(int32_t) * px, cudaMemcpyDeviceToHost, h->stream));
  h->motion_have_image = true;
  kb_frame g = *f;
  g.mask = KB_MASK_LAST_DETECTION;
  if ((st = kb_integrate_frames(h, &g, 1, 1, nullptr)) != KB_OK) return st;
  if ((st = updateTrackingImpl(h, f->stamp_ns)) != KB_OK) return st;
  KB_CUDA(h, cudaStreamSynchronize(h->stream));
  h->motion.n_seeds = h->h_mscal[kMsSeeds];
  h->motion_stale = h->h_mscal[kMsClusters] > 0;
  if (n_seeds) *n_seeds = h->h_mscal[kMsSeeds];
  if (n_clusters) *n_clusters = h->h_mscal[kMsClusters];
  return KB_OK;
}

int kb_detect_objects(kb_handle* h, const kb_object_detector_config* cfg, const kb_frame* f, int32_t* object_image_out,
                      int32_t* n_clusters) {
  if (!h || !cfg || !f || !object_image_out || (!f->depth && !f->depth_u16)) return fail(h, KB_ERR_INVALID, "null argument");
  if (!h->has_cam) return fail(h, KB_ERR_STATE, "kb_set_camera must be called first");
  if (cfg->use_3d && !(cfg->grid_size > 0.f)) return fail(h, KB_ERR_INVALID, "grid_size must be positive");
  KB_CUDA(h, cudaSetDevice(h->device));
  const kb_camera& c = h->cam;
  const size_t px = static_cast<size_t>(c.width) * c.height;
  int st;
  if ((st = ensureObjectBuffers(h, px)) != KB_OK) return st;
  // the object ranking stays bounded (single-CTA O(n^2) rank): more semantic clusters than this is a capacity error
  MotionTable ot = h->mt;
  ot.max_roots = std::min(ot.max_roots, 4096);
  if (ot.max_roots * 1024 < static_cast<int>(px)) return fail(h, KB_ERR_CAPACITY, "image too large for the 2D scan");
  h->obj_have = false;
  if (!f->label && !f->label_u8) {  // no semantic image: no objects (connected_semantics.cpp reads label_image only)
    std::memset(object_image_out, 0, sizeof(int32_t) * px);
    KB_CUDA(h, cudaMemsetAsync(h->d_object, 0, sizeof(int32_t) * px, h->stream));
    h->obj_image_host.assign(px, 0);
    h->obj_label_host.assign(px, 0);
    h->obj_have = true;
    if (n_clusters) *n_clusters = 0;
    return KB_OK;
  }
  ObjectParams p{};
  float R[9], t[3];
  poseToFloat(f->world_T_sensor, R, t, p.Rw, p.tw);
  p.W = c.width; p.H = c.height; p.fx = c.fx; p.fy = c.fy; p.cx = c.cx; p.cy = c.cy;
  p.inv_grid = cfg->use_3d ? 1.f / cfg->grid_size : 0.f;
  p.max_range = cfg->max_range;
  for (int i = 0; i < KB_MAX_LABELS; ++i)
    if (cfg->is_object[i]) p.object_mask |= 1ull << i;
  p.full = cfg->use_full_connectivity;
  p.min_size = cfg->min_cluster_size;
  p.max_size = cfg->max_cluster_size;
  p.image = h->d_object;
  // inputs: compact formats are expanded like everywhere else (float(u16) * scale, int32(u8))
  if (f->depth_u16) {
    const uint16_t* d16 = nullptr;
    if ((st = stage(h, f->depth_u16, h->mot_depth16, px, f->memory, &d16)) != KB_OK) return st;
    launchExpandDepth(d16, f->depth_u16_scale, h->obj_depth, static_cast<int>(px), h->stream);
    p.depth = h->obj_depth;
  } else if ((st = stage(h, f->depth, h->obj_depth, px, f->memory, &p.depth)) != KB_OK) {
    return st;
  }
  h->obj_label_host.resize(px);
  if (f->label_u8) {
    std::vector<uint8_t> tmp(px);  // rare path: expand the 8-bit ids on the host side of the staging copy
    if (f->memory == KB_MEM_DEVICE) KB_CUDA(h, cudaMemcpy(tmp.data(), f->label_u8, px, cudaMemcpyDeviceToHost));
    else std::memcpy(tmp.data(), f->label_u8, px);
    for (size_t i = 0; i < px; ++i) h->obj_label_host[i] = tmp[i];
    KB_CUDA(h, cudaMemcpyAsync(h->obj_label, h->obj_label_host.data(), sizeof(int) * px, cudaMemcpyHostToDevice, h->stream));
    p.label = h->obj_label;
  } else {
    if ((st = stage(h, f->label, h->obj_label, px, f->memory, &p.label)) != KB_OK) return st;
    if (f->memory == KB_MEM_DEVICE) KB_CUDA(h, cudaMemcpyAsync(h->obj_label_host.data(), f->label, sizeof(int) * px, cudaMemcpyDeviceToHost, h->stream));
    else std::memcpy(h->obj_label_host.data(), f->label, sizeof(int) * px);
  }
  if (cfg->use_3d && (st = stage(h, f->vertex_world, h->stg_vertex, px * 3, f->memory, &p.vertex)) != KB_OK) return st;
  if (cfg->use_3d) launchObjectClustering3D(ot, p, h->stream);
  else launchObjectClustering2D(ot, p, h->stream);
  h->mt_dirty = true;  // shared table memory
  h->trk_have = false;
  KB_CUDA(h, cudaGetLastError());
  KB_CUDA(h, cudaMemcpyAsync(h->h_oscal, h->mt.scalars, sizeof(int) * kMsCount, cudaMemcpyDeviceToHost, h->stream));
  KB_CUDA(h, cudaMemcpyAsync(object_image_out, h->d_object, sizeof(int32_t) * px, cudaMemcpyDeviceToHost, h->stream));
  KB_CUDA(h, cudaStreamSynchronize(h->stream));
  if (cfg->use_3d && h->h_oscal[kMsRoots] > ot.max_roots)
    return fail(h, KB_ERR_CAPACITY, "too many semantic clusters for the device ranking");
  h->obj_image_host.assign(object_image_out, object_image_out + px);
  h->obj_have = true;
  if (n_clusters) *n_clusters = h->h_oscal[kMsClusters];
  return KB_OK;
}

int kb_forward_instances(kb_handle* h, const kb_instance_forwarding_config* cfg, const kb_frame* f, const uint8_t* id_is_background,
                         int32_t n_background, int32_t* object_image_out, int32_t* n_clusters) {
  if (!h || !cfg || !f || !object_image_out || (!f->depth && !f->depth_u16)) return fail(h, KB_ERR_INVALID, "null argument");
  if (!h->has_cam) return fail(h, KB_ERR_STATE, "kb_set_camera must be called first");
  KB_CUDA(h, cudaSetDevice(h->device));
  h->main_dirty = true;
  const kb_camera& c = h->cam;
  const size_t px = static_cast<size_t>(c.width) * c.height;
  int st;
  if ((st = ensureObjectBuffers(h, px)) != KB_OK) return st;
  h->inst_have = false;
  h->inst_clusters.clear();
  h->obj_label_host.assign(px, 0);
  h->inst_keep_host.assign(px, 0);
  if (!f->label && !f->label_u8) {
    std::memset(object_image_out, 0, sizeof(int32_t) * px);
    h->inst_have = true;
    if (n_clusters) *n_clusters = 0;
    return KB_OK;
  }
  if (!h->inst_counts) {
    KB_CUDA(h, devAlloc(&h->inst_counts, KB_MAX_INSTANCE_IDS, 0));
    KB_CUDA(h, devAlloc(&h->inst_bbox, static_cast<size_t>(KB_MAX_INSTANCE_IDS) * 6, 0));
    KB_CUDA(h, devAlloc(&h->inst_background, KB_MAX_INSTANCE_IDS, 0));
    KB_CUDA(h, devAlloc(&h->inst_bad, 1, 0));
  }
  if (h->inst_pixels < px) {
    KB_CUDA(h, cudaStreamSynchronize(h->stream));
    cudaFree(h->inst_keep);
    h->inst_keep = nullptr;
    KB_CUDA(h, devAlloc(&h->inst_keep, px, 0));
    h->inst_pixels = px;
  }
  ObjectParams p{};
  float R[9], t[3];
  poseToFloat(f->world_T_sensor, R, t, p.Rw, p.tw);
  p.W = c.width; p.H = c.height; p.fx = c.fx; p.fy = c.fy; p.cx = c.cx; p.cy = c.cy;
  p.max_range = cfg->max_range;
  if (f->depth_u16) {
    const uint16_t* d16 = nullptr;
    if ((st = stage(h, f->depth_u16, h->mot_depth16, px, f->memory, &d16)) != KB_OK) return st;
    launchExpandDepth(d16, f->depth_u16_scale, h->obj_depth, static_cast<int>(px), h->stream);
    p.depth = h->obj_depth;
  } else if ((st = stage(h, f->depth, h->obj_depth, px, f->memory, &p.depth)) != KB_OK) {
    return st;
  }
  if (f->label_u8) {
    std::vector<uint8_t> tmp(px);
    if (f->memory == KB_MEM_DEVICE) KB_CUDA(h, cudaMemcpy(tmp.data(), f->label_u8, px, cudaMemcpyDeviceToHost));
    else std::memcpy(tmp.data(), f->label_u8, px);
    for (size_t i = 0; i < px; ++i) h->obj_label_host[i] = tmp[i];
    KB_CUDA(h, cudaMemcpyAsync(h->obj_label, h->obj_label_host.data(), sizeof(int) * px, cudaMemcpyHostToDevice, h->stream));
    p.label = h->obj_label;
  } else {
    if ((st = stage(h, f->label, h->obj_label, px, f->memory, &p.label)) != KB_OK) return st;
    if (f->memory == KB_MEM_DEVICE) KB_CUDA(h, cudaMemcpyAsync(h->obj_label_host.data(), f->label, sizeof(int) * px, cudaMemcpyDeviceToHost, h->stream));
    else std::memcpy(h->obj_label_host.data(), f->label, sizeof(int) * px);
  }
  if ((st = stage(h, f->vertex_world, h->stg_vertex, px * 3, f->memory, &p.vertex)) != KB_OK) return st;
  const uint8_t* bg = nullptr;
  if (id_is_background && n_background > 0) {
    std::vector<uint8_t> table(KB_MAX_INSTANCE_IDS, 0);
    std::memcpy(table.data(), id_is_background, static_cast<size_t>(std::min<int32_t>(n_background, KB_MAX_INSTANCE_IDS)));
    KB_CUDA(h, cudaMemcpyAsync(h->inst_background, table.data(), KB_MAX_INSTANCE_IDS, cudaMemcpyHostToDevice, h->stream));
    KB_CUDA(h, cudaStreamSynchronize(h->stream));  // `table` is a local
    bg = h->inst_background;
  }
  launchInstanceForward(p, bg, KB_MAX_INSTANCE_IDS, h->inst_counts, h->inst_bbox, h->inst_keep, h->inst_bad, h->stream);
  KB_CUDA(h, cudaGetLastError());
  std::vector<int> counts(KB_MAX_INSTANCE_IDS);
  std::vector<unsigned int> bbox(static_cast<size_t>(KB_MAX_INSTANCE_IDS) * 6);
  int bad = 0;
  KB_CUDA(h, cudaMemcpyAsync(counts.data(), h->inst_counts, sizeof(int) * counts.size(), cudaMemcpyDeviceToHost, h->stream));
  KB_CUDA(h, cudaMemcpyAsync(bbox.data(), h->inst_bbox, sizeof(unsigned int) * bbox.size(), cudaMemcpyDeviceToHost, h->stream));
  KB_CUDA(h, cudaMemcpyAsync(h->inst_keep_host.data(), h->inst_keep, px, cudaMemcpyDeviceToHost, h->stream));
  KB_CUDA(h, cudaMemcpyAsync(&bad, h->inst_bad, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  KB_CUDA(h, cudaStreamSynchronize(h->stream));
  if (bad) return fail(h, KB_ERR_INVALID, "instance id outside 0 .. KB_MAX_INSTANCE_IDS - 1");
  std::memcpy(object_image_out, h->obj_label_host.data(), sizeof(int32_t) * px);  // object_image = label image (:83)
  const bool filter_by_volume = cfg->min_object_volume > 0.0 || cfg->max_object_volume > 0.0;  // :68
  auto decode = [](unsigned int o) {
    const unsigned int b = (o & 0x80000000u) ? (o & 0x7FFFFFFFu) : ~o;
    float v;
    std::memcpy(&v, &b, 4);
    return v;
  };
  for (int id = 1; id < KB_MAX_INSTANCE_IDS; ++id) {
    const int n = counts[id];
    if (n == 0) continue;
    if (n < cfg->min_cluster_size || (cfg->max_cluster_size > 0 && n > cfg->max_cluster_size)) continue;  // :119-122
    kb_handle::InstCluster cl{};
    cl.id = id;
    cl.count = n;
    for (int k = 0; k < 6; ++k) cl.bbox[k] = decode(bbox[static_cast<size_t>(id) * 6 + k]);
    if (filter_by_volume) {  // :128-135, BoundingBox::volume() = product of the float dimensions
      const float volume = (cl.bbox[3] - cl.bbox[0]) * (cl.bbox[4] - cl.bbox[1]) * (cl.bbox[5] - cl.bbox[2]);
      if (volume < cfg->min_object_volume || (cfg->max_object_volume > 0.0 && volume > cfg->max_object_volume)) continue;
    }
    h->inst_clusters.push_back(cl);
  }
  h->inst_have = true;
  if (n_clusters) *n_clusters = static_cast<int32_t>(h->inst_clusters.size());
  return KB_OK;
}

int kb_get_instance_clusters(kb_handle* h, int32_t* id_count, float* bbox_min_max, int32_t* pixels_uv, int32_t* n_clusters,
                             int32_t* total_pixels) {
  if (!h) return KB_ERR_INVALID;
  if (!h->inst_have) return fail(h, KB_ERR_STATE, "kb_forward_instances has not been called");
  const int W = h->cam.width, H = h->cam.height;
  int32_t total = 0;
  std::vector<int> base(KB_MAX_INSTANCE_IDS, -1);
  for (size_t c = 0; c < h->inst_clusters.size(); ++c) {
    const auto& cl = h->inst_clusters[c];
    if (id_count) { id_count[2 * c] = cl.id; id_count[2 * c + 1] = cl.count; }
    if (bbox_min_max) std::memcpy(bbox_min_max + 6 * c, cl.bbox, sizeof(cl.bbox));
    base[cl.id] = total;
    total += cl.count;
  }
  if (pixels_uv && total > 0) {
    std::vector<int> fill(KB_MAX_INSTANCE_IDS, 0);
    for (int u = 0; u < W; ++u)      // the reference's scan order (:87-88)
      for (int v = 0; v < H; ++v) {
        const size_t px = static_cast<size_t>(v) * W + u;
        if (!h->inst_keep_host[px]) continue;
        const int id = h->obj_label_host[px];
        if (id <= 0 || id >= KB_MAX_INSTANCE_IDS || base[id] < 0) continue;
        const int k = base[id] + fill[id]++;
        pixels_uv[2 * k] = u;
        pixels_uv[2 * k + 1] = v;
      }
  }
  if (n_clusters) *n_clusters = static_cast<int32_t>(h->inst_clusters.size());
  if (total_pixels) *total_pixels = total;
  return KB_OK;
}

int kb_get_object_clusters(kb_handle* h, int32_t* id_semantic_count, int32_t* pixels_uv, int32_t* n_clusters,
                           int32_t* total_pixels) {
  if (!h) return KB_ERR_INVALID;
  if (!h->obj_have) return fail(h, KB_ERR_STATE, "no object detection result");
  // Cluster lists are derived on demand from the object image: ascending id, semantic id = the label under any of
  // the cluster's pixels (all agree), pixels in row-major order.
  const int W = h->cam.width;
  const size_t px = h->obj_image_host.size();
  std::vector<std::pair<int32_t, int32_t>> by_id;  // (id, pixel)
  by_id.reserve(px / 8);
  for (size_t i = 0; i < px; ++i)
    if (h->obj_image_host[i] != 0) by_id.emplace_back(h->obj_image_host[i], static_cast<int32_t>(i));
  std::stable_sort(by_id.begin(), by_id.end(), [](const auto& a, const auto& b) { return a.first < b.first; });
  int32_t nc = 0;
  size_t i = 0;
  while (i < by_id.size()) {
    size_t e = i;
    while (e < by_id.size() && by_id[e].first == by_id[i].first) ++e;
    if (id_semantic_count) {
      id_semantic_count[nc * 3] = by_id[i].first;
      id_semantic_count[nc * 3 + 1] = h->obj_label_host[by_id[i].second];
      id_semantic_count[nc * 3 + 2] = static_cast<int32_t>(e - i);
    }
    if (pixels_uv)
      for (size_t k = i; k < e; ++k) { pixels_uv[k * 2] = by_id[k].second % W; pixels_uv[k * 2 + 1] = by_id[k].second / W; }
    ++nc;
    i = e;
  }
  if (n_clusters) *n_clusters = nc;
  if (total_pixels) *total_pixels = static_cast<int32_t>(by_id.size());
  return KB_OK;
}

int kb_track_measurements(kb_handle* h, const kb_frame* f, const int32_t* id_image, int32_t n_clusters,
                          const int32_t* cluster_ids, float voxel_size, int32_t n_tracks, const int32_t* track_offsets, const int64_t* track_voxels_xyz,
                          int32_t* voxel_counts, int64_t* voxel_sums, int32_t* intersections, float* iou) {
  if (!h || !f || !id_image || (!f->depth && !f->depth_u16 && !f->vertex_world)) return fail(h, KB_ERR_INVALID, "null argument");
  if (!h->has_cam) return fail(h, KB_ERR_STATE, "kb_set_camera must be called first");
  if (n_clusters < 1 || n_clusters > kTrackMaxIds) return fail(h, KB_ERR_INVALID, "n_clusters must be in 1..1022");
  for (int i = 1; cluster_ids && i < n_clusters; ++i)
    if (cluster_ids[i] <= cluster_ids[i - 1]) return fail(h, KB_ERR_INVALID, "cluster_ids must be strictly ascending");
  const int max_id = n_clusters;  // rows
  if (!(voxel_size > 0.f)) return fail(h, KB_ERR_INVALID, "voxel_size must be positive");
  if (n_tracks < 0 || (n_tracks > 0 && (!track_offsets || !track_voxels_xyz))) return fail(h, KB_ERR_INVALID, "track lists missing");
  if (n_tracks > 0 && (track_offsets[0] != 0)) return fail(h, KB_ERR_INVALID, "track_offsets[0] must be 0");
  for (int t = 0; t < n_tracks; ++t)
    if (track_offsets[t + 1] < track_offsets[t]) return fail(h, KB_ERR_INVALID, "track_offsets must be non-decreasing");
  KB_CUDA(h, cudaSetDevice(h->device));
  const kb_camera& c = h->cam;
  const size_t px = static_cast<size_t>(c.width) * c.height;
  const size_t ntv = n_tracks > 0 ? static_cast<size_t>(track_offsets[n_tracks]) : 0;
  const size_t ninter = static_cast<size_t>(max_id) * static_cast<size_t>(std::max(n_tracks, 1));
  int st;
  if ((st = ensureObjectBuffers(h, px)) != KB_OK) return st;
  if ((st = ensureTrackBuffers(h, px, std::max<size_t>(ntv, 1), ninter)) != KB_OK) return st;
  h->trk_have = false;
  TrackParams p{};
  float R[9], t[3];
  poseToFloat(f->world_T_sensor, R, t, p.Rw, p.tw);
  p.W = c.width; p.H = c.height; p.fx = c.fx; p.fy = c.fy; p.cx = c.cx; p.cy = c.cy;
  p.n_ids = n_clusters;
  if (cluster_ids) {
    KB_CUDA(h, cudaMemcpyAsync(h->trk_idlist, cluster_ids, sizeof(int) * n_clusters, cudaMemcpyHostToDevice, h->stream));
    p.id_list = h->trk_idlist;
  }
  p.inv_voxel = 1.f / voxel_size;
  p.voxel_counts = h->trk_counts;
  p.sums = h->trk_sums;
  if ((st = stage(h, f->vertex_world, h->stg_vertex, px * 3, f->memory, &p.vertex)) != KB_OK) return st;
  if (!p.vertex) {
    if (f->depth_u16) {
      const uint16_t* d16 = nullptr;
      if ((st = stage(h, f->depth_u16, h->mot_depth16, px, f->memory, &d16)) != KB_OK) return st;
      launchExpandDepth(d16, f->depth_u16_scale, h->obj_depth, static_cast<int>(px), h->stream);
      p.depth = h->obj_depth;
    } else if ((st = stage(h, f->depth, h->obj_depth, px, f->memory, &p.depth)) != KB_OK) {
      return st;
    }
  }
  if ((st = stage(h, id_image, h->trk_ids, px, f->memory, &p.ids)) != KB_OK) return st;
  // The table needs 2 slots per cluster pixel at most. A host id image is counted on the way (a pass over 1.2 MB), so
  // that only that part of the shared 2^20-slot table is reset and probed; device images use all of it.
  MotionTable table = h->mt;
  if (f->memory != KB_MEM_DEVICE) {
    size_t cluster_pixels = 0;
    for (size_t i = 0; i < px; ++i) cluster_pixels += id_image[i] != 0;
    uint32_t cap = 1024;
    while (cap < 2 * cluster_pixels) cap <<= 1;
    if (cap - 1 < table.mask) table.mask = cap - 1;
  }
  launchTrackVoxelize(table, p, h->stream);
  h->mt_dirty = true;  // shared table memory
  KB_CUDA(h, cudaGetLastError());
  h->trk_counts_host.assign(static_cast<size_t>(max_id), 0);
  std::vector<unsigned long long> sums(static_cast<size_t>(max_id) * 3);
  KB_CUDA(h, cudaMemcpyAsync(h->trk_counts_host.data(), h->trk_counts, sizeof(int) * max_id, cudaMemcpyDeviceToHost, h->stream));
  KB_CUDA(h, cudaMemcpyAsync(sums.data(), h->trk_sums, sizeof(unsigned long long) * 3 * max_id, cudaMemcpyDeviceToHost, h->stream));
  KB_CUDA(h, cudaStreamSynchronize(h->stream));
  if (voxel_counts) std::memcpy(voxel_counts, h->trk_counts_host.data(), sizeof(int32_t) * max_id);
  if (voxel_sums)
    for (size_t i = 0; i < sums.size(); ++i) voxel_sums[i] = static_cast<int64_t>(sums[i]);
  h->trk_have = true;
  if (n_tracks == 0 || (!intersections && !iou)) return KB_OK;
  // computeIoUVoxels: probe every track voxel against the clusters that have voxels
  std::vector<int> present;
  for (int id = 1; id <= max_id; ++id)
    if (h->trk_counts_host[id - 1] > 0) present.push_back(id);
  std::vector<unsigned long long> keys;
  std::vector<int> track_of;
  keys.reserve(ntv); track_of.reserve(ntv);
  for (int tr = 0; tr < n_tracks; ++tr)
    for (int k = track_offsets[tr]; k < track_offsets[tr + 1]; ++k) {
      unsigned long long key;  // a voxel outside the key range cannot be in any cluster of this frame
      if (trackVoxelKey(track_voxels_xyz[3 * k], track_voxels_xyz[3 * k + 1], track_voxels_xyz[3 * k + 2], &key)) {
        keys.push_back(key);
        track_of.push_back(tr);
      }
    }
  std::vector<int32_t> inter(static_cast<size_t>(max_id) * n_tracks, 0);
  if (!present.empty() && !keys.empty()) {
    KB_CUDA(h, cudaMemsetAsync(h->trk_inter, 0, sizeof(int) * inter.size(), h->stream));
    KB_CUDA(h, cudaMemcpyAsync(h->trk_keys, keys.data(), sizeof(unsigned long long) * keys.size(), cudaMemcpyHostToDevice, h->stream));
    KB_CUDA(h, cudaMemcpyAsync(h->trk_of, track_of.data(), sizeof(int) * keys.size(), cudaMemcpyHostToDevice, h->stream));
    KB_CUDA(h, cudaMemcpyAsync(h->trk_present, present.data(), sizeof(int) * present.size(), cudaMemcpyHostToDevice, h->stream));
    launchTrackIntersect(table, h->trk_keys, h->trk_of, static_cast<int>(keys.size()), h->trk_present,
                         static_cast<int>(present.size()), n_tracks, h->trk_inter, h->stream);
    KB_CUDA(h, cudaGetLastError());
    KB_CUDA(h, cudaMemcpyAsync(inter.data(), h->trk_inter, sizeof(int) * inter.size(), cudaMemcpyDeviceToHost, h->stream));
    KB_CUDA(h, cudaStreamSynchronize(h->stream));
  }
  for (int id = 1; id <= max_id; ++id)
    for (int tr = 0; tr < n_tracks; ++tr) {
      const size_t o = static_cast<size_t>(id - 1) * n_tracks + tr;
      if (intersections) intersections[o] = inter[o];
      if (iou) {
        // max_iou_tracker.cpp:562: float intersection / (size_t + size_t - float intersection)
        const float in = static_cast<float>(inter[o]);
        const size_t sizes = static_cast<size_t>(h->trk_counts_host[id - 1]) +
                             static_cast<size_t>(track_offsets[tr + 1] - track_offsets[tr]);
        iou[o] = in / (static_cast<float>(sizes) - in);
      }
    }
  return KB_OK;
}

int kb_compute_vertex_map(kb_handle* h, const kb_frame* f, float* vertex_world_out) {
  if (!h || !f || !vertex_world_out || (!f->depth && !f->depth_u16)) return fail(h, KB_ERR_INVALID, "null argument");
  if (!h->has_cam) return fail(h, KB_ERR_STATE, "kb_set_camera must be called first");
  KB_CUDA(h, cudaSetDevice(h->device));
  const kb_camera& c = h->cam;
  const size_t px = static_cast<size_t>(c.width) * c.height;
  int st;
  if ((st = ensureObjectBuffers(h, px)) != KB_OK) return st;
  TrackParams p{};
  float R[9], t[3];
  poseToFloat(f->world_T_sensor, R, t, p.Rw, p.tw);
  p.W = c.width; p.H = c.height; p.fx = c.fx; p.fy = c.fy; p.cx = c.cx; p.cy = c.cy;
  if (f->depth_u16) {
    const uint16_t* d16 = nullptr;
    if ((st = stage(h, f->depth_u16, h->mot_depth16, px, f->memory, &d16)) != KB_OK) return st;
    launchExpandDepth(d16, f->depth_u16_scale, h->obj_depth, static_cast<int>(px), h->stream);
    p.depth = h->obj_depth;
  } else if ((st = stage(h, f->depth, h->obj_depth, px, f->memory, &p.depth)) != KB_OK) {
    return st;
  }
  const bool device_out = f->memory == KB_MEM_DEVICE;
  float* out = device_out ? vertex_world_out : h->stg_vertex;
  launchVertexMap(p, out, h->stream);
  KB_CUDA(h, cudaGetLastError());
  if (!device_out) KB_CUDA(h, cudaMemcpyAsync(vertex_world_out, out, sizeof(float) * 3 * px, cudaMemcpyDeviceToHost, h->stream));
  KB_CUDA(h, cudaStreamSynchronize(h->stream));
  return KB_OK;
}

int kb_get_cluster_voxels(kb_handle* h, int32_t* offsets, int64_t* voxels_xyz, int32_t capacity, int32_t* total) {
  if (!h) return KB_ERR_INVALID;
  if (!h->trk_have) return fail(h, KB_ERR_STATE, "no track measurement result");
  KB_CUDA(h, cudaSetDevice(h->device));
  const int max_id = static_cast<int>(h->trk_counts_host.size());
  size_t n = 0;
  for (int c : h->trk_counts_host) n += static_cast<size_t>(c);
  if (total) *total = static_cast<int32_t>(n);
  if (offsets) {
    offsets[0] = 0;
    for (int i = 0; i < max_id; ++i) offsets[i + 1] = offsets[i] + h->trk_counts_host[i];
  }
  if (!voxels_xyz) return KB_OK;
  if (static_cast<size_t>(std::max(capacity, 0)) < n) return fail(h, KB_ERR_CAPACITY, "voxel buffer too small");
  if (n == 0) return KB_OK;
  std::vector<unsigned long long> keys(n);
  launchTrackExportKeys(h->mt, h->trk_export, h->stream);
  KB_CUDA(h, cudaGetLastError());
  KB_CUDA(h, cudaMemcpyAsync(keys.data(), h->trk_export, sizeof(unsigned long long) * n, cudaMemcpyDeviceToHost, h->stream));
  KB_CUDA(h, cudaStreamSynchronize(h->stream));
  std::sort(keys.begin(), keys.end());  // order preserving keys: cluster id, then (z, y, x)
  for (size_t i = 0; i < n; ++i) {
    int id, x, y, z;
    trackKeyDecode(keys[i], &id, &x, &y, &z);
    voxels_xyz[3 * i] = x; voxels_xyz[3 * i + 1] = y; voxels_xyz[3 * i + 2] = z;
  }
  return KB_OK;
}

int kb_motion_lookup_local(kb_handle* h, const kb_frame* f, uint8_t* pixel_flags) {
  if (!h || !f || (!f->depth && !f->depth_u16) || !pixel_flags) return fail(h, KB_ERR_INVALID, "null argument");
  if (!h->has_mot || !h->map.with_tracking) return fail(h, KB_ERR_STATE, "motion detector not configured");
  if (!h->has_cam) return fail(h, KB_ERR_STATE, "kb_set_camera must be called first");
  if (!(h->mot.min_separation_distance > 0.f) || f->vertex_world != nullptr)
    return fail(h, KB_ERR_STATE, "the sharded motion path needs min_separation_distance > 0 and no caller-supplied vertex map");
  KB_CUDA(h, cudaSetDevice(h->device));
  return enqueueMotionLookup(h, f, pixel_flags);
}

int kb_motion_lookup_peers(kb_handle* h, const kb_frame* f, uint8_t* const* peer_flags, int32_t n_peers) {
  if (!h || !f || (!f->depth && !f->depth_u16)) return fail(h, KB_ERR_INVALID, "null argument");
  if (!h->has_mot || !h->map.with_tracking) return fail(h, KB_ERR_STATE, "motion detector not configured");
  if (!h->has_cam) return fail(h, KB_ERR_STATE, "kb_set_camera must be called first");
  if (!(h->mot.min_separation_distance > 0.f) || f->vertex_world != nullptr)
    return fail(h, KB_ERR_STATE, "the sharded motion path needs min_separation_distance > 0 and no caller-supplied vertex map");
  KB_CUDA(h, cudaSetDevice(h->device));
  PeerBuffers peers{};
  int st = makePeers(h, reinterpret_cast<void* const*>(peer_flags), n_peers, &peers);
  if (st != KB_OK) return st;
  const size_t px = static_cast<size_t>(h->cam.width) * h->cam.height;
  if (h->flags_local_pixels < px) {
    cudaFree(h->d_flags_local);
    h->d_flags_local = nullptr;
    KB_CUDA(h, devAlloc(&h->d_flags_local, px, 0));
    h->flags_local_pixels = px;
  }
  if ((st = enqueueMotionLookup(h, f, h->d_flags_local)) != KB_OK) return st;
  launchFlagScatter(h->d_flags_local, peers, static_cast<int>(px), h->stream);
  KB_CUDA(h, cudaGetLastError());
  return KB_OK;
}

int kb_motion_cluster_global(kb_handle* h, const uint8_t* pixel_flags) {
  if (h) h->main_dirty = true;  // KB_PIPELINE: the next prologue must wait for this main-stream work
  if (!h || !pixel_flags) return fail(h, KB_ERR_INVALID, "null argument");
  if (!h->has_mot || !h->has_cam) return fail(h, KB_ERR_STATE, "motion detector not configured");
  KB_CUDA(h, cudaSetDevice(h->device));
  const size_t px = static_cast<size_t>(h->cam.width) * h->cam.height;
  launchMotionFinalize(h->dm, pixel_flags, h->d_pixel_gidx, h->d_pixel_seed, static_cast<int>(px), h->stream);
  KB_CUDA(h, cudaGetLastError());
  int st = enqueueDeviceClustering(h);
  if (st != KB_OK) return st;
  h->motion_have_image = true;
  return KB_OK;
}

int kb_motion_result(kb_handle* h, int32_t* dynamic_image_out, int32_t* n_seeds, int32_t* n_clusters) {
  if (!h) return KB_ERR_INVALID;
  if (!h->motion_have_image) return fail(h, KB_ERR_STATE, "no motion detection result");
  KB_CUDA(h, cudaSetDevice(h->device));
  const size_t px = static_cast<size_t>(h->cam.width) * h->cam.height;
  if (dynamic_image_out)
    KB_CUDA(h, cudaMemcpyAsync(dynamic_image_out, h->d_dynamic, sizeof(int32_t) * px, cudaMemcpyDeviceToHost, h->stream));
  KB_CUDA(h, cudaStreamSynchronize(h->stream));
  h->motion.n_seeds = h->h_mscal[kMsSeeds];
  h->motion_stale = h->h_mscal[kMsClusters] > 0;
  if (n_seeds) *n_seeds = h->h_mscal[kMsSeeds];
  if (n_clusters) *n_clusters = h->h_mscal[kMsClusters];
  return KB_OK;
}

int kb_multicast_copy(void* multicast_dst, const void* src, size_t bytes, void* cuda_stream) {
  if (!multicast_dst || !src || (bytes % 16) != 0 || (reinterpret_cast<uintptr_t>(multicast_dst) % 16) != 0 ||
      (reinterpret_cast<uintptr_t>(src) % 16) != 0)
    return KB_ERR_INVALID;
  launchMulticastCopy(multicast_dst, src, bytes, static_cast<cudaStream_t>(cuda_stream));
  return cudaGetLastError() == cudaSuccess ? KB_OK : KB_ERR_CUDA;
}

int kb_host_cluster_motion(const kb_camera* camera, const kb_motion_config* motion, const double world_T_sensor[16],
                           const int32_t* pixel_voxel_xyz, const uint8_t* pixel_seed, const float* depth,
                           int32_t* dynamic_image_out, int32_t* n_seeds, int32_t* n_clusters) {
  if (!camera || !motion || !world_T_sensor || !pixel_voxel_xyz || !pixel_seed || !depth || !dynamic_image_out) return KB_ERR_INVALID;
  MotionHostParams mp{};
  float R[9], t[3];
  poseToFloat(world_T_sensor, R, t, mp.Rw, mp.tw);
  mp.W = camera->width; mp.H = camera->height; mp.fx = camera->fx; mp.fy = camera->fy; mp.cx = camera->cx; mp.cy = camera->cy;
  mp.connectivity = motion->neighbor_connectivity;
  mp.min_cluster_size = motion->min_cluster_size;
  mp.max_cluster_size = motion->max_cluster_size;
  mp.min_separation_distance = motion->min_separation_distance;
  std::memset(dynamic_image_out, 0, sizeof(int32_t) * static_cast<size_t>(mp.W) * mp.H);
  MotionResult res;
  clusterMotion(mp, pixel_voxel_xyz, pixel_seed, depth, nullptr, dynamic_image_out, &res);
  if (n_seeds) *n_seeds = res.n_seeds;
  if (n_clusters) *n_clusters = static_cast<int32_t>(res.clusters.size());
  return KB_OK;
}

int kb_get_motion_clusters(kb_handle* h, int32_t* counts, int32_t* pixels_uv, int64_t* voxels_xyz,
                           float* bbox_min_max, int32_t* total_pixels, int32_t* total_voxels) {
  if (!h) return KB_ERR_INVALID;
  if (h->motion_stale) {
    KB_CUDA(h, cudaSetDevice(h->device));
    const int st = buildMotionListsOnDevice(h);
    if (st != KB_OK) return st;
  }
  if (counts) std::memcpy(counts, h->mcl_counts.data(), sizeof(int32_t) * h->mcl_counts.size());
  if (pixels_uv) std::memcpy(pixels_uv, h->mcl_pixels.data(), sizeof(int32_t) * h->mcl_pixels.size());
  if (voxels_xyz) std::memcpy(voxels_xyz, h->mcl_voxels.data(), sizeof(int64_t) * h->mcl_voxels.size());
  if (bbox_min_max) std::memcpy(bbox_min_max, h->mcl_bbox.data(), sizeof(float) * h->mcl_bbox.size());
  if (total_pixels) *total_pixels = static_cast<int32_t>(h->mcl_pixels.size() / 2);
  if (total_voxels) *total_voxels = static_cast<int32_t>(h->mcl_voxels.size() / 3);
  return KB_OK;
}

// ---- export -------------------------------------------------------------------------------------------

static int collectSlots(kb_handle* h, int which, std::vector<int>* slots, std::vector<int3>* index,
                        std::vector<uint32_t>* flags, uint32_t need_flag = 0) {
  int st, n = 0;
  if ((st = slotHwm(h, &n)) != KB_OK) return st;
  std::vector<int3> bi(static_cast<size_t>(n));
  std::vector<uint32_t> bf(static_cast<size_t>(n));
  if (n > 0) {
    KB_CUDA(h, cudaMemcpy(bi.data(), h->dm.block_index, sizeof(int3) * n, cudaMemcpyDeviceToHost));
    KB_CUDA(h, cudaMemcpy(bf.data(), h->dm.block_flags, sizeof(uint32_t) * n, cudaMemcpyDeviceToHost));
  }
  std::vector<int> order;
  for (int s = 0; s < n; ++s) {
    if (!(bf[s] & kFlagAllocated)) continue;
    if (which == KB_EXPORT_UPDATED && !(bf[s] & KB_FLAG_UPDATED)) continue;
    if (need_flag && !(bf[s] & need_flag)) continue;
    order.push_back(s);
  }
  std::sort(order.begin(), order.end(), [&](int a, int b) {
    const int3 &p = bi[a], &q = bi[b];
    return p.x != q.x ? p.x < q.x : (p.y != q.y ? p.y < q.y : p.z < q.z);
  });
  slots->clear(); index->clear(); flags->clear();
  for (int s : order) { slots->push_back(s); index->push_back(bi[s]); flags->push_back(bf[s]); }
  return KB_OK;
}

int kb_generate_mesh(kb_handle* h, int only_mesh_updated, int clear_updated_flag, float min_weight, int32_t* n_blocks,
                     int64_t* n_vertices) {
  if (!h) return KB_ERR_INVALID;
  h->main_dirty = true;
  KB_CUDA(h, cudaSetDevice(h->device));
  std::vector<int> slots; std::vector<uint32_t> flags;
  int st = collectSlots(h, KB_EXPORT_ALL, &slots, &h->mesh_index, &flags, only_mesh_updated ? KB_FLAG_MESH_UPDATED : 0u);
  if (st != KB_OK) return st;
  const int n = static_cast<int>(slots.size());
  h->mesh_base.assign(static_cast<size_t>(n) + 1, 0);
  h->mesh_have = true;
  if (n_blocks) *n_blocks = n;
  if (n_vertices) *n_vertices = 0;
  if (n == 0) return KB_OK;
  const size_t V = h->dm.V;
  if (h->mesh_block_cap < static_cast<size_t>(n)) {
    KB_CUDA(h, cudaStreamSynchronize(h->stream));
    cudaFree(h->mesh_slots); cudaFree(h->mesh_cases); cudaFree(h->mesh_tri_count); cudaFree(h->mesh_tri_base);
    h->mesh_slots = nullptr; h->mesh_cases = nullptr; h->mesh_tri_count = nullptr; h->mesh_tri_base = nullptr;
    h->mesh_block_cap = 0;
    const size_t cap = static_cast<size_t>(n) + static_cast<size_t>(n) / 4 + 64;
    KB_CUDA(h, cudaMalloc(&h->mesh_slots, sizeof(int) * cap));
    KB_CUDA(h, cudaMalloc(&h->mesh_cases, cap * V));
    KB_CUDA(h, cudaMalloc(&h->mesh_tri_count, sizeof(int) * cap));
    KB_CUDA(h, cudaMalloc(&h->mesh_tri_base, sizeof(long long) * (cap + 1)));
    h->mesh_block_cap = cap;
  }
  KB_CUDA(h, cudaMemcpyAsync(h->mesh_slots, slots.data(), sizeof(int) * n, cudaMemcpyHostToDevice, h->stream));
  MeshParams p{};
  p.slots = h->mesh_slots;
  p.n_blocks = n;
  p.voxel_size = h->map.voxel_size;
  p.block_size = h->block_size;
  p.min_weight = min_weight;
  p.cases = h->mesh_cases;
  p.tri_count = h->mesh_tri_count;
  p.tri_base = h->mesh_tri_base;
  p.clear_flag = clear_updated_flag ? 1 : 0;
  launchMeshCount(h->dm, p, h->stream);
  launchMeshScan(h->mesh_tri_count, h->mesh_tri_base, n, h->stream);
  KB_CUDA(h, cudaGetLastError());
  KB_CUDA(h, cudaMemcpyAsync(h->mesh_base.data(), h->mesh_tri_base, sizeof(long long) * (n + 1), cudaMemcpyDeviceToHost, h->stream));
  KB_CUDA(h, cudaStreamSynchronize(h->stream));
  const size_t tris = static_cast<size_t>(h->mesh_base[n]);
  if (h->mesh_tri_cap < tris) {
    cudaFree(h->mesh_points); cudaFree(h->mesh_colors); cudaFree(h->mesh_labels);
    h->mesh_points = nullptr; h->mesh_colors = nullptr; h->mesh_labels = nullptr;
    h->mesh_tri_cap = 0;
    const size_t cap = tris + tris / 4 + 1024;
    KB_CUDA(h, cudaMalloc(&h->mesh_points, sizeof(float) * 9 * cap));
    KB_CUDA(h, cudaMalloc(&h->mesh_colors, 9 * cap));
    KB_CUDA(h, cudaMalloc(&h->mesh_labels, sizeof(unsigned int) * 3 * cap));
    h->mesh_tri_cap = cap;
  }
  p.points = h->mesh_points;
  p.colors = h->mesh_colors;
  p.labels = h->mesh_labels;
  launchMeshEmit(h->dm, p, h->stream);
  KB_CUDA(h, cudaGetLastError());
  if (n_vertices) *n_vertices = static_cast<int64_t>(tris) * 3;
  return KB_OK;
}

int kb_get_mesh(kb_handle* h, int32_t* block_index_xyz, int64_t* block_vertex_offsets, float* points_xyz, uint8_t* colors_rgb,
                uint32_t* labels, int64_t capacity_vertices) {
  if (!h) return KB_ERR_INVALID;
  if (!h->mesh_have) return fail(h, KB_ERR_STATE, "kb_generate_mesh has not been called");
  KB_CUDA(h, cudaSetDevice(h->device));
  const size_t n = h->mesh_index.size();
  const int64_t nv = static_cast<int64_t>(h->mesh_base[n]) * 3;
  if ((points_xyz || colors_rgb || labels) && capacity_vertices < nv) return fail(h, KB_ERR_CAPACITY, "mesh output buffers too small");
  for (size_t i = 0; i < n; ++i) {
    if (block_index_xyz) { block_index_xyz[3 * i] = h->mesh_index[i].x; block_index_xyz[3 * i + 1] = h->mesh_index[i].y; block_index_xyz[3 * i + 2] = h->mesh_index[i].z; }
    if (block_vertex_offsets) block_vertex_offsets[i] = static_cast<int64_t>(h->mesh_base[i]) * 3;
  }
  if (block_vertex_offsets) block_vertex_offsets[n] = nv;
  if (nv > 0) {
    if (points_xyz) KB_CUDA(h, cudaMemcpyAsync(points_xyz, h->mesh_points, sizeof(float) * 3 * nv, cudaMemcpyDeviceToHost, h->stream));
    if (colors_rgb) KB_CUDA(h, cudaMemcpyAsync(colors_rgb, h->mesh_colors, 3 * nv, cudaMemcpyDeviceToHost, h->stream));
    if (labels) KB_CUDA(h, cudaMemcpyAsync(labels, h->mesh_labels, sizeof(uint32_t) * nv, cudaMemcpyDeviceToHost, h->stream));
  }
  KB_CUDA(h, cudaStreamSynchronize(h->stream));
  return KB_OK;
}

int kb_num_blocks(kb_handle* h, int which, int32_t* n) {
  if (!h || !n) return KB_ERR_INVALID;
  KB_CUDA(h, cudaSetDevice(h->device));
  std::vector<int> slots; std::vector<int3> index; std::vector<uint32_t> flags;
  int st = collectSlots(h, which, &slots, &index, &flags);
  if (st != KB_OK) return st;
  *n = static_cast<int32_t>(slots.size());
  return KB_OK;
}

int kb_export_blocks(kb_handle* h, int which, int32_t max_blocks, kb_block_export* out, int32_t* n_written) {
  if (!h || !out) return KB_ERR_INVALID;
  KB_CUDA(h, cudaSetDevice(h->device));
  std::vector<int> slots; std::vector<int3> index; std::vector<uint32_t> flags;
  int st = collectSlots(h, which, &slots, &index, &flags);
  if (st != KB_OK) return st;
  const int n = std::min<int>(max_blocks, slots.size());
  const size_t V = h->dm.V, L = h->L;
  for (int i = 0; i < n; ++i) {
    if (out->block_index) { out->block_index[i * 3] = index[i].x; out->block_index[i * 3 + 1] = index[i].y; out->block_index[i * 3 + 2] = index[i].z; }
    if (out->block_flags) out->block_flags[i] = static_cast<uint8_t>(flags[i] & kPublicFlagMask);
  }
  if (out->color && n && !h->dm.color) std::memset(out->color, 0, static_cast<size_t>(n) * V * 3);  // no colour seen yet
  // Gather in chunks through dense device buffers, then copy out.
  const int chunk = 1024;
  int* d_slots = nullptr;
  unsigned long long* d_stamps = nullptr;
  char* d_buf = nullptr;
  const size_t per_block = V * (4 + 4) + V * (8 + 8 + 3) + V * (4 + 1) + V * L * 4 + 16;
  const size_t rgb_off = per_block * std::min(chunk, std::max(n, 1));  // colour gather area behind the other fields
  auto cleanup = [&]() { cudaFree(d_slots); cudaFree(d_stamps); cudaFree(d_buf); };
  auto body = [&]() -> int {
    if (n == 0) return KB_OK;
    KB_CUDA(h, cudaMalloc(&d_slots, sizeof(int) * n));
    KB_CUDA(h, cudaMemcpy(d_slots, slots.data(), sizeof(int) * n, cudaMemcpyHostToDevice));
    KB_CUDA(h, cudaMalloc(&d_stamps, sizeof(uint64_t) * h->stamps.size()));
    KB_CUDA(h, cudaMemcpy(d_stamps, h->stamps.data(), sizeof(uint64_t) * h->stamps.size(), cudaMemcpyHostToDevice));
    KB_CUDA(h, cudaMalloc(&d_buf, (per_block + V * 3) * std::min(chunk, n)));
    for (int b0 = 0; b0 < n; b0 += chunk) {
      const int nb = std::min(chunk, n - b0);
      char* q = d_buf;
      float* d_dist = reinterpret_cast<float*>(q); q += nb * V * 4;
      float* d_w = reinterpret_cast<float*>(q); q += nb * V * 4;
      unsigned long long* d_lo = reinterpret_cast<unsigned long long*>(q); q += nb * V * 8;
      unsigned long long* d_lc = reinterpret_cast<unsigned long long*>(q); q += nb * V * 8;
      uint32_t* d_lab = reinterpret_cast<uint32_t*>(q); q += nb * V * 4;
      float* d_lik = reinterpret_cast<float*>(q); q += nb * V * L * 4;
      uint8_t* d_ef = reinterpret_cast<uint8_t*>(q); q += nb * V;
      uint8_t* d_ac = reinterpret_cast<uint8_t*>(q); q += nb * V;
      uint8_t* d_tr = reinterpret_cast<uint8_t*>(q); q += nb * V;
      uint8_t* d_em = reinterpret_cast<uint8_t*>(q); q += nb * V;
      uint8_t* d_ba = reinterpret_cast<uint8_t*>(q); q += nb;
      uint8_t* d_rgb = reinterpret_cast<uint8_t*>(d_buf) + rgb_off;
      const size_t off = static_cast<size_t>(b0) * V;
      if (out->distance || out->weight) {
        launchGatherTsdf(h->dm, d_slots + b0, nb, d_dist, d_w, h->stream);
        if (out->distance) KB_CUDA(h, cudaMemcpyAsync(out->distance + off, d_dist, nb * V * 4, cudaMemcpyDeviceToHost, h->stream));
        if (out->weight) KB_CUDA(h, cudaMemcpyAsync(out->weight + off, d_w, nb * V * 4, cudaMemcpyDeviceToHost, h->stream));
      }
      if (out->color && h->dm.color) {
        launchGatherColor(h->dm, d_slots + b0, nb, d_rgb, h->stream);
        KB_CUDA(h, cudaMemcpyAsync(out->color + off * 3, d_rgb, nb * V * 3, cudaMemcpyDeviceToHost, h->stream));
      }
      const bool want_trk = out->last_observed || out->last_occupied || out->ever_free || out->active ||
                            out->to_remove || out->block_flags;
      if (want_trk) {
        if (h->map.with_tracking) {
          launchGatherTracking(h->dm, h->pass, d_slots + b0, nb, d_stamps, d_lo, d_lc, d_ef, d_ac, d_tr, d_ba, h->stream);
          if (out->block_flags) {
            std::vector<uint8_t> ba(nb);
            KB_CUDA(h, cudaMemcpyAsync(ba.data(), d_ba, nb, cudaMemcpyDeviceToHost, h->stream));
            KB_CUDA(h, cudaStreamSynchronize(h->stream));
            for (int i = 0; i < nb; ++i)
              out->block_flags[b0 + i] = static_cast<uint8_t>((out->block_flags[b0 + i] & ~KB_FLAG_HAS_ACTIVE_DATA) |
                                                              (ba[i] ? KB_FLAG_HAS_ACTIVE_DATA : 0));
          }
          if (out->last_observed) KB_CUDA(h, cudaMemcpyAsync(out->last_observed + off, d_lo, nb * V * 8, cudaMemcpyDeviceToHost, h->stream));
          if (out->last_occupied) KB_CUDA(h, cudaMemcpyAsync(out->last_occupied + off, d_lc, nb * V * 8, cudaMemcpyDeviceToHost, h->stream));
          if (out->ever_free) KB_CUDA(h, cudaMemcpyAsync(out->ever_free + off, d_ef, nb * V, cudaMemcpyDeviceToHost, h->stream));
          if (out->active) KB_CUDA(h, cudaMemcpyAsync(out->active + off, d_ac, nb * V, cudaMemcpyDeviceToHost, h->stream));
          if (out->to_remove) KB_CUDA(h, cudaMemcpyAsync(out->to_remove + off, d_tr, nb * V, cudaMemcpyDeviceToHost, h->stream));
        } else {
          if (out->last_observed) std::memset(out->last_observed + off, 0, nb * V * 8);
          if (out->last_occupied) std::memset(out->last_occupied + off, 0, nb * V * 8);
          if (out->ever_free) std::memset(out->ever_free + off, 0, nb * V);
          if (out->active) std::memset(out->active + off, 0, nb * V);
          if (out->to_remove) std::memset(out->to_remove + off, 0, nb * V);
        }
      }
      if (out->semantic_label || out->semantic_empty || out->semantic_likelihoods) {
        if (L > 0) {
          launchGatherSemantic(h->dm, d_slots + b0, nb, static_cast<int>(L), d_lab, d_em,
                               out->semantic_likelihoods ? d_lik : nullptr, h->stream);
          if (out->semantic_label) KB_CUDA(h, cudaMemcpyAsync(out->semantic_label + off, d_lab, nb * V * 4, cudaMemcpyDeviceToHost, h->stream));
          if (out->semantic_empty) KB_CUDA(h, cudaMemcpyAsync(out->semantic_empty + off, d_em, nb * V, cudaMemcpyDeviceToHost, h->stream));
          if (out->semantic_likelihoods) KB_CUDA(h, cudaMemcpyAsync(out->semantic_likelihoods + off * L, d_lik, nb * V * L * 4, cudaMemcpyDeviceToHost, h->stream));
        } else {
          if (out->semantic_label) std::memset(out->semantic_label + off, 0, nb * V * 4);
          if (out->semantic_empty) std::memset(out->semantic_empty + off, 1, nb * V);
        }
      }
      KB_CUDA(h, cudaGetLastError());
      KB_CUDA(h, cudaStreamSynchronize(h->stream));
    }
    return KB_OK;
  };
  st = body();
  cleanup();
  if (st != KB_OK) return st;
  if (n_written) *n_written = n;
  return KB_OK;
}

}  // extern "C"
