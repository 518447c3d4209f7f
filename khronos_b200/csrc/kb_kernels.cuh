// Kernel parameter blocks and launch wrappers (implemented in kb_kernels.cu).
#pragma once

#include "kb_device.cuh"

namespace kb {

constexpr int kTileLevels = 4;  // depth max-pyramid: 8, 16, 32, 64 pixel tiles
constexpr int kMaxBatch = 32;  // frames fused per launch pair (bits of the per-block frame mask)

// Per-frame part of a batch (pose, image pointers, frame index).
struct FrameView {
  float R[9], t[3];  // sensor_T_world (float, rounded once from the double inverse)
  const float* depth;
  const int* label;
  const int* mask;
  const int* object_image;
  const uint8_t* color;  // H*W*3 RGB (InputData::color_image, CV_8UC3) or null
  float* tiles;   // per-frame depth max-pyramid (levels concatenated, see BatchParams::lvl_*)
  const uint16_t* depth16;  // compact inputs (device pointers) expanded into depth / label by expandFramesKernel
  const uint8_t* label8;
  float depth_scale;
  uint32_t frame_idx;
  int target_id;
};

// Everything one batch's K0 (select) + K1 (fuse) launches need, passed by value (constant bank).
struct BatchParams {
  int W, H;
  float fx, fy, cx, cy, min_range, max_range;
  float pl[4][2];  // frustum side planes (left,right,top,bottom): {lateral coeff, z coeff}
  float voxel_size, block_size, trunc, infl;
  int use_dropoff;
  float dropoff_eps;
  int constant_weight;
  float max_weight;
  int interp;
  float adaptive_thr;
  int sem_mode, L;
  float mle_diag, mle_off, mle_init;
  uint32_t label_frames;  // bit b: frame b has a label image the semantic mode reads (object image in BINARY mode)
  uint32_t mask_frames;   // bit b: frame b carries a dynamic mask
  unsigned long long blocked_mask;
  int lo[3], dims[3];  // union candidate block AABB of the batch (allocate mode)
  int allocate;        // 1: enumerate AABB + frustum test + insert; 0: all live slots
  int n_slots;         // allocate == 0: number of pool slots to scan
  int rank, nranks;
  int with_tracking;
  TrackEval trk;       // lazy tracking: state of the last tracking pass (K1 folds it in when it rewrites a voxel)
  float occ_thr;       // tsdf distance below which a voxel is occupied
  int n_frames;
  int parity;          // which of the two work-list counters this batch uses
  int compact_taps;    // 1: every frame of the batch is compact (u16 depth, u8/no labels): kernels convert per tap
  int cull;            // 1: conservative depth culling enabled
  int has_color;       // 1: some frame of the batch carries a colour image (selects the colour-blending fuse kernel)
  int lvl_tx[kTileLevels], lvl_ty[kTileLevels], lvl_off[kTileLevels];  // pyramid level dims / offsets
  int* work_slots;     // [max_work] selected block slots
  uint32_t* work_masks;  // [max_work] bit b set: block is processed for frame b of the batch
  uint32_t* work_upd;    // [max_work] bit b set: some voxel of the block was updated by frame b
  uint32_t* item_fmask;  // [max_work * items_per_block] frames (bits) for which the item survived culling
  int pipelined;         // KB_PIPELINE: the host resets this batch's counters itself (K0 must not touch the other batch's)
  int fetch_ctr;         // counter index of this batch's work cursor (kCtrFetch, or kCtrFetchB for odd pipelined batches)
  int items_ctr;         // first of the 3 item-list counters of this batch (kCtrItems0 / kCtrItemsB0)
  int coop;              // KB_FUSE_COOP: CTA-cooperative two-phase fuse kernel for long listed batches (fuseKernelCoop)
  int mlp_group;         // optional (KB_FUSE_MLP = 2 | 4): frames per memory-level-parallel group of fuseKernelMlp; 0 = fuseKernel
  int* item_list;        // optional (KB_FUSE_ITEM_LIST): 3 segments of item_list_cap box indices, non-empty boxes by
  int item_list_cap;     //   descending frame count (>= 20, >= 8, the rest): no empty fetches, heavy items start first
  int items_per_block;   // 32 (16^3 blocks) or 4 (8^3): 128-voxel culling boxes
  int layers_per_item;   // z-layers of a box one fuse item covers: 1 (long batches) or 4 (short ones)
  int max_work;
  FrameView f[kMaxBatch];
};

struct TrackingParams {
  TrackEval ev;             // state of this pass (k_last = this pass)
  uint32_t prev_pass;       // frame index of the previous pass (next_pass[] is filled for (prev, k_last])
  int connectivity;         // 6 | 18 | 26
  int n_slots;              // pool slots to scan
  int* pending;             // [max_blocks] ever-free work list (slots whose TSDF was updated since the last pass)
  int everfree_v2;          // KB_EVERFREE_V2 experiment: vectorised halo fill (everFreeKernelV2)
  // sharded pass only (everFreeKernel<true>): free masks of neighbour blocks owned by other ranks
  int rank, nranks;
  const int32_t* ghost_bits;             // the all-gathered halo buffers (see ShardExchange)
  const unsigned long long* ghost_keys;  // open-addressed block key -> int offset of the block's mask words
  const int* ghost_vals;
  uint32_t ghost_mask;
};

// Peer-memory variant of the exchanges: instead of writing a local buffer that an all-gather distributes, the producing
// kernel stores this rank's part straight into every rank's buffer (slot `rank` of the all_* layout) over NVLink peer
// mappings; the host only places a barrier between producer and consumer.
constexpr int kMaxPeers = 16;
struct PeerBuffers {
  void* p[kMaxPeers];  // base address of each rank's buffer as mapped on this device (p[rank] = the local one)
  int n;
};

// Exchange buffers of the sharded tracking pass (SURVEY.md §8e step 1), all int32 words, one per rank, concatenated
// by the all-gather:
//   pending buffer  [0] count  [1] overflow  [2..3] 0   then count x (bx, by, bz)                  (4 + 3*cap_pending words)
//   halo buffer     [0] count  [1] overflow  [2..3] 0   then count x (bx, by, bz, 0, V/32 mask words) (4 + cap_halo*(4 + V/32))
// A mask bit is the K3 neighbour predicate "ever_free || voxelIsFree at this pass" of one voxel (linear index order).
struct ShardExchange {
  int rank, nranks;
  int cap_pending, cap_halo;
  int mask_words;            // V / 32
  int* halo_mark;            // [max_blocks] 0/1: slot already in this pass's publish list
  int* publish;              // [cap_halo] slots to publish
  unsigned long long* ghost_keys;
  int* ghost_vals;
  uint32_t ghost_mask;
  __host__ __device__ int pending_stride() const { return 4 + 3 * cap_pending; }
  __host__ __device__ int halo_entry() const { return 4 + mask_words; }
  __host__ __device__ int halo_stride() const { return 4 + cap_halo * halo_entry(); }
};

struct MotionParams {
  float Rw[9], tw[3];
  int W, H;
  float fx, fy, cx, cy;
  float max_range, min_z_world;
  float block_size, block_size_inv, voxel_size_inv;
  const float* depth;
  const float* vertex;  // may be null -> computed from depth
  int3* pixel_gidx;     // out: global voxel index per pixel, x = INT_MIN if the pixel is dropped
  uint8_t* pixel_seed;  // out: 1 if the pixel's voxel is ever-free
  uint8_t* pixel_flags; // sharded lookup only: bit0 = the pixel's block exists on this rank (pixel is in the point
                        // map), bit1 = its voxel is ever-free; pixel_gidx is then written for every valid voxel index
};

void launchTileMax(const BatchParams& p, cudaStream_t s);
void launchExpandFrames(const BatchParams& p, cudaStream_t s);  // compact u16 depth / u8 labels -> f32 / i32
void launchExpandDepth(const uint16_t* src, float scale, float* dst, int n, cudaStream_t s);
void launchSelectBlocks(const DeviceMap& m, const BatchParams& p, int cull_grid, cudaStream_t s);
void launchFuse(const DeviceMap& m, const BatchParams& p, int grid, cudaStream_t s);
int fuseBlocksPerSm(int vps, int Lp);  // resident 128-thread CTAs per SM (occupancy API)
void launchTrackingPass(const DeviceMap& m, const TrackingParams& p, int everfree_grid, cudaStream_t s);
void launchResetInactive(const DeviceMap& m, const TrackEval& ev, int n_slots, int3* removed, int max_removed, cudaStream_t s);
// Rebuilds the block hash from the live slots (drops the tombstones block removal leaves behind; without this the empty
// entries of an open-addressed table only ever get fewer, and failed lookups — M1, K3 neighbours — degrade to full scans
// on long runs with block turnover).
void launchRehash(const DeviceMap& m, int n_slots, cudaStream_t s);
void launchMarkAllInactive(const DeviceMap& m, int n_slots, cudaStream_t s);
void launchClearUpdated(const DeviceMap& m, int n_slots, cudaStream_t s);
void launchMotionLookup(const DeviceMap& m, const MotionParams& p, cudaStream_t s);
// Sharded M1 (SURVEY.md §8e step 2): local lookup -> per-pixel flags; after the MAX all-reduce of the flags the
// finalize kernel drops pixels no rank has a block for, writes the seed bytes and counts the seed pixels.
void launchMotionLookupLocal(const DeviceMap& m, const MotionParams& p, cudaStream_t s);
void launchMotionFinalize(const DeviceMap& m, const uint8_t* flags, int3* gidx, uint8_t* seed, int n, cudaStream_t s);
// Sharded K2/K3: begin = K2 + export of the local ever-free work list; pack = free masks of local blocks that
// neighbour other ranks' pending blocks; finish = ghost table + K3.
void launchTrackingBegin(const DeviceMap& m, const TrackingParams& p, const ShardExchange& x, int32_t* pending_out, cudaStream_t s);
void launchHaloPack(const DeviceMap& m, const TrackingParams& p, const ShardExchange& x, const int32_t* all_pending,
                    int32_t* halo_out, cudaStream_t s);
// Peer-memory producers (see PeerBuffers): K2 + pending list into slot `rank` of every rank's all_pending buffer; free
// masks into slot `rank` of every rank's all_halo buffer; non-zero pixel flags into every rank's reduced flag image.
void launchTrackingBeginPeers(const DeviceMap& m, const TrackingParams& p, const ShardExchange& x, const PeerBuffers& peers, cudaStream_t s);
void launchHaloPackPeers(const DeviceMap& m, const TrackingParams& p, const ShardExchange& x, const int32_t* all_pending,
                         const PeerBuffers& peers, cudaStream_t s);
void launchFlagScatter(const uint8_t* local_flags, const PeerBuffers& peers, int n, cudaStream_t s);
void launchMulticastCopy(void* mc_dst, const void* src, size_t bytes, cudaStream_t s);  // bytes, both 16 B aligned
void launchTrackingFinish(const DeviceMap& m, const TrackingParams& p, const ShardExchange& x, const int32_t* all_pending,
                          const int32_t* all_halo, int everfree_grid, cudaStream_t s);
void launchAllocateBox(const DeviceMap& m, int3 lo, int3 dims, int rank, int nranks, uint32_t born, cudaStream_t s);
void launchScanConfidence(const DeviceMap& m, float min_conf, float min_obs, float trunc, int n_slots,
                          cudaStream_t s);

// Export gathers: slot_list[n] -> dense arrays (device), see kb_api.cu.
void launchGatherTsdf(const DeviceMap& m, const int* slots, int n, float* dist, float* weight, cudaStream_t s);
void launchGatherTracking(const DeviceMap& m, const TrackEval& ev, const int* slots, int n,
                          const unsigned long long* stamps, unsigned long long* last_obs,
                          unsigned long long* last_occ, uint8_t* ever_free, uint8_t* active, uint8_t* to_remove,
                          uint8_t* block_active, cudaStream_t s);
void launchGatherColor(const DeviceMap& m, const int* slots, int n, uint8_t* rgb, cudaStream_t s);
void launchGatherSemantic(const DeviceMap& m, const int* slots, int n, int L, uint32_t* label,
                          uint8_t* empty, float* lik, cudaStream_t s);

// Order-independent checksum of the whole map (see checksumKernel): out[4] = {sum, xor, blocks, observed voxels}, zeroed by
// the caller; stamps = the handle's frame index -> stamp table on the device.
void launchChecksum(const DeviceMap& m, int n_slots, const unsigned long long* stamps, unsigned long long* out, cudaStream_t s);

}  // namespace kb
