// Device-side data layout and helpers of the volumetric map (sm_90a).
//
// HBM layout (all arrays are structure-of-arrays over a fixed pool of block slots, V = vps^3):
//   hash_keys[H] u64, hash_vals[H] i32      open-addressed block hash (linear probing, tombstones)
//   block_index[S] int3, block_flags[S] u32, block_sem[S] i32 (semantic slot or -1)
//   tsdf[S][V] float2 {distance, weight}    one 8 B RMW per integrated voxel, 256 B per warp
//   last_obs[S][V] u32, last_occ[S][V] u32  frame *indices* (1-based, 0 = never); the host keeps the
//                                            index -> u64 stamp table, halving tracking traffic
//   vflags[S][V] u8                         bit0 ever_free, bit1 active, bit2 to_remove
//   sem_label[Q][V] u16 (0xFFFF = empty), sem_lik[Q][V][Lp] f32   lazily assigned semantic slots
//   color[S][V] uchar4                      TsdfVoxel::color, allocated on the first frame that carries colour
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace kb {

constexpr unsigned long long kEmptyKey = ~0ull;
constexpr unsigned long long kTombKey = ~0ull - 1ull;
constexpr uint32_t kFlagAllocated = 1u << 8;      // slot is live
constexpr uint32_t kFlagEverFreePending = 1u << 9;  // tracking_updated latched by K2 for K3
constexpr uint32_t kPublicFlagMask = 0x1Fu;
constexpr uint16_t kSemEmpty = 0xFFFFu;
// vflags bits. The tracking state is kept *lazily* (SURVEY §7 hard part 3): kVoxActive / kVoxToRemove hold
// the values as of the voxel's last write by K1 (the end of its previous observation epoch); the values
// the reference's per-frame all-block pass would have produced are derived on demand by evalTracking().
constexpr uint8_t kVoxEverFree = 1, kVoxActive = 2, kVoxToRemove = 4;
constexpr uint8_t kVoxNotOccupied = 8;  // distance >= occupancy threshold after the last write (0 = occupied,
                                        // which is also the state of a fresh voxel: distance 0 < thr)
constexpr uint32_t kFlagInactiveOverride = 1u << 10;  // kb_mark_all_inactive until the next tracking pass

struct DeviceMap {
  unsigned long long* hash_keys;
  int* hash_vals;
  uint32_t hash_mask;
  int max_blocks, max_sem;
  int vps, V, Lp;  // Lp = padded likelihood stride (multiple of 4 floats)
  int* counters;   // see Counter enum
  int* free_list;      // recycled block slots (stack)
  int* sem_free_list;  // recycled semantic slots
  int3* block_index;
  uint32_t* block_flags;
  int* block_sem;
  float2* tsdf;
  uint32_t* last_obs;
  uint32_t* last_occ;
  uint8_t* vflags;
  uint32_t* born_frame;  // [S] frame index at which the block was allocated
  uint32_t* next_pass;   // [frame idx] index of the first tracking pass at or after that frame (0 = none yet)
  uint32_t* act_min;     // [frame idx of a pass] smallest last_observed index that is 'active' at that pass
  int frame_capacity;
  uint16_t* sem_label;
  float* sem_lik;
  uchar4* color;  // [S][V] TsdfVoxel::color (rgb, w unused); null until the first frame with a colour image
  // Shard layout (kb_set_shard / kb_set_shard_cells). shard_cell == 0: per-block hash (blockOwner). shard_cell > 0:
  // square cells of shard_cell x shard_cell blocks in x/y (all z), tiled periodically over a shard_gx x shard_gy grid
  // of ranks, so spatially coherent frames touch few ranks (cellOwner).
  int shard_cell, shard_gx, shard_gy;
  // Optional explicit cell -> rank table (kb_set_shard_table): cells (cx, cy) with cx - tab_ox in [0, tab_w) and cy - tab_oy
  // in [0, tab_h) take their owner from the table (row-major, y outer); cells outside fall back to the periodic tiling.
  const uint8_t* shard_table;
  int tab_ox, tab_oy, tab_w, tab_h;
};

// Cumulative device counters (never reset on the hot path; the host reports differences).
enum Counter {
  kCtrPoolHwm = 0,     // high-water mark of block slots
  kCtrFreeCount = 1,   // entries in free_list
  kCtrSemHwm = 2,
  kCtrSemFreeCount = 3,
  kCtrLiveBlocks = 4,
  kCtrCapacityExceeded = 5,
  kCtrFrustum = 6,
  kCtrAllocated = 7,
  kCtrBlocksUpdated = 8,
  kCtrVoxelsUpdated = 9,
  kCtrVoxelsBand = 10,
  kCtrVoxelsSemantic = 11,
  kCtrSeeds = 12,
  kCtrRemoved = 13,
  kCtrErased = 14,
  kCtrWork0 = 15,  // two work-list counters used alternately by consecutive batches
  kCtrWork1 = 16,
  kCtrPairs = 17,  // (block, frame) pairs that survived K0 culling
  kCtrPending = 18,  // ever-free work list length of the current tracking pass
  kCtrFetch = 19,    // dynamic work cursor of the fuse kernel
  kCtrHalo = 20,     // sharded ever-free pass: locally owned blocks whose free masks are published this pass
  kCtrFetchB = 24,   // pipelined batches: second work cursor, so that the prologue of batch i+1 can run while the fuse
                     //   kernel of batch i is still fetching
  kCtrRehash = 28,   // number of hash-table rebuilds (tombstone garbage collection, kb_reset_inactive)
  kCtrItems0 = 32,   // item lists: non-empty culling boxes of the batch in kItemClasses weight classes (heaviest first);
  kCtrItemsB0 = 40,  //   second set for odd pipelined batches
  kNumCounters = 48
};
constexpr int kItemClasses = 8;  // by frame count: 32..29, 28..25, ..., 4..1 frames

// 64-bit cumulative totals (kb_get_totals64): the int counters above wrap after ~36 k frames of the bench workload
// (119 k voxel updates per frame). They live behind the int counters in the same allocation (8-byte aligned), so one
// device->host copy reads both.
enum Total64 {
  kTotVoxelsUpdated = 0,
  kTotVoxelsBand = 1,
  kTotVoxelsSemantic = 2,
  kTotFrustum = 3,
  kTotPairs = 4,
  kTotBlocksUpdated = 5,
  kTotAllocated = 6,
  kNumTotals = 8
};
constexpr int kCounterInts = kNumCounters + 2 * kNumTotals;  // ints in the counter allocation
__host__ __device__ inline unsigned long long* totals64(int* counters) {
  return reinterpret_cast<unsigned long long*>(counters + kNumCounters);
}

__host__ __device__ inline unsigned long long packKey(int x, int y, int z) {
  const unsigned long long o = 1ull << 20, m = (1ull << 21) - 1ull;
  return ((static_cast<unsigned long long>(x + static_cast<long long>(o)) & m)) |
         ((static_cast<unsigned long long>(y + static_cast<long long>(o)) & m) << 21) |
         ((static_cast<unsigned long long>(z + static_cast<long long>(o)) & m) << 42);
}

__host__ __device__ inline unsigned long long mix64(unsigned long long k) {
  k ^= k >> 33;
  k *= 0xff51afd7ed558ccdull;
  k ^= k >> 33;
  k *= 0xc4ceb9fe1a85ec53ull;
  k ^= k >> 33;
  return k;
}

// Shard owner of a block: upper hash bits, so it is independent of the table slot (lower bits).
__host__ __device__ inline int blockOwner(int x, int y, int z, int nranks) {
  return static_cast<int>((mix64(packKey(x, y, z)) >> 40) % static_cast<unsigned long long>(nranks));
}

// Periodic cell tiling: cell (cx, cy) = floor(block / cell) belongs to rank ((cx mod gx) + gx * (cy mod gy)) mod nranks.
__host__ __device__ inline int cellOwner(int x, int y, int cell, int gx, int gy, int nranks) {
  const int cx = (x >= 0 ? x : x - cell + 1) / cell, cy = (y >= 0 ? y : y - cell + 1) / cell;  // floor division
  const int mx = ((cx % gx) + gx) % gx, my = ((cy % gy) + gy) % gy;
  return (mx + gx * my) % nranks;
}
__host__ __device__ inline int floorDiv(int a, int b) { return (a >= 0 ? a : a - b + 1) / b; }
// Owner under an explicit cell table (`table` readable where this runs: device memory in kernels, a host copy on the host).
__host__ __device__ inline int tableOwner(const uint8_t* table, int ox, int oy, int w, int h, int cell, int gx, int gy, int x, int y,
                                          int nranks) {
  const int cx = floorDiv(x, cell) - ox, cy = floorDiv(y, cell) - oy;
  if (cx >= 0 && cx < w && cy >= 0 && cy < h) return table[cy * w + cx] % nranks;
  return cellOwner(x, y, cell, gx, gy, nranks);
}
// Owner rank of a block under the map's shard layout (device side; the host uses kb_handle's copy of the table).
__device__ inline int mapOwner(const DeviceMap& m, int x, int y, int z, int nranks) {
  if (m.shard_cell <= 0) return blockOwner(x, y, z, nranks);
  if (m.shard_table) return tableOwner(m.shard_table, m.tab_ox, m.tab_oy, m.tab_w, m.tab_h, m.shard_cell, m.shard_gx, m.shard_gy, x, y, nranks);
  return cellOwner(x, y, m.shard_cell, m.shard_gx, m.shard_gy, nranks);
}

#ifdef __CUDACC__
__device__ inline int hashLookup(const DeviceMap& m, int x, int y, int z) {
  const unsigned long long key = packKey(x, y, z);
  uint32_t h = static_cast<uint32_t>(mix64(key)) & m.hash_mask;
  for (uint32_t probe = 0; probe <= m.hash_mask; ++probe) {
    const unsigned long long k = m.hash_keys[h];
    if (k == key) return m.hash_vals[h];
    if (k == kEmptyKey) return -1;
    h = (h + 1) & m.hash_mask;
  }
  return -1;
}

// Pops a recycled slot or bumps the high-water mark. Returns -1 when the pool is exhausted.
__device__ inline int allocSlot(int* counters, int ctr_hwm, int ctr_free, const int* free_list, int cap) {
  int nfree = atomicSub(&counters[ctr_free], 1);
  if (nfree > 0) return free_list[nfree - 1];
  atomicAdd(&counters[ctr_free], 1);
  const int s = atomicAdd(&counters[ctr_hwm], 1);
  if (s >= cap) {
    atomicSub(&counters[ctr_hwm], 1);
    atomicExch(&counters[kCtrCapacityExceeded], 1);
    return -1;
  }
  return s;
}

// Finds or inserts a block. At most one thread per key calls this in any launch. *created = 1 if new.
__device__ inline int hashFindOrInsert(const DeviceMap& m, int x, int y, int z, uint32_t born, int* created) {
  const unsigned long long key = packKey(x, y, z);
  uint32_t h = static_cast<uint32_t>(mix64(key)) & m.hash_mask;
  *created = 0;
  // Pass 1: is the key present? remember the first tombstone.
  int64_t tomb = -1;
  uint32_t hh = h;
  for (uint32_t probe = 0; probe <= m.hash_mask; ++probe) {
    const unsigned long long k = m.hash_keys[hh];
    if (k == key) return m.hash_vals[hh];
    if (k == kEmptyKey) break;
    if (k == kTombKey && tomb < 0) tomb = hh;
    hh = (hh + 1) & m.hash_mask;
  }
  const int slot = allocSlot(m.counters, kCtrPoolHwm, kCtrFreeCount, m.free_list, m.max_blocks);
  if (slot < 0) return -1;
  // Pass 2: claim the tombstone or the first empty entry (other keys may race for the same entry).
  if (tomb >= 0 && atomicCAS(&m.hash_keys[tomb], kTombKey, key) == kTombKey) {
    m.hash_vals[tomb] = slot;
  } else {
    hh = h;
    bool done = false;
    for (uint32_t probe = 0; probe <= m.hash_mask && !done; ++probe) {
      unsigned long long k = m.hash_keys[hh];
      if (k == kEmptyKey || k == kTombKey) {
        if (atomicCAS(&m.hash_keys[hh], k, key) == k) {
          m.hash_vals[hh] = slot;
          done = true;
          break;
        }
      }
      hh = (hh + 1) & m.hash_mask;
    }
    if (!done) {
      atomicExch(&m.counters[kCtrCapacityExceeded], 1);
      return -1;
    }
  }
  m.block_index[slot] = make_int3(x, y, z);
  m.block_flags[slot] = kFlagAllocated;
  m.block_sem[slot] = -1;
  if (m.born_frame) m.born_frame[slot] = born;
  atomicAdd(&m.counters[kCtrLiveBlocks], 1);
  *created = 1;
  return slot;
}

// Parameters of the lazy tracking evaluation: the state of "the last tracking pass" (frame index k_last).
struct TrackEval {
  uint32_t k_last;      // frame index of the most recent tracking pass (0: none yet)
  uint32_t act_min;     // last_observed >= act_min  <=> active at pass k_last (double-seconds compare, host)
  uint32_t zero_max;    // a never-observed voxel (stamp 0) counts as active at pass k iff k <= zero_max
  uint32_t free_max;    // last_occupied < free_max  <=> toSeconds(last_occ) < toSeconds(now) - temporal_buffer
  int zero_free;        // the same predicate for last_occupied == 0
};

// Values the reference's brute-force pass (tracking_integrator.cpp:133-166,224-246) would hold for a
// voxel right after pass k_last, derived from the lazily kept state (see kb_kernels.cu, fuseKernel).
__device__ __forceinline__ void evalTracking(const DeviceMap& m, const TrackEval& t, uint32_t born, uint32_t o,
                                             uint32_t c_stored, uint8_t f, uint32_t* last_occ, bool* active,
                                             bool* to_remove) {
  const uint32_t e = o > born ? o : born;
  const bool has_pass = t.k_last != 0 && t.k_last >= e;  // a pass saw the voxel in its current epoch
  *last_occ = (has_pass && !(f & kVoxNotOccupied)) ? t.k_last : c_stored;
  bool act = (f & kVoxActive) != 0, rem = (f & kVoxToRemove) != 0;
  if (has_pass) {
    const bool act_last = o == 0 ? (t.k_last <= t.zero_max) : (o >= t.act_min);
    if (!act_last && !rem) {
      bool was = act;
      if (!was) {
        const uint32_t first = m.next_pass[e];
        was = o == 0 ? (first <= t.zero_max) : (o >= m.act_min[first]);
      }
      rem = was;
    }
    act = act_last;
  }
  *active = act;
  *to_remove = rem;
}
#endif

// Streaming multiprocessors of the current device (132 on an H100 SXM): the grid unit of the persistent,
// grid-stride kernels, whose results do not depend on the grid size.
inline int smCount() {
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
    return 1;
  return n;
}

}  // namespace kb
