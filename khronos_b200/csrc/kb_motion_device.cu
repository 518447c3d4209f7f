// Device-side motion clustering: M2-M4 of FreeSpaceMotionDetector (clusterDynamicVoxels / mergeClusters /
// applyClusterLevelFilters / writeClustersToData, khronos/src/active_window/motion_detection/
// free_space_motion_detector.cpp:205-399) as connected-component labelling on the sparse set of voxels that
// contain points, so the per-frame pipeline keeps the dynamic image on the GPU.
//
// Equivalence with the reference (for min_separation_distance > 0; the host path handles <= 0):
//   raw cluster     = connected component of seed voxels under the 6/18/26 neighbourhood (the DFS only expands
//                     seeds) + every non-seed voxel with points adjacent to one of its seeds ("absorbed")
//   pixel count     = sum_seeds count(s) + sum_absorbed count(n) * #(adjacent seeds)   (the reference appends an
//                     absorbed voxel's pixels once per adjacent processed seed, :255-265)
//   merging         = clusters containing voxels a, b with int(sqrt(|a-b|^2)) < d, i.e. |a-b|^2 < ceil(d)^2;
//                     a shared absorbed voxel has distance 0, so with d > 0 every voxel ends in exactly one
//                     final cluster = one component of {seed-seed adjacency, seed-absorbed adjacency, near pairs}
//   order / ids     = final clusters ordered by their smallest seed in (z,y,x) order (the lowest raw index of a
//                     merged group), size-filtered, ids 1..255 saturating
// Compile with -fmad=false like the other kernels (no float math here matters for parity).
#include <limits.h>

#include <algorithm>

#include <cub/device/device_segmented_sort.cuh>

#include "kb_motion_device.cuh"
#include "kb_unionfind.cuh"

namespace kb {

namespace {

constexpr unsigned long long kVtEmpty = ~0ull;

__device__ __forceinline__ unsigned long long voxKey(int x, int y, int z) {
  // order-preserving in (z, y, x): z in the top bits
  const unsigned long long o = 1ull << 20, m = (1ull << 21) - 1ull;
  return ((static_cast<unsigned long long>(z + static_cast<long long>(o)) & m) << 42) |
         ((static_cast<unsigned long long>(y + static_cast<long long>(o)) & m) << 21) |
         (static_cast<unsigned long long>(x + static_cast<long long>(o)) & m);
}

__device__ __forceinline__ uint32_t vtHash(unsigned long long k, uint32_t mask) {
  return static_cast<uint32_t>(mix64(k)) & mask;
}

__device__ __forceinline__ int vtLookup(const MotionTable& t, int x, int y, int z) {
  const unsigned long long key = voxKey(x, y, z);
  uint32_t h = vtHash(key, t.mask);
  for (uint32_t probe = 0; probe <= t.mask; ++probe) {
    const unsigned long long k = t.keys[h];
    if (k == key) return static_cast<int>(h);
    if (k == kVtEmpty) return -1;
    h = (h + 1) & t.mask;
  }
  return -1;
}

// C1: the reference's BlockToPointsMap: every valid pixel inserts its voxel; slots double as entry ids.
__global__ void vtInsertKernel(MotionTable t, const int3* __restrict__ gidx, const uint8_t* __restrict__ seed, int P) {
  const int px = blockIdx.x * blockDim.x + threadIdx.x;
  if (px >= P || *t.gate == 0) return;
  const int3 g = gidx[px];
  int slot = -1;
  if (g.x != INT_MIN) {
    const unsigned long long key = voxKey(g.x, g.y, g.z);
    uint32_t h = vtHash(key, t.mask);
    for (uint32_t probe = 0; probe <= t.mask; ++probe) {
      unsigned long long k = t.keys[h];
      if (k == kVtEmpty) {
        k = atomicCAS(&t.keys[h], kVtEmpty, key);
        if (k == kVtEmpty) {  // this thread created the entry
          t.parent[h] = static_cast<int>(h);
          t.occupied[atomicAdd(&t.scalars[kMsOccupied], 1)] = static_cast<int>(h);
          k = key;
        }
      }
      if (k == key) { slot = static_cast<int>(h); break; }
      h = (h + 1) & t.mask;
    }
    if (slot >= 0) {
      atomicAdd(&t.count[slot], 1u);
      if (seed[px]) t.flags[slot] = kMvSeed;  // all pixels of a voxel agree on the seed bit
    }
  }
  t.pix_slot[px] = slot;
}

__device__ __forceinline__ bool inConn(int dx, int dy, int dz, int conn) {
  const int nnz = (dx != 0) + (dy != 0) + (dz != 0);
  return nnz != 0 && !(conn == 6 && nnz > 1) && !(conn == 18 && nnz > 2);
}

__device__ __forceinline__ void keyToVox(unsigned long long k, int& x, int& y, int& z) {
  const long long o = 1ll << 20;
  const unsigned long long m = (1ull << 21) - 1ull;
  x = static_cast<int>(static_cast<long long>(k & m) - o);
  y = static_cast<int>(static_cast<long long>((k >> 21) & m) - o);
  z = static_cast<int>(static_cast<long long>((k >> 42) & m) - o);
}

// C2: seed-seed and seed-absorbed adjacency; counts an absorbed voxel's adjacent seeds (deg).
// One warp per occupied voxel, lane = neighbour offset (27 cells of the 3x3x3 cube), so the hash probes of a
// voxel's neighbourhood run in parallel instead of as 26 dependent chains.
__global__ void __launch_bounds__(256) vtLinkKernel(MotionTable t, int conn) {
  if (*t.gate == 0) return;
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = (gridDim.x * blockDim.x) >> 5;
  const int n = t.scalars[kMsOccupied];
  const int dx = lane % 3 - 1, dy = (lane / 3) % 3 - 1, dz = lane / 9 - 1;
  const bool active = lane < 27 && inConn(dx, dy, dz, conn);
  for (int w = warp; w < n; w += n_warps) {
    const int slot = t.occupied[w];
    int x, y, z;
    keyToVox(t.keys[slot], x, y, z);
    const bool is_seed = t.flags[slot] & kMvSeed;
    bool nb_seed = false;
    if (active) {
      const int nb = vtLookup(t, x + dx, y + dy, z + dz);
      nb_seed = nb >= 0 && (t.flags[nb] & kMvSeed);
      if (nb_seed && (!is_seed || nb < slot)) ufUnion(t.parent, slot, nb);  // each seed pair once; absorbed -> all its seeds
    }
    const int deg = __popc(__ballot_sync(0xffffffffu, nb_seed));
    if (lane == 0) {
      if (is_seed) {
        atomicAdd(&t.scalars[kMsSeeds], 1);
        t.deg[slot] = 1;
      } else {
        t.deg[slot] = deg;  // 0: not part of any cluster
      }
    }
  }
}

// C3: merge clusters closer than min_separation_distance: |a-b|^2 < D^2 with D = ceil(d). One warp per cluster
// voxel; the lanes stride over the (2D-1)^3 offset cube.
__global__ void __launch_bounds__(256) vtMergeNearKernel(MotionTable t, int D) {
  if (*t.gate == 0) return;
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = (gridDim.x * blockDim.x) >> 5;
  const int n = t.scalars[kMsOccupied];
  const int side = 2 * D - 1, cells = side * side * side, D2 = D * D;
  for (int w = warp; w < n; w += n_warps) {
    const int slot = t.occupied[w];
    if (t.deg[slot] == 0) continue;
    int x, y, z;
    keyToVox(t.keys[slot], x, y, z);
    for (int c = lane; c < cells; c += 32) {
      const int dx = c % side - (D - 1), dy = (c / side) % side - (D - 1), dz = c / (side * side) - (D - 1);
      const int s = dx * dx + dy * dy + dz * dz;
      if (s == 0 || s >= D2) continue;
      const int nb = vtLookup(t, x + dx, y + dy, z + dz);
      if (nb >= 0 && nb < slot && t.deg[nb] != 0) ufUnion(t.parent, slot, nb);
    }
  }
}

// C4: per-component reductions: pixel multiset size, smallest seed, member list of roots.
__global__ void vtReduceKernel(MotionTable t) {
  const int slot = blockIdx.x * blockDim.x + threadIdx.x;
  if (slot > static_cast<int>(t.mask) || *t.gate == 0) return;
  const unsigned long long key = t.keys[slot];
  if (key == kVtEmpty || t.deg[slot] == 0) return;
  const int root = ufFind(t.parent, slot);
  const bool is_seed = t.flags[slot] & kMvSeed;
  atomicAdd(&t.pix_total[root], static_cast<unsigned long long>(t.count[slot]) * static_cast<unsigned long long>(is_seed ? 1 : t.deg[slot]));
  if (is_seed) atomicMin(&t.min_seed[root], key);
  if (root == slot) {
    const int i = atomicAdd(&t.scalars[kMsRoots], 1);
    if (i < t.max_roots) t.roots[i] = slot;
  }
}

// C5: size filter + ranking by smallest seed -> cluster ids. Single CTA, quadratic in the number of roots: cheap for the
// usual handful of clusters; a frame with thousands of isolated components (up to one root per pixel) pays n^2 / 1024
// steps per thread, which only pathological frames reach.
__global__ void vtRankKernel(MotionTable t, int min_size, int max_size) {
  if (*t.gate == 0) return;
  const int n = min(t.scalars[kMsRoots], t.max_roots);
  __shared__ int s_kept;
  if (threadIdx.x == 0) s_kept = 0;
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int r = t.roots[i];
    const unsigned long long px = t.pix_total[r];
    const bool keep = px >= static_cast<unsigned long long>(max(min_size, 0)) && px <= static_cast<unsigned long long>(max(max_size, 0));
    int id = 0;
    if (keep) {
      const unsigned long long mine = t.min_seed[r];
      int rank = 0;
      for (int j = 0; j < n; ++j) {
        const int q = t.roots[j];
        const unsigned long long pq = t.pix_total[q];
        if (pq >= static_cast<unsigned long long>(max(min_size, 0)) && pq <= static_cast<unsigned long long>(max(max_size, 0)) && t.min_seed[q] < mine) ++rank;
      }
      id = rank + 1;  // the image saturates it at 255 (:390-395); the cluster lists need the rank itself
      atomicAdd(&s_kept, 1);
    }
    t.cluster_id[r] = id;
  }
  __syncthreads();
  if (threadIdx.x == 0) t.scalars[kMsClusters] = s_kept;
}

// C6: writeClustersToData: every pixel of a cluster voxel gets the cluster id.
__global__ void vtWriteImageKernel(MotionTable t, int32_t* __restrict__ image, int P) {
  const int px = blockIdx.x * blockDim.x + threadIdx.x;
  if (px >= P) return;
  int id = 0;
  if (*t.gate != 0) {
    const int slot = t.pix_slot[px];
    if (slot >= 0 && t.deg[slot] != 0) id = min(t.cluster_id[ufFind(t.parent, slot)], 255);
  }
  image[px] = id;  // no seeds: an all-zero dynamic image
}

__global__ void vtInitKernel(MotionTable t) {
  const int slot = blockIdx.x * blockDim.x + threadIdx.x;
  if (slot < kMsCount) t.scalars[slot] = 0;
  if (slot > static_cast<int>(t.mask) || *t.gate == 0) return;
  t.keys[slot] = kVtEmpty;
  t.count[slot] = 0;
  t.flags[slot] = 0;
  t.deg[slot] = 0;
  t.pix_total[slot] = 0;
  t.min_seed[slot] = ~0ull;
  t.cluster_id[slot] = 0;
}

// ---- sparse variants (KB_MOTION_SPARSE=1): the table is kept clean between frames by resetting only the slots the frame
// occupied (vtCleanupKernel), so neither the init nor the reduction has to walk all 2^20 slots (~8 us each at 640x480).
// Unconditional full reset (vtInitKernel skips the table when the frame has no seeds, which would leave another user's
// entries behind for the first frame that has some).
__global__ void vtInitFullKernel(MotionTable t) {
  const int slot = blockIdx.x * blockDim.x + threadIdx.x;
  if (slot < kMsCount) t.scalars[slot] = 0;
  if (slot > static_cast<int>(t.mask)) return;
  t.keys[slot] = kVtEmpty;
  t.count[slot] = 0;
  t.flags[slot] = 0;
  t.deg[slot] = 0;
  t.pix_total[slot] = 0;
  t.min_seed[slot] = ~0ull;
  t.cluster_id[slot] = 0;
}

__global__ void vtInitSparseKernel(MotionTable t) {
  if (threadIdx.x < kMsCount) t.scalars[threadIdx.x] = 0;
}

__global__ void vtReduceSparseKernel(MotionTable t) {
  if (*t.gate == 0) return;
  const int n = t.scalars[kMsOccupied];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int slot = t.occupied[i];
    if (t.deg[slot] == 0) continue;
    const unsigned long long key = t.keys[slot];
    const int root = ufFind(t.parent, slot);
    const bool is_seed = t.flags[slot] & kMvSeed;
    atomicAdd(&t.pix_total[root], static_cast<unsigned long long>(t.count[slot]) * static_cast<unsigned long long>(is_seed ? 1 : t.deg[slot]));
    if (is_seed) atomicMin(&t.min_seed[root], key);
    if (root == slot) {
      const int r = atomicAdd(&t.scalars[kMsRoots], 1);
      if (r < t.max_roots) t.roots[r] = slot;
    }
  }
}

__global__ void vtCleanupKernel(MotionTable t) {
  if (*t.gate == 0) return;
  const int n = t.scalars[kMsOccupied];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int slot = t.occupied[i];
    t.keys[slot] = kVtEmpty;
    t.count[slot] = 0;
    t.flags[slot] = 0;
    t.deg[slot] = 0;
    t.pix_total[slot] = 0;
    t.min_seed[slot] = ~0ull;
    t.cluster_id[slot] = 0;
  }
}

// ---- cluster lists (kb_get_motion_clusters) ----

// Cluster index (0-based rank, not saturating) of an occupied slot, or -1 when the slot is in no kept cluster.
__device__ __forceinline__ int listCluster(const MotionTable& t, int slot) {
  if (slot < 0 || t.deg[slot] == 0) return -1;
  return t.cluster_id[ufFind(t.parent, slot)] - 1;
}

// Reserves n consecutive entries of ctr[c] for each lane with c >= 0 and returns the first; lanes that share c take one
// atomic between them (a cluster's voxels and pixels arrive in runs). Every lane of the warp must call it.
__device__ __forceinline__ int warpReserve(int* ctr, int c, int n) {
  const unsigned peers = __match_any_sync(0xffffffffu, c);
  const int lane = threadIdx.x & 31;
  int before = 0, total = 0;
  for (int l = 0; l < 32; ++l) {
    const int v = __shfl_sync(0xffffffffu, n, l);
    if ((peers >> l) & 1u) {
      total += v;
      if (l < lane) before += v;
    }
  }
  const int leader = __ffs(peers) - 1;
  int base = 0;
  if (lane == leader && c >= 0) base = atomicAdd(&ctr[c], total);
  return __shfl_sync(0xffffffffu, base, leader) + before;
}

// Order-preserving integer image of a float: min / max of the images is the IEEE 754-2019 minimum / maximum, which
// puts -0 below +0, so a box does not depend on the (unspecified) order of the cluster's pixels.
__device__ __forceinline__ unsigned int floatOrder(float f) {
  const unsigned int b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float orderFloat(unsigned int o) {
  return __uint_as_float((o & 0x80000000u) ? (o & 0x7FFFFFFFu) : ~o);
}

// Per-cluster pixel counts (from the roots) and voxel counts. Warps walk the occupied list together (warpReserve).
__global__ void __launch_bounds__(256) lsCountKernel(MotionTable t, MotionLists l) {
  const int n = t.scalars[kMsOccupied];
  const int lane = threadIdx.x & 31;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i - lane < n; i += gridDim.x * blockDim.x) {
    const int slot = i < n ? t.occupied[i] : -1;
    const int c = listCluster(t, slot);
    warpReserve(l.vox_count, c, 1);
    if (c >= 0 && t.parent[slot] == slot) l.pix_count[c] = static_cast<int>(t.pix_total[slot]);
  }
}

// Places every kept voxel's key in its cluster's voxel range and reserves count * multiplicity pixel positions for it
// (the reference appends an absorbed voxel's pixels once per adjacent seed).
__global__ void __launch_bounds__(256) lsVoxelKernel(MotionTable t, MotionLists l) {
  const int n = t.scalars[kMsOccupied];
  const int lane = threadIdx.x & 31;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i - lane < n; i += gridDim.x * blockDim.x) {
    const int slot = i < n ? t.occupied[i] : -1;
    const int c = listCluster(t, slot);
    const int mult = c < 0 ? 0 : ((t.flags[slot] & kMvSeed) ? 1 : t.deg[slot]);
    const int v = warpReserve(l.vox_fill, c, 1);
    const int p = warpReserve(l.pix_fill, c, c < 0 ? 0 : static_cast<int>(t.count[slot]) * mult);
    if (c >= 0) {
      l.vox_keys[l.vox_off[c] + v] = t.keys[slot];
      l.vox_next[slot] = l.pix_off[c] + p;
    }
  }
}

// Writes each pixel of a kept voxel at its voxel's next position and at the same place in every further copy, and folds
// its world point into the cluster's box (one atomic per run of same-cluster lanes per bound).
__global__ void __launch_bounds__(256) lsPixelKernel(MotionTable t, MotionLists l, const __grid_constant__ MotionBoxParams b, int P) {
  const int px = blockIdx.x * blockDim.x + threadIdx.x;
  const int slot = px < P ? t.pix_slot[px] : -1;
  const int c = listCluster(t, slot);
  const int u = px % b.W, v = px / b.W;
  float w[3] = {0.f, 0.f, 0.f};
  if (c >= 0) {
    const int n = static_cast<int>(t.count[slot]);
    const int mult = (t.flags[slot] & kMvSeed) ? 1 : t.deg[slot];
    const int pos = atomicAdd(&l.vox_next[slot], 1);
    for (int k = 0; k < mult; ++k) {
      l.pixels_uv[2 * (pos + k * n)] = u;
      l.pixels_uv[2 * (pos + k * n) + 1] = v;
    }
    if (b.vertex) {
      w[0] = b.vertex[3 * px]; w[1] = b.vertex[3 * px + 1]; w[2] = b.vertex[3 * px + 2];
    } else {  // kb_motion_host.cpp's back-projection, op for op
      const float d = b.depth[px];
      const float x = __fmul_rn(__fdiv_rn(__fsub_rn(static_cast<float>(u), b.cx), b.fx), d);
      const float y = __fmul_rn(__fdiv_rn(__fsub_rn(static_cast<float>(v), b.cy), b.fy), d);
      for (int a = 0; a < 3; ++a)
        w[a] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(b.Rw[3 * a], x), __fmul_rn(b.Rw[3 * a + 1], y)), __fmul_rn(b.Rw[3 * a + 2], d)), b.tw[a]);
    }
  }
  const unsigned peers = __match_any_sync(0xffffffffu, c);
  const bool leader = (threadIdx.x & 31) == __ffs(peers) - 1;
  for (int a = 0; a < 3; ++a) {
    const unsigned int o = floatOrder(w[a]);
    const unsigned int lo = __reduce_min_sync(peers, o), hi = __reduce_max_sync(peers, o);
    if (leader && c >= 0) {
      atomicMin(&l.box_min[3 * c + a], lo);
      atomicMax(&l.box_max[3 * c + a], hi);
    }
  }
}

__global__ void lsDecodeKernel(MotionLists l, int n_voxels, int n_clusters) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_voxels; i += gridDim.x * blockDim.x) {
    int x, y, z;
    keyToVox(l.vox_sorted[i], x, y, z);
    l.voxels_xyz[3 * i] = x; l.voxels_xyz[3 * i + 1] = y; l.voxels_xyz[3 * i + 2] = z;
  }
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < n_clusters; c += gridDim.x * blockDim.x)
    for (int a = 0; a < 3; ++a) {
      l.bbox[6 * c + a] = orderFloat(l.box_min[3 * c + a]);
      l.bbox[6 * c + 3 + a] = orderFloat(l.box_max[3 * c + a]);
    }
}

}  // namespace

void launchMotionListCounts(const MotionTable& t, const MotionLists& l, const int3* gidx, const uint8_t* seed, int P, int conn,
                            int D, int min_size, int max_size, int n_clusters, cudaStream_t s) {
  vtInitSparseKernel<<<1, 32, 0, s>>>(t);
  vtInsertKernel<<<(P + 255) / 256, 256, 0, s>>>(t, gidx, seed, P);
  vtLinkKernel<<<smCount() * 4, 256, 0, s>>>(t, conn);
  if (D > 1) vtMergeNearKernel<<<smCount() * 4, 256, 0, s>>>(t, D);
  vtReduceSparseKernel<<<smCount(), 256, 0, s>>>(t);
  vtRankKernel<<<1, 1024, 0, s>>>(t, min_size, max_size);
  cudaMemsetAsync(l.vox_count, 0, sizeof(int) * n_clusters, s);
  lsCountKernel<<<smCount() * 4, 256, 0, s>>>(t, l);
}

cudaError_t launchMotionListFill(const MotionTable& t, const MotionLists& l, const MotionBoxParams& b, int P, int n_clusters,
                                 int total_voxels, void* sort_tmp, size_t* sort_tmp_bytes, cudaStream_t s) {
  if (!sort_tmp)  // size query only
    return cub::DeviceSegmentedSort::SortKeys(nullptr, *sort_tmp_bytes, l.vox_keys, l.vox_sorted, total_voxels, n_clusters,
                                              l.vox_off, l.vox_off + 1, s);
  cudaMemsetAsync(l.pix_fill, 0, sizeof(int) * n_clusters, s);
  cudaMemsetAsync(l.vox_fill, 0, sizeof(int) * n_clusters, s);
  cudaMemsetAsync(l.box_min, 0xFF, sizeof(unsigned int) * 3 * n_clusters, s);
  cudaMemsetAsync(l.box_max, 0, sizeof(unsigned int) * 3 * n_clusters, s);
  lsVoxelKernel<<<smCount() * 4, 256, 0, s>>>(t, l);
  lsPixelKernel<<<(P + 255) / 256, 256, 0, s>>>(t, l, b, P);
  const cudaError_t e = cub::DeviceSegmentedSort::SortKeys(sort_tmp, *sort_tmp_bytes, l.vox_keys, l.vox_sorted, total_voxels,
                                                           n_clusters, l.vox_off, l.vox_off + 1, s);
  if (e != cudaSuccess) return e;
  lsDecodeKernel<<<smCount(), 256, 0, s>>>(l, total_voxels, n_clusters);
  vtCleanupKernel<<<smCount(), 256, 0, s>>>(t);  // the list table stays clean for the next call
  return cudaGetLastError();
}

void launchMotionClusteringSparse(const MotionTable& t, const int3* gidx, const uint8_t* seed, int P, int conn, int D,
                                  int min_size, int max_size, int32_t* image, bool table_dirty, cudaStream_t s) {
  const int cap = static_cast<int>(t.mask) + 1;
  if (table_dirty) vtInitFullKernel<<<(cap + 255) / 256, 256, 0, s>>>(t);  // someone else used the table: full reset once
  else vtInitSparseKernel<<<1, 32, 0, s>>>(t);
  vtInsertKernel<<<(P + 255) / 256, 256, 0, s>>>(t, gidx, seed, P);
  vtLinkKernel<<<smCount() * 4, 256, 0, s>>>(t, conn);
  if (D > 1) vtMergeNearKernel<<<smCount() * 4, 256, 0, s>>>(t, D);
  vtReduceSparseKernel<<<smCount(), 256, 0, s>>>(t);
  vtRankKernel<<<1, 1024, 0, s>>>(t, min_size, max_size);
  vtWriteImageKernel<<<(P + 255) / 256, 256, 0, s>>>(t, image, P);
  vtCleanupKernel<<<smCount(), 256, 0, s>>>(t);
}

void launchMotionClustering(const MotionTable& t, const int3* gidx, const uint8_t* seed, int P, int conn, int D,
                            int min_size, int max_size, int32_t* image, cudaStream_t s) {
  const int cap = static_cast<int>(t.mask) + 1;
  vtInitKernel<<<(cap + 255) / 256, 256, 0, s>>>(t);
  vtInsertKernel<<<(P + 255) / 256, 256, 0, s>>>(t, gidx, seed, P);
  vtLinkKernel<<<smCount() * 4, 256, 0, s>>>(t, conn);     // persistent warps over the occupied-voxel list
  if (D > 1) vtMergeNearKernel<<<smCount() * 4, 256, 0, s>>>(t, D);
  vtReduceKernel<<<(cap + 255) / 256, 256, 0, s>>>(t);
  vtRankKernel<<<1, 1024, 0, s>>>(t, min_size, max_size);
  vtWriteImageKernel<<<(P + 255) / 256, 256, 0, s>>>(t, image, P);
}

}  // namespace kb
