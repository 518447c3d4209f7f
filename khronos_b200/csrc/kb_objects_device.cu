// Device-side semantic object detection: khronos::ConnectedSemantics::processInput
// (khronos/src/active_window/object_detection/connected_semantics.cpp:60-217) as connected-component labelling, so
// that FrameData::object_image — the label source of the ObjectIntegrator (object_integrator.cpp:76-79) — is produced
// on the GPU from the frame that is already there (SURVEY.md §8f row 2).
//
//   3D mode (semanticClustering3D :71-122 + computeCandidateVoxels :124-146): the reference groups the object-class
//     pixels by (semantic id, voxel of the world-frame vertex at grid_size) and region-grows over the 6/26
//     neighbourhood per semantic id. Here: every candidate pixel inserts its (id, voxel) key into an open-addressed
//     table (O1), one warp per occupied entry probes its neighbourhood and unions through a lock-free union-find (O2),
//     per-root atomics accumulate pixel counts and the smallest key (O3), one CTA filters by size and ranks the kept
//     roots by smallest key — semantic id ascending like the reference's std::map, then smallest voxel in (z,y,x)
//     order (the determinisation of the unordered_map iteration, docs/ORACLE_SPEC.md §13) — into ids 1..N (O4), and
//     every pixel reads its root's id (O5).
//   2D mode (semanticClustering2D :148-163 + growCluster2D :165-198 + filterClusters :200-217): union-find over the
//     pixels in the reference's column-major scan order (index u*H + v, smaller index wins, so a component's root IS
//     its first pixel in scan order); ids = 1 + number of roots before it (prefix sum), small clusters are zeroed
//     without renumbering, exactly like filterClusters.
#include <limits.h>

#include <algorithm>

#include "kb_objects_device.cuh"
#include "kb_unionfind.cuh"

namespace kb {

namespace {

constexpr unsigned long long kOsEmpty = ~0ull;
constexpr int kCoordBits = 18;  // +-131072 voxels per axis (13 km at the default 0.1 m grid)
constexpr long long kCoordBias = 1ll << (kCoordBits - 1);
constexpr unsigned long long kCoordMask = (1ull << kCoordBits) - 1ull;

// Order preserving in (semantic id, z, y, x).
__device__ __forceinline__ unsigned long long objKey(int label, int x, int y, int z) {
  return (static_cast<unsigned long long>(label) << (3 * kCoordBits)) |
         ((static_cast<unsigned long long>(z + kCoordBias) & kCoordMask) << (2 * kCoordBits)) |
         ((static_cast<unsigned long long>(y + kCoordBias) & kCoordMask) << kCoordBits) |
         (static_cast<unsigned long long>(x + kCoordBias) & kCoordMask);
}

__device__ __forceinline__ void objKeyDecode(unsigned long long k, int& label, int& x, int& y, int& z) {
  x = static_cast<int>(static_cast<long long>(k & kCoordMask) - kCoordBias);
  y = static_cast<int>(static_cast<long long>((k >> kCoordBits) & kCoordMask) - kCoordBias);
  z = static_cast<int>(static_cast<long long>((k >> (2 * kCoordBits)) & kCoordMask) - kCoordBias);
  label = static_cast<int>(k >> (3 * kCoordBits));
}

__device__ __forceinline__ bool coordOk(int c) { return c >= -kCoordBias && c < kCoordBias; }

__device__ __forceinline__ int osLookup(const MotionTable& t, unsigned long long key) {
  uint32_t h = static_cast<uint32_t>(mix64(key)) & t.mask;
  for (uint32_t probe = 0; probe <= t.mask; ++probe) {
    const unsigned long long k = t.keys[h];
    if (k == key) return static_cast<int>(h);
    if (k == kOsEmpty) return -1;
    h = (h + 1) & t.mask;
  }
  return -1;
}

__device__ __forceinline__ bool isObject(const ObjectParams& p, int label) {
  return label >= 0 && label < 64 && ((p.object_mask >> label) & 1ull);
}

// ---- 3D mode ------------------------------------------------------------------------------------------------
__global__ void osInitKernel(MotionTable t) {
  const int slot = blockIdx.x * blockDim.x + threadIdx.x;
  if (slot < kMsCount) t.scalars[slot] = 0;
  if (slot > static_cast<int>(t.mask)) return;
  t.keys[slot] = kOsEmpty;
  t.count[slot] = 0;
  t.pix_total[slot] = 0;
  t.min_seed[slot] = ~0ull;
  t.cluster_id[slot] = 0;
}

// O1: computeCandidateVoxels. No depth-validity test, like the reference (:127-145).
__global__ void osInsertKernel(MotionTable t, const __grid_constant__ ObjectParams p) {
  const int px = blockIdx.x * blockDim.x + threadIdx.x;
  if (px >= p.W * p.H) return;
  int slot = -1;
  const float range = __ldg(&p.depth[px]);
  const int label = __ldg(&p.label[px]);
  if (!(p.max_range > 0.f && range > p.max_range) && isObject(p, label)) {
    float wx, wy, wz;
    if (p.vertex) {
      wx = __ldg(&p.vertex[3 * px]); wy = __ldg(&p.vertex[3 * px + 1]); wz = __ldg(&p.vertex[3 * px + 2]);
    } else {
      const int u = px % p.W, v = px / p.W;
      const float cxn = (static_cast<float>(u) - p.cx) / p.fx * range;
      const float cyn = (static_cast<float>(v) - p.cy) / p.fy * range;
      wx = ((p.Rw[0] * cxn + p.Rw[1] * cyn) + p.Rw[2] * range) + p.tw[0];
      wy = ((p.Rw[3] * cxn + p.Rw[4] * cyn) + p.Rw[5] * range) + p.tw[1];
      wz = ((p.Rw[6] * cxn + p.Rw[7] * cyn) + p.Rw[8] * range) + p.tw[2];
    }
    const int gx = static_cast<int>(floorf(wx * p.inv_grid)), gy = static_cast<int>(floorf(wy * p.inv_grid)),
              gz = static_cast<int>(floorf(wz * p.inv_grid));
    if (coordOk(gx) && coordOk(gy) && coordOk(gz)) {
      const unsigned long long key = objKey(label, gx, gy, gz);
      uint32_t h = static_cast<uint32_t>(mix64(key)) & t.mask;
      for (uint32_t probe = 0; probe <= t.mask; ++probe) {
        unsigned long long k = t.keys[h];
        if (k == kOsEmpty) {
          k = atomicCAS(&t.keys[h], kOsEmpty, key);
          if (k == kOsEmpty) {  // this thread created the entry
            t.parent[h] = static_cast<int>(h);
            t.occupied[atomicAdd(&t.scalars[kMsOccupied], 1)] = static_cast<int>(h);
            k = key;
          }
        }
        if (k == key) { slot = static_cast<int>(h); break; }
        h = (h + 1) & t.mask;
      }
      if (slot >= 0) atomicAdd(&t.count[slot], 1u);
    }
  }
  t.pix_slot[px] = slot;
}

// O2: region growing == connected components over same-id voxels. One warp per occupied entry, lane = offset.
__global__ void __launch_bounds__(256) osLinkKernel(MotionTable t, int full) {
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = (gridDim.x * blockDim.x) >> 5;
  const int n = t.scalars[kMsOccupied];
  const int dx = lane % 3 - 1, dy = (lane / 3) % 3 - 1, dz = lane / 9 - 1;
  const int nnz = (dx != 0) + (dy != 0) + (dz != 0);
  const bool active = lane < 27 && nnz != 0 && (full || nnz == 1);
  for (int w = warp; w < n; w += n_warps) {
    const int slot = t.occupied[w];
    int label, x, y, z;
    objKeyDecode(t.keys[slot], label, x, y, z);
    if (active && coordOk(x + dx) && coordOk(y + dy) && coordOk(z + dz)) {
      const int nb = osLookup(t, objKey(label, x + dx, y + dy, z + dz));
      if (nb >= 0 && nb < slot) ufUnion(t.parent, slot, nb);  // each adjacent pair once
    }
  }
}

// O3: per-component pixel count, smallest key, list of roots.
__global__ void osReduceKernel(MotionTable t) {
  const int slot = blockIdx.x * blockDim.x + threadIdx.x;
  if (slot > static_cast<int>(t.mask)) return;
  const unsigned long long key = t.keys[slot];
  if (key == kOsEmpty) return;
  const int root = ufFind(t.parent, slot);
  atomicAdd(&t.pix_total[root], static_cast<unsigned long long>(t.count[slot]));
  atomicMin(&t.min_seed[root], key);
  if (root == slot) {
    const int i = atomicAdd(&t.scalars[kMsRoots], 1);
    if (i < t.max_roots) t.roots[i] = slot;
  }
}

// O4: size filter (:107-111) and ids = 1 + rank of the smallest key among the kept clusters (:112). Single CTA.
__global__ void osRankKernel(MotionTable t, int min_size, int max_size) {
  const int n = min(t.scalars[kMsRoots], t.max_roots);
  __shared__ int s_kept;
  if (threadIdx.x == 0) s_kept = 0;
  __syncthreads();
  const unsigned long long lo = static_cast<unsigned long long>(max(min_size, 0));
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int r = t.roots[i];
    const unsigned long long px = t.pix_total[r];
    int id = 0;
    if (px >= lo && (max_size <= 0 || px <= static_cast<unsigned long long>(max_size))) {
      const unsigned long long mine = t.min_seed[r];
      int rank = 0;
      for (int j = 0; j < n; ++j) {
        const int q = t.roots[j];
        const unsigned long long pq = t.pix_total[q];
        if (pq >= lo && (max_size <= 0 || pq <= static_cast<unsigned long long>(max_size)) && t.min_seed[q] < mine) ++rank;
      }
      id = rank + 1;
      atomicAdd(&s_kept, 1);
    }
    t.cluster_id[r] = id;
  }
  __syncthreads();
  if (threadIdx.x == 0) t.scalars[kMsClusters] = s_kept;
}

// O5: object_image (:114-116).
__global__ void osWriteKernel(MotionTable t, int32_t* __restrict__ image, int P) {
  const int px = blockIdx.x * blockDim.x + threadIdx.x;
  if (px >= P) return;
  const int slot = t.pix_slot[px];
  image[px] = slot >= 0 ? t.cluster_id[ufFind(t.parent, slot)] : 0;
}

// ---- 2D mode ------------------------------------------------------------------------------------------------
// Element index c = u*H + v (the reference's scan order); the table arrays are reused as plain per-pixel arrays.
__global__ void o2InitKernel(MotionTable t, const __grid_constant__ ObjectParams p) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < kMsCount) t.scalars[c] = 0;
  if (c >= p.W * p.H) return;
  const int u = c / p.H, v = c % p.H;
  t.parent[c] = isObject(p, __ldg(&p.label[v * p.W + u])) ? c : -1;
  t.count[c] = 0;
}

__global__ void o2LinkKernel(MotionTable t, const __grid_constant__ ObjectParams p) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= p.W * p.H || t.parent[c] < 0) return;
  const int u = c / p.H, v = c % p.H;
  const int label = __ldg(&p.label[v * p.W + u]);
  // forward half of the 4 / 8 neighbourhood: every adjacent pair is visited once
  const int du[4] = {1, 0, 1, 1}, dv[4] = {0, 1, 1, -1};
  const int n = p.full ? 4 : 2;
  for (int k = 0; k < n; ++k) {
    const int nu = u + du[k], nv = v + dv[k];
    if (nu < 0 || nv < 0 || nu >= p.W || nv >= p.H) continue;
    if (__ldg(&p.label[nv * p.W + nu]) == label) ufUnion(t.parent, c, nu * p.H + nv);  // same id => also an object
  }
}

// Pixel counts per root and root flags (deg[c] = 1 for a component's first pixel in scan order).
__global__ void o2CountKernel(MotionTable t, int P) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= P) return;
  int flag = 0;
  if (t.parent[c] >= 0) {
    const int r = ufFind(t.parent, c);
    atomicAdd(&t.count[r], 1u);
    flag = r == c ? 1 : 0;
  }
  t.deg[c] = flag;
}

// Inclusive scan of deg[] in tiles of 1024 (cluster_id[c] = inclusive count within the tile, roots[b] = tile total).
__global__ void __launch_bounds__(1024) o2ScanTilesKernel(MotionTable t, int P) {
  __shared__ int s_warp[32];
  const int c = blockIdx.x * 1024 + threadIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int v = c < P ? t.deg[c] : 0;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int n = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += n;
  }
  if (lane == 31) s_warp[warp] = v;
  __syncthreads();
  if (warp == 0) {
    int w = s_warp[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int n = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += n;
    }
    s_warp[lane] = w;
  }
  __syncthreads();
  if (warp > 0) v += s_warp[warp - 1];
  if (c < P) t.cluster_id[c] = v;
  if (threadIdx.x == 1023) t.roots[blockIdx.x] = v;
}

// Exclusive scan of the tile totals in place (single CTA; at most max_roots tiles) + number of components.
__global__ void __launch_bounds__(1024) o2ScanTotalsKernel(MotionTable t, int n_tiles) {
  __shared__ int s_carry;
  __shared__ int s_warp[32];
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int base = 0; base < n_tiles; base += 1024) {
    const int i = base + threadIdx.x;
    const int own = i < n_tiles ? t.roots[i] : 0;
    int v = own;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int n = __shfl_up_sync(0xffffffffu, v, o);
      if (lane >= o) v += n;
    }
    if (lane == 31) s_warp[warp] = v;
    __syncthreads();
    if (warp == 0) {
      int w = s_warp[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int n = __shfl_up_sync(0xffffffffu, w, o);
        if (lane >= o) w += n;
      }
      s_warp[lane] = w;
    }
    __syncthreads();
    if (warp > 0) v += s_warp[warp - 1];
    const int carry = s_carry;
    if (i < n_tiles) t.roots[i] = carry + v - own;  // exclusive
    __syncthreads();
    if (threadIdx.x == 1023) s_carry = carry + v;
    __syncthreads();
  }
  if (threadIdx.x == 0) t.scalars[kMsRoots] = s_carry;
}

// object_image: id = 1 + number of roots before the component's root; clusters below min_cluster_size are zeroed
// but keep their id slot (filterClusters :200-217). Also counts the kept clusters.
__global__ void o2WriteKernel(MotionTable t, const __grid_constant__ ObjectParams p) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= p.W * p.H) return;
  const int u = c / p.H, v = c % p.H;
  int id = 0;
  if (t.parent[c] >= 0) {
    const int r = ufFind(t.parent, c);
    const bool keep = static_cast<int>(t.count[r]) >= p.min_size;
    if (keep) id = t.cluster_id[r] + t.roots[r >> 10];
    if (keep && r == c) atomicAdd(&t.scalars[kMsClusters], 1);
  }
  p.image[v * p.W + u] = id;
}

// ---- InstanceForwarding (khronos/src/active_window/object_detection/instance_forwarding.cpp:80-149) -------------------
// The detector that forwards instance ids of an upstream segmenter: per pixel a range / background test, per id a pixel
// count and the world-frame bounding box of its vertices (for the volume filter). One pass over the image with per-id
// atomics (ids < kMaxInstanceIds); floats are ordered through the usual sign-flip encoding so atomicMin / atomicMax apply.
__device__ __forceinline__ unsigned int orderedBits(float f) {
  const unsigned int b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

__global__ void instanceForwardKernel(const __grid_constant__ ObjectParams p, const uint8_t* __restrict__ background, int max_ids,
                                      int* __restrict__ counts, unsigned int* __restrict__ bbox, uint8_t* __restrict__ keep,
                                      int* __restrict__ bad_id) {
  const int px = blockIdx.x * blockDim.x + threadIdx.x;
  if (px >= p.W * p.H) return;
  const int id = __ldg(&p.label[px]);
  uint8_t k = 0;
  if (id != 0) {
    if (id < 0 || id >= max_ids) {
      atomicExch(bad_id, 1);
    } else {
      const float range = __ldg(&p.depth[px]);
      if (!(background && background[id]) && !(p.max_range > 0.f && range > p.max_range)) {
        float wx, wy, wz;
        if (p.vertex) {
          wx = __ldg(&p.vertex[3 * px]); wy = __ldg(&p.vertex[3 * px + 1]); wz = __ldg(&p.vertex[3 * px + 2]);
        } else {
          const int u = px % p.W, v = px / p.W;
          const float cxn = (static_cast<float>(u) - p.cx) / p.fx * range;
          const float cyn = (static_cast<float>(v) - p.cy) / p.fy * range;
          wx = ((p.Rw[0] * cxn + p.Rw[1] * cyn) + p.Rw[2] * range) + p.tw[0];
          wy = ((p.Rw[3] * cxn + p.Rw[4] * cyn) + p.Rw[5] * range) + p.tw[1];
          wz = ((p.Rw[6] * cxn + p.Rw[7] * cyn) + p.Rw[8] * range) + p.tw[2];
        }
        atomicAdd(&counts[id], 1);
        unsigned int* b = bbox + static_cast<size_t>(id) * 6;
        atomicMin(&b[0], orderedBits(wx)); atomicMin(&b[1], orderedBits(wy)); atomicMin(&b[2], orderedBits(wz));
        atomicMax(&b[3], orderedBits(wx)); atomicMax(&b[4], orderedBits(wy)); atomicMax(&b[5], orderedBits(wz));
        k = 1;
      }
    }
  }
  keep[px] = k;
}

__global__ void instanceInitKernel(int max_ids, int* __restrict__ counts, unsigned int* __restrict__ bbox, int* __restrict__ bad_id) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) *bad_id = 0;
  if (i >= max_ids) return;
  counts[i] = 0;
#pragma unroll
  for (int k = 0; k < 3; ++k) { bbox[static_cast<size_t>(i) * 6 + k] = 0xFFFFFFFFu; bbox[static_cast<size_t>(i) * 6 + 3 + k] = 0u; }
}

}  // namespace

void launchObjectClustering3D(const MotionTable& t, const ObjectParams& p, cudaStream_t s) {
  const int cap = static_cast<int>(t.mask) + 1, P = p.W * p.H;
  osInitKernel<<<(cap + 255) / 256, 256, 0, s>>>(t);
  osInsertKernel<<<(P + 255) / 256, 256, 0, s>>>(t, p);
  osLinkKernel<<<smCount() * 4, 256, 0, s>>>(t, p.full);
  osReduceKernel<<<(cap + 255) / 256, 256, 0, s>>>(t);
  osRankKernel<<<1, 1024, 0, s>>>(t, p.min_size, p.max_size);
  osWriteKernel<<<(P + 255) / 256, 256, 0, s>>>(t, p.image, P);
}

void launchObjectClustering2D(const MotionTable& t, const ObjectParams& p, cudaStream_t s) {
  const int P = p.W * p.H, tiles = (P + 1023) / 1024;
  o2InitKernel<<<(P + 255) / 256, 256, 0, s>>>(t, p);
  o2LinkKernel<<<(P + 255) / 256, 256, 0, s>>>(t, p);
  o2CountKernel<<<(P + 255) / 256, 256, 0, s>>>(t, P);
  o2ScanTilesKernel<<<tiles, 1024, 0, s>>>(t, P);
  o2ScanTotalsKernel<<<1, 1024, 0, s>>>(t, tiles);
  o2WriteKernel<<<(P + 255) / 256, 256, 0, s>>>(t, p);
}

void launchInstanceForward(const ObjectParams& p, const uint8_t* background, int max_ids, int* counts, unsigned int* bbox,
                           uint8_t* keep, int* bad_id, cudaStream_t s) {
  instanceInitKernel<<<(max_ids + 255) / 256, 256, 0, s>>>(max_ids, counts, bbox, bad_id);
  const int P = p.W * p.H;
  instanceForwardKernel<<<(P + 255) / 256, 256, 0, s>>>(p, background, max_ids, counts, bbox, keep, bad_id);
}

}  // namespace kb
