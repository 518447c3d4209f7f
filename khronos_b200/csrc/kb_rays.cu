// Ray index: khronos::RayVerificator on the device (khronos/src/backend/change_detection/ray_verificator.cpp; SURVEY.md
// §8f row 3 — "the only real ray-march in the repo"). The verificator hashes every measurement ray (sensor position at a
// pose-graph node -> mesh vertex) into the coarse blocks it passes through (addRayToHash :326-350) and later asks, for a
// query point, which of the rays through the point's block saw it, saw through it, or were occluded before it
// (check :66-146). Both halves are data parallel over rays / points and run on the same block-hash machinery as the map:
//
//   R0  one thread per new ray marches it in steps of block_size / 4 and counts the distinct blocks it enters. Along a
//       straight ray every coordinate of source + d * direction is monotone in d, so a ray never re-enters a block: "the
//       index changed since the previous step" is exactly the reference's set insertion.
//   R1  (after a host-side exclusive scan of the counts) the same march writes (block key, ray) pairs.
//   B1-B3  CSR "block -> rays" over ALL pairs: open-addressed table of block keys (sized by the distinct blocks, grown 4x when
//       the count pass finds it more than half full) with a count per slot, one-CTA
//       exclusive scan over the slots, scatter of the ray indices (order within a block is unspecified, as in the
//       reference's unordered_set<size_t>).
//   C1  one warp per query point: table lookup of the point's block, lanes stride over the block's rays, classify each
//       (time window, radial distance, depth test: no overlap / occluded / absent / match), warp-reduce the counts.
//   C2  (after a host-side scan) the same loop writes the rays' timestamps into the point's absent / present segments
//       (ballot + popc ranks); the host sorts each segment ascending — the consumers bucket the stamps into a time series
//       (ray_change_detector.cpp:72-81), so order is immaterial and sorting makes the result deterministic.
//
// Rays are "deformable": the reference looks the endpoints up in the current scene graph at every check (RayLookup,
// :88, :330) but hashes a ray only once, with the endpoints it had when it was added. kb_rays_add therefore stores the
// endpoints it is given, and kb_rays_set_endpoints replaces all of them after a deformation without touching the hash.
#include <stdint.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include <cuda_runtime.h>
#include <cub/device/device_scan.cuh>

#include "../../include/khronos_b200.h"
#include "kb_device.cuh"

namespace kb {
namespace {

constexpr unsigned long long kRaysEmpty = ~0ull;
constexpr int kMaxMarchSteps = 1 << 22;  // guard: 4 M steps of block_size / 4 (1000 km at 1 m blocks)

struct RayTable {
  unsigned long long* keys;  // block keys (packKey), ~0 = empty
  int* count;                // rays in the block
  int* offset;               // start of the block's ray list
  int* cursor;               // fill cursor
  uint32_t mask;
};

struct Vec3 { float x, y, z; };

__device__ __forceinline__ Vec3 load3(const float* p, long long i) { return Vec3{p[3 * i], p[3 * i + 1], p[3 * i + 2]}; }
__device__ __forceinline__ Vec3 sub(Vec3 a, Vec3 b) { return Vec3{a.x - b.x, a.y - b.y, a.z - b.z}; }
// Eigen (unvectorised 3-vectors): squaredNorm = (x*x + y*y) + z*z, norm = sqrt(squaredNorm), normalized = v / sqrt(n) if n > 0
__device__ __forceinline__ float sqnorm(Vec3 a) { return (a.x * a.x + a.y * a.y) + a.z * a.z; }
__device__ __forceinline__ float dot(Vec3 a, Vec3 b) { return (a.x * b.x + a.y * b.y) + a.z * b.z; }
__device__ __forceinline__ Vec3 normalized(Vec3 a) {
  const float n = sqnorm(a);
  if (n > 0.f) { const float s = sqrtf(n); return Vec3{a.x / s, a.y / s, a.z / s}; }
  return a;
}
__device__ __forceinline__ Vec3 cross(Vec3 a, Vec3 b) {
  return Vec3{a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x};
}

__device__ __forceinline__ bool blockOf(Vec3 p, float inv_block, unsigned long long* key) {
  const float fx = floorf(p.x * inv_block), fy = floorf(p.y * inv_block), fz = floorf(p.z * inv_block);
  const float lim = 1048576.f;  // 2^20 blocks per axis (packKey)
  if (!(fabsf(fx) < lim && fabsf(fy) < lim && fabsf(fz) < lim)) return false;
  *key = packKey(static_cast<int>(fx), static_cast<int>(fy), static_cast<int>(fz));
  return true;
}

// addRayToHash (:326-350). WRITE = false counts the blocks, WRITE = true stores (key, ray) pairs at out[offset...].
template <bool WRITE>
__global__ void rayMarchKernel(const float* __restrict__ src, const float* __restrict__ dst, int first, int n, float block_size,
                               int* __restrict__ counts, const long long* __restrict__ offsets,
                               unsigned long long* __restrict__ pair_keys, int* __restrict__ pair_rays) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int ray = first + i;
  const Vec3 source = load3(src, ray), target = load3(dst, ray);
  const Vec3 d = sub(target, source);
  const Vec3 direction = normalized(d);
  const float max_depth = sqrtf(sqnorm(d));
  const float ray_step = block_size / 4;
  const float inv_block = 1.f / block_size;
  float ray_distance = 0.f;
  unsigned long long prev = kRaysEmpty;
  int c = 0;
  long long o = WRITE ? offsets[i] : 0;
  for (int step = 0; step < kMaxMarchSteps && ray_distance <= max_depth; ++step) {
    ray_distance += ray_step;
    const Vec3 p{source.x + ray_distance * direction.x, source.y + ray_distance * direction.y, source.z + ray_distance * direction.z};
    unsigned long long key;
    if (!blockOf(p, inv_block, &key)) continue;
    if (key == prev) continue;
    prev = key;
    if (WRITE) { pair_keys[o] = key; pair_rays[o] = ray; ++o; }
    ++c;
  }
  if (!WRITE) counts[i] = c;
}

__global__ void tableClearKernel(RayTable t) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > t.mask) return;
  t.keys[i] = kRaysEmpty;
  t.count[i] = 0;
  t.cursor[i] = 0;
}

__device__ __forceinline__ int tableFind(const RayTable& t, unsigned long long key) {
  uint32_t h = static_cast<uint32_t>(mix64(key)) & t.mask;
  for (uint32_t probe = 0; probe <= t.mask; ++probe) {
    const unsigned long long k = t.keys[h];
    if (k == key) return static_cast<int>(h);
    if (k == kRaysEmpty) return -1;
    h = (h + 1) & t.mask;
  }
  return -1;
}

// flags[0] = number of distinct blocks inserted, flags[1] = set when a key found no slot (the host then retries with a larger table)
__global__ void tableCountKernel(RayTable t, const unsigned long long* __restrict__ pair_keys, long long n, int* __restrict__ flags) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const unsigned long long key = pair_keys[i];
  uint32_t h = static_cast<uint32_t>(mix64(key)) & t.mask;
  for (uint32_t probe = 0; probe <= t.mask; ++probe) {
    unsigned long long k = t.keys[h];
    if (k == kRaysEmpty) {
      k = atomicCAS(&t.keys[h], kRaysEmpty, key);
      if (k == kRaysEmpty) { k = key; atomicAdd(&flags[0], 1); }
    }
    if (k == key) { atomicAdd(&t.count[h], 1); return; }
    h = (h + 1) & t.mask;
  }
  flags[1] = 1;
}

// Exclusive scan of count[] into offset[] by one CTA of 1024 threads (contiguous chunks + a shared scan of the chunk sums).
__global__ void __launch_bounds__(1024) tableScanKernel(RayTable t) {
  __shared__ int sums[1024];
  const uint32_t n = t.mask + 1, chunk = (n + 1023) / 1024;
  const uint32_t b = threadIdx.x * chunk, e = b + chunk < n ? b + chunk : n;
  int s = 0;
  for (uint32_t i = b; i < e; ++i) s += t.count[i];
  sums[threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    int run = 0;
    for (int i = 0; i < 1024; ++i) { const int v = sums[i]; sums[i] = run; run += v; }
  }
  __syncthreads();
  int run = sums[threadIdx.x];
  for (uint32_t i = b; i < e; ++i) { t.offset[i] = run; run += t.count[i]; }
}

__global__ void tableFillKernel(RayTable t, const unsigned long long* __restrict__ pair_keys, const int* __restrict__ pair_rays,
                                long long n, int* __restrict__ block_rays) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const int slot = tableFind(t, pair_keys[i]);
  if (slot < 0) return;
  block_rays[t.offset[slot] + atomicAdd(&t.cursor[slot], 1)] = pair_rays[i];
}

// check (:66-146): 0 = not counted (out of the time window, no overlap, occluded), 1 = absent, 2 = present.
__device__ __forceinline__ int classify(Vec3 point, Vec3 source, Vec3 vertex, float radial_tolerance, float depth_tolerance) {
  const Vec3 ps = sub(point, source);
  const Vec3 direction = normalized(ps);
  const float depth = sqrtf(sqnorm(ps));
  const float radial_distance = sqrtf(sqnorm(cross(ps, sub(source, vertex)))) / depth;
  if (radial_distance > radial_tolerance) return 0;
  const float depth_distance = dot(sub(vertex, source), direction);
  if (depth - depth_distance > depth_tolerance) return 0;
  if (depth_distance - depth > depth_tolerance) return 1;
  return 2;
}

template <bool WRITE>
__global__ void __launch_bounds__(256) rayCheckKernel(RayTable t, const int* __restrict__ block_rays, const float* __restrict__ src,
                                                      const float* __restrict__ dst, const unsigned long long* __restrict__ stamps,
                                                      const float* __restrict__ points, const unsigned long long* __restrict__ earliest,
                                                      const unsigned long long* __restrict__ latest, int n_points, float inv_block,
                                                      float radial_tolerance, float depth_tolerance, int* __restrict__ counts,
                                                      const long long* __restrict__ out_offsets, unsigned long long* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = (gridDim.x * blockDim.x) >> 5;
  for (int pt = warp; pt < n_points; pt += n_warps) {
    const Vec3 point = load3(points, pt);
    unsigned long long key;
    int slot = -1;
    if (blockOf(point, inv_block, &key)) slot = tableFind(t, key);
    int n_absent = 0, n_present = 0;
    if (slot >= 0) {
      const int off = t.offset[slot], cnt = t.count[slot];
      const unsigned long long lo = earliest[pt], hi = latest[pt];
      long long base_a = 0, base_p = 0;
      if (WRITE) { base_a = out_offsets[pt]; base_p = base_a + counts[2 * pt]; }
      for (int b = 0; b < cnt; b += 32) {
        int cls = 0;
        unsigned long long ts = 0;
        if (b + lane < cnt) {
          const int ray = block_rays[off + b + lane];
          ts = stamps[ray];
          if (!(ts < lo || ts > hi)) cls = classify(point, load3(src, ray), load3(dst, ray), radial_tolerance, depth_tolerance);
        }
        const unsigned ma = __ballot_sync(0xffffffffu, cls == 1), mp = __ballot_sync(0xffffffffu, cls == 2);
        if (WRITE) {
          const unsigned below = (1u << lane) - 1u;
          if (cls == 1) out[base_a + n_absent + __popc(ma & below)] = ts;
          if (cls == 2) out[base_p + n_present + __popc(mp & below)] = ts;
        }
        n_absent += __popc(ma);
        n_present += __popc(mp);
      }
    }
    if (!WRITE && lane == 0) { counts[2 * pt] = n_absent; counts[2 * pt + 1] = n_present; }
  }
}

}  // namespace
}  // namespace kb

using namespace kb;

struct kb_ray_index {
  int device = 0;
  cudaStream_t stream = nullptr;
  kb_ray_config cfg{};
  // rays
  int n_rays = 0, cap_rays = 0;
  float* d_src = nullptr;
  float* d_dst = nullptr;
  unsigned long long* d_stamps = nullptr;
  // (block, ray) pairs of all rays, ray-major
  long long n_pairs = 0, cap_pairs = 0;
  unsigned long long* d_pair_keys = nullptr;
  int* d_pair_rays = nullptr;
  int* d_block_rays = nullptr;
  RayTable table{};
  uint32_t table_cap = 0;
  int* d_flags = nullptr;  // tableCountKernel: distinct blocks, overflow
  void* scan_tmp = nullptr;  // cub::DeviceScan temporary storage (large tables)
  size_t scan_tmp_bytes = 0;
  bool csr_valid = false;
  // scratch
  int* d_counts = nullptr; long long* d_offsets = nullptr; size_t cap_scratch = 0;
  float* d_points = nullptr; unsigned long long* d_early = nullptr; unsigned long long* d_late = nullptr;
  int* d_pt_counts = nullptr; long long* d_pt_offsets = nullptr; size_t cap_points = 0;
  unsigned long long* d_out = nullptr; size_t cap_out = 0;
  // scene-graph ids of the rays added through kb_rays_add_vertices (Ray::source_node as pose index, Ray::target_index); -1 otherwise
  std::vector<int32_t> ray_pose, ray_vertex;
  // last check
  std::vector<uint64_t> result_stamps;
  bool have_result = false;
  std::string err;
};

namespace {

#define KR_CUDA(h, call)                                                 \
  do {                                                                   \
    cudaError_t e_ = (call);                                             \
    if (e_ != cudaSuccess) {                                             \
      (h)->err = std::string(#call) + ": " + cudaGetErrorString(e_);     \
      return KB_ERR_CUDA;                                                \
    }                                                                    \
  } while (0)

int rfail(kb_ray_index* h, int code, const char* msg) {
  if (h) h->err = msg;
  return code;
}

template <typename T>
int growBuffer(kb_ray_index* h, T** p, size_t have_elems, size_t old_cap, size_t new_cap) {
  T* q = nullptr;
  KR_CUDA(h, cudaMalloc(reinterpret_cast<void**>(&q), std::max<size_t>(new_cap, 1) * sizeof(T)));
  if (*p && have_elems) KR_CUDA(h, cudaMemcpyAsync(q, *p, have_elems * sizeof(T), cudaMemcpyDeviceToDevice, h->stream));
  KR_CUDA(h, cudaStreamSynchronize(h->stream));
  cudaFree(*p);
  *p = q;
  (void)old_cap;
  return KB_OK;
}

bool finite3(const float* p, size_t n) {
  for (size_t i = 0; i < 3 * n; ++i)
    if (!std::isfinite(p[i])) return false;
  return true;
}

int allocTable(kb_ray_index* h, uint32_t cap) {
  // allocate the new table first: an out-of-memory during growth must leave the old (valid) table in place
  RayTable t{};
  cudaError_t e = cudaMalloc(reinterpret_cast<void**>(&t.keys), sizeof(unsigned long long) * cap);
  if (e == cudaSuccess) e = cudaMalloc(reinterpret_cast<void**>(&t.count), sizeof(int) * cap);
  if (e == cudaSuccess) e = cudaMalloc(reinterpret_cast<void**>(&t.offset), sizeof(int) * cap);
  if (e == cudaSuccess) e = cudaMalloc(reinterpret_cast<void**>(&t.cursor), sizeof(int) * cap);
  if (e != cudaSuccess) {
    cudaFree(t.keys); cudaFree(t.count); cudaFree(t.offset); cudaFree(t.cursor);
    h->err = std::string("ray table allocation: ") + cudaGetErrorString(e);
    return KB_ERR_CUDA;
  }
  cudaStreamSynchronize(h->stream);
  cudaFree(h->table.keys); cudaFree(h->table.count); cudaFree(h->table.offset); cudaFree(h->table.cursor);
  h->table = t;
  h->table_cap = cap;
  return KB_OK;
}

// The table is sized by the number of distinct blocks (usually thousands), not by the number of (block, ray) pairs
// (millions): start small, and when the count pass reports a full or more than half-full table, grow 4x and redo it.
int rebuildCsr(kb_ray_index* h) {
  if (h->csr_valid) return KB_OK;
  int st;
  if (!h->d_flags) KR_CUDA(h, cudaMalloc(reinterpret_cast<void**>(&h->d_flags), sizeof(int) * 2));
  if (h->table_cap == 0 && (st = allocTable(h, 1u << 14)) != KB_OK) return st;
  const unsigned blocks = static_cast<unsigned>((std::max<long long>(h->n_pairs, 1) + 255) / 256);
  for (;;) {
    h->table.mask = h->table_cap - 1;
    tableClearKernel<<<(h->table_cap + 255) / 256, 256, 0, h->stream>>>(h->table);
    if (h->n_pairs == 0) break;
    KR_CUDA(h, cudaMemsetAsync(h->d_flags, 0, sizeof(int) * 2, h->stream));
    tableCountKernel<<<blocks, 256, 0, h->stream>>>(h->table, h->d_pair_keys, h->n_pairs, h->d_flags);
    KR_CUDA(h, cudaGetLastError());
    int flags[2] = {0, 0};
    KR_CUDA(h, cudaMemcpyAsync(flags, h->d_flags, sizeof(int) * 2, cudaMemcpyDeviceToHost, h->stream));
    KR_CUDA(h, cudaStreamSynchronize(h->stream));
    if (!flags[1] && static_cast<uint32_t>(flags[0]) * 2u <= h->table_cap) break;
    if (h->table_cap >= (1u << 30)) return rfail(h, KB_ERR_CAPACITY, "too many distinct blocks");
    if ((st = allocTable(h, h->table_cap * 4u)) != KB_OK) return st;
  }
  if (h->table_cap <= (1u << 16)) {
    tableScanKernel<<<1, 1024, 0, h->stream>>>(h->table);  // small tables: one CTA is latency-optimal
  } else {
    // large tables (many distinct blocks): multi-CTA device scan, so a big map does not serialise on one SM
    size_t tmp_bytes = 0;
    KR_CUDA(h, cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, h->table.count, h->table.offset, static_cast<int>(h->table_cap), h->stream));
    if (tmp_bytes > h->scan_tmp_bytes) {
      KR_CUDA(h, cudaStreamSynchronize(h->stream));
      cudaFree(h->scan_tmp);
      h->scan_tmp = nullptr;
      h->scan_tmp_bytes = 0;
      KR_CUDA(h, cudaMalloc(&h->scan_tmp, tmp_bytes));
      h->scan_tmp_bytes = tmp_bytes;
    }
    KR_CUDA(h, cub::DeviceScan::ExclusiveSum(h->scan_tmp, tmp_bytes, h->table.count, h->table.offset, static_cast<int>(h->table_cap), h->stream));
  }
  if (h->n_pairs > 0) tableFillKernel<<<blocks, 256, 0, h->stream>>>(h->table, h->d_pair_keys, h->d_pair_rays, h->n_pairs, h->d_block_rays);
  KR_CUDA(h, cudaGetLastError());
  h->csr_valid = true;
  return KB_OK;
}

}  // namespace

extern "C" {

int kb_rays_create(const kb_ray_config* config, int device, kb_ray_index** out) {
  if (!config || !out) return KB_ERR_INVALID;
  *out = nullptr;
  // RayVerificator::Config checks (ray_verificator.cpp:56-61)
  if (!(config->block_size > 0.f) || !(config->radial_tolerance > 0.f) || !(config->depth_tolerance > 0.f)) return KB_ERR_INVALID;
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0 || device < 0 || device >= n) return KB_ERR_NO_DEVICE;
  if (cudaSetDevice(device) != cudaSuccess) return KB_ERR_CUDA;
  kb_ray_index* h = new kb_ray_index();
  h->device = device;
  h->cfg = *config;
  if (cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess) { delete h; return KB_ERR_CUDA; }
  *out = h;
  return KB_OK;
}

int kb_rays_destroy(kb_ray_index* h) {
  if (!h) return KB_OK;
  cudaSetDevice(h->device);
  if (h->stream) { cudaStreamSynchronize(h->stream); cudaStreamDestroy(h->stream); }
  cudaFree(h->d_src); cudaFree(h->d_dst); cudaFree(h->d_stamps); cudaFree(h->d_pair_keys); cudaFree(h->d_pair_rays);
  cudaFree(h->d_block_rays); cudaFree(h->table.keys); cudaFree(h->table.count); cudaFree(h->table.offset); cudaFree(h->table.cursor);
  cudaFree(h->d_counts); cudaFree(h->d_offsets); cudaFree(h->d_points); cudaFree(h->d_early); cudaFree(h->d_late);
  cudaFree(h->d_pt_counts); cudaFree(h->d_pt_offsets); cudaFree(h->d_out); cudaFree(h->d_flags); cudaFree(h->scan_tmp);
  delete h;
  return KB_OK;
}

const char* kb_rays_last_error(const kb_ray_index* h) { return h ? h->err.c_str() : "null handle"; }

int kb_rays_clear(kb_ray_index* h) {
  if (!h) return KB_ERR_INVALID;
  h->n_rays = 0;
  h->n_pairs = 0;
  h->csr_valid = false;
  h->have_result = false;
  h->ray_pose.clear();
  h->ray_vertex.clear();
  return KB_OK;
}

int kb_rays_size(kb_ray_index* h, int32_t* n_rays, int64_t* n_block_entries) {
  if (!h) return KB_ERR_INVALID;
  if (n_rays) *n_rays = h->n_rays;
  if (n_block_entries) *n_block_entries = h->n_pairs;
  return KB_OK;
}

int kb_rays_add(kb_ray_index* h, int32_t n, const float* sources_xyz, const float* targets_xyz, const uint64_t* timestamps,
                int32_t* observed_blocks_xyz, int32_t max_observed, int32_t* n_observed) {
  if (!h || n < 0 || (n > 0 && (!sources_xyz || !targets_xyz || !timestamps))) return rfail(h, KB_ERR_INVALID, "null argument");
  if (n_observed) *n_observed = 0;
  if (n == 0) return KB_OK;
  if (!finite3(sources_xyz, n) || !finite3(targets_xyz, n)) return rfail(h, KB_ERR_INVALID, "non-finite ray endpoint");
  KR_CUDA(h, cudaSetDevice(h->device));
  const size_t total = static_cast<size_t>(h->n_rays) + n;
  if (total > static_cast<size_t>(h->cap_rays)) {
    const size_t cap = std::max<size_t>(total, static_cast<size_t>(h->cap_rays) * 2);
    int st;
    if ((st = growBuffer(h, &h->d_src, static_cast<size_t>(h->n_rays) * 3, 0, cap * 3)) != KB_OK) return st;
    if ((st = growBuffer(h, &h->d_dst, static_cast<size_t>(h->n_rays) * 3, 0, cap * 3)) != KB_OK) return st;
    if ((st = growBuffer(h, &h->d_stamps, static_cast<size_t>(h->n_rays), 0, cap)) != KB_OK) return st;
    h->cap_rays = static_cast<int>(cap);
  }
  if (static_cast<size_t>(n) > h->cap_scratch) {
    cudaFree(h->d_counts); cudaFree(h->d_offsets);
    KR_CUDA(h, cudaMalloc(reinterpret_cast<void**>(&h->d_counts), sizeof(int) * n));
    KR_CUDA(h, cudaMalloc(reinterpret_cast<void**>(&h->d_offsets), sizeof(long long) * n));
    h->cap_scratch = n;
  }
  const int first = h->n_rays;
  KR_CUDA(h, cudaMemcpyAsync(h->d_src + 3ll * first, sources_xyz, sizeof(float) * 3 * n, cudaMemcpyHostToDevice, h->stream));
  KR_CUDA(h, cudaMemcpyAsync(h->d_dst + 3ll * first, targets_xyz, sizeof(float) * 3 * n, cudaMemcpyHostToDevice, h->stream));
  KR_CUDA(h, cudaMemcpyAsync(h->d_stamps + first, timestamps, sizeof(uint64_t) * n, cudaMemcpyHostToDevice, h->stream));
  rayMarchKernel<false><<<(n + 127) / 128, 128, 0, h->stream>>>(h->d_src, h->d_dst, first, n, h->cfg.block_size, h->d_counts, nullptr, nullptr, nullptr);
  KR_CUDA(h, cudaGetLastError());
  std::vector<int> counts(n);
  KR_CUDA(h, cudaMemcpyAsync(counts.data(), h->d_counts, sizeof(int) * n, cudaMemcpyDeviceToHost, h->stream));
  KR_CUDA(h, cudaStreamSynchronize(h->stream));
  std::vector<long long> offsets(n);
  long long run = h->n_pairs;
  for (int i = 0; i < n; ++i) { offsets[i] = run; run += counts[i]; }
  if (run > (1ll << 31) - 1) return rfail(h, KB_ERR_CAPACITY, "more than 2^31 block entries");
  if (run > h->cap_pairs) {
    const size_t cap = std::max<size_t>(static_cast<size_t>(run), static_cast<size_t>(h->cap_pairs) * 2);
    int st;
    if ((st = growBuffer(h, &h->d_pair_keys, static_cast<size_t>(h->n_pairs), 0, cap)) != KB_OK) return st;
    if ((st = growBuffer(h, &h->d_pair_rays, static_cast<size_t>(h->n_pairs), 0, cap)) != KB_OK) return st;
    cudaFree(h->d_block_rays);
    h->d_block_rays = nullptr;
    KR_CUDA(h, cudaMalloc(reinterpret_cast<void**>(&h->d_block_rays), sizeof(int) * cap));
    h->cap_pairs = static_cast<long long>(cap);
  }
  KR_CUDA(h, cudaMemcpyAsync(h->d_offsets, offsets.data(), sizeof(long long) * n, cudaMemcpyHostToDevice, h->stream));
  rayMarchKernel<true><<<(n + 127) / 128, 128, 0, h->stream>>>(h->d_src, h->d_dst, first, n, h->cfg.block_size, h->d_counts, h->d_offsets, h->d_pair_keys, h->d_pair_rays);
  KR_CUDA(h, cudaGetLastError());
  const long long new_pairs = run - h->n_pairs;
  // observed blocks of the new rays (addVertices' return value, :222-276): unique keys of the new pairs
  if (n_observed || observed_blocks_xyz) {
    std::vector<unsigned long long> keys(static_cast<size_t>(new_pairs));
    if (new_pairs) KR_CUDA(h, cudaMemcpyAsync(keys.data(), h->d_pair_keys + h->n_pairs, sizeof(unsigned long long) * new_pairs, cudaMemcpyDeviceToHost, h->stream));
    KR_CUDA(h, cudaStreamSynchronize(h->stream));
    std::sort(keys.begin(), keys.end());
    keys.erase(std::unique(keys.begin(), keys.end()), keys.end());
    if (n_observed) *n_observed = static_cast<int32_t>(keys.size());
    if (observed_blocks_xyz) {
      if (static_cast<size_t>(std::max(max_observed, 0)) < keys.size()) {
        // the rays are not added: the caller retries with a larger buffer
        return rfail(h, KB_ERR_CAPACITY, "observed block buffer too small");
      }
      const long long o = 1ll << 20, m = (1ll << 21) - 1;
      for (size_t i = 0; i < keys.size(); ++i) {  // packKey order = (z, y, x) ascending
        observed_blocks_xyz[3 * i] = static_cast<int32_t>(static_cast<long long>(keys[i] & m) - o);
        observed_blocks_xyz[3 * i + 1] = static_cast<int32_t>(static_cast<long long>((keys[i] >> 21) & m) - o);
        observed_blocks_xyz[3 * i + 2] = static_cast<int32_t>(static_cast<long long>((keys[i] >> 42) & m) - o);
      }
    }
  }
  h->n_rays = static_cast<int>(total);
  h->n_pairs = run;
  h->csr_valid = false;
  h->have_result = false;
  h->ray_pose.resize(total, -1);
  h->ray_vertex.resize(total, -1);
  return KB_OK;
}

int kb_rays_add_vertices(kb_ray_index* h, int32_t policy, float active_window_duration, int32_t n_poses, const uint64_t* pose_stamps,
                         const float* pose_positions_xyz, int32_t n_vertices, int32_t vertex_index_base, const float* vertices_xyz,
                         const uint64_t* first_seen, const uint64_t* last_seen, int32_t* observed_blocks_xyz, int32_t max_observed,
                         int32_t* n_observed, int32_t* n_rays_added) {
  if (!h || n_poses < 0 || n_vertices < 0 || (n_poses > 0 && (!pose_stamps || !pose_positions_xyz)) ||
      (n_vertices > 0 && (!vertices_xyz || !first_seen || !last_seen)))
    return rfail(h, KB_ERR_INVALID, "null argument");
  if (policy < KB_RAYS_FIRST || policy > KB_RAYS_ALL) return rfail(h, KB_ERR_INVALID, "unsupported ray policy (the random policies are not reproducible)");
  for (int i = 1; i < n_poses; ++i)
    if (pose_stamps[i] < pose_stamps[i - 1]) return rfail(h, KB_ERR_INVALID, "pose stamps must be ascending");
  if (n_observed) *n_observed = 0;
  if (n_rays_added) *n_rays_added = 0;
  // addVertices (:222-276): last_seen is shifted back by the active-window duration (:246-251), unsigned like the reference
  const uint64_t offset_ns = active_window_duration > 0.f ? static_cast<uint64_t>(active_window_duration * 1e9) : 0ull;
  const uint64_t* tb = pose_stamps;
  const uint64_t* te = pose_stamps + n_poses;
  std::vector<float> src, dst;
  std::vector<uint64_t> ts;
  std::vector<int32_t> pose_of, vertex_of;
  std::vector<size_t> sources;
  for (int v = 0; v < n_vertices; ++v) {
    const uint64_t first = first_seen[v], last = last_seen[v] - offset_ns;
    sources.clear();
    // computeVertexSources (:278-330); the result set is listed ascending
    if (policy == KB_RAYS_FIRST || policy == KB_RAYS_FIRST_AND_LAST) {
      const uint64_t* it = std::upper_bound(tb, te, first);
      if (it != te) sources.push_back(static_cast<size_t>(it - tb));
    }
    if (policy == KB_RAYS_LAST || policy == KB_RAYS_FIRST_AND_LAST) {
      const uint64_t* it = std::lower_bound(tb, te, last);
      if (it != te) sources.push_back(static_cast<size_t>(it - tb));
    }
    if (policy == KB_RAYS_MIDDLE) {
      const uint64_t stamp = (last + first) / 2;
      const uint64_t* it = std::lower_bound(tb, te, stamp);
      if (it != te) sources.push_back(static_cast<size_t>(it - tb));
    }
    if (policy == KB_RAYS_ALL) {
      const uint64_t* lo = std::upper_bound(tb, te, first);
      const uint64_t* hi = std::lower_bound(tb, te, last);
      for (const uint64_t* it = lo; it < hi; ++it) sources.push_back(static_cast<size_t>(it - tb));
    }
    std::sort(sources.begin(), sources.end());
    sources.erase(std::unique(sources.begin(), sources.end()), sources.end());
    for (size_t sidx : sources) {
      for (int a = 0; a < 3; ++a) { src.push_back(pose_positions_xyz[3 * sidx + a]); dst.push_back(vertices_xyz[3 * static_cast<size_t>(v) + a]); }
      ts.push_back(pose_stamps[sidx]);
      pose_of.push_back(static_cast<int32_t>(sidx));
      vertex_of.push_back(vertex_index_base + v);
    }
  }
  const int n = static_cast<int>(ts.size());
  const int before = h->n_rays;
  const int st = kb_rays_add(h, n, src.data(), dst.data(), ts.data(), observed_blocks_xyz, max_observed, n_observed);
  if (st != KB_OK) return st;
  for (int i = 0; i < n; ++i) { h->ray_pose[before + i] = pose_of[i]; h->ray_vertex[before + i] = vertex_of[i]; }
  if (n_rays_added) *n_rays_added = n;
  return KB_OK;
}

int kb_rays_get_ray_ids(kb_ray_index* h, int32_t* pose_index, int32_t* vertex_index, uint64_t* timestamps, int32_t capacity) {
  if (!h) return KB_ERR_INVALID;
  if (capacity < h->n_rays) return rfail(h, KB_ERR_CAPACITY, "ray id buffer too small");
  if (h->n_rays == 0) return KB_OK;
  if (pose_index) std::memcpy(pose_index, h->ray_pose.data(), sizeof(int32_t) * h->n_rays);
  if (vertex_index) std::memcpy(vertex_index, h->ray_vertex.data(), sizeof(int32_t) * h->n_rays);
  if (timestamps) {
    KR_CUDA(h, cudaSetDevice(h->device));
    KR_CUDA(h, cudaMemcpyAsync(timestamps, h->d_stamps, sizeof(uint64_t) * h->n_rays, cudaMemcpyDeviceToHost, h->stream));
    KR_CUDA(h, cudaStreamSynchronize(h->stream));
  }
  return KB_OK;
}

int kb_rays_set_endpoints(kb_ray_index* h, int32_t n_rays, const float* sources_xyz, const float* targets_xyz) {
  if (!h || !sources_xyz || !targets_xyz) return rfail(h, KB_ERR_INVALID, "null argument");
  if (n_rays != h->n_rays) return rfail(h, KB_ERR_INVALID, "endpoint count differs from the number of rays");
  if (n_rays == 0) return KB_OK;
  // same validation as kb_rays_add: a non-finite endpoint would make a later kb_rays_rehash drop rays (the reference's
  // recomputeHash never does)
  for (size_t i = 0; i < 3 * static_cast<size_t>(n_rays); ++i)
    if (!std::isfinite(sources_xyz[i]) || !std::isfinite(targets_xyz[i])) return rfail(h, KB_ERR_INVALID, "non-finite ray endpoint");
  KR_CUDA(h, cudaSetDevice(h->device));
  KR_CUDA(h, cudaMemcpyAsync(h->d_src, sources_xyz, sizeof(float) * 3 * n_rays, cudaMemcpyHostToDevice, h->stream));
  KR_CUDA(h, cudaMemcpyAsync(h->d_dst, targets_xyz, sizeof(float) * 3 * n_rays, cudaMemcpyHostToDevice, h->stream));
  KR_CUDA(h, cudaStreamSynchronize(h->stream));
  h->have_result = false;
  return KB_OK;
}

int kb_rays_rehash(kb_ray_index* h) {
  // recomputeHash (:314-324): march all rays again with their current endpoints
  if (!h) return KB_ERR_INVALID;
  const int n = h->n_rays;
  if (n == 0) return KB_OK;
  KR_CUDA(h, cudaSetDevice(h->device));
  std::vector<float> src(3 * static_cast<size_t>(n)), dst(3 * static_cast<size_t>(n));
  std::vector<uint64_t> ts(n);
  KR_CUDA(h, cudaMemcpyAsync(src.data(), h->d_src, sizeof(float) * 3 * n, cudaMemcpyDeviceToHost, h->stream));
  KR_CUDA(h, cudaMemcpyAsync(dst.data(), h->d_dst, sizeof(float) * 3 * n, cudaMemcpyDeviceToHost, h->stream));
  KR_CUDA(h, cudaMemcpyAsync(ts.data(), h->d_stamps, sizeof(uint64_t) * n, cudaMemcpyDeviceToHost, h->stream));
  KR_CUDA(h, cudaStreamSynchronize(h->stream));
  // endpoints were validated when they were set (kb_rays_add / kb_rays_set_endpoints), so the re-add cannot reject rays
  std::vector<int32_t> pose = h->ray_pose, vertex = h->ray_vertex;
  kb_rays_clear(h);
  const int st = kb_rays_add(h, n, src.data(), dst.data(), ts.data(), nullptr, 0, nullptr);
  h->ray_pose = pose;  // the scene-graph ids survive either way; after a CUDA failure the index is empty and says so
  h->ray_vertex = vertex;
  if (st != KB_OK) { h->ray_pose.resize(static_cast<size_t>(h->n_rays)); h->ray_vertex.resize(static_cast<size_t>(h->n_rays)); }
  return st;
}

int kb_rays_check(kb_ray_index* h, int32_t n_points, const float* points_xyz, const uint64_t* earliest, const uint64_t* latest,
                  int32_t* counts, int64_t* total_stamps) {
  if (!h || n_points < 0 || (n_points > 0 && (!points_xyz || !earliest || !latest || !counts))) return rfail(h, KB_ERR_INVALID, "null argument");
  h->have_result = false;
  h->result_stamps.clear();
  if (total_stamps) *total_stamps = 0;
  if (n_points == 0) { h->have_result = true; return KB_OK; }
  if (h->n_rays == 0) {  // :73-76: no measurements
    std::memset(counts, 0, sizeof(int32_t) * 2 * n_points);
    h->have_result = true;
    return KB_OK;
  }
  KR_CUDA(h, cudaSetDevice(h->device));
  int st;
  if ((st = rebuildCsr(h)) != KB_OK) return st;
  if (static_cast<size_t>(n_points) > h->cap_points) {
    cudaFree(h->d_points); cudaFree(h->d_early); cudaFree(h->d_late); cudaFree(h->d_pt_counts); cudaFree(h->d_pt_offsets);
    KR_CUDA(h, cudaMalloc(reinterpret_cast<void**>(&h->d_points), sizeof(float) * 3 * n_points));
    KR_CUDA(h, cudaMalloc(reinterpret_cast<void**>(&h->d_early), sizeof(uint64_t) * n_points));
    KR_CUDA(h, cudaMalloc(reinterpret_cast<void**>(&h->d_late), sizeof(uint64_t) * n_points));
    KR_CUDA(h, cudaMalloc(reinterpret_cast<void**>(&h->d_pt_counts), sizeof(int) * 2 * n_points));
    KR_CUDA(h, cudaMalloc(reinterpret_cast<void**>(&h->d_pt_offsets), sizeof(long long) * n_points));
    h->cap_points = n_points;
  }
  KR_CUDA(h, cudaMemcpyAsync(h->d_points, points_xyz, sizeof(float) * 3 * n_points, cudaMemcpyHostToDevice, h->stream));
  KR_CUDA(h, cudaMemcpyAsync(h->d_early, earliest, sizeof(uint64_t) * n_points, cudaMemcpyHostToDevice, h->stream));
  KR_CUDA(h, cudaMemcpyAsync(h->d_late, latest, sizeof(uint64_t) * n_points, cudaMemcpyHostToDevice, h->stream));
  const int blocks = std::min((n_points + 7) / 8, kb::smCount() * 8);
  const float inv_block = 1.f / h->cfg.block_size;
  rayCheckKernel<false><<<blocks, 256, 0, h->stream>>>(h->table, h->d_block_rays, h->d_src, h->d_dst, h->d_stamps, h->d_points, h->d_early, h->d_late, n_points, inv_block, h->cfg.radial_tolerance, h->cfg.depth_tolerance, h->d_pt_counts, nullptr, nullptr);
  KR_CUDA(h, cudaGetLastError());
  KR_CUDA(h, cudaMemcpyAsync(counts, h->d_pt_counts, sizeof(int) * 2 * n_points, cudaMemcpyDeviceToHost, h->stream));
  KR_CUDA(h, cudaStreamSynchronize(h->stream));
  std::vector<long long> offsets(n_points);
  long long run = 0;
  for (int i = 0; i < n_points; ++i) { offsets[i] = run; run += counts[2 * i] + counts[2 * i + 1]; }
  if (total_stamps) *total_stamps = run;
  h->result_stamps.resize(static_cast<size_t>(run));
  if (run > 0) {
    if (static_cast<size_t>(run) > h->cap_out) {
      cudaFree(h->d_out);
      KR_CUDA(h, cudaMalloc(reinterpret_cast<void**>(&h->d_out), sizeof(uint64_t) * run));
      h->cap_out = static_cast<size_t>(run);
    }
    KR_CUDA(h, cudaMemcpyAsync(h->d_pt_offsets, offsets.data(), sizeof(long long) * n_points, cudaMemcpyHostToDevice, h->stream));
    rayCheckKernel<true><<<blocks, 256, 0, h->stream>>>(h->table, h->d_block_rays, h->d_src, h->d_dst, h->d_stamps, h->d_points, h->d_early, h->d_late, n_points, inv_block, h->cfg.radial_tolerance, h->cfg.depth_tolerance, h->d_pt_counts, h->d_pt_offsets, h->d_out);
    KR_CUDA(h, cudaGetLastError());
    KR_CUDA(h, cudaMemcpyAsync(h->result_stamps.data(), h->d_out, sizeof(uint64_t) * run, cudaMemcpyDeviceToHost, h->stream));
    KR_CUDA(h, cudaStreamSynchronize(h->stream));
    for (int i = 0; i < n_points; ++i) {  // deterministic order within each absent / present segment
      uint64_t* a = h->result_stamps.data() + offsets[i];
      std::sort(a, a + counts[2 * i]);
      std::sort(a + counts[2 * i], a + counts[2 * i] + counts[2 * i + 1]);
    }
  }
  h->have_result = true;
  return KB_OK;
}

int kb_rays_get_stamps(kb_ray_index* h, uint64_t* stamps, int64_t capacity) {
  if (!h) return KB_ERR_INVALID;
  if (!h->have_result) return rfail(h, KB_ERR_STATE, "no check result");
  if (capacity < static_cast<int64_t>(h->result_stamps.size())) return rfail(h, KB_ERR_CAPACITY, "stamp buffer too small");
  if (!h->result_stamps.empty()) {
    if (!stamps) return rfail(h, KB_ERR_INVALID, "null argument");
    std::memcpy(stamps, h->result_stamps.data(), sizeof(uint64_t) * h->result_stamps.size());
  }
  return KB_OK;
}

}  // extern "C"
