// Hand-written sm_90a kernels of the active-window fusion hot path.
// Compile with -fmad=false: the per-voxel arithmetic must round exactly like the fp32 reference
// (no FMA contraction), integer outputs (labels, indices, flags) are bit-exact by construction.
//
//   K0     selectBlocksKernel   per batch: frustum test (+ conservative depth culling), block hash
//                               insert, semantic slot assignment, compaction into a work list
//   K1     fuseKernel           persistent CTAs over (block, z-slab) items: projective TSDF + semantic
//                               fusion of up to 32 frames with the voxel state held in registers
//   K2     trackingPassKernel   lazy tracking pass: O(blocks) bookkeeping; per-voxel last_occupied / active /
//                               to_remove are derived on demand (evalTracking) instead of rewritten per frame
//   K3     everFreeKernel       ever-free labelling with 6/18/26 neighbourhood across blocks
//   K2r    resetInactiveKernel  block removal + slot recycling
//   M1     motionLookupKernel   per-pixel endpoint voxel lookup + ever-free seed test
//   K4     scanConfidenceKernel object-extraction low-confidence erase
#include <limits.h>

#include <algorithm>
#include <type_traits>

#include "../../include/khronos_b200.h"
#include "kb_kernels.cuh"

namespace kb {

namespace {

constexpr int kThreads = 256;
constexpr int kFuseThreads = 128;  // 4 independent warps per CTA
// Floats per thread of the fuse kernels' likelihood rows (s_rows[thread][S]): Lp rounded up to an odd multiple of 4, so the
// 16 B row accesses of a quarter-warp (8 lanes) fall on 8 disjoint groups of 4 banks. BINARY rows (Lp = 2) keep the
// transposed [2][thread] layout.
__host__ __device__ constexpr int fuseRowStride(int Lp) { return Lp <= 2 ? 2 : ((Lp >> 2) | 1) << 2; }
#ifndef KB_FUSE_MIN_BLOCKS
#define KB_FUSE_MIN_BLOCKS 10      // resident CTAs per SM the fuse kernel is compiled for (register cap 65536/(128*N))
#endif
#ifndef KB_FUSE_COLOR_MIN_BLOCKS
#define KB_FUSE_COLOR_MIN_BLOCKS 8  // the colour-blending variant carries a few more live registers
#endif

__device__ __forceinline__ void xform(const float* R, const float* t, float x, float y, float z,
                                      float& ox, float& oy, float& oz) {
  ox = ((R[0] * x + R[1] * y) + R[2] * z) + t[0];
  oy = ((R[3] * x + R[4] * y) + R[5] * z) + t[1];
  oz = ((R[6] * x + R[7] * y) + R[8] * z) + t[2];
}

// hydra::Camera::pointIsInViewFrustum restated (oracle.cpp pointInFrustum): z, range and 4 planes.
__device__ __forceinline__ bool inFrustum(const BatchParams& p, float x, float y, float z) {
  const float infl = p.infl;
  if (z < -infl) return false;
  const float r = sqrtf((x * x + y * y) + z * z);
  if (r < p.min_range - infl || r > p.max_range + infl) return false;
  if (p.pl[0][0] * x + p.pl[0][1] * z < -infl) return false;
  if (p.pl[1][0] * x + p.pl[1][1] * z < -infl) return false;
  if (p.pl[2][0] * y + p.pl[2][1] * z < -infl) return false;
  if (p.pl[3][0] * y + p.pl[3][1] * z < -infl) return false;
  return true;
}

// Image reads. COMPACT: the frame's depth is 16-bit millimetres and its labels 8-bit ids; the conversion hydra's
// parseInputPacket does on the host (float(u16) * scale, int32(u8)) happens per tap, so compact batches need no
// expansion pass and their taps touch 2 B / 1 B instead of 4 B.
template <bool COMPACT>
__device__ __forceinline__ float depthAt(const FrameView& f, int i) {
  if (COMPACT) return static_cast<float>(__ldg(&f.depth16[i])) * f.depth_scale;
  return __ldg(&f.depth[i]);
}
template <bool COMPACT>
__device__ __forceinline__ int labelAt(const FrameView& f, int i) {
  if (COMPACT) return static_cast<int>(__ldg(&f.label8[i]));
  return __ldg(&f.label[i]);
}

__device__ __forceinline__ float measurementWeight(const BatchParams& p, float depth, float sdf) {
  float w = (p.fx * p.fy) * (p.voxel_size * p.voxel_size) / (depth * depth);
  if (!p.constant_weight) w = w / (depth * depth);
  if (p.use_dropoff && sdf < -p.dropoff_eps) {
    w = w * ((p.trunc + sdf) / (p.trunc - p.dropoff_eps));
    w = fmaxf(w, 0.f);
  }
  return w;
}

// ProjectionInterpolator::interpolateColor (UP App. A.6 step 5; docs/ORACLE_SPEC.md §5.6): nearest -> the colour of
// pixel i; bilinear -> per channel ((w0 c0 + w1 c1) + w2 c2) + w3 c3 over the taps (u,v), (u,v+1), (u+1,v), (u+1,v+1)
// with pixel i = (u,v), truncated to u8.
__device__ __forceinline__ uchar3 measuredColor(const BatchParams& p, const FrameView& f, int i, bool bilinear, float w0,
                                                float w1, float w2, float w3) {
  const uint8_t* __restrict__ p0 = f.color + static_cast<size_t>(i) * 3;
  if (!bilinear) return make_uchar3(__ldg(p0), __ldg(p0 + 1), __ldg(p0 + 2));
  const uint8_t* __restrict__ p1 = p0 + static_cast<size_t>(p.W) * 3;
  uint8_t o[3];
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    const float s = ((w0 * static_cast<float>(__ldg(p0 + ch)) + w1 * static_cast<float>(__ldg(p1 + ch))) +
                     w2 * static_cast<float>(__ldg(p0 + 3 + ch))) + w3 * static_cast<float>(__ldg(p1 + 3 + ch));
    o[ch] = static_cast<uint8_t>(static_cast<int>(s));
  }
  return make_uchar3(o[0], o[1], o[2]);
}

// spark_dsg Color::merge as called by updateVoxel: c = u8(c * (1 - ratio) + c_m * ratio).
__device__ __forceinline__ uint8_t mergeChannel(uint8_t c, uint8_t cm, float ratio) {
  return static_cast<uint8_t>(static_cast<int>(static_cast<float>(c) * (1.f - ratio) + static_cast<float>(cm) * ratio));
}

__device__ __forceinline__ int warpSum(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---- input conversion: compact sensor formats -> the f32 / i32 images the fusion reads ------------------------
// hydra's parseInputPacket (call site khronos/src/active_window/active_window.cpp:275) converts 16UC1 depth in
// millimetres to 32FC1 metres and class ids to 32SC1 on the host; here the 3 B/pixel cross PCIe / NVLink and
// are expanded on the device: depth = float(u16) * scale (one fp32 multiply), label = int32(u8).
__global__ void __launch_bounds__(256) expandFramesKernel(const __grid_constant__ BatchParams p) {
  const FrameView& f = p.f[blockIdx.y];
  const int n = p.W * p.H;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (f.depth16) const_cast<float*>(f.depth)[i] = static_cast<float>(__ldg(&f.depth16[i])) * f.depth_scale;
    if (f.label8) const_cast<int*>(f.label)[i] = static_cast<int>(__ldg(&f.label8[i]));
  }
}

__global__ void expandDepthKernel(const uint16_t* __restrict__ src, float scale, float* __restrict__ dst, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = static_cast<float>(src[i]) * scale;
}

// ---- per-frame tile maxima of the depth image (input of the conservative culling) ---------------------
// A max-pyramid with 8/16/32/64-pixel tiles: a culling query reads the level at which its footprint spans
// only a handful of tiles. Levels 0 and 1 come from this kernel, the coarser ones from tilePyramidKernel.
// One warp reduces a 16-row x 32-column strip: coalesced row reads, vertical max in registers,
// horizontal max over 8-/16-lane groups by shuffles -> eight 8x8 and two 16x16 maxima per warp.
__global__ void __launch_bounds__(256) tileMaxKernel(const __grid_constant__ BatchParams p) {
  const int b = blockIdx.y;
  const int warps_x = (p.W + 31) / 32;
  const int warp = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (warp >= warps_x * p.lvl_ty[1]) return;
  const int ty16 = warp / warps_x, wx = warp % warps_x;
  const int u = wx * 32 + lane;
  const FrameView& f = p.f[b];
  float d[2] = {0.f, 0.f};
#pragma unroll
  for (int r = 0; r < 16; ++r) {
    const int v = ty16 * 16 + r;
    if (u < p.W && v < p.H)
      d[r >> 3] = fmaxf(d[r >> 3], p.compact_taps ? depthAt<true>(f, v * p.W + u) : depthAt<false>(f, v * p.W + u));
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    d[h] = fmaxf(d[h], __shfl_xor_sync(0xffffffffu, d[h], 1));
    d[h] = fmaxf(d[h], __shfl_xor_sync(0xffffffffu, d[h], 2));
    d[h] = fmaxf(d[h], __shfl_xor_sync(0xffffffffu, d[h], 4));
    const int tx = wx * 4 + (lane >> 3), ty = ty16 * 2 + h;
    if ((lane & 7) == 0 && tx < p.lvl_tx[0] && ty < p.lvl_ty[0]) p.f[b].tiles[p.lvl_off[0] + ty * p.lvl_tx[0] + tx] = d[h];
  }
  float m16 = fmaxf(d[0], d[1]);
  m16 = fmaxf(m16, __shfl_xor_sync(0xffffffffu, m16, 8));
  const int tx16 = wx * 2 + (lane >> 4);
  if ((lane & 15) == 0 && tx16 < p.lvl_tx[1]) p.f[b].tiles[p.lvl_off[1] + ty16 * p.lvl_tx[1] + tx16] = m16;
}

// Vectorised variant for f32 depth images whose rows are 16-byte aligned (W % 4 == 0, 16-byte aligned base): one warp
// reduces a 16-row x 128-column strip, each lane streaming a 4-pixel column group with 16 independent 16-byte loads
// (8 KB in flight per warp; the round-1 kernel moved 39 MB per batch at 1.3 TB/s, a fifth of HBM speed, and sits on the
// critical path of every rank of a sharded replay). 8x8 tile = 2 lanes x 8 rows, 16x16 tile = 4 lanes x 16 rows.
__global__ void __launch_bounds__(256) tileMaxVec4Kernel(const __grid_constant__ BatchParams p) {
  const int b = blockIdx.y;
  const int strips_x = (p.W + 127) / 128;
  const int warp = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (warp >= strips_x * p.lvl_ty[1]) return;
  const int ty16 = warp / strips_x, sx = warp % strips_x;
  const int u = sx * 128 + lane * 4;
  const FrameView& f = p.f[b];
  float d[2] = {0.f, 0.f};
  if (u < p.W) {
    const float4* __restrict__ base = reinterpret_cast<const float4*>(f.depth + u);
    const int w4 = p.W >> 2;
    float4 v[16];
#pragma unroll
    for (int r = 0; r < 16; ++r) {
      const int row = ty16 * 16 + r;
      v[r] = row < p.H ? __ldcs(base + static_cast<size_t>(row) * w4) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int r = 0; r < 16; ++r) d[r >> 3] = fmaxf(d[r >> 3], fmaxf(fmaxf(v[r].x, v[r].y), fmaxf(v[r].z, v[r].w)));
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    d[h] = fmaxf(d[h], __shfl_xor_sync(0xffffffffu, d[h], 1));
    const int tx = sx * 16 + (lane >> 1), ty = ty16 * 2 + h;
    if ((lane & 1) == 0 && tx < p.lvl_tx[0] && ty < p.lvl_ty[0]) p.f[b].tiles[p.lvl_off[0] + ty * p.lvl_tx[0] + tx] = d[h];
  }
  float m16 = fmaxf(d[0], d[1]);
  m16 = fmaxf(m16, __shfl_xor_sync(0xffffffffu, m16, 2));
  const int tx16 = sx * 8 + (lane >> 2);
  if ((lane & 3) == 0 && tx16 < p.lvl_tx[1]) p.f[b].tiles[p.lvl_off[1] + ty16 * p.lvl_tx[1] + tx16] = m16;
}

// Coarser pyramid levels (32 and 64 pixel tiles) from the 16-pixel level: one CTA per frame.
__global__ void __launch_bounds__(256) tilePyramidKernel(const __grid_constant__ BatchParams p) {
  float* __restrict__ t = p.f[blockIdx.x].tiles;
  for (int l = 2; l < kTileLevels; ++l) {
    const int n = p.lvl_tx[l] * p.lvl_ty[l];
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const int tx = i % p.lvl_tx[l], ty = i / p.lvl_tx[l];
      float d = 0.f;
#pragma unroll
      for (int j = 0; j < 2; ++j)
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          const int x = tx * 2 + k, y = ty * 2 + j;
          if (x < p.lvl_tx[l - 1] && y < p.lvl_ty[l - 1]) d = fmaxf(d, t[p.lvl_off[l - 1] + y * p.lvl_tx[l - 1] + x]);
        }
      t[p.lvl_off[l] + i] = d;
    }
    __syncthreads();
  }
}

// Conservative culling rule for an axis-aligned box of voxel centres [lo, hi] (world frame) against frame
// f: a (box, frame) pair is skipped only if NO voxel centre inside the box can receive a valid measurement,
// so skipping cannot change any result (SURVEY §7 hard part 4): the box projects entirely outside the
// image, or every depth pixel its voxels could tap is invalid, or every voxel lies more than the truncation
// distance behind the farthest of those depths (sdf < -trunc). Margins (1 mm, 2 px) are far above the fp32
// rounding of the per-voxel arithmetic.

// ---- culling helpers (lane-serial) ----------------------------------------------------------------------------
// Box of voxel centres of work item `it` of a block (4x8x4 voxels; x fastest).
template <int VPS>
__device__ __forceinline__ void itemOrigin(int it, int& x0, int& y0, int& z0) {
  constexpr int IX = VPS / 4, IY = VPS / 8;
  x0 = (it % IX) * 4;
  y0 = ((it / IX) % IY) * 8;
  z0 = (it / (IX * IY)) * 4;
}

// One lane tests one box: 8 corner projections, then the tile-maximum rectangle they span.
__device__ __forceinline__ bool boxCulledPose(const BatchParams& p, const float* R, const float* t, const float* __restrict__ frame_tiles,
                                              float lox, float loy, float loz, float hix, float hiy, float hiz) {
  float zmin = 3.0e38f, umin = 3.0e38f, umax = -3.0e38f, vmin = 3.0e38f, vmax = -3.0e38f;
#pragma unroll 1
  for (int c = 0; c < 8; ++c) {
    float x, y, z;
    xform(R, t, (c & 1) ? hix : lox, (c & 2) ? hiy : loy, (c & 4) ? hiz : loz, x, y, z);
    if (z < 1e-2f) return false;  // reaches behind / near the camera plane: keep
    const float u = p.fx * x / z + p.cx, v = p.fy * y / z + p.cy;
    zmin = fminf(zmin, z);
    umin = fminf(umin, u); umax = fmaxf(umax, u);
    vmin = fminf(vmin, v); vmax = fmaxf(vmax, v);
  }
  if (umax < -0.5f || vmax < -0.5f || umin > static_cast<float>(p.W - 1) + 0.5f || vmin > static_cast<float>(p.H - 1) + 0.5f)
    return true;
  const int u0 = max(static_cast<int>(floorf(umin)) - 2, 0), u1 = min(static_cast<int>(floorf(umax)) + 3, p.W - 1);
  const int v0 = max(static_cast<int>(floorf(vmin)) - 2, 0), v1 = min(static_cast<int>(floorf(vmax)) + 3, p.H - 1);
  // pyramid level: the footprint spans at most ~9 x 9 tiles (coarser tiles only loosen the bound)
  int l = 0;
  while (l < kTileLevels - 1 && max(u1 - u0, v1 - v0) > (64 << l)) ++l;
  const int sh = 3 + l;
  const int tx0 = u0 >> sh, tx1 = u1 >> sh, ty0 = v0 >> sh, ty1 = v1 >> sh;
  const float* __restrict__ tiles = frame_tiles + p.lvl_off[l];
  const int tiles_x = p.lvl_tx[l];
  float dmax = 0.f;
  for (int ty = ty0; ty <= ty1; ++ty) {
    const float* __restrict__ row = tiles + ty * tiles_x;
#pragma unroll 4
    for (int tx = tx0; tx <= tx1; ++tx) dmax = fmaxf(dmax, __ldg(&row[tx]));
  }
  if (!(dmax > 0.f)) return true;
  return zmin - p.trunc - 1e-3f > dmax;
}
__device__ __forceinline__ bool boxCulledLane(const BatchParams& p, const FrameView& f, float lox, float loy, float loz,
                                              float hix, float hiy, float hiz) {
  return boxCulledPose(p, f.R, f.t, f.tiles, lox, loy, loz, hix, hiy, hiz);
}

// ---- K0: block selection for a batch of frames ---------------------------------------------------------
// One WARP per candidate block of the batch's AABB (allocate mode; hydra findBlocksInViewFrustum,
// SURVEY App. A.5) or per pool slot (allocate == 0: all allocated blocks, mesh_object_extractor.cpp:242).
// Lane b evaluates frame b of the batch: frustum test -> ballot -> 32-bit frame mask.
// PIPE (KB_PIPELINE): the host zeroes this batch's own counters on the prologue stream; the other batch's counters may
// be in use by its fuse kernel, so K0 must not touch them.
template <bool PIPE>
__global__ void __launch_bounds__(128) selectBlocksKernel(const DeviceMap m, const __grid_constant__ BatchParams p) {
  const int c0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  // lane = frame: every lane needs ITS frame's pose. Indexing the parameter block with the lane id serialises the constant
  // cache 32 ways per load (r2 capture: 6 % issue utilisation, stalls 46 % short scoreboard + 36 % MIO throttle, 40 us for
  // 1.3 M instructions); a structure-of-arrays copy in shared memory is conflict free.
  __shared__ float s_pose[12][kMaxBatch];
  __shared__ const float* s_tiles[kMaxBatch];
  for (int i = threadIdx.x; i < 12 * kMaxBatch; i += blockDim.x) {
    const int b = i % kMaxBatch, k = i / kMaxBatch;
    s_pose[k][b] = b < p.n_frames ? (k < 9 ? p.f[b].R[k] : p.f[b].t[k - 9]) : 0.f;
  }
  if (threadIdx.x < kMaxBatch) s_tiles[threadIdx.x] = threadIdx.x < p.n_frames ? p.f[threadIdx.x].tiles : nullptr;
  __syncthreads();
  float Rl[9], tl[3];
#pragma unroll
  for (int k = 0; k < 9; ++k) Rl[k] = s_pose[k][lane];
#pragma unroll
  for (int k = 0; k < 3; ++k) tl[k] = s_pose[9 + k][lane];
  if (!PIPE && c0 == 0 && lane == 0) {  // reset the next batch's work counter and this batch's fetch cursor
    m.counters[kCtrWork0 + (p.parity ^ 1)] = 0;
    m.counters[kCtrFetch] = 0;
  }
  int slot = -1, bx = 0, by = 0, bz = 0;
  uint32_t mask = 0;
  int created = 0;
  if (p.allocate) {
    if (c0 >= p.dims[0] * p.dims[1] * p.dims[2]) return;
    int c = c0;
    bx = p.lo[0] + c % p.dims[0];
    c /= p.dims[0];
    by = p.lo[1] + c % p.dims[1];
    bz = p.lo[2] + c / p.dims[1];
    const float cx = (static_cast<float>(bx) + 0.5f) * p.block_size;
    const float cy = (static_cast<float>(by) + 0.5f) * p.block_size;
    const float cz = (static_cast<float>(bz) + 0.5f) * p.block_size;
    // shard filter first: at N ranks (N-1)/N of the candidate warps retire here
    if (p.nranks > 1 && mapOwner(m, bx, by, bz, p.nranks) != p.rank) return;
    bool in = false;
    if (lane < p.n_frames) {
      float x, y, z;
      xform(Rl, tl, cx, cy, cz, x, y, z);
      in = inFrustum(p, x, y, z);
    }
    mask = __ballot_sync(0xffffffffu, in);
    if (!mask) return;
    if (lane == 0) slot = hashFindOrInsert(m, bx, by, bz, p.f[__ffs(mask) - 1].frame_idx, &created);
    slot = __shfl_sync(0xffffffffu, slot, 0);
    if (slot < 0) return;
  } else {
    if (c0 >= p.n_slots || !(m.block_flags[c0] & kFlagAllocated)) return;
    slot = c0;
    const int3 bi = m.block_index[slot];
    bx = bi.x; by = bi.y; bz = bi.z;
    mask = p.n_frames >= 32 ? 0xffffffffu : ((1u << p.n_frames) - 1u);
  }
  if (lane == 0) {
    atomicAdd(&m.counters[kCtrFrustum], __popc(mask));
    atomicAdd(&totals64(m.counters)[kTotFrustum], static_cast<unsigned long long>(__popc(mask)));
    if (created) {
      atomicAdd(&m.counters[kCtrAllocated], 1);
      atomicAdd(&totals64(m.counters)[kTotAllocated], 1ull);
    }
  }
  if (p.cull) {
    // block-level culling, lane = frame: each lane tests the whole block against its own frame
    const float ox = static_cast<float>(bx) * p.block_size, oy = static_cast<float>(by) * p.block_size,
                oz = static_cast<float>(bz) * p.block_size;
    const float lo = 0.5f * p.voxel_size, hi = p.block_size - 0.5f * p.voxel_size;
    bool keep = false;
    if ((mask >> lane) & 1u)
      keep = !boxCulledPose(p, Rl, tl, s_tiles[lane], ox + lo, oy + lo, oz + lo, ox + hi, oy + hi, oz + hi);
    mask = __ballot_sync(0xffffffffu, keep);
    if (!mask) return;
  }
  int i = 0;
  if (lane == 0) {
    // Blocks that may receive measurements get their semantic slot here (one thread per block, so no
    // allocation race inside the fuse kernel); never-measured blocks cost no semantic memory.
    if (p.L > 0 && m.block_sem[slot] < 0) {
      m.block_sem[slot] = allocSlot(m.counters, kCtrSemHwm, kCtrSemFreeCount, m.sem_free_list, m.max_sem);
    }
    atomicAdd(&m.counters[kCtrPairs], __popc(mask));
    atomicAdd(&totals64(m.counters)[kTotPairs], static_cast<unsigned long long>(__popc(mask)));
    i = atomicAdd(&m.counters[kCtrWork0 + p.parity], 1);
    if (i < p.max_work) {
      p.work_slots[i] = slot;
      p.work_masks[i] = mask;
      p.work_upd[i] = 0;
    } else {
      atomicExch(&m.counters[kCtrCapacityExceeded], 1);
    }
  }
  i = __shfl_sync(0xffffffffu, i, 0);
  // per-item frame masks: all of the block's frames without culling, else filled by itemCullKernel
  if (i < p.max_work && lane < p.items_per_block) p.item_fmask[static_cast<size_t>(i) * p.items_per_block + lane] = p.cull ? 0u : mask;
}

// ---- K0b: work-item culling --------------------------------------------------------------------------------
// One warp per (work block, chunk of kCullChunk frames); lane = work item of the block. Fills
// item_fmask[block][item] with the frames for which the item may receive a measurement.
constexpr int kCullChunk = 1;
template <int VPS>
__global__ void __launch_bounds__(128) itemCullKernel(const DeviceMap m, const __grid_constant__ BatchParams p) {
  constexpr int ITEMS = (VPS / 4) * (VPS / 8) * (VPS / 4);
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int n_warps = (gridDim.x * blockDim.x) >> 5;
  const int chunks = (p.n_frames + kCullChunk - 1) / kCullChunk;
  const int n = min(m.counters[kCtrWork0 + p.parity], p.max_work) * chunks;
  for (int w = warp; w < n; w += n_warps) {
    const int wi = w / chunks, ch = w % chunks;
    const uint32_t bmask = p.work_masks[wi] & (((kCullChunk >= 32 ? 0u : (1u << kCullChunk)) - 1u) << (ch * kCullChunk));
    if (!bmask || lane >= ITEMS) continue;
    const int3 bi = m.block_index[p.work_slots[wi]];
    int x0, y0, z0;
    itemOrigin<VPS>(lane, x0, y0, z0);
    const float ox = static_cast<float>(bi.x) * p.block_size, oy = static_cast<float>(bi.y) * p.block_size,
                oz = static_cast<float>(bi.z) * p.block_size;
    const float lx = ox + (static_cast<float>(x0) + 0.5f) * p.voxel_size, hx = ox + (static_cast<float>(x0 + 3) + 0.5f) * p.voxel_size;
    const float ly = oy + (static_cast<float>(y0) + 0.5f) * p.voxel_size, hy = oy + (static_cast<float>(y0 + 7) + 0.5f) * p.voxel_size;
    const float lz = oz + (static_cast<float>(z0) + 0.5f) * p.voxel_size, hz = oz + (static_cast<float>(z0 + 3) + 0.5f) * p.voxel_size;
    uint32_t keep = 0, rem = bmask;
    while (rem) {
      const int b = __ffs(rem) - 1;
      rem &= rem - 1;
      if (!boxCulledLane(p, p.f[b], lx, ly, lz, hx, hy, hz)) keep |= 1u << b;
    }
    if (keep) atomicOr(&p.item_fmask[static_cast<size_t>(wi) * ITEMS + lane], keep);
  }
}

// ---- K0c (optional, KB_FUSE_ITEM_LIST): compaction of the non-empty culling boxes, heaviest first ----------------
// The fuse kernel's warps fetch items from a shared cursor; with ~4 items per warp and item costs between 1 and 32
// frame iterations, the order matters (longest-processing-time first shortens the tail) and every empty box costs a
// cursor round trip. This pass lists the boxes whose frame mask is non-zero in three weight classes.
template <int VPS, bool PB>
__global__ void __launch_bounds__(256) itemCompactKernel(const DeviceMap m, const __grid_constant__ BatchParams p) {
  constexpr int kItems = PB ? kCtrItemsB0 : kCtrItems0;  // PB: second counter set (odd pipelined batches)
  constexpr int BOXES = (VPS / 4) * (VPS / 8) * (VPS / 4);
  const int n = min(m.counters[kCtrWork0 + p.parity], p.max_work) * BOXES;
  const int lane = threadIdx.x & 31;
  for (int base = (blockIdx.x * blockDim.x + threadIdx.x) - lane; base < n; base += gridDim.x * blockDim.x) {
    const int i = base + lane;
    const uint32_t fm = i < n ? p.item_fmask[i] : 0u;
    const int cls = fm ? (32 - __popc(fm)) >> 2 : -1;  // 0: 32..29 frames, ..., 7: 4..1 frames
    // lanes of the same class aggregate their append into one atomic
    const unsigned peers = __match_any_sync(0xffffffffu, cls);
    if (cls < 0) continue;
    const int leader = __ffs(peers) - 1;
    int start = 0;
    if (lane == leader) start = atomicAdd(&m.counters[kItems + cls], __popc(peers));
    start = __shfl_sync(peers, start, leader);
    const int idx = start + __popc(peers & ((1u << lane) - 1u));
    if (idx < p.item_list_cap) p.item_list[static_cast<size_t>(cls) * p.item_list_cap + idx] = i;
  }
}

// Item j of the concatenated class lists -> box index.
template <bool PB>
__device__ __forceinline__ int listedBox(const BatchParams& p, const int (&n_cls)[kItemClasses], int j) {
  int k = 0;
#pragma unroll
  for (int c = 0; c < kItemClasses - 1; ++c) {
    if (k == c && j >= n_cls[c]) { j -= n_cls[c]; k = c + 1; }
  }
  return p.item_list[static_cast<size_t>(k) * p.item_list_cap + j];
}

// ---- K1: the per-voxel steps of the fuse kernels ---------------------------------------------------------------
// fuseKernel, fuseKernelCoop and fuseKernelMlp are built from the same steps and differ only in how they order them over an
// item's frames: the measurement of a voxel in a frame (projectQuad -> resolveQuad -> labelTap -> measurementWeight) and
// its fold into the voxel state (VoxelState, LikelihoodRow), then the item's and the warp's bookkeeping.
// ProjectiveIntegrator::updateBlock / getVoxelMeasurement / computeLabel / updateVoxel (UP App. A.6; computeLabel structure
// pinned by khronos/src/active_window/integration/object_integrator.cpp:58-81); SemanticIntegrator::updateLikelihoods
// (UP App. A.8).
constexpr int kBoxLayers = 4;  // z-layers per 4x8x4 culling box
template <int VPS>
constexpr int kBoxes = (VPS / 4) * (VPS / 8) * (VPS / kBoxLayers);  // 32 (16^3) or 4 (8^3) boxes of 128 voxels

// Items of the batch, an item being one of the IPB layer groups of a box. LIST: the boxes of itemCompactKernel's class
// lists (n_cls: the class sizes, for listedBox); else every box of every work block.
template <int VPS, int IPB, bool LIST, bool PB>
__device__ __forceinline__ int fuseItemCount(const DeviceMap& m, const BatchParams& p, int (&n_cls)[kItemClasses]) {
  if constexpr (LIST) {
    constexpr int kItems = PB ? kCtrItemsB0 : kCtrItems0;
    int n = 0;
#pragma unroll
    for (int c = 0; c < kItemClasses; ++c) {
      n_cls[c] = min(m.counters[kItems + c], p.item_list_cap);
      n += n_cls[c];
    }
    return n * IPB;
  } else {
    return min(m.counters[kCtrWork0 + p.parity], p.max_work) * kBoxes<VPS> * IPB;
  }
}

// The voxel of `lane` in layer k of box `it` of the block in pool slot `slot` (block index bi): its index in the block, its
// index in the pool and its centre in world coordinates.
struct VoxelSite {
  int lin;
  size_t gi;
  float x, y, z;
};
template <int VPS>
__device__ __forceinline__ VoxelSite voxelSite(const BatchParams& p, int slot, int3 bi, int it, int k, int lane) {
  int x0, y0, z0;
  itemOrigin<VPS>(it, x0, y0, z0);
  const int vx = x0 + (lane & 3), vy = y0 + (lane >> 2), vz = z0 + k;
  VoxelSite s;
  s.lin = vx + VPS * (vy + VPS * vz);
  s.gi = static_cast<size_t>(slot) * (VPS * VPS * VPS) + s.lin;
  s.x = static_cast<float>(bi.x) * p.block_size + (static_cast<float>(vx) + 0.5f) * p.voxel_size;
  s.y = static_cast<float>(bi.y) * p.block_size + (static_cast<float>(vy) + 0.5f) * p.voxel_size;
  s.z = static_cast<float>(bi.z) * p.block_size + (static_cast<float>(vz) + 0.5f) * p.voxel_size;
  return s;
}

// Measurement, step 1: the voxel centre's projection and the four depth taps around it, loaded together at clamped
// addresses (on the last column / row the second column / row collapses onto the first). The nearest pixel,
// round(u) = floor(u) + (du >= 0.5) for u >= 0, is one of the four, so no interpolator needs a second, dependent depth load.
// False: the centre is behind the camera or projects outside the image.
struct DepthQuad {
  float z, du, dv;       // camera depth of the centre; its pixel position minus (u0, v0)
  int i0, su, sv;        // pixel (u0, v0) = (floor(u), floor(v)); offsets of the second column and row (0 on the last one)
  float r0, r1, r2, r3;  // depths at (u0, v0), (u0, v0 + 1), (u0 + 1, v0), (u0 + 1, v0 + 1)
};
template <bool COMPACT>
__device__ __forceinline__ bool projectQuad(const BatchParams& p, const FrameView& f, float wx, float wy, float wz, DepthQuad& q) {
  float x, y;
  xform(f.R, f.t, wx, wy, wz, x, y, q.z);
  if (q.z <= 0.f) return false;
  const float u = p.fx * x / q.z + p.cx;
  const float v = p.fy * y / q.z + p.cy;
  if (u < 0.f || u > static_cast<float>(p.W - 1) || v < 0.f || v > static_cast<float>(p.H - 1)) return false;
  const int u0 = static_cast<int>(floorf(u)), v0 = static_cast<int>(floorf(v));
  q.du = u - static_cast<float>(u0);
  q.dv = v - static_cast<float>(v0);
  q.i0 = v0 * p.W + u0;
  q.su = u0 + 1 < p.W ? 1 : 0;
  q.sv = v0 + 1 < p.H ? p.W : 0;
  q.r0 = depthAt<COMPACT>(f, q.i0);
  q.r2 = depthAt<COMPACT>(f, q.i0 + q.su);
  q.r1 = depthAt<COMPACT>(f, q.i0 + q.sv);
  q.r3 = depthAt<COMPACT>(f, q.i0 + q.sv + q.su);
  return true;
}

// Measurement, step 2: ProjectionInterpolator{Nearest,Bilinear,Adaptive}::computeWeights (UP, SURVEY App. A.7) on the quad,
// the sdf, and interpolateID's pixel: the dominant bilinear tap (ties -> the lowest tap index) or the nearest pixel.
// False: no valid range, or the voxel lies more than trunc behind it. (Older comments and test docstrings call this step
// computeTaps.)
struct Measurement {
  float sdf;
  bool in_band, bilinear;
  float w0, w1, w2, w3;  // bilinear weights of the taps in DepthQuad order
  int ti;                // label / mask pixel (meaningful in band)
  int ti_near;           // nearest pixel
};
__device__ __forceinline__ bool resolveQuad(const BatchParams& p, const DepthQuad& q, Measurement& ms) {
  const bool inside = q.su != 0 && q.sv != 0;
  const bool ru = q.du >= 0.5f, rv = q.dv >= 0.5f;
  const int ti_near = q.i0 + (ru ? 1 : 0) + (rv ? p.W : 0);  // du = 0 on the last column, dv = 0 on the last row
  ms.w0 = (1.f - q.du) * (1.f - q.dv);
  ms.w1 = (1.f - q.du) * q.dv;
  ms.w2 = q.du * (1.f - q.dv);
  ms.w3 = q.du * q.dv;
  ms.bilinear = false;
  if (p.interp != KB_INTERP_NEAREST) {
    if (inside) {
      const bool all_valid = q.r0 > 0.f && q.r1 > 0.f && q.r2 > 0.f && q.r3 > 0.f;
      if (p.interp == KB_INTERP_ADAPTIVE) {
        const float mx = fmaxf(fmaxf(q.r0, q.r1), fmaxf(q.r2, q.r3));
        const float mn = fminf(fminf(q.r0, q.r1), fminf(q.r2, q.r3));
        ms.bilinear = all_valid && mx - mn < p.adaptive_thr;
      } else {
        if (!all_valid) return false;  // bilinear: invalid
        ms.bilinear = true;
      }
    } else if (p.interp != KB_INTERP_ADAPTIVE) {
      return false;
    }
  }
  float range;
  if (ms.bilinear) {
    range = ((ms.w0 * q.r0 + ms.w1 * q.r1) + ms.w2 * q.r2) + ms.w3 * q.r3;
  } else {
    range = ru ? (rv ? q.r3 : q.r2) : (rv ? q.r1 : q.r0);
    if (!(range > 0.f)) return false;
  }
  ms.sdf = range - q.z;
  if (ms.sdf < -p.trunc) return false;
  ms.in_band = fabsf(ms.sdf) < p.trunc;
  ms.ti_near = ti_near;
  ms.ti = ti_near;
  if (ms.in_band && ms.bilinear) {
    int best = 0;
    float bw = ms.w0;
    if (ms.w1 > bw) { best = 1; bw = ms.w1; }
    if (ms.w2 > bw) { best = 2; bw = ms.w2; }
    if (ms.w3 > bw) { best = 3; }
    ms.ti = q.i0 + (best >> 1) + ((best & 1) ? p.W : 0);
  }
  return true;
}

// Whether frame b has the label image the semantic mode reads (the object image in BINARY mode).
__device__ __forceinline__ bool hasLabelImage(const BatchParams& p, int b) { return (p.label_frames >> b) & 1u; }

// Measurement, step 3, in band only: the dynamic mask and the label at pixel ti. label: the class id (BINARY: 1 on the target
// object, else 0), 0 when the frame has no label image. False: the measurement is dropped (masked, or a blocked label).
template <bool COMPACT>
__device__ __forceinline__ bool labelTap(const BatchParams& p, const FrameView& f, int b, int ti, uint32_t& label) {
  if (((p.mask_frames >> b) & 1u) && __ldg(&f.mask[ti]) != 0) return false;
  if (hasLabelImage(p, b)) {
    if (p.sem_mode == KB_SEMANTICS_BINARY) {
      label = __ldg(&f.object_image[ti]) == f.target_id ? 1u : 0u;
    } else {
      label = static_cast<uint32_t>(labelAt<COMPACT>(f, ti));
      if (label < static_cast<uint32_t>(KB_MAX_LABELS) && ((p.blocked_mask >> label) & 1ull)) return false;
    }
  }
  return true;
}

// Lazy tracking fold (see evalTracking): what the tracking passes since the voxel's last write would have
// done to it. Returns the flag byte to carry (ever_free, active, to_remove); refreshes last_occupied.
// Out of line so that the fuse kernel's item loop keeps its register budget. The arguments are references into the
// calling kernel's __grid_constant__ parameters: passed by value, the DeviceMap (~200 B) and TrackEval would be copied to
// the stack at every call, i.e. once per voxel and batch.
__device__ __noinline__ uint32_t trackingFold(const DeviceMap& m, const TrackEval& t, uint32_t born, size_t gi) {
  const uint8_t fl = m.vflags[gi];
  const uint32_t c_stored = m.last_occ[gi];
  uint32_t c_true;
  bool act, rem;
  evalTracking(m, t, born, m.last_obs[gi], c_stored, fl, &c_true, &act, &rem);
  if (c_true != c_stored) m.last_occ[gi] = c_true;
  return (fl & kVoxEverFree) | (act ? kVoxActive : 0) | (rem ? kVoxToRemove : 0);
}

// The voxel's {distance, weight, last_observed, flags} (and colour) in registers while its frames are folded in, in frame
// order: read at the first valid measurement, written back once. COLOR: TsdfVoxel::color is carried too.
template <bool COLOR>
struct VoxelState {
  float2 st = make_float2(0.f, 0.f);
  uint32_t lobs = 0, vfl = 0, upd_frames = 0;  // last observing frame, carried tracking flags, frames b that updated it
  bool have = false;
  uchar4 col = make_uchar4(0, 0, 0, 0);
  bool col_dirty = false;

  // updateVoxel's TSDF recurrence for frame b; returns the weight before it (the colour merge's denominator).
  __device__ __forceinline__ float integrate(const DeviceMap& m, const BatchParams& p, int slot, size_t gi, const FrameView& f,
                                             int b, float sdf, float wm) {
    if (!have) {
      st = m.tsdf[gi];
      have = true;
      if (p.with_tracking) vfl = trackingFold(m, p.trk, m.born_frame[slot], gi);
      if constexpr (COLOR) col = m.color[gi];
    }
    const float sdf_c = fminf(fmaxf(sdf, -p.trunc), p.trunc);
    const float2 old = st;
    st.x = (old.x * old.y + sdf_c * wm) / (old.y + wm);
    st.y = fminf(old.y + wm, p.max_weight);
    lobs = f.frame_idx;
    upd_frames |= 1u << b;
    return old.y;
  }
  // updateVoxel: colour is merged near the surface only, from frames that carry a colour image.
  __device__ __forceinline__ void mergeColor(const BatchParams& p, const FrameView& f, const DepthQuad& q, const Measurement& ms,
                                             float wm, float w_old) {
    if (f.color == nullptr) return;
    const uchar3 cm = measuredColor(p, f, ms.bilinear ? q.i0 : ms.ti_near, ms.bilinear, ms.w0, ms.w1, ms.w2, ms.w3);
    const float tot = w_old + wm;
    const float ratio = tot > 0.f ? wm / tot : 0.f;
    col.x = mergeChannel(col.x, cm.x, ratio);
    col.y = mergeChannel(col.y, cm.y, ratio);
    col.z = mergeChannel(col.z, cm.z, ratio);
    col_dirty = true;
  }
  __device__ __forceinline__ void store(const DeviceMap& m, const BatchParams& p, size_t gi) const {
    m.tsdf[gi] = st;
    if constexpr (COLOR) {
      if (col_dirty) m.color[gi] = col;
    }
    if (p.with_tracking) {
      m.last_obs[gi] = lobs;
      m.vflags[gi] = static_cast<uint8_t>(vfl | (st.x < p.occ_thr ? 0 : kVoxNotOccupied));
    }
  }
};

// The voxel's semantic likelihood row, on chip in dynamic shared memory while its frames are folded in: MLE rows as
// [thread][fuseRowStride(Lp)] (moved with conflict-free 16 B accesses), BINARY counts as [2][T]. T: the threads that share
// the row array (kFuseThreads, or the 32 lanes of fuseKernelCoop's folding warp); V: voxels per block.
template <int T, int V>
struct LikelihoodRow {
  bool resident = false;
  int best_label = 0;

  // likelihoods += logM[:, label] (BINARY: count[label] += 1); the first call brings the row on chip, or starts it.
  __device__ __forceinline__ void add(const DeviceMap& m, const BatchParams& p, float4* s_rows4, int sem, int lin, uint32_t label) {
    const bool binary = p.sem_mode == KB_SEMANTICS_BINARY;
    float* const s_rows = reinterpret_cast<float*>(s_rows4);
    if (!resident) {
      resident = true;
      const size_t si = static_cast<size_t>(sem) * V + lin;
      const bool empty = m.sem_label[si] == kSemEmpty;
      if (binary) {
        const float2 c = empty ? make_float2(0.f, 0.f) : *reinterpret_cast<const float2*>(m.sem_lik + si * 2);
        s_rows[threadIdx.x] = c.x;
        s_rows[T + threadIdx.x] = c.y;
      } else {
        const float4* __restrict__ lk = reinterpret_cast<const float4*>(m.sem_lik + si * m.Lp);
        float4* const row = s_rows4 + threadIdx.x * (fuseRowStride(m.Lp) >> 2);
        const float4 init = make_float4(p.mle_init, p.mle_init, p.mle_init, p.mle_init);
#pragma unroll
        for (int q = 0; q < KB_MAX_LABELS / 4; ++q) {
          if (4 * q >= m.Lp) break;
          row[q] = empty ? init : lk[q];
        }
      }
    }
    if (binary) {
      const float c = s_rows[label * T + threadIdx.x] + 1.f;
      s_rows[label * T + threadIdx.x] = c;
      best_label = s_rows[T + threadIdx.x] > s_rows[threadIdx.x] ? 1 : 0;
    } else {
      // mle_off on every entry but the label's, which gets mle_diag. Every entry still receives exactly one addition per
      // frame: the label entry is read first, the whole row (padding included, which nobody reads) takes mle_off in 16 B
      // steps, then the label entry is overwritten with old + mle_diag. The arg max is taken once, in store: only its final
      // value is ever stored, and it only depends on the final row.
      float* const row = s_rows + threadIdx.x * fuseRowStride(m.Lp);
      float4* const row4 = reinterpret_cast<float4*>(row);
      const float c_label = row[label];
      const float off = p.mle_off;
#pragma unroll
      for (int q = 0; q < KB_MAX_LABELS / 4; ++q) {
        if (4 * q >= m.Lp) break;
        float4 c = row4[q];
        c.x += off;
        c.y += off;
        c.z += off;
        c.w += off;
        row4[q] = c;
      }
      row[label] = c_label + p.mle_diag;
    }
  }
  // Writes the row back with SemanticVoxel::semantic_label, the first maximum of the final likelihoods over 0..L-1
  // (UP App. A.8), taken from the values being written.
  __device__ __forceinline__ void store(const DeviceMap& m, const BatchParams& p, const float4* s_rows4, int sem, int lin) {
    if (!resident) return;
    const size_t si = static_cast<size_t>(sem) * V + lin;
    if (p.sem_mode == KB_SEMANTICS_BINARY) {
      const float* const s_rows = reinterpret_cast<const float*>(s_rows4);
      *reinterpret_cast<float2*>(m.sem_lik + si * 2) = make_float2(s_rows[threadIdx.x], s_rows[T + threadIdx.x]);
    } else {
      float4* __restrict__ lk = reinterpret_cast<float4*>(m.sem_lik + si * m.Lp);
      const float4* const row = s_rows4 + threadIdx.x * (fuseRowStride(m.Lp) >> 2);
      const int L = p.L;
      float bestv = 0.f;
      best_label = 0;
#pragma unroll
      for (int q = 0; q < KB_MAX_LABELS / 4; ++q) {
        if (4 * q >= m.Lp) break;
        const float4 c = row[q];
        lk[q] = c;
        if (q == 0) bestv = c.x;
        else if (4 * q < L && c.x > bestv) { bestv = c.x; best_label = 4 * q; }
        if (4 * q + 1 < L && c.y > bestv) { bestv = c.y; best_label = 4 * q + 1; }
        if (4 * q + 2 < L && c.z > bestv) { bestv = c.z; best_label = 4 * q + 2; }
        if (4 * q + 3 < L && c.w > bestv) { bestv = c.w; best_label = 4 * q + 3; }
      }
    }
    m.sem_label[si] = static_cast<uint16_t>(best_label);
  }
};

// Once per item, by its warp: block flags and the per-(block, frame) update bookkeeping. blocks_updated counts (block,
// frame) pairs once even though many items report them.
__device__ __forceinline__ void itemUpdated(const DeviceMap& m, const BatchParams& p, int slot, int wi, bool any_have,
                                            uint32_t upd_frames) {
  if (!__any_sync(0xffffffffu, any_have)) return;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) upd_frames |= __shfl_xor_sync(0xffffffffu, upd_frames, o);
  if ((threadIdx.x & 31) == 0) {
    const uint32_t all = KB_FLAG_UPDATED | KB_FLAG_MESH_UPDATED | KB_FLAG_ESDF_UPDATED | KB_FLAG_TRACKING_UPDATED;
    if ((m.block_flags[slot] & all) != all) atomicOr(&m.block_flags[slot], all);
    if ((p.work_upd[wi] & upd_frames) != upd_frames) {
      const uint32_t prev = atomicOr(&p.work_upd[wi], upd_frames);
      const int fresh = __popc(upd_frames & ~prev);
      if (fresh) {
        atomicAdd(&m.counters[kCtrBlocksUpdated], fresh);
        atomicAdd(&totals64(m.counters)[kTotBlocksUpdated], static_cast<unsigned long long>(fresh));
      }
    }
  }
}

// The warp's voxel counters, one atomic set per warp for the whole launch (32-bit per-call and 64-bit total counters).
__device__ __forceinline__ void flushFuseCounters(const DeviceMap& m, int n_valid, int n_band, int n_sem) {
  n_valid = warpSum(n_valid);
  if (!n_valid) return;
  n_band = warpSum(n_band);
  n_sem = warpSum(n_sem);
  if ((threadIdx.x & 31) == 0) {
    unsigned long long* t64 = totals64(m.counters);
    atomicAdd(&m.counters[kCtrVoxelsUpdated], n_valid);
    atomicAdd(&t64[kTotVoxelsUpdated], static_cast<unsigned long long>(n_valid));
    if (n_band) {
      atomicAdd(&m.counters[kCtrVoxelsBand], n_band);
      atomicAdd(&t64[kTotVoxelsBand], static_cast<unsigned long long>(n_band));
    }
    if (n_sem) {
      atomicAdd(&m.counters[kCtrVoxelsSemantic], n_sem);
      atomicAdd(&t64[kTotVoxelsSemantic], static_cast<unsigned long long>(n_sem));
    }
  }
}

// ---- K1: projective TSDF + semantic fusion ----------------------------------------------------------------
// Persistent warps fetch work items from a shared cursor. An item = one z-layer (4x8 voxels, one per lane) of
// a 4x8x4 box that survived culling, together with the box's frame mask. The lane keeps its voxel's state in registers
// (VoxelState) and its semantic likelihood row in shared memory (LikelihoodRow) while the warp walks the surviving frames
// in order: TSDF and likelihoods are read and written once per batch, every warp access covers whole 32 B sectors, and the
// serial dependency chain per item is one voxel deep, so ~25 k items per batch balance over the SMs.
// Warps never synchronise with each other.
// COLOR: some frame of the batch carries a colour image; band voxels blend it into TsdfVoxel::color (kept in a
// register like the rest of the voxel state: one 4 B read + write per batch). The colour-less instantiations
// are the ones the BASELINE workloads run and are unchanged by this parameter.
// LIST: items come from the compacted, heaviest-first box lists of itemCompactKernel instead of the dense box range.
// PB: the batch uses the second cursor / item-list counter set (odd batches of KB_PIPELINE).
template <int VPS, int LPI, bool COMPACT, bool COLOR, bool LIST = false, bool PB = false>
__global__ void __launch_bounds__(kFuseThreads, COLOR ? KB_FUSE_COLOR_MIN_BLOCKS : KB_FUSE_MIN_BLOCKS) fuseKernel(const __grid_constant__ DeviceMap m, const __grid_constant__ BatchParams p) {
  constexpr int kFetch = PB ? kCtrFetchB : kCtrFetch;
  // Short batches have little work per voxel, so an item then covers all layers of its box (amortising the fetch); long
  // batches use one layer per item for balance.
  constexpr int ipb = kBoxLayers / LPI;  // items per box
  extern __shared__ float4 s_rows4[];    // likelihood rows of the CTA's threads
  const int lane = threadIdx.x & 31;
  int n_cls[kItemClasses] = {0};
  const int n_items = fuseItemCount<VPS, ipb, LIST, PB>(m, p, n_cls);
  const int L = p.L;
  int n_valid = 0, n_band = 0, n_sem = 0;

  // The cursor fetch for the NEXT item is issued before the current item is processed, so the atomic's
  // L2 round trip overlaps useful work.
  int pending = 0;
  if (lane == 0) pending = atomicAdd(&m.counters[kFetch], 1);
  for (;;) {
    const int w = __shfl_sync(0xffffffffu, pending, 0);
    if (w >= n_items) break;
    if (lane == 0) pending = atomicAdd(&m.counters[kFetch], 1);
    int box = w / ipb;
    if constexpr (LIST) {
      box = listedBox<PB>(p, n_cls, box);
    }
    const uint32_t fmask = p.item_fmask[box];
    if (!fmask) continue;
    const int wi = box / kBoxes<VPS>, it = box % kBoxes<VPS>;
    const int slot = p.work_slots[wi];
    const int3 bi = m.block_index[slot];
    const int sem = L > 0 ? m.block_sem[slot] : -1;
    uint32_t upd_all = 0;
    bool any_have = false;
#pragma unroll 1
    for (int k = (w % ipb) * LPI; k < (w % ipb) * LPI + LPI; ++k) {
      const VoxelSite vs = voxelSite<VPS>(p, slot, bi, it, k, lane);
      VoxelState<COLOR> vox;
      LikelihoodRow<kFuseThreads, VPS * VPS * VPS> row;
      uint32_t rem = fmask;
      while (rem) {
        const int b = __ffs(rem) - 1;
        rem &= rem - 1;
        const FrameView& f = p.f[b];
        DepthQuad q;
        Measurement ms;
        uint32_t label = 0;
        if (!projectQuad<COMPACT>(p, f, vs.x, vs.y, vs.z, q) || !resolveQuad(p, q, ms)) continue;
        if (ms.in_band && !labelTap<COMPACT>(p, f, b, ms.ti, label)) continue;
        const float wm = measurementWeight(p, q.z, ms.sdf);
        const float w_old = vox.integrate(m, p, slot, vs.gi, f, b, ms.sdf, wm);
        ++n_valid;
        if (!ms.in_band) continue;
        ++n_band;
        if constexpr (COLOR) vox.mergeColor(p, f, q, ms, wm, w_old);
        if (sem >= 0 && hasLabelImage(p, b) && label < static_cast<uint32_t>(L)) {
          row.add(m, p, s_rows4, sem, vs.lin, label);
          ++n_sem;
        }
      }
      if (vox.have) {  // write the voxel back once
        vox.store(m, p, vs.gi);
        row.store(m, p, s_rows4, sem, vs.lin);
      }
      upd_all |= vox.upd_frames;
      any_have |= vox.have;
    }
    itemUpdated(m, p, slot, wi, any_have, upd_all);
  }
  flushFuseCounters(m, n_valid, n_band, n_sem);
}

// ---- K1, CTA-cooperative two-phase variant (KB_FUSE_COOP) ----------------------------------------------------------
// fuseKernel's unit of serial work is one warp walking up to 32 frames of its 32 voxels: ~280 instructions per frame, so
// the dependency chain of a heavy item is about half the kernel and the SMs drain long before the last warp is done (r2
// capture: SMs idle 26-36 % of the kernel). Only the last ~40 instructions of a frame depend on the voxel state. Here the
// four warps of a CTA share one item: phase A — warp w computes the measurements (projection, taps, sdf, weight, label)
// of the item's frames w, w+4, ... for all 32 voxels and parks them in shared memory; phase B — warp 0 folds them into
// the voxel state in frame order (TSDF recurrence, likelihood row, bookkeeping). Same steps in the same order per
// voxel, so results are bit-identical; the chain per item shrinks to a quarter of the frames plus a short fold, and the
// scheduling unit becomes the CTA (~15 items each instead of ~4 per warp).
template <int VPS, bool COMPACT, bool PB>
__global__ void __launch_bounds__(kFuseThreads, KB_FUSE_MIN_BLOCKS) fuseKernelCoop(const __grid_constant__ DeviceMap m, const __grid_constant__ BatchParams p) {
  constexpr int kFetch = PB ? kCtrFetchB : kCtrFetch;
  constexpr uint8_t kInvalid = 0xFE, kNoSem = 0xFF;
  extern __shared__ float4 s_rows4[];  // [32][S] likelihood rows of the folding warp (BINARY: [2][32]), then the records
  float* __restrict__ s_w = reinterpret_cast<float*>(s_rows4) + fuseRowStride(m.Lp) * 32;  // [32 frames][32 voxels] weight
  float* __restrict__ s_s = s_w + 32 * 32;                                                  // [32][32] sdf (unclamped)
  uint8_t* __restrict__ s_l = reinterpret_cast<uint8_t*>(s_s + 32 * 32);  // [32][32] label | kNoSem | kInvalid
  __shared__ int s_item;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int n_cls[kItemClasses];
  const int n_items = fuseItemCount<VPS, kBoxLayers, true, PB>(m, p, n_cls);
  const int L = p.L;
  int n_valid = 0, n_band = 0, n_sem = 0;
  int pending = 0;
  if (threadIdx.x == 0) pending = atomicAdd(&m.counters[kFetch], 1);
  for (;;) {
    if (threadIdx.x == 0) s_item = pending;
    __syncthreads();  // item index visible; the previous item's fold is done, its records may be overwritten
    const int w = s_item;
    if (w >= n_items) break;
    if (threadIdx.x == 0) pending = atomicAdd(&m.counters[kFetch], 1);  // next item: the round trip overlaps this one
    const int box = listedBox<PB>(p, n_cls, w / kBoxLayers);
    const uint32_t fmask = p.item_fmask[box];
    const int wi = box / kBoxes<VPS>, it = box % kBoxes<VPS>;
    const int slot = p.work_slots[wi];
    const int sem = L > 0 ? m.block_sem[slot] : -1;
    const VoxelSite vs = voxelSite<VPS>(p, slot, m.block_index[slot], it, w % kBoxLayers, lane);
    const int nf = __popc(fmask);
    // ---- phase A: measurements of frames (rank r among the item's frames) r = warp, warp + 4, ...
    for (int r = warp; r < nf; r += 4) {
      const int b = __fns(fmask, 0, r + 1);
      const FrameView& f = p.f[b];
      DepthQuad q;
      Measurement ms;
      uint32_t label = 0;
      uint8_t tag = kInvalid;
      float sdf = 0.f, wm = 0.f;
      if (projectQuad<COMPACT>(p, f, vs.x, vs.y, vs.z, q) && resolveQuad(p, q, ms) &&
          (!ms.in_band || labelTap<COMPACT>(p, f, b, ms.ti, label))) {
        sdf = ms.sdf;
        wm = measurementWeight(p, q.z, ms.sdf);
        tag = ms.in_band && sem >= 0 && hasLabelImage(p, b) && label < static_cast<uint32_t>(L) ? static_cast<uint8_t>(label) : kNoSem;
      }
      s_w[r * 32 + lane] = wm;
      s_s[r * 32 + lane] = sdf;
      s_l[r * 32 + lane] = tag;
    }
    __syncthreads();  // all measurements of the item are in shared memory
    // ---- phase B: warp 0 folds the frames into the voxel state, in frame order
    if (warp == 0) {
      VoxelState<false> vox;
      LikelihoodRow<32, VPS * VPS * VPS> row;
      uint32_t rem = fmask;
      for (int r = 0; rem; ++r) {
        const int b = __ffs(rem) - 1;
        rem &= rem - 1;
        const uint8_t tag = s_l[r * 32 + lane];
        if (tag == kInvalid) continue;
        const float sdf = s_s[r * 32 + lane];
        vox.integrate(m, p, slot, vs.gi, p.f[b], b, sdf, s_w[r * 32 + lane]);
        ++n_valid;
        if (!(fabsf(sdf) < p.trunc)) continue;
        ++n_band;
        if (tag == kNoSem) continue;
        row.add(m, p, s_rows4, sem, vs.lin, tag);
        ++n_sem;
      }
      if (vox.have) {
        vox.store(m, p, vs.gi);
        row.store(m, p, s_rows4, sem, vs.lin);
      }
      itemUpdated(m, p, slot, wi, vox.have, vox.upd_frames);
    }
  }
  if (warp == 0) flushFuseCounters(m, n_valid, n_band, n_sem);
}

// ---- K1, memory-level-parallel variant (experiment, KB_FUSE_MLP=G; off by default) -------------------------------
// fuseKernel walks an item's frames one at a time: projection -> 4 depth taps -> label/mask tap -> update, i.e. two
// dependent memory round trips per in-band frame and voxel (three, with the nearest-pixel reload it had when this variant
// was measured), with ~26 resident warps per SM to hide them (ncu, then: issue slots 54 % busy, the rest is latency).
// Only the last step depends on the voxel state. This variant processes the frames of an item in groups of G: phase A
// projects the voxel into all G frames and issues their depth quads together; phase B1 resolves the quads and issues the
// G label + mask taps together; phase B2 applies the G updates in frame order. Steps, order and results are those of
// fuseKernel; registers go up (G x ~9 live values), occupancy down.
#ifndef KB_FUSE_MLP_MIN_BLOCKS
#define KB_FUSE_MLP_MIN_BLOCKS 5
#endif
template <int VPS, int LPI, bool COMPACT, int G, bool LIST, bool PB = false>
__global__ void __launch_bounds__(kFuseThreads, KB_FUSE_MLP_MIN_BLOCKS) fuseKernelMlp(const __grid_constant__ DeviceMap m, const __grid_constant__ BatchParams p) {
  constexpr int kFetch = PB ? kCtrFetchB : kCtrFetch;
  constexpr int ipb = kBoxLayers / LPI;
  extern __shared__ float4 s_rows4[];
  const int lane = threadIdx.x & 31;
  int n_cls[kItemClasses] = {0};
  const int n_items = fuseItemCount<VPS, ipb, LIST, PB>(m, p, n_cls);
  const int L = p.L;
  int n_valid = 0, n_band = 0, n_sem = 0;

  int pending = 0;
  if (lane == 0) pending = atomicAdd(&m.counters[kFetch], 1);
  for (;;) {
    const int w = __shfl_sync(0xffffffffu, pending, 0);
    if (w >= n_items) break;
    if (lane == 0) pending = atomicAdd(&m.counters[kFetch], 1);
    int box = w / ipb;
    if constexpr (LIST) {
      box = listedBox<PB>(p, n_cls, box);
    }
    const uint32_t fmask = p.item_fmask[box];
    if (!fmask) continue;
    const int wi = box / kBoxes<VPS>, it = box % kBoxes<VPS>;
    const int slot = p.work_slots[wi];
    const int3 bi = m.block_index[slot];
    const int sem = L > 0 ? m.block_sem[slot] : -1;
    uint32_t upd_all = 0;
    bool any_have = false;
#pragma unroll 1
    for (int k = (w % ipb) * LPI; k < (w % ipb) * LPI + LPI; ++k) {
      const VoxelSite vs = voxelSite<VPS>(p, slot, bi, it, k, lane);
      VoxelState<false> vox;
      LikelihoodRow<kFuseThreads, VPS * VPS * VPS> row;
      uint32_t rem = fmask;  // warp-uniform
#pragma unroll 1
      while (rem) {
        int fb[G];
        bool ok[G];
        DepthQuad q[G];
        // ---- phase A: projections and depth taps of up to G frames (no dependence on the voxel state)
#pragma unroll
        for (int g = 0; g < G; ++g) {
          fb[g] = 0;
          ok[g] = false;
          if (rem) {
            fb[g] = __ffs(rem) - 1;
            rem &= rem - 1;
            ok[g] = projectQuad<COMPACT>(p, p.f[fb[g]], vs.x, vs.y, vs.z, q[g]);
          }
        }
        // ---- phase B1: interpolation, sdf and weight; the label / mask taps of the G frames issued together
        Measurement ms[G];
        float wm[G];
        uint32_t label[G];
#pragma unroll
        for (int g = 0; g < G; ++g) {
          label[g] = 0;
          ok[g] = ok[g] && resolveQuad(p, q[g], ms[g]) &&
                  (!ms[g].in_band || labelTap<COMPACT>(p, p.f[fb[g]], fb[g], ms[g].ti, label[g]));
          wm[g] = ok[g] ? measurementWeight(p, q[g].z, ms[g].sdf) : 0.f;
        }
        // ---- phase B2: the G updates in frame order (the only part that depends on the voxel state)
#pragma unroll
        for (int g = 0; g < G; ++g) {
          if (!ok[g]) continue;
          const int b = fb[g];
          vox.integrate(m, p, slot, vs.gi, p.f[b], b, ms[g].sdf, wm[g]);
          ++n_valid;
          if (!ms[g].in_band) continue;
          ++n_band;
          if (sem >= 0 && hasLabelImage(p, b) && label[g] < static_cast<uint32_t>(L)) {
            row.add(m, p, s_rows4, sem, vs.lin, label[g]);
            ++n_sem;
          }
        }
      }
      if (vox.have) {
        vox.store(m, p, vs.gi);
        row.store(m, p, s_rows4, sem, vs.lin);
      }
      upd_all |= vox.upd_frames;
      any_have |= vox.have;
    }
    itemUpdated(m, p, slot, wi, any_have, upd_all);
  }
  flushFuseCounters(m, n_valid, n_band, n_sem);
}

// ---- K2 (lazy): TrackingIntegrator::updateBlockTracking (tracking_integrator.cpp:133-166,224-246) ------
// The reference rewrites last_occupied / active / to_remove of EVERY voxel of EVERY allocated block each
// frame (~10 GB/frame at 50 k blocks). All three are pure functions of (distance, last_observed, the
// pass history), so the pass itself only (1) records the pass in two small per-frame-index tables,
// (2) latches tracking_updated into the ever-free work list and clears it, (3) clears the
// finishMapping override. Per-voxel values are derived by evalTracking() when someone needs them
// (K1 when it rewrites a voxel, K3, K2r, export) — bit-identical to the brute-force pass
// (tests/test_parity_gpu.py, tests/test_golden.py).
__global__ void trackingPassKernel(const DeviceMap m, const TrackingParams p) {
  const int slot = blockIdx.x * blockDim.x + threadIdx.x;
  if (slot == 0) {
    for (uint32_t i = p.prev_pass + 1; i <= p.ev.k_last; ++i) m.next_pass[i] = p.ev.k_last;
    m.act_min[p.ev.k_last] = p.ev.act_min;
  }
  if (slot >= p.n_slots) return;
  const uint32_t flags = m.block_flags[slot];
  if (!(flags & kFlagAllocated)) return;
  uint32_t f = flags & ~(static_cast<uint32_t>(KB_FLAG_TRACKING_UPDATED) | kFlagInactiveOverride);
  if (flags & KB_FLAG_TRACKING_UPDATED) p.pending[atomicAdd(&m.counters[kCtrPending], 1)] = slot;
  if (f != flags) m.block_flags[slot] = f;
}

// ---- K3: TrackingIntegrator::updateBlockEverFree (tracking_integrator.cpp:168-222) ------------------
// "free(v)" = ever_free(v) || voxelIsFree(v). Neighbours set ever_free concurrently, but a voxel set
// in this pass necessarily satisfies voxelIsFree, so the predicate is stable under the race.
// During a pass every voxel of an existing block has been seen by it, so last_occupied is "now" for
// occupied voxels and the stored value otherwise.
__device__ __forceinline__ bool voxelFreeNow(const DeviceMap& m, const TrackEval& t, size_t idx, uint8_t f) {
  if (f & kVoxEverFree) return true;
  if (!(f & kVoxNotOccupied)) return false;  // occupied => last_occupied == now (also: never observed)
  const uint32_t oc = m.last_occ[idx];
  return oc == 0 ? (t.zero_free != 0) : (oc < t.free_max);
}

// One CTA per pending block. The "free or ever-free" predicate of the block's voxels and of a one-voxel halo
// (taken from the 26 neighbour blocks, resolved once into shared memory) is first materialised in shared
// memory by all threads in parallel; the 6/18/26-neighbourhood test of every candidate voxel then only reads
// shared memory, instead of chasing up to 18 dependent global loads per candidate.
// SHARD: neighbour blocks owned by another rank are not in the local hash; their predicate bits come from the
// all-gathered halo masks (ShardExchange), found through the ghost table; s_nbr then holds -(2 + word offset).
__device__ __forceinline__ int ghostLookup(const TrackingParams& p, int x, int y, int z) {
  const unsigned long long key = packKey(x, y, z);
  uint32_t h = static_cast<uint32_t>(mix64(key)) & p.ghost_mask;
  for (uint32_t probe = 0; probe <= p.ghost_mask; ++probe) {
    const unsigned long long k = p.ghost_keys[h];
    if (k == key) return p.ghost_vals[h];
    if (k == kEmptyKey) return -1;
    h = (h + 1) & p.ghost_mask;
  }
  return -1;
}

template <bool SHARD>
__global__ void __launch_bounds__(kThreads) everFreeKernel(const DeviceMap m, const TrackingParams p) {
  __shared__ int s_nbr[27];
  __shared__ uint8_t s_free[18 * 18 * 18];  // bit0: free or ever-free, bit1: ever-free (halo of the largest block)
  const int n = m.counters[kCtrPending];
  const int vps = m.vps, V = m.V, hs = vps + 2;
  for (int w = blockIdx.x; w < n; w += gridDim.x) {
    const int slot = p.pending[w];
    __syncthreads();
    if (threadIdx.x < 27) {
      const int3 bi = m.block_index[slot];
      const int dx = threadIdx.x % 3 - 1, dy = (threadIdx.x / 3) % 3 - 1, dz = threadIdx.x / 9 - 1;
      int ns = (dx == 0 && dy == 0 && dz == 0) ? slot : hashLookup(m, bi.x + dx, bi.y + dy, bi.z + dz);
      if (SHARD && ns < 0 && mapOwner(m, bi.x + dx, bi.y + dy, bi.z + dz, p.nranks) != p.rank) {
        const int off = ghostLookup(p, bi.x + dx, bi.y + dy, bi.z + dz);
        if (off >= 0) ns = -(2 + off);
      }
      s_nbr[threadIdx.x] = ns;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < hs * hs * hs; i += kThreads) {
      int x = i % hs - 1, y = (i / hs) % hs - 1, z = i / (hs * hs) - 1;
      int bx = 1, by = 1, bz = 1;
      if (x < 0) { x += vps; bx = 0; } else if (x >= vps) { x -= vps; bx = 2; }
      if (y < 0) { y += vps; by = 0; } else if (y >= vps) { y -= vps; by = 2; }
      if (z < 0) { z += vps; bz = 0; } else if (z >= vps) { z -= vps; bz = 2; }
      const int ns = s_nbr[bx + 3 * by + 9 * bz];
      uint8_t v = 0;  // missing neighbour block: blocks its neighbours (:198-202)
      if (ns >= 0) {
        const size_t idx = static_cast<size_t>(ns) * V + (x + vps * (y + vps * z));
        const uint8_t f = m.vflags[idx];
        v = (voxelFreeNow(m, p.ev, idx, f) ? 1 : 0) | ((f & kVoxEverFree) ? 2 : 0);
      } else if (SHARD && ns <= -2) {  // remote neighbour: bit of its published mask (halo voxels only need bit 0)
        const int lin = x + vps * (y + vps * z);
        v = (static_cast<uint32_t>(__ldg(&p.ghost_bits[(-ns - 2) + (lin >> 5)])) >> (lin & 31)) & 1u;
      }
      s_free[i] = v;
    }
    __syncthreads();
    const size_t base = static_cast<size_t>(slot) * V;
    for (int lin = threadIdx.x; lin < V; lin += kThreads) {
      const int vx = lin % vps, vy = (lin / vps) % vps, vz = lin / (vps * vps);
      const int c = (vx + 1) + hs * ((vy + 1) + hs * (vz + 1));
      if (s_free[c] != 1) continue;  // needs: free now, not yet ever-free
      bool blocked = false;
      for (int dz = -1; dz <= 1 && !blocked; ++dz)
        for (int dy = -1; dy <= 1 && !blocked; ++dy)
          for (int dx = -1; dx <= 1; ++dx) {
            const int nnz = (dx != 0) + (dy != 0) + (dz != 0);
            if (nnz == 0 || (p.connectivity == 6 && nnz > 1) || (p.connectivity == 18 && nnz > 2)) continue;
            if (!(s_free[c + dx + hs * (dy + hs * dz)] & 1)) { blocked = true; break; }
          }
      if (!blocked) m.vflags[base + lin] |= kVoxEverFree;
    }
  }
}

// KB_EVERFREE_V2 (experiment, same results): the halo fill of everFreeKernel walks all (vps+2)^3 cells with one scalar byte
// load each (23 dependent iterations per thread at vps 16). Here the block's own vps^3 flag bytes arrive as 16-byte vector
// loads (one per thread at vps 16) and only the one-voxel shell taken from the 26 neighbour blocks (1736 of 5832 cells) is
// gathered cell by cell.
template <bool SHARD>
__global__ void __launch_bounds__(kThreads) everFreeKernelV2(const DeviceMap m, const TrackingParams p) {
  __shared__ int s_nbr[27];
  __shared__ uint8_t s_free[18 * 18 * 18];
  const int n = m.counters[kCtrPending];
  const int vps = m.vps, V = m.V, hs = vps + 2;
  const int planeA = hs * hs, planeB = vps * hs, planeC = vps * vps, n_shell = 2 * (planeA + planeB + planeC);
  for (int w = blockIdx.x; w < n; w += gridDim.x) {
    const int slot = p.pending[w];
    __syncthreads();
    if (threadIdx.x < 27) {
      const int3 bi = m.block_index[slot];
      const int dx = threadIdx.x % 3 - 1, dy = (threadIdx.x / 3) % 3 - 1, dz = threadIdx.x / 9 - 1;
      int ns = (dx == 0 && dy == 0 && dz == 0) ? slot : hashLookup(m, bi.x + dx, bi.y + dy, bi.z + dz);
      if (SHARD && ns < 0 && mapOwner(m, bi.x + dx, bi.y + dy, bi.z + dz, p.nranks) != p.rank) {
        const int off = ghostLookup(p, bi.x + dx, bi.y + dy, bi.z + dz);
        if (off >= 0) ns = -(2 + off);
      }
      s_nbr[threadIdx.x] = ns;
    }
    const size_t base = static_cast<size_t>(slot) * V;
    // centre block: 16 flag bytes per vector load (does not need s_nbr)
    for (int q = threadIdx.x; q < V / 16; q += kThreads) {
      const uint4 f16 = *reinterpret_cast<const uint4*>(m.vflags + base + static_cast<size_t>(q) * 16);
      const uint32_t wds[4] = {f16.x, f16.y, f16.z, f16.w};
#pragma unroll
      for (int k = 0; k < 16; ++k) {
        const uint8_t f = static_cast<uint8_t>((wds[k >> 2] >> (8 * (k & 3))) & 0xFFu);
        const int lin = q * 16 + k;
        const int vx = lin % vps, vy = (lin / vps) % vps, vz = lin / (vps * vps);
        s_free[(vx + 1) + hs * ((vy + 1) + hs * (vz + 1))] =
            static_cast<uint8_t>((voxelFreeNow(m, p.ev, base + lin, f) ? 1 : 0) | ((f & kVoxEverFree) ? 2 : 0));
      }
    }
    __syncthreads();  // s_nbr complete
    // one-voxel shell from the neighbour blocks: two z planes, two y slabs, two x slabs
    for (int j = threadIdx.x; j < n_shell; j += kThreads) {
      int x, y, z;
      if (j < 2 * planeA) {
        const int r = j % planeA;
        x = r % hs - 1; y = r / hs - 1; z = (j / planeA) ? vps : -1;
      } else if (j < 2 * (planeA + planeB)) {
        const int jj = j - 2 * planeA, r = jj % planeB;
        x = r % hs - 1; z = r / hs; y = (jj / planeB) ? vps : -1;
      } else {
        const int jj = j - 2 * (planeA + planeB), r = jj % planeC;
        y = r % vps; z = r / vps; x = (jj / planeC) ? vps : -1;
      }
      const int cell = (x + 1) + hs * ((y + 1) + hs * (z + 1));
      int bx = 1, by = 1, bz = 1;
      if (x < 0) { x += vps; bx = 0; } else if (x >= vps) { x -= vps; bx = 2; }
      if (y < 0) { y += vps; by = 0; } else if (y >= vps) { y -= vps; by = 2; }
      if (z < 0) { z += vps; bz = 0; } else if (z >= vps) { z -= vps; bz = 2; }
      const int ns = s_nbr[bx + 3 * by + 9 * bz];
      uint8_t v = 0;  // missing neighbour block: blocks its neighbours (:198-202)
      if (ns >= 0) {
        const size_t idx = static_cast<size_t>(ns) * V + (x + vps * (y + vps * z));
        const uint8_t f = m.vflags[idx];
        v = (voxelFreeNow(m, p.ev, idx, f) ? 1 : 0) | ((f & kVoxEverFree) ? 2 : 0);
      } else if (SHARD && ns <= -2) {
        const int lin = x + vps * (y + vps * z);
        v = (static_cast<uint32_t>(__ldg(&p.ghost_bits[(-ns - 2) + (lin >> 5)])) >> (lin & 31)) & 1u;
      }
      s_free[cell] = v;
    }
    __syncthreads();
    for (int lin = threadIdx.x; lin < V; lin += kThreads) {
      const int vx = lin % vps, vy = (lin / vps) % vps, vz = lin / (vps * vps);
      const int c = (vx + 1) + hs * ((vy + 1) + hs * (vz + 1));
      if (s_free[c] != 1) continue;
      bool blocked = false;
      for (int dz = -1; dz <= 1 && !blocked; ++dz)
        for (int dy = -1; dy <= 1 && !blocked; ++dy)
          for (int dx = -1; dx <= 1; ++dx) {
            const int nnz = (dx != 0) + (dy != 0) + (dz != 0);
            if (nnz == 0 || (p.connectivity == 6 && nnz > 1) || (p.connectivity == 18 && nnz > 2)) continue;
            if (!(s_free[c + dx + hs * (dy + hs * dz)] & 1)) { blocked = true; break; }
          }
      if (!blocked) m.vflags[base + lin] |= kVoxEverFree;
    }
  }
}

// Resets the ever-free work counter after K3 (separate tiny launch: K3's CTAs all read it).
__global__ void resetPendingKernel(const DeviceMap m) { m.counters[kCtrPending] = 0; }

// ---- sharded K2/K3 exchange (SURVEY.md §8e step 1; buffer layouts: ShardExchange in kb_kernels.cuh) ----------
// Exports this rank's ever-free work list as block indices.
__global__ void exportPendingKernel(const DeviceMap m, const int* __restrict__ pending, int32_t* __restrict__ out, int cap) {
  const int n = m.counters[kCtrPending];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) {
    out[0] = min(n, cap);
    out[1] = n > cap ? 1 : 0;
    out[2] = out[3] = 0;
    m.counters[kCtrHalo] = 0;
  }
  if (i < min(n, cap)) {
    const int3 bi = m.block_index[pending[i]];
    out[4 + 3 * i] = bi.x; out[4 + 3 * i + 1] = bi.y; out[4 + 3 * i + 2] = bi.z;
  }
}

// One thread per (rank r != me, pending block i of r, neighbour offset k): if the neighbour is owned by this rank
// and exists, its slot joins the publish list (once).
__global__ void haloMarkKernel(const DeviceMap m, const ShardExchange x, const int32_t* __restrict__ all_pending) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  const int per_rank = x.cap_pending * 27;
  if (t >= x.nranks * per_rank) return;
  const int r = t / per_rank, i = (t % per_rank) / 27, k = t % 27;
  if (r == x.rank || k == 13) return;
  const int32_t* __restrict__ buf = all_pending + static_cast<size_t>(r) * x.pending_stride();
  if (i >= buf[0]) return;
  const int bx = buf[4 + 3 * i] + (k % 3 - 1), by = buf[4 + 3 * i + 1] + ((k / 3) % 3 - 1), bz = buf[4 + 3 * i + 2] + (k / 9 - 1);
  if (mapOwner(m, bx, by, bz, x.nranks) != x.rank) return;
  const int slot = hashLookup(m, bx, by, bz);
  if (slot < 0) return;
  if (atomicExch(&x.halo_mark[slot], 1) != 0) return;
  const int j = atomicAdd(&m.counters[kCtrHalo], 1);
  if (j < x.cap_halo) x.publish[j] = slot;
}

// One CTA per published block: 1 bit per voxel = "ever_free || voxelIsFree at this pass" (the K3 neighbour predicate).
__global__ void __launch_bounds__(kThreads) haloPackKernel(const DeviceMap m, const TrackingParams p, const ShardExchange x,
                                                           int32_t* __restrict__ out) {
  const int n_all = m.counters[kCtrHalo];
  const int n = min(n_all, x.cap_halo);
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    out[0] = n;
    out[1] = n_all > x.cap_halo ? 1 : 0;
    out[2] = out[3] = 0;
  }
  const int V = m.V;
  for (int j = blockIdx.x; j < n_all; j += gridDim.x) {
    const int slot = j < x.cap_halo ? x.publish[j] : -1;
    if (slot < 0) continue;
    if (threadIdx.x == 0) x.halo_mark[slot] = 0;
    int32_t* __restrict__ e = out + 4 + static_cast<size_t>(j) * x.halo_entry();
    if (threadIdx.x == 0) {
      const int3 bi = m.block_index[slot];
      e[0] = bi.x; e[1] = bi.y; e[2] = bi.z; e[3] = 0;
    }
    const size_t base = static_cast<size_t>(slot) * V;
    for (int lin = threadIdx.x; lin < V; lin += kThreads) {  // V and kThreads are multiples of 32: full warps
      const bool fr = voxelFreeNow(m, p.ev, base + lin, m.vflags[base + lin]);
      const unsigned bits = __ballot_sync(0xffffffffu, fr);
      if ((threadIdx.x & 31) == 0) e[4 + (lin >> 5)] = static_cast<int32_t>(bits);
    }
  }
}

// ---- peer-memory producers: the same lists / masks, stored into slot `rank` of EVERY rank's buffer --------------------
__global__ void exportPendingPeersKernel(const DeviceMap m, const int* __restrict__ pending, const PeerBuffers peers, int rank,
                                         int stride, int cap) {
  const int n = m.counters[kCtrPending];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) m.counters[kCtrHalo] = 0;
  const bool entry = i < min(n, cap);
  int3 bi = make_int3(0, 0, 0);
  if (entry) bi = m.block_index[pending[i]];
  for (int q = 0; q < peers.n; ++q) {
    int32_t* __restrict__ out = static_cast<int32_t*>(peers.p[q]) + static_cast<size_t>(rank) * stride;
    if (i == 0) {
      out[0] = min(n, cap);
      out[1] = n > cap ? 1 : 0;
      out[2] = out[3] = 0;
    }
    if (entry) { out[4 + 3 * i] = bi.x; out[4 + 3 * i + 1] = bi.y; out[4 + 3 * i + 2] = bi.z; }
  }
}

__global__ void __launch_bounds__(kThreads) haloPackPeersKernel(const DeviceMap m, const TrackingParams p, const ShardExchange x,
                                                                const PeerBuffers peers) {
  const int n_all = m.counters[kCtrHalo];
  const int n = min(n_all, x.cap_halo);
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    for (int q = 0; q < peers.n; ++q) {
      int32_t* out = static_cast<int32_t*>(peers.p[q]) + static_cast<size_t>(x.rank) * x.halo_stride();
      out[0] = n;
      out[1] = n_all > x.cap_halo ? 1 : 0;
      out[2] = out[3] = 0;
    }
  }
  const int V = m.V;
  for (int j = blockIdx.x; j < n_all; j += gridDim.x) {
    const int slot = j < x.cap_halo ? x.publish[j] : -1;
    if (slot < 0) continue;
    if (threadIdx.x == 0) x.halo_mark[slot] = 0;
    const size_t eoff = static_cast<size_t>(x.rank) * x.halo_stride() + 4 + static_cast<size_t>(j) * x.halo_entry();
    if (threadIdx.x == 0) {
      const int3 bi = m.block_index[slot];
      for (int q = 0; q < peers.n; ++q) {
        int32_t* e = static_cast<int32_t*>(peers.p[q]) + eoff;
        e[0] = bi.x; e[1] = bi.y; e[2] = bi.z; e[3] = 0;
      }
    }
    const size_t base = static_cast<size_t>(slot) * V;
    for (int lin = threadIdx.x; lin < V; lin += kThreads) {
      const bool fr = voxelFreeNow(m, p.ev, base + lin, m.vflags[base + lin]);
      const unsigned bits = __ballot_sync(0xffffffffu, fr);
      if ((threadIdx.x & 31) == 0)
        for (int q = 0; q < peers.n; ++q) static_cast<int32_t*>(peers.p[q])[eoff + 4 + (lin >> 5)] = static_cast<int32_t>(bits);
    }
  }
}

// M1 exchange without a reduction: a pixel's flag byte is non-zero on at most one rank (the owner of its block), so every
// rank simply stores its non-zero bytes into all reduced flag images (zeroed by their owners after the previous use).
__global__ void flagScatterKernel(const uint8_t* __restrict__ local_flags, const PeerBuffers peers, int n) {
  const int px = blockIdx.x * blockDim.x + threadIdx.x;
  if (px >= n) return;
  const uint8_t f = local_flags[px];
  if (f == 0) return;
  for (int q = 0; q < peers.n; ++q) static_cast<uint8_t*>(peers.p[q])[px] = f;
}

// ---- NVLS frame broadcast: rank 0 stores the step's frames ONCE to the multicast mapping of the symmetric receive buffer;
// NVSwitch replicates every store to all ranks (multimem.st; SASS: STG.E.128.STRONG.SYS on a multicast address), so the
// ingest rank's egress is 1x the frame bytes instead of a ring / tree of point-to-point copies.
__global__ void __launch_bounds__(256) multicastCopyKernel(float4* __restrict__ mc_dst, const float4* __restrict__ src, size_t n16) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n16; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const float4 v = __ldg(&src[i]);
#ifdef KB_CUDA_EMU
    mc_dst[i] = v;
#else
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(mc_dst + i), "f"(v.x), "f"(v.y), "f"(v.z),
                 "f"(v.w)
                 : "memory");
#endif
  }
}

// Overflowed publish lists leave marks behind: clear the marks of the slots that did not fit (rare; error path).
__global__ void haloUnmarkKernel(const DeviceMap m, const ShardExchange x, int n_slots) {
  const int slot = blockIdx.x * blockDim.x + threadIdx.x;
  if (slot < n_slots && m.counters[kCtrHalo] > x.cap_halo) x.halo_mark[slot] = 0;
}

// Builds the ghost table from the other ranks' halo buffers: block key -> word offset of its mask.
__global__ void ghostBuildKernel(const DeviceMap m, const ShardExchange x, const int32_t* __restrict__ all_pending,
                                 const int32_t* __restrict__ all_halo) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= x.nranks * x.cap_halo) return;
  const int r = t / x.cap_halo, i = t % x.cap_halo;
  const int32_t* __restrict__ buf = all_halo + static_cast<size_t>(r) * x.halo_stride();
  if (i == 0 && (buf[1] != 0 || all_pending[static_cast<size_t>(r) * x.pending_stride() + 1] != 0))
    atomicExch(&m.counters[kCtrCapacityExceeded], 1);  // a list did not fit its exchange buffer: results incomplete
  if (r == x.rank || i >= buf[0]) return;
  const int off = r * x.halo_stride() + 4 + i * x.halo_entry();
  const unsigned long long key = packKey(all_halo[off], all_halo[off + 1], all_halo[off + 2]);
  uint32_t h = static_cast<uint32_t>(mix64(key)) & x.ghost_mask;
  for (uint32_t probe = 0; probe <= x.ghost_mask; ++probe) {
    if (atomicCAS(&x.ghost_keys[h], kEmptyKey, key) == kEmptyKey) {  // keys are unique: each block has one owner
      x.ghost_vals[h] = off + 4;
      return;
    }
    h = (h + 1) & x.ghost_mask;
  }
}

// ---- K2r: TrackingIntegrator::resetInactive (tracking_integrator.cpp:106-131) -----------------------
__global__ void __launch_bounds__(kThreads) resetInactiveKernel(const DeviceMap m, const TrackEval ev, int3* removed, int max_removed) {
  const int slot = blockIdx.x;
  const uint32_t flags = m.block_flags[slot];
  if (!(flags & kFlagAllocated)) return;
  const int V = m.V;
  const size_t base = static_cast<size_t>(slot) * V;
  const uint32_t born = m.born_frame[slot];
  // read before the block-wide reductions below: thread 0 resets block_sem at the end, and without a barrier in
  // between a slow warp could otherwise see -1 and skip scrubbing its part of the semantic slot (found by running
  // the kernels under tools/cuda_emu, whose sequential fiber schedule makes thread 0 finish first)
  const int sem = m.block_sem[slot];
  int all_remove = 1, any_active = 0;
  for (int lin = threadIdx.x; lin < V; lin += kThreads) {
    uint32_t c;
    bool act, rem;
    evalTracking(m, ev, born, m.last_obs[base + lin], m.last_occ[base + lin], m.vflags[base + lin], &c, &act, &rem);
    all_remove &= rem ? 1 : 0;
    any_active |= act ? 1 : 0;
  }
  all_remove = __syncthreads_and(all_remove);
  any_active = __syncthreads_or(any_active);
  // has_active_data: set by the last pass that saw the block; false before any pass and after finishMapping
  const bool seen = ev.k_last != 0 && ev.k_last >= born;
  const bool has_active = seen && any_active && !(flags & kFlagInactiveOverride);
  if (has_active && !all_remove) return;
  // Remove: scrub the slot so that a later allocation starts from the default voxel state.
  for (int lin = threadIdx.x; lin < V; lin += kThreads) {
    m.tsdf[base + lin] = make_float2(0.f, 0.f);
    m.last_obs[base + lin] = 0;
    m.last_occ[base + lin] = 0;
    m.vflags[base + lin] = 0;
    if (m.color) m.color[base + lin] = make_uchar4(0, 0, 0, 0);
    if (sem >= 0) m.sem_label[static_cast<size_t>(sem) * V + lin] = kSemEmpty;
  }
  if (threadIdx.x == 0) {
    const int3 bi = m.block_index[slot];
    const unsigned long long key = packKey(bi.x, bi.y, bi.z);
    uint32_t h = static_cast<uint32_t>(mix64(key)) & m.hash_mask;
    for (uint32_t probe = 0; probe <= m.hash_mask; ++probe) {
      const unsigned long long k = m.hash_keys[h];
      if (k == key) { m.hash_keys[h] = kTombKey; break; }
      if (k == kEmptyKey) break;
      h = (h + 1) & m.hash_mask;
    }
    m.block_flags[slot] = 0;
    m.block_sem[slot] = -1;
    m.free_list[atomicAdd(&m.counters[kCtrFreeCount], 1)] = slot;
    if (sem >= 0) m.sem_free_list[atomicAdd(&m.counters[kCtrSemFreeCount], 1)] = sem;
    atomicSub(&m.counters[kCtrLiveBlocks], 1);
    const int r = atomicAdd(&m.counters[kCtrRemoved], 1);
    if (r < max_removed) removed[r] = bi;
  }
}

// Tombstone garbage collection: the table was cleared; every live slot re-inserts its key (keys are unique).
__global__ void rehashKernel(const DeviceMap m, int n) {
  const int slot = blockIdx.x * blockDim.x + threadIdx.x;
  if (slot == 0) atomicAdd(&m.counters[kCtrRehash], 1);
  if (slot >= n || !(m.block_flags[slot] & kFlagAllocated)) return;
  const int3 bi = m.block_index[slot];
  const unsigned long long key = packKey(bi.x, bi.y, bi.z);
  uint32_t h = static_cast<uint32_t>(mix64(key)) & m.hash_mask;
  for (uint32_t probe = 0; probe <= m.hash_mask; ++probe) {
    if (atomicCAS(&m.hash_keys[h], kEmptyKey, key) == kEmptyKey) {
      m.hash_vals[h] = slot;
      return;
    }
    h = (h + 1) & m.hash_mask;
  }
}

__global__ void markAllInactiveKernel(const DeviceMap m, int n) {
  const int slot = blockIdx.x * blockDim.x + threadIdx.x;
  if (slot < n && (m.block_flags[slot] & kFlagAllocated)) m.block_flags[slot] |= kFlagInactiveOverride;
}

__global__ void clearUpdatedKernel(const DeviceMap m, int n) {
  const int slot = blockIdx.x * blockDim.x + threadIdx.x;
  if (slot < n && (m.block_flags[slot] & kFlagAllocated)) m.block_flags[slot] &= ~static_cast<uint32_t>(KB_FLAG_UPDATED);
}

// ---- M1: FreeSpaceMotionDetector::setUpPointMapPart (free_space_motion_detector.cpp:158-203) --------
// SHARD (block-hash sharded map, SURVEY.md §8e step 2): only the owner rank knows whether the pixel's block exists
// and whether its voxel is ever-free, so the kernel writes the voxel index of every pixel with a valid index plus a
// flag byte (bit0 block exists here, bit1 ever-free) that is MAX-reduced over the ranks; motionFinalizeKernel then
// produces what the unsharded kernel writes directly.
template <bool SHARD>
__global__ void motionLookupKernel(const DeviceMap m, const __grid_constant__ MotionParams p) {
  const int px = blockIdx.x * blockDim.x + threadIdx.x;
  if (px >= p.W * p.H) return;
  int3 g = make_int3(INT_MIN, 0, 0);
  uint8_t seed = 0, flags = 0;
  const float range = __ldg(&p.depth[px]);
  if (range > 0.f && range <= p.max_range) {
    float wx, wy, wz;
    if (p.vertex) {
      wx = __ldg(&p.vertex[3 * px]); wy = __ldg(&p.vertex[3 * px + 1]); wz = __ldg(&p.vertex[3 * px + 2]);
    } else {
      const int u = px % p.W, v = px / p.W;
      const float cxn = (static_cast<float>(u) - p.cx) / p.fx * range;
      const float cyn = (static_cast<float>(v) - p.cy) / p.fy * range;
      xform(p.Rw, p.tw, cxn, cyn, range, wx, wy, wz);
    }
    if (!(wz < p.min_z_world)) {
      const int bx = static_cast<int>(floorf(wx * p.block_size_inv));
      const int by = static_cast<int>(floorf(wy * p.block_size_inv));
      const int bz = static_cast<int>(floorf(wz * p.block_size_inv));
      const int slot = hashLookup(m, bx, by, bz);
      if (SHARD || slot >= 0) {
        const int vps = m.vps;
        const int vx = static_cast<int>(floorf((wx - static_cast<float>(bx) * p.block_size) * p.voxel_size_inv));
        const int vy = static_cast<int>(floorf((wy - static_cast<float>(by) * p.block_size) * p.voxel_size_inv));
        const int vz = static_cast<int>(floorf((wz - static_cast<float>(bz) * p.block_size) * p.voxel_size_inv));
        if (vx >= 0 && vy >= 0 && vz >= 0 && vx < vps && vy < vps && vz < vps) {
          g = make_int3(bx * vps + vx, by * vps + vy, bz * vps + vz);
          if (slot >= 0) {
            seed = (m.vflags[static_cast<size_t>(slot) * m.V + (vx + vps * (vy + vps * vz))] & kVoxEverFree) ? 1 : 0;
            flags = static_cast<uint8_t>(1 | (seed << 1));
          }
        }
      }
    }
  }
  p.pixel_gidx[px] = g;
  if (SHARD) {
    p.pixel_flags[px] = flags;
    return;
  }
  p.pixel_seed[px] = seed;
  // one counter update per warp
  const unsigned ballot = __ballot_sync(__activemask(), seed != 0);
  if (ballot && (threadIdx.x & 31) == (__ffs(ballot) - 1)) atomicAdd(&m.counters[kCtrSeeds], __popc(ballot));
}

// Sharded M1, second half: flags = MAX over the ranks of the per-rank flag bytes.
__global__ void motionFinalizeKernel(const DeviceMap m, const uint8_t* __restrict__ flags, int3* __restrict__ gidx,
                                     uint8_t* __restrict__ seed_out, int n) {
  const int px = blockIdx.x * blockDim.x + threadIdx.x;
  uint8_t seed = 0;
  if (px < n) {
    const uint8_t f = flags[px];
    if (!(f & 1)) gidx[px] = make_int3(INT_MIN, 0, 0);  // no rank holds the pixel's block: not in the point map
    seed = (f >> 1) & 1;
    seed_out[px] = seed;
  }
  const unsigned ballot = __ballot_sync(0xffffffffu, seed != 0);  // n-tail threads stay in the warp (no early return)
  if (ballot && (threadIdx.x & 31) == (__ffs(ballot) - 1)) atomicAdd(&m.counters[kCtrSeeds], __popc(ballot));
}

// ---- E0: dense allocation (mesh_object_extractor.cpp:220-228) ----------------------------------------
__global__ void allocateBoxKernel(const DeviceMap m, int3 lo, int3 dims, int rank, int nranks, uint32_t born) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= dims.x * dims.y * dims.z) return;
  const int bx = lo.x + c % dims.x;
  c /= dims.x;
  const int by = lo.y + c % dims.y, bz = lo.z + c / dims.y;
  if (nranks > 1 && mapOwner(m, bx, by, bz, nranks) != rank) return;
  int created;
  hashFindOrInsert(m, bx, by, bz, born, &created);
}

// ---- K4: low-confidence erase (mesh_object_extractor.cpp:246-264, computeConfidence :342-356) -------
__global__ void __launch_bounds__(kThreads) scanConfidenceKernel(const DeviceMap m, float min_conf, float min_obs, float trunc) {
  const int slot = blockIdx.x;
  if (!(m.block_flags[slot] & kFlagAllocated)) return;
  const int V = m.V;
  const int sem = m.block_sem[slot];
  int erased = 0;
  for (int lin = threadIdx.x; lin < V; lin += kThreads) {
    float2 t = m.tsdf[static_cast<size_t>(slot) * V + lin];
    if (t.x > 0.f) continue;
    float conf = 0.f;  // empty voxel
    if (sem >= 0 && m.sem_label[static_cast<size_t>(sem) * V + lin] != kSemEmpty) {
      const float2 c = *reinterpret_cast<const float2*>(m.sem_lik + (static_cast<size_t>(sem) * V + lin) * 2);
      const float total = c.x + c.y;
      conf = total < min_obs ? -1.f : c.y / total;
    }
    if (conf < min_conf) {
      t.x = trunc;
      m.tsdf[static_cast<size_t>(slot) * V + lin] = t;
      ++erased;
    }
  }
  erased = warpSum(erased);
  if ((threadIdx.x & 31) == 0 && erased) atomicAdd(&m.counters[kCtrErased], erased);
}

// ---- export gathers -------------------------------------------------------------------------------------
__global__ void gatherTsdfKernel(const DeviceMap m, const int* slots, float* dist, float* weight) {
  const int V = m.V, slot = slots[blockIdx.x];
  for (int lin = threadIdx.x; lin < V; lin += blockDim.x) {
    const float2 t = m.tsdf[static_cast<size_t>(slot) * V + lin];
    dist[static_cast<size_t>(blockIdx.x) * V + lin] = t.x;
    weight[static_cast<size_t>(blockIdx.x) * V + lin] = t.y;
  }
}

__global__ void gatherTrackingKernel(const DeviceMap m, const TrackEval ev, const int* slots,
                                     const unsigned long long* stamps, unsigned long long* last_obs,
                                     unsigned long long* last_occ, uint8_t* ever_free, uint8_t* active,
                                     uint8_t* to_remove, uint8_t* block_active) {
  const int V = m.V, slot = slots[blockIdx.x];
  const uint32_t born = m.born_frame[slot];
  int any_active = 0;
  for (int lin = threadIdx.x; lin < V; lin += blockDim.x) {
    const size_t src = static_cast<size_t>(slot) * V + lin, dst = static_cast<size_t>(blockIdx.x) * V + lin;
    const uint8_t f = m.vflags[src];
    const uint32_t o = m.last_obs[src];
    uint32_t c;
    bool act, rem;
    evalTracking(m, ev, born, o, m.last_occ[src], f, &c, &act, &rem);
    last_obs[dst] = stamps[o];
    last_occ[dst] = stamps[c];
    ever_free[dst] = (f & kVoxEverFree) ? 1 : 0;
    active[dst] = act ? 1 : 0;
    to_remove[dst] = rem ? 1 : 0;
    any_active |= act ? 1 : 0;
  }
  any_active = __syncthreads_or(any_active);
  if (threadIdx.x == 0) {
    const bool seen = ev.k_last != 0 && ev.k_last >= born;
    block_active[blockIdx.x] = (seen && any_active && !(m.block_flags[slot] & kFlagInactiveOverride)) ? 1 : 0;
  }
}

__global__ void gatherColorKernel(const DeviceMap m, const int* slots, uint8_t* rgb) {
  const int V = m.V, slot = slots[blockIdx.x];
  for (int lin = threadIdx.x; lin < V; lin += blockDim.x) {
    const uchar4 c = m.color[static_cast<size_t>(slot) * V + lin];
    uint8_t* o = rgb + (static_cast<size_t>(blockIdx.x) * V + lin) * 3;
    o[0] = c.x; o[1] = c.y; o[2] = c.z;
  }
}

__global__ void gatherSemanticKernel(const DeviceMap m, const int* slots, int L, uint32_t* label,
                                     uint8_t* empty, float* lik) {
  const int V = m.V, slot = slots[blockIdx.x];
  const int sem = m.block_sem[slot];
  for (int lin = threadIdx.x; lin < V; lin += blockDim.x) {
    const size_t dst = static_cast<size_t>(blockIdx.x) * V + lin;
    uint16_t lb = kSemEmpty;
    if (sem >= 0) lb = m.sem_label[static_cast<size_t>(sem) * V + lin];
    const bool is_empty = lb == kSemEmpty;
    label[dst] = is_empty ? 0u : lb;
    empty[dst] = is_empty ? 1 : 0;
    if (lik) {
      for (int k = 0; k < L; ++k)
        lik[dst * L + k] = is_empty ? 0.f : m.sem_lik[(static_cast<size_t>(sem) * V + lin) * m.Lp + k];
    }
  }
}

}  // namespace

void launchExpandFrames(const BatchParams& p, cudaStream_t s) {
  expandFramesKernel<<<dim3(smCount(), p.n_frames), 256, 0, s>>>(p);
}
void launchExpandDepth(const uint16_t* src, float scale, float* dst, int n, cudaStream_t s) {
  expandDepthKernel<<<(n + 255) / 256, 256, 0, s>>>(src, scale, dst, n);
}
void launchTileMax(const BatchParams& p, cudaStream_t s) {
  bool vec4 = !p.compact_taps && (p.W % 4) == 0;
  for (int b = 0; b < p.n_frames && vec4; ++b) vec4 = (reinterpret_cast<uintptr_t>(p.f[b].depth) & 15u) == 0;
  if (vec4) {
    const int warps = ((p.W + 127) / 128) * p.lvl_ty[1];
    tileMaxVec4Kernel<<<dim3((warps + 7) / 8, p.n_frames), 256, 0, s>>>(p);
  } else {
    const int warps = ((p.W + 31) / 32) * p.lvl_ty[1];
    tileMaxKernel<<<dim3((warps + 7) / 8, p.n_frames), 256, 0, s>>>(p);
  }
  tilePyramidKernel<<<p.n_frames, 256, 0, s>>>(p);
}
void launchSelectBlocks(const DeviceMap& m, const BatchParams& p, int cull_grid, cudaStream_t s) {
  const int n = p.allocate ? p.dims[0] * p.dims[1] * p.dims[2] : p.n_slots;
  if (p.pipelined) selectBlocksKernel<true><<<(std::max(n, 1) + 3) / 4, 128, 0, s>>>(m, p);  // one warp per candidate
  else selectBlocksKernel<false><<<(std::max(n, 1) + 3) / 4, 128, 0, s>>>(m, p);
  if (p.cull) {
    if (m.vps == 16) itemCullKernel<16><<<cull_grid, 128, 0, s>>>(m, p);
    else itemCullKernel<8><<<cull_grid, 128, 0, s>>>(m, p);
  }
  if (p.item_list) {
    const bool pb = p.fetch_ctr == kCtrFetchB;
    cudaMemsetAsync(m.counters + (pb ? kCtrItemsB0 : kCtrItems0), 0, kItemClasses * sizeof(int), s);
    if (m.vps == 16) { if (pb) itemCompactKernel<16, true><<<cull_grid, 256, 0, s>>>(m, p); else itemCompactKernel<16, false><<<cull_grid, 256, 0, s>>>(m, p); }
    else { if (pb) itemCompactKernel<8, true><<<cull_grid, 256, 0, s>>>(m, p); else itemCompactKernel<8, false><<<cull_grid, 256, 0, s>>>(m, p); }
  }
}
// fuseKernel's and fuseKernelMlp's likelihood rows ([kFuseThreads][fuseRowStride(Lp)]; BINARY: [2][kFuseThreads])
static size_t fuseSmemBytes(int Lp) { return static_cast<size_t>(fuseRowStride(Lp)) * kFuseThreads * sizeof(float); }
// fuseKernelCoop: the folding warp's rows, then the weight, sdf and label tag of each (frame, voxel) of the item
static size_t fuseCoopSmemBytes(int Lp) {
  return static_cast<size_t>(fuseRowStride(Lp)) * 32 * sizeof(float) + 2 * 32 * 32 * sizeof(float) + 32 * 32;
}
int fuseBlocksPerSm(int vps, int Lp) {
  int n = 0;
  if (vps == 16) cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, fuseKernel<16, 1, false, false>, kFuseThreads, fuseSmemBytes(Lp));
  else cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, fuseKernel<8, 1, false, false>, kFuseThreads, fuseSmemBytes(Lp));
  return n > 0 ? n : 4;
}
// Calls f(std::integral_constant<int, V>{}) for the V of Vs that equals v: turns a launch flag into a template argument.
template <int... Vs, typename F>
static void withConstant(int v, F&& f) {
  (void)((v == Vs && (f(std::integral_constant<int, Vs>{}), true)) || ...);
}
void launchFuse(const DeviceMap& m, const BatchParams& p, int grid, cudaStream_t s) {
  if (grid <= 0) return;
  const bool col = p.has_color != 0 && m.color != nullptr, list = p.item_list != nullptr;
  // CTA-cooperative two-phase items (long listed batches); the memory-level-parallel experiment has no colour instantiation
  const bool coop = p.coop && list && p.layers_per_item == 1 && !col && p.mlp_group == 0;
  const int mlp = col || p.mlp_group == 0 ? 0 : (p.mlp_group == 2 ? 2 : 4);
  const size_t smem = fuseSmemBytes(m.Lp);
  withConstant<8, 16>(m.vps == 16 ? 16 : 8, [&](auto vps) {
    withConstant<0, 1>(p.compact_taps != 0, [&](auto compact) {
      withConstant<0, 1>(p.fetch_ctr == kCtrFetchB, [&](auto pb) {  // odd batch of KB_PIPELINE: second counter set
        constexpr int VPS = decltype(vps)::value;
        constexpr bool C = decltype(compact)::value, PB = decltype(pb)::value;
        if (coop) {
          fuseKernelCoop<VPS, C, PB><<<grid, kFuseThreads, fuseCoopSmemBytes(m.Lp), s>>>(m, p);
          return;
        }
        withConstant<1, 4>(p.layers_per_item == 1 ? 1 : 4, [&](auto lpi) {
          withConstant<0, 1>(list, [&](auto listed) {
            constexpr int LPI = decltype(lpi)::value;
            constexpr bool LIST = decltype(listed)::value;
            if (mlp) {
              withConstant<2, 4>(mlp, [&](auto g) {
                fuseKernelMlp<VPS, LPI, C, decltype(g)::value, LIST, PB><<<grid, kFuseThreads, smem, s>>>(m, p);
              });
            } else if (col) {
              fuseKernel<VPS, LPI, C, true, false, PB><<<grid, kFuseThreads, smem, s>>>(m, p);
            } else {
              fuseKernel<VPS, LPI, C, false, LIST, PB><<<grid, kFuseThreads, smem, s>>>(m, p);
            }
          });
        });
      });
    });
  });
}
void launchTrackingPass(const DeviceMap& m, const TrackingParams& p, int everfree_grid, cudaStream_t s) {
  trackingPassKernel<<<(std::max(p.n_slots, 1) + 255) / 256, 256, 0, s>>>(m, p);
  if (p.everfree_v2) everFreeKernelV2<false><<<everfree_grid, kThreads, 0, s>>>(m, p);
  else everFreeKernel<false><<<everfree_grid, kThreads, 0, s>>>(m, p);
  resetPendingKernel<<<1, 1, 0, s>>>(m);
}
void launchTrackingBegin(const DeviceMap& m, const TrackingParams& p, const ShardExchange& x, int32_t* pending_out, cudaStream_t s) {
  trackingPassKernel<<<(std::max(p.n_slots, 1) + 255) / 256, 256, 0, s>>>(m, p);
  exportPendingKernel<<<(x.cap_pending + 255) / 256, 256, 0, s>>>(m, p.pending, pending_out, x.cap_pending);
}
void launchHaloPack(const DeviceMap& m, const TrackingParams& p, const ShardExchange& x, const int32_t* all_pending,
                    int32_t* halo_out, cudaStream_t s) {
  const int n = x.nranks * x.cap_pending * 27;
  haloMarkKernel<<<(n + 255) / 256, 256, 0, s>>>(m, x, all_pending);
  haloPackKernel<<<smCount() * 4, kThreads, 0, s>>>(m, p, x, halo_out);
  haloUnmarkKernel<<<(m.max_blocks + 255) / 256, 256, 0, s>>>(m, x, m.max_blocks);
}
void launchTrackingBeginPeers(const DeviceMap& m, const TrackingParams& p, const ShardExchange& x, const PeerBuffers& peers, cudaStream_t s) {
  trackingPassKernel<<<(std::max(p.n_slots, 1) + 255) / 256, 256, 0, s>>>(m, p);
  exportPendingPeersKernel<<<(x.cap_pending + 255) / 256, 256, 0, s>>>(m, p.pending, peers, x.rank, x.pending_stride(), x.cap_pending);
}
void launchHaloPackPeers(const DeviceMap& m, const TrackingParams& p, const ShardExchange& x, const int32_t* all_pending,
                         const PeerBuffers& peers, cudaStream_t s) {
  const int n = x.nranks * x.cap_pending * 27;
  haloMarkKernel<<<(n + 255) / 256, 256, 0, s>>>(m, x, all_pending);
  haloPackPeersKernel<<<smCount() * 4, kThreads, 0, s>>>(m, p, x, peers);
  haloUnmarkKernel<<<(m.max_blocks + 255) / 256, 256, 0, s>>>(m, x, m.max_blocks);
}
void launchMulticastCopy(void* mc_dst, const void* src, size_t bytes, cudaStream_t s) {
  const size_t n16 = bytes / 16;
  if (n16 == 0) return;
  const int grid = static_cast<int>(std::min<size_t>((n16 + 255) / 256, static_cast<size_t>(smCount()) * 8));
  multicastCopyKernel<<<grid, 256, 0, s>>>(static_cast<float4*>(mc_dst), static_cast<const float4*>(src), n16);
}
void launchFlagScatter(const uint8_t* local_flags, const PeerBuffers& peers, int n, cudaStream_t s) {
  flagScatterKernel<<<(n + 255) / 256, 256, 0, s>>>(local_flags, peers, n);
}
void launchTrackingFinish(const DeviceMap& m, const TrackingParams& p, const ShardExchange& x, const int32_t* all_pending,
                          const int32_t* all_halo, int everfree_grid, cudaStream_t s) {
  cudaMemsetAsync(x.ghost_keys, 0xFF, (static_cast<size_t>(x.ghost_mask) + 1) * sizeof(unsigned long long), s);
  const int n = x.nranks * x.cap_halo;
  ghostBuildKernel<<<(n + 255) / 256, 256, 0, s>>>(m, x, all_pending, all_halo);
  if (p.everfree_v2) everFreeKernelV2<true><<<everfree_grid, kThreads, 0, s>>>(m, p);
  else everFreeKernel<true><<<everfree_grid, kThreads, 0, s>>>(m, p);
  resetPendingKernel<<<1, 1, 0, s>>>(m);
}
void launchResetInactive(const DeviceMap& m, const TrackEval& ev, int n, int3* removed, int max_removed, cudaStream_t s) {
  if (n > 0) resetInactiveKernel<<<n, kThreads, 0, s>>>(m, ev, removed, max_removed);
}
void launchRehash(const DeviceMap& m, int n, cudaStream_t s) {
  cudaMemsetAsync(m.hash_keys, 0xFF, (static_cast<size_t>(m.hash_mask) + 1) * sizeof(unsigned long long), s);
  rehashKernel<<<(std::max(n, 1) + 255) / 256, 256, 0, s>>>(m, n);
}
void launchMarkAllInactive(const DeviceMap& m, int n, cudaStream_t s) {
  if (n > 0) markAllInactiveKernel<<<(n + 255) / 256, 256, 0, s>>>(m, n);
}
void launchClearUpdated(const DeviceMap& m, int n, cudaStream_t s) {
  if (n > 0) clearUpdatedKernel<<<(n + 255) / 256, 256, 0, s>>>(m, n);
}
void launchMotionLookup(const DeviceMap& m, const MotionParams& p, cudaStream_t s) {
  const int n = p.W * p.H;
  motionLookupKernel<false><<<(n + 255) / 256, 256, 0, s>>>(m, p);
}
void launchMotionLookupLocal(const DeviceMap& m, const MotionParams& p, cudaStream_t s) {
  const int n = p.W * p.H;
  motionLookupKernel<true><<<(n + 255) / 256, 256, 0, s>>>(m, p);
}
void launchMotionFinalize(const DeviceMap& m, const uint8_t* flags, int3* gidx, uint8_t* seed, int n, cudaStream_t s) {
  motionFinalizeKernel<<<(n + 255) / 256, 256, 0, s>>>(m, flags, gidx, seed, n);
}
void launchAllocateBox(const DeviceMap& m, int3 lo, int3 dims, int rank, int nranks, uint32_t born, cudaStream_t s) {
  const int n = dims.x * dims.y * dims.z;
  if (n > 0) allocateBoxKernel<<<(n + 127) / 128, 128, 0, s>>>(m, lo, dims, rank, nranks, born);
}
void launchScanConfidence(const DeviceMap& m, float min_conf, float min_obs, float trunc, int n, cudaStream_t s) {
  if (n > 0) scanConfidenceKernel<<<n, kThreads, 0, s>>>(m, min_conf, min_obs, trunc);
}
void launchGatherTsdf(const DeviceMap& m, const int* slots, int n, float* dist, float* weight, cudaStream_t s) {
  if (n > 0) gatherTsdfKernel<<<n, 256, 0, s>>>(m, slots, dist, weight);
}
void launchGatherTracking(const DeviceMap& m, const TrackEval& ev, const int* slots, int n,
                          const unsigned long long* stamps, unsigned long long* last_obs,
                          unsigned long long* last_occ, uint8_t* ever_free, uint8_t* active, uint8_t* to_remove,
                          uint8_t* block_active, cudaStream_t s) {
  if (n > 0) gatherTrackingKernel<<<n, 256, 0, s>>>(m, ev, slots, stamps, last_obs, last_occ, ever_free, active, to_remove, block_active);
}
void launchGatherColor(const DeviceMap& m, const int* slots, int n, uint8_t* rgb, cudaStream_t s) {
  if (n > 0) gatherColorKernel<<<n, 256, 0, s>>>(m, slots, rgb);
}
void launchGatherSemantic(const DeviceMap& m, const int* slots, int n, int L, uint32_t* label, uint8_t* empty,
                          float* lik, cudaStream_t s) {
  if (n > 0) gatherSemanticKernel<<<n, 256, 0, s>>>(m, slots, L, label, empty, lik);
}

// ---- order-independent map checksum (kb_map_checksum) ----------------------------------------------------------
// One CTA per pool slot; every voxel of every allocated block contributes
//   v = mix64(mix64(mix64(mix64(packKey(block) ^ mix64(lin + 1)) ^ (distance bits | weight bits << 32)) ^ label) ^ stamp)
// (label = semantic_label, 0xFFFFFFFF when empty / no semantic layer; stamp = last_observed in ns, 0 = never) to a
// wrapping 64-bit sum and an xor; out[2] counts blocks, out[3] voxels observed at least once. The same function over
// a kb_block_export is tests/harness.py::map_checksum.
namespace {
__global__ void __launch_bounds__(256) checksumKernel(const DeviceMap m, int n_slots, const unsigned long long* __restrict__ stamps,
                                                      unsigned long long* __restrict__ out) {
  const int slot = blockIdx.x;
  if (slot >= n_slots || !(m.block_flags[slot] & kFlagAllocated)) return;
  const int3 bi = m.block_index[slot];
  const unsigned long long key = packKey(bi.x, bi.y, bi.z);
  const int sem = m.block_sem[slot];
  unsigned long long sum = 0, xr = 0, seen = 0;
  for (int lin = threadIdx.x; lin < m.V; lin += blockDim.x) {
    const size_t gi = static_cast<size_t>(slot) * m.V + lin;
    const float2 st = m.tsdf[gi];
    uint32_t label = 0xFFFFFFFFu;
    if (sem >= 0 && m.sem_label) {
      const uint16_t lb = m.sem_label[static_cast<size_t>(sem) * m.V + lin];
      if (lb != kSemEmpty) label = lb;
    }
    const unsigned long long stamp = m.last_obs ? stamps[m.last_obs[gi]] : 0ull;
    unsigned long long v = mix64(key ^ mix64(static_cast<unsigned long long>(lin) + 1ull));
    v = mix64(v ^ (static_cast<unsigned long long>(__float_as_uint(st.x)) | (static_cast<unsigned long long>(__float_as_uint(st.y)) << 32)));
    v = mix64(v ^ static_cast<unsigned long long>(label));
    v = mix64(v ^ stamp);
    sum += v;
    xr ^= v;
    seen += (stamp != 0ull || st.y > 0.f) ? 1ull : 0ull;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    sum += __shfl_xor_sync(0xffffffffu, sum, o);
    xr ^= __shfl_xor_sync(0xffffffffu, xr, o);
    seen += __shfl_xor_sync(0xffffffffu, seen, o);
  }
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(&out[0], sum);
    atomicXor(&out[1], xr);
    atomicAdd(&out[3], seen);
  }
  if (threadIdx.x == 0) atomicAdd(&out[2], 1ull);
}
}  // namespace

void launchChecksum(const DeviceMap& m, int n_slots, const unsigned long long* stamps, unsigned long long* out, cudaStream_t s) {
  if (n_slots > 0) checksumKernel<<<n_slots, 256, 0, s>>>(m, n_slots, stamps, out);
}


}  // namespace kb
