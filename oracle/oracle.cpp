// TEST INFRASTRUCTURE — NOT PRODUCT CODE. See oracle.hpp. PARITY UNPINNED (no reference tests).
// Compile with -ffp-contract=off: every float expression below is evaluated op by op in fp32.
#include "oracle.hpp"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <map>
#include <set>
#include <mutex>
#include <thread>

namespace ko {

namespace {

inline double toSeconds(uint64_t ns) { return static_cast<double>(ns) / 1e9; }  // UP App. A.2 [M]

inline int floorDiv(int64_t a, int64_t b) {
  int64_t q = a / b, r = a % b;
  if (r != 0 && ((r < 0) != (b < 0))) --q;
  return static_cast<int>(q);
}

template <typename F>
void parallelFor(int n, int num_threads, F&& fn) {
  // Same model as hydra::IndexGetter + std::thread workers (tracking_integrator.cpp:83-90): a shared
  // cursor hands out block indices.
  num_threads = std::max(1, std::min(num_threads, n));
  if (num_threads == 1) {
    for (int i = 0; i < n; ++i) fn(i);
    return;
  }
  std::atomic<int> cursor{0};
  std::vector<std::thread> threads;
  for (int t = 0; t < num_threads; ++t) {
    threads.emplace_back([&]() {
      int i;
      while ((i = cursor.fetch_add(1)) < n) fn(i);
    });
  }
  for (auto& t : threads) t.join();
}

int resolveThreads(int n) {
  if (n > 0) return n;
  int hc = static_cast<int>(std::thread::hardware_concurrency());
  return hc > 0 ? hc : 1;  // ThreadNumConversion: -1 => hardware concurrency (tracking_integrator.cpp:59)
}

// spatial_hash::NeighborSearch offsets (UP App. A.1): 6 faces, +12 edges (18), +8 corners (26).
std::vector<std::array<int, 3>> neighborOffsets(int connectivity) {
  std::vector<std::array<int, 3>> out;
  for (int pass = 1; pass <= 3; ++pass) {
    if ((pass == 2 && connectivity < 18) || (pass == 3 && connectivity < 26)) break;
    for (int dz = -1; dz <= 1; ++dz)
      for (int dy = -1; dy <= 1; ++dy)
        for (int dx = -1; dx <= 1; ++dx) {
          int nz = (dx != 0) + (dy != 0) + (dz != 0);
          if (nz == pass) out.push_back({dx, dy, dz});
        }
  }
  return out;
}

}  // namespace

Oracle::Oracle(const kb_map_config& map, const kb_integrator_config& integ,
               const kb_tracking_config* trk, const kb_motion_config* mot)
    : map_(map), integ_(integ) {
  if (trk) { trk_ = *trk; has_trk_ = true; }
  if (mot) { mot_ = *mot; has_mot_ = true; }
  vps_ = map.voxels_per_side;
  V_ = vps_ * vps_ * vps_;
  L_ = integ.semantic_mode == KB_SEMANTICS_MLE ? integ.num_labels
       : integ.semantic_mode == KB_SEMANTICS_BINARY ? 2 : 0;
  if (!map.with_semantics) L_ = 0;
  block_size_ = map.voxel_size * static_cast<float>(vps_);
  voxel_size_inv_ = 1.f / map.voxel_size;
  block_size_inv_ = 1.f / block_size_;
  if (integ.semantic_mode == KB_SEMANTICS_MLE && integ.num_labels > 1) {
    // MLESemanticIntegrator (UP App. A.8): log-likelihood matrix with diag log(c), off-diag
    // log((1-c)/(N-1)); prior log(1/N). Constants are formed in double and rounded once to float.
    const double c = static_cast<double>(integ.label_confidence);
    const double N = static_cast<double>(integ.num_labels);
    mle_diag_ = static_cast<float>(std::log(c));
    mle_off_ = static_cast<float>(std::log((1.0 - c) / (N - 1.0)));
    mle_init_ = static_cast<float>(std::log(1.0 / N));
  }
  if (vps_ != 8 && vps_ != 16) error_ = "voxels_per_side must be 8 or 16";
  if (!(map.voxel_size > 0) || !(map.truncation_distance > 0)) error_ = "invalid map config";
}

Block* Oracle::getBlock(const Idx3& idx) const {
  auto it = blocks_.find(idx);
  return it == blocks_.end() ? nullptr : it->second.get();
}

Block* Oracle::allocateBlock(const Idx3& idx) {
  auto it = blocks_.find(idx);
  if (it != blocks_.end()) return it->second.get();
  auto b = std::make_unique<Block>();
  b->index = idx;
  b->distance.assign(V_, 0.f);
  b->weight.assign(V_, 0.f);
  b->color.assign(3 * V_, 0);
  if (map_.with_tracking) {
    b->last_observed.assign(V_, 0);
    b->last_occupied.assign(V_, 0);
    b->ever_free.assign(V_, 0);
    b->active.assign(V_, 0);     // TrackingVoxel::active default [L]: false
    b->to_remove.assign(V_, 0);
  }
  if (L_ > 0) {
    b->semantic_label.assign(V_, 0);
    b->semantic_empty.assign(V_, 1);
    // likelihoods are sized on the block's first semantic update (hydra sizes each voxel's VectorXf
    // on its first update, App. A.8) — keeps block allocation cheap like the reference.
  }
  Block* raw = b.get();
  blocks_.emplace(idx, std::move(b));
  return raw;
}

// ---- camera (hydra::Camera, UP App. A.3) -------------------------------------------------------

bool Oracle::project(const float p[3], float* u, float* v) const {
  if (p[2] <= 0.f) return false;
  *u = cam_.fx * p[0] / p[2] + cam_.cx;
  *v = cam_.fy * p[1] / p[2] + cam_.cy;
  if (*u < 0.f || *u > static_cast<float>(cam_.width - 1) || *v < 0.f ||
      *v > static_cast<float>(cam_.height - 1)) {
    return false;
  }
  return true;
}

bool Oracle::pointInFrustum(const float p[3], float infl) const {
  if (p[2] < -infl) return false;
  const float r = std::sqrt((p[0] * p[0] + p[1] * p[1]) + p[2] * p[2]);
  if (r < cam_.min_range - infl || r > cam_.max_range + infl) return false;
  // Four side planes through the optical centre, inward unit normals, offset by the inflation.
  const float xl = (0.f - cam_.cx) / cam_.fx;
  const float xr = (static_cast<float>(cam_.width - 1) - cam_.cx) / cam_.fx;
  const float yt = (0.f - cam_.cy) / cam_.fy;
  const float yb = (static_cast<float>(cam_.height - 1) - cam_.cy) / cam_.fy;
  const float il = 1.f / std::sqrt(1.f + xl * xl), ir = 1.f / std::sqrt(1.f + xr * xr);
  const float it = 1.f / std::sqrt(1.f + yt * yt), ib = 1.f / std::sqrt(1.f + yb * yb);
  if (il * p[0] + (-xl * il) * p[2] < -infl) return false;
  if ((-ir) * p[0] + (xr * ir) * p[2] < -infl) return false;
  if (it * p[1] + (-yt * it) * p[2] < -infl) return false;
  if ((-ib) * p[1] + (yb * ib) * p[2] < -infl) return false;
  return true;
}

// ---- interpolators (hydra ProjectionInterpolator*, UP App. A.7) ------------------------------------

Oracle::Weights Oracle::computeWeights(float u, float v, const float* range) const {
  Weights w;
  const int W = cam_.width, H = cam_.height;
  auto nearest = [&]() {
    Weights n;
    n.u = static_cast<int>(std::round(u));
    n.v = static_cast<int>(std::round(v));
    n.bilinear = false;
    n.valid = n.u >= 0 && n.u < W && n.v >= 0 && n.v < H && range[n.v * W + n.u] > 0.f;
    return n;
  };
  if (integ_.interpolation_method == KB_INTERP_NEAREST) return nearest();
  const int u0 = static_cast<int>(std::floor(u)), v0 = static_cast<int>(std::floor(v));
  const bool inside = u0 >= 0 && v0 >= 0 && u0 + 1 < W && v0 + 1 < H;
  if (!inside) {
    return integ_.interpolation_method == KB_INTERP_ADAPTIVE ? nearest() : w;  // bilinear: invalid
  }
  // Neighbour order (u,v), (u,v+1), (u+1,v), (u+1,v+1).
  const float r0 = range[v0 * W + u0], r1 = range[(v0 + 1) * W + u0];
  const float r2 = range[v0 * W + u0 + 1], r3 = range[(v0 + 1) * W + u0 + 1];
  const bool all_valid = r0 > 0.f && r1 > 0.f && r2 > 0.f && r3 > 0.f;
  if (integ_.interpolation_method == KB_INTERP_ADAPTIVE) {
    const float mx = std::max(std::max(r0, r1), std::max(r2, r3));
    const float mn = std::min(std::min(r0, r1), std::min(r2, r3));
    if (!all_valid || !(mx - mn < integ_.adaptive_max_depth_difference)) return nearest();
  } else if (!all_valid) {
    return w;
  }
  const float du = u - static_cast<float>(u0), dv = v - static_cast<float>(v0);
  w.valid = true;
  w.bilinear = true;
  w.u = u0;
  w.v = v0;
  w.w[0] = (1.f - du) * (1.f - dv);
  w.w[1] = (1.f - du) * dv;
  w.w[2] = du * (1.f - dv);
  w.w[3] = du * dv;
  return w;
}

float Oracle::interpolateRange(const float* range, const Weights& w) const {
  const int W = cam_.width;
  if (!w.bilinear) return range[w.v * W + w.u];
  return ((w.w[0] * range[w.v * W + w.u] + w.w[1] * range[(w.v + 1) * W + w.u]) +
          w.w[2] * range[w.v * W + w.u + 1]) +
         w.w[3] * range[(w.v + 1) * W + w.u + 1];
}

int32_t Oracle::interpolateID(const int32_t* img, const Weights& w) const {
  const int W = cam_.width;
  if (!w.bilinear) return img[w.v * W + w.u];
  int best = 0;  // value at the neighbour with the largest weight; ties -> lowest neighbour index
  for (int i = 1; i < 4; ++i) {
    if (w.w[i] > w.w[best]) best = i;
  }
  const int du = best >> 1, dv = best & 1;
  return img[(w.v + dv) * W + w.u + du];
}

void Oracle::interpolateColor(const uint8_t* rgb, const Weights& w, uint8_t out[3]) const {
  const int W = cam_.width;
  const uint8_t* p0 = rgb + (static_cast<size_t>(w.v) * W + w.u) * 3;
  if (!w.bilinear) {
    out[0] = p0[0]; out[1] = p0[1]; out[2] = p0[2];
    return;
  }
  const uint8_t* p1 = p0 + static_cast<size_t>(W) * 3;  // (u, v+1)
  const uint8_t* p2 = p0 + 3;                            // (u+1, v)
  const uint8_t* p3 = p1 + 3;                            // (u+1, v+1)
  for (int ch = 0; ch < 3; ++ch) {
    const float s = ((w.w[0] * static_cast<float>(p0[ch]) + w.w[1] * static_cast<float>(p1[ch])) +
                     w.w[2] * static_cast<float>(p2[ch])) + w.w[3] * static_cast<float>(p3[ch]);
    out[ch] = static_cast<uint8_t>(static_cast<int>(s));
  }
}

float Oracle::computeWeight(float depth, float sdf) const {
  // UP App. A.6 step 4: ray density fx*fy*vs^2/z^2, optional 1/z^2, linear drop-off behind surface.
  const float vs = map_.voxel_size;
  float weight = (cam_.fx * cam_.fy) * (vs * vs) / (depth * depth);
  if (!integ_.use_constant_weight) weight = weight / (depth * depth);
  if (integ_.use_weight_dropoff) {
    const float eps = integ_.weight_dropoff_epsilon > 0.f ? integ_.weight_dropoff_epsilon
                                                          : integ_.weight_dropoff_epsilon * -vs;
    if (sdf < -eps) {
      weight = weight * ((map_.truncation_distance + sdf) / (map_.truncation_distance - eps));
      weight = std::max(weight, 0.f);
    }
  }
  return weight;
}

// ---- K0 + K1 ---------------------------------------------------------------------------------------

static void invertPose(const double T[16], float R[9], float t[3], float Rw[9], float tw[3]) {
  // sensor_T_world = world_T_sensor^-1 for a rigid transform, formed in double, rounded once to float.
  double Rd[9], td[3];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) Rd[r * 3 + c] = T[c * 4 + r];
  for (int r = 0; r < 3; ++r)
    td[r] = -(Rd[r * 3 + 0] * T[3] + Rd[r * 3 + 1] * T[7] + Rd[r * 3 + 2] * T[11]);
  for (int i = 0; i < 9; ++i) R[i] = static_cast<float>(Rd[i]);
  for (int i = 0; i < 3; ++i) t[i] = static_cast<float>(td[i]);
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) Rw[r * 3 + c] = static_cast<float>(T[r * 4 + c]);
    tw[r] = static_cast<float>(T[r * 4 + 3]);
  }
}

static inline void transform(const float R[9], const float t[3], const float p[3], float out[3]) {
  out[0] = ((R[0] * p[0] + R[1] * p[1]) + R[2] * p[2]) + t[0];
  out[1] = ((R[3] * p[0] + R[4] * p[1]) + R[5] * p[2]) + t[1];
  out[2] = ((R[6] * p[0] + R[7] * p[1]) + R[8] * p[2]) + t[2];
}

int Oracle::owner(const Idx3& b) const {
  if (cell_ <= 0) return blockOwner(b, nranks_);
  if (!table_.empty()) {
    auto fdiv = [](int a, int c) { return (a >= 0 ? a : a - c + 1) / c; };
    const int cx = fdiv(b.x, cell_) - tab_ox_, cy = fdiv(b.y, cell_) - tab_oy_;
    if (cx >= 0 && cx < tab_w_ && cy >= 0 && cy < tab_h_) return table_[static_cast<size_t>(cy) * tab_w_ + cx] % nranks_;
  }
  return cellOwner(b.x, b.y, cell_, gx_, gy_, nranks_);
}

void Oracle::setShardTable(int rank, int nranks, int cell, int ox, int oy, int w, int h, const uint8_t* owners) {
  rank_ = rank; nranks_ = nranks; cell_ = cell;
  int gy = 1;
  for (int g = 1; g * g <= nranks; ++g) if (nranks % g == 0) gy = g;  // same fallback tiling as the product
  gy_ = gy; gx_ = nranks / gy;
  table_.assign(owners, owners + static_cast<size_t>(w) * h);
  tab_ox_ = ox; tab_oy_ = oy; tab_w_ = w; tab_h_ = h;
}

void Oracle::frameCells(const kb_frame& f, int cell, int ox, int oy, int w, int h, uint8_t* touched) const {
  float R[9], t[3], Rw[9], tw[3];
  invertPose(f.world_T_sensor, R, t, Rw, tw);
  const float infl = block_size_ * 0.8660254f;
  const float reach = cam_.max_range + infl;
  int lo[3], hi[3];
  for (int a = 0; a < 3; ++a) {
    lo[a] = static_cast<int>(std::floor((tw[a] - reach) * block_size_inv_));
    hi[a] = static_cast<int>(std::floor((tw[a] + reach) * block_size_inv_));
  }
  auto fdiv = [](int a, int c) { return (a >= 0 ? a : a - c + 1) / c; };
  for (int bz = lo[2]; bz <= hi[2]; ++bz)
    for (int by = lo[1]; by <= hi[1]; ++by)
      for (int bx = lo[0]; bx <= hi[0]; ++bx) {
        const int cx = fdiv(bx, cell) - ox, cy = fdiv(by, cell) - oy;
        if (cx < 0 || cx >= w || cy < 0 || cy >= h || touched[static_cast<size_t>(cy) * w + cx]) continue;
        const float c[3] = {(static_cast<float>(bx) + 0.5f) * block_size_, (static_cast<float>(by) + 0.5f) * block_size_,
                            (static_cast<float>(bz) + 0.5f) * block_size_};
        float cC[3];
        transform(R, t, c, cC);
        if (pointInFrustum(cC, infl)) touched[static_cast<size_t>(cy) * w + cx] = 1;
      }
}

// kb_frame_owners on the oracle: the exact frustum selection of integrateFrame (no safety inflation), reduced to the set
// of owner ranks. The product's mask must be a superset.
uint32_t Oracle::frameOwners(const kb_frame& f) const {
  float R[9], t[3], Rw[9], tw[3];
  invertPose(f.world_T_sensor, R, t, Rw, tw);
  const float infl = block_size_ * 0.8660254f;
  const float reach = cam_.max_range + infl;
  int lo[3], hi[3];
  for (int a = 0; a < 3; ++a) {
    lo[a] = static_cast<int>(std::floor((tw[a] - reach) * block_size_inv_));
    hi[a] = static_cast<int>(std::floor((tw[a] + reach) * block_size_inv_));
  }
  uint32_t mask = 0;
  for (int bz = lo[2]; bz <= hi[2]; ++bz)
    for (int by = lo[1]; by <= hi[1]; ++by)
      for (int bx = lo[0]; bx <= hi[0]; ++bx) {
        const float c[3] = {(static_cast<float>(bx) + 0.5f) * block_size_, (static_cast<float>(by) + 0.5f) * block_size_,
                            (static_cast<float>(bz) + 0.5f) * block_size_};
        float cC[3];
        transform(R, t, c, cC);
        if (!pointInFrustum(cC, infl)) continue;
        mask |= 1u << (nranks_ > 1 ? owner(Idx3{bx, by, bz}) : 0);
      }
  return mask;
}

void Oracle::integrateFrame(const kb_frame& f, bool allocate_blocks, kb_frame_stats* stats) {
  if (!has_cam_) { error_ = "camera not set"; return; }
  if (f.stamp_ns == 0) { error_ = "stamp must be > 0"; return; }
  float R[9], t[3], Rw[9], tw[3];
  invertPose(f.world_T_sensor, R, t, Rw, tw);

  std::vector<Block*> todo;
  int n_new = 0;
  if (allocate_blocks) {
    // findBlocksInViewFrustum (UP App. A.5): block centres inside the frustum inflated by the block
    // half-diagonal, within [min_range, max_range].
    const float infl = block_size_ * 0.8660254f;
    const float reach = cam_.max_range + infl;
    int lo[3], hi[3];
    for (int a = 0; a < 3; ++a) {
      lo[a] = static_cast<int>(std::floor((tw[a] - reach) * block_size_inv_));
      hi[a] = static_cast<int>(std::floor((tw[a] + reach) * block_size_inv_));
    }
    for (int bz = lo[2]; bz <= hi[2]; ++bz)
      for (int by = lo[1]; by <= hi[1]; ++by)
        for (int bx = lo[0]; bx <= hi[0]; ++bx) {
          const float c[3] = {(static_cast<float>(bx) + 0.5f) * block_size_,
                              (static_cast<float>(by) + 0.5f) * block_size_,
                              (static_cast<float>(bz) + 0.5f) * block_size_};
          float cC[3];
          transform(R, t, c, cC);
          if (!pointInFrustum(cC, infl)) continue;
          const Idx3 idx{bx, by, bz};
          if (nranks_ > 1 && owner(idx) != rank_) continue;  // block-hash / cell shard (§8e)
          if (!getBlock(idx)) ++n_new;
          todo.push_back(allocateBlock(idx));
        }
  } else {
    for (auto& kv : blocks_) todo.push_back(kv.second.get());
  }

  std::atomic<int> counters[4];
  for (auto& c : counters) c = 0;
  parallelFor(static_cast<int>(todo.size()), resolveThreads(integ_.num_threads),
              [&](int i) { updateBlock(*todo[i], f, R, t, counters); });
  if (stats) {
    stats->blocks_in_frustum = static_cast<int>(todo.size());
    stats->blocks_allocated = n_new;
    stats->blocks_updated = counters[0];
    stats->voxels_updated = counters[1];
    stats->voxels_in_band = counters[2];
    stats->voxels_semantic = counters[3];
    stats->total_blocks = static_cast<int>(blocks_.size());
    stats->capacity_exceeded = 0;
  }
}

void Oracle::updateBlock(Block& b, const kb_frame& f, const float R[9], const float t[3],
                         std::atomic<int>* counters) {
  // ProjectiveIntegrator::updateBlock / getVoxelMeasurement / computeLabel / updateVoxel
  // (UP App. A.6; computeLabel structure pinned by object_integrator.cpp:58-81).
  const float vs = map_.voxel_size, trunc = map_.truncation_distance;
  const float ox = static_cast<float>(b.index.x) * block_size_;
  const float oy = static_cast<float>(b.index.y) * block_size_;
  const float oz = static_cast<float>(b.index.z) * block_size_;
  const bool binary = integ_.semantic_mode == KB_SEMANTICS_BINARY;
  const bool has_sem = L_ > 0 && (binary ? f.object_image != nullptr : f.label != nullptr);
  int n_valid = 0, n_band = 0, n_sem = 0;
  for (int lin = 0; lin < V_; ++lin) {
    const int vx = lin % vps_, vy = (lin / vps_) % vps_, vz = lin / (vps_ * vps_);
    const float pW[3] = {ox + (static_cast<float>(vx) + 0.5f) * vs,
                         oy + (static_cast<float>(vy) + 0.5f) * vs,
                         oz + (static_cast<float>(vz) + 0.5f) * vs};
    float pC[3];
    transform(R, t, pW, pC);
    // 1. interpolatePoint
    float u, v;
    if (!project(pC, &u, &v)) continue;
    const Weights w = computeWeights(u, v, f.depth);
    if (!w.valid) continue;
    // 2. sdf
    const float depth = pC[2];
    const float sdf = interpolateRange(f.depth, w) - depth;
    if (sdf < -trunc) continue;
    // 3. computeLabel
    const bool in_band = std::fabs(sdf) < trunc;
    uint32_t label = 0;
    bool have_label = false;
    if (in_band) {
      if (f.mask && interpolateID(f.mask, w) != 0) continue;
      if (has_sem) {
        if (binary) {
          label = interpolateID(f.object_image, w) == f.object_target_id ? 1u : 0u;
          have_label = true;
        } else {
          label = static_cast<uint32_t>(interpolateID(f.label, w));
          // SemanticIntegrator::canIntegrate: dynamic / invalid labels are not integrated at all.
          if (label < static_cast<uint32_t>(KB_MAX_LABELS) && integ_.label_blocked[label]) continue;
          have_label = true;
        }
      }
    }
    // 4. weight
    const float wm = computeWeight(depth, sdf);
    // updateVoxel
    const float d_old = b.distance[lin], w_old = b.weight[lin];
    const float sdf_c = std::min(std::max(sdf, -trunc), trunc);
    b.distance[lin] = (d_old * w_old + sdf_c * wm) / (w_old + wm);
    b.weight[lin] = std::min(w_old + wm, integ_.max_weight);
    if (map_.with_tracking) b.last_observed[lin] = f.stamp_ns;
    ++n_valid;
    if (!in_band) continue;
    ++n_band;
    // colour (UP App. A.6 step 5 / updateVoxel): only near the surface, only with a colour image.
    // interpolateColor: nearest -> that pixel; bilinear -> per channel ((w0 c0 + w1 c1) + w2 c2) + w3 c3,
    // truncated to u8. Color::merge with ratio = w_m / (w_old + w_m): c = u8(c (1 - ratio) + c_m ratio).
    if (f.color) {
      uint8_t cm[3];
      interpolateColor(f.color, w, cm);
      const float tot = w_old + wm;
      const float ratio = tot > 0.f ? wm / tot : 0.f;
      for (int ch = 0; ch < 3; ++ch) {
        uint8_t& c = b.color[static_cast<size_t>(lin) * 3 + ch];
        c = static_cast<uint8_t>(static_cast<int>(static_cast<float>(c) * (1.f - ratio) + static_cast<float>(cm[ch]) * ratio));
      }
    }
    if (have_label && label < static_cast<uint32_t>(L_)) {  // isValidLabel
      if (b.likelihoods.empty()) b.likelihoods.assign(static_cast<size_t>(V_) * L_, 0.f);
      float* lik = &b.likelihoods[static_cast<size_t>(lin) * L_];
      if (b.semantic_empty[lin]) {
        b.semantic_empty[lin] = 0;
        for (int k = 0; k < L_; ++k) lik[k] = binary ? 0.f : mle_init_;
      }
      if (binary) {
        lik[label] = lik[label] + 1.f;
      } else {
        for (int k = 0; k < L_; ++k)
          lik[k] = lik[k] + (static_cast<uint32_t>(k) == label ? mle_diag_ : mle_off_);
      }
      int best = 0;
      for (int k = 1; k < L_; ++k)
        if (lik[k] > lik[best]) best = k;
      b.semantic_label[lin] = static_cast<uint32_t>(best);
      ++n_sem;
    }
  }
  if (n_valid > 0) {
    b.updated = b.mesh_updated = b.esdf_updated = b.tracking_updated = true;  // setUpdated()
    counters[0] += 1;
    counters[1] += n_valid;
    counters[2] += n_band;
    counters[3] += n_sem;
  }
}

// ---- K2 / K3 / K2r -----------------------------------------------------------------------------------

bool Oracle::voxelIsFree(const Block& b, int lin, uint64_t stamp) const {
  // tracking_integrator.cpp:248-252 (uses temporal_buffer; burn_in_period is unused by the reference).
  return toSeconds(b.last_occupied[lin]) < toSeconds(stamp) - trk_.temporal_buffer &&
         b.last_observed[lin] != 0u;
}

void Oracle::updateBlockTracking(Block& b, uint64_t stamp, float thr) {
  // tracking_integrator.cpp:133-166 + updateTrackingDuration :224-246.
  b.tracking_updated = false;
  bool any_active = false;
  for (int lin = 0; lin < V_; ++lin) {
    if (b.distance[lin] < thr) b.last_occupied[lin] = stamp;
    const bool was_active = b.active[lin] != 0;
    const bool now_active =
        toSeconds(b.last_observed[lin]) >= toSeconds(stamp) - trk_.temporal_window;
    b.active[lin] = now_active;
    if (was_active && !now_active) b.to_remove[lin] = 1;
    any_active = any_active || now_active;
  }
  b.has_active_data = any_active;
}

void Oracle::updateBlockEverFree(const Block& b, uint64_t stamp, std::vector<int>* to_set, const GhostMap* ghosts) const {
  // tracking_integrator.cpp:168-222. The reference writes ever_free while other threads read it; the
  // outcome is order independent because a neighbour that became ever-free during this pass
  // necessarily satisfies voxelIsFree at this stamp. We therefore evaluate every voxel against the
  // pre-pass flags ("neighbour ever_free OR neighbour free now") and apply the writes afterwards,
  // which is race free and gives the identical result.
  const auto offs = neighborOffsets(trk_.neighbor_connectivity);
  for (int lin = 0; lin < V_; ++lin) {
    if (b.ever_free[lin] || !voxelIsFree(b, lin, stamp)) continue;
    const int vx = lin % vps_, vy = (lin / vps_) % vps_, vz = lin / (vps_ * vps_);
    bool blocked = false;
    for (const auto& o : offs) {
      int nx = vx + o[0], ny = vy + o[1], nz = vz + o[2];
      Idx3 nb = b.index;
      if (nx < 0) { nx += vps_; --nb.x; } else if (nx >= vps_) { nx -= vps_; ++nb.x; }
      if (ny < 0) { ny += vps_; --nb.y; } else if (ny >= vps_) { ny -= vps_; ++nb.y; }
      if (nz < 0) { nz += vps_; --nb.z; } else if (nz >= vps_) { nz -= vps_; ++nb.z; }
      const Block* nblk = (nb == b.index) ? &b : getBlock(nb);
      const int nlin = nx + vps_ * (ny + vps_ * nz);
      if (!nblk && ghosts) {  // sharded: the neighbour block lives on another rank, which published this predicate
        auto git = ghosts->find(nb);
        if (git != ghosts->end()) {
          if ((git->second[nlin >> 5] >> (nlin & 31)) & 1u) continue;
          blocked = true;
          break;
        }
      }
      if (!nblk) { blocked = true; break; }  // :198-202 missing neighbour block
      if (nblk->ever_free[nlin]) continue;
      if (!voxelIsFree(*nblk, nlin, stamp)) { blocked = true; break; }
    }
    if (!blocked) to_set->push_back(lin);
  }
}

std::vector<Block*> Oracle::trackingPassLocal(uint64_t stamp) {
  // tracking_integrator.cpp:71-104: all blocks get the tracking pass, then blocks whose TSDF was
  // updated this frame get the ever-free pass.
  std::vector<Block*> all, updated;
  for (auto& kv : blocks_) {
    all.push_back(kv.second.get());
    if (kv.second->tracking_updated) updated.push_back(kv.second.get());
  }
  const float thr = trk_.tsdf_occupancy_threshold < 0
                        ? trk_.tsdf_occupancy_threshold * -map_.voxel_size
                        : trk_.tsdf_occupancy_threshold;
  const int nt = resolveThreads(trk_.num_threads);
  parallelFor(static_cast<int>(all.size()), nt, [&](int i) { updateBlockTracking(*all[i], stamp, thr); });
  return updated;
}

void Oracle::applyEverFree(const std::vector<Block*>& updated, uint64_t stamp, const GhostMap* ghosts) {
  const int nt = resolveThreads(trk_.num_threads);
  std::vector<std::vector<int>> to_set(updated.size());
  parallelFor(static_cast<int>(updated.size()), nt,
              [&](int i) { updateBlockEverFree(*updated[i], stamp, &to_set[i], ghosts); });
  for (size_t i = 0; i < updated.size(); ++i)
    for (int lin : to_set[i]) updated[i]->ever_free[lin] = 1;
}

void Oracle::updateTracking(uint64_t stamp) {
  if (!has_trk_ || !map_.with_tracking) { error_ = "tracking not configured"; return; }
  const std::vector<Block*> updated = trackingPassLocal(stamp);
  applyEverFree(updated, stamp, nullptr);
}

// ---- sharded K2/K3 (buffer layouts: csrc/kb_kernels.cuh ShardExchange) ---------------------------------

static inline uint64_t shardMix64(uint64_t k) {
  k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
  return k;
}

int Oracle::blockOwner(const Idx3& b, int nranks) {
  // restates csrc/kb_device.cuh packKey/blockOwner: 21-bit biased coordinates, upper hash bits modulo nranks
  if (nranks <= 1) return 0;
  const uint64_t o = 1ull << 20, m = (1ull << 21) - 1ull;
  const uint64_t key = ((static_cast<uint64_t>(static_cast<int64_t>(b.x) + static_cast<int64_t>(o)) & m)) |
                       ((static_cast<uint64_t>(static_cast<int64_t>(b.y) + static_cast<int64_t>(o)) & m) << 21) |
                       ((static_cast<uint64_t>(static_cast<int64_t>(b.z) + static_cast<int64_t>(o)) & m) << 42);
  return static_cast<int>((shardMix64(key) >> 40) % static_cast<uint64_t>(nranks));
}

int Oracle::cellOwner(int bx, int by, int cell, int gx, int gy, int nranks) {
  // restates csrc/kb_device.cuh cellOwner: floor division into cells, periodic gx x gy tiling
  if (nranks <= 1 || cell < 1) return 0;
  auto fdiv = [](int a, int b) { return (a >= 0 ? a : a - b + 1) / b; };
  const int cx = fdiv(bx, cell), cy = fdiv(by, cell);
  const int mx = ((cx % gx) + gx) % gx, my = ((cy % gy) + gy) % gy;
  return (mx + gx * my) % nranks;
}

void Oracle::trackingBegin(uint64_t stamp, int32_t* out, int cap) {
  if (!has_trk_ || !map_.with_tracking) { error_ = "tracking not configured"; return; }
  open_pending_ = trackingPassLocal(stamp);
  std::sort(open_pending_.begin(), open_pending_.end(), [](const Block* a, const Block* b) { return a->index < b->index; });
  open_stamp_ = stamp;
  const int n = static_cast<int>(open_pending_.size());
  out[0] = std::min(n, cap); out[1] = n > cap ? 1 : 0; out[2] = out[3] = 0;
  for (int i = 0; i < std::min(n, cap); ++i) {
    out[4 + 3 * i] = open_pending_[i]->index.x; out[4 + 3 * i + 1] = open_pending_[i]->index.y; out[4 + 3 * i + 2] = open_pending_[i]->index.z;
  }
}

void Oracle::packHalo(const int32_t* all_pending, int cap_pending, int32_t* out, int cap_halo) {
  const int stride = 4 + 3 * cap_pending, W = V_ / 32, entry = 4 + W;
  std::map<Idx3, const Block*> publish;  // ordered: deterministic buffer contents
  for (int r = 0; r < nranks_; ++r) {
    if (r == rank_) continue;
    const int32_t* buf = all_pending + static_cast<size_t>(r) * stride;
    for (int i = 0; i < buf[0]; ++i)
      for (int k = 0; k < 27; ++k) {
        if (k == 13) continue;
        const Idx3 nb{buf[4 + 3 * i] + (k % 3 - 1), buf[4 + 3 * i + 1] + ((k / 3) % 3 - 1), buf[4 + 3 * i + 2] + (k / 9 - 1)};
        if (owner(nb) != rank_) continue;
        if (const Block* b = getBlock(nb)) publish.emplace(nb, b);
      }
  }
  const int n = static_cast<int>(publish.size());
  out[0] = std::min(n, cap_halo); out[1] = n > cap_halo ? 1 : 0; out[2] = out[3] = 0;
  int j = 0;
  for (const auto& kv : publish) {
    if (j >= cap_halo) break;
    int32_t* e = out + 4 + static_cast<size_t>(j) * entry;
    e[0] = kv.first.x; e[1] = kv.first.y; e[2] = kv.first.z; e[3] = 0;
    for (int w = 0; w < W; ++w) {
      uint32_t bits = 0;
      for (int b = 0; b < 32; ++b) {
        const int lin = w * 32 + b;
        if (kv.second->ever_free[lin] || voxelIsFree(*kv.second, lin, open_stamp_)) bits |= 1u << b;
      }
      e[4 + w] = static_cast<int32_t>(bits);
    }
    ++j;
  }
}

void Oracle::trackingFinish(const int32_t* all_pending, int cap_pending, const int32_t* all_halo, int cap_halo) {
  const int W = V_ / 32, entry = 4 + W, stride = 4 + cap_halo * entry;
  GhostMap ghosts;
  for (int r = 0; r < nranks_; ++r) {
    const int32_t* buf = all_halo + static_cast<size_t>(r) * stride;
    if (buf[1] != 0 || all_pending[static_cast<size_t>(r) * (4 + 3 * cap_pending) + 1] != 0) error_ = "shard exchange buffer overflow";
    if (r == rank_) continue;
    for (int i = 0; i < buf[0]; ++i) {
      const int32_t* e = buf + 4 + static_cast<size_t>(i) * entry;
      ghosts.emplace(Idx3{e[0], e[1], e[2]}, reinterpret_cast<const uint32_t*>(e + 4));
    }
  }
  applyEverFree(open_pending_, open_stamp_, &ghosts);
  open_pending_.clear();
}

void Oracle::resetInactive(std::vector<Idx3>* removed) {
  // tracking_integrator.cpp:106-131.
  std::vector<Idx3> to_erase;
  for (auto& kv : blocks_) {
    Block& b = *kv.second;
    if (b.to_remove.empty()) continue;  // no tracking block
    bool remove_block = true;
    for (int lin = 0; lin < V_; ++lin)
      if (!b.to_remove[lin]) { remove_block = false; break; }
    if (!b.has_active_data || remove_block) to_erase.push_back(b.index);
  }
  std::sort(to_erase.begin(), to_erase.end());
  for (const auto& i : to_erase) blocks_.erase(i);
  if (removed) *removed = to_erase;
}

void Oracle::markAllInactive() {
  for (auto& kv : blocks_) kv.second->has_active_data = false;  // active_window.cpp:181-183
}

void Oracle::clearUpdated() {
  for (auto& kv : blocks_) kv.second->updated = false;  // active_window.cpp:169-171
}

// ---- M1 - M4 --------------------------------------------------------------------------------------------

// M1 is split into three steps so that the block-hash sharded protocol (SURVEY.md §8e step 2) can exchange the
// per-pixel "block exists / voxel ever-free" answers between ranks; unsharded, the three run back to back and
// give exactly FreeSpaceMotionDetector::setUpPointMap (free_space_motion_detector.cpp:105-203).

void Oracle::computePixelKeys(const kb_frame& f) {
  const int W = cam_.width, H = cam_.height;
  float R[9], t[3], Rw[9], tw[3];
  invertPose(f.world_T_sensor, R, t, Rw, tw);
  // vertex map in the world frame (hydra parseInputPacket, UP): back-project depth, then transform.
  const float* vertex = f.vertex_world;
  if (!vertex) {
    vertex_scratch_.resize(static_cast<size_t>(W) * H * 3);
    for (int v = 0; v < H; ++v)
      for (int u = 0; u < W; ++u) {
        const float d = f.depth[v * W + u];
        const float pC[3] = {(static_cast<float>(u) - cam_.cx) / cam_.fx * d,
                             (static_cast<float>(v) - cam_.cy) / cam_.fy * d, d};
        transform(Rw, tw, pC, &vertex_scratch_[(static_cast<size_t>(v) * W + u) * 3]);
      }
    vertex = vertex_scratch_.data();
  }
  vertex_ = vertex;
  const float min_z_world = tw[2] + mot_.min_z_coordinate;  // :80
  pix_keys_.assign(static_cast<size_t>(W) * H, PixKey{});
  const int nt = std::max(1, std::min(resolveThreads(mot_.num_threads), W));
  int u_step = W / nt;
  if (u_step * nt < W) ++u_step;  // :112-115
  std::vector<std::thread> threads;
  for (int i = 0; i < nt; ++i) {
    threads.emplace_back([&, i]() {
      const int u_start = u_step * i, u_stop = std::min(u_step * (i + 1), W);
      for (int v = 0; v < H; ++v)
        for (int u = u_start; u < u_stop; ++u) {
          const float range = f.depth[v * W + u];
          if (range <= 0.f || range > mot_.max_range) continue;  // :169-172
          const float* p = &vertex[(static_cast<size_t>(v) * W + u) * 3];
          if (p[2] < min_z_world) continue;  // :176-178
          const Idx3 bi{static_cast<int>(std::floor(p[0] * block_size_inv_)),
                        static_cast<int>(std::floor(p[1] * block_size_inv_)),
                        static_cast<int>(std::floor(p[2] * block_size_inv_))};
          // block->getVoxelIndex(p): floor((p - origin) * voxel_size_inv), may be out of range.
          const int vx = static_cast<int>(std::floor((p[0] - static_cast<float>(bi.x) * block_size_) * voxel_size_inv_));
          const int vy = static_cast<int>(std::floor((p[1] - static_cast<float>(bi.y) * block_size_) * voxel_size_inv_));
          const int vz = static_cast<int>(std::floor((p[2] - static_cast<float>(bi.z) * block_size_) * voxel_size_inv_));
          // The reference appends the pixel under (block, voxel_index) before the validity check
          // (:187-196); invalid indices can never be looked up again (keyFromGlobalIndex always
          // yields valid voxel indices, :234), so such pixels never reach a cluster. We drop them.
          if (vx < 0 || vy < 0 || vz < 0 || vx >= vps_ || vy >= vps_ || vz >= vps_) continue;
          PixKey& k = pix_keys_[static_cast<size_t>(v) * W + u];
          k.valid = true;
          k.block = bi;
          k.lin = vx + vps_ * (vy + vps_ * vz);
          k.g = GIdx{static_cast<int64_t>(bi.x) * vps_ + vx, static_cast<int64_t>(bi.y) * vps_ + vy,
                     static_cast<int64_t>(bi.z) * vps_ + vz};
        }
    });
  }
  for (auto& th : threads) th.join();
}

void Oracle::motionLookupLocal(const kb_frame& f, uint8_t* flags) {
  if (!has_mot_ || !map_.with_tracking) { error_ = "motion detector not configured"; return; }
  computePixelKeys(f);
  // bit0: tracking_layer.getBlockPtr(p_W) exists (:180-183) -> the pixel is in the point map;
  // bit1: that voxel is ever-free (:197-200) -> seed.
  for (size_t px = 0; px < pix_keys_.size(); ++px) {
    uint8_t fl = 0;
    const PixKey& k = pix_keys_[px];
    if (k.valid) {
      if (const Block* blk = getBlock(k.block)) fl = static_cast<uint8_t>(1 | (blk->ever_free[k.lin] ? 2 : 0));
    }
    flags[px] = fl;
  }
}

void Oracle::motionClusterGlobal(const uint8_t* flags, int32_t* dynamic_image, int32_t* n_seeds, int32_t* n_clusters) {
  if (pix_keys_.size() != static_cast<size_t>(cam_.width) * cam_.height) { error_ = "motionLookupLocal must run first"; return; }
  clusterFromFlags(flags, dynamic_image, n_seeds, n_clusters);
}

void Oracle::detectMotion(const kb_frame& f, int32_t* dynamic_image, int32_t* n_seeds_out,
                          int32_t* n_clusters_out) {
  if (!has_mot_ || !map_.with_tracking) { error_ = "motion detector not configured"; return; }
  flags_scratch_.resize(static_cast<size_t>(cam_.width) * cam_.height);
  motionLookupLocal(f, flags_scratch_.data());
  clusterFromFlags(flags_scratch_.data(), dynamic_image, n_seeds_out, n_clusters_out);
}

void Oracle::clusterFromFlags(const uint8_t* flags, int32_t* dynamic_image, int32_t* n_seeds_out,
                              int32_t* n_clusters_out) {
  const int W = cam_.width, H = cam_.height;
  const float* vertex = vertex_;
  std::memset(dynamic_image, 0, sizeof(int32_t) * W * H);
  clusters_.clear();

  // setUpPointMap (:105-156): per-thread strip maps merged under a mutex.
  using VoxelPoints = std::unordered_map<GIdx, std::vector<Pixel>, GIdxHash>;
  VoxelPoints point_map;  // keyed by global voxel index of *valid* voxel indices
  std::unordered_set<GIdx, GIdxHash> seeds;
  const int nt = std::max(1, std::min(resolveThreads(mot_.num_threads), W));
  int u_step = W / nt;
  if (u_step * nt < W) ++u_step;  // :112-115
  std::mutex mtx;
  std::vector<std::thread> threads;
  for (int i = 0; i < nt; ++i) {
    threads.emplace_back([&, i]() {
      VoxelPoints local_map;
      std::unordered_set<GIdx, GIdxHash> local_seeds;
      const int u_start = u_step * i, u_stop = std::min(u_step * (i + 1), W);
      for (int v = 0; v < H; ++v)
        for (int u = u_start; u < u_stop; ++u) {
          const size_t px = static_cast<size_t>(v) * W + u;
          if (!pix_keys_[px].valid || !(flags[px] & 1)) continue;
          local_map[pix_keys_[px].g].push_back({u, v});
          if (flags[px] & 2) local_seeds.insert(pix_keys_[px].g);
        }
      std::lock_guard<std::mutex> lock(mtx);
      seeds.insert(local_seeds.begin(), local_seeds.end());
      for (auto& kv : local_map) {
        auto& dst = point_map[kv.first];
        dst.insert(dst.end(), kv.second.begin(), kv.second.end());
      }
    });
  }
  for (auto& th : threads) th.join();
  if (n_seeds_out) *n_seeds_out = static_cast<int32_t>(seeds.size());

  // M2: clusterDynamicVoxels (:205-272). Seeds iterate in ascending (z,y,x) — a deliberate
  // determinisation of the reference's unordered_set order (SURVEY App. A.10).
  std::vector<GIdx> seed_list(seeds.begin(), seeds.end());
  std::sort(seed_list.begin(), seed_list.end(), GIdxZyxLess());
  const auto offs = neighborOffsets(mot_.neighbor_connectivity);
  std::unordered_set<GIdx, GIdxHash> closed;
  std::vector<Cluster> clusters;
  for (const GIdx& seed : seed_list) {
    if (closed.count(seed)) continue;
    std::vector<GIdx> stack = {seed};
    Cluster cluster;
    while (!stack.empty()) {
      const GIdx g = stack.back();
      stack.pop_back();
      if (closed.count(g)) continue;
      closed.insert(g);
      auto it = point_map.find(g);
      if (it == point_map.end()) continue;
      cluster.pixels.insert(cluster.pixels.end(), it->second.begin(), it->second.end());
      cluster.voxels.insert(g);
      for (const auto& o : offs) {
        const GIdx n{g.x + o[0], g.y + o[1], g.z + o[2]};
        if (seeds.count(n)) {
          stack.push_back(n);
        } else {
          // Non-seed neighbour that contains points: absorbed (pixels appended once per adjacent
          // processed seed voxel — no closed-set check in the reference, :255-265) and closed.
          auto it2 = point_map.find(n);
          if (it2 != point_map.end()) {
            cluster.pixels.insert(cluster.pixels.end(), it2->second.begin(), it2->second.end());
            cluster.voxels.insert(n);
            closed.insert(n);
          }
        }
      }
    }
    clusters.emplace_back(std::move(cluster));
  }

  // M3: mergeClusters (:274-322): connected components of the overlap graph merge into the lowest
  // index. checkClusterOverlap (:345-355): Eigen integer norm() truncates sqrt to an integer.
  const size_t C = clusters.size();
  std::vector<std::vector<uint8_t>> overlap(C, std::vector<uint8_t>(C, 0));
  for (size_t i = 0; i < C; ++i)
    for (size_t j = i + 1; j < C; ++j) {
      bool ov = false;
      for (const GIdx& a : clusters[i].voxels) {
        for (const GIdx& b : clusters[j].voxels) {
          const int64_t dx = a.x - b.x, dy = a.y - b.y, dz = a.z - b.z;
          const int64_t n = static_cast<int64_t>(std::sqrt(static_cast<double>(dx * dx + dy * dy + dz * dz)));
          if (static_cast<float>(n) < mot_.min_separation_distance) { ov = true; break; }
        }
        if (ov) break;
      }
      overlap[i][j] = overlap[j][i] = ov;
    }
  std::vector<bool> merged(C, false), keep(C, false);
  std::function<void(size_t, std::vector<size_t>&)> collect = [&](size_t c, std::vector<size_t>& out) {
    for (size_t i = 0; i < C; ++i) {
      if (merged[i]) continue;
      if (overlap[c][i]) {
        merged[i] = true;
        out.push_back(i);
        collect(i, out);
      }
    }
  };
  for (size_t cur = 0; cur < C; ++cur) {
    if (merged[cur]) continue;
    std::vector<size_t> conn;
    collect(cur, conn);
    for (size_t i : conn) {
      if (i == cur) continue;
      clusters[cur].pixels.insert(clusters[cur].pixels.end(), clusters[i].pixels.begin(),
                                  clusters[i].pixels.end());
      clusters[cur].voxels.insert(clusters[i].voxels.begin(), clusters[i].voxels.end());
    }
    keep[cur] = true;
  }
  std::vector<Cluster> kept;
  for (size_t i = 0; i < C; ++i)
    if (keep[i]) kept.emplace_back(std::move(clusters[i]));

  // M4: applyClusterLevelFilters (:365-379) + writeClustersToData (:381-399).
  for (auto& c : kept) {
    const int sz = static_cast<int>(c.pixels.size());
    if (sz < mot_.min_cluster_size || sz > mot_.max_cluster_size) continue;
    clusters_.emplace_back(std::move(c));
  }
  int id = 1;
  for (auto& c : clusters_) {
    c.id = id;
    bool first = true;
    for (const Pixel& px : c.pixels) {
      dynamic_image[px.v * W + px.u] = id;
      const float* p = &vertex[(static_cast<size_t>(px.v) * W + px.u) * 3];
      for (int a = 0; a < 3; ++a) {
        c.bbox_min[a] = first ? p[a] : std::min(c.bbox_min[a], p[a]);
        c.bbox_max[a] = first ? p[a] : std::max(c.bbox_max[a], p[a]);
      }
      first = false;
    }
    if (id < 255) ++id;  // ids saturate at 255 (:390-395)
  }
  if (n_clusters_out) *n_clusters_out = static_cast<int32_t>(clusters_.size());
}

// ---- object detection: ConnectedSemantics (object_detection/connected_semantics.cpp, fully in-tree) -----------

void Oracle::detectObjects(const kb_object_detector_config& cfg, const kb_frame& f, int32_t* object_image,
                           std::vector<ObjectCluster>* clusters_out) {
  if (!has_cam_) { error_ = "camera not set"; return; }
  const int W = cam_.width, H = cam_.height;
  std::memset(object_image, 0, sizeof(int32_t) * W * H);  // createData: cv::Mat::zeros (active_window.cpp:284)
  object_clusters_.clear();
  if (!f.label) { if (clusters_out) clusters_out->clear(); return; }
  auto isObject = [&](int id) { return id >= 0 && id < KB_MAX_LABELS && cfg.is_object[id] != 0; };
  if (cfg.use_3d) {
    // computeCandidateVoxels (:124-146): pixels of object classes within max_range, grouped by semantic id and by
    // the voxel (grid_size) of their world-frame vertex. NOTE: like the reference, no depth-validity test here; a
    // vertex with a non-finite coordinate or a voxel outside +-2^17 cells makes no candidate (ORACLE_SPEC §10), where
    // the reference's float-to-integer conversion is undefined.
    float R[9], t[3], Rw[9], tw[3];
    invertPose(f.world_T_sensor, R, t, Rw, tw);
    const float inv = 1.f / cfg.grid_size;  // semanticClustering3D(data, config.grid_size) -> 1.f / grid_size (:76)
    // std::map<int, VoxelPixelMap> (connected_semantics.h:88): semantic ids ascending. The inner map is an
    // unordered_map in the reference; ordering its voxels by (z, y, x) makes `begin()` (:87) deterministic.
    std::map<int, std::map<GIdx, std::vector<Pixel>, GIdxZyxLess>> maps;
    for (int u = 0; u < W; ++u)
      for (int v = 0; v < H; ++v) {
        const size_t px = static_cast<size_t>(v) * W + u;
        const float range = f.depth[px];
        if (cfg.max_range > 0.f && range > cfg.max_range) continue;
        const int semantic_id = f.label[px];
        if (!isObject(semantic_id)) continue;
        float p[3];
        if (f.vertex_world) {
          p[0] = f.vertex_world[px * 3]; p[1] = f.vertex_world[px * 3 + 1]; p[2] = f.vertex_world[px * 3 + 2];
        } else {
          const float pC[3] = {(static_cast<float>(u) - cam_.cx) / cam_.fx * range,
                               (static_cast<float>(v) - cam_.cy) / cam_.fy * range, range};
          transform(Rw, tw, pC, p);
        }
        const float c[3] = {std::floor(p[0] * inv), std::floor(p[1] * inv), std::floor(p[2] * inv)};
        constexpr float kCellLimit = 131072.f;  // 2^17
        bool inside = true;
        for (float x : c) inside = inside && x >= -kCellLimit && x < kCellLimit;  // false for NaN and +-inf
        if (!inside) continue;
        const GIdx g{static_cast<int64_t>(c[0]), static_cast<int64_t>(c[1]), static_cast<int64_t>(c[2])};  // spatial_hash::indexFromPoint (:142-143)
        maps[semantic_id][g].push_back({u, v});
      }
    const auto offs = neighborOffsets(cfg.use_full_connectivity ? 26 : 6);  // :58
    for (auto& sm : maps) {
      auto& voxel_to_pixels = sm.second;
      while (!voxel_to_pixels.empty()) {  // :84-121
        ObjectCluster cluster;
        std::vector<GIdx> stack;
        auto item = voxel_to_pixels.begin();
        stack.push_back(item->first);
        cluster.pixels.insert(cluster.pixels.end(), item->second.begin(), item->second.end());
        voxel_to_pixels.erase(item);
        while (!stack.empty()) {
          const GIdx g = stack.back();
          stack.pop_back();
          for (const auto& o : offs) {
            auto it = voxel_to_pixels.find(GIdx{g.x + o[0], g.y + o[1], g.z + o[2]});
            if (it == voxel_to_pixels.end()) continue;
            stack.push_back(it->first);
            cluster.pixels.insert(cluster.pixels.end(), it->second.begin(), it->second.end());
            voxel_to_pixels.erase(it);
          }
        }
        const int size = static_cast<int>(cluster.pixels.size());
        if (size < cfg.min_cluster_size || (cfg.max_cluster_size > 0 && size > cfg.max_cluster_size)) continue;  // :107-111
        cluster.id = static_cast<int>(object_clusters_.size()) + 1;
        cluster.semantic_id = sm.first;
        for (const Pixel& px : cluster.pixels) object_image[px.v * W + px.u] = cluster.id;
        object_clusters_.emplace_back(std::move(cluster));
      }
    }
  } else {
    // semanticClustering2D (:148-163) + growCluster2D (:165-198): column-major scan, region growing over pixels
    // with the same semantic id; then filterClusters (:200-217) zeroes small clusters without renumbering.
    std::vector<ObjectCluster> all;
    for (int u = 0; u < W; ++u)
      for (int v = 0; v < H; ++v) {
        if (object_image[v * W + u] != 0) continue;
        const int semantic_id = f.label[v * W + u];
        if (!isObject(semantic_id)) continue;
        ObjectCluster cluster;
        cluster.id = static_cast<int>(all.size()) + 1;
        cluster.semantic_id = semantic_id;
        std::vector<Pixel> stack{{u, v}};
        cluster.pixels.push_back({u, v});
        object_image[v * W + u] = cluster.id;
        while (!stack.empty()) {
          const Pixel p = stack.back();
          stack.pop_back();
          for (int dv = -1; dv <= 1; ++dv)
            for (int du = -1; du <= 1; ++du) {
              if ((du == 0 && dv == 0) || (!cfg.use_full_connectivity && du != 0 && dv != 0)) continue;
              const int nu = p.u + du, nv = p.v + dv;
              if (nu < 0 || nv < 0 || nu >= W || nv >= H) continue;
              if (object_image[nv * W + nu] != 0) continue;
              if (f.label[nv * W + nu] != semantic_id) continue;
              cluster.pixels.push_back({nu, nv});
              object_image[nv * W + nu] = cluster.id;
              stack.push_back({nu, nv});
            }
        }
        all.emplace_back(std::move(cluster));
      }
    for (auto& c : all) {
      if (static_cast<int>(c.pixels.size()) < cfg.min_cluster_size) {
        for (const Pixel& px : c.pixels) object_image[px.v * W + px.u] = 0;
      } else {
        object_clusters_.emplace_back(std::move(c));
      }
    }
  }
  if (clusters_out) *clusters_out = object_clusters_;
}

// ---- track measurements: MaxIoUTracker, track_by = voxels (tracking/max_iou_tracker.cpp, fully in-tree) --------

void Oracle::trackMeasurements(const kb_frame& f, const int32_t* id_image, int max_id, const int32_t* cluster_ids, float voxel_size, int n_tracks,
                               const int32_t* track_offsets, const int64_t* track_voxels_xyz) {
  track_result_ = TrackMeasurements{};
  if (!has_cam_) { error_ = "camera not set"; return; }
  const int W = cam_.width, H = cam_.height;
  float R[9], t[3], Rw[9], tw[3];
  invertPose(f.world_T_sensor, R, t, Rw, tw);
  // spatial_hash::Grid(voxel_size) (max_iou_tracker.cpp:158): toIndex(p) = floor(p * voxel_size_inv), voxel_size_inv = 1.f / voxel_size
  const float inv = 1.f / voxel_size;
  // setupTrackMeasurementVoxels (:450-459) for every cluster: the set of voxels under the cluster's pixels
  std::vector<std::set<GIdx, GIdxZyxLess>> sets(static_cast<size_t>(max_id));
  for (int v = 0; v < H; ++v)
    for (int u = 0; u < W; ++u) {
      const size_t px = static_cast<size_t>(v) * W + u;
      int id = id_image[px];  // -> row + 1
      if (cluster_ids) {
        const int32_t* it = std::find(cluster_ids, cluster_ids + max_id, id);
        if (it == cluster_ids + max_id) continue;
        id = static_cast<int>(it - cluster_ids) + 1;
      } else if (id < 1 || id > max_id) {
        continue;
      }
      float p[3];
      if (f.vertex_world) {
        p[0] = f.vertex_world[px * 3]; p[1] = f.vertex_world[px * 3 + 1]; p[2] = f.vertex_world[px * 3 + 2];
      } else {
        const float range = f.depth[px];
        const float pC[3] = {(static_cast<float>(u) - cam_.cx) / cam_.fx * range,
                             (static_cast<float>(v) - cam_.cy) / cam_.fy * range, range};
        transform(Rw, tw, pC, p);
      }
      sets[id - 1].insert(GIdx{static_cast<int64_t>(std::floor(p[0] * inv)), static_cast<int64_t>(std::floor(p[1] * inv)),
                               static_cast<int64_t>(std::floor(p[2] * inv))});
    }
  track_result_.voxels.resize(static_cast<size_t>(max_id));
  for (int i = 0; i < max_id; ++i) track_result_.voxels[i].assign(sets[i].begin(), sets[i].end());
  // computeIoUVoxels (:551-562) for every (cluster, track) pair
  track_result_.intersections.assign(static_cast<size_t>(max_id) * n_tracks, 0);
  track_result_.iou.assign(static_cast<size_t>(max_id) * n_tracks, 0.f);
  for (int tr = 0; tr < n_tracks; ++tr) {
    std::set<GIdx, GIdxZyxLess> last_voxels;
    for (int k = track_offsets[tr]; k < track_offsets[tr + 1]; ++k)
      last_voxels.insert(GIdx{track_voxels_xyz[3 * k], track_voxels_xyz[3 * k + 1], track_voxels_xyz[3 * k + 2]});
    const size_t track_size = static_cast<size_t>(track_offsets[tr + 1] - track_offsets[tr]);  // Track::last_voxels.size()
    for (int i = 0; i < max_id; ++i) {
      float intersection = 0.f;
      for (const GIdx& voxel : sets[i])
        if (last_voxels.count(voxel)) intersection += 1.f;
      const size_t o = static_cast<size_t>(i) * n_tracks + tr;
      track_result_.intersections[o] = static_cast<int32_t>(intersection);
      track_result_.iou[o] = intersection / (sets[i].size() + track_size - intersection);
    }
  }
}

bool Oracle::computeVertexMap(const kb_frame& f, float* out) {
  if (!has_cam_) { error_ = "camera not set"; return false; }
  float R[9], t[3], Rw[9], tw[3];
  invertPose(f.world_T_sensor, R, t, Rw, tw);
  for (int v = 0; v < cam_.height; ++v)
    for (int u = 0; u < cam_.width; ++u) {
      const size_t px = static_cast<size_t>(v) * cam_.width + u;
      const float d = f.depth[px];
      const float pC[3] = {(static_cast<float>(u) - cam_.cx) / cam_.fx * d, (static_cast<float>(v) - cam_.cy) / cam_.fy * d, d};
      transform(Rw, tw, pC, &out[3 * px]);
    }
  return true;
}

// ---- E0 / K4 ----------------------------------------------------------------------------------------------

void Oracle::allocateBox(const int32_t mn[3], const int32_t mx[3]) {
  for (int x = mn[0]; x <= mx[0]; ++x)
    for (int y = mn[1]; y <= mx[1]; ++y)
      for (int z = mn[2]; z <= mx[2]; ++z) {
        if (nranks_ > 1 && owner(Idx3{x, y, z}) != rank_) continue;
        allocateBlock(Idx3{x, y, z});
      }
}

int Oracle::scanObjectConfidence(float min_confidence, int min_observations) {
  // mesh_object_extractor.cpp:246-264 with computeConfidence :342-356.
  int erased = 0;
  if (L_ < 2) { error_ = "scanObjectConfidence needs binary semantics"; return 0; }
  for (auto& kv : blocks_) {
    Block& b = *kv.second;
    for (int lin = 0; lin < V_; ++lin) {
      if (b.distance[lin] > 0.f) continue;
      float conf;
      if (b.semantic_empty[lin] || b.likelihoods.empty()) {
        conf = 0.f;
      } else {
        const float total = b.likelihoods[static_cast<size_t>(lin) * L_] +
                            b.likelihoods[static_cast<size_t>(lin) * L_ + 1];
        conf = total < static_cast<float>(min_observations)
                   ? -1.f
                   : b.likelihoods[static_cast<size_t>(lin) * L_ + 1] / total;
      }
      if (conf < min_confidence) {
        b.distance[lin] = map_.truncation_distance;
        ++erased;
      }
    }
  }
  return erased;
}

std::vector<const Block*> Oracle::sortedBlocks(int which) const {
  std::vector<const Block*> out;
  for (auto& kv : blocks_)
    if (which == KB_EXPORT_ALL || kv.second->updated) out.push_back(kv.second.get());
  std::sort(out.begin(), out.end(), [](const Block* a, const Block* b) { return a->index < b->index; });
  return out;
}

}  // namespace ko
