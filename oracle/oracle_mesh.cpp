// TEST INFRASTRUCTURE — NOT PRODUCT CODE.
// CPU restatement of hydra::MeshIntegrator::generateMesh (UPSTREAM MIT-SPARK/Hydra @ main, not under /root/reference;
// Khronos calls it at khronos/src/active_window/active_window.cpp:223 and
// khronos/src/active_window/object_extraction/mesh_object_extractor.cpp:267 and concatenates the per-block meshes with
// khronos/src/utils/geometry_utils.cpp:61-86). PARITY UNPINNED: restated from the published voxblox algorithm
// (MeshIntegrator::extractMeshInsideBlock / extractMeshOnBorder, MarchingCubes::meshCube) it derives from; the frozen
// behaviour is docs/ORACLE_SPEC.md §13.
#include <algorithm>
#include <cmath>
#include <limits>

#include "oracle.hpp"
#include "oracle_mc_tables.hpp"

namespace ko {

namespace {
const int kCornerOffsets[8][3] = {{0, 0, 0}, {1, 0, 0}, {1, 1, 0}, {0, 1, 0}, {0, 0, 1}, {1, 0, 1}, {1, 1, 1}, {0, 1, 1}};
constexpr float kMinSdfDifference = 1e-6f;  // voxblox MarchingCubes::interpolateVertex
}  // namespace

void Oracle::generateMesh(bool only_mesh_updated, bool clear_updated_flag, float min_weight) {
  mesh_.clear();
  std::vector<Block*> todo;
  for (auto& kv : blocks_)
    if (!only_mesh_updated || kv.second->mesh_updated) todo.push_back(kv.second.get());
  std::sort(todo.begin(), todo.end(), [](const Block* a, const Block* b) { return a->index < b->index; });
  const int vps = vps_;
  const float vs = map_.voxel_size;
  mesh_.resize(todo.size());
  for (size_t bi = 0; bi < todo.size(); ++bi) {
    Block& b = *todo[bi];
    MeshBlock& out = mesh_[bi];
    out.index = b.index;
    // One cube: corner voxels (x,y,z) + offsets; corners beyond the block's last voxel come from the +x/+y/+z neighbour
    // blocks (extractMeshOnBorder); a missing neighbour block or a corner below min_weight drops the cube.
    auto cube = [&](int x, int y, int z) {
      float sdf[8], pos[8][3];
      const Block* cb[8];
      int clin[8];
      for (int c = 0; c < 8; ++c) {
        int vx = x + kCornerOffsets[c][0], vy = y + kCornerOffsets[c][1], vz = z + kCornerOffsets[c][2];
        Idx3 bidx = b.index;
        if (vx == vps) { vx = 0; ++bidx.x; }
        if (vy == vps) { vy = 0; ++bidx.y; }
        if (vz == vps) { vz = 0; ++bidx.z; }
        const Block* nb = (bidx == b.index) ? &b : getBlock(bidx);
        if (!nb) return;
        const int lin = vx + vps * (vy + vps * vz);
        if (!(nb->weight[lin] >= min_weight)) return;
        sdf[c] = nb->distance[lin];
        pos[c][0] = static_cast<float>(bidx.x) * block_size_ + (static_cast<float>(vx) + 0.5f) * vs;
        pos[c][1] = static_cast<float>(bidx.y) * block_size_ + (static_cast<float>(vy) + 0.5f) * vs;
        pos[c][2] = static_cast<float>(bidx.z) * block_size_ + (static_cast<float>(vz) + 0.5f) * vs;
        cb[c] = nb;
        clin[c] = lin;
      }
      int index = 0;
      for (int c = 0; c < 8; ++c)
        if (sdf[c] < 0.f) index |= 1 << c;  // calculateVertexConfiguration
      if (index == 0 || index == 255) return;
      float ev[12][3];
      int near[12];
      for (int e = 0; e < 12; ++e) {
        const int c0 = kEdgeIndexPairs[e][0], c1 = kEdgeIndexPairs[e][1];
        near[e] = -1;
        if (!((sdf[c0] < 0.f) != (sdf[c1] < 0.f))) continue;  // only edges with a zero crossing
        const float diff = sdf[c0] - sdf[c1];
        float t = 0.5f;
        if (std::fabs(diff) >= kMinSdfDifference) {
          t = sdf[c0] / diff;
          for (int a = 0; a < 3; ++a) ev[e][a] = pos[c0][a] + t * (pos[c1][a] - pos[c0][a]);
        } else {
          for (int a = 0; a < 3; ++a) ev[e][a] = 0.5f * (pos[c0][a] + pos[c1][a]);
        }
        near[e] = t < 0.5f ? c0 : c1;  // vertex attributes come from the nearer corner voxel
      }
      const signed char* row = kTriangleTable[index];
      for (int k = 0; row[k] != -1; k += 3) {
        for (int j = 2; j >= 0; --j) {  // voxblox meshCube emits (row[k+2], row[k+1], row[k])
          const int e = row[k + j];
          out.points.insert(out.points.end(), {ev[e][0], ev[e][1], ev[e][2]});
          const Block* nb = cb[near[e]];
          const int lin = clin[near[e]];
          for (int ch = 0; ch < 3; ++ch) out.colors.push_back(nb->color.empty() ? 0 : nb->color[static_cast<size_t>(lin) * 3 + ch]);
          out.labels.push_back((nb->semantic_empty.empty() || nb->semantic_empty[lin]) ? 0u : nb->semantic_label[lin]);
        }
      }
    };
    const int m = vps - 1;
    // extractMeshInsideBlock: x outermost, z innermost
    for (int x = 0; x < m; ++x)
      for (int y = 0; y < m; ++y)
        for (int z = 0; z < m; ++z) cube(x, y, z);
    // extractMeshOnBorder: max-x plane, then max-y plane without the x edge, then max-z plane without both
    for (int z = 0; z < vps; ++z)
      for (int y = 0; y < vps; ++y) cube(m, y, z);
    for (int z = 0; z < vps; ++z)
      for (int x = 0; x < m; ++x) cube(x, m, z);
    for (int y = 0; y < m; ++y)
      for (int x = 0; x < m; ++x) cube(x, y, m);
    if (clear_updated_flag) b.mesh_updated = false;
  }
}

// ---- InstanceForwarding (khronos/src/active_window/object_detection/instance_forwarding.cpp:80-149) ----------------------
void Oracle::forwardInstances(const kb_instance_forwarding_config& cfg, const kb_frame& f, const uint8_t* background, int n_background,
                              int32_t* object_image) {
  instance_clusters_.clear();
  const int W = cam_.width, H = cam_.height;
  const size_t P = static_cast<size_t>(W) * H;
  if (!f.label) { std::fill(object_image, object_image + P, 0); return; }
  std::copy(f.label, f.label + P, object_image);  // :83 (shared buffer: filtered pixels keep their id)
  std::vector<float> vertex;
  const float* vm = f.vertex_world;
  if (!vm) { vertex.resize(P * 3); computeVertexMap(f, vertex.data()); vm = vertex.data(); }
  std::map<int32_t, std::vector<Pixel>> clusters;  // ascending id: determinisation of the unordered_map at :86
  for (int u = 0; u < W; ++u)
    for (int v = 0; v < H; ++v) {  // :87-88 column-major scan
      const size_t px = static_cast<size_t>(v) * W + u;
      const int32_t id = f.label[px];
      if (id == 0) continue;                                                  // :90
      if (background && id > 0 && id < n_background && background[id]) continue;  // :96-104, decided per id by the caller
      if (cfg.max_range > 0.f && f.depth[px] > cfg.max_range) continue;       // :107-112
      clusters[id].push_back(Pixel{u, v});                                    // :114
    }
  const bool filter_by_volume = cfg.min_object_volume > 0.0 || cfg.max_object_volume > 0.0;  // :68
  for (const auto& kv : clusters) {
    const int n = static_cast<int>(kv.second.size());
    if (n < cfg.min_cluster_size || (cfg.max_cluster_size > 0 && n > cfg.max_cluster_size)) continue;  // :119-122
    InstanceCluster cl;
    cl.id = kv.first;
    cl.pixels = kv.second;
    // Per axis the IEEE 754-2019 minimum / maximum over the non-NaN coordinates (-0 below +0), so the box does not
    // depend on the pixel order; an axis without a non-NaN coordinate is NaN at both ends.
    for (int a = 0; a < 3; ++a) cl.bbox[a] = cl.bbox[3 + a] = std::numeric_limits<float>::quiet_NaN();
    for (const Pixel& p : cl.pixels)
      for (int a = 0; a < 3; ++a) {
        const float x = vm[(static_cast<size_t>(p.v) * W + p.u) * 3 + a];
        if (std::isnan(x)) continue;
        float& lo = cl.bbox[a];
        float& hi = cl.bbox[3 + a];
        if (std::isnan(lo) || x < lo || (x == lo && std::signbit(x))) lo = x;
        if (std::isnan(hi) || x > hi || (x == hi && !std::signbit(x))) hi = x;
      }
    if (filter_by_volume) {  // :128-135
      const float volume = (cl.bbox[3] - cl.bbox[0]) * (cl.bbox[4] - cl.bbox[1]) * (cl.bbox[5] - cl.bbox[2]);
      if (volume < cfg.min_object_volume || (cfg.max_object_volume > 0.0 && volume > cfg.max_object_volume)) continue;
    }
    instance_clusters_.push_back(std::move(cl));
  }
}

}  // namespace ko
