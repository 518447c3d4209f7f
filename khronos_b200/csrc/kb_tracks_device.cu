// Device-side measurements of khronos::MaxIoUTracker in its shipped mode, track_by = "voxels"
// (khronos_ros/config/mapper/uHumans2.yaml:72; SURVEY.md §8f row 4). The tracker itself — greedy association, track
// bookkeeping — is a few dozen list operations per frame and stays with the caller; what it iterates pixels and voxel
// sets for moves here, next to the id images the device already holds:
//
//   T1  setupTrackMeasurementVoxels (khronos/src/active_window/tracking/max_iou_tracker.cpp:450-459): the voxels of a
//       cluster are the set { grid.toIndex(vertex_map(pixel)) : pixel in cluster } at the tracker's own voxel size.
//       Every pixel of the id image inserts (cluster row + 1, voxel) into an open-addressed table; the thread that creates an entry
//       adds it to the id's count and integer index sums (computeCentroid's voxel mode, :534-539, is the mean of the
//       voxel centres = (sum / n + 0.5) * voxel_size; integer sums do not depend on the iteration order of the set).
//   T2  computeIoUVoxels (:551-562): |cluster.voxels ∩ track.last_voxels| for every (cluster, track) pair: one thread
//       per (track voxel, present cluster id) probes the table. The IoU quotient is formed by the host from the counts.
//   T3  the table's keys are order preserving in (id, z, y, x): exported as they are, sorted by the host when the caller
//       asks for the voxel lists (Track::last_voxels of the associated tracks).
#include "kb_tracks_device.cuh"

namespace kb {

namespace {

constexpr unsigned long long kTkEmpty = ~0ull;

__global__ void tkInitKernel(MotionTable t, TrackParams p) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < kMsCount) t.scalars[i] = 0;
  if (i < p.n_ids) {
    p.voxel_counts[i] = 0;
    p.sums[3 * i] = 0; p.sums[3 * i + 1] = 0; p.sums[3 * i + 2] = 0;
  }
  if (i <= static_cast<int>(t.mask)) t.keys[i] = kTkEmpty;
}

__global__ void tkInsertKernel(MotionTable t, const __grid_constant__ TrackParams p) {
  const int px = blockIdx.x * blockDim.x + threadIdx.x;
  if (px >= p.W * p.H) return;
  const int value = __ldg(&p.ids[px]);
  int id;  // row + 1
  if (p.id_list) {  // sparse ids (2D object images keep their creation-order ids): position in the ascending list
    int lo = 0, hi = p.n_ids - 1;
    id = 0;
    while (lo <= hi) {
      const int mid = (lo + hi) >> 1;
      const int m = __ldg(&p.id_list[mid]);
      if (m == value) { id = mid + 1; break; }
      if (m < value) lo = mid + 1; else hi = mid - 1;
    }
    if (id == 0) return;
  } else {
    id = value;
    if (id < 1 || id > p.n_ids) return;
  }
  float wx, wy, wz;
  if (p.vertex) {
    wx = __ldg(&p.vertex[3 * px]); wy = __ldg(&p.vertex[3 * px + 1]); wz = __ldg(&p.vertex[3 * px + 2]);
  } else {
    const float range = __ldg(&p.depth[px]);
    const int u = px % p.W, v = px / p.W;
    const float cxn = (static_cast<float>(u) - p.cx) / p.fx * range;
    const float cyn = (static_cast<float>(v) - p.cy) / p.fy * range;
    wx = ((p.Rw[0] * cxn + p.Rw[1] * cyn) + p.Rw[2] * range) + p.tw[0];
    wy = ((p.Rw[3] * cxn + p.Rw[4] * cyn) + p.Rw[5] * range) + p.tw[1];
    wz = ((p.Rw[6] * cxn + p.Rw[7] * cyn) + p.Rw[8] * range) + p.tw[2];
  }
  const float fx = floorf(wx * p.inv_voxel), fy = floorf(wy * p.inv_voxel), fz = floorf(wz * p.inv_voxel);
  const float lim = static_cast<float>(1 << (kTrackCoordBits - 1));
  if (!(fabsf(fx) < lim && fabsf(fy) < lim && fabsf(fz) < lim)) return;  // also drops NaN vertices
  const int gx = static_cast<int>(fx), gy = static_cast<int>(fy), gz = static_cast<int>(fz);
  unsigned long long key;
  trackVoxelKey(gx, gy, gz, &key);
  key |= static_cast<unsigned long long>(id) << (3 * kTrackCoordBits);
  uint32_t h = static_cast<uint32_t>(mix64(key)) & t.mask;
  for (uint32_t probe = 0; probe <= t.mask; ++probe) {
    unsigned long long k = t.keys[h];
    if (k == kTkEmpty) {
      k = atomicCAS(&t.keys[h], kTkEmpty, key);
      if (k == kTkEmpty) {  // this thread created the entry: a new voxel of cluster `id`
        t.occupied[atomicAdd(&t.scalars[kMsOccupied], 1)] = static_cast<int>(h);
        atomicAdd(&p.voxel_counts[id - 1], 1);
        atomicAdd(&p.sums[3 * (id - 1)], static_cast<unsigned long long>(static_cast<long long>(gx)));
        atomicAdd(&p.sums[3 * (id - 1) + 1], static_cast<unsigned long long>(static_cast<long long>(gy)));
        atomicAdd(&p.sums[3 * (id - 1) + 2], static_cast<unsigned long long>(static_cast<long long>(gz)));
        return;
      }
    }
    if (k == key) return;
    h = (h + 1) & t.mask;
  }
}

// Input conversion (upstream parseInputPacket, call site active_window.cpp:275): world-frame vertex map of a depth image.
__global__ void vertexMapKernel(TrackParams p, float* __restrict__ out) {
  const int px = blockIdx.x * blockDim.x + threadIdx.x;
  if (px >= p.W * p.H) return;
  const float range = __ldg(&p.depth[px]);
  const int u = px % p.W, v = px / p.W;
  const float cxn = (static_cast<float>(u) - p.cx) / p.fx * range;
  const float cyn = (static_cast<float>(v) - p.cy) / p.fy * range;
  out[3 * px] = ((p.Rw[0] * cxn + p.Rw[1] * cyn) + p.Rw[2] * range) + p.tw[0];
  out[3 * px + 1] = ((p.Rw[3] * cxn + p.Rw[4] * cyn) + p.Rw[5] * range) + p.tw[1];
  out[3 * px + 2] = ((p.Rw[6] * cxn + p.Rw[7] * cyn) + p.Rw[8] * range) + p.tw[2];
}

__global__ void tkIntersectKernel(MotionTable t, const unsigned long long* __restrict__ track_keys,
                                  const int* __restrict__ track_of, int n_track_voxels, const int* __restrict__ present_ids,
                                  int n_present, int n_tracks, int* intersections) {
  const long long total = static_cast<long long>(n_track_voxels) * n_present;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int tv = static_cast<int>(i / n_present);
    const int id = present_ids[static_cast<int>(i % n_present)];
    const unsigned long long key = track_keys[tv] | (static_cast<unsigned long long>(id) << (3 * kTrackCoordBits));
    uint32_t h = static_cast<uint32_t>(mix64(key)) & t.mask;
    for (uint32_t probe = 0; probe <= t.mask; ++probe) {
      const unsigned long long k = t.keys[h];
      if (k == key) {
        atomicAdd(&intersections[static_cast<size_t>(id - 1) * n_tracks + track_of[tv]], 1);
        break;
      }
      if (k == kTkEmpty) break;
      h = (h + 1) & t.mask;
    }
  }
}

__global__ void tkExportKernel(MotionTable t, unsigned long long* out) {
  const int n = t.scalars[kMsOccupied];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) out[i] = t.keys[t.occupied[i]];
}

}  // namespace

void launchTrackVoxelize(const MotionTable& t, const TrackParams& p, cudaStream_t s) {
  const int slots = static_cast<int>(t.mask) + 1;
  const int n_init = slots > p.n_ids ? slots : p.n_ids;
  tkInitKernel<<<(n_init + 255) / 256, 256, 0, s>>>(t, p);
  tkInsertKernel<<<(p.W * p.H + 255) / 256, 256, 0, s>>>(t, p);
}

void launchTrackIntersect(const MotionTable& t, const unsigned long long* track_keys, const int* track_of, int n_track_voxels,
                          const int* present_ids, int n_present, int n_tracks, int* intersections, cudaStream_t s) {
  if (n_track_voxels <= 0 || n_present <= 0) return;
  const long long total = static_cast<long long>(n_track_voxels) * n_present;
  const int blocks = static_cast<int>(std::min<long long>(total / 256 + 1, smCount() * 8LL));
  tkIntersectKernel<<<blocks, 256, 0, s>>>(t, track_keys, track_of, n_track_voxels, present_ids, n_present, n_tracks, intersections);
}

void launchVertexMap(const TrackParams& p, float* out, cudaStream_t s) {
  vertexMapKernel<<<(p.W * p.H + 255) / 256, 256, 0, s>>>(p, out);
}

void launchTrackExportKeys(const MotionTable& t, unsigned long long* out, cudaStream_t s) {
  tkExportKernel<<<smCount(), 256, 0, s>>>(t, out);
}

}  // namespace kb
