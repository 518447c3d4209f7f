// Device-side motion clustering (M2-M4), see kb_motion_device.cu.
#pragma once

#include "kb_device.cuh"

namespace kb {

constexpr uint8_t kMvSeed = 1;
enum MotionScalar { kMsSeeds = 0, kMsRoots = 1, kMsClusters = 2, kMsOccupied = 3, kMsCount = 4 };

// Open-addressed table of the voxels that contain points of the current frame; a slot index is the voxel's
// id in all per-voxel arrays (capacity = mask + 1 >= 2 * pixels).
struct MotionTable {
  unsigned long long* keys;       // packed (z,y,x), order preserving; ~0 = empty
  uint32_t mask;
  uint32_t* count;                // pixels in the voxel
  uint8_t* flags;                 // kMvSeed
  int* deg;                       // seeds: 1; absorbed voxels: number of adjacent seeds; 0: not in a cluster
  int* parent;                    // union-find
  unsigned long long* pix_total;  // per root: pixel multiset size of the cluster
  unsigned long long* min_seed;   // per root: smallest seed key (z,y,x order)
  int* cluster_id;                // per root: 0 = filtered, else 1 + rank (the image saturates ids at 255)
  int* occupied;                  // compact list of occupied slots (capacity = pixels)
  int* roots;                     // compact list of roots
  int max_roots;
  int* scalars;                   // MotionScalar
  int* pix_slot;                  // [pixels] slot of the pixel's voxel or -1
  const int* gate;                // device counter of seed pixels of this frame: 0 => every stage is a no-op
};

// Per-cluster lists of a clustering (kb_get_motion_clusters). Cluster c (0-based, not saturating) is the root with
// cluster_id == c + 1. Per-cluster arrays hold n_clusters entries, pix_off / vox_off n_clusters + 1.
struct MotionLists {
  int* pix_count;                 // pixels with duplicates (the root's pix_total)
  int* vox_count;
  int* pix_off;                   // exclusive offsets into pixels_uv / voxels (filled by the host)
  int* vox_off;
  int* pix_fill;                  // reservation cursors
  int* vox_fill;
  int* vox_next;                  // [table slots] next pixel position of the voxel's first copy
  unsigned int* box_min;          // [3 * clusters] order-preserving integer images of the floats
  unsigned int* box_max;
  float* bbox;                    // [6 * clusters] min xyz, max xyz
  int32_t* pixels_uv;             // [2 * total pixels]
  unsigned long long* vox_keys;   // [total voxels] unsorted, grouped by cluster
  unsigned long long* vox_sorted;
  int64_t* voxels_xyz;            // [3 * total voxels]
};

// Where the bounding boxes' vertices come from: the kept vertex map, or the kept depth back-projected with the pose.
struct MotionBoxParams {
  const float* vertex;            // H*W*3 or null
  const float* depth;
  int W;
  float fx, fy, cx, cy;
  float Rw[9], tw[3];
};

// Runs C1-C6 on `s`; writes the dynamic image (device) and scalars (seeds, roots, clusters). All stages read the
// device-side seed-pixel counter t.gate, so the sequence can be enqueued before the host knows whether M1 found seeds.
void launchMotionClustering(const MotionTable& t, const int3* gidx, const uint8_t* seed, int P, int conn, int D,
                            int min_size, int max_size, int32_t* image, cudaStream_t s);

// KB_MOTION_SPARSE experiment: same result; the table is reset slot by slot after use instead of wholesale before use
// (table_dirty: another user — the object detector — left entries behind, do one full reset).
void launchMotionClusteringSparse(const MotionTable& t, const int3* gidx, const uint8_t* seed, int P, int conn, int D,
                                  int min_size, int max_size, int32_t* image, bool table_dirty, cudaStream_t s);

// The cluster lists of the M1 output (gidx, seed), in a table of their own (`t`, kept clean between calls, gate != 0).
// Step 1 clusters again (C1-C5) and writes the per-cluster pixel and voxel counts; the host then fills pix_off /
// vox_off. Step 2 writes pixels, voxels (sorted per cluster) and bounding boxes, and resets the table.
void launchMotionListCounts(const MotionTable& t, const MotionLists& l, const int3* gidx, const uint8_t* seed, int P, int conn,
                            int D, int min_size, int max_size, int n_clusters, cudaStream_t s);
cudaError_t launchMotionListFill(const MotionTable& t, const MotionLists& l, const MotionBoxParams& b, int P, int n_clusters,
                                 int total_voxels, void* sort_tmp, size_t* sort_tmp_bytes, cudaStream_t s);

}  // namespace kb
