// Internal interface of ls_filters.cu for ls_api.cu: the per-scan input filters (ls_point_filter chains) enqueued on
// device buffers and a stream.  Not part of the C ABI.
#ifndef LS_FILTERS_CUH_
#define LS_FILTERS_CUH_

#include <cstddef>
#include <cstdint>

#include <cuda_runtime.h>

#include "../../include/ls_b200.h"
#include "ls_buffer.cuh"

namespace lsf {

// Device scratch of one chain run, grown to the largest cloud seen (reserve()); pts[0]'s capacity is the group's.  The
// chain ping-pongs between pts[0]/nrm[0] and pts[1]/nrm[1].
struct ChainBuffers {
  ls::Buffer<float4> pts[2], nrm[2];
  ls::Buffer<int> keep, pos;  // per-point flags and their exclusive scan
  ls::Buffer<int> small;      // 8 ints: voxel cell bounds (6), kept count
  ls::Buffer<unsigned long long> key, key2;
  ls::Buffer<int> idx, idx2, head, slot;
  ls::Buffer<unsigned long long> sums;  // 7 per voxel: x, y, z, count, nx, ny, nz (fixed point)
  ls::Buffer<unsigned char> tmp;        // CUB temporary storage
  size_t tmp_bytes = 0;
};
// All or nothing: on a failure every array is freed and the error returned.
cudaError_t reserve(ChainBuffers& b, int n);

// Flag / compact one run of mask filters (point-wise tests and index samplers) that starts at filters[0].  `n` points in
// pts/nrm (nrm may be NULL).  Writes the survivors to out/out_nrm and their number to b.small[6]; the caller reads it
// back.  *used = filters consumed.  Launch count added to *launches (own kernels; the CUB scans are not counted).
cudaError_t enqueue_mask_run(const ls_point_filter* filters, int n_filters, const float4* pts, const float4* nrm, int n,
                             float4* out, float4* out_nrm, ChainBuffers& b, cudaStream_t st, int* used, uint64_t* launches);
bool is_mask_filter(int type);

// pcl::VoxelGrid centroids (ls_voxel_grid) of n device points, with the normals averaged alongside when in_nrm != NULL.
// Synchronises `st` twice (cell bounds, voxel count).  *m_out = voxels written to out / out_nrm.  Returns LS_OK,
// LS_ERR_ARG (leaf too small for the cloud's extent) or LS_ERR_CUDA.
// min_points > 1 keeps only the voxels with at least that many points (pcl::VoxelGrid::setMinimumPointsNumberPerVoxel):
// the centroids go to b.cent first, then one flag / scan / compaction into out, and `st` is synchronised a third time.
// It needs b.cent (n float4) and no normals.  min_points 0 or 1 launches exactly the kernels of the plain grid.
struct VoxelBuffers {
  int* mm;  // 6 ints
  unsigned long long *key, *key2, *sums;
  int *idx, *idx2, *head, *slot;
  void* tmp;
  size_t tmp_bytes;
  float4* cent = nullptr;  // centroids before the minimum-count compaction
};
size_t voxel_temp_bytes(int n);
int enqueue_voxel_grid(const float4* in, const float4* in_nrm, int n, const float leaf[3], float4* out, float4* out_nrm,
                       int min_points, const VoxelBuffers& b, cudaStream_t st, int* m_out, uint64_t* launches);
VoxelBuffers voxel_buffers(const ChainBuffers& b);

// ---- local map (ls_local_map_*): scratch is a ChainBuffers reserved for the largest cloud of the call; each helper
// synchronises `st` once and returns LS_OK or LS_ERR_CUDA.
// Append: the n points of a ring slot moved by T (an exact identity when `identity`: verbatim) into b.pts[0], ground points
// ((double)z <= z_min) dropped when remove_ground, the rest compacted in order to BOTH local_tail and queue_tail.
int enqueue_local_map_append(const float4* scan, int n, const float T[16], bool identity, bool remove_ground, double z_min,
                             float4* local_tail, float4* queue_tail, ChainBuffers& b, cudaStream_t st, int* kept,
                             uint64_t* launches);
// updateLocalMap's move of n device points in place (the xform_point order, no identity shortcut); enqueued only.
int enqueue_transform_in_place(float4* pts, int n, const float T[16], cudaStream_t st, uint64_t* launches);
// ls_filter_cylinder's inside rule (d_xy^2 <= r^2 and |dz| <= h/2) from device `in` to device `out`, input order kept.
int enqueue_cylinder_crop(const float4* in, int n, const double center[3], double radius_m, double height_m, float4* out,
                          ChainBuffers& b, cudaStream_t st, int* kept, uint64_t* launches);
// One stable two-way partition: the inside points (<=) to `inside`, the outside points (>= on either) to `outside`; a
// point on the boundary goes to both.  Uses b.key / b.key2 as its 64-bit flags and their scan.
int enqueue_cylinder_split(const float4* in, int n, const double center[3], double radius_m, double height_m, float4* inside,
                           float4* outside, ChainBuffers& b, cudaStream_t st, int* n_inside, int* n_outside, uint64_t* launches);

}  // namespace lsf

#endif  // LS_FILTERS_CUH_
