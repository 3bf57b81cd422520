// Internal interface of ls_filters.cu for ls_api.cu: the per-scan input filters (ls_point_filter chains) enqueued on
// device buffers and a stream.  Not part of the C ABI.
#ifndef LS_FILTERS_CUH_
#define LS_FILTERS_CUH_

#include <cstddef>
#include <cstdint>

#include <cuda_runtime.h>

#include "../../include/ls_b200.h"

namespace lsf {

// Device scratch of one chain run, grown to the largest cloud seen (reserve()).  The chain ping-pongs between
// pts[0]/nrm[0] and pts[1]/nrm[1].
struct ChainBuffers {
  int cap = 0;
  float4* pts[2] = {nullptr, nullptr};
  float4* nrm[2] = {nullptr, nullptr};
  int *keep = nullptr, *pos = nullptr;  // per-point flags and their exclusive scan
  int* small = nullptr;                 // 8 ints: voxel cell bounds (6), kept count
  unsigned long long *key = nullptr, *key2 = nullptr;
  int *idx = nullptr, *idx2 = nullptr, *head = nullptr, *slot = nullptr;
  unsigned long long* sums = nullptr;   // 7 per voxel: x, y, z, count, nx, ny, nz (fixed point)
  void* tmp = nullptr;                  // CUB temporary storage
  size_t tmp_bytes = 0;
};
cudaError_t reserve(ChainBuffers& b, int n);
void release(ChainBuffers& b);

// Flag / compact one run of mask filters (point-wise tests and index samplers) that starts at filters[0].  `n` points in
// pts/nrm (nrm may be NULL).  Writes the survivors to out/out_nrm and their number to b.small[6]; the caller reads it
// back.  *used = filters consumed.  Launch count added to *launches (own kernels; the CUB scans are not counted).
cudaError_t enqueue_mask_run(const ls_point_filter* filters, int n_filters, const float4* pts, const float4* nrm, int n,
                             float4* out, float4* out_nrm, ChainBuffers& b, cudaStream_t st, int* used, uint64_t* launches);
bool is_mask_filter(int type);

// pcl::VoxelGrid centroids (ls_voxel_grid) of n device points, with the normals averaged alongside when in_nrm != NULL.
// Synchronises `st` twice (cell bounds, voxel count).  *m_out = voxels written to out / out_nrm.  Returns LS_OK,
// LS_ERR_ARG (leaf too small for the cloud's extent) or LS_ERR_CUDA.
struct VoxelBuffers {
  int* mm;  // 6 ints
  unsigned long long *key, *key2, *sums;
  int *idx, *idx2, *head, *slot;
  void* tmp;
  size_t tmp_bytes;
};
size_t voxel_temp_bytes(int n);
int enqueue_voxel_grid(const float4* in, const float4* in_nrm, int n, const float leaf[3], float4* out, float4* out_nrm,
                       const VoxelBuffers& b, cudaStream_t st, int* m_out, uint64_t* launches);
VoxelBuffers voxel_buffers(const ChainBuffers& b);

}  // namespace lsf

#endif  // LS_FILTERS_CUH_
