// Input / map-maintenance side of the path (SURVEY.md §8 row f4): the steps either side of the registration that
// laser_slam_ros runs on the CPU per scan or per map publication --
//   PointCloud2 -> DataPoints        reference laser_slam_ros/src/laser_slam_worker.cpp:125 (pcl::fromROSMsg + conversion)
//   applyCylindricalFilter           reference laser_slam_ros/include/laser_slam_ros/common.hpp:194-223 (used by
//                                    LaserSlamWorker::getFilteredMap, laser_slam_worker.cpp:415-488)
//   pcl::VoxelGrid                   laser_slam_worker.cpp:434-441 (voxel_filter_, leaf from params)
//   velodyne assembler de-skew       reference sensor_drivers/velodyne_assembler/src/velodyne_assembler_ros.cpp:57-143: the
//                                    packets of one revolution, each moved into the frame of the revolution's last packet
// as device kernels behind the C ABI.  Not the hot path: the radix sort and the scans are CUB (library code), the
// kernels around them are ours.  Order of the outputs is defined so that results are reproducible: the cylinder filter
// keeps the input order (as the reference's sequential push_back), the voxel grid emits voxels by ascending cell index
// (as PCL does) with the centroid of each voxel computed from EXACT fixed-point sums (2^-24 m), one rounding.
#include <cstdint>
#include <cstring>
#include <string>

#include <cub/cub.cuh>
#include <cuda_runtime.h>

#include "../../include/ls_b200.h"

namespace {

__global__ void ingest_kernel(const unsigned char* __restrict__ data, int point_step, int off_x, int off_y, int off_z, int n,
                              float4* __restrict__ out) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const unsigned char* p = data + (size_t)i * point_step;
    float x, y, z;
    memcpy(&x, p + off_x, 4);
    memcpy(&y, p + off_y, 4);
    memcpy(&z, p + off_z, 4);
    out[i] = make_float4(x, y, z, 1.0f);
  }
}

// keep[i] = 1 iff the point passes applyCylindricalFilter's test (double arithmetic as the reference: pow(), abs()).
__global__ void cylinder_flag_kernel(const float4* __restrict__ in, int n, double cx, double cy, double cz, double r2, double hh,
                                     int remove_inside, int* __restrict__ keep) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float4 p = in[i];
    const double dx = (double)p.x - cx, dy = (double)p.y - cy;
    const double d2 = dx * dx + dy * dy;
    const double dz = fabs((double)p.z - cz);
    const bool inside = d2 <= r2 && dz <= hh;             // kept when remove_inside == 0 (reference :213-216)
    const bool outside = d2 >= r2 || dz >= hh;            // kept when remove_inside != 0 (reference :205-209)
    keep[i] = remove_inside ? (outside ? 1 : 0) : (inside ? 1 : 0);
  }
}

__global__ void compact_kernel(const float4* __restrict__ in, const int* __restrict__ keep, const int* __restrict__ pos, int n,
                               float4* __restrict__ out) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    if (keep[i]) out[pos[i]] = in[i];
}

// ---- de-skew of one revolution: out = T_final (x) (T_packet (x) p), two float32 transforms in the reference's order
// (velodyne_assembler_ros.cpp:129-133 transforms a packet into the frame of the revolution's start when it arrives,
// :107-108 moves the assembled cloud to the frame of its last packet before publishing).  An exact identity matrix copies
// the point verbatim -- the reference does not transform the first packet at all.  Same arithmetic as ls_transform_cloud.
__device__ __forceinline__ void xform3(const float* T, float x, float y, float z, float& ox, float& oy, float& oz) {
  float a, b, c, s;
  a = T[0] * x; b = T[4] * y; c = T[8] * z; s = a + b; s = s + c; ox = s + T[12];
  a = T[1] * x; b = T[5] * y; c = T[9] * z; s = a + b; s = s + c; oy = s + T[13];
  a = T[2] * x; b = T[6] * y; c = T[10] * z; s = a + b; s = s + c; oz = s + T[14];
}
__device__ __forceinline__ bool is_identity(const float* T) {
  bool id = true;
  for (int k = 0; k < 16; ++k) id = id && T[k] == ((k % 5 == 0) ? 1.0f : 0.0f);
  return id;
}
__global__ void deskew_kernel(const float4* __restrict__ in, int m, const int* __restrict__ offs, int n_packets,
                              const float* __restrict__ T_packets, const float* __restrict__ T_final, float4* __restrict__ out) {
  __shared__ float Tf[16];
  __shared__ int final_identity;
  if (threadIdx.x < 16) Tf[threadIdx.x] = T_final[threadIdx.x];
  __syncthreads();
  if (threadIdx.x == 0) final_identity = is_identity(Tf) ? 1 : 0;
  __syncthreads();
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += gridDim.x * blockDim.x) {
    int lo = 0, hi = n_packets - 1;  // last packet whose first point is <= i (empty packets share an offset: skipped)
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (offs[mid] <= i) lo = mid;
      else hi = mid - 1;
    }
    const float* Tk = T_packets + 16 * (size_t)lo;
    const float4 p = in[i];
    float x = p.x, y = p.y, z = p.z;
    if (!is_identity(Tk)) xform3(Tk, p.x, p.y, p.z, x, y, z);
    if (!final_identity) {
      const float a = x, b = y, c = z;
      xform3(Tf, a, b, c, x, y, z);
    }
    out[i] = make_float4(x, y, z, p.w);
  }
}

// ---- voxel grid
__global__ void minmax_kernel(const float4* __restrict__ in, int n, int* __restrict__ mn, int* __restrict__ mx, float ix, float iy, float iz) {
  int lo[3] = {INT_MAX, INT_MAX, INT_MAX}, hi[3] = {INT_MIN, INT_MIN, INT_MIN};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float4 p = in[i];
    if (!(isfinite(p.x) && isfinite(p.y) && isfinite(p.z))) continue;
    const int c[3] = {(int)floorf(p.x * ix), (int)floorf(p.y * iy), (int)floorf(p.z * iz)};
    for (int a = 0; a < 3; ++a) { lo[a] = min(lo[a], c[a]); hi[a] = max(hi[a], c[a]); }
  }
  for (int a = 0; a < 3; ++a) {
    atomicMin(&mn[a], lo[a]);
    atomicMax(&mx[a], hi[a]);
  }
}

__global__ void voxel_key_kernel(const float4* __restrict__ in, int n, const int* __restrict__ mn, const int* __restrict__ mx, float ix,
                                 float iy, float iz, unsigned long long* __restrict__ key, int* __restrict__ idx) {
  const long long dx = (long long)mx[0] - mn[0] + 1, dy = (long long)mx[1] - mn[1] + 1;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float4 p = in[i];
    unsigned long long k = ~0ull;  // non-finite points sort last and are dropped (PCL skips them too)
    if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z)) {
      const long long a = (long long)floorf(p.x * ix) - mn[0], b = (long long)floorf(p.y * iy) - mn[1],
                      c = (long long)floorf(p.z * iz) - mn[2];
      k = (unsigned long long)(a + b * dx + c * dx * dy);
    }
    key[i] = k;
    idx[i] = i;
  }
}

__global__ void voxel_head_kernel(const unsigned long long* __restrict__ key, int n, int* __restrict__ head) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    head[i] = (key[i] != ~0ull && (i == 0 || key[i] != key[i - 1])) ? 1 : 0;
}

// slot[i] = inclusive scan of head - 1: every sorted point adds its exact fixed-point coordinates to its voxel
__global__ void voxel_accumulate_kernel(const float4* __restrict__ in, const unsigned long long* __restrict__ key,
                                        const int* __restrict__ idx, const int* __restrict__ slot, int n,
                                        unsigned long long* __restrict__ sums /* 4 per voxel: x, y, z, count */) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (key[i] == ~0ull) continue;
    const float4 p = in[idx[i]];
    unsigned long long* s = sums + 4 * (size_t)(slot[i] - 1);
    atomicAdd(&s[0], (unsigned long long)__double2ll_rn((double)p.x * 16777216.0));
    atomicAdd(&s[1], (unsigned long long)__double2ll_rn((double)p.y * 16777216.0));
    atomicAdd(&s[2], (unsigned long long)__double2ll_rn((double)p.z * 16777216.0));
    atomicAdd(&s[3], 1ull);
  }
}

__global__ void voxel_centroid_kernel(const unsigned long long* __restrict__ sums, int m, float4* __restrict__ out) {
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < m; v += gridDim.x * blockDim.x) {
    const double c = (double)sums[4 * (size_t)v + 3] * 16777216.0;
    out[v] = make_float4((float)((double)(long long)sums[4 * (size_t)v] / c), (float)((double)(long long)sums[4 * (size_t)v + 1] / c),
                         (float)((double)(long long)sums[4 * (size_t)v + 2] / c), 1.0f);
  }
}

struct Scratch {  // freed on every exit path
  void* p[12] = {};
  int n = 0;
  template <typename T>
  cudaError_t alloc(T** out, size_t count) {
    cudaError_t e = cudaMalloc((void**)out, (count ? count : 1) * sizeof(T));
    if (e == cudaSuccess) p[n++] = *out;
    return e;
  }
  ~Scratch() {
    for (int i = 0; i < n; ++i) cudaFree(p[i]);
  }
};

// grid-stride kernels: at most 8 CTAs of 256 threads per SM of the current device (set by every entry point)
inline int blocks(int n) {
  int dev = 0, sms = 1;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
      sms < 1)
    sms = 1;
  const int b = (n + 255) / 256;
  return b < 1 ? 1 : (b > sms * 8 ? sms * 8 : b);
}

#define FCU(call)                              \
  do {                                         \
    if ((call) != cudaSuccess) return LS_ERR_CUDA; \
  } while (0)

}  // namespace

extern "C" {

int ls_ingest_pointcloud2(int device, const void* data, int point_step, int off_x, int off_y, int off_z, int n, float* out4) {
  if (!data || !out4 || n < 0 || point_step < 12 || off_x < 0 || off_y < 0 || off_z < 0 || off_x + 4 > point_step ||
      off_y + 4 > point_step || off_z + 4 > point_step)
    return LS_ERR_ARG;
  if (n == 0) return LS_OK;
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || device < 0 || device >= count) return LS_ERR_CUDA;  // no CPU fallback
  FCU(cudaSetDevice(device));
  Scratch s;
  unsigned char* d_in;
  float4* d_out;
  FCU(s.alloc(&d_in, (size_t)n * point_step));
  FCU(s.alloc(&d_out, (size_t)n));
  FCU(cudaMemcpy(d_in, data, (size_t)n * point_step, cudaMemcpyHostToDevice));
  ingest_kernel<<<blocks(n), 256>>>(d_in, point_step, off_x, off_y, off_z, n, d_out);
  FCU(cudaMemcpy(out4, d_out, (size_t)n * sizeof(float4), cudaMemcpyDeviceToHost));
  return LS_OK;
}

int ls_filter_cylinder(int device, const float* in4, int n, const double center[3], double radius_m, double height_m,
                       int remove_points_inside, float* out4, int* n_out) {
  if (!in4 || !out4 || !n_out || !center || n < 0) return LS_ERR_ARG;
  *n_out = 0;
  if (n == 0) return LS_OK;
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || device < 0 || device >= count) return LS_ERR_CUDA;
  FCU(cudaSetDevice(device));
  Scratch s;
  float4 *d_in, *d_out;
  int *d_keep, *d_pos;
  FCU(s.alloc(&d_in, (size_t)n));
  FCU(s.alloc(&d_out, (size_t)n));
  FCU(s.alloc(&d_keep, (size_t)n));
  FCU(s.alloc(&d_pos, (size_t)n));
  FCU(cudaMemcpy(d_in, in4, (size_t)n * sizeof(float4), cudaMemcpyHostToDevice));
  cylinder_flag_kernel<<<blocks(n), 256>>>(d_in, n, center[0], center[1], center[2], radius_m * radius_m, height_m / 2.0,
                                          remove_points_inside, d_keep);
  size_t tmp_bytes = 0;
  FCU(cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, d_keep, d_pos, n));
  void* d_tmp;
  FCU(s.alloc((unsigned char**)&d_tmp, tmp_bytes));
  FCU(cub::DeviceScan::ExclusiveSum(d_tmp, tmp_bytes, d_keep, d_pos, n));
  compact_kernel<<<blocks(n), 256>>>(d_in, d_keep, d_pos, n, d_out);
  int last_pos = 0, last_keep = 0;
  FCU(cudaMemcpy(&last_pos, d_pos + (n - 1), sizeof(int), cudaMemcpyDeviceToHost));
  FCU(cudaMemcpy(&last_keep, d_keep + (n - 1), sizeof(int), cudaMemcpyDeviceToHost));
  *n_out = last_pos + last_keep;
  FCU(cudaMemcpy(out4, d_out, (size_t)*n_out * sizeof(float4), cudaMemcpyDeviceToHost));
  return LS_OK;
}

int ls_deskew_revolution(int device, const float* points4, const int* packet_offsets, int n_packets, const float* T_packets,
                         const float T_final[16], float* out4) {
  if (!packet_offsets || n_packets < 1 || !T_packets || !T_final) return LS_ERR_ARG;
  const int m = packet_offsets[n_packets];
  if (packet_offsets[0] != 0 || m < 0) return LS_ERR_ARG;
  for (int k = 0; k < n_packets; ++k)
    if (packet_offsets[k + 1] < packet_offsets[k]) return LS_ERR_ARG;
  if (m == 0) return LS_OK;
  if (!points4 || !out4) return LS_ERR_ARG;
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || device < 0 || device >= count) return LS_ERR_CUDA;
  FCU(cudaSetDevice(device));
  Scratch s;
  float4 *d_in, *d_out;
  int* d_offs;
  float* d_T;
  FCU(s.alloc(&d_in, (size_t)m));
  FCU(s.alloc(&d_out, (size_t)m));
  FCU(s.alloc(&d_offs, (size_t)n_packets + 1));
  FCU(s.alloc(&d_T, 16 * ((size_t)n_packets + 1)));
  FCU(cudaMemcpy(d_in, points4, (size_t)m * sizeof(float4), cudaMemcpyHostToDevice));
  FCU(cudaMemcpy(d_offs, packet_offsets, ((size_t)n_packets + 1) * sizeof(int), cudaMemcpyHostToDevice));
  FCU(cudaMemcpy(d_T, T_packets, 16 * (size_t)n_packets * sizeof(float), cudaMemcpyHostToDevice));
  FCU(cudaMemcpy(d_T + 16 * (size_t)n_packets, T_final, 16 * sizeof(float), cudaMemcpyHostToDevice));
  deskew_kernel<<<blocks(m), 256>>>(d_in, m, d_offs, n_packets, d_T, d_T + 16 * (size_t)n_packets, d_out);
  FCU(cudaGetLastError());
  FCU(cudaMemcpy(out4, d_out, (size_t)m * sizeof(float4), cudaMemcpyDeviceToHost));
  return LS_OK;
}

int ls_voxel_grid(int device, const float* in4, int n, const float leaf_size[3], float* out4, int* n_out) {
  if (!in4 || !out4 || !n_out || !leaf_size || n < 0 || !(leaf_size[0] > 0.f) || !(leaf_size[1] > 0.f) || !(leaf_size[2] > 0.f))
    return LS_ERR_ARG;
  *n_out = 0;
  if (n == 0) return LS_OK;
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || device < 0 || device >= count) return LS_ERR_CUDA;
  FCU(cudaSetDevice(device));
  const float ix = 1.0f / leaf_size[0], iy = 1.0f / leaf_size[1], iz = 1.0f / leaf_size[2];  // PCL: inverse_leaf_size_
  Scratch s;
  float4 *d_in, *d_out;
  int *d_mm, *d_idx, *d_idx2, *d_head, *d_slot;
  unsigned long long *d_key, *d_key2, *d_sums;
  FCU(s.alloc(&d_in, (size_t)n));
  FCU(s.alloc(&d_out, (size_t)n));
  FCU(s.alloc(&d_mm, 6));
  FCU(s.alloc(&d_idx, (size_t)n));
  FCU(s.alloc(&d_idx2, (size_t)n));
  FCU(s.alloc(&d_head, (size_t)n));
  FCU(s.alloc(&d_slot, (size_t)n));
  FCU(s.alloc(&d_key, (size_t)n));
  FCU(s.alloc(&d_key2, (size_t)n));
  FCU(cudaMemcpy(d_in, in4, (size_t)n * sizeof(float4), cudaMemcpyHostToDevice));
  const int init[6] = {INT_MAX, INT_MAX, INT_MAX, INT_MIN, INT_MIN, INT_MIN};
  FCU(cudaMemcpy(d_mm, init, sizeof(init), cudaMemcpyHostToDevice));
  minmax_kernel<<<blocks(n), 256>>>(d_in, n, d_mm, d_mm + 3, ix, iy, iz);
  int mm[6];
  FCU(cudaMemcpy(mm, d_mm, sizeof(mm), cudaMemcpyDeviceToHost));
  if (mm[0] > mm[3]) return LS_OK;  // no finite point
  const double cells = ((double)mm[3] - mm[0] + 1) * ((double)mm[4] - mm[1] + 1) * ((double)mm[5] - mm[2] + 1);
  if (cells >= 9.0e18) return LS_ERR_ARG;  // PCL: "Leaf size is too small for the input dataset"
  voxel_key_kernel<<<blocks(n), 256>>>(d_in, n, d_mm, d_mm + 3, ix, iy, iz, d_key, d_idx);
  size_t tmp_bytes = 0, tmp2 = 0;
  FCU(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, d_key, d_key2, d_idx, d_idx2, n));
  FCU(cub::DeviceScan::InclusiveSum(nullptr, tmp2, d_head, d_slot, n));
  void* d_tmp;
  FCU(s.alloc((unsigned char**)&d_tmp, tmp_bytes > tmp2 ? tmp_bytes : tmp2));
  FCU(cub::DeviceRadixSort::SortPairs(d_tmp, tmp_bytes, d_key, d_key2, d_idx, d_idx2, n));  // stable: input order inside a voxel
  voxel_head_kernel<<<blocks(n), 256>>>(d_key2, n, d_head);
  FCU(cub::DeviceScan::InclusiveSum(d_tmp, tmp2, d_head, d_slot, n));
  int m = 0;
  FCU(cudaMemcpy(&m, d_slot + (n - 1), sizeof(int), cudaMemcpyDeviceToHost));
  if (m > 0) {
    FCU(s.alloc(&d_sums, (size_t)m * 4));
    FCU(cudaMemset(d_sums, 0, (size_t)m * 4 * sizeof(unsigned long long)));
    voxel_accumulate_kernel<<<blocks(n), 256>>>(d_in, d_key2, d_idx2, d_slot, n, d_sums);
    voxel_centroid_kernel<<<blocks(m), 256>>>(d_sums, m, d_out);
    FCU(cudaMemcpy(out4, d_out, (size_t)m * sizeof(float4), cudaMemcpyDeviceToHost));
  }
  FCU(cudaGetLastError());
  *n_out = m;
  return LS_OK;
}

}  // extern "C"
