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
#include "ls_filters.cuh"

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

// Stable compaction by the exclusive scan `pos` of `keep`; normals (may be NULL) move with their points, and the thread of
// the last point stores the number kept (count may be NULL).
__global__ void compact_kernel(const float4* __restrict__ in, const float4* __restrict__ in_nrm, const int* __restrict__ keep,
                               const int* __restrict__ pos, int n, float4* __restrict__ out, float4* __restrict__ out_nrm,
                               int* __restrict__ count) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (keep[i]) {
      out[pos[i]] = in[i];
      if (in_nrm) out_nrm[pos[i]] = in_nrm[i];
    }
    if (count && i == n - 1) *count = pos[i] + keep[i];
  }
}

// ---- per-scan input filters (ls_point_filter): one flag kernel per run of point-wise tests, samplers on the rank the
// preceding exclusive scan gives each point
constexpr int kMaxPw = 8;
struct PwOp {
  int type, dim, remove_inside, pad;
  float dist;
  float box[6];
};
struct MaskStage {
  int n_pw;
  int sampler;  // 0, LS_PF_RANDOM_SAMPLING, LS_PF_FIX_STEP_SAMPLING or LS_PF_SAMPLING_SURFACE_NORMAL
  float prob;
  uint32_t salt;
  int step;
  PwOp pw[kMaxPw];
};

// ls_keep_point (ls_yaml.cpp) on the device
__device__ __forceinline__ bool keep_point_dev(uint32_t index, uint32_t salt, float prob) {
  if (!(prob < 1.0f)) return true;
  if (!(prob > 0.0f)) return false;
  uint32_t h = index * 0x9E3779B1u + salt * 0x85EBCA77u + 0x165667B1u;
  h ^= h >> 15; h *= 0x2C1B3C6Du;
  h ^= h >> 12; h *= 0x297A2D39u;
  h ^= h >> 15;
  return (double)h < (double)prob * 4294967296.0;
}

// float32, each operation rounded (the library is built with -fmad=false): fl(fl(fl(x*x) + fl(y*y)) + fl(z*z))
__device__ __forceinline__ bool pass_pw(const PwOp& o, const float4 p) {
  if (o.type == LS_PF_REMOVE_NAN) return !(isnan(p.x) || isnan(p.y) || isnan(p.z));
  if (o.type == LS_PF_MAX_DIST || o.type == LS_PF_MIN_DIST) {
    float v, lim;
    if (o.dim < 0) {
      const float a = p.x * p.x, b = p.y * p.y, c = p.z * p.z;
      v = a + b;
      v = v + c;
      lim = o.dist * o.dist;
    } else {
      v = fabsf(o.dim == 0 ? p.x : (o.dim == 1 ? p.y : p.z));
      lim = o.dist;
    }
    return o.type == LS_PF_MAX_DIST ? v < lim : v > lim;
  }
  // LS_PF_BOUNDING_BOX: a point on a face is outside
  const bool inside = o.box[0] < p.x && p.x < o.box[1] && o.box[2] < p.y && p.y < o.box[3] && o.box[4] < p.z && p.z < o.box[5];
  return o.remove_inside ? !inside : inside;
}

// keep_out[i] = keep_in[i] (1 if NULL) && sampler(rank[i] (i if NULL)) && every point-wise test.  keep_in may be keep_out.
__global__ void mask_kernel(const float4* __restrict__ pts, int n, const int* keep_in, const int* __restrict__ rank, MaskStage s,
                            int* keep_out) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    bool k = keep_in ? keep_in[i] != 0 : true;
    if (k && s.sampler) {
      const uint32_t r = rank ? (uint32_t)rank[i] : (uint32_t)i;
      k = s.sampler == LS_PF_FIX_STEP_SAMPLING ? (r % (uint32_t)s.step) == 0u : keep_point_dev(r, s.salt, s.prob);
    }
    if (k && s.n_pw) {
      const float4 p = pts[i];
      for (int j = 0; j < s.n_pw; ++j) k = k && pass_pw(s.pw[j], p);
    }
    keep_out[i] = k ? 1 : 0;
  }
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
// Normals (nrm != NULL) are summed the same way into sums[4..6] of a voxel (stride 7 then, 4 without).
__global__ void voxel_accumulate_kernel(const float4* __restrict__ in, const float4* __restrict__ nrm,
                                        const unsigned long long* __restrict__ key, const int* __restrict__ idx,
                                        const int* __restrict__ slot, int n, int stride,
                                        unsigned long long* __restrict__ sums /* per voxel: x, y, z, count[, nx, ny, nz] */) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (key[i] == ~0ull) continue;
    const float4 p = in[idx[i]];
    unsigned long long* s = sums + (size_t)stride * (size_t)(slot[i] - 1);
    atomicAdd(&s[0], (unsigned long long)__double2ll_rn((double)p.x * 16777216.0));
    atomicAdd(&s[1], (unsigned long long)__double2ll_rn((double)p.y * 16777216.0));
    atomicAdd(&s[2], (unsigned long long)__double2ll_rn((double)p.z * 16777216.0));
    atomicAdd(&s[3], 1ull);
    if (nrm) {
      const float4 q = nrm[idx[i]];
      atomicAdd(&s[4], (unsigned long long)__double2ll_rn((double)q.x * 16777216.0));
      atomicAdd(&s[5], (unsigned long long)__double2ll_rn((double)q.y * 16777216.0));
      atomicAdd(&s[6], (unsigned long long)__double2ll_rn((double)q.z * 16777216.0));
    }
  }
}

__global__ void voxel_centroid_kernel(const unsigned long long* __restrict__ sums, int m, int stride, float4* __restrict__ out,
                                      float4* __restrict__ out_nrm) {
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < m; v += gridDim.x * blockDim.x) {
    const unsigned long long* s = sums + (size_t)stride * (size_t)v;
    const double c = (double)s[3] * 16777216.0;
    out[v] = make_float4((float)((double)(long long)s[0] / c), (float)((double)(long long)s[1] / c),
                         (float)((double)(long long)s[2] / c), 1.0f);
    if (out_nrm)  // mean of the voxel's normals, one rounding, not renormalised
      out_nrm[v] = make_float4((float)((double)(long long)s[4] / c), (float)((double)(long long)s[5] / c),
                               (float)((double)(long long)s[6] / c), 0.0f);
  }
}

// pcl::VoxelGrid's minimum point number: keep[v] = 1 iff voxel v holds at least min_points points
__global__ void voxel_min_count_kernel(const unsigned long long* __restrict__ sums, int m, int stride, int min_points,
                                       int* __restrict__ keep) {
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < m; v += gridDim.x * blockDim.x)
    keep[v] = sums[(size_t)stride * (size_t)v + 3] >= (unsigned long long)min_points ? 1 : 0;
}

// ---- local map (ls_local_map_*): the map maintenance of LaserSlamWorker
// The scan of a ring slot moved into the world frame (xform3: the xform_point order of ls_map_assemble; an exact identity
// copies verbatim), and keep[i] = 0 for a ground point: (double)z <= z_min when remove_ground.
struct Xform16 {
  float T[16];
};
__global__ void local_map_append_kernel(const float4* __restrict__ in, int n, Xform16 T, int identity, int remove_ground,
                                        double z_min, float4* __restrict__ out, int* __restrict__ keep) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    float4 p = in[i];
    if (!identity) {
      float x, y, z;
      xform3(T.T, p.x, p.y, p.z, x, y, z);
      p.x = x; p.y = y; p.z = z;
    }
    out[i] = p;
    keep[i] = (!remove_ground || (double)p.z > z_min) ? 1 : 0;
  }
}

// updateLocalMap's move, in place: every thread reads its point and writes it back (no restrict pointers)
__global__ void local_map_transform_kernel(float4* pts, int n, Xform16 T) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    float4 p = pts[i];
    float x, y, z;
    xform3(T.T, p.x, p.y, p.z, x, y, z);
    p.x = x; p.y = y; p.z = z;
    pts[i] = p;
  }
}

// Two-way split of the voxelised map by the cylinder: flag[i] = inside (d_xy^2 <= r^2 and |dz| <= h/2) in the low word,
// outside (>= on either) in the high word -- a point exactly on the boundary is both, as in the reference.  One 64-bit
// exclusive scan then places both streams at once.
__global__ void split_flag_kernel(const float4* __restrict__ in, int n, double cx, double cy, double cz, double r2, double hh,
                                  unsigned long long* __restrict__ flag) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float4 p = in[i];
    const double dx = (double)p.x - cx, dy = (double)p.y - cy;
    const double d2 = dx * dx + dy * dy;
    const double dz = fabs((double)p.z - cz);
    const bool inside = d2 <= r2 && dz <= hh;
    const bool outside = d2 >= r2 || dz >= hh;
    flag[i] = (inside ? 1ull : 0ull) | (outside ? (1ull << 32) : 0ull);
  }
}

// Scatter by the exclusive scan `pos` of `flag`: inside points to in_out[lo], outside points to out_out[hi]; the thread of
// the last point stores both totals in counts[0..1].
__global__ void split_scatter_kernel(const float4* __restrict__ in, const unsigned long long* __restrict__ flag,
                                     const unsigned long long* __restrict__ pos, int n, float4* __restrict__ in_out,
                                     float4* __restrict__ out_out, int* __restrict__ counts) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const unsigned long long f = flag[i], q = pos[i];
    if (f & 0xffffffffull) in_out[q & 0xffffffffull] = in[i];
    if (f >> 32) out_out[q >> 32] = in[i];
    if (i == n - 1) {
      const unsigned long long t = q + f;
      counts[0] = (int)(t & 0xffffffffull);
      counts[1] = (int)(t >> 32);
    }
  }
}

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
  const size_t bytes = (size_t)n * point_step;
  ls::Buffer<unsigned char> d_in;
  ls::Buffer<float4> d_out;
  FCU(d_in.reserve(bytes, bytes));
  FCU(d_out.reserve(n, n));
  FCU(cudaMemcpy(d_in.get(), data, bytes, cudaMemcpyHostToDevice));
  ingest_kernel<<<blocks(n), 256>>>(d_in.get(), point_step, off_x, off_y, off_z, n, d_out.get());
  FCU(cudaMemcpy(out4, d_out.get(), (size_t)n * sizeof(float4), cudaMemcpyDeviceToHost));
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
  ls::Buffer<float4> d_in, d_out;
  ls::Buffer<int> d_keep, d_pos;
  FCU(d_in.reserve(n, n));
  FCU(d_out.reserve(n, n));
  FCU(d_keep.reserve(n, n));
  FCU(d_pos.reserve(n, n));
  FCU(cudaMemcpy(d_in.get(), in4, (size_t)n * sizeof(float4), cudaMemcpyHostToDevice));
  cylinder_flag_kernel<<<blocks(n), 256>>>(d_in.get(), n, center[0], center[1], center[2], radius_m * radius_m, height_m / 2.0,
                                          remove_points_inside, d_keep.get());
  size_t tmp_bytes = 0;
  FCU(cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, d_keep.get(), d_pos.get(), n));
  ls::Buffer<unsigned char> d_tmp;
  FCU(d_tmp.reserve(tmp_bytes, tmp_bytes));
  FCU(cub::DeviceScan::ExclusiveSum(d_tmp.get(), tmp_bytes, d_keep.get(), d_pos.get(), n));
  compact_kernel<<<blocks(n), 256>>>(d_in.get(), nullptr, d_keep.get(), d_pos.get(), n, d_out.get(), nullptr, nullptr);
  int last_pos = 0, last_keep = 0;
  FCU(cudaMemcpy(&last_pos, d_pos.get() + (n - 1), sizeof(int), cudaMemcpyDeviceToHost));
  FCU(cudaMemcpy(&last_keep, d_keep.get() + (n - 1), sizeof(int), cudaMemcpyDeviceToHost));
  *n_out = last_pos + last_keep;
  FCU(cudaMemcpy(out4, d_out.get(), (size_t)*n_out * sizeof(float4), cudaMemcpyDeviceToHost));
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
  const size_t np = (size_t)n_packets;
  ls::Buffer<float4> d_in, d_out;
  ls::Buffer<int> d_offs;
  ls::Buffer<float> d_T;
  FCU(d_in.reserve(m, m));
  FCU(d_out.reserve(m, m));
  FCU(d_offs.reserve(np + 1, np + 1));
  FCU(d_T.reserve(16 * (np + 1), 16 * (np + 1)));
  FCU(cudaMemcpy(d_in.get(), points4, (size_t)m * sizeof(float4), cudaMemcpyHostToDevice));
  FCU(cudaMemcpy(d_offs.get(), packet_offsets, (np + 1) * sizeof(int), cudaMemcpyHostToDevice));
  FCU(cudaMemcpy(d_T.get(), T_packets, 16 * np * sizeof(float), cudaMemcpyHostToDevice));
  FCU(cudaMemcpy(d_T.get() + 16 * np, T_final, 16 * sizeof(float), cudaMemcpyHostToDevice));
  deskew_kernel<<<blocks(m), 256>>>(d_in.get(), m, d_offs.get(), n_packets, d_T.get(), d_T.get() + 16 * np, d_out.get());
  FCU(cudaGetLastError());
  FCU(cudaMemcpy(out4, d_out.get(), (size_t)m * sizeof(float4), cudaMemcpyDeviceToHost));
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
  const size_t tmp_bytes = lsf::voxel_temp_bytes(n);
  ls::Buffer<float4> d_in, d_out;
  ls::Buffer<int> mm, idx, idx2, head, slot;
  ls::Buffer<unsigned long long> key, key2, sums;
  ls::Buffer<unsigned char> tmp;
  FCU(d_in.reserve(n, n));
  FCU(d_out.reserve(n, n));
  FCU(mm.reserve(6, 6));
  FCU(idx.reserve(n, n));
  FCU(idx2.reserve(n, n));
  FCU(head.reserve(n, n));
  FCU(slot.reserve(n, n));
  FCU(key.reserve(n, n));
  FCU(key2.reserve(n, n));
  FCU(sums.reserve((size_t)n * 4, (size_t)n * 4));
  FCU(tmp.reserve(tmp_bytes, tmp_bytes));
  lsf::VoxelBuffers vb;
  vb.mm = mm.get();
  vb.key = key.get();
  vb.key2 = key2.get();
  vb.sums = sums.get();
  vb.idx = idx.get();
  vb.idx2 = idx2.get();
  vb.head = head.get();
  vb.slot = slot.get();
  vb.tmp = tmp.get();
  vb.tmp_bytes = tmp_bytes;
  FCU(cudaMemcpy(d_in.get(), in4, (size_t)n * sizeof(float4), cudaMemcpyHostToDevice));
  uint64_t launches = 0;
  int m = 0;
  const int rc = lsf::enqueue_voxel_grid(d_in.get(), nullptr, n, leaf_size, d_out.get(), nullptr, 0, vb, 0, &m, &launches);
  if (rc != LS_OK) return rc;
  if (m > 0) FCU(cudaMemcpy(out4, d_out.get(), (size_t)m * sizeof(float4), cudaMemcpyDeviceToHost));
  *n_out = m;
  return LS_OK;
}

}  // extern "C"

// ---- per-scan input filters: what ls_api.cu enqueues ----------------------------------------------------------------
namespace lsf {

namespace {
bool is_pointwise(int type) {
  return type == LS_PF_REMOVE_NAN || type == LS_PF_MAX_DIST || type == LS_PF_MIN_DIST || type == LS_PF_BOUNDING_BOX;
}
size_t scan_temp_bytes(int n) {
  size_t a = 0, b = 0, c = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, a, (const int*)nullptr, (int*)nullptr, n);
  cub::DeviceScan::InclusiveSum(nullptr, b, (const int*)nullptr, (int*)nullptr, n);
  cub::DeviceScan::ExclusiveSum(nullptr, c, (const unsigned long long*)nullptr, (unsigned long long*)nullptr, n);  // split
  a = a > b ? a : b;
  return a > c ? a : c;
}
}  // namespace

bool is_mask_filter(int type) {
  return is_pointwise(type) || type == LS_PF_RANDOM_SAMPLING || type == LS_PF_FIX_STEP_SAMPLING;
}

size_t voxel_temp_bytes(int n) {
  size_t sort = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, sort, (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                  (const int*)nullptr, (int*)nullptr, n);
  const size_t scan = scan_temp_bytes(n);
  return sort > scan ? sort : scan;
}

cudaError_t reserve(ChainBuffers& b, int n) {
  if (b.pts[0].get() && (size_t)n <= b.pts[0].capacity()) return cudaSuccess;
  b = ChainBuffers();  // the old arrays go before the new ones are allocated
  const int cap = n + n / 8 + 1024;
  const size_t c = (size_t)cap, tmp_bytes = voxel_temp_bytes(cap);
  cudaError_t e;
  if ((e = b.pts[0].reserve(c, c)) || (e = b.pts[1].reserve(c, c)) || (e = b.nrm[0].reserve(c, c)) ||
      (e = b.nrm[1].reserve(c, c)) || (e = b.keep.reserve(c, c)) || (e = b.pos.reserve(c, c)) || (e = b.small.reserve(8, 8)) ||
      (e = b.key.reserve(c, c)) || (e = b.key2.reserve(c, c)) || (e = b.idx.reserve(c, c)) || (e = b.idx2.reserve(c, c)) ||
      (e = b.head.reserve(c, c)) || (e = b.slot.reserve(c, c)) || (e = b.sums.reserve(7 * c, 7 * c)) ||
      (e = b.tmp.reserve(tmp_bytes, tmp_bytes))) {
    b = ChainBuffers();
    return e;
  }
  b.tmp_bytes = tmp_bytes;
  return cudaSuccess;
}

VoxelBuffers voxel_buffers(const ChainBuffers& b) {
  VoxelBuffers v;
  v.mm = b.small.get();
  v.key = b.key.get();
  v.key2 = b.key2.get();
  v.sums = b.sums.get();
  v.idx = b.idx.get();
  v.idx2 = b.idx2.get();
  v.head = b.head.get();
  v.slot = b.slot.get();
  v.tmp = b.tmp.get();
  v.tmp_bytes = b.tmp_bytes;
  return v;
}

cudaError_t enqueue_mask_run(const ls_point_filter* filters, int n_filters, const float4* pts, const float4* nrm, int n,
                             float4* out, float4* out_nrm, ChainBuffers& b, cudaStream_t st, int* used, uint64_t* launches) {
  cudaError_t e;
  int j = 0;
  bool have_keep = false;
  while (j < n_filters && (j == 0 || is_mask_filter(filters[j].type))) {
    MaskStage s;
    memset(&s, 0, sizeof(s));
    const int* rank = nullptr;
    const int t = filters[j].type;
    if (!is_pointwise(t)) {  // a sampler: rank of every point in the cloud entering it = exclusive scan of the flags so far
      if (have_keep) {
        if ((e = cub::DeviceScan::ExclusiveSum(b.tmp.get(), b.tmp_bytes, b.keep.get(), b.pos.get(), n, st))) return e;
        rank = b.pos.get();
      }
      s.sampler = t;
      s.prob = filters[j].prob;
      s.salt = t == LS_PF_SAMPLING_SURFACE_NORMAL ? 0x5a17u : 0x7e11u;
      s.step = filters[j].step;
      ++j;
    }
    while (j < n_filters && is_pointwise(filters[j].type) && s.n_pw < kMaxPw) {
      const ls_point_filter& f = filters[j++];
      PwOp& o = s.pw[s.n_pw++];
      o.type = f.type;
      o.dim = f.dim;
      o.remove_inside = f.remove_inside;
      o.dist = f.dist;
      for (int a = 0; a < 6; ++a) o.box[a] = f.box[a];
    }
    mask_kernel<<<blocks(n), 256, 0, st>>>(pts, n, have_keep ? b.keep.get() : nullptr, rank, s, b.keep.get());
    ++*launches;
    if ((e = cudaGetLastError())) return e;
    have_keep = true;
  }
  *used = j;
  if ((e = cub::DeviceScan::ExclusiveSum(b.tmp.get(), b.tmp_bytes, b.keep.get(), b.pos.get(), n, st))) return e;
  compact_kernel<<<blocks(n), 256, 0, st>>>(pts, nrm, b.keep.get(), b.pos.get(), n, out, out_nrm, b.small.get() + 6);
  ++*launches;
  return cudaGetLastError();
}

int enqueue_voxel_grid(const float4* in, const float4* in_nrm, int n, const float leaf[3], float4* out, float4* out_nrm,
                       int min_points, const VoxelBuffers& b, cudaStream_t st, int* m_out, uint64_t* launches) {
  *m_out = 0;
  const bool min_filter = min_points > 1;  // 0 and 1 keep every voxel: exactly the kernels of the plain grid
  if (min_filter && (in_nrm || !b.cent)) return LS_ERR_ARG;
  if (n == 0) return LS_OK;
  const float ix = 1.0f / leaf[0], iy = 1.0f / leaf[1], iz = 1.0f / leaf[2];  // PCL: inverse_leaf_size_
  const int init[6] = {INT_MAX, INT_MAX, INT_MAX, INT_MIN, INT_MIN, INT_MIN};
  FCU(cudaMemcpyAsync(b.mm, init, sizeof(init), cudaMemcpyHostToDevice, st));
  minmax_kernel<<<blocks(n), 256, 0, st>>>(in, n, b.mm, b.mm + 3, ix, iy, iz);
  ++*launches;
  int mm[6];
  FCU(cudaMemcpyAsync(mm, b.mm, sizeof(mm), cudaMemcpyDeviceToHost, st));
  FCU(cudaStreamSynchronize(st));
  if (mm[0] > mm[3]) return LS_OK;  // no finite point
  const double cells = ((double)mm[3] - mm[0] + 1) * ((double)mm[4] - mm[1] + 1) * ((double)mm[5] - mm[2] + 1);
  if (cells >= 9.0e18) return LS_ERR_ARG;  // PCL: "Leaf size is too small for the input dataset"
  voxel_key_kernel<<<blocks(n), 256, 0, st>>>(in, n, b.mm, b.mm + 3, ix, iy, iz, b.key, b.idx);
  ++*launches;
  size_t bytes = b.tmp_bytes;
  // stable: input order inside a voxel
  FCU(cub::DeviceRadixSort::SortPairs(b.tmp, bytes, b.key, b.key2, b.idx, b.idx2, n, 0, (int)sizeof(unsigned long long) * 8, st));
  voxel_head_kernel<<<blocks(n), 256, 0, st>>>(b.key2, n, b.head);
  ++*launches;
  bytes = b.tmp_bytes;
  FCU(cub::DeviceScan::InclusiveSum(b.tmp, bytes, b.head, b.slot, n, st));
  int m = 0;
  FCU(cudaMemcpyAsync(&m, b.slot + (n - 1), sizeof(int), cudaMemcpyDeviceToHost, st));
  FCU(cudaStreamSynchronize(st));
  if (m > 0) {
    const int stride = in_nrm ? 7 : 4;
    FCU(cudaMemsetAsync(b.sums, 0, (size_t)m * stride * sizeof(unsigned long long), st));
    voxel_accumulate_kernel<<<blocks(n), 256, 0, st>>>(in, in_nrm, b.key2, b.idx2, b.slot, n, stride, b.sums);
    voxel_centroid_kernel<<<blocks(m), 256, 0, st>>>(b.sums, m, stride, min_filter ? b.cent : out, in_nrm ? out_nrm : nullptr);
    *launches += 2;
    if (min_filter) {  // flag, scan, stable compaction of the voxels (head / slot are free again after the accumulation)
      voxel_min_count_kernel<<<blocks(m), 256, 0, st>>>(b.sums, m, stride, min_points, b.head);
      bytes = b.tmp_bytes;
      FCU(cub::DeviceScan::ExclusiveSum(b.tmp, bytes, b.head, b.slot, m, st));
      compact_kernel<<<blocks(m), 256, 0, st>>>(b.cent, nullptr, b.head, b.slot, m, out, nullptr, b.mm);
      *launches += 2;
      FCU(cudaMemcpyAsync(&m, b.mm, sizeof(int), cudaMemcpyDeviceToHost, st));
      FCU(cudaStreamSynchronize(st));
    }
  }
  FCU(cudaGetLastError());
  *m_out = m;
  return LS_OK;
}

int enqueue_local_map_append(const float4* scan, int n, const float T[16], bool identity, bool remove_ground, double z_min,
                             float4* local_tail, float4* queue_tail, ChainBuffers& b, cudaStream_t st, int* kept,
                             uint64_t* launches) {
  *kept = 0;
  if (n == 0) return LS_OK;
  Xform16 x;
  memcpy(x.T, T, sizeof(x.T));
  local_map_append_kernel<<<blocks(n), 256, 0, st>>>(scan, n, x, identity ? 1 : 0, remove_ground ? 1 : 0, z_min, b.pts[0].get(),
                                                     b.keep.get());
  size_t bytes = b.tmp_bytes;
  FCU(cub::DeviceScan::ExclusiveSum(b.tmp.get(), bytes, b.keep.get(), b.pos.get(), n, st));
  // one compaction fills both: the local map's tail as the points, the queue's tail as the "normals" of the same points
  compact_kernel<<<blocks(n), 256, 0, st>>>(b.pts[0].get(), b.pts[0].get(), b.keep.get(), b.pos.get(), n, local_tail, queue_tail,
                                            b.small.get() + 6);
  *launches += 2;
  FCU(cudaGetLastError());
  FCU(cudaMemcpyAsync(kept, b.small.get() + 6, sizeof(int), cudaMemcpyDeviceToHost, st));
  FCU(cudaStreamSynchronize(st));
  return LS_OK;
}

int enqueue_transform_in_place(float4* pts, int n, const float T[16], cudaStream_t st, uint64_t* launches) {
  if (n == 0) return LS_OK;
  Xform16 x;
  memcpy(x.T, T, sizeof(x.T));
  local_map_transform_kernel<<<blocks(n), 256, 0, st>>>(pts, n, x);
  ++*launches;
  FCU(cudaGetLastError());
  return LS_OK;
}

int enqueue_cylinder_crop(const float4* in, int n, const double center[3], double radius_m, double height_m, float4* out,
                          ChainBuffers& b, cudaStream_t st, int* kept, uint64_t* launches) {
  *kept = 0;
  if (n == 0) return LS_OK;
  cylinder_flag_kernel<<<blocks(n), 256, 0, st>>>(in, n, center[0], center[1], center[2], radius_m * radius_m, height_m / 2.0, 0,
                                                  b.keep.get());
  size_t bytes = b.tmp_bytes;
  FCU(cub::DeviceScan::ExclusiveSum(b.tmp.get(), bytes, b.keep.get(), b.pos.get(), n, st));
  compact_kernel<<<blocks(n), 256, 0, st>>>(in, nullptr, b.keep.get(), b.pos.get(), n, out, nullptr, b.small.get() + 6);
  *launches += 2;
  FCU(cudaGetLastError());
  FCU(cudaMemcpyAsync(kept, b.small.get() + 6, sizeof(int), cudaMemcpyDeviceToHost, st));
  FCU(cudaStreamSynchronize(st));
  return LS_OK;
}

int enqueue_cylinder_split(const float4* in, int n, const double center[3], double radius_m, double height_m, float4* inside,
                           float4* outside, ChainBuffers& b, cudaStream_t st, int* n_inside, int* n_outside, uint64_t* launches) {
  *n_inside = *n_outside = 0;
  if (n == 0) return LS_OK;
  split_flag_kernel<<<blocks(n), 256, 0, st>>>(in, n, center[0], center[1], center[2], radius_m * radius_m, height_m / 2.0,
                                               b.key.get());
  size_t bytes = b.tmp_bytes;
  FCU(cub::DeviceScan::ExclusiveSum(b.tmp.get(), bytes, b.key.get(), b.key2.get(), n, st));
  split_scatter_kernel<<<blocks(n), 256, 0, st>>>(in, b.key.get(), b.key2.get(), n, inside, outside, b.small.get() + 6);
  *launches += 2;
  FCU(cudaGetLastError());
  int c[2];
  FCU(cudaMemcpyAsync(c, b.small.get() + 6, sizeof(c), cudaMemcpyDeviceToHost, st));
  FCU(cudaStreamSynchronize(st));
  *n_inside = c[0];
  *n_outside = c[1];
  return LS_OK;
}

}  // namespace lsf
