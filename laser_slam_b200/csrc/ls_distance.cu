// Euclidean distance map of the resident occupancy map: octomap's DynamicEDTOctomap (dynamicEDT3D) over the finest cells of
// an axis-aligned box, recomputed in full at every update.  The rules are DESIGN.md §4b'''''''''.  Per update:
//   (a) dt_extract_kernel  one block per pool brick, one thread per voxel; a brick whose key range misses the box leaves at
//                          once.  The grid (one byte per cell) was set to 0, or to 1 in unknown-as-occupied mode; a voxel
//                          inside the box writes 1 when occupied (known, v >= L_occ), or 0 when known free in that mode
//   (b) dt_row_kernel      one warp per x row: the nearest obstacle at or left of each cell (a max-scan over the warp with a
//                          carry), then at or right of it (a min-scan from the right); the left one wins ties.  Writes
//                          s = dx^2 and the obstacle's cell index, or no site when s > M; counts the obstacles
//   (c) dt_col_kernel      one thread per column over adjacent x, once along y and once along z: Meijster's lower envelope
//                          of the parabolas f(u) + (x - u)^2 of the column's sites (a stack of (site, start, f(site)) per
//                          column in scratch laid out [entry][column]), then the backward scan that reads each cell's
//                          value off it
// A site is dropped as soon as its partial sum exceeds M: every partial sum of a cell whose final s <= M is <= s, so the
// capped field is exact while every stored value fits int32.  Sums are formed in int64.  Ties: a parabola leaves the stack
// only when strictly worse, and the intersection's floor hands the tie point to the lower site, so every 1-D pass takes the
// minimal value first and the lower coordinate second; over x, y, z in turn that is the smallest packed key.
// Queries and the download read the last field only.
#include <climits>
#include <cmath>
#include <cstdint>
#include <cstring>

#include <cuda_runtime.h>

#include "../../include/ls_b200.h"
#include "ls_occupancy.cuh"

namespace lso {
namespace {

constexpr int kNoSite = INT_MAX;  // the value of a cell without a site in (b) and (c)
constexpr unsigned kNanBits = 0x7fc00000u;

struct Box {
  int kmin[3], size[3];
};

__global__ void __launch_bounds__(512) dt_extract_kernel(const unsigned long long* __restrict__ bkey,
                                                         const unsigned* __restrict__ known, const float* __restrict__ lo,
                                                         Box B, float l_occ, int unknown_occ, unsigned char* __restrict__ grid) {
  const int b = blockIdx.x, t = threadIdx.x;
  int base[3];  // the brick's first voxel
  voxel_keys(bkey[b], 0, base);
  for (int a = 0; a < 3; ++a)
    if (base[a] + 7 < B.kmin[a] || base[a] > B.kmin[a] + B.size[a] - 1) return;  // the whole block: the brick misses the box
  const int c[3] = {base[0] + (t & 7) - B.kmin[0], base[1] + ((t >> 3) & 7) - B.kmin[1], base[2] + (t >> 6) - B.kmin[2]};
  for (int a = 0; a < 3; ++a)
    if (c[a] < 0 || c[a] >= B.size[a]) return;
  if (!((known[(size_t)b * 16 + (t >> 5)] >> (t & 31)) & 1u)) return;
  const bool occ = lo[(size_t)b * 512 + t] >= l_occ;
  const size_t cell = ((size_t)c[2] * B.size[1] + c[1]) * B.size[0] + c[0];
  if (occ && !unknown_occ) grid[cell] = 1;
  if (!occ && unknown_occ) grid[cell] = 0;
}

__device__ __forceinline__ int warp_max_scan(int v) {
  const int lane = threadIdx.x & 31;
  for (int o = 1; o < 32; o <<= 1) {
    const int u = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v = max(v, u);
  }
  return v;
}

__device__ __forceinline__ int warp_min_suffix(int v) {
  const int lane = threadIdx.x & 31;
  for (int o = 1; o < 32; o <<= 1) {
    const int u = __shfl_down_sync(0xffffffffu, v, o);
    if (lane + o < 32) v = min(v, u);
  }
  return v;
}

// (b): rows = sy * sz, one warp each.  site holds the left obstacle between the two sweeps.
__global__ void dt_row_kernel(const unsigned char* __restrict__ grid, int sx, long long rows, long long M, int* __restrict__ val,
                              int* __restrict__ site, unsigned long long* __restrict__ obstacles) {
  const long long r = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (r >= rows) return;  // whole warps only: blockDim is a multiple of 32
  const int lane = threadIdx.x & 31;
  const size_t base = (size_t)r * sx;
  unsigned long long count = 0;
  int carry = -1;
  for (int x0 = 0; x0 < sx; x0 += 32) {
    const int x = x0 + lane;
    const bool ob = x < sx && grid[base + x];
    count += __popc(__ballot_sync(0xffffffffu, ob));
    const int left = max(warp_max_scan(ob ? x : -1), carry);
    carry = __shfl_sync(0xffffffffu, left, 31);
    if (x < sx) site[base + x] = left;
  }
  carry = INT_MAX;
  for (int x0 = (sx - 1) & ~31; x0 >= 0; x0 -= 32) {
    const int x = x0 + lane;
    const bool ob = x < sx && grid[base + x];
    const int right = min(warp_min_suffix(ob ? x : INT_MAX), carry);
    carry = __shfl_sync(0xffffffffu, right, 0);
    if (x < sx) {
      const int left = site[base + x];
      int s = -1;
      if (left >= 0 && (right == INT_MAX || x - left <= right - x)) s = left;
      else if (right != INT_MAX) s = right;
      const long long d = s < 0 ? 0 : (long long)(x - s) * (x - s);
      const bool keep = s >= 0 && d <= M;
      val[base + x] = keep ? (int)d : kNoSite;
      site[base + x] = keep ? (int)(base + s) : -1;
    }
  }
  if (lane == 0 && count) atomicAdd(obstacles, count);
}

__device__ __forceinline__ long long floor_div(long long a, long long b) {  // b > 0
  const long long q = a / b;
  return (q * b > a) ? q - 1 : q;
}

// (c): one thread per column.  Column i starts at (i / sx) * outer + i % sx and has n cells `stride` apart.  stack: entry q of
// column i at q * cols + i, {site position | start << 16, f(site)}.  last: the z pass, storing M and no obstacle for a cell
// without a site.
__global__ void dt_col_kernel(const int* __restrict__ gin, const int* __restrict__ sin, int* __restrict__ gout,
                              int* __restrict__ sout, uint2* __restrict__ stack, long long cols, int sx, long long outer,
                              long long stride, int n, long long M, int last) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= cols) return;
  const size_t base = (size_t)(i / sx) * outer + (size_t)(i % sx);
  int q = -1, ts = 0, tt = 0;
  long long tg = 0;
  for (int u = 0; u < n; ++u) {
    const int g = gin[base + (size_t)u * stride];
    if (g == kNoSite) continue;
    while (q >= 0) {
      const long long a = tt - ts, b = tt - u;
      if (a * a + tg <= b * b + g) break;
      if (--q >= 0) {
        const uint2 e = stack[(size_t)q * cols + i];
        ts = (int)(e.x & 0xffffu), tt = (int)(e.x >> 16), tg = (int)e.y;
      }
    }
    if (q < 0) {
      q = 0, ts = u, tt = 0, tg = g;
      continue;
    }
    const long long w = 1 + floor_div((long long)u * u - (long long)ts * ts + g - tg, 2LL * (u - ts));
    if (w < n) {
      stack[(size_t)q * cols + i] = make_uint2((unsigned)ts | ((unsigned)tt << 16), (unsigned)tg);
      ++q, ts = u, tt = (int)w, tg = g;
    }
  }
  for (int u = n - 1; u >= 0; --u) {
    const size_t o = base + (size_t)u * stride;
    long long d = M + 1;
    if (q >= 0) d = (long long)(u - ts) * (u - ts) + tg;
    const bool keep = d <= M;
    gout[o] = keep ? (int)d : (last ? (int)M : kNoSite);
    sout[o] = keep ? sin[base + (size_t)ts * stride] : -1;
    if (q >= 0 && u == tt && --q >= 0) {
      const uint2 e = stack[(size_t)q * cols + i];
      ts = (int)(e.x & 0xffffu), tt = (int)(e.x >> 16), tg = (int)e.y;
    }
  }
}

// One thread per point: the key of each float coordinate (key_of), inside the box or -1 / NaN.
__global__ void dt_query_kernel(const float* __restrict__ pts3, int n, Box B, double inv, double res, const int* __restrict__ val,
                                const int* __restrict__ site, float* __restrict__ dist, int* __restrict__ sq,
                                float* __restrict__ obst3, unsigned long long* __restrict__ outside) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  bool out = false;
  if (i < n) {
    int c[3];
    bool in = true;
    for (int a = 0; a < 3; ++a) {
      int k;
      if (!key_of(inv, pts3[3 * (size_t)i + a], k)) {
        in = false;
        continue;
      }
      c[a] = k - B.kmin[a];
      if (c[a] < 0 || c[a] >= B.size[a]) in = false;
    }
    int s = -1, w = -1;
    if (in) {
      const size_t cell = ((size_t)c[2] * B.size[1] + c[1]) * B.size[0] + c[0];
      s = val[cell];
      w = site[cell];
    }
    out = !in;
    if (dist) dist[i] = in ? (float)((double)(float)sqrt((double)s) * res) : -1.0f;
    if (sq) sq[i] = s;
    if (obst3) {
      if (w >= 0) {
        const int wx = w % B.size[0], wy = (w / B.size[0]) % B.size[1], wz = w / B.size[0] / B.size[1];
        obst3[3 * (size_t)i] = centre_of(B.kmin[0] + wx, res);
        obst3[3 * (size_t)i + 1] = centre_of(B.kmin[1] + wy, res);
        obst3[3 * (size_t)i + 2] = centre_of(B.kmin[2] + wz, res);
      } else {
        for (int a = 0; a < 3; ++a) obst3[3 * (size_t)i + a] = __uint_as_float(kNanBits);
      }
    }
  }
  const unsigned o = __ballot_sync(0xffffffffu, out);
  if ((threadIdx.x & 31) == 0 && o) atomicAdd(outside, (unsigned long long)__popc(o));
}

// The obstacle of each cell as a packed key, all ones when none.
__global__ void dt_keys_kernel(const int* __restrict__ site, long long cells, Box B, unsigned long long* __restrict__ keys) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= cells) return;
  const int w = site[i];
  if (w < 0) {
    keys[i] = ~0ull;
    return;
  }
  const int wx = w % B.size[0], wy = (w / B.size[0]) % B.size[1], wz = w / B.size[0] / B.size[1];
  keys[i] = pack(B.kmin[0] + wx, B.kmin[1] + wy, B.kmin[2] + wz);
}

Box box_of(const DistanceField& f) {
  Box B;
  for (int a = 0; a < 3; ++a) B.kmin[a] = f.kmin[a], B.size[a] = f.size[a];
  return B;
}

}  // namespace

int distance_reserve(DistanceField& f, long long cells) {
  const size_t c = (size_t)cells;
  cudaError_t e = f.grid.reserve(c, c);
  for (int k = 0; k < 2 && e == cudaSuccess; ++k) {
    e = f.val[k].reserve(c, c);
    if (e == cudaSuccess) e = f.site[k].reserve(c, c);
  }
  if (e == cudaSuccess) e = f.stack.reserve(c, c);
  if (e == cudaSuccess) e = f.cnt_dev.reserve(1, 1);
  if (e == cudaSuccess) e = f.cnt_host.reserve(1, 1);
  if (e != cudaSuccess) {
    f.grid.reset(), f.stack.reset();
    for (int k = 0; k < 2; ++k) f.val[k].reset(), f.site[k].reset();
    return code(e);
  }
  return LS_OK;
}

int distance_update(DistanceField& f, const Map& m, float l_occ, bool unknown_occ, cudaStream_t st, uint64_t* launches) {
  const Box B = box_of(f);
  const long long sx = f.size[0], sy = f.size[1], sz = f.size[2], cells = f.cells, M = f.M;
  LSO_TRY(cudaMemsetAsync(f.grid.get(), unknown_occ ? 1 : 0, (size_t)cells, st));
  LSO_TRY(cudaMemsetAsync(f.cnt_dev.get(), 0, sizeof(unsigned long long), st));
  if (m.pool_n > 0) {
    dt_extract_kernel<<<m.pool_n, 512, 0, st>>>(m.bkey.get(), m.known.get(), m.lo.get(), B, l_occ, unknown_occ ? 1 : 0,
                                                f.grid.get());
    LSO_LAUNCHED();
  }
  dt_row_kernel<<<blocks(sy * sz * 32, 256), 256, 0, st>>>(f.grid.get(), (int)sx, sy * sz, M, f.val[0].get(), f.site[0].get(),
                                                           f.cnt_dev.get());
  LSO_LAUNCHED();
  // y: columns (x, z), outer sx * sy; z: columns (x, y), outer sx
  dt_col_kernel<<<blocks(sx * sz, 128), 128, 0, st>>>(f.val[0].get(), f.site[0].get(), f.val[1].get(), f.site[1].get(),
                                                      f.stack.get(), sx * sz, (int)sx, sx * sy, sx, (int)sy, M, 0);
  LSO_LAUNCHED();
  dt_col_kernel<<<blocks(sx * sy, 128), 128, 0, st>>>(f.val[1].get(), f.site[1].get(), f.val[0].get(), f.site[0].get(),
                                                      f.stack.get(), sx * sy, (int)sx, sx, sx * sy, (int)sz, M, 1);
  LSO_LAUNCHED();
  LSO_TRY(cudaMemcpyAsync(f.cnt_host.get(), f.cnt_dev.get(), sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  LSO_TRY(cudaStreamSynchronize(st));
  f.obstacles = (long long)*f.cnt_host.get();
  return LS_OK;
}

int distance_query(DistanceField& f, const float* pts3, int n, float* dist, int* sq, float* obst3, long long* outside,
                   cudaStream_t st, uint64_t* launches) {
  *outside = 0;
  if (n <= 0) return LS_OK;
  const size_t N = (size_t)n;
  size_t off = 0;
  const size_t o_cnt = take(off, sizeof(unsigned long long)), o_p = take(off, 12 * N), o_d = dist ? take(off, 4 * N) : 0,
               o_s = sq ? take(off, 4 * N) : 0, o_o = obst3 ? take(off, 12 * N) : 0;
  if (f.qbuf.capacity() < off) LSO_TRY(f.qbuf.reserve(off, 2 * off));
  char* q = f.qbuf.get();
  auto* cnt = reinterpret_cast<unsigned long long*>(q + o_cnt);
  LSO_TRY(cudaMemsetAsync(cnt, 0, sizeof(unsigned long long), st));
  LSO_TRY(cudaMemcpyAsync(q + o_p, pts3, 12 * N, cudaMemcpyHostToDevice, st));
  dt_query_kernel<<<blocks(n, 256), 256, 0, st>>>(reinterpret_cast<const float*>(q + o_p), n, box_of(f), f.inv, f.res,
                                                  f.val[0].get(), f.site[0].get(), dist ? (float*)(q + o_d) : nullptr,
                                                  sq ? (int*)(q + o_s) : nullptr, obst3 ? (float*)(q + o_o) : nullptr, cnt);
  LSO_LAUNCHED();
  if (dist) LSO_TRY(cudaMemcpyAsync(dist, q + o_d, 4 * N, cudaMemcpyDeviceToHost, st));
  if (sq) LSO_TRY(cudaMemcpyAsync(sq, q + o_s, 4 * N, cudaMemcpyDeviceToHost, st));
  if (obst3) LSO_TRY(cudaMemcpyAsync(obst3, q + o_o, 12 * N, cudaMemcpyDeviceToHost, st));
  unsigned long long h = 0;
  LSO_TRY(cudaMemcpyAsync(&h, cnt, sizeof h, cudaMemcpyDeviceToHost, st));
  LSO_TRY(cudaStreamSynchronize(st));
  *outside = (long long)h;
  return LS_OK;
}

int distance_download(DistanceField& f, int* sq, uint64_t* keys, cudaStream_t st, uint64_t* launches) {
  const size_t c = (size_t)f.cells;
  if (sq) LSO_TRY(cudaMemcpyAsync(sq, f.val[0].get(), 4 * c, cudaMemcpyDeviceToHost, st));
  if (keys) {
    // the stack is scratch between updates: 8 bytes per cell, as a key
    auto* k = reinterpret_cast<unsigned long long*>(f.stack.get());
    dt_keys_kernel<<<blocks(f.cells, 256), 256, 0, st>>>(f.site[0].get(), f.cells, box_of(f), k);
    LSO_LAUNCHED();
    LSO_TRY(cudaMemcpyAsync(keys, k, 8 * c, cudaMemcpyDeviceToHost, st));
  }
  LSO_TRY(cudaStreamSynchronize(st));
  return LS_OK;
}

size_t distance_bytes(const DistanceField& f) {
  return f.grid.capacity() + 4 * (f.val[0].capacity() + f.val[1].capacity() + f.site[0].capacity() + f.site[1].capacity()) +
         sizeof(uint2) * f.stack.capacity() + f.qbuf.capacity() + sizeof(unsigned long long) * f.cnt_dev.capacity();
}

}  // namespace lso
