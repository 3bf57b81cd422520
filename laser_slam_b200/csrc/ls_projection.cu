// octomap_server's projected_map of the resident occupancy map (DESIGN.md §4b'''''''''''''): the leaves of the .bt tree
// (toMaxLikelihood + prune) painted into a 2D occupancy grid, as handlePreNodeTraversal sizes it and update2DMap fills it at
// m_maxTreeDepth = 16 with a complete projection.  Per call, on the map's stream:
//   (p0) lv_down_kernel / lv_emit_kernel over the cached .bt build's records (ls_occupancy.cu): every leaf as a packed key,
//        depth and state, in pre-order
//   (p1) pj_leaf_kernel   one thread per leaf: calcMinMax's corners, reduced per block and merged with one atomic per
//                         block and bound (doubles as order-preserving integers); the (leaf, row) spans a leaf in the z band
//                         paints, 2^(16-d) of them
//   a CUB scan of the spans; the bounds and the span total come back, the host sizes the grid
//   (p2) pj_paint_kernel  one thread per (leaf, row) span: the leaf found by a binary search of the scan, its row's words of
//                         the occupied or known-free bit-plane set with atomicOr, so the work follows the footprint
//   (p3) pj_cells_kernel  one thread per cell: 100 where occupied, else 0 where known free, else -1; counts per value
// Occupied wins and free only fills unknown cells, so the grid is a per-cell maximum and does not depend on leaf order.
#include <algorithm>
#include <cstring>

#include <cub/cub.cuh>
#include <cuda_runtime.h>

#include "../../include/ls_b200.h"
#include "ls_occupancy.cuh"

namespace lso {
namespace {

constexpr int kLeafThreads = 256;
constexpr long long kMaxCells = 0x7fffffffLL;

// A double as an unsigned integer of the same order (no NaN reaches it), so bounds merge with atomicMin / atomicMax.
__host__ __device__ __forceinline__ unsigned long long ordered(unsigned long long bits) {
  return (bits >> 63) ? ~bits : bits | (1ull << 63);
}
double unordered(unsigned long long u) {
  const unsigned long long bits = (u >> 63) ? u & ~(1ull << 63) : ~u;
  double x;
  std::memcpy(&x, &bits, sizeof x);
  return x;
}

struct MinU {
  __device__ __forceinline__ unsigned long long operator()(unsigned long long a, unsigned long long b) const {
    return b < a ? b : a;
  }
};
struct MaxU {
  __device__ __forceinline__ unsigned long long operator()(unsigned long long a, unsigned long long b) const {
    return a < b ? b : a;
  }
};

// (p1) stat[0 ... 2]: the least lower corner per axis, stat[3 ... 5] the largest upper corner (calcMinMax: centre - size / 2,
// then that + size, in double); span[i]: 2^(16-d) when leaf i meets the band (z + size / 2 > min_z && z - size / 2 < max_z)
__global__ void __launch_bounds__(kLeafThreads) pj_leaf_kernel(const unsigned long long* __restrict__ rec, long long n,
                                                               double res, double min_z, double max_z,
                                                               unsigned long long* __restrict__ span,
                                                               unsigned long long* __restrict__ stat) {
  using Reduce = cub::BlockReduce<unsigned long long, kLeafThreads>;
  __shared__ typename Reduce::TempStorage red;
  const long long i = blockIdx.x * (long long)kLeafThreads + threadIdx.x;
  unsigned long long lo[3] = {~0ull, ~0ull, ~0ull}, hi[3] = {0ull, 0ull, 0ull};
  if (i < n) {
    const unsigned long long r = rec[i];
    const int s = 16 - (int)((r >> 48) & 0xff);
    const double size = res * (double)(1 << s), half = size / 2.0;
    double z = 0.0;
    for (int a = 0; a < 3; ++a) {
      const double c = leaf_centre_d((int)((r >> (16 * a)) & 0xffff), s, res);
      const double l = c - half;
      lo[a] = ordered((unsigned long long)__double_as_longlong(l));
      hi[a] = ordered((unsigned long long)__double_as_longlong(l + size));
      z = c;
    }
    span[i] = z + half > min_z && z - half < max_z ? 1ull << s : 0ull;
  }
  for (int a = 0; a < 3; ++a) {
    unsigned long long v = Reduce(red).Reduce(lo[a], MinU());
    __syncthreads();
    if (threadIdx.x == 0) atomicMin(&stat[a], v);
    v = Reduce(red).Reduce(hi[a], MaxU());
    __syncthreads();
    if (threadIdx.x == 0) atomicMax(&stat[3 + a], v);
  }
}

// (p2) span s of the scan off (n leaves, total spans): leaf j = the last with off[j] <= s paints row s - off[j] of its
// footprint, cells [kx - px, kx - px + 2^(16-d)) of grid row ky - py + (s - off[j]).  planes: occupied, then known-free,
// `plane` words each, rows of W words.
__global__ void pj_paint_kernel(const unsigned long long* __restrict__ rec, const unsigned long long* __restrict__ off, long long n,
                                unsigned long long total, int px, int py, long long W, long long plane,
                                unsigned* __restrict__ planes) {
  for (unsigned long long s = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; s < total;
       s += (unsigned long long)gridDim.x * blockDim.x) {
    long long lo = 0, hi = n - 1;
    while (lo < hi) {
      const long long mid = (lo + hi + 1) >> 1;
      if (off[mid] <= s) lo = mid;
      else hi = mid - 1;
    }
    const unsigned long long r = rec[lo];
    const int side = 1 << (16 - (int)((r >> 48) & 0xff));
    const long long row = (long long)((r >> 16) & 0xffff) - py + (long long)(s - off[lo]);
    const int x0 = (int)(r & 0xffff) - px, x1 = x0 + side;
    unsigned* w = planes + ((r >> 56) & 1 ? 0 : plane) + row * W;
    for (int k = x0 >> 5; k <= (x1 - 1) >> 5; ++k) {
      const int a = max(x0 - 32 * k, 0), b = min(x1 - 32 * k, 32);  // bits [a, b) of word k
      atomicOr(&w[k], b - a == 32 ? ~0u : ((1u << (b - a)) - 1u) << a);
    }
  }
}

// (p3) cell i = (x, y) at y * width + x: its value, and count[0 ... 2] the cells of -1, 0 and 100.  The index is 64-bit:
// with a grid of up to 2^31 - 1 cells, an index plus the grid's stride passes INT_MAX.
__global__ void __launch_bounds__(256) pj_cells_kernel(const unsigned* __restrict__ planes, long long plane, long long W,
                                                       long long width, long long cells, signed char* __restrict__ grid,
                                                       unsigned long long* __restrict__ count) {
  __shared__ unsigned h[3];
  if (threadIdx.x < 3) h[threadIdx.x] = 0;
  __syncthreads();
  unsigned c0 = 0, c1 = 0, c2 = 0;  // scalars, not an array indexed by v: that would live in local memory
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < cells; i += (long long)gridDim.x * blockDim.x) {
    const long long y = i / width, x = i - y * width;
    const long long k = y * W + (x >> 5);
    const unsigned bit = 1u << (x & 31);
    const int v = (planes[k] & bit) ? 2 : (planes[plane + k] & bit) ? 1 : 0;
    grid[i] = (signed char)(v == 2 ? 100 : v - 1);
    c0 += v == 0, c1 += v == 1, c2 += v == 2;
  }
  if (c0) atomicAdd(&h[0], c0);
  if (c1) atomicAdd(&h[1], c1);
  if (c2) atomicAdd(&h[2], c2);
  __syncthreads();
  if (threadIdx.x < 3 && h[threadIdx.x]) atomicAdd(&count[threadIdx.x], (unsigned long long)h[threadIdx.x]);
}

// Every per-leaf buffer for n leaves, all or nothing.
int reserve_leaf_scratch(Projection& p, long long n, cudaStream_t st) {
  LSO_TRY(p.stat.reserve(7, 7));
  LSO_TRY(p.stat_host.reserve(7, 7));
  if ((size_t)n + 1 <= p.rec.capacity()) return LS_OK;
  if (n >= (1LL << 30)) return LS_ERR_NOMEM;  // CUB's item counts are int
  LSO_TRY(cudaStreamSynchronize(st));
  const size_t c = (size_t)(n + 1 + n / 8);
  size_t scan = 0;
  cudaError_t e;
  if ((e = p.rec.reserve(c, c)) || (e = p.span.reserve(c, c)) || (e = p.off.reserve(c, c)) ||
      (e = cub::DeviceScan::ExclusiveSum(nullptr, scan, p.span.get(), p.off.get(), (int)c, st)) ||
      (e = p.cub_tmp.reserve(scan, scan))) {
    p.rec.reset(), p.span.reset(), p.off.reset(), p.cub_tmp.reset();
    p.cub_bytes = 0;
    return code(e);
  }
  p.cub_bytes = scan;
  return LS_OK;
}

// octomap's coordToKeyChecked(point3d, 16): the double corner as a float, keyed on every axis.
bool corner_keys(const Params& P, const double c[3], int k[3]) {
  for (int a = 0; a < 3; ++a)
    if (!key_of(P.inv, (double)(float)c[a], k[a])) return false;
  return true;
}

}  // namespace

int build_projection(const Map& m, const Params& P, Octree& t, const ProjectionArgs& A, Projection& p, const char** why,
                     cudaStream_t st, uint64_t* launches) {
  *why = "";
  const long long n = t.nodes - t.bytes / 2;  // the root is inner, so no leaves iff no nodes
  if (t.nodes == 0 || n <= 0) {              // octomap_server publishes nothing for a tree of size <= 1
    p.width = p.height = 0;
    p.cells[0] = p.cells[1] = p.cells[2] = 0;
    p.origin[0] = p.origin[1] = 0.0;
    return LS_OK;
  }
  int rc;
  if ((rc = reserve_leaf_scratch(p, n, st))) return *why = "out of device memory for the leaves", rc;
  unsigned long long* stat = p.stat.get();
  LSO_TRY(cudaMemsetAsync(stat, 0xff, 3 * sizeof(unsigned long long), st));
  LSO_TRY(cudaMemsetAsync(stat + 3, 0, 4 * sizeof(unsigned long long), st));
  LSO_TRY(cudaMemsetAsync(p.span.get() + n, 0, sizeof(unsigned long long), st));
  if ((rc = tree_leaf_records(m, P, t, p.rec.get(), st, launches))) return rc;
  pj_leaf_kernel<<<blocks(n, kLeafThreads), kLeafThreads, 0, st>>>(p.rec.get(), n, P.res, A.min_z, A.max_z, p.span.get(), stat);
  LSO_LAUNCHED();
  size_t bytes = p.cub_bytes;
  LSO_TRY(cub::DeviceScan::ExclusiveSum(p.cub_tmp.get(), bytes, p.span.get(), p.off.get(), (int)(n + 1), st));
  ++*launches;
  LSO_TRY(cudaMemcpyAsync(stat + 6, p.off.get() + n, sizeof(unsigned long long), cudaMemcpyDeviceToDevice, st));
  LSO_TRY(cudaMemcpyAsync(p.stat_host.get(), stat, 7 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  LSO_TRY(cudaStreamSynchronize(st));
  const unsigned long long* h = p.stat_host.get();
  double lo[3], hi[3];
  for (int a = 0; a < 3; ++a) lo[a] = unordered(h[a]), hi[a] = unordered(h[3 + a]);
  const unsigned long long spans = h[6];

  // handlePreNodeTraversal: the padded corners (std::min / std::max against -+min_size / 2 in x and y), keyed as floats
  const double hx = 0.5 * A.min_size_x, hy = 0.5 * A.min_size_y;
  const double pmin[3] = {std::min(lo[0], -hx), std::min(lo[1], -hy), lo[2]};
  const double pmax[3] = {std::max(hi[0], hx), std::max(hi[1], hy), hi[2]};
  int kmin[3], kmax[3];
  if (!corner_keys(P, pmin, kmin)) return *why = "the padded minimum corner is outside the key space", LS_ERR_ARG;
  if (!corner_keys(P, pmax, kmax)) return *why = "the padded maximum corner is outside the key space", LS_ERR_ARG;
  const long long width = (long long)kmax[0] - kmin[0] + 1, height = (long long)kmax[1] - kmin[1] + 1;
  const long long cells = width * height;
  if (cells > kMaxCells) return *why = "the grid has more than 2^31 - 1 cells", LS_ERR_ARG;

  // Only now are the planes and (when it must grow) a new grid allocated; the last grid stays until the call succeeds.
  const long long W = (width + 31) / 32, plane = W * height;
  if (p.planes.capacity() < (size_t)(2 * plane)) {
    LSO_TRY(cudaStreamSynchronize(st));
    if ((rc = code(p.planes.reserve((size_t)(2 * plane), (size_t)(2 * plane))))) return *why = "out of device memory for the grid", rc;
  }
  ls::Buffer<signed char> grown;
  signed char* grid = p.grid.get();
  if (p.grid.capacity() < (size_t)cells) {
    if ((rc = code(grown.reserve((size_t)cells, (size_t)cells)))) return *why = "out of device memory for the grid", rc;
    grid = grown.get();
  }
  LSO_TRY(cudaMemsetAsync(p.planes.get(), 0, (size_t)(2 * plane) * sizeof(unsigned), st));
  if (spans > 0) {
    const unsigned g = (unsigned)std::min<unsigned long long>((spans + 255) / 256, 8192);
    pj_paint_kernel<<<g, 256, 0, st>>>(p.rec.get(), p.off.get(), n, spans, kmin[0], kmin[1], W, plane, p.planes.get());
    LSO_LAUNCHED();
  }
  LSO_TRY(cudaMemsetAsync(stat, 0, 3 * sizeof(unsigned long long), st));
  pj_cells_kernel<<<std::min(blocks(cells, 256), 8192u), 256, 0, st>>>(p.planes.get(), plane, W, width, cells, grid,
                                                                       stat);
  LSO_LAUNCHED();
  LSO_TRY(cudaMemcpyAsync(p.stat_host.get(), stat, 3 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  LSO_TRY(cudaStreamSynchronize(st));
  if (grown.get()) p.grid = std::move(grown);
  p.width = width, p.height = height;
  for (int v = 0; v < 3; ++v) p.cells[v] = (long long)p.stat_host.get()[v];
  // keyToCoord(paddedMinKey) as a float point, less half a cell, in double
  p.origin[0] = (double)centre_of(kmin[0], P.res) - P.res * 0.5;
  p.origin[1] = (double)centre_of(kmin[1], P.res) - P.res * 0.5;
  return LS_OK;
}

int download_projection(const Projection& p, int8_t* cells, cudaStream_t st) {
  const long long c = p.width * p.height;
  if (c > 0) LSO_TRY(cudaMemcpyAsync(cells, p.grid.get(), (size_t)c, cudaMemcpyDeviceToHost, st));
  LSO_TRY(cudaStreamSynchronize(st));
  return LS_OK;
}

}  // namespace lso
