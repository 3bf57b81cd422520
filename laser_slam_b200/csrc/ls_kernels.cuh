// CUDA kernels of the registration hot path (sm_90a).  No tensor cores: there is no dense
// contraction on this path; every kernel is an HBM/L2-bound gather, scatter, histogram or reduction.
//
//   K0  assemble_kernel      sub-map = concat_p( T_p * scan_p ), exact mean sums, bounding box
//                            (LaserTrack::localScanToSubMap, reference laser_slam/src/laser_track.cpp:476-486)
//   K1  setup/count/scan/table/scatter kernels: two-level spatial hash + occupancy pyramid build (counting sort)
//                            (matcher->init(reference) inside ICP::compute, laser_track.cpp:496)
//   K2..K4 icp_kernel        ONE persistent cooperative kernel for the whole ICP loop: per iteration
//                            NN query (K2) -> exact trimmed-quantile radix select (K3) -> point-to-plane
//                            normal equations, order-independent int64 reduction, 6x6 solve (K4),
//                            transformation checkers; grid-wide barriers between phases.
//                            (KDTreeMatcher / TrimmedDistOutlierFilter / PointToPlaneErrorMinimizer /
//                            Counter+Differential checkers, icp_default.yaml:9-27)
#pragma once
#include <cuda_runtime.h>
#include <cooperative_groups.h>

#include "ls_grid.cuh"

namespace ls {

constexpr int kMaxParts = 16;
constexpr int kScanTile = 4096;       // level-0 cells per scan block
constexpr int kScanThreads = 512;
constexpr int kIcpThreads = 512;
constexpr int kIcpCtasPerSm = 1024 / kIcpThreads;
constexpr int kMaxSmooth = 15;
constexpr uint32_t kTag1 = 1u << 31, kKeyMask = (1u << 31) - 1u;  // pkey: tag | key (fine keys < 2^31)
// Untagged pkey between count0 and scatter: the fine sub-index (< LS_FB3 = 2^9) above the level-0 cell (< 2^22: the
// device caps max_cells there).
constexpr int kSubShift = 22;
constexpr uint32_t kCellMask = (1u << kSubShift) - 1u;

struct Parts {
  int n_parts;
  int offset[kMaxParts + 1];
  const float4* pts[kMaxParts];
  const float4* nrm[kMaxParts];
  float T[kMaxParts][16];
  int identity[kMaxParts];
};

struct BuildState {
  unsigned long long sum[3];         // exact fixed-point (2^-24 m) coordinate sums
  unsigned int minkey[3], maxkey[3];  // order-preserving integer images of float min/max
  Grid grid;
  float T_pre[16];                    // T_refMean_dataIn = [R0 | t0 - mu]
  unsigned int tile_sums[1024];
};

struct BuildArrays {
  float4* sub_pts;   // assembled sub-map, original order (not centred: scatter_kernel centres the sorted copy)
  float4* sub_nrm;
  float4* srt_pts;   // sorted {x,y,z,idx}
  float4* srt_nrm;
  uint32_t* pkey;    // per point: tag | deepest cell key found so far
  Entry* top;
  uint32_t* cnt0;
  Entry* tab1;           // fine tables, LS_FB3 entries each
  uint32_t* cnt1;
  uint32_t* tab1_cell;   // level-0 cell of each fine table
  int tab_cap;
  unsigned long long* pyr;  // occupancy pyramid masks
  unsigned long long* topmask;  // per level-0 cell with a table: non-empty rows (GridView::topmask)
  // query ordering (same keys as the map): rank -> query
  uint32_t* qkey;        // per query: tag | cell key
  uint32_t* qtop_start;  // per level-0 cell: first rank
  uint32_t* qtab_local;  // per fine cell: rank offset inside its table
  uint32_t* qtab_total;  // per table: number of queries
  uint32_t* qperm;       // rank -> original query index
  float4* rd_s;          // pre-transformed reading in rank order
};

// One map build (+ optional reading sort) of a launch: every build kernel takes an array of these and serves job
// blockIdx.y, so a step that registers B scans issues each build phase ONCE for all B problems instead of B times
// (a registration's build is a chain of ~17 short kernels: launched per problem it is bound by launch latency).
struct BuildJob {
  Parts parts;            // the sub-map: resident scans + per-scan transforms
  BuildState* bs;
  BuildArrays A;
  int m;                  // map points (= parts.offset[parts.n_parts])
  int n;                  // reading points (0: no reading)
  const float4* reading;  // raw reading, device
  float4* rd;             // reading pre-transformed by T_refMean_dataIn
  float T0[16];           // initial guess (column-major)
};

struct IcpParamsDev {
  int max_iterations;
  float trim_ratio;
  int use_differential;
  float min_diff_rot, min_diff_trans;
  int smooth_length;
};

struct alignas(16) IcpWork {
  unsigned int barrier;
  unsigned int pad0[31];
  unsigned int hist[2][5][2048];  // per parity: radix levels 1-3, then the speculative copies of levels 2 and 3
  unsigned long long acc[2][32];
  unsigned int qctr[2];  // phase-A work counters (next unclaimed query), one per iteration parity
  float T_out[16];
  int status, iterations, converged, max_iter_reached, last_kept;
  float last_limit;
  int fail_code;       // 1 no finite match, 2 nothing kept, 3 non-finite solve, 4 NaN in checker, 5 non-finite T
  unsigned int xsignals;  // query-sharded: arrivals this registration consumed from the local exchange flag
  unsigned int dbg_total, dbg_bin[3], dbg_rem[3];  // written by CTA 0 in phase E, read by nothing (see LS_STAMP)
  double dbg_A[6], dbg_x[6];
};

// What the host reads back of one registration: the results at the tail of its IcpWork and its grid's statistics.  A
// launch gathers them for all its problems into one array (collect_results_kernel), which comes back in one copy.
struct IcpResult {
  float T_out[16];
  int status, iterations, converged, max_iter_reached, last_kept;
  float last_limit;
  unsigned int xsignals;
  int n_cells0, n_tab1, overflow;
};

// Query-sharded registration: how one GPU reaches the others.  Every GPU owns an array of `shard_count` IcpWork
// "slots" plus an arrival counter.  Slot [self] is where the GPU's own CTAs accumulate (L2 atomics, as in the unsharded
// kernel); slot [r] receives, by plain stores over NVLink, the sections of shard r's slot [r] that the next step reads.
// A reader sums the slots -- all of them local memory.  Nothing is ever LOADED or polled across NVLink.
constexpr int kMaxShards = 8;
struct ShardLink {
  IcpWork* slots;                       // this GPU's slots [shard_count]
  IcpWork* peer_slots[kMaxShards];      // peer g's slot array, mapped into this GPU's address space (CUDA IPC)
  unsigned int* flag;                   // this GPU's arrival counter; never reset while the buffer lives
  unsigned int* peer_flag[kMaxShards];
  unsigned int flag_base;               // arrivals consumed by earlier registrations
};

struct IcpProblem {
  const BuildState* bs;
  GridView view;
  const float4* nrm;  // sorted normals
  const float4* rd;   // pre-transformed reading
  int n;
  int* pos;
  float* d2;            // per rank (internal)
  int* ids;             // original order, written by the final pass only
  float* d2_out;        // original order, written by the final pass only
  const uint32_t* qperm;  // rank -> original query index
  VLists lists;           // certified candidate lists (ls_grid.cuh), rank order
  IcpWork* work;
  // Query-sharded registration (one registration, its queries split over several GPUs; shard_count <= 1: not sharded)
  int shard_rank, shard_count;
  ShardLink link;
  float* T_hist;  // max_iterations*16 floats or null
  int want_matches;  // 1: finish with an uncapped NN pass so ids/d2 hold every point's true match
  unsigned long long* phase_ns;  // always null (see LS_STAMP)
  float T0[16];
};

// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned int float_order_key(float f) {
  const unsigned int u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float float_from_order_key(unsigned int k) {
  const unsigned int u = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
  return __uint_as_float(u);
}

__device__ __forceinline__ long long warp_sum_ll(long long v) {
  // 3 x 21-bit limbs through the integer warp-reduce unit (REDUX); exact, order independent
  unsigned int lo = (unsigned int)(v & 0x1FFFFF);
  unsigned int mid = (unsigned int)((v >> 21) & 0x1FFFFF);
  int hi = (int)(v >> 42);
  lo = __reduce_add_sync(0xffffffffu, lo);
  mid = __reduce_add_sync(0xffffffffu, mid);
  hi = __reduce_add_sync(0xffffffffu, hi);
  return ((long long)hi << 42) + ((long long)mid << 21) + (long long)lo;
}

// Histogram counters of the build.  Consecutive points of a lidar ring fall into the same cell, so the 32 lanes of a
// warp often carry one or two distinct keys: the lanes with equal keys (`active` = the lanes taking part) form a group
// whose leader does one atomic for all of them.  Every lane of `active` must make the call with the key (tagged
// pkey/qkey or level-0 cell) that names its counter `ctr` uniquely.
__device__ __forceinline__ void warp_count(uint32_t* ctr, uint32_t key, unsigned int active) {
  const unsigned int peers = __match_any_sync(active, key);
  if ((threadIdx.x & 31) == (unsigned int)(__ffs(peers) - 1)) atomicAdd(ctr, (unsigned int)__popc(peers));
}
// Scatter cursor: takes one slot per lane from *ctr (counting down) and returns the lane's slot; the group of lanes
// with equal keys takes its slots with one atomicSub.  The counter ends at zero once every point is placed.
__device__ __forceinline__ uint32_t warp_take(uint32_t* ctr, uint32_t key, unsigned int active) {
  const unsigned int peers = __match_any_sync(active, key);
  const int leader = __ffs(peers) - 1;
  const unsigned int lane = threadIdx.x & 31;
  uint32_t old = 0;
  if (lane == (unsigned int)leader) old = atomicSub(ctr, (unsigned int)__popc(peers));
  old = __shfl_sync(peers, old, leader);
  return old - 1u - (uint32_t)__popc(peers & ((1u << lane) - 1u));
}

// ---- K0: assemble + statistics -------------------------------------------------------------------
__global__ void __launch_bounds__(256) assemble_kernel(const BuildJob* __restrict__ jobs) {
  const BuildJob& J = jobs[blockIdx.y];
  const Parts& parts = J.parts;
  float4* __restrict__ sub_pts = J.A.sub_pts;
  float4* __restrict__ sub_nrm = J.A.sub_nrm;
  BuildState* bs = J.bs;
  const int total = parts.offset[parts.n_parts];
  long long s0 = 0, s1 = 0, s2 = 0;
  float mn0 = INFINITY, mn1 = INFINITY, mn2 = INFINITY, mx0 = -INFINITY, mx1 = -INFINITY, mx2 = -INFINITY;
  int p = 0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    while (i >= parts.offset[p + 1]) ++p;
    const int j = i - parts.offset[p];
    float4 a = __ldg(parts.pts[p] + j);
    float4 nn = __ldg(parts.nrm[p] + j);
    if (!parts.identity[p]) {
      float x, y, z;
      xform_point(parts.T[p], a.x, a.y, a.z, x, y, z);
      a.x = x; a.y = y; a.z = z;
      rotate_vec(parts.T[p], nn.x, nn.y, nn.z, x, y, z);
      nn.x = x; nn.y = y; nn.z = z;
    }
    sub_pts[i] = a;
    sub_nrm[i] = nn;
    s0 += __double2ll_rn((double)a.x * 16777216.0);
    s1 += __double2ll_rn((double)a.y * 16777216.0);
    s2 += __double2ll_rn((double)a.z * 16777216.0);
    mn0 = fminf(mn0, a.x); mx0 = fmaxf(mx0, a.x);
    mn1 = fminf(mn1, a.y); mx1 = fmaxf(mx1, a.y);
    mn2 = fminf(mn2, a.z); mx2 = fmaxf(mx2, a.z);
  }
  s0 = warp_sum_ll(s0); s1 = warp_sum_ll(s1); s2 = warp_sum_ll(s2);
  for (int o = 16; o > 0; o >>= 1) {
    mn0 = fminf(mn0, __shfl_xor_sync(0xffffffffu, mn0, o)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, o));
    mn1 = fminf(mn1, __shfl_xor_sync(0xffffffffu, mn1, o)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, o));
    mn2 = fminf(mn2, __shfl_xor_sync(0xffffffffu, mn2, o)); mx2 = fmaxf(mx2, __shfl_xor_sync(0xffffffffu, mx2, o));
  }
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(&bs->sum[0], (unsigned long long)s0);
    atomicAdd(&bs->sum[1], (unsigned long long)s1);
    atomicAdd(&bs->sum[2], (unsigned long long)s2);
    atomicMin(&bs->minkey[0], float_order_key(mn0)); atomicMax(&bs->maxkey[0], float_order_key(mx0));
    atomicMin(&bs->minkey[1], float_order_key(mn1)); atomicMax(&bs->maxkey[1], float_order_key(mx1));
    atomicMin(&bs->minkey[2], float_order_key(mn2)); atomicMax(&bs->maxkey[2], float_order_key(mx2));
  }
}

// points only (the reading side of a sub-map <-> sub-map registration): same arithmetic as assemble_kernel
__global__ void __launch_bounds__(256) assemble_points_kernel(const __grid_constant__ Parts parts, float4* __restrict__ out) {
  const int total = parts.offset[parts.n_parts];
  int p = 0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    while (i >= parts.offset[p + 1]) ++p;
    float4 a = __ldg(parts.pts[p] + (i - parts.offset[p]));
    if (!parts.identity[p]) {
      float x, y, z;
      xform_point(parts.T[p], a.x, a.y, a.z, x, y, z);
      a.x = x; a.y = y; a.z = z;
    }
    out[i] = a;
  }
}

// normals descriptor (stride floats per point) -> float4
__global__ void expand_normals_kernel(const float* __restrict__ raw, int stride, int n, float4* __restrict__ out) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float* r = raw + (size_t)i * stride;
    out[i] = make_float4(r[0], r[1], r[2], 0.f);
  }
}

__global__ void reset_build_kernel(const BuildJob* __restrict__ jobs) {
  BuildState* bs = jobs[blockIdx.y].bs;
  const int t = threadIdx.x;
  if (t < 3) {
    bs->sum[t] = 0ull;
    bs->minkey[t] = 0xffffffffu;
    bs->maxkey[t] = 0u;
  }
}

// ---- K1a: mean, bounding box, grid geometry, T_pre -------------------------------------------------
__global__ void setup_kernel(const BuildJob* __restrict__ jobs, float cell_size, int max_cells, int leaf_split) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const BuildJob& J = jobs[blockIdx.y];
  BuildState* bs = J.bs;
  const int m = J.m;
  const float* T0 = J.T0;
  float mu[3], lo[3], hi[3];
  for (int a = 0; a < 3; ++a) {
    const long long s = (long long)bs->sum[a];
    mu[a] = (float)((double)s / ((double)m * 16777216.0));
    // min over fl(x - mu) == fl(min x - mu): rounding is monotone
    lo[a] = float_from_order_key(bs->minkey[a]) - mu[a];
    hi[a] = float_from_order_key(bs->maxkey[a]) - mu[a];
  }
  Grid g;
  grid_setup(g, lo, hi, cell_size, max_cells, leaf_split, m);
  for (int a = 0; a < 3; ++a) g.mu[a] = mu[a];
  bs->grid = g;
  for (int i = 0; i < 16; ++i) bs->T_pre[i] = T0[i];
  for (int a = 0; a < 3; ++a) bs->T_pre[12 + a] = T0[12 + a] - mu[a];
}

// ---- K1b: level-0 histogram, and each point's level-0 cell and fine sub-index ----------------------------------
// The sub-map stays as assembled (the scatter centres it); the cell expressions take the centred coordinates, so
// membership is exactly what the queries assume.
// The point loops of the build run a whole warp per step (the warp-aggregated counters need all its lanes there): a
// warp takes 32 consecutive points, `active` holds the lanes that have one.
__global__ void __launch_bounds__(256) count0_kernel(const BuildJob* __restrict__ jobs) {
  const BuildJob& J = jobs[blockIdx.y];
  const BuildState* __restrict__ bs = J.bs;
  const BuildArrays A = J.A;
  const int m = J.m;
  __shared__ Grid g;
  if (threadIdx.x == 0) g = bs->grid;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i - lane < m; i += gridDim.x * blockDim.x) {
    const unsigned int active = __ballot_sync(0xffffffffu, i < m);
    if (i >= m) break;
    const float4 p = A.sub_pts[i];
    const float x = p.x - g.mu[0], y = p.y - g.mu[1], z = p.z - g.mu[2];
    const int c0 = top_index(g, x, y, z);
    float lx, ly, lz;
    top_origin(g, c0, lx, ly, lz);
    warp_count(A.cnt0 + c0, (uint32_t)c0, active);
    A.pkey[i] = ((uint32_t)sub_index(x, y, z, lx, ly, lz, g.inv1) << kSubShift) | (uint32_t)c0;
  }
}

// ---- K1c: exclusive scan of the level-0 histogram (two kernels, no spin-waits) ----------------------
__global__ void __launch_bounds__(kScanThreads) scan_reduce_kernel(const BuildJob* __restrict__ jobs) {
  BuildState* bs = jobs[blockIdx.y].bs;
  const uint32_t* __restrict__ cnt0 = jobs[blockIdx.y].A.cnt0;
  const int n = bs->grid.n_cells0;
  const int base = blockIdx.x * kScanTile;
  if (base >= n) return;
  unsigned int s = 0;
  for (int k = threadIdx.x; k < kScanTile; k += kScanThreads) {
    const int c = base + k;
    if (c < n) s += cnt0[c];
  }
  s = __reduce_add_sync(0xffffffffu, s);
  __shared__ unsigned int ws[kScanThreads / 32];
  if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned int t = 0;
    for (int w = 0; w < kScanThreads / 32; ++w) t += ws[w];
    bs->tile_sums[blockIdx.x] = t;
  }
}

__global__ void __launch_bounds__(kScanThreads) scan_apply_kernel(const BuildJob* __restrict__ jobs) {
  BuildState* bs = jobs[blockIdx.y].bs;
  const BuildArrays A = jobs[blockIdx.y].A;
  const int n = bs->grid.n_cells0;
  const int base = blockIdx.x * kScanTile;
  if (base >= n) return;
  const int split = bs->grid.leaf_split;
  __shared__ unsigned int ws[kScanThreads / 32];
  __shared__ unsigned int tile_off;
  // offset of this tile = sum of the previous tile sums
  unsigned int s = 0;
  for (int u = threadIdx.x; u < (int)blockIdx.x; u += kScanThreads) s += bs->tile_sums[u];
  s = __reduce_add_sync(0xffffffffu, s);
  if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned int t = 0;
    for (int w = 0; w < kScanThreads / 32; ++w) t += ws[w];
    tile_off = t;
  }
  __syncthreads();
  // each thread owns 8 consecutive cells
  constexpr int per = kScanTile / kScanThreads;
  unsigned int c[per], loc = 0;
  const int first = base + threadIdx.x * per;
#pragma unroll
  for (int k = 0; k < per; ++k) {
    c[k] = (first + k < n) ? A.cnt0[first + k] : 0u;
    loc += c[k];
  }
  unsigned int incl = loc;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned int v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  __syncthreads();
  if (lane == 31) ws[warp] = incl;
  __syncthreads();
  unsigned int woff = 0;
  for (int w = 0; w < warp; ++w) woff += ws[w];
  unsigned int run = tile_off + woff + incl - loc;
#pragma unroll
  for (int k = 0; k < per; ++k) {
    const int cell = first + k;
    if (cell < n) {
      Entry e;
      e.start = run;
      e.meta = (int)c[k];
      if ((int)c[k] > split) {
        const int t = atomicAdd(&bs->grid.n_tab1, 1);
        if (t < A.tab_cap) {
          e.meta = ~t;
          A.tab1_cell[t] = (uint32_t)cell;
          A.cnt0[cell] = 0u;  // not a scatter cursor; leave the array clean for the next build
        } else {
          bs->grid.overflow = 1;
        }
      }
      A.top[cell] = e;
    }
    run += c[k];
  }
}

// ---- K1c': occupancy pyramid (level 1 from the level-0 entries, upper levels by one CTA) -------------
__device__ __forceinline__ unsigned long long pyramid_mask(const Grid& g, int l, int x, int y, int z, const Entry* top,
                                                           const unsigned long long* pyr) {
  const int* cd = g.pdim[l - 1];
  unsigned long long mask = 0ull;
  for (int k = 0; k < 4; ++k) {
    const int cz = 4 * z + k;
    if (cz >= cd[2]) break;
    for (int j = 0; j < 4; ++j) {
      const int cy = 4 * y + j;
      if (cy >= cd[1]) break;
      for (int i = 0; i < 4; ++i) {
        const int cx = 4 * x + i;
        if (cx >= cd[0]) break;
        const size_t ci = ((size_t)cz * cd[1] + cy) * cd[0] + cx;
        const bool occ = (l == 1) ? (top[ci].meta != 0) : (pyr[g.poff[l - 1] + ci] != 0ull);
        if (occ) mask |= 1ull << ((k * 4 + j) * 4 + i);
      }
    }
  }
  return mask;
}

__global__ void __launch_bounds__(256) pyramid1_kernel(const BuildJob* __restrict__ jobs) {
  const BuildState* __restrict__ bs = jobs[blockIdx.y].bs;
  const BuildArrays A = jobs[blockIdx.y].A;
  __shared__ Grid g;
  if (threadIdx.x == 0) g = bs->grid;
  __syncthreads();
  const int* pd = g.pdim[1];
  const int n = pd[0] * pd[1] * pd[2];
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < n; c += gridDim.x * blockDim.x) {
    const int x = c % pd[0], y = (c / pd[0]) % pd[1], z = c / (pd[0] * pd[1]);
    A.pyr[g.poff[1] + c] = pyramid_mask(g, 1, x, y, z, A.top, A.pyr);
  }
}

__global__ void __launch_bounds__(1024) pyramid_up_kernel(const BuildJob* __restrict__ jobs) {
  const BuildState* __restrict__ bs = jobs[blockIdx.y].bs;
  const BuildArrays A = jobs[blockIdx.y].A;
  __shared__ Grid g;
  if (threadIdx.x == 0) g = bs->grid;
  __syncthreads();
  for (int l = 2; l <= g.n_pyr; ++l) {
    const int* pd = g.pdim[l];
    const int n = pd[0] * pd[1] * pd[2];
    for (int c = threadIdx.x; c < n; c += blockDim.x) {
      const int x = c % pd[0], y = (c / pd[0]) % pd[1], z = c / (pd[0] * pd[1]);
      A.pyr[g.poff[l] + c] = pyramid_mask(g, l, x, y, z, A.top, A.pyr);
    }
    __threadfence_block();
    __syncthreads();
  }
}

// ---- K1d: level-1 histogram (from the keys count0 left: the points are not read again) ----------------------
__global__ void __launch_bounds__(256) count1_kernel(const BuildJob* __restrict__ jobs) {
  const BuildArrays A = jobs[blockIdx.y].A;
  const int m = jobs[blockIdx.y].m;
  const int lane = threadIdx.x & 31;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i - lane < m; i += gridDim.x * blockDim.x) {
    const uint32_t k = i < m ? A.pkey[i] : 0u;
    const int meta = i < m ? A.top[k & kCellMask].meta : 0;
    const unsigned int active = __ballot_sync(0xffffffffu, meta < 0);
    if (meta >= 0) continue;
    const uint32_t key = (uint32_t)(~meta) * (uint32_t)LS_FB3 + (k >> kSubShift);
    warp_count(A.cnt1 + key, key, active);
    A.pkey[i] = kTag1 | key;
  }
}

// one CTA per fine table: exclusive scan of its LS_FB3 counts -> Entry{start, count}
__global__ void __launch_bounds__(256) tables_kernel(const BuildJob* __restrict__ jobs) {
  BuildState* bs = jobs[blockIdx.y].bs;
  const BuildArrays A = jobs[blockIdx.y].A;
  const int n_tab = min(bs->grid.n_tab1, A.tab_cap);
  constexpr int per = LS_FB3 / 256;  // 2 consecutive cells per thread
  __shared__ unsigned int ws[8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int t = blockIdx.x; t < n_tab; t += gridDim.x) {
    const uint32_t* cnt = A.cnt1 + (size_t)t * LS_FB3;
    Entry* tab = A.tab1 + (size_t)t * LS_FB3;
    const uint32_t base = A.top[A.tab1_cell[t]].start;
    unsigned int c[per], loc = 0;
#pragma unroll
    for (int k = 0; k < per; ++k) {
      c[k] = cnt[threadIdx.x * per + k];
      loc += c[k];
    }
    unsigned int incl = loc;
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned int v = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += v;
    }
    __syncthreads();
    if (lane == 31) ws[warp] = incl;
    __syncthreads();
    unsigned int woff = 0;
    for (int w = 0; w < warp; ++w) woff += ws[w];
    unsigned int run = base + woff + incl - loc;
#pragma unroll
    for (int k = 0; k < per; ++k) {
      Entry e;
      e.start = run;
      e.meta = (int)c[k];
      tab[threadIdx.x * per + k] = e;
      run += c[k];
    }
    // non-empty rows: a row is 8 consecutive cells = 4 consecutive threads; warp w covers rows 8w .. 8w+7
    const unsigned int occ = __ballot_sync(0xffffffffu, loc != 0u);
    unsigned int rows8 = 0u;
#pragma unroll
    for (int r = 0; r < 8; ++r)
      if ((occ >> (4 * r)) & 0xFu) rows8 |= 1u << r;
    __syncthreads();  // ws was read above
    if (lane == 0) ws[warp] = rows8;
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned long long m = 0ull;
      for (int w = 0; w < 8; ++w) m |= (unsigned long long)ws[w] << (8 * w);
      A.topmask[A.tab1_cell[t]] = m;
    }
  }
}

// ---- K1f: centre and scatter into sorted order (the leaf histograms double as cursors and end at zero) -----------
__global__ void __launch_bounds__(256) scatter_kernel(const BuildJob* __restrict__ jobs) {
  const BuildArrays A = jobs[blockIdx.y].A;
  const int m = jobs[blockIdx.y].m;
  const float* mu = jobs[blockIdx.y].bs->grid.mu;
  const float mx = mu[0], my = mu[1], mz = mu[2];
  const int lane = threadIdx.x & 31;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i - lane < m; i += gridDim.x * blockDim.x) {
    const unsigned int active = __ballot_sync(0xffffffffu, i < m);
    if (i >= m) break;
    const uint32_t k = A.pkey[i];
    const bool fine = (k & kTag1) != 0u;
    const uint32_t key = fine ? k : (k & kCellMask);  // tagged: never equal to a level-0 cell
    const Entry* e = fine ? A.tab1 + (key & kKeyMask) : A.top + key;
    uint32_t* ctr = fine ? A.cnt1 + (key & kKeyMask) : A.cnt0 + key;
    const uint32_t pos = e->start + warp_take(ctr, key, active);
    float4 p = A.sub_pts[i];
    p.x = p.x - mx;
    p.y = p.y - my;
    p.z = p.z - mz;
    p.w = __int_as_float(i);
    A.srt_pts[pos] = p;
    A.srt_nrm[pos] = A.sub_nrm[i];
  }
}

// ---- query ordering ----------------------------------------------------------------------------------------
// The reading is processed in the order of the map's own cell keys (level-0 cell, fine cell): threads of a warp
// then walk the same rows and candidates (L1 reuse, convergent loops) instead of 32 different places along a
// lidar ring.  It is a counting sort that borrows the map's histogram arrays -- they are all zero again once the
// map's scatter has run, and the cursors below return them to zero.  Results do not depend on the order: every
// reduction of the ICP kernel is an exact integer sum.
// q_count_kernel also pre-transforms the reading, R' = T_refMean_dataIn * R, into `rd` (reading_kernel's arithmetic).
__global__ void __launch_bounds__(256) q_count_kernel(const BuildJob* __restrict__ jobs) {
  const BuildState* __restrict__ bs = jobs[blockIdx.y].bs;
  const BuildArrays A = jobs[blockIdx.y].A;
  const float4* __restrict__ in = jobs[blockIdx.y].reading;
  float4* __restrict__ rd = jobs[blockIdx.y].rd;
  const int n = jobs[blockIdx.y].n;
  __shared__ Grid g;
  __shared__ float T[16];
  if (threadIdx.x == 0) g = bs->grid;
  if (threadIdx.x < 16) T[threadIdx.x] = bs->T_pre[threadIdx.x];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i - lane < n; i += gridDim.x * blockDim.x) {
    const unsigned int active = __ballot_sync(0xffffffffu, i < n);
    if (i >= n) break;
    const float4 a = __ldg(in + i);
    float4 p;
    xform_point(T, a.x, a.y, a.z, p.x, p.y, p.z);
    p.w = a.w;
    rd[i] = p;
    const int c0 = top_index(g, p.x, p.y, p.z);
    const Entry e = A.top[c0];
    uint32_t key;
    uint32_t* ctr;
    if (e.meta < 0) {
      float lx, ly, lz;
      top_origin(g, c0, lx, ly, lz);
      key = (uint32_t)(~e.meta) * (uint32_t)LS_FB3 + (uint32_t)sub_index(p.x, p.y, p.z, lx, ly, lz, g.inv1);
      ctr = A.cnt1 + key;
      key |= kTag1;
    } else {
      key = (uint32_t)c0;
      ctr = A.cnt0 + c0;
    }
    warp_count(ctr, key, active);
    A.qkey[i] = key;
  }
}

__global__ void __launch_bounds__(256) q_tables_kernel(const BuildJob* __restrict__ jobs) {
  BuildState* bs = jobs[blockIdx.y].bs;
  const BuildArrays A = jobs[blockIdx.y].A;
  const int n_tab = min(bs->grid.n_tab1, A.tab_cap);
  constexpr int per = LS_FB3 / 256;
  __shared__ unsigned int ws[8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int t = blockIdx.x; t < n_tab; t += gridDim.x) {
    const uint32_t* cnt = A.cnt1 + (size_t)t * LS_FB3;
    unsigned int c[per], loc = 0;
#pragma unroll
    for (int k = 0; k < per; ++k) {
      c[k] = cnt[threadIdx.x * per + k];
      loc += c[k];
    }
    unsigned int incl = loc;
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned int v = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += v;
    }
    __syncthreads();
    if (lane == 31) ws[warp] = incl;
    __syncthreads();
    unsigned int woff = 0, total = 0;
    for (int w = 0; w < 8; ++w) {
      if (w < warp) woff += ws[w];
      total += ws[w];
    }
    unsigned int run = woff + incl - loc;
#pragma unroll
    for (int k = 0; k < per; ++k) {
      A.qtab_local[(size_t)t * LS_FB3 + threadIdx.x * per + k] = run;
      run += c[k];
    }
    if (threadIdx.x == 0) A.qtab_total[t] = total;
  }
}

__device__ __forceinline__ unsigned int q_cell_count(const BuildArrays& A, int c) {
  const Entry e = A.top[c];
  return e.meta < 0 ? A.qtab_total[~e.meta] : A.cnt0[c];
}

__global__ void __launch_bounds__(kScanThreads) q_scan_reduce_kernel(const BuildJob* __restrict__ jobs) {
  BuildState* bs = jobs[blockIdx.y].bs;
  const BuildArrays A = jobs[blockIdx.y].A;
  const int n = bs->grid.n_cells0;
  const int base = blockIdx.x * kScanTile;
  if (base >= n) return;
  unsigned int s = 0;
  for (int k = threadIdx.x; k < kScanTile; k += kScanThreads) {
    const int c = base + k;
    if (c < n) s += q_cell_count(A, c);
  }
  s = __reduce_add_sync(0xffffffffu, s);
  __shared__ unsigned int ws[kScanThreads / 32];
  if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned int t = 0;
    for (int w = 0; w < kScanThreads / 32; ++w) t += ws[w];
    bs->tile_sums[blockIdx.x] = t;
  }
}

__global__ void __launch_bounds__(kScanThreads) q_scan_apply_kernel(const BuildJob* __restrict__ jobs) {
  BuildState* bs = jobs[blockIdx.y].bs;
  const BuildArrays A = jobs[blockIdx.y].A;
  const int n = bs->grid.n_cells0;
  const int base = blockIdx.x * kScanTile;
  if (base >= n) return;
  __shared__ unsigned int ws[kScanThreads / 32];
  __shared__ unsigned int tile_off;
  unsigned int s = 0;
  for (int u = threadIdx.x; u < (int)blockIdx.x; u += kScanThreads) s += bs->tile_sums[u];
  s = __reduce_add_sync(0xffffffffu, s);
  if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned int t = 0;
    for (int w = 0; w < kScanThreads / 32; ++w) t += ws[w];
    tile_off = t;
  }
  __syncthreads();
  constexpr int per = kScanTile / kScanThreads;
  unsigned int c[per], loc = 0;
  const int first = base + threadIdx.x * per;
#pragma unroll
  for (int k = 0; k < per; ++k) {
    c[k] = (first + k < n) ? q_cell_count(A, first + k) : 0u;
    loc += c[k];
  }
  unsigned int incl = loc;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned int v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  __syncthreads();
  if (lane == 31) ws[warp] = incl;
  __syncthreads();
  unsigned int woff = 0;
  for (int w = 0; w < warp; ++w) woff += ws[w];
  unsigned int run = tile_off + woff + incl - loc;
#pragma unroll
  for (int k = 0; k < per; ++k) {
    if (first + k < n) A.qtop_start[first + k] = run;
    run += c[k];
  }
}

__global__ void __launch_bounds__(256) q_scatter_kernel(const BuildJob* __restrict__ jobs) {
  const BuildArrays A = jobs[blockIdx.y].A;
  const float4* __restrict__ rd = jobs[blockIdx.y].rd;
  const int n = jobs[blockIdx.y].n;
  const int lane = threadIdx.x & 31;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i - lane < n; i += gridDim.x * blockDim.x) {
    const unsigned int active = __ballot_sync(0xffffffffu, i < n);
    if (i >= n) break;
    const uint32_t k = A.qkey[i];
    uint32_t start;
    uint32_t* ctr;
    if (k & kTag1) {
      const uint32_t key = k & kKeyMask;
      start = A.qtop_start[A.tab1_cell[key / (uint32_t)LS_FB3]] + A.qtab_local[key];
      ctr = A.cnt1 + key;
    } else {
      start = A.qtop_start[k];
      ctr = A.cnt0 + k;
    }
    const uint32_t rank = start + warp_take(ctr, k, active);
    A.rd_s[rank] = __ldg(rd + i);
    A.qperm[rank] = (uint32_t)i;
  }
}

// Query-sharded registration: narrow a staged problem to this shard's range of the cell-sorted reading.  The order
// of the queries INSIDE a cell depends on the scatter's atomics and differs from GPU to GPU; where a cell starts does not
// (it is a prefix sum of counts).  So the cuts are moved to the next cell start: every shard computes the same cuts and
// every query belongs to exactly one shard.  One thread; qtop_start is non-decreasing over the level-0 cells.
__global__ void shard_slice_kernel(IcpProblem* P, const BuildJob* __restrict__ job, int shard_rank, int shard_count) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const BuildArrays A = job->A;
  const int n_cells = job->bs->grid.n_cells0, n = job->n;
  auto cut = [&](int s) -> int {
    if (s <= 0) return 0;
    if (s >= shard_count) return n;
    const unsigned int target = (unsigned int)((long long)n * s / shard_count);
    int lo = 0, hi = n_cells;  // first cell whose start is >= target
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (A.qtop_start[mid] < target) lo = mid + 1;
      else hi = mid;
    }
    return lo < n_cells ? (int)A.qtop_start[lo] : n;
  };
  const int q0 = cut(shard_rank), q1 = cut(shard_rank + 1);
  P->rd += q0;
  P->qperm += q0;
  P->pos += q0;
  P->d2 += q0;
  P->lists.vq += q0;
  P->lists.vpts += q0;  // the candidate slots keep their stride (lists.n = the whole reading)
  P->n = q1 - q0;
}

// one CTA per problem of an ICP launch, after it: results -> out[problem]
__global__ void collect_results_kernel(const IcpProblem* __restrict__ probs, IcpResult* __restrict__ out) {
  const IcpProblem& P = probs[blockIdx.x];
  const IcpWork* W = P.work;
  IcpResult& r = out[blockIdx.x];
  if (threadIdx.x < 16) r.T_out[threadIdx.x] = W->T_out[threadIdx.x];
  if (threadIdx.x == 0) {
    r.status = W->status;
    r.iterations = W->iterations;
    r.converged = W->converged;
    r.max_iter_reached = W->max_iter_reached;
    r.last_kept = W->last_kept;
    r.last_limit = W->last_limit;
    r.xsignals = W->xsignals;
    r.n_cells0 = P.bs->grid.n_cells0;
    r.n_tab1 = P.bs->grid.n_tab1;
    r.overflow = P.bs->grid.overflow;
  }
}

// ---- reading pre-transform: R' = T_refMean_dataIn * R ----------------------------------------------
__global__ void __launch_bounds__(256) reading_kernel(const BuildJob* __restrict__ jobs) {
  const BuildState* __restrict__ bs = jobs[blockIdx.y].bs;
  const float4* __restrict__ in = jobs[blockIdx.y].reading;
  float4* __restrict__ out = jobs[blockIdx.y].rd;
  const int n = jobs[blockIdx.y].n;
  __shared__ float T[16];
  if (threadIdx.x < 16) T[threadIdx.x] = bs->T_pre[threadIdx.x];
  __syncthreads();
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float4 a = __ldg(in + i);
    float4 o;
    xform_point(T, a.x, a.y, a.z, o.x, o.y, o.z);
    o.w = a.w;
    out[i] = o;
  }
}

// plain RigidTransformation::compute on a cloud
__global__ void __launch_bounds__(256) transform_kernel(const float* __restrict__ Tg, const float4* __restrict__ in,
                                                        const float4* __restrict__ nin, int n, float4* __restrict__ out,
                                                        float4* __restrict__ nout) {
  __shared__ float T[16];
  if (threadIdx.x < 16) T[threadIdx.x] = Tg[threadIdx.x];
  __syncthreads();
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float4 a = __ldg(in + i);
    float4 o;
    xform_point(T, a.x, a.y, a.z, o.x, o.y, o.z);
    o.w = a.w;
    out[i] = o;
    if (nin) {
      const float4 b = __ldg(nin + i);
      float4 r;
      rotate_vec(T, b.x, b.y, b.z, r.x, r.y, r.z);
      r.w = 0.f;
      nout[i] = r;
    }
  }
}

// float4 normals -> packed 3 floats (download helper)
__global__ void pack_normals_kernel(const float4* __restrict__ in, int n, float* __restrict__ out3) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float4 a = in[i];
    out3[3 * (size_t)i] = a.x;
    out3[3 * (size_t)i + 1] = a.y;
    out3[3 * (size_t)i + 2] = a.z;
  }
}

// ---- matcher-only kernel (ls_nn_query): cold exact NN for every pre-transformed reading point -------
__global__ void __launch_bounds__(256) nn_query_kernel(const BuildState* __restrict__ bs, GridView view,
                                                       const float4* __restrict__ rd, int n, int* __restrict__ ids,
                                                       float* __restrict__ d2) {
  __shared__ Grid g;
  if (threadIdx.x == 0) g = bs->grid;
  __syncthreads();
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float4 q = __ldg(rd + i);
    const Best b = nn_search(g, view, q.x, q.y, q.z, -1, INFINITY);
    ids[i] = b.idx;
    d2[i] = b.d2;
  }
}

// ---- surface normals (SURVEY.md §8 row f1) ---------------------------------------------------------------------
// Replaces the SurfaceNormal / SamplingSurfaceNormal DataPointsFilters the reference runs on every scan and on the
// whole sub-map (reference laser_slam/configurations/icp_default.yaml:5-7, laser_slam/src/laser_track.cpp:27,146):
// exact K nearest neighbours (self included) over the cloud's own spatial hash, covariance of the neighbourhood
// accumulated in double in (d2, index) order, eigenvector of the smallest eigenvalue, flipped towards the sensor
// (the origin of the scan frame).  Deterministic; bit-comparable with the CPU restatement in oracle/.
__global__ void __launch_bounds__(128) knn_normals_kernel(const BuildState* __restrict__ bs, GridView view,
                                                           const float4* __restrict__ pts /* assembled, original order */,
                                                           int n, int k, float4* __restrict__ out) {
  __shared__ Grid g;
  if (threadIdx.x == 0) g = bs->grid;
  __syncthreads();
  // the centred coordinates, as scatter_kernel computes them for the hash
  auto centred = [&](int j) {
    float4 p = __ldg(pts + j);
    p.x = p.x - g.mu[0];
    p.y = p.y - g.mu[1];
    p.z = p.z - g.mu[2];
    return p;
  };
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float4 q = centred(i);
    TopK t;
    knn_search(g, view, q.x, q.y, q.z, k, t);
    int cnt = 0;
    double mx = 0.0, my = 0.0, mz = 0.0;
    for (int j = 0; j < k; ++j) {
      if (t.id[j] == INT_MAX) break;
      const float4 p = centred(t.id[j]);
      mx = mx + (double)p.x;
      my = my + (double)p.y;
      mz = mz + (double)p.z;
      ++cnt;
    }
    float4 nn = make_float4(0.f, 0.f, 0.f, 0.f);
    if (cnt >= 3) {
      const double inv = 1.0 / (double)cnt;
      mx = mx * inv; my = my * inv; mz = mz * inv;
      double C[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
      for (int j = 0; j < cnt; ++j) {
        const float4 p = centred(t.id[j]);
        const double dx = (double)p.x - mx, dy = (double)p.y - my, dz = (double)p.z - mz;
        C[0] = C[0] + dx * dx; C[1] = C[1] + dx * dy; C[2] = C[2] + dx * dz;
        C[4] = C[4] + dy * dy; C[5] = C[5] + dy * dz; C[8] = C[8] + dz * dz;
      }
      C[3] = C[1]; C[6] = C[2]; C[7] = C[5];
      double nv[3];
      smallest_eigvec3(C, nv);
      // towards the sensor: the vector from the point to the scan-frame origin is -(p_centred + mu)
      const double ox = (double)q.x + (double)g.mu[0], oy = (double)q.y + (double)g.mu[1], oz = (double)q.z + (double)g.mu[2];
      const double dot = nv[0] * ox + (nv[1] * oy + nv[2] * oz);
      const double sgn = dot > 0.0 ? -1.0 : 1.0;
      nn = make_float4((float)(sgn * nv[0]), (float)(sgn * nv[1]), (float)(sgn * nv[2]), 0.f);
    }
    out[i] = nn;
  }
}

// ================================================================================================
// Persistent ICP kernel
// ================================================================================================
__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
// Per-phase globaltimer stamps of CTA 0 into IcpProblem::phase_ns, which the library always sets to null.  Neither these
// sites nor the IcpWork::dbg_* stores of phase E contribute to the result, but removing them changes icp_kernel's register
// allocation, and the batched launch then ran about 1% slower (H100 SXM, 700 W power limit, bench.py configs 2 and 5).
#define LS_STAMP(slot)                                                                   \
  do {                                                                                   \
    if (P.phase_ns && cta == 0 && tid == 0) P.phase_ns[iter * 6 + (slot)] = globaltimer_ns(); \
  } while (0)

__device__ __forceinline__ unsigned int ld_relaxed_u32(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_release_inc(unsigned int* p) {
  asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(p) : "memory");
}
// system-scope flavours for the exchange buffer of a query-sharded registration (peer memory over NVLink)
__device__ __forceinline__ unsigned int ld_relaxed_sys_u32(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ unsigned long long ld_relaxed_sys_u64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_release_sys_inc(unsigned int* p) {
  asm volatile("red.release.sys.global.add.u32 [%0], 1;" ::"l"(p) : "memory");
}

// All CTAs of one problem.  `epoch` is the number of arrivals expected so far (kept in a register).
//
// Deliberately NOT an acquire: an acquire at gpu scope makes ptxas emit CCTL.IVALL (invalidate the whole
// L1) -- per poll, that let a waiting CTA keep flushing the L1 of the CTA still searching on the same SM.
// Everything one CTA produces for another (histograms, accumulators, their clearing) is either an L2
// atomic or read back with ld.global.cg, i.e. served by L2, the point of coherence; per-query state
// (pos/d2/ids) is only ever touched by its owning thread.  So the arrive is a release (prior writes are
// performed at L2 before the counter moves) and the wait is a relaxed poll: L1 keeps the read-only map.
__device__ __forceinline__ void problem_barrier(unsigned int* ctr, unsigned int n_ctas, unsigned int& epoch) {
  __syncthreads();
  if (threadIdx.x == 0) {
    epoch += n_ctas;
    red_release_inc(ctr);
    unsigned int polls = 0;
    unsigned long long t0 = 0ull;
    while (ld_relaxed_u32(ctr) < epoch) {
      __nanosleep(64);  // the polling thread shares its SM's issue slots with a CTA that is still working
      // watchdog: a barrier that does not complete within seconds is a bug (or a launch that was not co-resident);
      // fail the launch loudly instead of hanging the device
      if ((++polls & 0x3fffu) == 0u) {
        const unsigned long long now = globaltimer_ns();
        if (t0 == 0ull) t0 = now;
        else if (now - t0 > 8000000000ull) {
          printf("[ls] icp_kernel barrier timeout: block %d waits for %u, counter %u\n", (int)blockIdx.x, epoch, ld_relaxed_u32(ctr));
          __trap();
        }
      }
    }
  }
  __syncthreads();
}

struct SelectOut {
  unsigned int bin, rem, total;
};
constexpr size_t kWorkWords = sizeof(IcpWork) / 4;
static_assert(sizeof(IcpWork) % 16 == 0 && offsetof(IcpWork, hist) % 16 == 0 && offsetof(IcpWork, acc) % 16 == 0, "sections move as uint4");

// Query-sharded registration: the cross-GPU step that takes the place of problem_barrier.
//   1. local barrier: this GPU's contribution to the sections is complete (in L2)
//   2. CTA c < shard_count-1 pushes the sections to peer c's slot for this shard (16-byte stores over NVLink), then
//      bumps that peer's arrival counter with a system-scope release
//   3. every CTA waits until all peers have bumped THIS GPU's counter (a local poll), after which the peers' sections
//      are in this GPU's memory
// A section is rewritten by a peer two iterations later at the earliest (the buffers alternate with the iteration's
// parity), and the peer gets there only through exchanges this GPU feeds after all its CTAs have read -- so no reader is
// ever overtaken.  Sections are word offsets into IcpWork, multiples of 4.
__device__ __forceinline__ void shard_exchange(const IcpProblem& P, IcpWork* X, int cta, unsigned int G, unsigned int& epoch,
                                               unsigned int& xepoch, int off0, int n0, int off1, int n1, int off2, int n2) {
  problem_barrier(&X->barrier, G, epoch);
  const int peers = P.shard_count - 1;
  if (cta < peers) {
    const int g = cta + (cta >= P.shard_rank ? 1 : 0);
    const uint4* src = reinterpret_cast<const uint4*>(X);
    uint4* dst = reinterpret_cast<uint4*>(P.link.peer_slots[g] + P.shard_rank);
    for (int k = threadIdx.x; k < n0 / 4; k += kIcpThreads) __stcg(dst + off0 / 4 + k, __ldcg(src + off0 / 4 + k));
    for (int k = threadIdx.x; k < n1 / 4; k += kIcpThreads) __stcg(dst + off1 / 4 + k, __ldcg(src + off1 / 4 + k));
    for (int k = threadIdx.x; k < n2 / 4; k += kIcpThreads) __stcg(dst + off2 / 4 + k, __ldcg(src + off2 / 4 + k));
    __syncthreads();
    if (threadIdx.x == 0) {
      __threadfence_system();
      red_release_sys_inc(P.link.peer_flag[g]);
    }
  }
  xepoch += (unsigned int)peers;
  if (threadIdx.x == 0) {
    const unsigned int target = P.link.flag_base + xepoch;
    unsigned int polls = 0;
    unsigned long long t0 = 0ull;
    while ((int)(ld_relaxed_sys_u32(P.link.flag) - target) < 0) {
      __nanosleep(64);
      if ((++polls & 0x3fffu) == 0u) {
        const unsigned long long now = globaltimer_ns();
        if (t0 == 0ull) t0 = now;
        else if (now - t0 > 8000000000ull) {
          printf("[ls] icp_kernel shard %d: a peer did not arrive (block %d waits for %u, counter %u)\n", P.shard_rank, (int)blockIdx.x,
                 target, ld_relaxed_sys_u32(P.link.flag));
          __trap();
        }
      }
    }
  }
  __syncthreads();
}

__device__ __forceinline__ unsigned long long sum_slots_u64(const unsigned long long* p, int n_slots) {
  unsigned long long v = 0ull;
  for (int g = 0; g < n_slots; ++g) v += __ldcg(p + (size_t)g * (kWorkWords / 2));
  return v;
}

// Block-wide: find the histogram bin holding the element of 0-based rank k.
// If `first` the rank is derived from the total: k = (unsigned)((float)total * ratio), clamped.
__device__ __forceinline__ void block_select(const unsigned int* ghist, int nbins, unsigned int k, bool first,
                                             float ratio, SelectOut* out, unsigned int* ws, int n_slots = 1) {
  const int per = nbins / kIcpThreads;
  unsigned int c[2048 / kIcpThreads], loc = 0;
  for (int j = 0; j < per; ++j) {
    unsigned int v = 0;  // sharded: the histogram is the sum of the shards' (slot g sits kWorkWords after slot g-1)
    for (int g = 0; g < n_slots; ++g) v += __ldcg(ghist + (size_t)g * kWorkWords + threadIdx.x * per + j);
    c[j] = v;
    loc += v;
  }
  unsigned int incl = loc;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned int v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  __syncthreads();  // ws reuse
  if (lane == 31) ws[warp] = incl;
  __syncthreads();
  unsigned int woff = 0, total = 0;
  for (int w = 0; w < kIcpThreads / 32; ++w) {
    const unsigned int v = ws[w];
    if (w < warp) woff += v;
    total += v;
  }
  if (first) {
    k = (unsigned int)((float)total * ratio);
    if (total > 0 && k >= total) k = total - 1;
  }
  unsigned int run = woff + incl - loc;
  for (int j = 0; j < per; ++j) {
    if (k >= run && k < run + c[j]) {
      out->bin = threadIdx.x * per + j;
      out->rem = k - run;
    }
    run += c[j];
  }
  if (threadIdx.x == 0) out->total = total;
  __syncthreads();
}

// ---- phase A building blocks ------------------------------------------------------------------------------------
// Per-query state (pos, d2, candidate lists) crosses CTAs -- it is written by whichever warp claimed the query in
// phase A and read by the static owner of the query in the select / correction passes -- so it always goes through
// L2 (.cg loads and stores), never through L1.

// Per-CTA histograms of the trimmed-quantile select (3-level radix over the float bits of d2: 10 + 11 + 10 bits).
// Level 1 is always built in phase A.  Levels 2 and 3 need the bin chosen at the level above -- which is only known
// a grid-wide barrier later -- so phase A builds them SPECULATIVELY for the bins of the previous iteration's limit;
// when the limit has moved by less than a bin (almost always once the registration settles) the whole select needs
// no further pass and no further barrier.
struct SelHists {
  unsigned int h1[1024];  // key >> 21
  unsigned int h2[2048];  // (key >> 10) & 2047 of the keys in the predicted level-1 bin
  unsigned int h3[1024];  // key & 1023 of the keys under the predicted (level-1, level-2) prefix
};
constexpr unsigned int kNoPrediction = 0xffffffffu;

// outcome of one query: remember the last real match as the next warm start, record d2, count it
__device__ __forceinline__ void phase_a_record(const IcpProblem& P, int i, const Best& b, SelHists* H, unsigned int pred_bin1,
                                               unsigned int pred_pref12) {
  if (b.pos >= 0) __stcg(P.pos + i, b.pos);
  const float d = b.pos >= 0 ? b.d2 : INFINITY;
  __stcg(P.d2 + i, d);
  const unsigned int key = __float_as_uint(d);
  if (key <= 0x7f800000u) {  // non-negative, not NaN; +inf (no match inside the cap) -> bin 1020
    atomicAdd(&H->h1[key >> 21], 1u);
    if ((key >> 21) == pred_bin1) {
      atomicAdd(&H->h2[(key >> 10) & 2047u], 1u);
      if ((key >> 10) == pred_pref12) atomicAdd(&H->h3[key & 1023u], 1u);
    }
  }
}

// Point-to-plane terms of one pair (PointToPlaneErrorMinimizer): f = [s x n; n], e = (s - q) . n, every operation
// individually rounded in this fixed order (oracle/icp_oracle.cpp).  The same function serves phase A and the
// correction pass, so a pair added in one and removed in the other cancels exactly.
__device__ __forceinline__ void residual_terms(float sx, float sy, float sz, const float4 q, const float4 nn, float* f, float& e) {
  float u = sy * nn.z, v = sz * nn.y;
  f[0] = u - v;
  u = sz * nn.x; v = sx * nn.z;
  f[1] = u - v;
  u = sx * nn.y; v = sy * nn.x;
  f[2] = u - v;
  f[3] = nn.x; f[4] = nn.y; f[5] = nn.z;
  const float dx = sx - q.x, dy = sy - q.y, dz = sz - q.z;
  e = dx * nn.x;
  float t = dy * nn.y;
  e = e + t;
  t = dz * nn.z;
  e = e + t;
}

// ---- normal equations: A = sum f f^T (21 unique entries), b = sum f e (6), number of pairs (1) -------------------
// Every product is a float32 product quantised to 2^-22 and summed as int64 -- exact, hence independent of any
// ordering (oracle/icp_oracle.cpp).  Pairs are not reduced across lanes as they come (that took 81 warp-wide integer
// reductions per 32 queries): each warp queues the pairs that count as 8-float records {f0..f5, e, sign} in shared
// memory and, whenever 32 are waiting, lane k walks all 32 records for ITS entry of the system -- 28 lanes, 28
// private int64 sums held in registers for the whole pass, no cross-lane traffic at all.  A record with sign -1
// removes a pair that an earlier pass added (same floats, same products: cancels exactly).
constexpr int kPairSlots = 64;  // per warp: up to 31 waiting + 32 arriving
constexpr int kIcpPairBytes = (kIcpThreads / 32) * kPairSlots * 8 * (int)sizeof(float);  // dynamic shared memory of icp_kernel
__constant__ unsigned char kPairRow[32] = {0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 4, 4, 5, 0, 1, 2, 3, 4, 5, 7, 7, 7, 7, 7};
__constant__ unsigned char kPairCol[32] = {0, 1, 2, 3, 4, 5, 1, 2, 3, 4, 5, 2, 3, 4, 5, 3, 4, 5, 4, 5, 5, 6, 6, 6, 6, 6, 6, 7, 7, 7, 7, 7};

struct PairQueue {
  float* recs;    // kPairSlots x 8 floats, shared memory, this warp's
  int head, cnt;  // warp-uniform
  long long acc;  // lane k < 28: its entry's running sum
};

// lanes 0..20: upper triangle of A; 21..26: b; 27: count (sign * sign quantised with scale 1); 28..31 idle copies of 27
__device__ __noinline__ long long consume_pairs(const float* recs, int head, int count, long long acc) {
  const int lane = threadIdx.x & 31;
  const int ro = kPairRow[lane], co = kPairCol[lane];
  const float scale = lane < 27 ? 4194304.0f : 1.0f;
#pragma unroll 4
  for (int j = 0; j < count; ++j) {
    const float* r = recs + ((head + j) & (kPairSlots - 1)) * 8;
    const float a = r[ro], b = r[co], sg = r[7];
    long long v = __float2ll_rn((a * b) * scale);
    if (sg < 0.f) v = -v;
    acc += v;
  }
  return acc;
}

// Warp-collective (all 32 lanes, converged): lanes with sign != 0 queue the pair (query at s, matched point q at sorted
// position pos, its normal fetched here).
__device__ __forceinline__ void push_pairs(const IcpProblem& P, PairQueue& Q, int sign, float sx, float sy, float sz,
                                           const float4 q, int pos) {
  const unsigned int m = __ballot_sync(0xffffffffu, sign != 0);
  if (m == 0u) return;  // warp-uniform
  if (sign) {
    float f[6], e;
    residual_terms(sx, sy, sz, q, __ldg(P.nrm + pos), f, e);
    const int slot = (Q.head + Q.cnt + __popc(m & ((1u << (threadIdx.x & 31)) - 1u))) & (kPairSlots - 1);
    float4* r = reinterpret_cast<float4*>(Q.recs + slot * 8);
    r[0] = make_float4(f[0], f[1], f[2], f[3]);
    r[1] = make_float4(f[4], f[5], e, (float)sign);
  }
  Q.cnt += __popc(m);
  __syncwarp();
  if (Q.cnt >= 32) {
    Q.acc = consume_pairs(Q.recs, Q.head, 32, Q.acc);
    Q.head = (Q.head + 32) & (kPairSlots - 1);
    Q.cnt -= 32;
    __syncwarp();
  }
}

// end of a pass: consume what is waiting, hand the lane sums to the CTA (slab), start from zero
__device__ __forceinline__ void drain_pairs(PairQueue& Q, unsigned long long* slab) {
  if (Q.cnt > 0) {
    Q.acc = consume_pairs(Q.recs, Q.head, Q.cnt, Q.acc);
    Q.head = (Q.head + Q.cnt) & (kPairSlots - 1);
    Q.cnt = 0;
  }
  const int lane = threadIdx.x & 31;
  if (lane < 28) slab[lane] = (unsigned long long)Q.acc;
  Q.acc = 0ll;
  __syncwarp();
}

// Slow path of phase A: the search itself (warm-started, inside the cap) -- from the second iteration on together with
// the list that lets later iterations skip it, in the same walk (nn_search_collect decides whether a list can pay off
// from how far the last step moved this query: T_prev is the previous iteration's T_iter).  Not inlined: the search
// wants the whole register budget for itself, not the caller's loop state spilled into its inner loops.  Called by all
// 32 lanes (i < 0: nothing to do); the outcome is left in the query's state (P.pos / P.d2), where the caller -- the
// same thread -- reads it back.
__device__ __noinline__ void phase_a_search(const Grid* gp, const IcpProblem* Pp, const float* T_iter, const float* T_prev,
                                            int i, float cap, SelHists* H, unsigned int pred_bin1, unsigned int pred_pref12) {
  if (i < 0) return;
  const Grid& g = *gp;
  const IcpProblem& P = *Pp;
  const float4 r = __ldg(P.rd + i);
  float sx, sy, sz;
  xform_point(T_iter, r.x, r.y, r.z, sx, sy, sz);
  const int warm = __ldcg(P.pos + i);
  Best b;
  if (T_prev) {
    float px, py, pz;
    xform_point(T_prev, r.x, r.y, r.z, px, py, pz);
    b = nn_search_collect(g, P.view, P.lists, i, sx, sy, sz, warm, cap, sqrtf(dist2(sx, sy, sz, px, py, pz)));
  } else {
    b = nn_search(g, P.view, sx, sy, sz, warm, cap);
  }
  phase_a_record(P, i, b, H, pred_bin1, pred_pref12);
}

// Warp-collective: the queries just searched (j < 0: none on this lane) whose match lies inside the accumulation
// limit queue their pairs.  The match is read back from the query's state, written by this very thread.
__device__ __forceinline__ void push_searched(const IcpProblem& P, PairQueue& Q, const float* T_iter, int j, float acc_limit) {
  if (!(acc_limit >= 0.0f)) return;  // uniform: nothing enters the normal equations during phase A
  float d = INFINITY;
  if (j >= 0) d = __ldcg(P.d2 + j);
  const bool keep = d <= acc_limit;  // finite d2 <=> matched in this iteration, P.pos[j] is that match
  if (__ballot_sync(0xffffffffu, keep) == 0u) return;
  float4 q = make_float4(0.f, 0.f, 0.f, 0.f);
  float sx = 0.f, sy = 0.f, sz = 0.f;
  int pos = -1;
  if (keep) {
    pos = __ldcg(P.pos + j);
    const float4 r = __ldg(P.rd + j);
    xform_point(T_iter, r.x, r.y, r.z, sx, sy, sz);
    q = __ldg(P.view.pts + pos);
  }
  push_pairs(P, Q, keep ? 1 : 0, sx, sy, sz, q, pos);
}

// After the loop, when the caller asked for correspondences: every point's true (uncapped) match under T.
__device__ __noinline__ void final_match(const Grid* gp, const IcpProblem* Pp, const float* T, int i) {
  if (i < 0) return;  // called by whole warps (a divergent call of a non-inlined function miscompiled once: never again)
  const IcpProblem& P = *Pp;
  const float4 r = __ldg(P.rd + i);
  float sx, sy, sz;
  xform_point(T, r.x, r.y, r.z, sx, sy, sz);
  const Best b = nn_search(*gp, P.view, sx, sy, sz, __ldcg(P.pos + i), INFINITY);
  const uint32_t orig = __ldg(P.qperm + i);
  P.d2_out[orig] = b.d2;
  P.ids[orig] = b.idx;
}

// CTA-wide: fold the warps' sums (drain_pairs) into the problem's accumulators (L2 atomics).
__device__ __forceinline__ void flush_slabs(unsigned long long (*acc_w)[28], unsigned long long* gacc) {
  __syncthreads();
  if (threadIdx.x < 28) {
    unsigned long long t = 0ull;
#pragma unroll
    for (int w = 0; w < kIcpThreads / 32; ++w) t += acc_w[w][threadIdx.x];
    if (t != 0ull) atomicAdd(&gacc[threadIdx.x], t);
  }
  __syncthreads();  // the slabs may be rewritten
}

__device__ __forceinline__ void flush_hist(const unsigned int* hs, int nbins, unsigned int* gh) {
  for (int k = threadIdx.x; k < nbins; k += kIcpThreads) {
    const unsigned int v = hs[k];
    if (v) atomicAdd(&gh[k], v);
  }
}

// One iteration, seen from one problem's group of CTAs (G of them, each owning a contiguous chunk of the queries for
// the passes that read per-query state back):
//   A   every query gets its match -- from its certified candidate list when that proves the answer, from the search
//       otherwise -- and on the spot: its d2 enters the select histograms (all three radix levels, the lower two
//       speculatively) and, when d2 <= the PREVIOUS iteration's limit, its pair enters the normal equations
//   --  barrier
//   S   every CTA resolves the trimmed limit from the histograms (a pass over d2 + a barrier per level only where
//       the speculation missed), then corrects the normal equations for the queries between the previous and the
//       actual limit: +pair / -pair, exact because the sums are integers
//   --  barrier
//   E   every CTA solves the 6x6 system, updates T_iter and runs the transformation checkers, identically
// i.e. two grid-wide barriers per iteration once the limit moves by less than a histogram bin per iteration.
__global__ void __launch_bounds__(kIcpThreads, kIcpCtasPerSm)
icp_kernel(const IcpProblem* __restrict__ probs, int ctas_per_problem, IcpParamsDev prm, int dynamic) {
  const int pi = blockIdx.x / ctas_per_problem;
  const int cta = blockIdx.x - pi * ctas_per_problem;
  const IcpProblem& P = probs[pi];
  IcpWork* W = P.work;                 // work counters, results
  const bool xg = P.shard_count > 1;   // query-sharded over several GPUs (ShardLink)
  IcpWork* X = xg ? P.link.slots + P.shard_rank : W;   // where this GPU's CTAs accumulate histograms and sums
  const IcpWork* S0 = xg ? P.link.slots : W;           // first of the n_slots slots a reader sums
  const int n_slots = xg ? P.shard_count : 1;
  const unsigned int G = (unsigned int)ctas_per_problem;
  unsigned int xepoch = 0;             // arrivals expected from the peers so far
  const int tid = threadIdx.x, lane = tid & 31;

  __shared__ Grid g;
  __shared__ float T_iter[16], T_last[16];
  __shared__ SelHists hs;
  __shared__ unsigned long long acc_w[kIcpThreads / 32][28];
  __shared__ SelectOut sel;
  __shared__ unsigned int ws[kIcpThreads / 32];
  __shared__ double qh[kMaxSmooth + 2][4];
  __shared__ double th[kMaxSmooth + 2][3];
  __shared__ int flag_stop, flag_status;
  __shared__ int miss_buf[kIcpThreads / 32][64];  // per-warp queue of queries whose list did not certify
  extern __shared__ __align__(16) float pair_buf[];  // kIcpPairBytes, dynamic: per-warp queues of pairs (PairQueue)

  if (tid == 0) {
    g = P.bs->grid;
    for (int i = 0; i < 16; ++i) T_iter[i] = (i % 5 == 0) ? 1.f : 0.f;
    quat_from_T(T_iter, qh[0]);
    th[0][0] = th[0][1] = th[0][2] = 0.0;
    flag_stop = 0;
    flag_status = 0;
  }
  __syncthreads();
  PairQueue Q;
  Q.recs = pair_buf + (tid >> 5) * (kPairSlots * 8);
  Q.head = 0;
  Q.cnt = 0;
  Q.acc = 0ll;

  // contiguous chunk of queries per CTA (spatially compact, coalesced)
  const int n = P.n;
  int chunk = (n + (int)G - 1) / (int)G;
  chunk = (chunk + 31) & ~31;
  const int q_begin = min(n, cta * chunk), q_end = min(n, q_begin + chunk);

  for (int i = q_begin + tid; i < q_end; i += kIcpThreads) {
    __stcg(P.pos + i, -1);
    __stcg(P.lists.vq + i, make_float4(0.f, 0.f, 0.f, 0.f));  // no list yet
  }

  // Trim-aware search cap (squared metres).  TrimmedDistOutlierFilter keeps matches with d2 <= limit,
  // so a match only has to be exact if d2 <= limit; searching inside a ball of radius sqrt(cap) with
  // cap >= limit finds exactly those.  cap is a GUESS (first iteration: 0.04 m^2; second: half the first limit;
  // then twice the previous limit) that is VERIFIED every iteration: points without a match inside
  // the cap are counted in the +inf histogram bin, and if the quantile lands in that bin the queries that found
  // nothing -- only those: a match found inside a smaller cap is the nearest neighbour under any cap -- are
  // searched again with a 4x larger cap (`redo` counts these rounds).
  float cap = 0.04f;
  int redo = 0;
  unsigned int epoch = 0;
  // grid-wide step: a barrier, or -- sharded -- a barrier + the exchange of up to three sections of the scratch
  constexpr int kHistOff = (int)(offsetof(IcpWork, hist) / 4), kAccOff = (int)(offsetof(IcpWork, acc) / 4);
  auto meet = [&](int off0, int n0, int off1, int n1, int off2, int n2) {
    if (xg) shard_exchange(P, X, cta, G, epoch, xepoch, off0, n0, off1, n1, off2, n2);
    else problem_barrier(&X->barrier, G, epoch);
  };
  problem_barrier(&X->barrier, G, epoch);  // the state initialised above is read by other CTAs
  int hist_count = 1;  // entries in qh/th
  int iter = 0, converged = 0, max_reached = 0, last_kept = 0;
  float last_limit = 0.f;
  // what the previous iteration predicts for this one (uniform over the CTA, identical in every CTA)
  unsigned int pred_bin1 = kNoPrediction, pred_pref12 = kNoPrediction;
  float acc_limit = -1.0f;  // pairs with d2 <= acc_limit enter the normal equations in phase A (< 0: none do)

  for (;;) {
    const int par = iter & 1;
    LS_STAMP(0);
    // ---------------- phase A ----------------
    for (int k = tid; k < (int)(sizeof(SelHists) / 4); k += kIcpThreads) reinterpret_cast<unsigned int*>(&hs)[k] = 0u;
    __syncthreads();
    {
      // Every warp walks its share of the queries 32 at a time.  A query whose candidate list certifies the answer
      // is done on the spot (one round trip of coalesced loads); the others are queued PER WARP and searched 32 at
      // a time, so the expensive, divergent search always runs on full warps even when only a few percent of the
      // queries need it.
      const float* T_prev = iter >= 1 ? T_last : nullptr;  // lists are built from the second iteration on
      int* mq = miss_buf[tid >> 5];
      int n_miss = 0;                    // warp-uniform
      int next = q_begin + (tid & ~31);  // static schedule: this warp's next 32 queries
      for (;;) {
        int base;
        if (dynamic) {
          // Several problems per launch: warps claim 32 consecutive queries at a time from the problem's counter, so
          // every warp of the problem runs out of work at (almost) the same moment instead of parking at the
          // barrier -- and starving the co-resident CTA of another problem.
          unsigned int bb = 0;
          if (lane == 0) bb = atomicAdd(&W->qctr[par], 32u);
          bb = __shfl_sync(0xffffffffu, bb, 0);
          if (bb >= (unsigned int)n) break;
          base = (int)bb;
        } else {
          if (next >= q_end) break;  // one problem owns the whole grid: contiguous chunk per CTA
          base = next;
          next += kIcpThreads;
        }
        const int i = base + lane;
        bool valid = i < (dynamic ? n : q_end);
        if (redo && valid) valid = !(__ldcg(P.d2 + i) < INFINITY);  // matched in an earlier round of this iteration: final
        bool hit = false;
        Best b;
        b.d2 = INFINITY; b.idx = INT_MAX; b.pos = -1;
        float4 c = make_float4(0.f, 0.f, 0.f, 0.f);
        float sx = 0.f, sy = 0.f, sz = 0.f;
        if (valid) {
          // reading point, list header, first candidate: three addresses known up front, one round trip
          const float4 r = __ldg(P.rd + i);
          const float4 v = __ldcg(P.lists.vq + i);
          const float4 c0 = __ldcg(P.lists.vpts + i);
          xform_point(T_iter, r.x, r.y, r.z, sx, sy, sz);
          hit = vlist_query(P.lists, P.view.pts, i, v, c0, sx, sy, sz, cap, b, c);
          if (hit) phase_a_record(P, i, b, &hs, pred_bin1, pred_pref12);
        }
        push_pairs(P, Q, (hit && b.pos >= 0 && b.d2 <= acc_limit) ? 1 : 0, sx, sy, sz, c, b.pos);
        const unsigned int mm = __ballot_sync(0xffffffffu, valid && !hit);
        if (mm) {
          if (valid && !hit) mq[n_miss + __popc(mm & ((1u << lane) - 1u))] = i;
          n_miss += __popc(mm);
          __syncwarp();
          if (n_miss >= 32) {
            n_miss -= 32;
            const int j = mq[n_miss + lane];
            __syncwarp();
            phase_a_search(&g, &P, T_iter, T_prev, j, cap, &hs, pred_bin1, pred_pref12);
            push_searched(P, Q, T_iter, j, acc_limit);
          }
        }
      }
      if (n_miss > 0) {  // warp-uniform: the last, partial batch of searches
        __syncwarp();
        const int j = lane < n_miss ? mq[lane] : -1;
        phase_a_search(&g, &P, T_iter, T_prev, j, cap, &hs, pred_bin1, pred_pref12);
        __syncwarp();
        push_searched(P, Q, T_iter, j, acc_limit);
      }
    }
    drain_pairs(Q, acc_w[tid >> 5]);
    flush_slabs(acc_w, X->acc[par]);  // (starts with a __syncthreads: every warp is done with phase A)
    flush_hist(hs.h1, 1024, X->hist[par][0]);
    if (pred_bin1 != kNoPrediction) {
      flush_hist(hs.h2, 2048, X->hist[par][3]);
      flush_hist(hs.h3, 1024, X->hist[par][4]);
    }
    {
      const int hb = kHistOff + par * 5 * 2048;
      const bool pr = pred_bin1 != kNoPrediction;
      meet(hb, 1024, hb + 3 * 2048, pr ? 2048 : 0, hb + 4 * 2048, pr ? 1024 : 0);
    }
    LS_STAMP(1);

    // ---------------- select, level 1 ----------------
    block_select(S0->hist[par][0], 1024, 0u, true, prm.trim_ratio, &sel, ws, n_slots);
    if (sel.total == 0u) {  // no point at all -> ConvergenceError
      if (tid == 0) { flag_status = 1; if (cta == 0) W->fail_code = 1; }
      __syncthreads();
      break;
    }
    if (sel.bin >= 1020u) {
      // the quantile fell among the points with no match inside the cap: the cap was too small.
      if (!(cap < INFINITY)) {  // uncapped and still +inf: empty map
        if (tid == 0) { flag_status = 1; if (cta == 0) W->fail_code = 1; }
        __syncthreads();
        break;
      }
      cap = cap < 64.0f ? cap * 4.0f : INFINITY;
      ++redo;
      meet(0, 0, 0, 0, 0, 0);  // everyone, on every shard, has read the histogram
      if (cta == 0 && tid == 0) {
        X->hist[par][0][1020] = 0u;  // the unmatched queries are counted again; everything else stands
        W->qctr[par] = 0u;
      }
      problem_barrier(&X->barrier, G, epoch);
      continue;  // phase A again, for the queries without a match, with the larger cap
    }
    const unsigned int bin1 = sel.bin, rem1 = sel.rem;
    if (cta == 0) {  // clear the other parity's scratch for the next iteration (nobody touches it before the next barrier)
      unsigned int* h = &X->hist[par ^ 1][0][0];
      for (int k = tid; k < 5 * 2048; k += kIcpThreads) h[k] = 0u;
      if (tid < 32) X->acc[par ^ 1][tid] = 0ull;
    }
    if (cta == 0 && tid == 0) W->qctr[par ^ 1] = 0u;
    // ---------------- level 2: from the speculative histogram, or a pass over d2 + barrier ----------------
    const bool spec2 = bin1 == pred_bin1;
    if (!spec2) {
      for (int k = tid; k < 2048; k += kIcpThreads) hs.h2[k] = 0u;
      __syncthreads();
      for (int i = q_begin + tid; i < q_end; i += kIcpThreads) {
        const unsigned int key = __float_as_uint(__ldcg(P.d2 + i));
        if (key < 0x7f800000u && (key >> 21) == bin1) atomicAdd(&hs.h2[(key >> 10) & 2047u], 1u);
      }
      __syncthreads();
      flush_hist(hs.h2, 2048, X->hist[par][1]);
      meet(kHistOff + (par * 5 + 1) * 2048, 2048, 0, 0, 0, 0);
    }
    LS_STAMP(2);
    block_select(S0->hist[par][spec2 ? 3 : 1], 2048, rem1, false, 0.f, &sel, ws, n_slots);
    const unsigned int bin2 = sel.bin, rem2 = sel.rem;
    const unsigned int prefix12 = (bin1 << 11) | bin2;
    // ---------------- level 3 ----------------
    const bool spec3 = spec2 && prefix12 == pred_pref12;
    if (!spec3) {
      for (int k = tid; k < 1024; k += kIcpThreads) hs.h3[k] = 0u;
      __syncthreads();
      for (int i = q_begin + tid; i < q_end; i += kIcpThreads) {
        const unsigned int key = __float_as_uint(__ldcg(P.d2 + i));
        if (key < 0x7f800000u && (key >> 10) == prefix12) atomicAdd(&hs.h3[key & 1023u], 1u);
      }
      __syncthreads();
      flush_hist(hs.h3, 1024, X->hist[par][2]);
      meet(kHistOff + (par * 5 + 2) * 2048, 1024, 0, 0, 0, 0);
    }
    LS_STAMP(3);
    block_select(S0->hist[par][spec3 ? 4 : 2], 1024, rem2, false, 0.f, &sel, ws, n_slots);
    const float limit = __uint_as_float((prefix12 << 10) | sel.bin);
    // guess for the next iteration (verified there): the first step removes most of the initial misalignment, so the
    // limit drops sharply once and then settles -- a guess that turns out too small costs one more round for the
    // unmatched queries only
    cap = fmaxf(limit * (iter == 0 ? 0.5f : 2.0f), 1e-12f);
    redo = 0;

    // ---------------- correction pass: pairs between the predicted and the actual limit ----------------
    // Phase A added every pair with d2 <= acc_limit; the minimiser wants exactly those with d2 <= limit.
    for (int base = q_begin; base < q_end; base += kIcpThreads) {
      const int i = base + tid;
      int sign = 0, pos = -1;
      if (i < q_end) {
        const float d = __ldcg(P.d2 + i);
        pos = __ldcg(P.pos + i);
        sign = ((d <= limit && pos >= 0) ? 1 : 0) - ((d <= acc_limit) ? 1 : 0);  // d2 is +inf where nothing was found
      }
      if (__ballot_sync(0xffffffffu, sign != 0) == 0u) continue;  // warp-uniform
      float sx = 0.f, sy = 0.f, sz = 0.f;
      float4 q = make_float4(0.f, 0.f, 0.f, 0.f);
      if (sign) {
        const float4 r = __ldg(P.rd + i);
        xform_point(T_iter, r.x, r.y, r.z, sx, sy, sz);
        q = __ldg(P.view.pts + pos);
      }
      push_pairs(P, Q, sign, sx, sy, sz, q, pos);
    }
    drain_pairs(Q, acc_w[tid >> 5]);
    flush_slabs(acc_w, X->acc[par]);
    meet(kAccOff + par * 64, 64, 0, 0, 0, 0);
    LS_STAMP(4);

    // ---------------- phase E: solve, update, checkers (every CTA, identically) ----------------
    if (tid == 0) {
      double A[36], b[6], x[6];
      int k = 0;
      for (int rr = 0; rr < 6; ++rr)
        for (int cc = rr; cc < 6; ++cc, ++k) {
          const double v = (double)(long long)sum_slots_u64(&S0->acc[par][k], n_slots) / 4194304.0;
          A[rr * 6 + cc] = v;
          A[cc * 6 + rr] = v;
        }
      for (int rr = 0; rr < 6; ++rr) b[rr] = -((double)(long long)sum_slots_u64(&S0->acc[par][21 + rr], n_slots) / 4194304.0);
      last_kept = (int)sum_slots_u64(&S0->acc[par][27], n_slots);
      last_limit = limit;
      int status = 0, stop = 0;
      if (last_kept == 0) {
        status = 1;
        if (cta == 0) W->fail_code = 2;
      } else {
        if (!chol6(A, b, x)) jacobi_pinv_solve6(A, b, x);
        for (int i = 0; i < 6; ++i)
          if (!is_finite_d(x[i])) status = 1;
        if (status && cta == 0) W->fail_code = 3;
      }
      if (cta == 0) {
        W->dbg_total = sel.total; W->dbg_bin[0] = bin1; W->dbg_bin[1] = bin2; W->dbg_bin[2] = sel.bin;
        W->dbg_rem[0] = rem1; W->dbg_rem[1] = rem2; W->dbg_rem[2] = sel.rem;
        for (int i = 0; i < 6; ++i) { W->dbg_A[i] = A[i * 6 + i]; W->dbg_x[i] = x[i]; }
      }
      if (!status) {
        float T_step[16];
        step_matrix(x, T_step);
        for (int i = 0; i < 16; ++i) T_last[i] = T_iter[i];
        mat4_mul(T_step, T_iter, T_iter);
        if (P.T_hist && cta == 0)
          for (int i = 0; i < 16; ++i) P.T_hist[iter * 16 + i] = T_iter[i];
        if (iter + 1 >= prm.max_iterations) { stop = 1; max_reached = 1; }
        if (prm.use_differential) {
          const int L = prm.smooth_length;
          // ring buffer of the last L+1 (quaternion, translation) samples
          if (hist_count == L + 1) {
            for (int i = 0; i < L; ++i) {
              for (int c = 0; c < 4; ++c) qh[i][c] = qh[i + 1][c];
              for (int c = 0; c < 3; ++c) th[i][c] = th[i + 1][c];
            }
            --hist_count;
          }
          quat_from_T(T_iter, qh[hist_count]);
          th[hist_count][0] = (double)T_iter[12];
          th[hist_count][1] = (double)T_iter[13];
          th[hist_count][2] = (double)T_iter[14];
          ++hist_count;
          if (hist_count > L) {
            double mr = 0.0, mt = 0.0;
            for (int i = hist_count - 1; i >= hist_count - L; --i) {
              mr += fabs(quat_angular_distance(qh[i], qh[i - 1]));
              const double ddx = th[i][0] - th[i - 1][0], ddy = th[i][1] - th[i - 1][1], ddz = th[i][2] - th[i - 1][2];
              mt += sqrt(ddx * ddx + ddy * ddy + ddz * ddz);
            }
            mr /= (double)L;
            mt /= (double)L;
            if (mr != mr || mt != mt) { status = 1; if (cta == 0) W->fail_code = 4; }
            else if (mr < (double)prm.min_diff_rot && mt < (double)prm.min_diff_trans) { stop = 1; converged = 1; }
          }
        }
      }
      flag_status = status;
      flag_stop = stop | status;
      LS_STAMP(5);
    }
    __syncthreads();
    if (!flag_status) ++iter;  // every thread tracks the iteration count (parity, warm start)
    if (flag_stop) break;
    // what this iteration predicts for the next: the select bins of its limit, and -- once the limit has stopped
    // falling by large factors -- the limit itself as the threshold of phase A's accumulation
    pred_bin1 = bin1;
    pred_pref12 = prefix12;
    acc_limit = iter >= 2 ? limit : -1.0f;
  }

  if (P.want_matches && !flag_status && iter > 0) {
    // The loop ended right after the update of T_iter; the matches reported are those of the LAST
    // iteration, i.e. of the reading under T_last.  Redo that query without a cap.
    for (int base = q_begin; base < q_end; base += kIcpThreads) final_match(&g, &P, T_last, base + tid < q_end ? base + tid : -1);
  }

  if (cta == 0 && tid == 0) {
    int status = flag_status;
    float T_mean[16], tmp[16], T_fin[16];
    for (int i = 0; i < 16; ++i) T_mean[i] = (i % 5 == 0) ? 1.f : 0.f;
    T_mean[12] = g.mu[0]; T_mean[13] = g.mu[1]; T_mean[14] = g.mu[2];
    mat4_mul(T_mean, T_iter, tmp);
    mat4_mul(tmp, P.bs->T_pre, T_fin);
    for (int i = 0; i < 16; ++i)
      if (!is_finite_f(T_fin[i])) { status = 1; W->fail_code = 5; }
    for (int i = 0; i < 16; ++i) W->T_out[i] = status ? P.T0[i] : T_fin[i];
    W->status = status;
    W->iterations = iter;
    W->converged = converged;
    W->max_iter_reached = max_reached;
    W->last_kept = last_kept;
    W->last_limit = last_limit;
    W->xsignals = xepoch;
  }
}

}  // namespace ls
