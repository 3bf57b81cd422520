// Box status and robot collision on the resident occupancy map: volumetric_mapping's getCellStatusBoundingBox,
// checkCollisionWithRobot and checkPathForCollisionsWithRobot, batched (DESIGN.md §4b''''''''''').  Reads the map only
// (tab_keys / tab_vals, known, lo) on the map's stream; the insert, edit, query and tree kernels do not know it exists.
//   (a) co_axis_kernel    one thread per (box, axis): the size check, the corners and their keys, the unknown loop run
//                         sequentially as written (its point count, first and last valid key, any invalid point), the
//                         cube test of every key between the corner keys (the passing keys), the axis's brick range
//   (b) co_box_kernel     one thread per box: steps 1 and 2 (the centre's state in double, the float centre's key); a box
//                         they decide gets no work, the others the product of their axes' brick counts
//       CUB inclusive scans over the per-axis brick counts and the per-box items; one readback: the refusal flags and the
//       totals, which size the masks and the voxel pass.  A call whose boxes span more than 2^36 (box, brick) items (counted
//       from the boxes alone, whatever the map holds) is refused, so the item numbers fit and the pass takes bounded time
//   (c) co_mask_kernel    one thread per (box, axis): per brick of the axis, the 8-bit mask of its keys the loop reaches
//                         and the 8-bit mask of its keys that pass the cube test
//   (d) co_voxel_kernel   one warp per (box, brick) item, each warp of a grid of at most 2^16 blocks striding over the
//                         items: the brick's known words and log-odds against the masks; raises
//                         the box's occupied or unknown flag, and in path mode lowers the path's first collision with
//                         atomicMin.  Items of a box already occupied (or of a pose at or after its path's first
//                         collision) stop
//   (e) co_result_kernel  per box its status, or per path its first collision; one readback with the keys visited
// The result does not depend on the scheduling: occupied beats unknown, unknown beats free, and the minimum is exact.
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <vector>

#include <cub/cub.cuh>
#include <cuda_runtime.h>

#include "../../include/ls_b200.h"
#include "ls_occupancy.cuh"

namespace lso {
namespace {

constexpr long long kMaxAxisPoints = 1LL << 17;  // loop points per box axis
constexpr unsigned kFlagOcc = 1u, kFlagUnk = 2u;
constexpr unsigned kNone = 0xffffffffu;  // a path without a collision (yet)
constexpr int kWarpsPerBlock = 8;
constexpr unsigned kVoxelBlocks = 1u << 16;    // (d)'s grid: its warps stride over the items
constexpr double kMaxWork = 68719476736.0;    // 2^36 (box, brick) items per call, counted whatever the map holds

// The counters of one call: refusal bits (1 a size, 2 a loop of more than 2^17 points) and the (box, brick) items every
// box with a valid centre spans, whatever the map holds (a sum of integers below 2^42 each, exact in double below 2^53).
struct CallCounters {
  unsigned refused, pad;
  double work;
};

// One axis of one box after (a).  The passing keys [oa, ob] (empty when oa > ob) are those between the corner keys whose
// cube meets [bmin, bmax]; `corners` is 0 when a corner key is invalid (no occupied pass for the box).  The axis's bricks
// are b0 ... b0 + nb - 1.
struct Axis {
  int b0, nb;
  int oa, ob;
  int corners, invalid;  // invalid: some loop point has an invalid key
};

// The centre of box i has a valid key on every axis by the double rule, octomap's search(x, y, z) (step 1 can look it up).
// Every other key of the call is a float coordinate's.
__device__ __forceinline__ bool centre_keys(const double* c3, long long i, double inv, int k[3]) {
  return key_of(inv, c3[3 * i], k[0]) && key_of(inv, c3[3 * i + 1], k[1]) && key_of(inv, c3[3 * i + 2], k[2]);
}

// (a): one thread per (box, axis).  s_stride 3: a size per box; 0: one size for every box (the robot's).
__global__ void co_axis_kernel(const double* __restrict__ c3, const double* __restrict__ s3, int s_stride, long long n,
                               double res, double inv, Axis* __restrict__ axes, long long* __restrict__ nb_out,
                               CallCounters* __restrict__ ctr) {
  unsigned* refused = &ctr->refused;
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= 3 * n) return;
  const long long i = t / 3;
  const int a = (int)(t % 3);
  Axis A{0, 0, 1, 0, 0, 0};
  const double s = s3[(size_t)s_stride * i + a];
  int kc[3];
  if (!(s >= 0.0) || isinf(s)) {
    atomicOr(refused, 1u);
  } else if (centre_keys(c3, i, inv, kc)) {  // a centre with an invalid key is unknown: no loop, no refusal
    const double p = c3[3 * i + a];
    const float bmin = (float)(p - s / 2), bmax = (float)(p + s / 2);
    // the unknown pass's loop, accumulated as written
    long long points = 0;
    int first = -1, last = -1, k;
    for (double x = bmin; x <= bmax; x += res) {
      if (++points > kMaxAxisPoints) {
        atomicOr(refused, 2u);
        break;
      }
      if (key_of(inv, (float)x, k)) {
        if (first < 0) first = k;
        last = k;
      } else {
        A.invalid = 1;
      }
    }
    if (points <= kMaxAxisPoints) {
      int kmin, kmax;
      const double half = res / 2;
      if (key_of(inv, bmin, kmin) && key_of(inv, bmax, kmax)) {
        A.corners = 1;
        for (int q = kmin; q <= kmax; ++q) {  // the cube test of every key in the range
          const double c = centre_d(q, res);
          if (c + half < (double)bmin || c - half > (double)bmax) continue;
          if (A.oa > A.ob) A.oa = q;
          A.ob = q;
        }
      }
      int lo = first, hi = last;
      if (A.oa <= A.ob) {
        lo = lo < 0 ? A.oa : min(lo, A.oa);
        hi = hi < 0 ? A.ob : max(hi, A.ob);
      }
      if (lo >= 0) A.b0 = lo >> 3, A.nb = (hi >> 3) - (lo >> 3) + 1;
    }
  }
  axes[t] = A;
  nb_out[t] = A.nb;
}

// (b): one thread per box.  dec: the status steps 1 and 2 decide, or -1; flags: kFlagUnk when a loop point is invalid;
// items: the box's bricks for (d), 0 when decided (its axes' brick counts are zeroed so (c) skips them).  Path mode (pid
// not NULL): the pose's path, and a pose that collides already lowers best.
__global__ void co_box_kernel(const double* __restrict__ c3, long long n, double inv, const unsigned long long* __restrict__ tab_keys,
                              const int* __restrict__ tab_vals, unsigned tab_mask, const unsigned* __restrict__ known,
                              const float* __restrict__ lo, float l_occ, const Axis* __restrict__ axes,
                              long long* __restrict__ nb, long long* __restrict__ items, signed char* __restrict__ dec,
                              unsigned* __restrict__ flags, const long long* __restrict__ offsets, int n_paths,
                              int unknown_occ, int* __restrict__ pid, unsigned* __restrict__ best,
                              unsigned long long* __restrict__ visited, CallCounters* __restrict__ ctr) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  unsigned long long v = 0;
  double work = 0.0;
  if (i < n) {
    int k[3];
    int st = -1;
    if (!centre_keys(c3, i, inv, k)) {
      st = LS_CELL_UNKNOWN;  // step 1: an invalid key is unknown
    } else {
      ++v;
      const int b = lookup_brick(tab_keys, tab_vals, tab_mask, brick_key(k));
      const int s = b < 0 ? LS_CELL_UNKNOWN : voxel_state(known, lo, l_occ, b, local_of(k), nullptr);
      if (s != LS_CELL_FREE) st = s;
      else if (!(key_of(inv, (float)c3[3 * i], k[0]) && key_of(inv, (float)c3[3 * i + 1], k[1]) &&
                 key_of(inv, (float)c3[3 * i + 2], k[2])))
        st = LS_CELL_UNKNOWN;  // step 2: the float centre's key is invalid
    }
    const Axis X = axes[3 * i], Y = axes[3 * i + 1], Z = axes[3 * i + 2];
    work = (double)X.nb * Y.nb * Z.nb;  // < 2^42: exact
    unsigned f = (X.invalid | Y.invalid | Z.invalid) ? kFlagUnk : 0u;
    dec[i] = (signed char)st;
    flags[i] = st < 0 ? f : 0u;
    items[i] = st < 0 ? (long long)X.nb * Y.nb * Z.nb : 0;
    if (st >= 0) nb[3 * i] = nb[3 * i + 1] = nb[3 * i + 2] = 0;
    if (pid) {
      long long l = 0, h = n_paths;  // the last path whose first pose is <= i (empty paths share their offset)
      while (h - l > 1) {
        const long long mid = (l + h) >> 1;
        if (offsets[mid] <= i) l = mid;
        else h = mid;
      }
      pid[i] = (int)l;
      const bool hit = st >= 0 ? (st == LS_CELL_OCCUPIED || (unknown_occ && st == LS_CELL_UNKNOWN))
                               : (unknown_occ && f != 0u);
      if (hit) atomicMin(&best[l], (unsigned)(i - offsets[l]));
    }
  }
  for (int o = 16; o > 0; o >>= 1) {
    v += __shfl_down_sync(0xffffffffu, v, o);
    work += __shfl_down_sync(0xffffffffu, work, o);
  }
  if ((threadIdx.x & 31) == 0) {
    if (v) atomicAdd(visited, v);
    if (work > 0.0) atomicAdd(&ctr->work, work);
  }
}

// (c): one thread per (box, axis) with bricks: masks[moff + j] = loop mask | passing mask << 8 of brick b0 + j.
__global__ void co_mask_kernel(const double* __restrict__ c3, const double* __restrict__ s3, int s_stride, long long n,
                               double res, double inv, const Axis* __restrict__ axes, const long long* __restrict__ nb,
                               const long long* __restrict__ moff_incl, unsigned short* __restrict__ masks) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= 3 * n) return;
  const long long cnt = nb[t];
  if (cnt == 0) return;
  const Axis A = axes[t];
  unsigned short* m = masks + (moff_incl[t] - cnt);
  for (int j = 0; j < A.nb; ++j) {
    unsigned occ = 0;
    for (int q = 0; q < 8; ++q) {
      const int key = (A.b0 + j) * 8 + q;
      if (key >= A.oa && key <= A.ob) occ |= 1u << q;
    }
    m[j] = (unsigned short)(occ << 8);
  }
  const long long i = t / 3;
  const int a = (int)(t % 3);
  const double p = c3[3 * i + a], s = s3[(size_t)s_stride * i + a];
  const float bmin = (float)(p - s / 2), bmax = (float)(p + s / 2);
  int cur = -1, k;
  unsigned bits = 0;
  for (double x = bmin; x <= bmax; x += res) {  // (a) counted it: at most 2^17 points
    if (!key_of(inv, (float)x, k)) continue;
    const int j = (k >> 3) - A.b0;
    if (j != cur) {
      if (cur >= 0) m[cur] |= (unsigned short)bits;
      cur = j;
      bits = 0;
    }
    bits |= 1u << (k & 7);
  }
  if (cur >= 0) m[cur] |= (unsigned short)bits;
}

// (d): one warp per (box, brick) item; the grid's warps stride over the items, so any item count up to the call's bound
// runs.  Lane l holds voxels l + 32 w of the brick (w = 0 ... 15): x = l & 7, y = (l >> 3 & 3) | (w & 1) << 2, z = w >> 1.
// An occupied candidate passes the cube test on every axis (and the box's corners are valid); an unknown candidate is
// reached by the loop on every axis.  loop_needed 0 (path mode without unknown as occupied): the unknown flag cannot
// change a result, so only the occupied pass runs.  Every value a lane branches on is read by lane 0 and broadcast, so
// the warp stays converged for its collectives.
__global__ void __launch_bounds__(32 * kWarpsPerBlock) co_voxel_kernel(
    long long total, long long n, const long long* __restrict__ item_incl, const Axis* __restrict__ axes,
    const long long* __restrict__ nb, const long long* __restrict__ moff_incl, const unsigned short* __restrict__ masks,
    const unsigned long long* __restrict__ tab_keys, const int* __restrict__ tab_vals, unsigned tab_mask,
    const unsigned* __restrict__ known, const float* __restrict__ lo, float l_occ, int loop_needed, unsigned* flags,
    const long long* __restrict__ offsets, const int* __restrict__ pid, int unknown_occ, unsigned* best,
    unsigned long long* __restrict__ visited) {
  const int lane = threadIdx.x & 31;
  const long long stride = (long long)gridDim.x * kWarpsPerBlock;
  unsigned long long v = 0;
  for (long long item = (long long)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5); item < total; item += stride) {
    long long box = 0;
    int done = 0;
    if (lane == 0) {
      long long l = 0, h = n - 1;  // the first box whose inclusive item count exceeds item
      while (l < h) {
        const long long mid = (l + h) >> 1;
        if (item_incl[mid] > item) h = mid;
        else l = mid + 1;
      }
      box = l;
      if (pid) done = *(volatile unsigned*)&best[pid[l]] <= (unsigned)(l - offsets[pid[l]]);  // an earlier pose collides
      else done = (*(volatile unsigned*)&flags[l] & kFlagOcc) != 0u;                          // decided: occupied
    }
    box = __shfl_sync(0xffffffffu, box, 0);
    if (__shfl_sync(0xffffffffu, done, 0)) continue;
    const long long path = pid ? pid[box] : -1;
    const unsigned pose = pid ? (unsigned)(box - offsets[path]) : 0u;
    const long long local = item - (item_incl[box] - (long long)nb[3 * box] * nb[3 * box + 1] * nb[3 * box + 2]);
    const Axis X = axes[3 * box], Y = axes[3 * box + 1], Z = axes[3 * box + 2];
    const long long jz = local % Z.nb, jy = (local / Z.nb) % Y.nb, jx = local / ((long long)Z.nb * Y.nb);
    const unsigned mx = masks[moff_incl[3 * box] - X.nb + jx], my = masks[moff_incl[3 * box + 1] - Y.nb + jy],
                   mz = masks[moff_incl[3 * box + 2] - Z.nb + jz];
    const bool corners = X.corners && Y.corners && Z.corners;
    const unsigned ox = corners ? mx >> 8 : 0u, oy = my >> 8, oz = mz >> 8;
    const unsigned lx = loop_needed ? mx & 0xffu : 0u, ly = my & 0xffu, lz = mz & 0xffu;
    if (!(ox && oy && oz) && !(lx && ly && lz)) continue;
    int b = -1;
    if (lane == 0) b = lookup_brick(tab_keys, tab_vals, tab_mask, brick_pack(X.b0 + (int)jx, Y.b0 + (int)jy, Z.b0 + (int)jz));
    b = __shfl_sync(0xffffffffu, b, 0);
    const unsigned kw = (b >= 0 && lane < 16) ? known[(size_t)b * 16 + lane] : 0u;
    const int x = lane & 7, ylo = (lane >> 3) & 3;
    const bool occ_x = (ox >> x) & 1u, loop_x = (lx >> x) & 1u;
    bool f_occ = false, f_unk = false;
#pragma unroll
    for (int w = 0; w < 16; ++w) {
      const unsigned word = __shfl_sync(0xffffffffu, kw, w);
      const int y = ylo | ((w & 1) << 2), z = w >> 1;
      const bool oc = occ_x && ((oy >> y) & 1u) && ((oz >> z) & 1u);
      const bool uc = loop_x && ((ly >> y) & 1u) && ((lz >> z) & 1u);
      if (!(oc || uc)) continue;
      ++v;
      if (!((word >> lane) & 1u)) f_unk |= uc;
      else if (oc && lo[(size_t)b * 512 + w * 32 + lane] >= l_occ) f_occ = true;
    }
    const bool w_occ = __any_sync(0xffffffffu, f_occ), w_unk = __any_sync(0xffffffffu, f_unk);
    if (lane == 0) {
      if (w_occ || w_unk) atomicOr(&flags[box], (w_occ ? kFlagOcc : 0u) | (w_unk ? kFlagUnk : 0u));
      if (pid && (w_occ || (unknown_occ && w_unk))) atomicMin(&best[path], pose);
    }
  }
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  if (lane == 0 && v) atomicAdd(visited, v);
}

// (e): per box its status (box mode), or per path its first collision (path mode: n = n_paths).
__global__ void co_result_kernel(long long n, const signed char* __restrict__ dec, const unsigned* __restrict__ flags,
                                 const unsigned* __restrict__ best, signed char* __restrict__ status,
                                 long long* __restrict__ first) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (best) {
    first[i] = best[i] == kNone ? -1LL : (long long)best[i];
    return;
  }
  const int d = dec[i];
  const unsigned f = flags[i];
  status[i] = (signed char)(d >= 0 ? d : (f & kFlagOcc) ? LS_CELL_OCCUPIED : (f & kFlagUnk) ? LS_CELL_UNKNOWN : LS_CELL_FREE);
}

// Both calls: n boxes (centres c3, sizes s3 with stride s_stride) on the device; path mode when offsets is not NULL.
int collide(Map& m, const Params& P, const double* c3, const double* s3, int s_stride, long long n, const int64_t* offsets,
            int n_paths, int unknown_occ, int8_t* status, int64_t* first, long long* visited, cudaStream_t st,
            uint64_t* launches) {
  const bool paths = offsets != nullptr;
  const long long n_out = paths ? n_paths : n;
  const size_t n3 = (size_t)n * 3;
  size_t off = 0;
  // the readback region first: the keys visited, then the results
  const size_t o_vis = take(off, sizeof(unsigned long long) + (paths ? 8 * (size_t)n_out : (size_t)n_out));
  const size_t o_res = o_vis + sizeof(unsigned long long);
  const size_t o_c = take(off, n3 * sizeof(double)), o_s = take(off, (s_stride ? n3 : 3) * sizeof(double)),
               o_off = take(off, paths ? ((size_t)n_paths + 1) * sizeof(long long) : 0),
               o_ax = take(off, n3 * sizeof(Axis)), o_nb = take(off, n3 * sizeof(long long)),
               o_moff = take(off, n3 * sizeof(long long)), o_items = take(off, (size_t)n * sizeof(long long)),
               o_iinc = take(off, (size_t)n * sizeof(long long)), o_dec = take(off, (size_t)n),
               o_flags = take(off, (size_t)n * sizeof(unsigned)), o_pid = take(off, paths ? (size_t)n * sizeof(int) : 0),
               o_best = take(off, paths ? (size_t)n_paths * sizeof(unsigned) : 0), o_ctr = take(off, sizeof(CallCounters));
  size_t cub_a = 0, cub_b = 0;
  LSO_TRY(cub::DeviceScan::InclusiveSum(nullptr, cub_a, (long long*)nullptr, (long long*)nullptr, (int64_t)n3, st));
  LSO_TRY(cub::DeviceScan::InclusiveSum(nullptr, cub_b, (long long*)nullptr, (long long*)nullptr, (int64_t)n, st));
  const size_t cub_bytes = cub_a > cub_b ? cub_a : cub_b;
  const size_t o_cub = take(off, cub_bytes);
  int rc;
  if ((rc = reserve_staging(m, off, 0, st))) return rc;
  char* q = m.qbuf.get();
  const double* dc = (const double*)(q + o_c);
  const double* ds = (const double*)(q + o_s);
  const long long* doff = paths ? (const long long*)(q + o_off) : nullptr;
  Axis* ax = (Axis*)(q + o_ax);
  long long *nb = (long long*)(q + o_nb), *moff = (long long*)(q + o_moff), *items = (long long*)(q + o_items),
            *iinc = (long long*)(q + o_iinc);
  signed char* dec = (signed char*)(q + o_dec);
  unsigned* flags = (unsigned*)(q + o_flags);
  int* pid = paths ? (int*)(q + o_pid) : nullptr;
  unsigned* best = paths ? (unsigned*)(q + o_best) : nullptr;
  CallCounters* ctr = (CallCounters*)(q + o_ctr);
  unsigned long long* vis = (unsigned long long*)(q + o_vis);
  LSO_TRY(cudaMemcpyAsync(q + o_c, c3, n3 * sizeof(double), cudaMemcpyHostToDevice, st));
  LSO_TRY(cudaMemcpyAsync(q + o_s, s3, (s_stride ? n3 : 3) * sizeof(double), cudaMemcpyHostToDevice, st));
  if (paths) {
    LSO_TRY(cudaMemcpyAsync(q + o_off, offsets, ((size_t)n_paths + 1) * sizeof(long long), cudaMemcpyHostToDevice, st));
    LSO_TRY(cudaMemsetAsync(best, 0xff, (size_t)n_paths * sizeof(unsigned), st));
  }
  LSO_TRY(cudaMemsetAsync(vis, 0, sizeof(unsigned long long), st));
  LSO_TRY(cudaMemsetAsync(ctr, 0, sizeof(CallCounters), st));
  const unsigned tab_mask = (unsigned)m.tab_cap() - 1u;
  co_axis_kernel<<<blocks(3 * n, 256), 256, 0, st>>>(dc, ds, s_stride, n, P.res, P.inv, ax, nb, ctr);
  LSO_LAUNCHED();
  co_box_kernel<<<blocks(n, 256), 256, 0, st>>>(dc, n, P.inv, m.tab_keys.get(), m.tab_vals.get(), tab_mask, m.known.get(),
                                                m.lo.get(), P.l_occ, ax, nb, items, dec, flags, doff, n_paths, unknown_occ,
                                                pid, best, vis, ctr);
  LSO_LAUNCHED();
  size_t bytes = cub_bytes;
  LSO_TRY(cub::DeviceScan::InclusiveSum(q + o_cub, bytes, nb, moff, (int64_t)n3, st));
  bytes = cub_bytes;
  LSO_TRY(cub::DeviceScan::InclusiveSum(q + o_cub, bytes, items, iinc, (int64_t)n, st));
  *launches += 2;
  struct {
    CallCounters c;
    long long masks, total;
  } h{};
  LSO_TRY(cudaMemcpyAsync(&h.c, ctr, sizeof(CallCounters), cudaMemcpyDeviceToHost, st));
  LSO_TRY(cudaMemcpyAsync(&h.masks, moff + n3 - 1, sizeof(long long), cudaMemcpyDeviceToHost, st));
  LSO_TRY(cudaMemcpyAsync(&h.total, iinc + n - 1, sizeof(long long), cudaMemcpyDeviceToHost, st));
  LSO_TRY(cudaStreamSynchronize(st));
  if (h.c.refused || !(h.c.work <= kMaxWork)) return LS_ERR_ARG;
  if (h.total > 0) {
    const size_t keep = off;
    const size_t o_mask = take(off, (size_t)h.masks * sizeof(unsigned short));
    if ((rc = reserve_staging(m, off, keep, st))) return rc;
    q = m.qbuf.get();  // a growth moved the staging: every pointer again
    dc = (const double*)(q + o_c), ds = (const double*)(q + o_s);
    doff = paths ? (const long long*)(q + o_off) : nullptr;
    ax = (Axis*)(q + o_ax), nb = (long long*)(q + o_nb), moff = (long long*)(q + o_moff), iinc = (long long*)(q + o_iinc);
    dec = (signed char*)(q + o_dec), flags = (unsigned*)(q + o_flags);
    pid = paths ? (int*)(q + o_pid) : nullptr, best = paths ? (unsigned*)(q + o_best) : nullptr;
    vis = (unsigned long long*)(q + o_vis);
    unsigned short* masks = (unsigned short*)(q + o_mask);
    co_mask_kernel<<<blocks(3 * n, 256), 256, 0, st>>>(dc, ds, s_stride, n, P.res, P.inv, ax, nb, moff, masks);
    LSO_LAUNCHED();
    const unsigned grid = (unsigned)std::min<long long>((h.total + kWarpsPerBlock - 1) / kWarpsPerBlock, kVoxelBlocks);
    co_voxel_kernel<<<grid, 32 * kWarpsPerBlock, 0, st>>>(
        h.total, n, iinc, ax, nb, moff, masks, m.tab_keys.get(), m.tab_vals.get(), tab_mask, m.known.get(), m.lo.get(),
        P.l_occ, paths ? unknown_occ : 1, flags, doff, pid, unknown_occ, best, vis);
    LSO_LAUNCHED();
  }
  co_result_kernel<<<blocks(n_out, 256), 256, 0, st>>>(n_out, dec, flags, best, (signed char*)(q + o_res),
                                                       (long long*)(q + o_res));
  LSO_LAUNCHED();
  std::vector<char> back(sizeof(unsigned long long) + (paths ? 8 * (size_t)n_out : (size_t)n_out));
  LSO_TRY(cudaMemcpyAsync(back.data(), q + o_vis, back.size(), cudaMemcpyDeviceToHost, st));
  LSO_TRY(cudaStreamSynchronize(st));
  unsigned long long v;
  std::memcpy(&v, back.data(), sizeof v);
  *visited = (long long)v;
  if (paths) std::memcpy(first, back.data() + sizeof v, 8 * (size_t)n_out);
  else std::memcpy(status, back.data() + sizeof v, (size_t)n_out);
  return LS_OK;
}

}  // namespace

int box_status(Map& m, const Params& P, const double* centres3, const double* sizes3, int n, int8_t* status,
               long long* visited, cudaStream_t st, uint64_t* launches) {
  *visited = 0;
  if (n <= 0) return LS_OK;
  return collide(m, P, centres3, sizes3, 3, n, nullptr, 0, 0, status, nullptr, visited, st, launches);
}

int check_paths(Map& m, const Params& P, const double* positions3, const int64_t* offsets, int n_paths,
                const double robot3[3], int unknown_occ, int64_t* first, long long* visited, cudaStream_t st,
                uint64_t* launches) {
  *visited = 0;
  if (n_paths <= 0) return LS_OK;
  const long long poses = offsets[n_paths];
  if (poses == 0) {
    for (int p = 0; p < n_paths; ++p) first[p] = -1;
    return LS_OK;
  }
  return collide(m, P, positions3, robot3, 0, poses, offsets, n_paths, unknown_occ != 0, nullptr, first, visited, st,
                 launches);
}

}  // namespace lso
