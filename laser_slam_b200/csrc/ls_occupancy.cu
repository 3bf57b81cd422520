// Resident occupancy map: laser_to_octomap's insertion loop (reference laser_slam_tools/src/laser_to_octomap.cpp, through
// volumetric_mapping's OctomapManager) as device kernels.  The rules, shared with oracle/occupancy_oracle.cpp, are
// oracle/OCCUPANCY.md.  Per scan:
//   (a) occ_classify_kernel  one thread per point: world-frame point, ray end (cut at the max range), endpoint key; an
//                            in-range point with a valid key enters the per-scan endpoint table with atomicMin of its index
//   (b) occ_cast_kernel      one thread per point that casts (no in-range earlier point has its endpoint key): the DDA over
//                            keys, setting free marks and the occupied mark of the endpoint; bricks are found or inserted in
//                            the brick hash and listed the first time they are marked in the scan
//   (c) occ_update_kernel    one block per touched brick, one thread per voxel: the single log-odds update (occupied wins
//                            over free), known bits set, marks cleared
// Log-odds change only in (c).  When the pool or the hash overflows in (b) the host clears every mark, grows what filled
// and runs (b) again, so a failed insert leaves the known voxels and their values as they were.
//
// Octree export and read, one pipeline each over a format trait (BinaryTree: octomap's writeBinary / readBinary after
// toMaxLikelihood and prune, the .bt payload, rules in oracle/OCTREE.md; FullTree: OcTree::write / readData, the .ot
// payload with every node's float value, DESIGN.md §4b''''''').  Each kernel below is a template over the format, which
// supplies the node record, the merge of 8 children and its subtree totals, a brick's levels, and which nodes the stream
// holds.
// Export, reading the map only:
//   (d) oct_code_kernel      Morton code of each brick key; a CUB radix sort puts the bricks in pre-order at depth 13
//   (e) oct_brick_kernel     one block per brick: its 512 voxels merged in shared memory through levels 15, 14 and 13
//                            (the format's levels), the brick's state, value and subtree totals
//   (f) oct_up_kernel        one block: levels 12 ... 0, each level's sorted list segmented by code >> 3 with a block scan,
//                            the format's merge per parent (the root never collapses), subtree totals summed
//   the root's totals come back once and size the outputs
//   (g) oct_down_kernel      one block: levels 0 ... 12, each inner node's record and its children's offsets (its own +
//                            its record + the earlier siblings' totals); .bt writes occupied leaves' centres, .ot leaf nodes
//   (h) oct_emit_kernel      one block per inner brick: (e)'s levels again, its nodes below depth 13 written at the offset
//                            (g) gave it, so no per-brick staging is kept; one specialisation per format
// A brick without a known voxel (an insert that failed after placing it leaves one) has state 0 and adds nothing.
// Leaf lists (DESIGN.md §4b''''''''''''), over the records of a current .ot build, reading them and the map only; (l1) and
// (l2), templates over the format, also list the .bt build's leaves for the 2D projection (ls_projection.cu):
//   (l1) lv_down_kernel      one block: levels 0 ... 12 as (g), each node's leaf offset; leaves above the bricks written
//   (l2) lv_emit_kernel      one block per inner brick: (e)'s levels again, its leaves placed by a block scan
//   (l3) lv_compact_kernel   after a CUB scan of the region flags: the kept leaves in order, counts per (state, depth)
//   (l4) lv_gather_kernel    after a CUB radix sort by state (or state and depth): centres, tags and height colours
//
// Read (DESIGN.md §4b''''''), replacing the map.  The payload is uploaded once and parsed without a walk, one thread per
// stream record (.bt: inner nodes only; .ot: every node):
//   (r1) rd_excess_kernel + a CUB scan   the excess E_i of each record: stream nodes found but not yet read
//   (r2) rd_end_kernel                   the tree's end (the first E_i = 0) and each block's least excess
//   (r3) rd_parent_kernel                each node's parent (the last earlier record with E <= its own) and slot
//   (r4) rd_node_kernel                  depth and first key (at most 15 / 16 parents up), the depth-13 ancestor, the
//                                        format's checks and counts: nodes, leaves, known voxels and bricks; a CUB scan
//                                        gives each node its first brick, so the bricks are numbered in pre-order with
//                                        no deduplication
//   one readback validates the stream, checks the size line and the brick bound, and sizes the pool
//   (r5) rd_brick_kernel                 each new brick's key and state (uniform, or mixed)
//   the hash is built from those keys beside the old one (replace_map), so a failure up to here leaves the map as it was
//   (r6) rd_fill_kernel                  one block per brick: uniform bricks written whole, mixed ones cleared
//   (r7) rd_leaf_kernel                  the voxels of each leaf at depth 14 ... 16, each written once
#include <algorithm>
#include <cfloat>
#include <climits>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <functional>
#include <utility>
#include <vector>

#include <cub/cub.cuh>
#include <cuda_runtime.h>

#include "../../include/ls_b200.h"
#include "ls_occupancy.cuh"

namespace lso {
namespace {

constexpr unsigned long long kEmpty = ~0ull;
constexpr int kPending = -1, kFull = -2;
constexpr long long kMaxEditAxis = 1LL << 17;    // loop points per box axis (the key space has 2^16 per axis)
constexpr long long kMaxEditBricks = 1LL << 29;  // bricks of an edit plus those in use (the read's bound)
constexpr int kOverflowTable = 1, kOverflowPool = 2;

struct Xform16 {
  float T[16];
};

// ls_math.cuh's xform_point order (that header defines host functions and is included by ls_api.cu only)
__device__ __forceinline__ void xform3(const float* T, float x, float y, float z, float& ox, float& oy, float& oz) {
  float a, b, c, s;
  a = T[0] * x; b = T[4] * y; c = T[8] * z; s = a + b; s = s + c; ox = s + T[12];
  a = T[1] * x; b = T[5] * y; c = T[9] * z; s = a + b; s = s + c; oy = s + T[13];
  a = T[2] * x; b = T[6] * y; c = T[10] * z; s = a + b; s = s + c; oz = s + T[14];
}

// the views of Map the kernels need
struct Dev {
  unsigned long long* tab_keys;
  int* tab_vals;
  unsigned tab_mask;
  int pool_cap;
  float* lo;
  unsigned *known, *mfree, *mocc;
  unsigned long long* bkey;
  unsigned* touched;
  int* tlist;
};

Dev dev_of(const Map& m) {
  return Dev{m.tab_keys.get(), m.tab_vals.get(), (unsigned)m.tab_cap() - 1u, m.pool_cap(), m.lo.get(), m.known.get(),
             m.mfree.get(), m.mocc.get(), m.bkey.get(), m.touched.get(), m.tlist.get()};
}

__device__ __forceinline__ bool key3(double inv, const float p[3], int k[3]) {
  return key_of(inv, p[0], k[0]) && key_of(inv, p[1], k[1]) && key_of(inv, p[2], k[2]);
}
// |v|: squares and sums in float, the root in double
__device__ __forceinline__ double norm3(const float v[3]) {
  const float a = v[0] * v[0], b = v[1] * v[1], c = v[2] * v[2];
  float s = a + b;
  s = s + c;
  return sqrt((double)s);
}

// Pool index of brick `bk`, inserted if absent.  The inserting thread takes the next pool index and publishes it; a
// thread that finds the key waits for that.  kFull when the pool or the probe bound is exhausted (flagged in *overflow).
__device__ int brick_of(const Dev& D, Counters* cnt, unsigned long long bk) {
  unsigned h = hash64(bk) & D.tab_mask;
  for (int p = 0; p < kMaxProbe; ++p, h = (h + 1u) & D.tab_mask) {
    unsigned long long k = *(volatile unsigned long long*)&D.tab_keys[h];
    if (k == kEmpty) {
      k = atomicCAS(&D.tab_keys[h], kEmpty, bk);
      if (k == kEmpty) {
        int idx = atomicAdd(&cnt->pool_n, 1);
        if (idx >= D.pool_cap) {
          idx = kFull;
          atomicOr(&cnt->overflow, kOverflowPool);
        } else {
          D.bkey[idx] = bk;
        }
        __threadfence();
        atomicExch(&D.tab_vals[h], idx);
        return idx;
      }
    }
    if (k == bk) {
      int v;
      while ((v = *(volatile int*)&D.tab_vals[h]) == kPending) {
      }
      return v;
    }
  }
  atomicOr(&cnt->overflow, kOverflowTable);
  return kFull;
}

struct Cursor {
  unsigned long long bk = kEmpty;
  int b = -1;
};

// Set the free or occupied mark of voxel k; false when its brick could not be placed.
__device__ __forceinline__ bool mark(const Dev& D, Counters* cnt, Cursor& cur, const int k[3], bool occ) {
  const unsigned long long bk = brick_key(k);
  if (bk != cur.bk) {
    const int b = brick_of(D, cnt, bk);
    if (b < 0) return false;
    cur.bk = bk;
    cur.b = b;
    if (D.touched[b] == 0u && atomicExch(&D.touched[b], 1u) == 0u) D.tlist[atomicAdd(&cnt->n_touched, 1)] = b;
  }
  const int local = local_of(k);
  unsigned* w = (occ ? D.mocc : D.mfree) + (size_t)cur.b * 16 + (local >> 5);
  const unsigned bit = 1u << (local & 31);
  if (!(*w & bit)) atomicOr(w, bit);  // near the sensor thousands of rays share a voxel: read before the atomic
  return true;
}

// The Amanatides-Woo setup both of octomap's DDAs share, from key k at o along dir: step, tMax and tDelta per axis.  The
// border's half step is rounded to float in computeRayKeys (kFloatHalfStep) and kept in double in castRay.
template <bool kFloatHalfStep>
__device__ __forceinline__ void dda_setup(const int k[3], const float o[3], const float dir[3], double res, int step[3],
                                          double tmax[3], double tdelta[3]) {
  for (int i = 0; i < 3; ++i) {
    step[i] = dir[i] > 0.0f ? 1 : (dir[i] < 0.0f ? -1 : 0);
    if (step[i] != 0) {
      double border = centre_d(k[i], res);
      const double half = (double)step[i] * res * 0.5;
      border += kFloatHalfStep ? (double)(float)half : half;
      tmax[i] = (border - (double)o[i]) / (double)dir[i];
      tdelta[i] = res / (double)fabsf(dir[i]);
    } else {
      tmax[i] = DBL_MAX;
      tdelta[i] = DBL_MAX;
    }
  }
}

// The axis of the next step: the smallest tMax, ties to the later axis.
__device__ __forceinline__ int next_axis(const double tmax[3]) {
  if (tmax[0] < tmax[1]) return tmax[0] < tmax[2] ? 0 : 2;
  return tmax[1] < tmax[2] ? 1 : 2;
}

// octomap's computeRayKeys from o to e: visit(k) for the origin key and every key stepped into before the end key, in
// order.  False as soon as a visit returns false.  The insert marks each key free; the line queries read its state.
template <class Visit>
__device__ __forceinline__ bool walk(const Params& P, const float o[3], const float e[3], Visit&& visit) {
  int ko[3], ke[3];
  if (!key3(P.inv, o, ko) || !key3(P.inv, e, ke)) return true;
  if (ko[0] == ke[0] && ko[1] == ke[1] && ko[2] == ke[2]) return true;
  if (!visit(ko)) return false;
  float dir[3] = {e[0] - o[0], e[1] - o[1], e[2] - o[2]};
  const float length = (float)norm3(dir);
  for (int i = 0; i < 3; ++i) dir[i] = dir[i] / length;
  int step[3], k[3] = {ko[0], ko[1], ko[2]};
  double tmax[3], tdelta[3];
  dda_setup<true>(k, o, dir, P.res, step, tmax, tdelta);
  for (;;) {
    const int dim = next_axis(tmax);
    k[dim] += step[dim];
    tmax[dim] += tdelta[dim];
    if (k[0] == ke[0] && k[1] == ke[1] && k[2] == ke[2]) break;
    if (k[dim] < 0 || k[dim] > 65535) break;
    const double dist = fmin(fmin(tmax[0], tmax[1]), tmax[2]);
    if (dist > (double)length) break;
    if (!visit(k)) return false;
  }
  return true;
}

// (a) cls: 0 = no ray (non-finite), 1 = in range (free cells to the point, occupied endpoint), 2 = cut at the max range
__global__ void occ_classify_kernel(const float4* __restrict__ in, int n, Xform16 T, int identity, Params P,
                                    float4* __restrict__ ends, unsigned long long* __restrict__ pkey, int* __restrict__ cls,
                                    unsigned long long* ep_keys, int* ep_min, unsigned ep_mask) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float4 q = in[i];
  float p[3] = {q.x, q.y, q.z};
  if (!identity) xform3(T.T, q.x, q.y, q.z, p[0], p[1], p[2]);
  if (!isfinite(p[0]) || !isfinite(p[1]) || !isfinite(p[2])) {
    cls[i] = 0;
    pkey[i] = kEmpty;
    return;
  }
  int k[3];
  const unsigned long long key = key3(P.inv, p, k) ? pack(k[0], k[1], k[2]) : kEmpty;
  const float o[3] = {T.T[12], T.T[13], T.T[14]};
  const float d[3] = {p[0] - o[0], p[1] - o[1], p[2] - o[2]};
  const double len = norm3(d);
  float4 e = make_float4(p[0], p[1], p[2], 1.0f);
  int c = 1;
  if (!(P.max_range < 0.0 || len <= P.max_range)) {
    c = 2;
    const float fl = (float)len, fr = (float)P.max_range;
    float u, w;
    u = d[0] / fl; w = u * fr; e.x = o[0] + w;
    u = d[1] / fl; w = u * fr; e.y = o[1] + w;
    u = d[2] / fl; w = u * fr; e.z = o[2] + w;
  } else if (key != kEmpty) {
    unsigned h = hash64(key) & ep_mask;
    for (;;) {  // the table has twice the points' slots: it cannot fill
      unsigned long long cur = *(volatile unsigned long long*)&ep_keys[h];
      if (cur == kEmpty) {
        cur = atomicCAS(&ep_keys[h], kEmpty, key);
        if (cur == kEmpty) cur = key;
      }
      if (cur == key) {
        atomicMin(&ep_min[h], i);
        break;
      }
      h = (h + 1u) & ep_mask;
    }
  }
  ends[i] = e;
  pkey[i] = key;
  cls[i] = c;
}

// (b) one thread per point; the block size is a multiple of 32 so every lane of a warp takes part in the counts
__global__ void occ_cast_kernel(int n, Params P, float ox, float oy, float oz, const float4* __restrict__ ends,
                                const unsigned long long* __restrict__ pkey, const int* __restrict__ cls,
                                const unsigned long long* __restrict__ ep_keys, const int* __restrict__ ep_min, unsigned ep_mask,
                                Dev D, Counters* cnt) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const bool active = i < n;
  const int c = active ? cls[i] : 0;
  const unsigned long long key = active ? pkey[i] : kEmpty;
  bool cast = c != 0;
  if (cast && key != kEmpty) {  // already checked: an earlier in-range point has this endpoint key
    unsigned h = hash64(key) & ep_mask;
    for (;;) {
      const unsigned long long k = ep_keys[h];
      if (k == key) {
        if (ep_min[h] < i) cast = false;
        break;
      }
      if (k == kEmpty) break;
      h = (h + 1u) & ep_mask;
    }
  }
  const unsigned b_cast = __ballot_sync(0xffffffffu, cast), b_skip = __ballot_sync(0xffffffffu, active && !cast);
  if ((threadIdx.x & 31) == 0) {
    if (b_cast) atomicAdd(&cnt->rays_cast, __popc(b_cast));
    if (b_skip) atomicAdd(&cnt->rays_skipped, __popc(b_skip));
  }
  if (!cast || *(volatile int*)&cnt->overflow) return;
  const float4 e4 = ends[i];
  const float o[3] = {ox, oy, oz}, e[3] = {e4.x, e4.y, e4.z};
  Cursor cur;
  if (!walk(P, o, e, [&](const int* k) { return mark(D, cnt, cur, k, false); })) return;
  if (c == 1 && key != kEmpty) {
    const int k[3] = {(int)(key & 0xffff), (int)((key >> 16) & 0xffff), (int)((key >> 32) & 0xffff)};
    mark(D, cnt, cur, k, true);
  }
}

// (c) one block of 512 threads per touched brick; warp w owns mark / known word w
__global__ void occ_update_kernel(Dev D, Params P, Counters* cnt) {
  const int b = D.tlist[blockIdx.x];
  const int t = threadIdx.x, lane = t & 31;
  const size_t wi = (size_t)b * 16 + (t >> 5);
  const unsigned of = D.mfree[wi], oo = D.mocc[wi], kn = D.known[wi];
  const bool occ = (oo >> lane) & 1u, fr = !occ && ((of >> lane) & 1u);
  if (occ || fr) {
    float* v = D.lo + (size_t)b * 512 + t;
    float x = *v + (occ ? P.l_hit : P.l_miss);
    if (x < P.l_min) x = P.l_min;
    if (x > P.l_max) x = P.l_max;
    *v = x;
  }
  __syncwarp();
  if (lane == 0) {
    const unsigned upd = oo | of;
    D.known[wi] = kn | upd;
    D.mfree[wi] = 0u;
    D.mocc[wi] = 0u;
    const unsigned no = __popc(oo), nf = __popc(of & ~oo), nk = __popc(upd & ~kn);
    if (no) atomicAdd(&cnt->occ_upd, (unsigned long long)no);
    if (nf) atomicAdd(&cnt->free_upd, (unsigned long long)nf);
    if (nk) atomicAdd(&cnt->new_known, (unsigned long long)nk);
  }
  if (t == 0) D.touched[b] = 0u;
}

__global__ void occ_rehash_kernel(const unsigned long long* __restrict__ bkey, int n, unsigned long long* keys, int* vals,
                                  unsigned mask, Counters* cnt) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= n) return;
  const unsigned long long k = bkey[b];
  unsigned h = hash64(k) & mask;
  for (int p = 0; p < kMaxProbe; ++p, h = (h + 1u) & mask) {
    if (atomicCAS(&keys[h], kEmpty, k) == kEmpty) {
      vals[h] = b;
      return;
    }
  }
  atomicOr(&cnt->overflow, kOverflowTable);
}

// Known (which == LS_OCC_KNOWN) or occupied voxels of the first nvox pool voxels: counted into cnt->n_out and, with keys
// != NULL, written unordered as (packed key, log-odds bits).  Warp-aggregated slots.
__global__ void occ_select_kernel(Dev D, Params P, int which, long long nvox, unsigned long long* __restrict__ keys,
                                  unsigned* __restrict__ vals, Counters* cnt) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  const int lane = threadIdx.x & 31;
  for (long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x; v - lane < nvox; v += stride) {
    bool sel = false;
    float x = 0.0f;
    if (v < nvox) {
      const long long b = v >> 9;
      const int t = (int)(v & 511);
      if ((D.known[b * 16 + (t >> 5)] >> (t & 31)) & 1u) {
        x = D.lo[v];
        sel = which == LS_OCC_KNOWN || x >= P.l_occ;
      }
    }
    const unsigned bal = __ballot_sync(0xffffffffu, sel);
    if (!bal) continue;
    unsigned long long base = 0;
    if (lane == 0) base = atomicAdd(&cnt->n_out, (unsigned long long)__popc(bal));
    base = __shfl_sync(0xffffffffu, base, 0);
    if (sel && keys) {
      const unsigned long long pos = base + __popc(bal & ((1u << lane) - 1u));
      const unsigned long long bk = D.bkey[v >> 9];
      const int t = (int)(v & 511);
      int k[3];
      voxel_keys(bk, t, k);
      keys[pos] = pack(k[0], k[1], k[2]);
      vals[pos] = __float_as_uint(x);
    }
  }
}

__global__ void occ_centres_kernel(const unsigned long long* __restrict__ keys, long long n, double res, float4* __restrict__ out) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const unsigned long long k = keys[i];
    float c[3];
    for (int a = 0; a < 3; ++a) c[a] = centre_of((int)((k >> (16 * a)) & 0xffff), res);
    out[i] = make_float4(c[0], c[1], c[2], 1.0f);
  }
}

// ---- queries (volumetric_mapping's WorldBase and octomap's castRay; rules in oracle/QUERIES.md) -------------------------
// They read tab_keys / tab_vals, the known bits and the log-odds only; no insert runs during a query.
constexpr unsigned kNanBits = 0x7fc00000u;  // the NaN of an unknown cell's log-odds and an invalid ray's end

__device__ __forceinline__ int find_brick(const Dev& D, unsigned long long bk) {
  return lookup_brick(D.tab_keys, D.tab_vals, D.tab_mask, bk);
}

// State of voxel k (LS_CELL_*, voxel_state), the brick of the last lookup cached in cur.  *v: the log-odds of a known voxel.
__device__ __forceinline__ int state_of(const Dev& D, const Params& P, Cursor& cur, const int k[3], float* v) {
  const unsigned long long bk = brick_key(k);
  if (bk != cur.bk) {
    cur.bk = bk;
    cur.b = find_brick(D, bk);
  }
  if (cur.b < 0) return LS_CELL_UNKNOWN;
  return voxel_state(D.known, D.lo, P.l_occ, cur.b, local_of(k), v);
}

// Every lane of the warp calls it: the warp's keys_visited into cnt->n_out.
__device__ __forceinline__ void add_visited(Counters* cnt, unsigned long long v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0 && v) atomicAdd(&cnt->n_out, v);
}

// getCellStatusPoint / getCellProbabilityPoint: one thread per point
__global__ void occ_cell_kernel(const double* __restrict__ pts3, int n, Dev D, Params P, signed char* __restrict__ status,
                                float* __restrict__ log_odds, Counters* cnt) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  unsigned long long visited = 0;
  if (i < n) {
    int k[3];
    int s = LS_CELL_UNKNOWN;
    float v = __uint_as_float(kNanBits);
    if (key_of(P.inv, pts3[3 * (size_t)i], k[0]) && key_of(P.inv, pts3[3 * (size_t)i + 1], k[1]) &&
        key_of(P.inv, pts3[3 * (size_t)i + 2], k[2])) {  // octomap's search(double x, double y, double z)
      Cursor cur;
      ++visited;
      s = state_of(D, P, cur, k, &v);
      if (s == LS_CELL_UNKNOWN) v = __uint_as_float(kNanBits);
    }
    status[i] = (signed char)s;
    log_odds[i] = v;
  }
  add_visited(cnt, visited);
}

// getLineStatus / getVisibility over computeRayKeys(s, e): the state of the first occupied key, or of the first unknown
// key when stop_unknown, else free; *first its packed key (all ones when free).  cut(visited) ends the walk early (result
// -1): the bounding-box pass drops a line once a lower line of its segment has failed.
template <class Cut>
__device__ __forceinline__ int line_status(const Dev& D, const Params& P, const float s[3], const float e[3], bool stop_unknown,
                                           unsigned long long* first, unsigned long long& visited, Cut&& cut) {
  Cursor cur;
  int st = LS_CELL_FREE;
  unsigned long long fk = kEmpty;
  walk(P, s, e, [&](const int* k) {
    if (cut(visited)) {
      st = -1;
      return false;
    }
    ++visited;
    const int x = state_of(D, P, cur, k, nullptr);
    if (x == LS_CELL_OCCUPIED || (x == LS_CELL_UNKNOWN && stop_unknown)) {
      st = x;
      fk = pack(k[0], k[1], k[2]);
      return false;
    }
    return true;
  });
  *first = fk;
  return st;
}

// The float ends of line `l` of a segment: each coordinate cast to float once, after the box offset is added in double
// (kBox).  offs holds the box loop's x values, then its y values, then its z values; line l = (ix * ny + iy) * nz + iz.
template <bool kBox>
__device__ __forceinline__ void line_ends(const double* s3, const double* e3, int seg, const double* offs, int l, int nx, int ny,
                                          int nz, float s[3], float e[3]) {
  double off[3] = {0.0, 0.0, 0.0};
  if (kBox) off[0] = offs[l / (ny * nz)], off[1] = offs[nx + (l / nz) % ny], off[2] = offs[nx + ny + l % nz];
  for (int a = 0; a < 3; ++a) {
    s[a] = kBox ? (float)(s3[3 * (size_t)seg + a] + off[a]) : (float)s3[3 * (size_t)seg + a];
    e[a] = kBox ? (float)(e3[3 * (size_t)seg + a] + off[a]) : (float)e3[3 * (size_t)seg + a];
  }
}

// Plain lines (kBox false): one thread per segment, the result written.  Bounding boxes (kBox true): one thread per
// (segment, line); a failing line raises best[seg] to ~line with atomicMax, so best ends at the lowest failing line
// whatever the scheduling, and a line at or above the current lowest stops (checked every 16 keys).
template <bool kBox>
__global__ void occ_line_kernel(const double* __restrict__ s3, const double* __restrict__ e3, long long items, int lines,
                                const double* __restrict__ offs, int nx, int ny, int nz, int stop_unknown, Dev D, Params P,
                                signed char* __restrict__ status, unsigned long long* __restrict__ first, unsigned* best,
                                Counters* cnt) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  unsigned long long visited = 0;
  if (i < items) {
    const int seg = kBox ? (int)(i / lines) : (int)i;
    const int l = kBox ? (int)(i % lines) : 0;
    const unsigned mine = 0xffffffffu - (unsigned)l;
    if (!kBox || *(volatile unsigned*)&best[seg] < mine) {
      float s[3], e[3];
      line_ends<kBox>(s3, e3, seg, offs, l, nx, ny, nz, s, e);
      unsigned long long fk;
      const int st = line_status(D, P, s, e, stop_unknown != 0, &fk, visited, [&](unsigned long long v) {
        return kBox && (v & 15) == 15 && *(volatile unsigned*)&best[seg] >= mine;
      });
      if (!kBox) {
        status[seg] = (signed char)st;
        first[seg] = fk;
      } else if (st > 0) {
        atomicMax(&best[seg], mine);
      }
    }
  }
  add_visited(cnt, visited);
}

// The bounding box's result per segment: the lowest failing line walked again for its status and key, or free.
__global__ void occ_box_result_kernel(const double* __restrict__ s3, const double* __restrict__ e3, int n, int lines,
                                      const double* __restrict__ offs, int nx, int ny, int nz, int stop_unknown, Dev D, Params P,
                                      const unsigned* __restrict__ best, signed char* __restrict__ status,
                                      unsigned long long* __restrict__ first, Counters* cnt) {
  const int seg = blockIdx.x * blockDim.x + threadIdx.x;
  unsigned long long visited = 0;
  if (seg < n) {
    const unsigned b = best[seg];
    int st = LS_CELL_FREE;
    unsigned long long fk = kEmpty;
    if (b != 0u) {
      float s[3], e[3];
      line_ends<true>(s3, e3, seg, offs, (int)(0xffffffffu - b), nx, ny, nz, s, e);
      st = line_status(D, P, s, e, stop_unknown != 0, &fk, visited, [](unsigned long long) { return false; });
    }
    status[seg] = (signed char)st;
    first[seg] = fk;
  }
  add_visited(cnt, visited);
}

// octomap's castRay(origin, direction, end, ignore_unknown, max_range): the result code (LS_RAY_*), end[] the centre of
// the voxel it names (left alone for LS_RAY_INVALID).
__device__ __forceinline__ int cast_ray(const Dev& D, const Params& P, const float o[3], const float dir_in[3], bool ignore_unknown,
                                        double max_range, float end[3], unsigned long long& visited) {
  int k[3];
  if (!key3(P.inv, o, k)) return LS_RAY_INVALID;
  Cursor cur;
  ++visited;
  const int s0 = state_of(D, P, cur, k, nullptr);
  if (s0 == LS_CELL_OCCUPIED || (s0 == LS_CELL_UNKNOWN && !ignore_unknown)) {
    for (int a = 0; a < 3; ++a) end[a] = centre_of(k[a], P.res);
    return s0 == LS_CELL_OCCUPIED ? LS_RAY_HIT : LS_RAY_UNKNOWN;
  }
  float dir[3] = {dir_in[0], dir_in[1], dir_in[2]};
  const double len = norm3(dir);  // Vector3::normalize: divided by the float length only when it is > 0
  if (len > 0.0) {
    const float fl = (float)len;
    for (int a = 0; a < 3; ++a) dir[a] = dir[a] / fl;
  }
  int step[3];
  double tmax[3], tdelta[3];
  dda_setup<false>(k, o, dir, P.res, step, tmax, tdelta);
  if (step[0] == 0 && step[1] == 0 && step[2] == 0) return LS_RAY_INVALID;
  const bool range = max_range > 0.0;
  const double range_sq = max_range * max_range;
  for (;;) {
    const int dim = next_axis(tmax);
    if ((step[dim] < 0 && k[dim] == 0) || (step[dim] > 0 && k[dim] == 65535)) {
      for (int a = 0; a < 3; ++a) end[a] = centre_of(k[a], P.res);
      return LS_RAY_KEY_BOUND;
    }
    k[dim] += step[dim];
    tmax[dim] += tdelta[dim];
    for (int a = 0; a < 3; ++a) end[a] = centre_of(k[a], P.res);
    if (range) {
      double d = 0.0;
      for (int a = 0; a < 3; ++a) {
        const float x = end[a] - o[a];
        d += (double)(x * x);
      }
      if (d > range_sq) return LS_RAY_MAX_RANGE;
    }
    ++visited;
    const int s = state_of(D, P, cur, k, nullptr);
    if (s == LS_CELL_OCCUPIED) return LS_RAY_HIT;
    if (s == LS_CELL_UNKNOWN && !ignore_unknown) return LS_RAY_UNKNOWN;
  }
}

// one thread per ray
__global__ void occ_ray_kernel(const float* __restrict__ o3, const float* __restrict__ d3, int n, int ignore_unknown,
                               double max_range, Dev D, Params P, signed char* __restrict__ result, float* __restrict__ ends3,
                               Counters* cnt) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  unsigned long long visited = 0;
  if (i < n) {
    const float o[3] = {o3[3 * (size_t)i], o3[3 * (size_t)i + 1], o3[3 * (size_t)i + 2]};
    const float d[3] = {d3[3 * (size_t)i], d3[3 * (size_t)i + 1], d3[3 * (size_t)i + 2]};
    const float nan = __uint_as_float(kNanBits);
    float e[3] = {nan, nan, nan};
    const int r = cast_ray(D, P, o, d, ignore_unknown != 0, max_range, e, visited);
    if (r == LS_RAY_INVALID) e[0] = e[1] = e[2] = nan;
    result[i] = (signed char)r;
    for (int a = 0; a < 3; ++a) ends3[3 * (size_t)i + a] = e[a];
  }
  add_visited(cnt, visited);
}

// ---- octree export and read ------------------------------------------------------------------------------------------
constexpr int kTreeThreads = 1024;  // (f) and (g)
constexpr int kBrickDepth = 13;

// .bt node states: 0 no known voxel below, 1 free leaf, 2 occupied leaf, 3 inner -- also the bit pair of the payload.
static_assert(LS_CELL_FREE == 0 && LS_CELL_OCCUPIED == 1 && LS_CELL_UNKNOWN == 2, "a voxel's .bt state is (LS_CELL_* + 1) % 3");
// octomap's isNodeCollapsible after toMaxLikelihood: all 8 children exist, are leaves and have one state.
__device__ __forceinline__ int parent_state(int n_free, int n_occ, int n_any, bool may_prune) {
  if (may_prune && n_free == 8) return 1;
  if (may_prune && n_occ == 8) return 2;
  return n_any ? 3 : 0;
}

__device__ __forceinline__ unsigned long long spread3(unsigned v) {  // bit j to bit 3j, 13 bits
  unsigned long long x = 0;
  for (int j = 0; j < 13; ++j) x |= (unsigned long long)((v >> j) & 1u) << (3 * j);
  return x;
}
__device__ __forceinline__ int squeeze3(unsigned long long x) {  // bit 3j to bit j
  int v = 0;
  for (int j = 0; j < 13; ++j) v |= (int)((x >> (3 * j)) & 1ull) << j;
  return v;
}

// Morton index t within a brick (x, y, z bits of key bit 2, then 1, then 0) -> pool-local index x | y << 3 | z << 6
__device__ __forceinline__ int morton_local(int t) {
  const int x = (t & 1) | ((t >> 2) & 2) | ((t >> 4) & 4);
  const int y = ((t >> 1) & 1) | ((t >> 3) & 2) | ((t >> 5) & 4);
  const int z = ((t >> 2) & 1) | ((t >> 4) & 2) | ((t >> 6) & 4);
  return x | (y << 3) | (z << 6);
}

__device__ __forceinline__ int mask8(const unsigned char* s) {
  int m = 0;
  for (int i = 0; i < 8; ++i) m |= (int)s[i] << (2 * i);
  return m;
}

// octomap's keyToCoord(key, depth) of the node whose first voxel key is k0, s = 16 - depth
__device__ __forceinline__ float leaf_coord(int k0, int s, double res) { return (float)leaf_centre_d(k0, s, res); }

__device__ __forceinline__ void put_leaf(float4* cen, unsigned char* dep, unsigned long long i, int kx, int ky, int kz,
                                         int depth, double res) {
  const int s = 16 - depth;
  cen[i] = make_float4(leaf_coord(kx, s, res), leaf_coord(ky, s, res), leaf_coord(kz, s, res), 1.0f);
  dep[i] = (unsigned char)depth;
}

// Node records (Octree): bricks first, then each upper level.  tot: the subtree totals the format keeps, in its order.
struct Nodes {
  unsigned long long* code;
  int *pool, *first, *end;
  unsigned char* st;
  unsigned* val;  // FullTree only
  unsigned long long *tot[3], *off, *loff;
};

// ---- the two payloads ------------------------------------------------------------------------------------------------
// The export and the read below are written once over a format: BinaryTree (octomap's writeBinary / readBinary, the .bt
// payload; DESIGN.md §4b'''' and §4b'''''') or FullTree (OcTree::write / readData, the .ot payload; §4b''''''').  A
// format holds only what differs: the node record, the merge of 8 children and its totals, which nodes the stream holds
// and what a leaf writes into the map.
constexpr int kReadThreads = 256;
constexpr long long kMaxReadBricks = 1LL << 29;  // a hash of at most 2^30 slots at load <= 1/2
constexpr long long kMaxReadPairs = 1LL << 30;
constexpr int kBadDepth = 1, kBadValue = 2;

// The node whose bricks hold brick b: the last j < end with boff[j] <= b (a node without bricks has the next one's boff).
__device__ __forceinline__ int brick_owner(const long long* __restrict__ boff, int end, long long b) {
  int lo = 0, hi = end - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (boff[mid] <= b) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// The voxels [x0, x0 + side) x [y0, ...) x [z0, ...) of pool brick b hold v and become known.
__device__ __forceinline__ void fill_cube(const Dev& D, size_t b, int x0, int y0, int z0, int side, float v) {
  for (int z = z0; z < z0 + side; ++z)
    for (int y = y0; y < y0 + side; ++y) {
      unsigned bitsw = 0;
      const int row = (y << 3) | (z << 6);  // side <= 4 voxels of one row share a known word
      for (int x = x0; x < x0 + side; ++x) {
        D.lo[b * 512 + row + x] = v;
        bitsw |= 1u << ((row + x) & 31);
      }
      atomicOr(&D.known[b * 16 + (row >> 5)], bitsw);
    }
}

// .bt: node states as parent_state's.  Only inner nodes are in the stream, 2 bytes each (the bit pairs of their 8 children).  Totals: nodes, occupied leaves,
// payload bytes.
struct BinaryTree {
  static constexpr int kNodeBytes = 2, kTotals = 3;
  static constexpr bool kValued = false;
  static constexpr int kMaxDepth = 15;             // of a stream node
  static constexpr int kMaxExcess = 8 + 7 * 14;    // the largest excess of a tree whose inner nodes lie at depth <= 15
  static constexpr const char* kTooMany = "more than 2^30 inner nodes";
  static constexpr bool kCentres = true;  // (g) and (h) write the occupied leaves' centres and depths
  static long long payload_bytes(const unsigned long long* tot) { return (long long)tot[2]; }

  struct Merge {
    int nf = 0, no = 0, na = 0;
    __device__ __forceinline__ void add(int s, unsigned) { nf += s == 1, no += s == 2, na += s != 0; }
    __device__ __forceinline__ int state(bool may_prune, unsigned& v) const {
      v = 0;
      return parent_state(nf, no, na, may_prune);
    }
  };
  // (e) a brick's levels 16 ... 13 in shared memory, one block of 512 threads: thread t reads the voxel of Morton index t,
  // then levels 15, 14 and 13 merge their 8 children each
  struct Levels {
    unsigned char s16[512], s15[64], s14[8];
    int n15[64], l15[64], n14[8], l14[8], b14[8];
    int st, nodes, bytes, leaves;  // the depth-13 node
  };
  __device__ static void levels(const unsigned* __restrict__ known, const float* __restrict__ lo, int b, float l_occ,
                                Levels& T) {
    const int t = threadIdx.x;
    const int v = morton_local(t);
    const int s = voxel_state(known, lo, l_occ, b, v, nullptr);
    T.s16[t] = (unsigned char)((s + 1) % 3);  // LS_CELL_* (free 0, occupied 1, unknown 2) as the .bt state
    __syncthreads();
    if (t < 64) {
      int nf = 0, no = 0, na = 0;
      for (int i = 0; i < 8; ++i) {
        const int c = T.s16[8 * t + i];
        nf += c == 1, no += c == 2, na += c != 0;
      }
      const int st = parent_state(nf, no, na, true);
      T.s15[t] = (unsigned char)st;
      T.n15[t] = st == 3 ? 1 + na : st != 0;
      T.l15[t] = st == 3 ? no : st == 2;
    }
    __syncthreads();
    if (t < 8) {
      int nf = 0, no = 0, na = 0, n = 0, l = 0, by = 0;
      for (int i = 0; i < 8; ++i) {
        const int c = T.s15[8 * t + i];
        nf += c == 1, no += c == 2, na += c != 0;
        n += T.n15[8 * t + i], l += T.l15[8 * t + i], by += c == 3 ? 2 : 0;
      }
      const int st = parent_state(nf, no, na, true);
      T.s14[t] = (unsigned char)st;
      T.n14[t] = st == 3 ? 1 + n : st != 0;
      T.l14[t] = st == 3 ? l : st == 2;
      T.b14[t] = st == 3 ? 2 + by : 0;
    }
    __syncthreads();
    if (t == 0) {
      int nf = 0, no = 0, na = 0, n = 0, l = 0, by = 0;
      for (int i = 0; i < 8; ++i) {
        const int c = T.s14[i];
        nf += c == 1, no += c == 2, na += c != 0;
        n += T.n14[i], l += T.l14[i], by += T.b14[i];
      }
      const int st = parent_state(nf, no, na, true);
      T.st = st;
      T.nodes = st == 3 ? 1 + n : st != 0;
      T.leaves = st == 3 ? l : st == 2;
      T.bytes = st == 3 ? 2 + by : 0;
    }
    __syncthreads();
  }
  __device__ __forceinline__ static void record(const Levels& T, const Nodes& N, int r) {
    N.st[r] = (unsigned char)T.st;
    N.tot[0][r] = (unsigned long long)T.nodes;
    N.tot[1][r] = (unsigned long long)T.leaves;
    N.tot[2][r] = (unsigned long long)T.bytes;
  }
  // c: the children's totals summed, then the node's
  template <class T>
  __device__ __forceinline__ static void totals(int s, T* c) {
    c[0] = s == 3 ? c[0] + 1 : (T)(s != 0);
    c[1] = s == 3 ? c[1] : (T)(s == 2);
    c[2] = s == 3 ? c[2] + 2 : (T)0;
  }
  __device__ __forceinline__ static int child_bits(int s, int slot) { return s << (2 * slot); }
  __device__ __forceinline__ static void put_inner(unsigned char* p, const Nodes&, int, int mask) {
    p[0] = (unsigned char)(mask & 0xff), p[1] = (unsigned char)(mask >> 8);
  }
  // (g) child c of an inner node at depth d - 1 takes its offsets; an occupied leaf writes its centre
  __device__ __forceinline__ static void place(const Nodes& N, int c, int d, unsigned long long& o, unsigned long long& l,
                                               double res, unsigned char*, float4* cen, unsigned char* dep) {
    N.off[c] = o, N.loff[c] = l;
    if (N.st[c] == 2) {
      const unsigned long long k = N.code[c];
      const int sh = 16 - d;
      put_leaf(cen, dep, l, squeeze3(k) << sh, squeeze3(k >> 1) << sh, squeeze3(k >> 2) << sh, d, res);
    }
    o += N.tot[2][c], l += N.tot[1][c];
  }
  // The leaf walk (l1, l2): a leaf record's value is its state (1 free, 2 occupied); a subtree's leaves are its nodes less its
  // inner nodes (2 payload bytes each).
  __device__ __forceinline__ static bool walk_leaf(const Nodes& N, int c, unsigned& v) {
    v = N.st[c];
    return v == 1 || v == 2;
  }
  __device__ __forceinline__ static unsigned long long walk_leaves(const Nodes& N, int c) {
    return N.tot[0][c] - N.tot[2][c] / 2;
  }
  // the leaf of a brick whose first voxel has Morton index t, if any: its depth (0: none) and state
  __device__ __forceinline__ static int brick_leaf(const Levels& T, int t, unsigned& v) {
    const int i14 = t >> 6, i15 = t >> 3;
    int depth = 0;
    v = 0;
    if (T.s14[i14] != 3) {
      if ((t & 63) == 0 && T.s14[i14]) depth = 14, v = T.s14[i14];
    } else if (T.s15[i15] != 3) {
      if ((t & 7) == 0 && T.s15[i15]) depth = 15, v = T.s15[i15];
    } else if (T.s16[t]) {
      depth = 16, v = T.s16[t];
    }
    return depth;
  }

  __device__ __forceinline__ static int pair(const unsigned char* pay, int i) {
    return (int)pay[2 * (size_t)i] | ((int)pay[2 * (size_t)i + 1] << 8);
  }
  // the children of stream item i that are stream items too: its inner children
  __device__ __forceinline__ static int streamed(const unsigned char* pay, int i) {
    const int m = pair(pay, i);
    int c = 0;
    for (int s = 0; s < 8; ++s) c |= (((m >> (2 * s)) & 3) == 3) << s;
    return c;
  }
  __device__ __forceinline__ static unsigned long long* node_count(ReadCounters* cnt) { return &cnt->nodes; }
  // (r4) inner node j at depth d: its children's counts (nodes, free and occupied leaves, known voxels 8^(16-d) per leaf at
  // depth d) and bricks: 8^(13-d) per leaf at depth d <= 13, one for the node itself at depth 13
  __device__ __forceinline__ static int count(const unsigned char* pay, int j, int d, float, unsigned long long v[4],
                                              long long& bricks) {
    const int m = pair(pay, j);
    for (int s = 0; s < 8; ++s) {
      const int b = (m >> (2 * s)) & 3;
      if (!b) continue;
      ++v[0];
      if (b == 3) continue;
      ++v[b];
      v[3] += 1ull << (3 * (15 - d));
      if (d + 1 <= kBrickDepth) bricks += 1LL << (3 * (kBrickDepth - 1 - d));
    }
    if (d == kBrickDepth) bricks += 1;
    return 0;
  }
  // (r5) brick r of inner node j (depth d, first key k0): under a leaf child (its state; a leaf's bricks in Morton order),
  // or, at depth 13, the node's own brick (3: mixed)
  __device__ __forceinline__ static int brick(const unsigned char* pay, int j, int d, unsigned long long k0, long long r,
                                              int k[3]) {
    k[0] = (int)(k0 & 0xffff), k[1] = (int)((k0 >> 16) & 0xffff), k[2] = (int)((k0 >> 32) & 0xffff);
    if (d == kBrickDepth) return 3;
    const int m = pair(pay, j), sh = 15 - d;
    for (int s = 0; s < 8; ++s) {
      const int bits = (m >> (2 * s)) & 3;
      if (bits == 0 || bits == 3) continue;
      const long long c = 1LL << (3 * (kBrickDepth - 1 - d));
      if (r >= c) {
        r -= c;
        continue;
      }
      k[0] += ((s & 1) << sh) + (squeeze3((unsigned long long)r) << 3);
      k[1] += (((s >> 1) & 1) << sh) + (squeeze3((unsigned long long)r >> 1) << 3);
      k[2] += (((s >> 2) & 1) << sh) + (squeeze3((unsigned long long)r >> 2) << 3);
      return bits;
    }
    return 3;
  }
  // (r6) a uniform brick holds L_min or L_max
  __device__ __forceinline__ static float uniform(const Params& P, const unsigned char*, const long long*, int, int, int st) {
    return st == 1 ? P.l_min : st == 2 ? P.l_max : 0.0f;
  }
  // (r7) inner nodes at depth 13 ... 15 write the 64, 8 or 1 voxels of each of their leaves
  __device__ __forceinline__ static bool writes_leaves(const unsigned char*, int, int d) { return d >= kBrickDepth; }
  template <class Cube>
  __device__ __forceinline__ static void leaves(const Params& P, const unsigned char* pay, int j, int d,
                                                unsigned long long k0, Cube&& cube) {
    const int m = pair(pay, j), sh = 15 - d;
    for (int s = 0; s < 8; ++s) {
      const int bits = (m >> (2 * s)) & 3;
      if (bits == 0 || bits == 3) continue;
      cube(((int)(k0 & 7)) | ((s & 1) << sh), ((int)((k0 >> 16) & 7)) | (((s >> 1) & 1) << sh),
           ((int)((k0 >> 32) & 7)) | (((s >> 2) & 1) << sh), 1 << sh, bits == 1 ? P.l_min : P.l_max);
    }
  }

  static int check(const ReadCounters& c, long long, long long nodes, const char** why) {
    if (c.end == INT_MAX) return *why = "the payload is truncated", LS_ERR_ARG;
    if (c.bad) return *why = "an inner node at depth 16", LS_ERR_ARG;
    if ((long long)c.nodes + 1 != nodes) return *why = "the header's size does not count the payload's nodes", LS_ERR_ARG;
    return LS_OK;
  }
  static void counts(ReadCounters* out) {  // the root counts as a node; every stream item is inner
    out->nodes += 1;
    out->inner = (unsigned long long)out->end;
  }
};

// .ot: node states 0 no known voxel below, 1 leaf, 3 inner; values are float log-odds kept as their bits.  Every node is
// in the stream, 5 bytes each: its value, then the mask of its existing children.  Totals: nodes, leaves.
struct FullTree {
  static constexpr int kNodeBytes = 5, kTotals = 2;
  static constexpr bool kValued = true;
  static constexpr int kMaxDepth = 16;
  static constexpr int kMaxExcess = 8 + 7 * 15;  // the largest excess of a tree whose nodes lie at depth <= 16
  static constexpr const char* kTooMany = "more than 2^30 nodes";
  static constexpr bool kCentres = false;
  static long long payload_bytes(const unsigned long long* tot) { return kNodeBytes * (long long)tot[0]; }

  // octomap's isNodeCollapsible on values (all 8 children exist, are leaves and compare equal as floats; the collapsed
  // leaf keeps child 0's bits) and updateInnerOccupancy (an inner node holds its largest child, the earliest on ties).
  // Children are added in child order.
  struct Merge {
    int na = 0, nl = 0;
    bool eq = true;
    unsigned first = 0, best = 0;
    __device__ __forceinline__ void add(int s, unsigned v) {
      if (!s) return;
      if (na == 0) {
        first = best = v;
      } else {
        eq = eq && __uint_as_float(v) == __uint_as_float(first);
        if (__uint_as_float(v) > __uint_as_float(best)) best = v;
      }
      ++na;
      nl += s == 1;
    }
    __device__ __forceinline__ int state(bool may_prune, unsigned& v) const {
      if (may_prune && nl == 8 && eq) {
        v = first;
        return 1;
      }
      v = best;
      return na ? 3 : 0;
    }
  };
  // (e) as BinaryTree's, merging values
  struct Levels {
    unsigned v16[512], v15[64], v14[8];
    unsigned char s16[512], s15[64], s14[8];
    int n15[64], l15[64], n14[8], l14[8];
    int st, nodes, leaves;  // the depth-13 node
    unsigned val;
  };
  __device__ static void levels(const unsigned* __restrict__ known, const float* __restrict__ lo, int b, float, Levels& T) {
    const int t = threadIdx.x;
    const int v = morton_local(t);
    T.s16[t] = (unsigned char)((known[(size_t)b * 16 + (v >> 5)] >> (v & 31)) & 1u);
    T.v16[t] = __float_as_uint(lo[(size_t)b * 512 + v]);
    __syncthreads();
    if (t < 64) {
      Merge m;
      for (int i = 0; i < 8; ++i) m.add(T.s16[8 * t + i], T.v16[8 * t + i]);
      unsigned val;
      const int st = m.state(true, val);
      T.s15[t] = (unsigned char)st, T.v15[t] = val;
      T.n15[t] = st == 3 ? 1 + m.na : st != 0;
      T.l15[t] = st == 3 ? m.na : st != 0;
    }
    __syncthreads();
    if (t < 8) {
      Merge m;
      int n = 0, l = 0;
      for (int i = 0; i < 8; ++i) m.add(T.s15[8 * t + i], T.v15[8 * t + i]), n += T.n15[8 * t + i], l += T.l15[8 * t + i];
      unsigned val;
      const int st = m.state(true, val);
      T.s14[t] = (unsigned char)st, T.v14[t] = val;
      T.n14[t] = st == 3 ? 1 + n : st != 0;
      T.l14[t] = st == 3 ? l : st != 0;
    }
    __syncthreads();
    if (t == 0) {
      Merge m;
      int n = 0, l = 0;
      for (int i = 0; i < 8; ++i) m.add(T.s14[i], T.v14[i]), n += T.n14[i], l += T.l14[i];
      unsigned val;
      const int st = m.state(true, val);
      T.st = st, T.val = val;
      T.nodes = st == 3 ? 1 + n : st != 0;
      T.leaves = st == 3 ? l : st != 0;
    }
    __syncthreads();
  }
  __device__ __forceinline__ static void record(const Levels& T, const Nodes& N, int r) {
    N.st[r] = (unsigned char)T.st;
    N.val[r] = T.val;
    N.tot[0][r] = (unsigned long long)T.nodes;
    N.tot[1][r] = (unsigned long long)T.leaves;
  }
  template <class T>
  __device__ __forceinline__ static void totals(int s, T* c) {
    c[0] = s == 3 ? c[0] + 1 : (T)(s != 0);
    c[1] = s == 3 ? c[1] : (T)(s != 0);
  }
  __device__ __forceinline__ static void put_node(unsigned char* p, unsigned v, int mask) {
    p[0] = (unsigned char)(v & 0xff), p[1] = (unsigned char)((v >> 8) & 0xff), p[2] = (unsigned char)((v >> 16) & 0xff);
    p[3] = (unsigned char)(v >> 24), p[4] = (unsigned char)mask;
  }
  __device__ __forceinline__ static int child_bits(int s, int slot) { return (s != 0) << slot; }
  __device__ __forceinline__ static void put_inner(unsigned char* p, const Nodes& N, int i, int mask) {
    put_node(p, N.val[i], mask);
  }
  // (g) child c takes its offset; a leaf writes its node (an inner brick writes itself in (h))
  __device__ __forceinline__ static void place(const Nodes& N, int c, int, unsigned long long& o, unsigned long long&,
                                               double, unsigned char* payload, float4*, unsigned char*) {
    N.off[c] = o;
    if (N.st[c] == 1) put_node(payload + o, N.val[c], 0);
    o += kNodeBytes * N.tot[0][c];
  }
  // The leaf walk (l1, l2): a leaf record's value is its log-odds bits.
  __device__ __forceinline__ static bool walk_leaf(const Nodes& N, int c, unsigned& v) {
    if (N.st[c] != 1) return false;
    v = N.val[c];
    return true;
  }
  __device__ __forceinline__ static unsigned long long walk_leaves(const Nodes& N, int c) { return N.tot[1][c]; }
  __device__ __forceinline__ static int brick_leaf(const Levels& T, int t, unsigned& v) {
    const int i14 = t >> 6, i15 = t >> 3;
    int depth = 0;
    v = 0;
    if (T.s14[i14] != 3) {
      if ((t & 63) == 0 && T.s14[i14] == 1) depth = 14, v = T.v14[i14];
    } else if (T.s15[i15] != 3) {
      if ((t & 7) == 0 && T.s15[i15] == 1) depth = 15, v = T.v15[i15];
    } else if (T.s16[t]) {
      depth = 16, v = T.v16[t];
    }
    return depth;
  }

  __device__ __forceinline__ static int mask(const unsigned char* pay, int i) { return pay[(size_t)kNodeBytes * i + 4]; }
  __device__ __forceinline__ static unsigned value(const unsigned char* pay, int i) {
    const unsigned char* p = pay + (size_t)kNodeBytes * i;
    return (unsigned)p[0] | ((unsigned)p[1] << 8) | ((unsigned)p[2] << 16) | ((unsigned)p[3] << 24);
  }
  __device__ __forceinline__ static int streamed(const unsigned char* pay, int i) { return mask(pay, i); }
  __device__ __forceinline__ static unsigned long long* node_count(ReadCounters* cnt) { return &cnt->inner; }
  // (r4) node j at depth d: a node with children (one brick of its own at depth 13), or a leaf by state with 8^(16-d)
  // known voxels and 8^(13-d) bricks (d <= 13).  Children at depth 16 and leaf values that are not finite are refused.
  __device__ __forceinline__ static int count(const unsigned char* pay, int j, int d, float l_occ, unsigned long long v[4],
                                              long long& bricks) {
    const int m = mask(pay, j);
    const float val = __uint_as_float(value(pay, j));
    if (d == 16 && m) return kBadDepth;
    if (!m && !isfinite(val)) return kBadValue;
    if (m) {
      v[0] = 1;
      if (d == kBrickDepth) bricks = 1;
    } else {
      ++v[val >= l_occ ? 2 : 1];
      v[3] = 1ull << (3 * (16 - d));
      if (d <= kBrickDepth) bricks = 1LL << (3 * (kBrickDepth - d));
    }
    return 0;
  }
  // (r5) brick r of node j: a leaf's bricks in Morton order (1), or, at depth 13, the node's own brick (3: mixed)
  __device__ __forceinline__ static int brick(const unsigned char* pay, int j, int d, unsigned long long k0, long long r,
                                              int k[3]) {
    const bool mixed = d == kBrickDepth && mask(pay, j) != 0;
    const unsigned long long u = (unsigned long long)r;
    k[0] = (int)(k0 & 0xffff) + (mixed ? 0 : squeeze3(u) << 3);
    k[1] = (int)((k0 >> 16) & 0xffff) + (mixed ? 0 : squeeze3(u >> 1) << 3);
    k[2] = (int)((k0 >> 32) & 0xffff) + (mixed ? 0 : squeeze3(u >> 2) << 3);
    return mixed ? 3 : 1;
  }
  // (r6) a uniform brick holds its leaf's value
  __device__ __forceinline__ static float uniform(const Params&, const unsigned char* pay, const long long* boff, int end,
                                                  int b, int st) {
    return st == 1 ? __uint_as_float(value(pay, brick_owner(boff, end, b))) : 0.0f;
  }
  // (r7) leaves at depth 14 ... 16 write their 64, 8 or 1 voxels
  __device__ __forceinline__ static bool writes_leaves(const unsigned char* pay, int j, int d) {
    return d > kBrickDepth && !mask(pay, j);
  }
  template <class Cube>
  __device__ __forceinline__ static void leaves(const Params&, const unsigned char* pay, int j, int d, unsigned long long k0,
                                                Cube&& cube) {
    cube((int)(k0 & 7), (int)((k0 >> 16) & 7), (int)((k0 >> 32) & 7), 1 << (16 - d), __uint_as_float(value(pay, j)));
  }

  static int check(const ReadCounters& c, long long count, long long nodes, const char** why) {
    if (c.end == INT_MAX)
      return *why = count < nodes ? "the payload is truncated" : "the header's size does not count the payload's nodes",
             LS_ERR_ARG;
    if (c.bad & kBadDepth) return *why = "a node at depth 16 with children", LS_ERR_ARG;
    if (c.bad & kBadValue) return *why = "a leaf value that is NaN or infinite", LS_ERR_ARG;
    if ((long long)c.end != nodes) return *why = "the header's size does not count the payload's nodes", LS_ERR_ARG;
    return LS_OK;
  }
  static void counts(ReadCounters* out) { out->nodes = (unsigned long long)out->end; }
};

// ---- export: (d) ... (h) ---------------------------------------------------------------------------------------------
// (d)
__global__ void oct_code_kernel(const unsigned long long* __restrict__ bkey, int n, unsigned long long* __restrict__ code,
                                int* __restrict__ idx) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long k = bkey[i];
  code[i] = spread3((unsigned)(k & 0x1fff)) | (spread3((unsigned)((k >> 13) & 0x1fff)) << 1) |
            (spread3((unsigned)((k >> 26) & 0x1fff)) << 2);
  idx[i] = i;
}

// (e) one block per brick record, in pre-order: state, value and subtree totals
template <class F>
__global__ void __launch_bounds__(512) oct_brick_kernel(const unsigned* __restrict__ known, const float* __restrict__ lo,
                                                        Nodes N, float l_occ) {
  __shared__ typename F::Levels T;
  const int r = blockIdx.x;
  F::levels(known, lo, N.pool[r], l_occ, T);
  if (threadIdx.x == 0) F::record(T, N, r);
}

// (f) levels 12 ... 0 appended after the n_b brick records; levels[2d], levels[2d + 1]: first record and count at depth d.
// tot: the root's totals (all 0 when no voxel is known).
template <class F>
__global__ void __launch_bounds__(kTreeThreads) oct_up_kernel(Nodes N, int n_b, int* levels, unsigned long long* tot) {
  using Scan = cub::BlockScan<int, kTreeThreads>;
  __shared__ typename Scan::TempStorage scan;
  const int t = threadIdx.x;
  int cb = 0, cn = n_b;  // the level below
  if (t == 0) levels[2 * kBrickDepth] = 0, levels[2 * kBrickDepth + 1] = n_b;
  for (int d = kBrickDepth - 1; d >= 0; --d) {
    const int pb = cb + cn;
    int pn = 0;
    for (int c0 = 0; c0 < cn; c0 += kTreeThreads) {
      const int i = c0 + t;
      const int head = i < cn && (i == 0 || (N.code[cb + i] >> 3) != (N.code[cb + i - 1] >> 3));
      int pos, total;
      Scan(scan).ExclusiveSum(head, pos, total);
      if (head) {
        N.code[pb + pn + pos] = N.code[cb + i] >> 3;
        N.first[pb + pn + pos] = cb + i;
      }
      pn += total;
      __syncthreads();
    }
    for (int p = pb + t; p < pb + pn; p += kTreeThreads) {
      const int f = N.first[p], e = p + 1 < pb + pn ? N.first[p + 1] : pb;
      typename F::Merge m;
      unsigned long long sum[F::kTotals] = {};
      for (int c = f; c < e; ++c) {
        m.add(N.st[c], F::kValued ? N.val[c] : 0u);
        for (int k = 0; k < F::kTotals; ++k) sum[k] += N.tot[k][c];
      }
      unsigned v;
      const int s = m.state(d > 0, v);  // octomap's prune() stops at depth 1: the root stays inner
      N.st[p] = (unsigned char)s;
      if (F::kValued) N.val[p] = v;
      N.end[p] = e;
      F::totals(s, sum);
      for (int k = 0; k < F::kTotals; ++k) N.tot[k][p] = sum[k];
    }
    __syncthreads();
    if (t == 0) levels[2 * d] = pb, levels[2 * d + 1] = pn;
    cb = pb, cn = pn;
  }
  if (t == 0)
    for (int k = 0; k < F::kTotals; ++k) tot[k] = N.tot[k][cb];
}

// (g) levels 0 ... 12: each inner node writes its record and gives every child its offsets (its own + its record + the
// earlier siblings' totals)
template <class F>
__global__ void __launch_bounds__(kTreeThreads) oct_down_kernel(Nodes N, const int* __restrict__ levels, double res,
                                                                unsigned char* __restrict__ payload, float4* __restrict__ cen,
                                                                unsigned char* __restrict__ dep) {
  const int t = threadIdx.x;
  if (t == 0) N.off[levels[0]] = 0, N.loff[levels[0]] = 0;
  __syncthreads();
  for (int d = 0; d < kBrickDepth; ++d) {
    const int pb = levels[2 * d], pn = levels[2 * d + 1];
    for (int p = pb + t; p < pb + pn; p += kTreeThreads) {
      if (N.st[p] != 3) continue;  // only an inner node's children are in the tree
      const int f = N.first[p], e = N.end[p];
      int mask = 0;
      for (int c = f; c < e; ++c) mask |= F::child_bits(N.st[c], (int)(N.code[c] & 7));
      unsigned long long o = N.off[p], l = N.loff[p];
      F::put_inner(payload + o, N, p, mask);
      o += F::kNodeBytes;
      for (int c = f; c < e; ++c) F::place(N, c, d + 1, o, l, res, payload, cen, dep);
    }
    __syncthreads();
  }
}

// (h) one block per brick record; the inner ones write their nodes below depth 13 at the offset (g) gave them
template <class F>
__global__ void oct_emit_kernel(const unsigned* __restrict__ known, const float* __restrict__ lo,
                                const unsigned long long* __restrict__ bkey, Nodes N, float l_occ, double res,
                                unsigned char* __restrict__ payload, float4* __restrict__ cen, unsigned char* __restrict__ dep);

// .bt: the brick's pre-order bytes, and its occupied leaves
template <>
__global__ void __launch_bounds__(512) oct_emit_kernel<BinaryTree>(const unsigned* __restrict__ known,
                                                                   const float* __restrict__ lo,
                                                                   const unsigned long long* __restrict__ bkey, Nodes N,
                                                                   float l_occ, double res, unsigned char* __restrict__ payload,
                                                                   float4* __restrict__ cen, unsigned char* __restrict__ dep) {
  using Scan = cub::BlockScan<int, 512>;
  __shared__ BinaryTree::Levels T;
  __shared__ typename Scan::TempStorage scan;
  const int r = blockIdx.x;
  if (N.st[r] != 3) return;  // a leaf brick is written by its parent in (g)
  const int b = N.pool[r];
  BinaryTree::levels(known, lo, b, l_occ, T);
  const int t = threadIdx.x;
  if (t == 0) {  // pre-order: the brick, then each inner depth-14 node followed by its inner depth-15 nodes
    unsigned char* p = payload + N.off[r];
    int m = mask8(T.s14);
    *p++ = (unsigned char)(m & 0xff), *p++ = (unsigned char)(m >> 8);
    for (int i = 0; i < 8; ++i) {
      if (T.s14[i] != 3) continue;
      m = mask8(T.s15 + 8 * i);
      *p++ = (unsigned char)(m & 0xff), *p++ = (unsigned char)(m >> 8);
      for (int j = 0; j < 8; ++j) {
        if (T.s15[8 * i + j] != 3) continue;
        m = mask8(T.s16 + 64 * i + 8 * j);
        *p++ = (unsigned char)(m & 0xff), *p++ = (unsigned char)(m >> 8);
      }
    }
  }
  // the occupied leaf whose first voxel is t, in Morton order = pre-order
  const int s14 = T.s14[t >> 6], s15 = T.s15[t >> 3];
  int depth = 0;
  if (s14 != 3) depth = s14 == 2 && (t & 63) == 0 ? 14 : 0;
  else if (s15 != 3) depth = s15 == 2 && (t & 7) == 0 ? 15 : 0;
  else depth = T.s16[t] == 2 ? 16 : 0;
  int idx;
  Scan(scan).ExclusiveSum(depth != 0 ? 1 : 0, idx);
  if (depth) {
    int k[3];
    voxel_keys(bkey[b], morton_local(t), k);
    put_leaf(cen, dep, N.loff[r] + (unsigned long long)idx, k[0], k[1], k[2], depth, res);
  }
}

// .ot: the brick's up to 585 nodes placed in parallel.  Thread t owns, in pre-order, the depth-14 node starting at Morton
// index t (t % 64 == 0), the depth-15 one (t % 8 == 0) and voxel t, each when it is in the tree; a block scan over the
// owned counts gives each its place.
template <>
__global__ void __launch_bounds__(512) oct_emit_kernel<FullTree>(const unsigned* __restrict__ known, const float* __restrict__ lo,
                                                                 const unsigned long long* __restrict__, Nodes N, float l_occ,
                                                                 double, unsigned char* __restrict__ payload,
                                                                 float4* __restrict__, unsigned char* __restrict__) {
  using Scan = cub::BlockScan<int, 512>;
  __shared__ FullTree::Levels T;
  __shared__ typename Scan::TempStorage scan;
  const int r = blockIdx.x;
  if (N.st[r] != 3) return;  // a leaf brick is written by its parent in (g)
  FullTree::levels(known, lo, N.pool[r], l_occ, T);
  const int t = threadIdx.x;
  unsigned char* base = payload + N.off[r];
  if (t == 0) {
    int m = 0;
    for (int i = 0; i < 8; ++i) m |= (T.s14[i] != 0) << i;
    FullTree::put_node(base, T.val, m);
  }
  const int i14 = t >> 6, i15 = t >> 3;
  const bool a = (t & 63) == 0 && T.s14[i14] != 0;
  const bool b = (t & 7) == 0 && T.s14[i14] == 3 && T.s15[i15] != 0;
  const bool c = T.s14[i14] == 3 && T.s15[i15] == 3 && T.s16[t] != 0;
  int idx;
  Scan(scan).ExclusiveSum((int)a + (int)b + (int)c, idx);
  unsigned char* p = base + (size_t)FullTree::kNodeBytes * (1 + idx);
  if (a) {
    int m = 0;
    if (T.s14[i14] == 3)
      for (int i = 0; i < 8; ++i) m |= (T.s15[8 * i14 + i] != 0) << i;
    FullTree::put_node(p, T.v14[i14], m);
    p += FullTree::kNodeBytes;
  }
  if (b) {
    int m = 0;
    if (T.s15[i15] == 3)
      for (int i = 0; i < 8; ++i) m |= (T.s16[8 * i15 + i] != 0) << i;
    FullTree::put_node(p, T.v15[i15], m);
    p += FullTree::kNodeBytes;
  }
  if (c) FullTree::put_node(p, T.v16[t], 0);
}

// ---- leaf lists: (l1) ... (l4), over the records of a .ot build ---------------------------------------------------------
// A leaf's tag: its depth, plus kFreeTag when its value is below L_occ.  A radix sort over bit 5 splits the list by state,
// over bits 0 ... 5 by (state, depth), occupied first; both sorts are stable, so each part keeps the leaf iterator's order.
constexpr int kFreeTag = 32, kLeafBuckets = 34;  // bucket: depth, or 17 + depth for a free leaf

// The key range of a listing per axis: a leaf is kept iff its key cube [k0, k0 + side) meets [lo, hi] on every axis.
struct KeyRange {
  int lo[3], hi[3];
};

__device__ __forceinline__ void put_tree_leaf(int kx, int ky, int kz, int depth, unsigned v, float l_occ, double res,
                                              const KeyRange& R, unsigned long long i, float4* __restrict__ cen,
                                              unsigned char* __restrict__ tag, int* __restrict__ keep) {
  const int s = 16 - depth, side = 1 << s;
  cen[i] = make_float4(leaf_coord(kx, s, res), leaf_coord(ky, s, res), leaf_coord(kz, s, res), 1.0f);
  tag[i] = (unsigned char)(depth | (__uint_as_float(v) >= l_occ ? 0 : kFreeTag));
  keep[i] = kx <= R.hi[0] && kx + side - 1 >= R.lo[0] && ky <= R.hi[1] && ky + side - 1 >= R.lo[1] && kz <= R.hi[2] &&
            kz + side - 1 >= R.lo[2];
}

// What the walk writes per leaf: out(kx, ky, kz, depth, v, i) for the leaf whose first voxel key is (kx, ky, kz) and whose
// place in pre-order is i, v its value (F::walk_leaf's).  The leaf list writes a box (BoxOut, over a .ot build); the 2D
// projection a packed key (KeyOut, over a .bt build).
struct BoxOut {
  float l_occ;
  double res;
  KeyRange R;
  float4* __restrict__ cen;
  unsigned char* __restrict__ tag;
  int* __restrict__ keep;
  __device__ __forceinline__ void operator()(int kx, int ky, int kz, int depth, unsigned v, unsigned long long i) const {
    put_tree_leaf(kx, ky, kz, depth, v, l_occ, res, R, i, cen, tag, keep);
  }
};
struct KeyOut {
  unsigned long long* __restrict__ rec;
  __device__ __forceinline__ void operator()(int kx, int ky, int kz, int depth, unsigned v, unsigned long long i) const {
    rec[i] = leaf_record(kx, ky, kz, depth, v == 2);
  }
};

// (l1) levels 0 ... 12 as (g): each inner node gives its children their leaf offsets (its own + the earlier siblings'
// leaves); a leaf child, bricks at depth 13 included, writes itself
template <class F, class Out>
__global__ void __launch_bounds__(kTreeThreads) lv_down_kernel(Nodes N, const int* __restrict__ levels, Out out) {
  const int t = threadIdx.x;
  if (t == 0) N.loff[levels[0]] = 0;
  __syncthreads();
  for (int d = 0; d < kBrickDepth; ++d) {
    const int pb = levels[2 * d], pn = levels[2 * d + 1];
    for (int p = pb + t; p < pb + pn; p += kTreeThreads) {
      if (N.st[p] != 3) continue;
      unsigned long long l = N.loff[p];
      for (int c = N.first[p]; c < N.end[p]; ++c) {
        N.loff[c] = l;
        unsigned v;
        if (F::walk_leaf(N, c, v)) {
          const unsigned long long k = N.code[c];
          const int sh = 15 - d;
          out(squeeze3(k) << sh, squeeze3(k >> 1) << sh, squeeze3(k >> 2) << sh, d + 1, v, l);
        }
        l += F::walk_leaves(N, c);
      }
    }
    __syncthreads();
  }
}

// (l2) one block per inner brick: (e)'s levels again; thread t owns the leaf whose first voxel has Morton index t, if
// any (a depth-14 leaf at t % 64 == 0, a depth-15 one at t % 8 == 0 or voxel t), and a block scan places it
template <class F, class Out>
__global__ void __launch_bounds__(512) lv_emit_kernel(const unsigned* __restrict__ known, const float* __restrict__ lo,
                                                      const unsigned long long* __restrict__ bkey, Nodes N, float l_occ,
                                                      Out out) {
  using Scan = cub::BlockScan<int, 512>;
  __shared__ typename F::Levels T;
  __shared__ typename Scan::TempStorage scan;
  const int r = blockIdx.x;
  if (N.st[r] != 3) return;  // a leaf brick is written in (l1)
  const int b = N.pool[r];
  F::levels(known, lo, b, l_occ, T);
  const int t = threadIdx.x;
  unsigned v;
  const int depth = F::brick_leaf(T, t, v);
  int idx;
  Scan(scan).ExclusiveSum(depth != 0 ? 1 : 0, idx);
  if (depth) {
    int k[3];
    voxel_keys(bkey[b], morton_local(t), k);
    out(k[0], k[1], k[2], depth, v, N.loff[r] + (unsigned long long)idx);
  }
}

// (l3) after an exclusive scan of keep into pos: the kept leaves in order, their positions and the count per bucket
__global__ void __launch_bounds__(256) lv_compact_kernel(const float4* __restrict__ raw_c, const unsigned char* __restrict__ raw_tag,
                                                         const int* __restrict__ keep, const int* __restrict__ pos, int n,
                                                         float4* __restrict__ cen, unsigned char* __restrict__ tag,
                                                         int* __restrict__ idx, unsigned long long* __restrict__ count) {
  __shared__ unsigned hist[kLeafBuckets];
  if (threadIdx.x < kLeafBuckets) hist[threadIdx.x] = 0;
  __syncthreads();
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (!keep[i]) continue;
    const int j = pos[i], g = raw_tag[i];
    cen[j] = raw_c[i], tag[j] = (unsigned char)g, idx[j] = j;
    atomicAdd(&hist[(g & kFreeTag ? 17 : 0) + (g & 31)], 1u);
  }
  __syncthreads();
  if (threadIdx.x < kLeafBuckets && hist[threadIdx.x]) atomicAdd(&count[threadIdx.x], (unsigned long long)hist[threadIdx.x]);
}

// octomap_server's heightMapColor(h), in double and cast to float once: s = v = 1, so m = 0 and n = 1 - f
__device__ __forceinline__ float4 height_colour(double h) {
  h -= floor(h);
  h *= 6.0;
  const int i = (int)floor(h);
  double f = h - (double)i;
  if (!(i & 1)) f = 1.0 - f;
  const double n = 1.0 - f;
  double r = 1.0, g = 0.5, b = 0.5;
  switch (i) {
    case 6:
    case 0: r = 1.0, g = n, b = 0.0; break;
    case 1: r = n, g = 1.0, b = 0.0; break;
    case 2: r = 0.0, g = 1.0, b = n; break;
    case 3: r = 0.0, g = n, b = 1.0; break;
    case 4: r = n, g = 0.0, b = 1.0; break;
    case 5: r = 1.0, g = 0.0, b = n; break;
  }
  return make_float4((float)r, (float)g, (float)b, 1.0f);
}

// (l4) entries [first, first + n) of the sorted order gathered: centres and tags; the first n_col of them also take
// generateMarkerArray's height colour h = (1 - min(max((z - min_z) / (max_z - min_z), 0), 1)) * color_factor
__global__ void lv_gather_kernel(const float4* __restrict__ cen, const unsigned char* __restrict__ tag,
                                 const int* __restrict__ order, long long first, long long n, long long n_col, double min_z,
                                 double max_z, double color_factor, float4* __restrict__ out_c,
                                 unsigned char* __restrict__ out_tag, float4* __restrict__ rgba) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int j = order[first + i];
    const float4 c = cen[j];
    out_c[i] = c, out_tag[i] = tag[j];
    if (i < n_col) {
      double x = ((double)c.z - min_z) / (max_z - min_z);
      x = x < 0.0 ? 0.0 : x;  // std::max(x, 0.0)
      x = 1.0 < x ? 1.0 : x;  // std::min(x, 1.0)
      rgba[i] = height_colour((1.0 - x) * color_factor);
    }
  }
}

// ---- read: (r1) ... (r7) ---------------------------------------------------------------------------------------------
// Item i of the stream is the i-th node of it in pre-order.  With c_i its children in the stream, the excess E_0 = 1,
// E_{i+1} = E_i + c_i - 1 counts the stream nodes found but not yet read; the tree ends at the first i >= 1 with E_i = 0.
struct MinOp {
  __device__ __forceinline__ int operator()(int a, int b) const { return a < b ? a : b; }
};

// (r1) in[0] = 1 and in[i + 1] = c_i - 1: an inclusive sum gives E_0 ... E_n
template <class F>
__global__ void rd_excess_kernel(const unsigned char* __restrict__ pay, int n, int* __restrict__ in) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) in[0] = 1;
  if (i < n) in[i + 1] = __popc(F::streamed(pay, i)) - 1;
}

// (r2) the tree's end and, per block of kReadThreads items, the least excess (r3) skips blocks by
__global__ void __launch_bounds__(kReadThreads) rd_end_kernel(const int* __restrict__ ex, int n, int* __restrict__ bmin,
                                                             ReadCounters* cnt) {
  using Reduce = cub::BlockReduce<int, kReadThreads>;
  __shared__ typename Reduce::TempStorage tmp;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int e = i <= n ? ex[i] : INT_MAX;
  if (i >= 1 && i <= n && e == 0) atomicMin(&cnt->end, i);
  const int m = Reduce(tmp).Reduce(e, MinOp());
  if (threadIdx.x == 0) bmin[blockIdx.x] = m;
}

// (r3) per stream node j >= 1: its parent, the last i < j with E_i <= E_j, and its slot, the (E_p + c_p - 1 - E_j)-th
// stream child of p.  An excess above the format's bound proves a stream node too deep.
template <class F>
__global__ void rd_parent_kernel(const unsigned char* __restrict__ pay, const int* __restrict__ ex,
                                 const int* __restrict__ bmin, int n, int* __restrict__ par, unsigned char* __restrict__ slot,
                                 ReadCounters* cnt) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n || j >= cnt->end) return;
  const int e = ex[j];
  if (e > F::kMaxExcess) {
    atomicOr(&cnt->bad, kBadDepth);
    return;
  }
  if (j == 0) {
    par[0] = -1, slot[0] = 0;
    return;
  }
  const int b0 = j / kReadThreads * kReadThreads;
  int p = j - 1;
  while (p >= b0 && ex[p] > e) --p;
  if (p < b0) {  // E_0 = 1 <= e: some earlier block holds the parent
    int b = j / kReadThreads - 1;
    while (bmin[b] > e) --b;
    p = b * kReadThreads + kReadThreads - 1;
    while (ex[p] > e) --p;
  }
  const int m = F::streamed(pay, p);
  int rank = ex[p] + __popc(m) - 1 - e, s = 0;
  for (; s < 8; ++s)
    if (((m >> s) & 1) && rank-- == 0) break;
  par[j] = p;
  slot[j] = (unsigned char)s;
}

// (r4) per stream node j: depth and first key from at most F::kMaxDepth parents (more: too deep), its depth-13 ancestor,
// and the format's counts.  nb[j] = its bricks (0 past the tree, nb[n] = 0).
template <class F>
__global__ void __launch_bounds__(kReadThreads) rd_node_kernel(const unsigned char* __restrict__ pay,
                                                              const int* __restrict__ par,
                                                              const unsigned char* __restrict__ slot, int n, float l_occ,
                                                              unsigned char* __restrict__ depth,
                                                              unsigned long long* __restrict__ key, int* __restrict__ anc,
                                                              long long* __restrict__ nb, ReadCounters* cnt) {
  using Reduce = cub::BlockReduce<unsigned long long, kReadThreads>;
  __shared__ typename Reduce::TempStorage tmp;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  unsigned long long v[4] = {0, 0, 0, 0};  // F::node_count, free leaves, occupied leaves, known voxels
  long long bricks = 0;
  if (j < n && j < cnt->end && !cnt->bad) {
    // step i visits the ancestor at depth d - i: its slot is key bit 16 - d + i; the depth-13 one is among steps 0 ... 3
    int d = 0, x = j, a1 = j, a2 = j, a3 = j;
    unsigned long long slots = 0;
    while (x != 0 && d < F::kMaxDepth) {
      if (d == 1) a1 = x;
      if (d == 2) a2 = x;
      if (d == 3) a3 = x;
      slots |= (unsigned long long)slot[x] << (3 * d);
      ++d;
      x = par[x];
    }
    const int bad = x != 0 ? kBadDepth : F::count(pay, j, d, l_occ, v, bricks);
    if (bad) {
      atomicOr(&cnt->bad, bad);
    } else {
      unsigned kx = 0, ky = 0, kz = 0;
      for (int i = 0; i < d; ++i) {
        const unsigned s = (unsigned)(slots >> (3 * i)) & 7u, b = (unsigned)(16 - d + i);
        kx |= (s & 1u) << b, ky |= ((s >> 1) & 1u) << b, kz |= ((s >> 2) & 1u) << b;
      }
      depth[j] = (unsigned char)d;
      key[j] = pack((int)kx, (int)ky, (int)kz);
      anc[j] = d == kBrickDepth ? j : d == kBrickDepth + 1 ? a1 : d == kBrickDepth + 2 ? a2 : d == kBrickDepth + 3 ? a3 : -1;
    }
  }
  if (j <= n) nb[j] = bricks;
  for (int k = 0; k < 4; ++k) {
    const unsigned long long t = Reduce(tmp).Sum(v[k]);
    if (threadIdx.x == 0 && t) atomicAdd(k == 0 ? F::node_count(cnt) : k == 1 ? &cnt->free_leaves : k == 2 ? &cnt->occ_leaves
                                                                                                       : &cnt->known, t);
    __syncthreads();
  }
}

// (r5) per new brick, in pre-order: its key and state (1 free, 2 occupied: uniform; 3: below a node with children at depth
// 13), from the stream node whose bricks hold it
template <class F>
__global__ void rd_brick_kernel(const unsigned char* __restrict__ pay, const unsigned char* __restrict__ depth,
                                const unsigned long long* __restrict__ key, const long long* __restrict__ boff, int end,
                                int n_b, unsigned long long* __restrict__ bkey, unsigned char* __restrict__ bst) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= n_b) return;
  const int j = brick_owner(boff, end, b);
  int k[3];
  const int st = F::brick(pay, j, depth[j], key[j], b - boff[j], k);
  bkey[b] = brick_key(k);
  bst[b] = (unsigned char)st;
}

// (r6) one block of 512 threads per new brick: a uniform brick holds the format's value and is all known, a mixed one
// starts empty; marks and touched flags clear
template <class F>
__global__ void __launch_bounds__(512) rd_fill_kernel(Dev D, Params P, const unsigned char* __restrict__ pay,
                                                      const long long* __restrict__ boff, int end,
                                                      const unsigned long long* __restrict__ bkey,
                                                      const unsigned char* __restrict__ bst) {
  __shared__ float v;
  const int b = blockIdx.x, t = threadIdx.x, st = bst[b];
  if (t == 0) v = F::uniform(P, pay, boff, end, b, st);
  __syncthreads();
  D.lo[(size_t)b * 512 + t] = v;
  if (t < 16) {
    D.known[(size_t)b * 16 + t] = st == 3 ? 0u : ~0u;
    D.mfree[(size_t)b * 16 + t] = 0u;
    D.mocc[(size_t)b * 16 + t] = 0u;
  }
  if (t == 0) D.touched[b] = 0u, D.bkey[b] = bkey[b];
}

// (r7) per stream node: the voxels of the leaves below depth 13 it writes, each in its depth-13 ancestor's brick
template <class F>
__global__ void rd_leaf_kernel(Dev D, Params P, const unsigned char* __restrict__ pay, const unsigned char* __restrict__ depth,
                               const unsigned long long* __restrict__ key, const int* __restrict__ anc,
                               const long long* __restrict__ boff, int end) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= end) return;
  const int d = depth[j];
  if (!F::writes_leaves(pay, j, d)) return;
  const size_t b = (size_t)boff[anc[j]];
  F::leaves(P, pay, j, d, key[j], [&](int x0, int y0, int z0, int side, float v) { fill_cube(D, b, x0, y0, z0, side, v); });
}

// ---- edits (volumetric_mapping's setLogOddsBoundingBox, resetMap, getOccupiedPointcloudInBoundingBox and the map's
// extent; DESIGN.md §4b'''''''') -----------------------------------------------------------------------------------------
// A set box as the kernels see it: per axis, the bricks its loop reaches, axes[off[a] .. off[a] + n[a]) (brick index << 8 |
// the 8-bit mask of the brick's keys the loop reaches), and its first (box, brick) item over the whole call.
struct EditBox {
  int off[3], n[3];
  long long item0;
};

// Brick key of item j of box B (bricks x outer, z inner) and the masks of its keys in the box.
__device__ __forceinline__ unsigned long long edit_brick(const EditBox& B, const unsigned* __restrict__ axes, long long j,
                                                         unsigned m[3]) {
  const long long nyz = (long long)B.n[1] * B.n[2];
  const unsigned ax = axes[B.off[0] + (int)(j / nyz)], ay = axes[B.off[1] + (int)((j / B.n[2]) % B.n[1])],
                 az = axes[B.off[2] + (int)(j % B.n[2])];
  m[0] = ax & 0xffu, m[1] = ay & 0xffu, m[2] = az & 0xffu;
  return brick_pack(ax >> 8, ay >> 8, az >> 8);
}

// One thread per (box, brick) item of the call.  kClaim false: the items whose brick the hash lacks, counted into
// cnt->n_out (a brick missing from several boxes counts once per box).  kClaim true: every item's brick placed with
// brick_of, after the pool and the hash have grown for the count.
template <bool kClaim>
__global__ void ed_bricks_kernel(const EditBox* __restrict__ boxes, int nb, const unsigned* __restrict__ axes, long long items,
                                 Dev D, Counters* cnt) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  bool miss = false;
  if (i < items) {
    int lo = 0, hi = nb - 1;  // the last box whose first item is <= i (boxes without items share the next one's)
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (boxes[mid].item0 <= i) lo = mid;
      else hi = mid - 1;
    }
    unsigned m[3];
    const unsigned long long bk = edit_brick(boxes[lo], axes, i - boxes[lo].item0, m);
    if (kClaim) brick_of(D, cnt, bk);
    else miss = find_brick(D, bk) < 0;
  }
  if (!kClaim) {
    const unsigned bal = __ballot_sync(0xffffffffu, miss);
    if ((threadIdx.x & 31) == 0 && bal) atomicAdd(&cnt->n_out, (unsigned long long)__popc(bal));
  }
}

// One box: one block of 512 threads per brick item, one thread per voxel.  A voxel is in the box iff its key is in the
// box's key list on every axis; it takes `value` and becomes known.  Newly known voxels: one popcount per warp.
__global__ void __launch_bounds__(512) ed_write_kernel(EditBox B, const unsigned* __restrict__ axes, float value, Dev D,
                                                       Counters* cnt) {
  __shared__ int sb;
  unsigned m[3];
  const unsigned long long bk = edit_brick(B, axes, blockIdx.x, m);
  const int t = threadIdx.x, lane = t & 31;
  if (t == 0) sb = find_brick(D, bk);
  __syncthreads();
  const int b = sb;
  if (b < 0) return;
  const bool in = ((m[0] >> (t & 7)) & (m[1] >> ((t >> 3) & 7)) & (m[2] >> (t >> 6)) & 1u) != 0u;
  if (in) D.lo[(size_t)b * 512 + t] = value;
  const unsigned bits = __ballot_sync(0xffffffffu, in);
  if (lane == 0 && bits) {
    unsigned* w = D.known + (size_t)b * 16 + (t >> 5);
    const unsigned old = *w;
    *w = old | bits;
    const unsigned nk = __popc(bits & ~old);
    if (nk) atomicAdd(&cnt->new_known, (unsigned long long)nk);
  }
}

// The crop: one thread per loop point (x outer, z inner) over the valid keys of each axis (keys: x's, then y's, then
// z's); flag 1 when its voxel is in `which`.
__global__ void ed_flag_kernel(const int* __restrict__ keys, int nx, int ny, int nz, long long n, Dev D, Params P, int which,
                               int* __restrict__ flag) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int k[3] = {keys[(int)(i / ((long long)ny * nz))], keys[nx + (int)((i / nz) % ny)], keys[nx + ny + (int)(i % nz)]};
  Cursor cur;
  const int s = state_of(D, P, cur, k, nullptr);
  flag[i] = s == LS_CELL_OCCUPIED || (which == LS_OCC_KNOWN && s == LS_CELL_FREE);
}

// The flagged points in loop order at their inclusive-scan positions: packed key, log-odds bits and voxel centre.
__global__ void ed_scatter_kernel(const int* __restrict__ keys, int nx, int ny, int nz, long long n, Dev D, double res,
                                  const int* __restrict__ flag, const int* __restrict__ pos, unsigned long long* __restrict__ ok,
                                  unsigned* __restrict__ ov, float4* __restrict__ oc) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || !flag[i]) return;
  const int k[3] = {keys[(int)(i / ((long long)ny * nz))], keys[nx + (int)((i / nz) % ny)], keys[nx + ny + (int)(i % nz)]};
  const int b = find_brick(D, brick_key(k));
  const int p = pos[i] - 1;
  ok[p] = pack(k[0], k[1], k[2]);
  ov[p] = __float_as_uint(D.lo[(size_t)b * 512 + local_of(k)]);
  oc[p] = make_float4(centre_of(k[0], res), centre_of(k[1], res), centre_of(k[2], res), 1.0f);
}

// The extent: one block per brick in use; the smallest and largest known key per axis, one atomicMin / atomicMax per axis
// and block into mm (min x, y, z, then max x, y, z).
__global__ void __launch_bounds__(512) ed_bounds_kernel(Dev D, int* mm) {
  using Reduce = cub::BlockReduce<int, 512>;
  __shared__ typename Reduce::TempStorage tmp;
  const int b = blockIdx.x, t = threadIdx.x;
  const bool kn = (D.known[(size_t)b * 16 + (t >> 5)] >> (t & 31)) & 1u;
  int k[3];
  voxel_keys(D.bkey[b], t, k);
  for (int a = 0; a < 3; ++a) {
    const int lo = Reduce(tmp).Reduce(kn ? k[a] : INT_MAX, cub::Min());
    __syncthreads();
    const int hi = Reduce(tmp).Reduce(kn ? k[a] : -1, cub::Max());
    __syncthreads();
    if (t == 0 && hi >= 0) {
      atomicMin(&mm[a], lo);
      atomicMax(&mm[3 + a], hi);
    }
  }
}

int upload_counters(Map& m, cudaStream_t st) {
  std::memset(m.cnt_host.get(), 0, sizeof(Counters));
  m.cnt_host.get()->pool_n = m.pool_n;
  LSO_TRY(cudaMemcpyAsync(m.cnt_dev.get(), m.cnt_host.get(), sizeof(Counters), cudaMemcpyHostToDevice, st));
  return LS_OK;
}

int read_counters(Map& m, cudaStream_t st) {
  LSO_TRY(cudaMemcpyAsync(m.cnt_host.get(), m.cnt_dev.get(), sizeof(Counters), cudaMemcpyDeviceToHost, st));
  LSO_TRY(cudaStreamSynchronize(st));
  return LS_OK;
}

// A pool of `cap` bricks holding the first pool_n bricks of the old one; marks and touched flags start clear.  The old pool
// stays when an allocation fails.
int grow_pool(Map& m, int cap, cudaStream_t st) {
  Map q;
  const size_t c = (size_t)cap;
  cudaError_t e = q.lo.reserve(c * 512, c * 512);
  if (e == cudaSuccess) e = q.known.reserve(c * 16, c * 16);
  if (e == cudaSuccess) e = q.mfree.reserve(c * 16, c * 16);
  if (e == cudaSuccess) e = q.mocc.reserve(c * 16, c * 16);
  if (e == cudaSuccess) e = q.bkey.reserve(c, c);
  if (e == cudaSuccess) e = q.touched.reserve(c, c);
  if (e == cudaSuccess) e = q.tlist.reserve(c, c);
  const size_t n = (size_t)m.pool_n;
  if (e == cudaSuccess) e = cudaMemsetAsync(q.lo.get() + n * 512, 0, (c - n) * 512 * sizeof(float), st);
  if (e == cudaSuccess) e = cudaMemsetAsync(q.known.get() + n * 16, 0, (c - n) * 16 * sizeof(unsigned), st);
  if (e == cudaSuccess) e = cudaMemsetAsync(q.mfree.get(), 0, c * 16 * sizeof(unsigned), st);
  if (e == cudaSuccess) e = cudaMemsetAsync(q.mocc.get(), 0, c * 16 * sizeof(unsigned), st);
  if (e == cudaSuccess) e = cudaMemsetAsync(q.touched.get(), 0, c * sizeof(unsigned), st);
  if (e == cudaSuccess && n > 0) e = cudaMemcpyAsync(q.lo.get(), m.lo.get(), n * 512 * sizeof(float), cudaMemcpyDeviceToDevice,
                                                     st);
  if (e == cudaSuccess && n > 0)
    e = cudaMemcpyAsync(q.known.get(), m.known.get(), n * 16 * sizeof(unsigned), cudaMemcpyDeviceToDevice, st);
  if (e == cudaSuccess && n > 0)
    e = cudaMemcpyAsync(q.bkey.get(), m.bkey.get(), n * sizeof(unsigned long long), cudaMemcpyDeviceToDevice, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) return code(e);
  m.lo = std::move(q.lo), m.known = std::move(q.known), m.mfree = std::move(q.mfree), m.mocc = std::move(q.mocc);
  m.bkey = std::move(q.bkey), m.touched = std::move(q.touched), m.tlist = std::move(q.tlist);
  return LS_OK;
}

// A hash of at least `cap` slots (power of two) holding the n bricks of bkey (pool index = position) into keys / vals;
// doubles until the probe bound holds.  The map's own table is not touched.
int build_table(Map& m, const unsigned long long* bkey, int n, int cap, ls::Buffer<unsigned long long>& keys,
                ls::Buffer<int>& vals, cudaStream_t st, uint64_t* launches) {
  for (;; cap *= 2) {
    const size_t c = (size_t)cap;
    keys.reset(), vals.reset();
    cudaError_t e = keys.reserve(c, c);
    if (e == cudaSuccess) e = vals.reserve(c, c);
    if (e == cudaSuccess) e = cudaMemsetAsync(keys.get(), 0xff, c * sizeof(unsigned long long), st);
    if (e == cudaSuccess) e = cudaMemsetAsync(vals.get(), 0xff, c * sizeof(int), st);
    if (e == cudaSuccess) e = cudaMemsetAsync(&m.cnt_dev.get()->overflow, 0, sizeof(int), st);
    if (e == cudaSuccess && n > 0) {
      occ_rehash_kernel<<<(n + 255) / 256, 256, 0, st>>>(bkey, n, keys.get(), vals.get(), (unsigned)cap - 1u, m.cnt_dev.get());
      ++*launches;
      e = cudaGetLastError();
    }
    int overflow = 0;
    if (e == cudaSuccess) e = cudaMemcpyAsync(&overflow, &m.cnt_dev.get()->overflow, sizeof(int), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) {
      keys.reset(), vals.reset();
      return code(e);
    }
    if (!overflow) return LS_OK;
  }
}

// A hash of at least `cap` slots holding every pool brick.  The old table stays when an allocation fails.
int rebuild_table(Map& m, int cap, cudaStream_t st, uint64_t* launches) {
  ls::Buffer<unsigned long long> keys;
  ls::Buffer<int> vals;
  const int rc = build_table(m, m.bkey.get(), m.pool_n, cap, keys, vals, st, launches);
  if (rc) return rc;
  m.tab_keys = std::move(keys), m.tab_vals = std::move(vals);
  return LS_OK;
}

// The read's per-record scratch for n stream records of `bytes` payload bytes, grown all or nothing.
int reserve_read(Map& m, int n, size_t bytes, cudaStream_t st) {
  LSO_TRY(m.rd_cnt_dev.reserve(1, 1));
  LSO_TRY(m.rd_cnt_host.reserve(1, 1));
  if (bytes > m.rd_pay.capacity()) {
    LSO_TRY(cudaStreamSynchronize(st));
    LSO_TRY(m.rd_pay.reserve(bytes, bytes + bytes / 8));
  }
  if ((size_t)n + 1 <= m.rd_ex.capacity()) return LS_OK;
  LSO_TRY(cudaStreamSynchronize(st));
  const size_t c = (size_t)n + n / 8 + 1, blocks = c / kReadThreads + 1;
  size_t b1 = 0, b2 = 0;
  cudaError_t e;
  if ((e = m.rd_ex.reserve(c, c)) || (e = m.rd_tmp.reserve(c, c)) || (e = m.rd_par.reserve(c, c)) ||
      (e = m.rd_anc.reserve(c, c)) || (e = m.rd_bmin.reserve(blocks, blocks)) || (e = m.rd_slot.reserve(c, c)) ||
      (e = m.rd_depth.reserve(c, c)) || (e = m.rd_key.reserve(c, c)) || (e = m.rd_nb.reserve(c, c)) ||
      (e = m.rd_boff.reserve(c, c)) ||
      (e = cub::DeviceScan::InclusiveSum(nullptr, b1, m.rd_tmp.get(), m.rd_ex.get(), (int)c, st)) ||
      (e = cub::DeviceScan::ExclusiveSum(nullptr, b2, m.rd_nb.get(), m.rd_boff.get(), (int)c, st)) ||
      (e = m.rd_cub.reserve(std::max(b1, b2), std::max(b1, b2)))) {
    m.rd_ex.reset(), m.rd_tmp.reset(), m.rd_par.reset(), m.rd_anc.reset(), m.rd_bmin.reset(), m.rd_slot.reset();
    m.rd_depth.reset(), m.rd_key.reset(), m.rd_nb.reset(), m.rd_boff.reset(), m.rd_cub.reset();
    m.rd_cub_bytes = 0;
    return code(e);
  }
  m.rd_cub_bytes = std::max(b1, b2);
  return LS_OK;
}

int reserve_points(Map& m, int n, cudaStream_t st) {
  cudaError_t e;
  if ((size_t)n > m.ends.capacity()) {
    LSO_TRY(cudaStreamSynchronize(st));
    const size_t cap = (size_t)(n + n / 8);
    if ((e = m.ends.reserve(cap, cap)) || (e = m.pkey.reserve(cap, cap)) || (e = m.cls.reserve(cap, cap))) {
      m.ends.reset(), m.pkey.reset(), m.cls.reset();
      return code(e);
    }
  }
  size_t ep = 1024;
  while (ep < 2 * (size_t)n) ep *= 2;
  if (ep > m.ep_keys.capacity()) {
    LSO_TRY(cudaStreamSynchronize(st));
    if ((e = m.ep_keys.reserve(ep, ep)) || (e = m.ep_min.reserve(ep, ep))) {
      m.ep_keys.reset(), m.ep_min.reset();
      return code(e);
    }
  }
  return LS_OK;
}

int reserve_export(Map& m, long long n, cudaStream_t st) {
  if ((size_t)n <= m.ex_c.capacity()) return LS_OK;
  LSO_TRY(cudaStreamSynchronize(st));
  const long long cap = n + n / 8 + 1024;
  const size_t c = (size_t)cap;
  size_t bytes = 0;
  cudaError_t e;
  if ((e = m.ex_c.reserve(c, c)) || (e = m.ex_k[0].reserve(c, c)) || (e = m.ex_v[0].reserve(c, c)) ||
      (e = m.ex_k[1].reserve(c, c)) || (e = m.ex_v[1].reserve(c, c)) ||
      (e = cub::DeviceRadixSort::SortPairs(nullptr, bytes, m.ex_k[0].get(), m.ex_k[1].get(), m.ex_v[0].get(), m.ex_v[1].get(),
                                           (int)cap, 0, 48, st)) ||
      (e = m.cub_tmp.reserve(bytes, bytes))) {
    m.ex_c.reset(), m.ex_k[0].reset(), m.ex_v[0].reset(), m.ex_k[1].reset(), m.ex_v[1].reset(), m.cub_tmp.reset();
    m.cub_bytes = 0;
    return code(e);
  }
  m.cub_bytes = bytes;
  return LS_OK;
}

// the counting pass of the export: cnt->n_out (and, with keys, the unordered voxels)
int select(Map& m, const Params& P, int which, unsigned long long* keys, unsigned* vals, cudaStream_t st, uint64_t* launches) {
  int rc;
  if ((rc = upload_counters(m, st))) return rc;
  const long long nvox = (long long)m.pool_n * 512;
  if (nvox > 0) {
    long long blocks = (nvox + 255) / 256;
    if (blocks > 65536) blocks = 65536;
    occ_select_kernel<<<(int)blocks, 256, 0, st>>>(dev_of(m), P, which, nvox, keys, vals, m.cnt_dev.get());
    LSO_LAUNCHED();
  }
  return read_counters(m, st);
}

Nodes nodes_of(const Octree& t) {
  return Nodes{t.code.get(), t.pool.get(), t.first.get(), t.end.get(), t.st.get(), t.val.get(),
               {t.n_nodes.get(), t.n_leaves.get(), t.n_bytes.get()}, t.off.get(), t.loff.get()};
}

// Records for n_b bricks and every upper node they can have: at most min(n_b, 8^d) at depth d.
int reserve_tree(Octree& t, int n_b, cudaStream_t st) {
  LSO_TRY(t.levels.reserve(2 * (kBrickDepth + 1), 2 * (kBrickDepth + 1)));
  LSO_TRY(t.tot_dev.reserve(3, 3));
  LSO_TRY(t.tot_host.reserve(3, 3));
  if ((size_t)n_b <= t.pool.capacity()) return LS_OK;
  LSO_TRY(cudaStreamSynchronize(st));
  const int cap = n_b + n_b / 8;
  long long nodes = cap, level = 1;
  for (int d = 0; d < kBrickDepth; ++d, level *= 8) nodes += level < cap ? level : cap;
  const size_t n = (size_t)nodes, c = (size_t)cap;
  size_t bytes = 0;
  cudaError_t e;
  if ((e = t.pool.reserve(c, c)) || (e = t.code.reserve(n, n)) || (e = t.first.reserve(n, n)) || (e = t.end.reserve(n, n)) ||
      (e = t.st.reserve(n, n)) || (e = t.n_nodes.reserve(n, n)) || (e = t.n_bytes.reserve(n, n)) ||
      (e = t.n_leaves.reserve(n, n)) || (e = t.off.reserve(n, n)) || (e = t.loff.reserve(n, n)) ||
      (e = t.sort_k.reserve(c, c)) || (e = t.sort_v.reserve(c, c)) ||
      (e = cub::DeviceRadixSort::SortPairs(nullptr, bytes, t.sort_k.get(), t.code.get(), t.sort_v.get(), t.pool.get(), cap, 0,
                                           3 * kBrickDepth, st)) ||
      (e = t.cub_tmp.reserve(bytes, bytes))) {
    t.pool.reset(), t.code.reset(), t.first.reset(), t.end.reset(), t.st.reset(), t.n_nodes.reset(), t.n_bytes.reset();
    t.n_leaves.reset(), t.off.reset(), t.loff.reset(), t.sort_k.reset(), t.sort_v.reset(), t.cub_tmp.reset();
    t.cub_bytes = 0;
    return code(e);
  }
  t.cub_bytes = bytes;
  return LS_OK;
}

int reserve_tree_outputs(Octree& t, long long bytes, long long leaves, cudaStream_t st) {
  if ((size_t)bytes > t.payload.capacity()) {
    LSO_TRY(cudaStreamSynchronize(st));
    LSO_TRY(t.payload.reserve((size_t)bytes, (size_t)(bytes + bytes / 8)));
  }
  if ((size_t)leaves > t.centres.capacity()) {
    LSO_TRY(cudaStreamSynchronize(st));
    const size_t cap = (size_t)(leaves + leaves / 8);
    cudaError_t e;
    if ((e = t.centres.reserve(cap, cap)) || (e = t.depths.reserve(cap, cap))) {
      t.centres.reset(), t.depths.reset();
      return code(e);
    }
  }
  return LS_OK;
}

}  // namespace

int init(Map& m, int initial_bricks, cudaStream_t st) {
  m = Map();
  LSO_TRY(m.cnt_dev.reserve(1, 1));
  LSO_TRY(m.cnt_host.reserve(1, 1));
  int rc;
  if ((rc = grow_pool(m, initial_bricks, st))) return rc;
  int cap = 1024;
  while (cap < 2 * initial_bricks) cap *= 2;
  uint64_t launches = 0;
  return rebuild_table(m, cap, st, &launches);
}

size_t device_bytes(const Map& m) {
  const size_t pool = (size_t)m.pool_cap() * (512 * sizeof(float) + 48 * sizeof(unsigned) + sizeof(unsigned long long) +
                                              sizeof(unsigned) + sizeof(int));
  const size_t tab = (size_t)m.tab_cap() * (sizeof(unsigned long long) + sizeof(int));
  const size_t pts = m.ends.capacity() * (sizeof(float4) + sizeof(unsigned long long) + sizeof(int)) +
                     m.ep_keys.capacity() * (sizeof(unsigned long long) + sizeof(int));
  const size_t ex = m.ex_c.capacity() * (2 * sizeof(unsigned long long) + 2 * sizeof(unsigned) + sizeof(float4)) + m.cub_bytes;
  const size_t rd = m.rd_pay.capacity() + m.rd_ex.capacity() * (4 * sizeof(int) + 2 + sizeof(unsigned long long) +
                                                                2 * sizeof(long long)) +
                    m.rd_bmin.capacity() * sizeof(int) + m.rd_cub.capacity() +
                    m.rd_bkey.capacity() * (sizeof(unsigned long long) + 1) + m.rd_cnt_dev.capacity() * sizeof(ReadCounters);
  return pool + tab + pts + ex + m.qbuf.capacity() + sizeof(Counters) + rd;
}

int insert(Map& m, const Params& P, const float4* pts, int n, const float T[16], bool identity, cudaStream_t st, Counters* out,
           uint64_t* launches) {
  int rc;
  std::memset(out, 0, sizeof(Counters));
  if ((rc = reserve_points(m, n, st))) return rc;
  if (2LL * m.pool_n > m.tab_cap() && (rc = rebuild_table(m, m.tab_cap() * 2, st, launches))) return rc;
  if ((rc = upload_counters(m, st))) return rc;
  LSO_TRY(cudaMemsetAsync(m.ep_keys.get(), 0xff, m.ep_keys.capacity() * sizeof(unsigned long long), st));
  LSO_TRY(cudaMemsetAsync(m.ep_min.get(), 0x7f, m.ep_keys.capacity() * sizeof(int), st));  // 0x7f7f7f7f: above any point index
  Xform16 x;
  std::memcpy(x.T, T, sizeof(x.T));
  const int blocks = (n + 255) / 256;
  if (n > 0) {
    occ_classify_kernel<<<blocks, 256, 0, st>>>(pts, n, x, identity ? 1 : 0, P, m.ends.get(), m.pkey.get(), m.cls.get(),
                                                m.ep_keys.get(), m.ep_min.get(),
                                                 (unsigned)m.ep_keys.capacity() - 1u);
    LSO_LAUNCHED();
  }
  for (;;) {
    if (n > 0) {
      occ_cast_kernel<<<blocks, 256, 0, st>>>(n, P, T[12], T[13], T[14], m.ends.get(), m.pkey.get(), m.cls.get(), m.ep_keys.get(),
                                              m.ep_min.get(),
                                              (unsigned)m.ep_keys.capacity() - 1u, dev_of(m), m.cnt_dev.get());
      LSO_LAUNCHED();
    }
    if ((rc = read_counters(m, st))) return rc;
    const Counters c = *m.cnt_host.get();
    if (!c.overflow) break;
    // Undo the marking: clear every mark and touched flag, keep the bricks that got a pool index, drop the rest from the
    // hash, grow what filled and mark again.
    m.pool_n = c.pool_n < m.pool_cap() ? c.pool_n : m.pool_cap();
    LSO_TRY(cudaMemsetAsync(m.mfree.get(), 0, (size_t)m.pool_cap() * 16 * sizeof(unsigned), st));
    LSO_TRY(cudaMemsetAsync(m.mocc.get(), 0, (size_t)m.pool_cap() * 16 * sizeof(unsigned), st));
    LSO_TRY(cudaMemsetAsync(m.touched.get(), 0, (size_t)m.pool_cap() * sizeof(unsigned), st));
    int tab = m.tab_cap();
    if ((c.overflow & kOverflowTable) || 2LL * m.pool_n > tab) tab *= 2;
    if ((rc = rebuild_table(m, tab, st, launches))) return rc;
    if ((c.overflow & kOverflowPool) && (rc = grow_pool(m, m.pool_cap() * 2, st))) return rc;
    if ((rc = upload_counters(m, st))) return rc;
  }
  m.pool_n = m.cnt_host.get()->pool_n;
  if (m.cnt_host.get()->n_touched > 0) {
    occ_update_kernel<<<m.cnt_host.get()->n_touched, 512, 0, st>>>(dev_of(m), P, m.cnt_dev.get());
    LSO_LAUNCHED();
    if ((rc = read_counters(m, st))) return rc;
  }
  m.n_known += (long long)m.cnt_host.get()->new_known;
  *out = *m.cnt_host.get();
  return LS_OK;
}

int count(Map& m, const Params& P, int which, long long* n, cudaStream_t st, uint64_t* launches) {
  if (which == LS_OCC_KNOWN) {
    *n = m.n_known;
    return LS_OK;
  }
  int rc;
  if ((rc = select(m, P, which, nullptr, nullptr, st, launches))) return rc;
  *n = (long long)m.cnt_host.get()->n_out;
  return LS_OK;
}

int download(Map& m, const Params& P, int which, long long n, uint64_t* keys, float* log_odds, float* centres4, cudaStream_t st,
             uint64_t* launches) {
  if (n <= 0) return LS_OK;
  if (n > 0x7fffffffLL) return LS_ERR_NOMEM;
  int rc;
  if ((rc = reserve_export(m, n, st))) return rc;
  if ((rc = select(m, P, which, m.ex_k[0].get(), m.ex_v[0].get(), st, launches))) return rc;
  if ((long long)m.cnt_host.get()->n_out != n) return LS_ERR_CUDA;
  size_t bytes = m.cub_bytes;
  LSO_TRY(cub::DeviceRadixSort::SortPairs(m.cub_tmp.get(), bytes, m.ex_k[0].get(), m.ex_k[1].get(), m.ex_v[0].get(),
                                          m.ex_v[1].get(), (int)n, 0, 48, st));
  ++*launches;
  if (centres4) {
    long long blocks = (n + 255) / 256;
    if (blocks > 65536) blocks = 65536;
    occ_centres_kernel<<<(int)blocks, 256, 0, st>>>(m.ex_k[1].get(), n, P.res, m.ex_c.get());
    LSO_LAUNCHED();
    LSO_TRY(cudaMemcpyAsync(centres4, m.ex_c.get(), (size_t)n * sizeof(float4), cudaMemcpyDeviceToHost, st));
  }
  if (keys) LSO_TRY(cudaMemcpyAsync(keys, m.ex_k[1].get(), (size_t)n * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  if (log_odds) LSO_TRY(cudaMemcpyAsync(log_odds, m.ex_v[1].get(), (size_t)n * sizeof(float), cudaMemcpyDeviceToHost, st));
  LSO_TRY(cudaStreamSynchronize(st));
  return LS_OK;
}

int download_octree(const Octree& t, unsigned char* payload, float* centres4, unsigned char* depths, cudaStream_t st) {
  if (t.bytes > 0 && payload) LSO_TRY(cudaMemcpyAsync(payload, t.payload.get(), (size_t)t.bytes, cudaMemcpyDeviceToHost, st));
  if (t.leaves > 0 && centres4)
    LSO_TRY(cudaMemcpyAsync(centres4, t.centres.get(), (size_t)t.leaves * sizeof(float4), cudaMemcpyDeviceToHost, st));
  if (t.leaves > 0 && depths) LSO_TRY(cudaMemcpyAsync(depths, t.depths.get(), (size_t)t.leaves, cudaMemcpyDeviceToHost, st));
  LSO_TRY(cudaStreamSynchronize(st));
  return LS_OK;
}

namespace {

// The tail of a read whose stream is valid and numbers n_b new bricks: `keys` writes their keys and states to rd_bkey /
// rd_bst, the pool grows and the new hash is built beside the old one, so the map is unchanged if any of that fails; only
// then does `fill` write the new bricks (n_b > 0), and the map takes the new hash, n_b bricks and `known` voxels.
int replace_map(Map& m, int n_b, long long known, const std::function<int()>& keys, const std::function<int(const Dev&)>& fill,
                const char** why, cudaStream_t st, uint64_t* launches) {
  const char* nomem = "the map cannot grow";
  int rc;
  if (n_b > 0) {
    cudaError_t e = m.rd_bkey.capacity() >= (size_t)n_b ? cudaSuccess : m.rd_bkey.reserve(n_b, n_b + n_b / 8);
    if (e == cudaSuccess && m.rd_bst.capacity() < (size_t)n_b) e = m.rd_bst.reserve(n_b, n_b + n_b / 8);
    if (e != cudaSuccess) {
      m.rd_bkey.reset(), m.rd_bst.reset();
      return *why = nomem, code(e);
    }
    if ((rc = keys())) return rc;
  }
  if (n_b > m.pool_cap()) {
    long long cap = m.pool_cap() > 0 ? m.pool_cap() : 1;
    while (cap < n_b) cap *= 2;
    if ((rc = grow_pool(m, (int)cap, st))) return *why = nomem, rc;
  }
  int tab = 1024;
  while (tab < 2 * n_b) tab *= 2;
  ls::Buffer<unsigned long long> tkeys;
  ls::Buffer<int> tvals;
  if ((rc = build_table(m, m.rd_bkey.get(), n_b, tab, tkeys, tvals, st, launches))) return *why = nomem, rc;
  // Only now is the map written.
  if (n_b > 0 && (rc = fill(dev_of(m)))) return rc;
  if (m.pool_n > n_b) {  // bricks past the new pool start empty, as a grown pool's do
    const size_t a = (size_t)n_b, k = (size_t)(m.pool_n - n_b);
    LSO_TRY(cudaMemsetAsync(m.lo.get() + a * 512, 0, k * 512 * sizeof(float), st));
    LSO_TRY(cudaMemsetAsync(m.known.get() + a * 16, 0, k * 16 * sizeof(unsigned), st));
    LSO_TRY(cudaMemsetAsync(m.mfree.get() + a * 16, 0, k * 16 * sizeof(unsigned), st));
    LSO_TRY(cudaMemsetAsync(m.mocc.get() + a * 16, 0, k * 16 * sizeof(unsigned), st));
    LSO_TRY(cudaMemsetAsync(m.touched.get() + a, 0, k * sizeof(unsigned), st));
  }
  LSO_TRY(cudaStreamSynchronize(st));
  m.tab_keys = std::move(tkeys), m.tab_vals = std::move(tvals);
  m.pool_n = n_b;
  m.n_known = known;
  return LS_OK;
}

template <class F>
int build_tree_as(const Map& m, const Params& P, Octree& t, cudaStream_t st, uint64_t* launches) {
  t.nodes = t.bytes = t.leaves = 0;
  t.bricks = 0;
  const int n_b = m.pool_n;
  if (n_b == 0) return LS_OK;
  int rc;
  if ((rc = reserve_tree(t, n_b, st))) return rc;
  if (F::kValued && t.val.capacity() < t.code.capacity()) {
    LSO_TRY(cudaStreamSynchronize(st));
    t.val.reset();
    LSO_TRY(t.val.reserve(t.code.capacity(), t.code.capacity()));
  }
  const Nodes N = nodes_of(t);
  oct_code_kernel<<<(n_b + 255) / 256, 256, 0, st>>>(m.bkey.get(), n_b, t.sort_k.get(), t.sort_v.get());
  LSO_LAUNCHED();
  size_t bytes = t.cub_bytes;
  LSO_TRY(cub::DeviceRadixSort::SortPairs(t.cub_tmp.get(), bytes, t.sort_k.get(), t.code.get(), t.sort_v.get(), t.pool.get(), n_b,
                                          0, 3 * kBrickDepth, st));
  ++*launches;
  oct_brick_kernel<F><<<n_b, 512, 0, st>>>(m.known.get(), m.lo.get(), N, P.l_occ);
  LSO_LAUNCHED();
  oct_up_kernel<F><<<1, kTreeThreads, 0, st>>>(N, n_b, t.levels.get(), t.tot_dev.get());
  LSO_LAUNCHED();
  LSO_TRY(cudaMemcpyAsync(t.tot_host.get(), t.tot_dev.get(), F::kTotals * sizeof(unsigned long long), cudaMemcpyDeviceToHost,
                          st));
  LSO_TRY(cudaStreamSynchronize(st));
  const unsigned long long* tot = t.tot_host.get();
  const long long nodes = (long long)tot[0], leaves = (long long)tot[1], pay = F::payload_bytes(tot);
  if (nodes == 0) return LS_OK;
  if ((rc = reserve_tree_outputs(t, pay, F::kCentres ? leaves : 0, st))) return rc;
  oct_down_kernel<F><<<1, kTreeThreads, 0, st>>>(N, t.levels.get(), P.res, t.payload.get(), t.centres.get(), t.depths.get());
  LSO_LAUNCHED();
  oct_emit_kernel<F><<<n_b, 512, 0, st>>>(m.known.get(), m.lo.get(), m.bkey.get(), N, P.l_occ, P.res, t.payload.get(),
                                          t.centres.get(), t.depths.get());
  LSO_LAUNCHED();
  LSO_TRY(cudaStreamSynchronize(st));
  t.nodes = nodes, t.bytes = pay, t.leaves = leaves;
  t.bricks = n_b;
  return LS_OK;
}

template <class F>
int read_tree_as(Map& m, const Params& P, const unsigned char* payload, long long bytes, long long nodes, ReadCounters* out,
                 const char** why, cudaStream_t st, uint64_t* launches) {
  std::memset(out, 0, sizeof(ReadCounters));
  *why = "";
  int rc, n_b = 0, end = 0;
  // A valid tree has at most `nodes` stream nodes, so later records cannot belong to it.
  const long long count = nodes > 0 ? std::min(bytes / F::kNodeBytes, nodes) : 0;
  if (nodes > 0 && count == 0) return *why = "the payload is truncated", LS_ERR_ARG;
  if (count > kMaxReadPairs) return *why = F::kTooMany, LS_ERR_NOMEM;
  if (count > 0) {
    const int n = (int)count;
    const size_t pay = (size_t)F::kNodeBytes * n;
    if ((rc = reserve_read(m, n, pay, st))) return *why = "out of device memory for the parse", rc;
    ReadCounters* cnt = m.rd_cnt_dev.get();
    ReadCounters init{};
    init.end = INT_MAX;
    *m.rd_cnt_host.get() = init;
    LSO_TRY(cudaMemcpyAsync(cnt, m.rd_cnt_host.get(), sizeof(ReadCounters), cudaMemcpyHostToDevice, st));
    LSO_TRY(cudaMemcpyAsync(m.rd_pay.get(), payload, pay, cudaMemcpyHostToDevice, st));
    const int blocks = (n + kReadThreads) / kReadThreads;  // n + 1 items
    rd_excess_kernel<F><<<blocks, kReadThreads, 0, st>>>(m.rd_pay.get(), n, m.rd_tmp.get());
    LSO_LAUNCHED();
    size_t tb = m.rd_cub_bytes;
    LSO_TRY(cub::DeviceScan::InclusiveSum(m.rd_cub.get(), tb, m.rd_tmp.get(), m.rd_ex.get(), n + 1, st));
    ++*launches;
    rd_end_kernel<<<blocks, kReadThreads, 0, st>>>(m.rd_ex.get(), n, m.rd_bmin.get(), cnt);
    LSO_LAUNCHED();
    rd_parent_kernel<F><<<blocks, kReadThreads, 0, st>>>(m.rd_pay.get(), m.rd_ex.get(), m.rd_bmin.get(), n, m.rd_par.get(),
                                                         m.rd_slot.get(), cnt);
    LSO_LAUNCHED();
    rd_node_kernel<F><<<blocks, kReadThreads, 0, st>>>(m.rd_pay.get(), m.rd_par.get(), m.rd_slot.get(), n, P.l_occ,
                                                       m.rd_depth.get(), m.rd_key.get(), m.rd_anc.get(), m.rd_nb.get(), cnt);
    LSO_LAUNCHED();
    tb = m.rd_cub_bytes;
    LSO_TRY(cub::DeviceScan::ExclusiveSum(m.rd_cub.get(), tb, m.rd_nb.get(), m.rd_boff.get(), n + 1, st));
    ++*launches;
    LSO_TRY(cudaMemcpyAsync(&cnt->bricks, m.rd_boff.get() + n, sizeof(long long), cudaMemcpyDeviceToDevice, st));
    LSO_TRY(cudaMemcpyAsync(m.rd_cnt_host.get(), cnt, sizeof(ReadCounters), cudaMemcpyDeviceToHost, st));
    LSO_TRY(cudaStreamSynchronize(st));
    const ReadCounters c = *m.rd_cnt_host.get();
    if ((rc = F::check(c, count, nodes, why))) return rc;
    if (c.bricks > kMaxReadBricks) return *why = "the file covers more bricks than the map can index", LS_ERR_NOMEM;
    *out = c;
    F::counts(out);
    end = c.end;
    n_b = (int)c.bricks;
  }
  return replace_map(
      m, n_b, (long long)out->known,
      [&]() -> int {
        rd_brick_kernel<F><<<(n_b + 255) / 256, 256, 0, st>>>(m.rd_pay.get(), m.rd_depth.get(), m.rd_key.get(),
                                                              m.rd_boff.get(), end, n_b, m.rd_bkey.get(), m.rd_bst.get());
        LSO_LAUNCHED();
        return LS_OK;
      },
      [&](const Dev& D) -> int {
        rd_fill_kernel<F><<<n_b, 512, 0, st>>>(D, P, m.rd_pay.get(), m.rd_boff.get(), end, m.rd_bkey.get(), m.rd_bst.get());
        LSO_LAUNCHED();
        rd_leaf_kernel<F><<<(end + 255) / 256, 256, 0, st>>>(D, P, m.rd_pay.get(), m.rd_depth.get(), m.rd_key.get(),
                                                             m.rd_anc.get(), m.rd_boff.get(), end);
        LSO_LAUNCHED();
        return LS_OK;
      },
      why, st, launches);
}

}  // namespace

int build_tree(const Map& m, const Params& P, TreeFormat f, Octree& t, cudaStream_t st, uint64_t* launches) {
  return f == TreeFormat::Full ? build_tree_as<FullTree>(m, P, t, st, launches) : build_tree_as<BinaryTree>(m, P, t, st, launches);
}

int read_tree(Map& m, const Params& P, TreeFormat f, const unsigned char* payload, long long bytes, long long nodes,
              ReadCounters* out, const char** why, cudaStream_t st, uint64_t* launches) {
  return f == TreeFormat::Full ? read_tree_as<FullTree>(m, P, payload, bytes, nodes, out, why, st, launches)
                               : read_tree_as<BinaryTree>(m, P, payload, bytes, nodes, out, why, st, launches);
}

// ---- leaf lists ----------------------------------------------------------------------------------------------------------
namespace {

// Every buffer of a list of n leaves, all or nothing.
int reserve_leaves(Leaves& L, long long n, cudaStream_t st) {
  LSO_TRY(L.cnt_dev.reserve(kLeafBuckets, kLeafBuckets));
  LSO_TRY(L.cnt_host.reserve(kLeafBuckets, kLeafBuckets));
  if ((size_t)n <= L.raw_c.capacity()) return LS_OK;
  if (n > (1LL << 30)) return LS_ERR_NOMEM;  // CUB's item counts are int
  LSO_TRY(cudaStreamSynchronize(st));
  const size_t c = (size_t)(n + n / 8);
  size_t scan = 0, sort = 0;
  cudaError_t e;
  if ((e = L.raw_c.reserve(c, c)) || (e = L.cen.reserve(c, c)) || (e = L.rgba.reserve(c, c)) || (e = L.raw_tag.reserve(c, c)) ||
      (e = L.tag.reserve(c, c)) || (e = L.stag.reserve(c, c)) || (e = L.keep.reserve(c, c)) || (e = L.pos.reserve(c, c)) ||
      (e = L.idx.reserve(c, c)) || (e = L.sorted.reserve(c, c)) ||
      (e = cub::DeviceScan::ExclusiveSum(nullptr, scan, L.keep.get(), L.pos.get(), (int)c, st)) ||
      (e = cub::DeviceRadixSort::SortPairs(nullptr, sort, L.tag.get(), L.stag.get(), L.idx.get(), L.sorted.get(), (int)c, 0, 6,
                                           st)) ||
      (e = L.cub_tmp.reserve(std::max(scan, sort), std::max(scan, sort)))) {
    L.raw_c.reset(), L.cen.reset(), L.rgba.reset(), L.raw_tag.reset(), L.tag.reset(), L.stag.reset(), L.keep.reset();
    L.pos.reset(), L.idx.reset(), L.sorted.reset(), L.cub_tmp.reset();
    L.cub_bytes = 0;
    return code(e);
  }
  L.cub_bytes = std::max(scan, sort);
  return LS_OK;
}

int grid_of(long long n) { return (int)std::min<long long>((n + 255) / 256, 4096); }

// The list's positions stably sorted by tag bits [begin, 6) into L.sorted (tags into L.stag).
int sort_leaves(Leaves& L, int begin, cudaStream_t st, uint64_t* launches) {
  size_t bytes = L.cub_bytes;
  LSO_TRY(cub::DeviceRadixSort::SortPairs(L.cub_tmp.get(), bytes, L.tag.get(), L.stag.get(), L.idx.get(), L.sorted.get(),
                                          (int)L.n, begin, 6, st));
  ++*launches;
  return LS_OK;
}

// Entries [first, first + n) of L.sorted gathered into raw_c / raw_tag (the first n_col with colours), then copied out.
int gather_leaves(Leaves& L, long long first, long long n, long long n_col, double min_z, double max_z, double color_factor,
                  float* centres4, unsigned char* tags, float* rgba4, cudaStream_t st, uint64_t* launches) {
  if (n > 0) {
    lv_gather_kernel<<<grid_of(n), 256, 0, st>>>(L.cen.get(), L.tag.get(), L.sorted.get(), first, n, n_col, min_z, max_z,
                                                 color_factor, L.raw_c.get(), L.raw_tag.get(), L.rgba.get());
    LSO_LAUNCHED();
    if (centres4) LSO_TRY(cudaMemcpyAsync(centres4, L.raw_c.get(), (size_t)n * sizeof(float4), cudaMemcpyDeviceToHost, st));
    if (tags) LSO_TRY(cudaMemcpyAsync(tags, L.raw_tag.get(), (size_t)n, cudaMemcpyDeviceToHost, st));
    if (rgba4 && n_col > 0)
      LSO_TRY(cudaMemcpyAsync(rgba4, L.rgba.get(), (size_t)n_col * sizeof(float4), cudaMemcpyDeviceToHost, st));
  }
  LSO_TRY(cudaStreamSynchronize(st));
  return LS_OK;
}

}  // namespace

int build_leaves(const Map& m, const Params& P, Octree& t, const int kmin[3], const int kmax[3], Leaves& L, cudaStream_t st,
                 uint64_t* launches) {
  L.n = L.n_occupied = 0;
  std::fill(L.occupied, L.occupied + 17, 0LL), std::fill(L.free, L.free + 17, 0LL);
  const long long nl = t.leaves;
  if (nl == 0) return LS_OK;
  int rc;
  if ((rc = reserve_leaves(L, nl, st))) return rc;
  const KeyRange R{{kmin[0], kmin[1], kmin[2]}, {kmax[0], kmax[1], kmax[2]}};
  const Nodes N = nodes_of(t);
  const BoxOut out{P.l_occ, P.res, R, L.raw_c.get(), L.raw_tag.get(), L.keep.get()};
  lv_down_kernel<FullTree><<<1, kTreeThreads, 0, st>>>(N, t.levels.get(), out);
  LSO_LAUNCHED();
  lv_emit_kernel<FullTree><<<t.bricks, 512, 0, st>>>(m.known.get(), m.lo.get(), m.bkey.get(), N, P.l_occ, out);
  LSO_LAUNCHED();
  size_t bytes = L.cub_bytes;
  LSO_TRY(cub::DeviceScan::ExclusiveSum(L.cub_tmp.get(), bytes, L.keep.get(), L.pos.get(), (int)nl, st));
  ++*launches;
  LSO_TRY(cudaMemsetAsync(L.cnt_dev.get(), 0, kLeafBuckets * sizeof(unsigned long long), st));
  lv_compact_kernel<<<grid_of(nl), 256, 0, st>>>(L.raw_c.get(), L.raw_tag.get(), L.keep.get(), L.pos.get(), (int)nl,
                                                 L.cen.get(), L.tag.get(), L.idx.get(), L.cnt_dev.get());
  LSO_LAUNCHED();
  LSO_TRY(cudaMemcpyAsync(L.cnt_host.get(), L.cnt_dev.get(), kLeafBuckets * sizeof(unsigned long long), cudaMemcpyDeviceToHost,
                          st));
  LSO_TRY(cudaStreamSynchronize(st));
  for (int d = 0; d < 17; ++d) {
    L.occupied[d] = (long long)L.cnt_host.get()[d], L.free[d] = (long long)L.cnt_host.get()[17 + d];
    L.n_occupied += L.occupied[d], L.n += L.occupied[d] + L.free[d];
  }
  return LS_OK;
}

int tree_leaf_records(const Map& m, const Params& P, Octree& t, unsigned long long* rec, cudaStream_t st, uint64_t* launches) {
  if (t.nodes == 0) return LS_OK;
  const Nodes N = nodes_of(t);
  const KeyOut out{rec};
  lv_down_kernel<BinaryTree><<<1, kTreeThreads, 0, st>>>(N, t.levels.get(), out);
  LSO_LAUNCHED();
  lv_emit_kernel<BinaryTree><<<t.bricks, 512, 0, st>>>(m.known.get(), m.lo.get(), m.bkey.get(), N, P.l_occ, out);
  LSO_LAUNCHED();
  return LS_OK;
}

int download_leaves(Leaves& L, int which, float* centres4, unsigned char* tags, cudaStream_t st, uint64_t* launches) {
  if (L.n == 0) return LS_OK;
  if (which == 3) {
    if (centres4) LSO_TRY(cudaMemcpyAsync(centres4, L.cen.get(), (size_t)L.n * sizeof(float4), cudaMemcpyDeviceToHost, st));
    if (tags) LSO_TRY(cudaMemcpyAsync(tags, L.tag.get(), (size_t)L.n, cudaMemcpyDeviceToHost, st));
    LSO_TRY(cudaStreamSynchronize(st));
    return LS_OK;
  }
  int rc;
  if ((rc = sort_leaves(L, 5, st, launches))) return rc;
  const long long n_occ = L.n_occupied;
  return which == 2 ? gather_leaves(L, 0, n_occ, 0, 0.0, 1.0, 0.0, centres4, tags, nullptr, st, launches)
                    : gather_leaves(L, n_occ, L.n - n_occ, 0, 0.0, 1.0, 0.0, centres4, tags, nullptr, st, launches);
}

int marker_cubes(Leaves& L, double min_z, double max_z, double color_factor, float* centres4, float* rgba4, cudaStream_t st,
                 uint64_t* launches) {
  if (L.n == 0) return LS_OK;
  int rc;
  if ((rc = sort_leaves(L, 0, st, launches))) return rc;
  return gather_leaves(L, 0, L.n, L.n_occupied, min_z, max_z, color_factor, centres4, nullptr, rgba4, st, launches);
}

namespace {

int zero_visited(Map& m, cudaStream_t st) {
  LSO_TRY(cudaMemsetAsync(&m.cnt_dev.get()->n_out, 0, sizeof(unsigned long long), st));
  return LS_OK;
}

// The outputs' copies are queued; wait for them and the keys visited.
int finish_query(Map& m, cudaStream_t st, long long* visited) {
  LSO_TRY(cudaMemcpyAsync(&m.cnt_host.get()->n_out, &m.cnt_dev.get()->n_out, sizeof(unsigned long long), cudaMemcpyDeviceToHost,
                          st));
  LSO_TRY(cudaStreamSynchronize(st));
  *visited = (long long)m.cnt_host.get()->n_out;
  return LS_OK;
}

// One axis of getLineStatusBoundingBox's offset loop (at most cap values); false when it has more.
bool box_axis(double size, double res, long long cap, std::vector<double>* out) {
  out->clear();
  const double parts = std::ceil((size + 0.001) / res);
  if (!(parts <= (double)cap + 2.0)) return false;  // the loop below runs about parts + 1 times
  double disc = size / parts;
  if (disc <= 0.0) disc = 1.0;
  const double half = size * 0.5;
  for (double x = -half; x <= half; x += disc) {
    if ((long long)out->size() >= cap) return false;
    out->push_back(x);
  }
  return true;
}

}  // namespace

int query_cells(Map& m, const Params& P, const double* pts3, int n, int8_t* status, float* log_odds, long long* visited,
                cudaStream_t st, uint64_t* launches) {
  *visited = 0;
  if (n <= 0) return LS_OK;
  size_t off = 0;
  const size_t o_in = take(off, (size_t)n * 3 * sizeof(double)), o_st = take(off, (size_t)n),
               o_lo = take(off, (size_t)n * sizeof(float));
  int rc;
  if ((rc = reserve_staging(m, off, 0, st))) return rc;
  char* q = m.qbuf.get();
  LSO_TRY(cudaMemcpyAsync(q + o_in, pts3, (size_t)n * 3 * sizeof(double), cudaMemcpyHostToDevice, st));
  if ((rc = zero_visited(m, st))) return rc;
  occ_cell_kernel<<<blocks(n, 256), 256, 0, st>>>((const double*)(q + o_in), n, dev_of(m), P, (signed char*)(q + o_st),
                                                (float*)(q + o_lo), m.cnt_dev.get());
  LSO_LAUNCHED();
  LSO_TRY(cudaMemcpyAsync(status, q + o_st, (size_t)n, cudaMemcpyDeviceToHost, st));
  if (log_odds) LSO_TRY(cudaMemcpyAsync(log_odds, q + o_lo, (size_t)n * sizeof(float), cudaMemcpyDeviceToHost, st));
  return finish_query(m, st, visited);
}

int query_lines(Map& m, const Params& P, const double* starts3, const double* ends3, int n, const double* box3,
                int stop_at_unknown, int8_t* status, uint64_t* first_keys, long long* visited, cudaStream_t st,
                uint64_t* launches) {
  *visited = 0;
  if (n <= 0) return LS_OK;
  const long long kMaxLines = 0x7fffffffLL;
  std::vector<double> axes[3];
  long long lines = 1;
  if (box3) {
    for (int a = 0; a < 3; ++a) {
      if (!box_axis(box3[a], P.res, kMaxLines / n, &axes[a])) return LS_ERR_ARG;
      lines *= (long long)axes[a].size();
      if (lines * n > kMaxLines) return LS_ERR_ARG;
    }
  }
  const int nx = box3 ? (int)axes[0].size() : 1, ny = box3 ? (int)axes[1].size() : 1, nz = box3 ? (int)axes[2].size() : 1;
  const size_t seg_bytes = (size_t)n * 3 * sizeof(double);
  size_t off = 0;
  const size_t o_s = take(off, seg_bytes), o_e = take(off, seg_bytes), o_off = take(off, (size_t)(nx + ny + nz) * sizeof(double)),
               o_st = take(off, (size_t)n), o_fk = take(off, (size_t)n * sizeof(uint64_t)),
               o_best = take(off, (size_t)n * sizeof(unsigned));
  int rc;
  if ((rc = reserve_staging(m, off, 0, st))) return rc;
  char* q = m.qbuf.get();
  const double* s = (const double*)(q + o_s);
  const double* e = (const double*)(q + o_e);
  double* offs = (double*)(q + o_off);
  signed char* dst = (signed char*)(q + o_st);
  unsigned long long* dfk = (unsigned long long*)(q + o_fk);
  unsigned* best = (unsigned*)(q + o_best);
  LSO_TRY(cudaMemcpyAsync(q + o_s, starts3, seg_bytes, cudaMemcpyHostToDevice, st));
  LSO_TRY(cudaMemcpyAsync(q + o_e, ends3, seg_bytes, cudaMemcpyHostToDevice, st));
  if ((rc = zero_visited(m, st))) return rc;
  if (!box3) {
    occ_line_kernel<false><<<blocks(n, 256), 256, 0, st>>>(s, e, n, 1, nullptr, 1, 1, 1, stop_at_unknown, dev_of(m), P, dst, dfk,
                                                         nullptr, m.cnt_dev.get());
    LSO_LAUNCHED();
  } else {
    std::vector<double> flat;
    for (int a = 0; a < 3; ++a) flat.insert(flat.end(), axes[a].begin(), axes[a].end());
    LSO_TRY(cudaMemcpyAsync(offs, flat.data(), flat.size() * sizeof(double), cudaMemcpyHostToDevice, st));
    LSO_TRY(cudaMemsetAsync(best, 0, (size_t)n * sizeof(unsigned), st));  // 0: no line failed
    const long long items = lines * n;
    occ_line_kernel<true><<<blocks(items, 256), 256, 0, st>>>(s, e, items, (int)lines, offs, nx, ny, nz, stop_at_unknown,
                                                            dev_of(m), P, dst, dfk, best, m.cnt_dev.get());
    LSO_LAUNCHED();
    occ_box_result_kernel<<<blocks(n, 256), 256, 0, st>>>(s, e, n, (int)lines, offs, nx, ny, nz, stop_at_unknown, dev_of(m), P,
                                                         best, dst, dfk, m.cnt_dev.get());
    LSO_LAUNCHED();
    // the pageable copy of `flat` is staged before cudaMemcpyAsync returns, so it may go out of scope here
  }
  LSO_TRY(cudaMemcpyAsync(status, dst, (size_t)n, cudaMemcpyDeviceToHost, st));
  if (first_keys) LSO_TRY(cudaMemcpyAsync(first_keys, dfk, (size_t)n * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
  return finish_query(m, st, visited);
}

int query_rays(Map& m, const Params& P, const float* origins3, const float* directions3, int n, int ignore_unknown,
               double max_range, int8_t* result, float* ends3, long long* visited, cudaStream_t st, uint64_t* launches) {
  *visited = 0;
  if (n <= 0) return LS_OK;
  const size_t vec_bytes = (size_t)n * 3 * sizeof(float);
  size_t off = 0;
  const size_t o_o = take(off, vec_bytes), o_d = take(off, vec_bytes), o_r = take(off, (size_t)n), o_e = take(off, vec_bytes);
  int rc;
  if ((rc = reserve_staging(m, off, 0, st))) return rc;
  char* q = m.qbuf.get();
  LSO_TRY(cudaMemcpyAsync(q + o_o, origins3, vec_bytes, cudaMemcpyHostToDevice, st));
  LSO_TRY(cudaMemcpyAsync(q + o_d, directions3, vec_bytes, cudaMemcpyHostToDevice, st));
  if ((rc = zero_visited(m, st))) return rc;
  occ_ray_kernel<<<blocks(n, 256), 256, 0, st>>>((const float*)(q + o_o), (const float*)(q + o_d), n, ignore_unknown, max_range,
                                               dev_of(m), P, (signed char*)(q + o_r), (float*)(q + o_e), m.cnt_dev.get());
  LSO_LAUNCHED();
  LSO_TRY(cudaMemcpyAsync(result, q + o_r, (size_t)n, cudaMemcpyDeviceToHost, st));
  if (ends3) LSO_TRY(cudaMemcpyAsync(ends3, q + o_e, vec_bytes, cudaMemcpyDeviceToHost, st));
  return finish_query(m, st, visited);
}

// ---- edits -------------------------------------------------------------------------------------------------------------
namespace {

// One axis of setLogOddsBoundingBox's loop around p of size s: the keys of its points whose key is valid, in loop order
// (ascending, repeats kept).  False when the axis has more than kMaxEditAxis points.
bool edit_axis(double p, double s, const Params& P, std::vector<int>* keys) {
  keys->clear();
  const double c = P.res * std::floor(p / P.res) + P.res / 2.0;
  const double lo = (c - s / 2) + 0.001, hi = (c + s / 2) - 0.001;
  if (!((hi - lo) / P.res <= (double)kMaxEditAxis)) return false;  // bounds the loop below; a NaN is refused too
  long long points = 0;
  for (double x = lo; x <= hi; x += P.res) {
    if (++points > kMaxEditAxis) return false;
    int k;
    if (key_of(P.inv, (float)x, k)) keys->push_back(k);
  }
  return true;
}

// The bricks of one axis's keys appended to out: brick index << 8 | the mask of its keys (keys ascending, so each brick
// is one run).  Returns their number.
int axis_bricks(const std::vector<int>& keys, std::vector<unsigned>* out) {
  const size_t first = out->size();
  for (const int k : keys) {
    const unsigned b = (unsigned)(k >> 3) << 8, bit = 1u << (k & 7);
    if (out->size() > first && (out->back() & ~0xffu) == b) out->back() |= bit;
    else out->push_back(b | bit);
  }
  return (int)(out->size() - first);
}

}  // namespace

int set_boxes(Map& m, const Params& P, const double* centres3, const double* sizes3, const int8_t* occupied, int n,
              long long* voxels_set, long long* new_known, const char** why, cudaStream_t st, uint64_t* launches) {
  *voxels_set = *new_known = 0;
  *why = "";
  // Every box's loop first, on the host: nothing is allocated or written before the whole call is known to be valid.
  std::vector<EditBox> boxes((size_t)n);
  std::vector<unsigned> axes;
  std::vector<int> keys;
  long long items = 0, set = 0;
  for (int i = 0; i < n; ++i) {
    EditBox& B = boxes[(size_t)i];
    long long pts = 1, bricks = 1;
    for (int a = 0; a < 3; ++a) {
      if (!edit_axis(centres3[3 * (size_t)i + a], sizes3[3 * (size_t)i + a], P, &keys))
        return *why = "a box axis has more than 2^17 loop points", LS_ERR_ARG;
      B.off[a] = (int)axes.size();
      B.n[a] = axis_bricks(keys, &axes);
      pts *= (long long)keys.size();
      bricks *= B.n[a];
    }
    B.item0 = items;
    items += bricks;
    set += pts;
    if (items + m.pool_n > kMaxEditBricks) return *why = "the boxes cover more than 2^29 bricks", LS_ERR_NOMEM;
  }
  *voxels_set = set;
  if (items == 0) return LS_OK;
  size_t off = 0;
  const size_t o_box = take(off, boxes.size() * sizeof(EditBox)), o_ax = take(off, axes.size() * sizeof(unsigned));
  int rc;
  if ((rc = reserve_staging(m, off, 0, st))) return *why = "out of device memory for the boxes", rc;
  char* q = m.qbuf.get();
  const EditBox* dbox = (const EditBox*)(q + o_box);
  const unsigned* dax = (const unsigned*)(q + o_ax);
  LSO_TRY(cudaMemcpyAsync(q + o_box, boxes.data(), boxes.size() * sizeof(EditBox), cudaMemcpyHostToDevice, st));
  LSO_TRY(cudaMemcpyAsync(q + o_ax, axes.data(), axes.size() * sizeof(unsigned), cudaMemcpyHostToDevice, st));
  const int blocks = (int)((items + 255) / 256);
  // Count the missing bricks, grow the pool and the hash for them, then place them (the insert's retry when a probe
  // sequence overflows).  A failure here (a growth refused after some bricks were placed) leaves the known voxels as they
  // were: placed bricks hold none, as after a failed insert.  Both tree builds give a brick without a known voxel state 0
  // and no node, and the queries and the bounds test the known bits, so the cached trees and every answer stay current.
  if ((rc = upload_counters(m, st))) return rc;
  ed_bricks_kernel<false><<<blocks, 256, 0, st>>>(dbox, n, dax, items, dev_of(m), m.cnt_dev.get());
  LSO_LAUNCHED();
  if ((rc = read_counters(m, st))) return rc;
  const long long missing = (long long)m.cnt_host.get()->n_out;
  if (missing > 0) {
    const long long need = m.pool_n + missing;
    if (need > m.pool_cap()) {
      long long cap = m.pool_cap() > 0 ? m.pool_cap() : 1;
      while (cap < need) cap *= 2;
      if ((rc = grow_pool(m, (int)cap, st))) return *why = "the map cannot grow", rc;
    }
    long long tab = m.tab_cap();
    while (2 * need > tab) tab *= 2;
    if (tab > m.tab_cap() && (rc = rebuild_table(m, (int)tab, st, launches))) return *why = "the map cannot grow", rc;
    for (;;) {
      if ((rc = upload_counters(m, st))) return rc;
      ed_bricks_kernel<true><<<blocks, 256, 0, st>>>(dbox, n, dax, items, dev_of(m), m.cnt_dev.get());
      LSO_LAUNCHED();
      if ((rc = read_counters(m, st))) return rc;
      const Counters c = *m.cnt_host.get();
      m.pool_n = c.pool_n < m.pool_cap() ? c.pool_n : m.pool_cap();
      if (!c.overflow) break;
      if ((rc = rebuild_table(m, m.tab_cap() * 2, st, launches))) return *why = "the map cannot grow", rc;
    }
  }
  // Only now is the map written: one launch per box, in call order, so the last box covering a voxel sets it.
  if ((rc = upload_counters(m, st))) return rc;
  const Dev D = dev_of(m);
  for (int i = 0; i < n; ++i) {
    const EditBox& B = boxes[(size_t)i];
    const long long nb = (long long)B.n[0] * B.n[1] * B.n[2];
    if (nb == 0) continue;
    const float value = occupied[i] ? P.l_max : P.l_min;
    ed_write_kernel<<<(unsigned)nb, 512, 0, st>>>(B, dax, value, D, m.cnt_dev.get());
    LSO_LAUNCHED();
  }
  if ((rc = read_counters(m, st))) return rc;
  *new_known = (long long)m.cnt_host.get()->new_known;
  m.n_known += *new_known;
  return LS_OK;
}

int clear(Map& m, cudaStream_t st) {
  const size_t a = (size_t)m.pool_n;
  if (a > 0) {  // a claimed pool brick must start zeroed, as a grown pool's do
    LSO_TRY(cudaMemsetAsync(m.lo.get(), 0, a * 512 * sizeof(float), st));
    LSO_TRY(cudaMemsetAsync(m.known.get(), 0, a * 16 * sizeof(unsigned), st));
    LSO_TRY(cudaMemsetAsync(m.mfree.get(), 0, a * 16 * sizeof(unsigned), st));
    LSO_TRY(cudaMemsetAsync(m.mocc.get(), 0, a * 16 * sizeof(unsigned), st));
    LSO_TRY(cudaMemsetAsync(m.touched.get(), 0, a * sizeof(unsigned), st));
  }
  LSO_TRY(cudaMemsetAsync(m.tab_keys.get(), 0xff, (size_t)m.tab_cap() * sizeof(unsigned long long), st));
  LSO_TRY(cudaMemsetAsync(m.tab_vals.get(), 0xff, (size_t)m.tab_cap() * sizeof(int), st));
  LSO_TRY(cudaStreamSynchronize(st));
  m.pool_n = 0;
  m.n_known = 0;
  return LS_OK;
}

int box_voxels(Map& m, const Params& P, const double center3[3], const double size3[3], int which, uint64_t* keys,
               float* log_odds, float* centres4, long long cap, long long* n, cudaStream_t st, uint64_t* launches) {
  *n = 0;
  std::vector<int> axis[3];
  long long pts = 1;
  for (int a = 0; a < 3; ++a) {
    if (!edit_axis(center3[a], size3[a], P, &axis[a])) return LS_ERR_ARG;
    pts *= (long long)axis[a].size();
  }
  if (pts > 0x7fffffffLL) return LS_ERR_ARG;
  if (pts == 0) return LS_OK;
  const int nx = (int)axis[0].size(), ny = (int)axis[1].size(), nz = (int)axis[2].size();
  std::vector<int> flat;
  for (int a = 0; a < 3; ++a) flat.insert(flat.end(), axis[a].begin(), axis[a].end());
  size_t scan_bytes = 0;
  LSO_TRY(cub::DeviceScan::InclusiveSum(nullptr, scan_bytes, (int*)nullptr, (int*)nullptr, (int)pts, st));
  size_t off = 0;
  const size_t o_k = take(off, flat.size() * sizeof(int)), o_f = take(off, (size_t)pts * sizeof(int)),
               o_p = take(off, (size_t)pts * sizeof(int)), o_t = take(off, scan_bytes);
  int rc;
  if ((rc = reserve_staging(m, off, 0, st))) return rc;
  char* q = m.qbuf.get();
  const int* dk = (const int*)(q + o_k);
  int* flag = (int*)(q + o_f);
  int* pos = (int*)(q + o_p);
  LSO_TRY(cudaMemcpyAsync(q + o_k, flat.data(), flat.size() * sizeof(int), cudaMemcpyHostToDevice, st));
  const Dev D = dev_of(m);
  ed_flag_kernel<<<blocks(pts, 256), 256, 0, st>>>(dk, nx, ny, nz, pts, D, P, which, flag);
  LSO_LAUNCHED();
  LSO_TRY(cub::DeviceScan::InclusiveSum(q + o_t, scan_bytes, flag, pos, (int)pts, st));
  ++*launches;
  int total = 0;
  LSO_TRY(cudaMemcpyAsync(&total, pos + (pts - 1), sizeof(int), cudaMemcpyDeviceToHost, st));
  LSO_TRY(cudaStreamSynchronize(st));
  *n = total;
  if (total > cap) return LS_ERR_ARG;
  if (total == 0 || (!keys && !log_odds && !centres4)) return LS_OK;
  if ((rc = reserve_export(m, total, st))) return rc;
  ed_scatter_kernel<<<blocks(pts, 256), 256, 0, st>>>(dk, nx, ny, nz, pts, D, P.res, flag, pos, m.ex_k[0].get(), m.ex_v[0].get(),
                                                    m.ex_c.get());
  LSO_LAUNCHED();
  if (keys) LSO_TRY(cudaMemcpyAsync(keys, m.ex_k[0].get(), (size_t)total * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
  if (log_odds) LSO_TRY(cudaMemcpyAsync(log_odds, m.ex_v[0].get(), (size_t)total * sizeof(float), cudaMemcpyDeviceToHost, st));
  if (centres4) LSO_TRY(cudaMemcpyAsync(centres4, m.ex_c.get(), (size_t)total * sizeof(float4), cudaMemcpyDeviceToHost, st));
  LSO_TRY(cudaStreamSynchronize(st));
  return LS_OK;
}

int key_bounds(Map& m, int kmin[3], int kmax[3], bool* empty, cudaStream_t st, uint64_t* launches) {
  *empty = true;
  if (m.n_known == 0 || m.pool_n == 0) return LS_OK;
  size_t off = 0;
  const size_t o_mm = take(off, 6 * sizeof(int));
  int rc;
  if ((rc = reserve_staging(m, off, 0, st))) return rc;
  int* mm = (int*)(m.qbuf.get() + o_mm);
  LSO_TRY(cudaMemsetAsync(mm, 0x7f, 3 * sizeof(int), st));      // 0x7f7f7f7f: above any key
  LSO_TRY(cudaMemsetAsync(mm + 3, 0xff, 3 * sizeof(int), st));  // -1
  ed_bounds_kernel<<<m.pool_n, 512, 0, st>>>(dev_of(m), mm);
  LSO_LAUNCHED();
  int h[6];
  LSO_TRY(cudaMemcpyAsync(h, mm, sizeof h, cudaMemcpyDeviceToHost, st));
  LSO_TRY(cudaStreamSynchronize(st));
  if (h[3] < 0) return LS_OK;
  for (int a = 0; a < 3; ++a) kmin[a] = h[a], kmax[a] = h[3 + a];
  *empty = false;
  return LS_OK;
}

}  // namespace lso
