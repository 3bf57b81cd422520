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
#include <cfloat>
#include <cstdint>
#include <cstring>

#include <cub/cub.cuh>
#include <cuda_runtime.h>

#include "../../include/ls_b200.h"
#include "ls_occupancy.cuh"

namespace lso {
namespace {

constexpr unsigned long long kEmpty = ~0ull;
constexpr int kPending = -1, kFull = -2;
constexpr int kMaxProbe = 64;
constexpr int kKeyMax = 32768;
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
  return Dev{m.tab_keys, m.tab_vals, (unsigned)m.tab_cap - 1u, m.pool_cap, m.lo, m.known, m.mfree, m.mocc, m.bkey, m.touched,
             m.tlist};
}

__device__ __forceinline__ unsigned hash64(unsigned long long k) {
  k ^= k >> 33;
  k *= 0xff51afd7ed558ccdull;
  k ^= k >> 33;
  k *= 0xc4ceb9fe1a85ec53ull;
  k ^= k >> 33;
  return (unsigned)k;
}

// floor(c * (1/res)) + 32768, valid iff in [0, 65535]
__device__ __forceinline__ bool key_of(double inv, float c, int& k) {
  const double s = floor((double)c * inv);
  if (!(s >= -(double)kKeyMax && s < (double)kKeyMax)) return false;
  k = (int)s + kKeyMax;
  return true;
}
__device__ __forceinline__ bool key3(double inv, const float p[3], int k[3]) {
  return key_of(inv, p[0], k[0]) && key_of(inv, p[1], k[1]) && key_of(inv, p[2], k[2]);
}
__device__ __forceinline__ unsigned long long pack(int kx, int ky, int kz) {
  return (unsigned long long)kx | ((unsigned long long)ky << 16) | ((unsigned long long)kz << 32);
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
  const unsigned long long bk = (unsigned long long)(k[0] >> 3) | ((unsigned long long)(k[1] >> 3) << 13) |
                                ((unsigned long long)(k[2] >> 3) << 26);
  if (bk != cur.bk) {
    const int b = brick_of(D, cnt, bk);
    if (b < 0) return false;
    cur.bk = bk;
    cur.b = b;
    if (D.touched[b] == 0u && atomicExch(&D.touched[b], 1u) == 0u) D.tlist[atomicAdd(&cnt->n_touched, 1)] = b;
  }
  const int local = (k[0] & 7) | ((k[1] & 7) << 3) | ((k[2] & 7) << 6);
  unsigned* w = (occ ? D.mocc : D.mfree) + (size_t)cur.b * 16 + (local >> 5);
  const unsigned bit = 1u << (local & 31);
  if (!(*w & bit)) atomicOr(w, bit);  // near the sensor thousands of rays share a voxel: read before the atomic
  return true;
}

// octomap's computeRayKeys from o to e, marking every key before the end key free.
__device__ bool walk(const Dev& D, Counters* cnt, Cursor& cur, const Params& P, const float o[3], const float e[3]) {
  int ko[3], ke[3];
  if (!key3(P.inv, o, ko) || !key3(P.inv, e, ke)) return true;
  if (ko[0] == ke[0] && ko[1] == ke[1] && ko[2] == ke[2]) return true;
  if (!mark(D, cnt, cur, ko, false)) return false;
  float dir[3] = {e[0] - o[0], e[1] - o[1], e[2] - o[2]};
  const float length = (float)norm3(dir);
  for (int i = 0; i < 3; ++i) dir[i] = dir[i] / length;
  int step[3], k[3] = {ko[0], ko[1], ko[2]};
  double tmax[3], tdelta[3];
  for (int i = 0; i < 3; ++i) {
    step[i] = dir[i] > 0.0f ? 1 : (dir[i] < 0.0f ? -1 : 0);
    if (step[i] != 0) {
      double border = ((double)(k[i] - kKeyMax) + 0.5) * P.res;
      border += (double)(float)((double)step[i] * P.res * 0.5);
      tmax[i] = (border - (double)o[i]) / (double)dir[i];
      tdelta[i] = P.res / (double)fabsf(dir[i]);
    } else {
      tmax[i] = DBL_MAX;
      tdelta[i] = DBL_MAX;
    }
  }
  for (;;) {
    int dim;
    if (tmax[0] < tmax[1]) dim = tmax[0] < tmax[2] ? 0 : 2;
    else dim = tmax[1] < tmax[2] ? 1 : 2;
    k[dim] += step[dim];
    tmax[dim] += tdelta[dim];
    if (k[0] == ke[0] && k[1] == ke[1] && k[2] == ke[2]) break;
    if (k[dim] < 0 || k[dim] > 65535) break;
    const double dist = fmin(fmin(tmax[0], tmax[1]), tmax[2]);
    if (dist > (double)length) break;
    if (!mark(D, cnt, cur, k, false)) return false;
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
  if (!walk(D, cnt, cur, P, o, e)) return;
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
      const int kx = (int)(bk & 0x1fff) * 8 + (t & 7), ky = (int)((bk >> 13) & 0x1fff) * 8 + ((t >> 3) & 7),
                kz = (int)((bk >> 26) & 0x1fff) * 8 + (t >> 6);
      keys[pos] = pack(kx, ky, kz);
      vals[pos] = __float_as_uint(x);
    }
  }
}

__global__ void occ_centres_kernel(const unsigned long long* __restrict__ keys, long long n, double res, float4* __restrict__ out) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const unsigned long long k = keys[i];
    float c[3];
    for (int a = 0; a < 3; ++a) c[a] = (float)(((double)((int)((k >> (16 * a)) & 0xffff) - kKeyMax) + 0.5) * res);
    out[i] = make_float4(c[0], c[1], c[2], 1.0f);
  }
}

int code(cudaError_t e) {
  if (e == cudaSuccess) return LS_OK;
  cudaGetLastError();
  return e == cudaErrorMemoryAllocation ? LS_ERR_NOMEM : LS_ERR_CUDA;
}

#define OCC_TRY(call)           \
  do {                          \
    const int rc_ = code(call); \
    if (rc_) return rc_;        \
  } while (0)

#define OCC_LAUNCHED()                        \
  do {                                        \
    ++*launches;                              \
    OCC_TRY(cudaGetLastError());              \
  } while (0)

template <typename T>
cudaError_t alloc(T** p, size_t count) {
  *p = nullptr;
  return cudaMalloc((void**)p, (count ? count : 1) * sizeof(T));
}

template <typename T>
void free_ptr(T*& p) {
  if (p) cudaFree(p);
  p = nullptr;
}

int upload_counters(Map& m, cudaStream_t st) {
  std::memset(m.cnt_host, 0, sizeof(Counters));
  m.cnt_host->pool_n = m.pool_n;
  OCC_TRY(cudaMemcpyAsync(m.cnt_dev, m.cnt_host, sizeof(Counters), cudaMemcpyHostToDevice, st));
  return LS_OK;
}

int read_counters(Map& m, cudaStream_t st) {
  OCC_TRY(cudaMemcpyAsync(m.cnt_host, m.cnt_dev, sizeof(Counters), cudaMemcpyDeviceToHost, st));
  OCC_TRY(cudaStreamSynchronize(st));
  return LS_OK;
}

// A pool of `cap` bricks holding the first pool_n bricks of the old one; marks and touched flags start clear.  The old pool
// stays when an allocation fails.
int grow_pool(Map& m, int cap, cudaStream_t st) {
  Map q;
  const size_t c = (size_t)cap;
  cudaError_t e = alloc(&q.lo, c * 512);
  if (e == cudaSuccess) e = alloc(&q.known, c * 16);
  if (e == cudaSuccess) e = alloc(&q.mfree, c * 16);
  if (e == cudaSuccess) e = alloc(&q.mocc, c * 16);
  if (e == cudaSuccess) e = alloc(&q.bkey, c);
  if (e == cudaSuccess) e = alloc(&q.touched, c);
  if (e == cudaSuccess) e = alloc(&q.tlist, c);
  const size_t n = (size_t)m.pool_n;
  if (e == cudaSuccess) e = cudaMemsetAsync(q.lo + n * 512, 0, (c - n) * 512 * sizeof(float), st);
  if (e == cudaSuccess) e = cudaMemsetAsync(q.known + n * 16, 0, (c - n) * 16 * sizeof(unsigned), st);
  if (e == cudaSuccess) e = cudaMemsetAsync(q.mfree, 0, c * 16 * sizeof(unsigned), st);
  if (e == cudaSuccess) e = cudaMemsetAsync(q.mocc, 0, c * 16 * sizeof(unsigned), st);
  if (e == cudaSuccess) e = cudaMemsetAsync(q.touched, 0, c * sizeof(unsigned), st);
  if (e == cudaSuccess && n > 0) e = cudaMemcpyAsync(q.lo, m.lo, n * 512 * sizeof(float), cudaMemcpyDeviceToDevice, st);
  if (e == cudaSuccess && n > 0) e = cudaMemcpyAsync(q.known, m.known, n * 16 * sizeof(unsigned), cudaMemcpyDeviceToDevice, st);
  if (e == cudaSuccess && n > 0) e = cudaMemcpyAsync(q.bkey, m.bkey, n * sizeof(unsigned long long), cudaMemcpyDeviceToDevice, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  Map& drop = e == cudaSuccess ? m : q;
  free_ptr(drop.lo), free_ptr(drop.known), free_ptr(drop.mfree), free_ptr(drop.mocc), free_ptr(drop.bkey);
  free_ptr(drop.touched), free_ptr(drop.tlist);
  if (e != cudaSuccess) return code(e);
  m.lo = q.lo, m.known = q.known, m.mfree = q.mfree, m.mocc = q.mocc, m.bkey = q.bkey, m.touched = q.touched, m.tlist = q.tlist;
  m.pool_cap = cap;
  return LS_OK;
}

// A hash of at least `cap` slots (power of two) holding every pool brick; doubles until the probe bound holds.  The old
// table stays when an allocation fails.
int rebuild_table(Map& m, int cap, cudaStream_t st, uint64_t* launches) {
  for (;; cap *= 2) {
    unsigned long long* keys = nullptr;
    int* vals = nullptr;
    cudaError_t e = alloc(&keys, (size_t)cap);
    if (e == cudaSuccess) e = alloc(&vals, (size_t)cap);
    if (e == cudaSuccess) e = cudaMemsetAsync(keys, 0xff, (size_t)cap * sizeof(unsigned long long), st);
    if (e == cudaSuccess) e = cudaMemsetAsync(vals, 0xff, (size_t)cap * sizeof(int), st);
    if (e == cudaSuccess) e = cudaMemsetAsync(&m.cnt_dev->overflow, 0, sizeof(int), st);
    if (e == cudaSuccess && m.pool_n > 0) {
      occ_rehash_kernel<<<(m.pool_n + 255) / 256, 256, 0, st>>>(m.bkey, m.pool_n, keys, vals, (unsigned)cap - 1u, m.cnt_dev);
      ++*launches;
      e = cudaGetLastError();
    }
    int overflow = 0;
    if (e == cudaSuccess) e = cudaMemcpyAsync(&overflow, &m.cnt_dev->overflow, sizeof(int), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess || overflow) {
      free_ptr(keys), free_ptr(vals);
      if (e != cudaSuccess) return code(e);
      continue;
    }
    free_ptr(m.tab_keys), free_ptr(m.tab_vals);
    m.tab_keys = keys, m.tab_vals = vals, m.tab_cap = cap;
    return LS_OK;
  }
}

int reserve_points(Map& m, int n, cudaStream_t st) {
  if (n > m.pt_cap) {
    OCC_TRY(cudaStreamSynchronize(st));
    const int cap = n + n / 8;
    free_ptr(m.ends), free_ptr(m.pkey), free_ptr(m.cls);
    m.pt_cap = 0;
    OCC_TRY(alloc(&m.ends, (size_t)cap));
    OCC_TRY(alloc(&m.pkey, (size_t)cap));
    OCC_TRY(alloc(&m.cls, (size_t)cap));
    m.pt_cap = cap;
  }
  int ep = 1024;
  while (ep < 2 * n) ep *= 2;
  if (ep > m.ep_cap) {
    OCC_TRY(cudaStreamSynchronize(st));
    free_ptr(m.ep_keys), free_ptr(m.ep_min);
    m.ep_cap = 0;
    OCC_TRY(alloc(&m.ep_keys, (size_t)ep));
    OCC_TRY(alloc(&m.ep_min, (size_t)ep));
    m.ep_cap = ep;
  }
  return LS_OK;
}

int reserve_export(Map& m, long long n, cudaStream_t st) {
  if (n <= m.ex_cap && m.ex_c) return LS_OK;
  OCC_TRY(cudaStreamSynchronize(st));
  for (int j = 0; j < 2; ++j) free_ptr(m.ex_k[j]), free_ptr(m.ex_v[j]);
  free_ptr(m.ex_c);
  free_ptr(m.cub_tmp);
  m.ex_cap = 0;
  m.cub_bytes = 0;
  const long long cap = n + n / 8 + 1024;
  for (int j = 0; j < 2; ++j) {
    OCC_TRY(alloc(&m.ex_k[j], (size_t)cap));
    OCC_TRY(alloc(&m.ex_v[j], (size_t)cap));
  }
  OCC_TRY(alloc(&m.ex_c, (size_t)cap));
  size_t bytes = 0;
  OCC_TRY(cub::DeviceRadixSort::SortPairs(nullptr, bytes, m.ex_k[0], m.ex_k[1], m.ex_v[0], m.ex_v[1], (int)cap, 0, 48, st));
  OCC_TRY(alloc((unsigned char**)&m.cub_tmp, bytes));
  m.cub_bytes = bytes;
  m.ex_cap = cap;
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
    occ_select_kernel<<<(int)blocks, 256, 0, st>>>(dev_of(m), P, which, nvox, keys, vals, m.cnt_dev);
    OCC_LAUNCHED();
  }
  return read_counters(m, st);
}

}  // namespace

int init(Map& m, int initial_bricks, cudaStream_t st) {
  m = Map();
  OCC_TRY(cudaMalloc((void**)&m.cnt_dev, sizeof(Counters)));
  OCC_TRY(cudaMallocHost((void**)&m.cnt_host, sizeof(Counters)));
  int rc;
  if ((rc = grow_pool(m, initial_bricks, st))) return rc;
  int cap = 1024;
  while (cap < 2 * initial_bricks) cap *= 2;
  uint64_t launches = 0;
  return rebuild_table(m, cap, st, &launches);
}

void release(Map& m) {
  free_ptr(m.tab_keys), free_ptr(m.tab_vals);
  free_ptr(m.lo), free_ptr(m.known), free_ptr(m.mfree), free_ptr(m.mocc), free_ptr(m.bkey), free_ptr(m.touched);
  free_ptr(m.tlist);
  free_ptr(m.ends), free_ptr(m.pkey), free_ptr(m.cls), free_ptr(m.ep_keys), free_ptr(m.ep_min);
  for (int j = 0; j < 2; ++j) free_ptr(m.ex_k[j]), free_ptr(m.ex_v[j]);
  free_ptr(m.ex_c), free_ptr(m.cub_tmp), free_ptr(m.cnt_dev);
  if (m.cnt_host) cudaFreeHost(m.cnt_host);
  m.cnt_host = nullptr;
}

size_t device_bytes(const Map& m) {
  const size_t pool = (size_t)m.pool_cap * (512 * sizeof(float) + 48 * sizeof(unsigned) + sizeof(unsigned long long) +
                                            sizeof(unsigned) + sizeof(int));
  const size_t tab = (size_t)m.tab_cap * (sizeof(unsigned long long) + sizeof(int));
  const size_t pts = (size_t)m.pt_cap * (sizeof(float4) + sizeof(unsigned long long) + sizeof(int)) +
                     (size_t)m.ep_cap * (sizeof(unsigned long long) + sizeof(int));
  const size_t ex = (size_t)m.ex_cap * (2 * sizeof(unsigned long long) + 2 * sizeof(unsigned) + sizeof(float4)) + m.cub_bytes;
  return pool + tab + pts + ex + sizeof(Counters);
}

int insert(Map& m, const Params& P, const float4* pts, int n, const float T[16], bool identity, cudaStream_t st, Counters* out,
           uint64_t* launches) {
  int rc;
  std::memset(out, 0, sizeof(Counters));
  if ((rc = reserve_points(m, n, st))) return rc;
  if (2LL * m.pool_n > m.tab_cap && (rc = rebuild_table(m, m.tab_cap * 2, st, launches))) return rc;
  if ((rc = upload_counters(m, st))) return rc;
  OCC_TRY(cudaMemsetAsync(m.ep_keys, 0xff, (size_t)m.ep_cap * sizeof(unsigned long long), st));
  OCC_TRY(cudaMemsetAsync(m.ep_min, 0x7f, (size_t)m.ep_cap * sizeof(int), st));  // 0x7f7f7f7f: above any point index
  Xform16 x;
  std::memcpy(x.T, T, sizeof(x.T));
  const int blocks = (n + 255) / 256;
  if (n > 0) {
    occ_classify_kernel<<<blocks, 256, 0, st>>>(pts, n, x, identity ? 1 : 0, P, m.ends, m.pkey, m.cls, m.ep_keys, m.ep_min,
                                                 (unsigned)m.ep_cap - 1u);
    OCC_LAUNCHED();
  }
  for (;;) {
    if (n > 0) {
      occ_cast_kernel<<<blocks, 256, 0, st>>>(n, P, T[12], T[13], T[14], m.ends, m.pkey, m.cls, m.ep_keys, m.ep_min,
                                              (unsigned)m.ep_cap - 1u, dev_of(m), m.cnt_dev);
      OCC_LAUNCHED();
    }
    if ((rc = read_counters(m, st))) return rc;
    const Counters c = *m.cnt_host;
    if (!c.overflow) break;
    // Undo the marking: clear every mark and touched flag, keep the bricks that got a pool index, drop the rest from the
    // hash, grow what filled and mark again.
    m.pool_n = c.pool_n < m.pool_cap ? c.pool_n : m.pool_cap;
    OCC_TRY(cudaMemsetAsync(m.mfree, 0, (size_t)m.pool_cap * 16 * sizeof(unsigned), st));
    OCC_TRY(cudaMemsetAsync(m.mocc, 0, (size_t)m.pool_cap * 16 * sizeof(unsigned), st));
    OCC_TRY(cudaMemsetAsync(m.touched, 0, (size_t)m.pool_cap * sizeof(unsigned), st));
    int tab = m.tab_cap;
    if ((c.overflow & kOverflowTable) || 2LL * m.pool_n > tab) tab *= 2;
    if ((rc = rebuild_table(m, tab, st, launches))) return rc;
    if ((c.overflow & kOverflowPool) && (rc = grow_pool(m, m.pool_cap * 2, st))) return rc;
    if ((rc = upload_counters(m, st))) return rc;
  }
  m.pool_n = m.cnt_host->pool_n;
  if (m.cnt_host->n_touched > 0) {
    occ_update_kernel<<<m.cnt_host->n_touched, 512, 0, st>>>(dev_of(m), P, m.cnt_dev);
    OCC_LAUNCHED();
    if ((rc = read_counters(m, st))) return rc;
  }
  m.n_known += (long long)m.cnt_host->new_known;
  *out = *m.cnt_host;
  return LS_OK;
}

int count(Map& m, const Params& P, int which, long long* n, cudaStream_t st, uint64_t* launches) {
  if (which == LS_OCC_KNOWN) {
    *n = m.n_known;
    return LS_OK;
  }
  int rc;
  if ((rc = select(m, P, which, nullptr, nullptr, st, launches))) return rc;
  *n = (long long)m.cnt_host->n_out;
  return LS_OK;
}

int download(Map& m, const Params& P, int which, long long n, uint64_t* keys, float* log_odds, float* centres4, cudaStream_t st,
             uint64_t* launches) {
  if (n <= 0) return LS_OK;
  if (n > 0x7fffffffLL) return LS_ERR_NOMEM;
  int rc;
  if ((rc = reserve_export(m, n, st))) return rc;
  if ((rc = select(m, P, which, m.ex_k[0], m.ex_v[0], st, launches))) return rc;
  if ((long long)m.cnt_host->n_out != n) return LS_ERR_CUDA;
  size_t bytes = m.cub_bytes;
  OCC_TRY(cub::DeviceRadixSort::SortPairs(m.cub_tmp, bytes, m.ex_k[0], m.ex_k[1], m.ex_v[0], m.ex_v[1], (int)n, 0, 48, st));
  ++*launches;
  if (centres4) {
    long long blocks = (n + 255) / 256;
    if (blocks > 65536) blocks = 65536;
    occ_centres_kernel<<<(int)blocks, 256, 0, st>>>(m.ex_k[1], n, P.res, m.ex_c);
    OCC_LAUNCHED();
    OCC_TRY(cudaMemcpyAsync(centres4, m.ex_c, (size_t)n * sizeof(float4), cudaMemcpyDeviceToHost, st));
  }
  if (keys) OCC_TRY(cudaMemcpyAsync(keys, m.ex_k[1], (size_t)n * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  if (log_odds) OCC_TRY(cudaMemcpyAsync(log_odds, m.ex_v[1], (size_t)n * sizeof(float), cudaMemcpyDeviceToHost, st));
  OCC_TRY(cudaStreamSynchronize(st));
  return LS_OK;
}

}  // namespace lso
