// Change detection of the resident occupancy map: octomap's enableChangeDetection / changedKeysBegin / resetChangeDetection
// as a diff of the map against a baseline (DESIGN.md §4b'''''''''').  Reads the map only (tab_keys / tab_vals, lo, known,
// bkey); the insert, edit and read kernels do not know it exists.
//   capture  (a) ch_capture_kernel   one block per pool brick with a known voxel: its brick key, 16 known words and 16
//                                    occupied words, at a slot from one atomic per brick
//            a CUB radix sort over the 39 key bits orders the records, (b) ch_gather_kernel moves their words into place
//   diff     (c) ch_current_kernel   one block per pool brick: the brick's baseline record by binary search (none: every
//                                    voxel unknown then), each voxel's state now against its state then
//            (d) ch_baseline_kernel  one block per baseline brick: absent from the current hash, every voxel known then is
//                                    unknown now; present, (c) has compared it
//            (c) and (d) run once to count (one readback sizes the outputs) and once to emit with warp-aggregated slots; a
//            CUB radix sort over the 48 packed-key bits orders the voxels, (e) ch_finish_kernel writes states and centres
// A capture is built beside the baseline and swapped in only when it completes, so an error leaves the baseline as it was.
#include <cstdint>
#include <utility>

#include <cub/cub.cuh>
#include <cuda_runtime.h>

#include "../../include/ls_b200.h"
#include "ls_occupancy.cuh"

namespace lso {
namespace {

constexpr int kWords = 32;  // per baseline brick: 16 known words, then 16 occupied words

// (a): blockDim 512, warp w owns known word w of the brick.
__global__ void __launch_bounds__(512) ch_capture_kernel(const unsigned long long* __restrict__ bkey,
                                                         const unsigned* __restrict__ known, const float* __restrict__ lo,
                                                         float l_occ, unsigned long long* __restrict__ rec_key,
                                                         int* __restrict__ rec_idx, unsigned* __restrict__ rec_bits,
                                                         unsigned long long* __restrict__ count) {
  __shared__ int slot;
  const int b = blockIdx.x, t = threadIdx.x, lane = t & 31, w = t >> 5;
  const unsigned kn = known[(size_t)b * 16 + w];
  const bool occ = ((kn >> lane) & 1u) && lo[(size_t)b * 512 + t] >= l_occ;
  const unsigned oc = __ballot_sync(0xffffffffu, occ);
  if (!__syncthreads_or(kn != 0u)) return;  // the whole block: no known voxel (a brick left by a failed insert)
  if (t == 0) {
    slot = (int)atomicAdd(count, 1ull);
    rec_key[slot] = bkey[b];
    rec_idx[slot] = slot;
  }
  __syncthreads();
  if (lane == 0) {
    rec_bits[(size_t)slot * kWords + w] = kn;
    rec_bits[(size_t)slot * kWords + 16 + w] = oc;
  }
}

// (b): one thread per word of the sorted records.
__global__ void ch_gather_kernel(const int* __restrict__ order, const unsigned* __restrict__ rec_bits, long long words,
                                 unsigned* __restrict__ bits) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= words) return;
  bits[i] = rec_bits[(size_t)order[i / kWords] * kWords + (size_t)(i % kWords)];
}

__device__ __forceinline__ int state(unsigned known_w, unsigned occ_w, int lane) {
  if (!((known_w >> lane) & 1u)) return LS_CELL_UNKNOWN;
  return ((occ_w >> lane) & 1u) ? LS_CELL_OCCUPIED : LS_CELL_FREE;
}

// Voxel t of brick bk (every lane of the warp calls it): counted into *count and, with out_key, written at a
// warp-aggregated slot as (packed key, state now | state then << 2).
__device__ __forceinline__ void emit(bool changed, unsigned long long bk, int t, int now, int then,
                                     unsigned long long* __restrict__ out_key, unsigned* __restrict__ out_val,
                                     unsigned long long* __restrict__ count) {
  const unsigned bal = __ballot_sync(0xffffffffu, changed);
  if (!bal) return;
  const int lane = threadIdx.x & 31;
  unsigned long long base = 0;
  if (lane == 0) base = atomicAdd(count, (unsigned long long)__popc(bal));
  base = __shfl_sync(0xffffffffu, base, 0);
  if (changed && out_key) {
    const unsigned long long pos = base + __popc(bal & ((1u << lane) - 1u));
    int k[3];
    voxel_keys(bk, t, k);
    out_key[pos] = pack(k[0], k[1], k[2]);
    out_val[pos] = (unsigned)now | ((unsigned)then << 2);
  }
}

// (c): blockDim 512, one block per pool brick.
__global__ void __launch_bounds__(512) ch_current_kernel(const unsigned long long* __restrict__ bkey,
                                                         const unsigned* __restrict__ known, const float* __restrict__ lo,
                                                         float l_occ, const unsigned long long* __restrict__ base_keys,
                                                         const unsigned* __restrict__ base_bits, long long n_base,
                                                         unsigned long long* __restrict__ out_key,
                                                         unsigned* __restrict__ out_val, unsigned long long* __restrict__ count) {
  __shared__ long long found;
  const int b = blockIdx.x, t = threadIdx.x, lane = t & 31, w = t >> 5;
  const unsigned long long bk = bkey[b];
  if (t == 0) {
    long long l = 0, h = n_base;  // the first record with key >= bk
    while (l < h) {
      const long long mid = (l + h) >> 1;
      if (base_keys[mid] < bk) l = mid + 1;
      else h = mid;
    }
    found = (l < n_base && base_keys[l] == bk) ? l : -1;
  }
  __syncthreads();
  const long long j = found;
  const unsigned kn = known[(size_t)b * 16 + w];
  const bool occ = ((kn >> lane) & 1u) && lo[(size_t)b * 512 + t] >= l_occ;
  const int now = state(kn, __ballot_sync(0xffffffffu, occ), lane);
  const int then = j < 0 ? LS_CELL_UNKNOWN
                         : state(base_bits[(size_t)j * kWords + w], base_bits[(size_t)j * kWords + 16 + w], lane);
  emit(now != then, bk, t, now, then, out_key, out_val, count);
}

// (d): blockDim 512, one block per baseline brick.
__global__ void __launch_bounds__(512) ch_baseline_kernel(const unsigned long long* __restrict__ tab_keys,
                                                          const int* __restrict__ tab_vals, unsigned tab_mask,
                                                          const unsigned long long* __restrict__ base_keys,
                                                          const unsigned* __restrict__ base_bits,
                                                          unsigned long long* __restrict__ out_key,
                                                          unsigned* __restrict__ out_val, unsigned long long* __restrict__ count) {
  const int j = blockIdx.x, t = threadIdx.x, lane = t & 31, w = t >> 5;
  const unsigned long long bk = base_keys[j];
  if (lookup_brick(tab_keys, tab_vals, tab_mask, bk) >= 0) return;  // the whole block: (c) compares the brick
  const int then = state(base_bits[(size_t)j * kWords + w], base_bits[(size_t)j * kWords + 16 + w], lane);
  emit(then != LS_CELL_UNKNOWN, bk, t, LS_CELL_UNKNOWN, then, out_key, out_val, count);
}

// (e): per sorted voxel its two states and centre: at the map's resolution when known now, at the baseline's otherwise.
__global__ void ch_finish_kernel(const unsigned long long* __restrict__ keys, const unsigned* __restrict__ vals, long long n,
                                 double res_now, double res_base, signed char* __restrict__ status,
                                 signed char* __restrict__ previous, float4* __restrict__ centres) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned v = vals[i];
  const int now = (int)(v & 3u);
  status[i] = (signed char)now;
  previous[i] = (signed char)(v >> 2);
  const double res = now == LS_CELL_UNKNOWN ? res_base : res_now;
  const unsigned long long k = keys[i];
  float c[3];
  for (int a = 0; a < 3; ++a) c[a] = centre_of((int)((k >> (16 * a)) & 0xffff), res);
  centres[i] = make_float4(c[0], c[1], c[2], 1.0f);
}

// Grows an array of a group to at least `need` elements (an eighth more), after the stream's pending work.
template <class T>
int grow(ls::Buffer<T>& b, long long need, cudaStream_t st) {
  if ((size_t)need <= b.capacity()) return LS_OK;
  LSO_TRY(cudaStreamSynchronize(st));
  return code(b.reserve((size_t)need, (size_t)(need + need / 8 + 64)));
}

int grow_cub(Changes& c, size_t bytes, cudaStream_t st) {
  if (bytes <= c.cub_tmp.capacity()) return LS_OK;
  LSO_TRY(cudaStreamSynchronize(st));
  return code(c.cub_tmp.reserve(bytes, bytes + bytes / 8));
}

int read_count(Changes& c, cudaStream_t st, long long* n) {
  LSO_TRY(cudaMemcpyAsync(c.cnt_host.get(), c.cnt_dev.get(), sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  LSO_TRY(cudaStreamSynchronize(st));
  *n = (long long)*c.cnt_host.get();
  return LS_OK;
}

// One pass of (c) and (d): counts into cnt_dev, and with out_key emits.
int diff_pass(Changes& c, const Map& m, const Params& P, unsigned long long* out_key, unsigned* out_val, cudaStream_t st,
              uint64_t* launches) {
  LSO_TRY(cudaMemsetAsync(c.cnt_dev.get(), 0, sizeof(unsigned long long), st));
  if (m.pool_n > 0) {
    ch_current_kernel<<<m.pool_n, 512, 0, st>>>(m.bkey.get(), m.known.get(), m.lo.get(), P.l_occ, c.base.keys.get(),
                                                c.base.bits.get(), c.base.n, out_key, out_val, c.cnt_dev.get());
    LSO_LAUNCHED();
  }
  if (c.base.n > 0) {
    ch_baseline_kernel<<<(unsigned)c.base.n, 512, 0, st>>>(m.tab_keys.get(), m.tab_vals.get(), (unsigned)m.tab_cap() - 1u,
                                                           c.base.keys.get(), c.base.bits.get(), out_key, out_val,
                                                           c.cnt_dev.get());
    LSO_LAUNCHED();
  }
  return LS_OK;
}

}  // namespace

int capture_baseline(Changes& c, const Map& m, const Params& P, cudaStream_t st, uint64_t* launches) {
  LSO_TRY(c.cnt_dev.reserve(1, 1));
  LSO_TRY(c.cnt_host.reserve(1, 1));
  const long long nb = m.pool_n;
  int rc;
  if ((rc = grow(c.rec_key, nb, st)) || (rc = grow(c.rec_idx[0], nb, st)) ||
      (rc = grow(c.rec_idx[1], nb, st)) || (rc = grow(c.rec_bits, nb * kWords, st)))
    return rc;
  LSO_TRY(cudaMemsetAsync(c.cnt_dev.get(), 0, sizeof(unsigned long long), st));
  if (nb > 0) {
    ch_capture_kernel<<<(unsigned)nb, 512, 0, st>>>(m.bkey.get(), m.known.get(), m.lo.get(), P.l_occ, c.rec_key.get(),
                                                    c.rec_idx[0].get(), c.rec_bits.get(), c.cnt_dev.get());
    LSO_LAUNCHED();
  }
  long long n = 0;
  if ((rc = read_count(c, st, &n))) return rc;
  Baseline& nx = c.next;
  if ((rc = grow(nx.keys, n, st)) || (rc = grow(nx.bits, n * kWords, st))) return rc;
  if (n > 0) {
    size_t bytes = 0;
    LSO_TRY(cub::DeviceRadixSort::SortPairs(nullptr, bytes, c.rec_key.get(), nx.keys.get(), c.rec_idx[0].get(),
                                           c.rec_idx[1].get(), (int)n, 0, 39, st));
    if ((rc = grow_cub(c, bytes, st))) return rc;
    bytes = c.cub_tmp.capacity();
    LSO_TRY(cub::DeviceRadixSort::SortPairs(c.cub_tmp.get(), bytes, c.rec_key.get(), nx.keys.get(), c.rec_idx[0].get(),
                                           c.rec_idx[1].get(), (int)n, 0, 39, st));
    ++*launches;
    ch_gather_kernel<<<blocks(n * kWords, 256), 256, 0, st>>>(c.rec_idx[1].get(), c.rec_bits.get(), n * kWords,
                                                              nx.bits.get());
    LSO_LAUNCHED();
  }
  LSO_TRY(cudaStreamSynchronize(st));
  nx.n = n;
  nx.res = P.res;
  std::swap(c.base, c.next);
  return LS_OK;
}

int diff_changes(Changes& c, const Map& m, const Params& P, uint64_t* keys, int8_t* status, int8_t* previous, float* centres4,
                 long long cap, long long* n, cudaStream_t st, uint64_t* launches) {
  int rc;
  *n = 0;
  if ((rc = diff_pass(c, m, P, nullptr, nullptr, st, launches))) return rc;
  long long cnt = 0;
  if ((rc = read_count(c, st, &cnt))) return rc;
  *n = cnt;
  if (cnt > cap) return LS_ERR_ARG;
  if (cnt == 0) return LS_OK;
  if ((rc = grow(c.out_key[0], cnt, st)) || (rc = grow(c.out_key[1], cnt, st)) || (rc = grow(c.out_val[0], cnt, st)) ||
      (rc = grow(c.out_val[1], cnt, st)) || (rc = grow(c.out_st, 2 * cnt, st)) || (rc = grow(c.out_c, cnt, st)))
    return rc;
  if ((rc = diff_pass(c, m, P, c.out_key[0].get(), c.out_val[0].get(), st, launches))) return rc;
  size_t bytes = 0;
  LSO_TRY(cub::DeviceRadixSort::SortPairs(nullptr, bytes, c.out_key[0].get(), c.out_key[1].get(), c.out_val[0].get(),
                                         c.out_val[1].get(), (int)cnt, 0, 48, st));
  if ((rc = grow_cub(c, bytes, st))) return rc;
  bytes = c.cub_tmp.capacity();
  LSO_TRY(cub::DeviceRadixSort::SortPairs(c.cub_tmp.get(), bytes, c.out_key[0].get(), c.out_key[1].get(), c.out_val[0].get(),
                                         c.out_val[1].get(), (int)cnt, 0, 48, st));
  ++*launches;
  signed char* st_now = c.out_st.get();
  ch_finish_kernel<<<blocks(cnt, 256), 256, 0, st>>>(c.out_key[1].get(), c.out_val[1].get(), cnt, P.res, c.base.res, st_now,
                                                     st_now + cnt, c.out_c.get());
  LSO_LAUNCHED();
  const size_t N = (size_t)cnt;
  if (keys) LSO_TRY(cudaMemcpyAsync(keys, c.out_key[1].get(), 8 * N, cudaMemcpyDeviceToHost, st));
  if (status) LSO_TRY(cudaMemcpyAsync(status, st_now, N, cudaMemcpyDeviceToHost, st));
  if (previous) LSO_TRY(cudaMemcpyAsync(previous, st_now + cnt, N, cudaMemcpyDeviceToHost, st));
  if (centres4) LSO_TRY(cudaMemcpyAsync(centres4, c.out_c.get(), 16 * N, cudaMemcpyDeviceToHost, st));
  LSO_TRY(cudaStreamSynchronize(st));
  return LS_OK;
}

void release_changes(Changes& c) { c = Changes(); }

size_t changes_bytes(const Changes& c) {
  size_t b = (c.base.keys.capacity() + c.next.keys.capacity()) * sizeof(unsigned long long) +
             (c.base.bits.capacity() + c.next.bits.capacity() + c.rec_bits.capacity()) * sizeof(unsigned);
  b += c.rec_key.capacity() * sizeof(unsigned long long) +
       (c.rec_idx[0].capacity() + c.rec_idx[1].capacity()) * sizeof(int);
  b += (c.out_key[0].capacity() + c.out_key[1].capacity()) * sizeof(unsigned long long) +
       (c.out_val[0].capacity() + c.out_val[1].capacity()) * sizeof(unsigned) + c.out_st.capacity() +
       c.out_c.capacity() * sizeof(float4);
  return b + c.cub_tmp.capacity() + c.cnt_dev.capacity() * sizeof(unsigned long long);
}

}  // namespace lso
