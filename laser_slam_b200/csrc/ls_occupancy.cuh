// Resident occupancy map (ls_occupancy_*): laser_to_octomap's scan insertion on the device.  The rules are
// oracle/OCCUPANCY.md; the layout and kernels are described in ls_occupancy.cu and DESIGN.md.
#pragma once
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <utility>

#include <cuda_runtime.h>

#include "../../include/ls_b200.h"
#include "ls_buffer.cuh"

namespace lso {

// The rules' constants: log-odds computed on the host in double and rounded to float once.
struct Params {
  double res, inv, max_range;
  float l_hit, l_miss, l_min, l_max, l_occ;
};

// Device counters of one insert (or export), copied back whole.
struct Counters {
  unsigned long long free_upd, occ_upd, new_known, n_out;
  int pool_n, n_touched, overflow, rays_cast, rays_skipped, pad[3];
};

// Device counters of one tree read, copied back once after the parse: the node counts, the record after the tree (INT_MAX
// while none is found), the known voxels and bricks the file covers, and why it is malformed (0 when it is not).
struct ReadCounters {
  unsigned long long nodes, inner, free_leaves, occ_leaves, known;
  long long bricks;
  int end, bad, pad[2];
};

// Bricks of 8x8x8 voxels.  The hash maps a brick key (13 bits per axis) to a pool index; per brick the pool holds 512
// float log-odds, 16 words of known bits and 16 + 16 words of per-scan free / occupied marks.
// Each group of arrays grows all or nothing; its first array tells its capacity.
struct Map {
  ls::Buffer<unsigned long long> tab_keys;  // power-of-two slots
  ls::Buffer<int> tab_vals;
  int pool_n = 0;
  ls::Buffer<int> tlist;  // per pool brick: bricks marked in this scan
  ls::Buffer<float> lo;
  ls::Buffer<unsigned> known, mfree, mocc;
  ls::Buffer<unsigned long long> bkey;  // brick key of each pool brick
  ls::Buffer<unsigned> touched;         // per brick: marked in this scan
  // per-scan scratch: ray ends, endpoint keys and classes; the endpoint-key -> first point index table
  ls::Buffer<float4> ends;
  ls::Buffer<unsigned long long> pkey;
  ls::Buffer<int> cls;
  ls::Buffer<unsigned long long> ep_keys;
  ls::Buffer<int> ep_min;
  // export scratch
  ls::Buffer<float4> ex_c;
  ls::Buffer<unsigned long long> ex_k[2];
  ls::Buffer<unsigned> ex_v[2];
  ls::Buffer<unsigned char> cub_tmp;
  size_t cub_bytes = 0;
  // query staging (inputs and outputs of one call), grown by doubling
  ls::Buffer<char> qbuf;
  // tree read scratch: per stream record (the excess, parent, depth, first key, bricks) and per new brick (key, state)
  ls::Buffer<unsigned char> rd_pay;
  ls::Buffer<int> rd_ex, rd_tmp, rd_par, rd_anc, rd_bmin;
  ls::Buffer<unsigned char> rd_slot, rd_depth;
  ls::Buffer<unsigned long long> rd_key;
  ls::Buffer<long long> rd_nb, rd_boff;
  ls::Buffer<unsigned char> rd_cub;
  size_t rd_cub_bytes = 0;
  ls::Buffer<unsigned long long> rd_bkey;
  ls::Buffer<unsigned char> rd_bst;
  ls::Buffer<ReadCounters> rd_cnt_dev;
  ls::PinnedBuffer<ReadCounters> rd_cnt_host;
  ls::Buffer<Counters> cnt_dev;
  ls::PinnedBuffer<Counters> cnt_host;
  long long n_known = 0;

  int tab_cap() const { return (int)tab_keys.capacity(); }
  int pool_cap() const { return (int)tlist.capacity(); }
};

// The brick hash: a brick key's home slot (before the mask) and the probe bound of its linear probing.  The insert places
// keys with it (ls_occupancy.cu); the queries and change detection (ls_changes.cu) look them up.
constexpr int kMaxProbe = 64;
__device__ __forceinline__ unsigned hash64(unsigned long long k) {
  k ^= k >> 33;
  k *= 0xff51afd7ed558ccdull;
  k ^= k >> 33;
  k *= 0xc4ceb9fe1a85ec53ull;
  k ^= k >> 33;
  return (unsigned)k;
}

// Pool index of brick bk, or -1 when the hash does not hold it.  Read-only: no CAS, no allocation, no wait on a pending
// slot.  A slot whose value is negative (left by an insert whose pool filled) is absent.
__device__ __forceinline__ int lookup_brick(const unsigned long long* tab_keys, const int* tab_vals, unsigned mask,
                                            unsigned long long bk) {
  unsigned h = hash64(bk) & mask;
  for (int p = 0; p < kMaxProbe; ++p, h = (h + 1u) & mask) {
    const unsigned long long k = tab_keys[h];
    if (k == bk) {
      const int v = tab_vals[h];
      return v >= 0 ? v : -1;
    }
    if (k == ~0ull) return -1;
  }
  return -1;
}

// ---- the map's keys and bricks ---------------------------------------------------------------------------------------
// Every module that reads the map takes its key, centre, brick and voxel-state rules from here.  The key and centre rules
// are octomap's (16 levels), bit for bit under -fmad=false.

// A voxel key is floor(c / res) + kKeyOffset per axis, valid in [0, 65535].
constexpr int kKeyOffset = 32768;

// octomap's coordToKeyChecked: floor(c * inv) + 32768; false when outside [0, 65535] (NaN included).  A float coordinate
// is widened to double before the multiply.
__host__ __device__ __forceinline__ bool key_of(double inv, double c, int& k) {
  const double s = floor(c * inv);
  if (!(s >= -(double)kKeyOffset && s < (double)kKeyOffset)) return false;
  k = (int)s + kKeyOffset;
  return true;
}

// octomap's keyToCoord(key): the voxel centre on one axis in double (centre_d), and that rounded to float once (centre_of),
// as every output centre is.
__host__ __device__ __forceinline__ double centre_d(int k, double res) { return ((double)(k - kKeyOffset) + 0.5) * res; }
__host__ __device__ __forceinline__ float centre_of(int k, double res) { return (float)centre_d(k, res); }
// octomap's keyToCoord(key, depth) in double of the node whose first voxel key is k0, s = 16 - depth (key + 2^(s-1) is the
// node's key); at s = 0 it equals centre_d.
__host__ __device__ __forceinline__ double leaf_centre_d(int k0, int s, double res) {
  const int kc = k0 + (s > 0 ? 1 << (s - 1) : 0);
  const double scale = (double)(1 << s);
  return (floor(((double)kc - (double)kKeyOffset) / scale) + 0.5) * (res * scale);
}

// The packed key of a voxel: x | y << 16 | z << 32.
__host__ __device__ __forceinline__ unsigned long long pack(int kx, int ky, int kz) {
  return (unsigned long long)kx | ((unsigned long long)ky << 16) | ((unsigned long long)kz << 32);
}

// A brick key: the brick's coordinates (a voxel key >> 3 per axis), 13 bits each, x | y << 13 | z << 26.
__host__ __device__ __forceinline__ unsigned long long brick_pack(unsigned long long bx, unsigned long long by,
                                                                  unsigned long long bz) {
  return bx | (by << 13) | (bz << 26);
}
__host__ __device__ __forceinline__ unsigned long long brick_key(const int k[3]) {
  return brick_pack(k[0] >> 3, k[1] >> 3, k[2] >> 3);
}

// A voxel's local index in its brick, t = x | y << 3 | z << 6 of its key's low 3 bits, and back: the keys of voxel t of
// brick bk (t in [0, 512)).
__host__ __device__ __forceinline__ int local_of(const int k[3]) { return (k[0] & 7) | ((k[1] & 7) << 3) | ((k[2] & 7) << 6); }
__host__ __device__ __forceinline__ void voxel_keys(unsigned long long bk, int t, int k[3]) {
  k[0] = (int)(bk & 0x1fff) * 8 + (t & 7);
  k[1] = (int)((bk >> 13) & 0x1fff) * 8 + ((t >> 3) & 7);
  k[2] = (int)((bk >> 26) & 0x1fff) * 8 + (t >> 6);
}

// State (LS_CELL_*) of voxel `local` of pool brick b: unknown without its known bit, else occupied iff its log-odds >=
// l_occ.  The known bit decides "unknown", not the brick's presence: a brick placed by a failed insert holds no known
// voxel.  *v (when v is not NULL): the log-odds of a known voxel.
__host__ __device__ __forceinline__ int voxel_state(const unsigned* known, const float* lo, float l_occ, int b, int local,
                                                    float* v) {
  if (!((known[(size_t)b * 16 + (local >> 5)] >> (local & 31)) & 1u)) return LS_CELL_UNKNOWN;
  const float x = lo[(size_t)b * 512 + local];
  if (v) *v = x;
  return x >= l_occ ? LS_CELL_OCCUPIED : LS_CELL_FREE;
}

// ---- host: error codes, launches and staging -------------------------------------------------------------------------
// LS_OK, LS_ERR_NOMEM for a failed allocation, else LS_ERR_CUDA; the error is cleared from cudaGetLastError.
inline int code(cudaError_t e) {
  if (e == cudaSuccess) return LS_OK;
  cudaGetLastError();
  return e == cudaErrorMemoryAllocation ? LS_ERR_NOMEM : LS_ERR_CUDA;
}

#define LSO_TRY(call)                \
  do {                               \
    const int rc_ = lso::code(call); \
    if (rc_) return rc_;             \
  } while (0)

// After a launch: counts it in *launches and returns its error.
#define LSO_LAUNCHED()           \
  do {                           \
    ++*launches;                 \
    LSO_TRY(cudaGetLastError()); \
  } while (0)

inline unsigned blocks(long long n, int threads) { return (unsigned)((n + threads - 1) / threads); }

// The next 256-byte aligned region of `bytes` in a staging buffer whose first `off` bytes are taken.
inline size_t take(size_t& off, size_t bytes) {
  const size_t o = off;
  off += (bytes + 255) & ~(size_t)255;
  return o;
}

// The query staging m.qbuf of at least `bytes`, grown by doubling from 64 KiB after the stream's pending work.  The first
// `keep` bytes survive a growth; with keep 0 the old buffer is dropped first.
inline int reserve_staging(Map& m, size_t bytes, size_t keep, cudaStream_t st) {
  if (bytes <= m.qbuf.capacity()) return LS_OK;
  LSO_TRY(cudaStreamSynchronize(st));
  size_t cap = m.qbuf.capacity() ? 2 * m.qbuf.capacity() : (size_t)1 << 16;
  while (cap < bytes) cap *= 2;
  if (keep == 0) return code(m.qbuf.reserve(bytes, cap));
  ls::Buffer<char> grown;
  LSO_TRY(grown.reserve(bytes, cap));
  LSO_TRY(cudaMemcpyAsync(grown.get(), m.qbuf.get(), keep, cudaMemcpyDeviceToDevice, st));
  LSO_TRY(cudaStreamSynchronize(st));
  m.qbuf = std::move(grown);
  return LS_OK;
}

// Change detection (ls_changes.cu; DESIGN.md §4b'''''''''').  A baseline holds, per brick with a known voxel when it was
// taken, its brick key (ascending) and 32 words: 16 of known bits, then 16 of occupied bits (known and v >= L_occ); res is
// the map's resolution then.  Keys, not pool indices, so growth, rehashing, clear and reads cannot corrupt it.
struct Baseline {
  ls::Buffer<unsigned long long> keys;
  ls::Buffer<unsigned> bits;
  long long n = 0;
  double res = 0.0;
};
struct Changes {
  Baseline base, next;  // next: a capture in progress, swapped with base when it completes
  // capture records before the sort (key, order, bits); the diff's voxels (packed key, states) before and after the sort,
  // their status / previous bytes and centres
  ls::Buffer<unsigned long long> rec_key;
  ls::Buffer<int> rec_idx[2];
  ls::Buffer<unsigned> rec_bits;
  ls::Buffer<unsigned long long> out_key[2];
  ls::Buffer<unsigned> out_val[2];
  ls::Buffer<signed char> out_st;
  ls::Buffer<float4> out_c;
  ls::Buffer<unsigned char> cub_tmp;
  ls::Buffer<unsigned long long> cnt_dev;
  ls::PinnedBuffer<unsigned long long> cnt_host;
};

// The map as octomap's pruned tree: depth 16 over the map's keys, each brick a depth-13 node.  Node records hold the
// bricks by Morton code, then each upper level (12 ... 0) in turn; all scratch is O(bricks) plus the outputs.
struct Octree {
  ls::Buffer<int> levels;  // per depth d = 0 ... 13: first record, count
  ls::Buffer<int> pool;    // bricks: pool index (its capacity is the group's, in bricks)
  ls::Buffer<unsigned long long> code;  // Morton code of the node at its depth
  ls::Buffer<int> first, end;           // upper nodes: their children's records [first, end)
  ls::Buffer<unsigned char> st;         // 0 no known voxel below, 1 free leaf, 2 occupied leaf, 3 inner (full tree: 1 leaf)
  ls::Buffer<unsigned> val;             // full tree only: each node's float log-odds bits
  ls::Buffer<unsigned long long> n_nodes, n_bytes, n_leaves;  // subtree totals: nodes, payload bytes (.bt only), leaves
  ls::Buffer<unsigned long long> off, loff;  // payload byte and occupied-leaf offsets in pre-order
  ls::Buffer<unsigned long long> sort_k;
  ls::Buffer<int> sort_v;
  ls::Buffer<unsigned char> cub_tmp;
  size_t cub_bytes = 0;
  ls::Buffer<unsigned long long> tot_dev;    // nodes, payload bytes, occupied leaves of the whole tree
  ls::PinnedBuffer<unsigned long long> tot_host;
  ls::Buffer<unsigned char> payload;
  ls::Buffer<float4> centres;  // with depths
  ls::Buffer<unsigned char> depths;
  long long nodes = 0, bytes = 0, leaves = 0;  // of the last build (full tree: every leaf)
  // The last build's brick records (the map's pool_n then).  A failed edit can place empty bricks without invalidating a
  // build, so a pass over the build's records takes their number from here, not from the map.
  int bricks = 0;
};

// All return LS_OK, LS_ERR_NOMEM or LS_ERR_CUDA (include/ls_b200.h) and count their launches in *launches.
int init(Map& m, int initial_bricks, cudaStream_t st);
// One scan of n points (device, float4) moved by T (column-major float32; identity: copied).  Synchronous; *out holds the
// scan's counters.  On an error the known voxels and their log-odds are unchanged.
int insert(Map& m, const Params& P, const float4* pts, int n, const float T[16], bool identity, cudaStream_t st, Counters* out,
           uint64_t* launches);
// which: LS_OCC_KNOWN or LS_OCC_OCCUPIED.  count() gives the number of voxels; download() writes n of them (as counted)
// by ascending packed key: keys, log-odds and centres {x, y, z, 1}, each output may be NULL.
int count(Map& m, const Params& P, int which, long long* n, cudaStream_t st, uint64_t* launches);
int download(Map& m, const Params& P, int which, long long n, uint64_t* keys, float* log_odds, float* centres4, cudaStream_t st,
             uint64_t* launches);
size_t device_bytes(const Map& m);
// octomap's two tree payloads: the pruned max-likelihood tree of writeBinary (.bt, oracle/OCTREE.md) and the
// full-probability tree of OcTree::write (.ot, DESIGN.md §4b''''''': every node's float log-odds and child mask, 5 bytes
// per node in pre-order, pruned by value).
enum class TreeFormat { Binary, Full };
// Builds the map's tree in format f into t: the payload (and, for .bt, the occupied leaves' centres and depths) stays on
// the device, t.nodes / bytes / leaves hold the counts (leaves: occupied ones for .bt, every leaf for .ot).  Reads the map
// only.  Synchronous.
int build_tree(const Map& m, const Params& P, TreeFormat f, Octree& t, cudaStream_t st, uint64_t* launches);
// Copies the last build's payload (t.bytes) and, each when not NULL, its t.leaves centres {x, y, z, 1} and depths.
int download_octree(const Octree& t, unsigned char* payload, float* centres4, unsigned char* depths, cudaStream_t st);

// The leaves of the value-pruned tree as boxes (DESIGN.md §4b''''''''''''): getAllFreeBoxes / getAllOccupiedBoxes and
// generateMarkerArray's cube lists.  raw_*: every leaf of the tree in pre-order, then the gather target of a download;
// cen / tag: the listed leaves in pre-order, a tag being the depth plus 32 for a free leaf; idx / sorted: their
// positions, and those positions and tags after a stable sort by state (or state and depth).
struct Leaves {
  ls::Buffer<float4> raw_c, cen, rgba;
  ls::Buffer<unsigned char> raw_tag, tag, stag;
  ls::Buffer<int> keep, pos, idx, sorted;
  ls::Buffer<unsigned char> cub_tmp;
  size_t cub_bytes = 0;
  ls::Buffer<unsigned long long> cnt_dev;
  ls::PinnedBuffer<unsigned long long> cnt_host;
  long long n = 0, n_occupied = 0;              // listed leaves, of them occupied
  long long occupied[17] = {}, free[17] = {};  // listed leaves per depth
};
// Lists the leaves of t, which must be the current .ot build of m (TreeFormat::Full), whose key cube meets kmin ... kmax
// on every axis: L.n and the counts per state and depth are set.  Reads the map and t only; synchronous.
int build_leaves(const Map& m, const Params& P, Octree& t, const int kmin[3], const int kmax[3], Leaves& L, cudaStream_t st,
                 uint64_t* launches);
// Of the last list: which = 1 the free leaves, 2 the occupied ones, 3 all, each part in pre-order.  Writes their centres
// {x, y, z, 1} and tags (n of them, as counted).
int download_leaves(Leaves& L, int which, float* centres4, unsigned char* tags, cudaStream_t st, uint64_t* launches);
// The last list ordered by (occupied first, depth, pre-order): centres {x, y, z, 1} and, for the occupied leaves, the
// height colour {r, g, b, 1} (min_z < max_z, finite: checked by the caller).
int marker_cubes(Leaves& L, double min_z, double max_z, double color_factor, float* centres4, float* rgba4, cudaStream_t st,
                 uint64_t* launches);

// A leaf of a tree walk as one word: its first voxel key packed (bits 0 ... 47), its depth (48 ... 55) and 1 when it is
// occupied (bit 56).
__host__ __device__ __forceinline__ unsigned long long leaf_record(int kx, int ky, int kz, int depth, bool occupied) {
  return pack(kx, ky, kz) | ((unsigned long long)depth << 48) | ((unsigned long long)occupied << 56);
}
// The leaves of t, which must be the current .bt build of m (TreeFormat::Binary), in pre-order as leaf_record words: rec
// holds t.nodes - t.bytes / 2 of them (every node less the inner ones).  Reads the map; of t it writes only t.loff, which
// becomes each node's offset among all leaves (the .bt build leaves its occupied-leaf offsets there, read during the build
// only, so loff is scratch between builds).  Asynchronous on st.
int tree_leaf_records(const Map& m, const Params& P, Octree& t, unsigned long long* rec, cudaStream_t st, uint64_t* launches);

// octomap_server's projected_map of the .bt tree (ls_projection.cu; DESIGN.md §4b''''''''''''').  rec / span / off: per
// leaf, its record, the (leaf, row) spans it paints and their exclusive sum; stat: the ordered bounds (min x, y, z, max x,
// y, z) and the spans in all; planes: the occupied and known-free bit-planes; grid: the last projection's cells, row j at
// j * width, written only by a call that succeeds.
struct Projection {
  ls::Buffer<unsigned long long> rec, span, off, stat;
  ls::PinnedBuffer<unsigned long long> stat_host;
  ls::Buffer<unsigned char> cub_tmp;
  size_t cub_bytes = 0;
  ls::Buffer<unsigned> planes;
  ls::Buffer<signed char> grid;
  // the last projection: octomap_server's grid geometry and the cells per value (-1, 0, 100)
  long long width = 0, height = 0, cells[3] = {0, 0, 0};
  double origin[2] = {0.0, 0.0};
};
// The band, padding and map of one projection; the caller checks that the band has no NaN and that min_size is finite and
// >= 0.
struct ProjectionArgs {
  double min_z, max_z, min_size_x, min_size_y;
};
// Projects t, the current .bt build of m, into p (synchronous).  LS_ERR_ARG (*why says why) when a padded corner has no key
// or the grid has more than 2^31 - 1 cells; LS_ERR_NOMEM when its buffers cannot grow.  After any error p's last
// projection is as it was.
int build_projection(const Map& m, const Params& P, Octree& t, const ProjectionArgs& a, Projection& p, const char** why,
                     cudaStream_t st, uint64_t* launches);
// The last projection's width * height cells.
int download_projection(const Projection& p, int8_t* cells, cudaStream_t st);

// octomap's readBinary (.bt) or readData (.ot) of a payload (`bytes` bytes after "data\n", `nodes` the header's size) into
// the map, replacing it (DESIGN.md §4b'''''' and §4b''''''').  P: the map's parameters at the file's resolution (P.l_occ
// classifies a .ot's leaves in *out; a .ot leaf's voxels take its value verbatim).  Synchronous.  Validates the whole
// stream and the brick count before it grows or writes anything: LS_ERR_ARG for a malformed payload (for .ot, a leaf
// value that is not finite too), LS_ERR_NOMEM for more bricks than the map can index or a failed growth, and the map is
// unchanged after any error (*why then says why).  *out: the counts; out->inner: the nodes with children.
int read_tree(Map& m, const Params& P, TreeFormat f, const unsigned char* payload, long long bytes, long long nodes,
              ReadCounters* out, const char** why, cudaStream_t st, uint64_t* launches);

// Queries (oracle/QUERIES.md), reading the map only.  Synchronous; host inputs and outputs, *visited the voxel states the
// kernels read.  n <= 0 launches nothing.
// getCellStatusPoint: LS_CELL_* per point (double triples), the log-odds or NaN when unknown (log_odds may be NULL).
int query_cells(Map& m, const Params& P, const double* pts3, int n, int8_t* status, float* log_odds, long long* visited,
                cudaStream_t st, uint64_t* launches);
// getLineStatus / getVisibility (box3 NULL) or getLineStatusBoundingBox (box3: the box size): LS_CELL_* per segment and the
// packed key that decided it (all ones when free; first_keys may be NULL).  LS_ERR_ARG when the box has more than 2^31 - 1
// lines in all.  The box size must be finite and >= 0 (checked by the caller).
int query_lines(Map& m, const Params& P, const double* starts3, const double* ends3, int n, const double* box3,
                int stop_at_unknown, int8_t* status, uint64_t* first_keys, long long* visited, cudaStream_t st,
                uint64_t* launches);
// castRay: LS_RAY_* per ray and the voxel centre it names (NaN for LS_RAY_INVALID; ends3 may be NULL).
int query_rays(Map& m, const Params& P, const float* origins3, const float* directions3, int n, int ignore_unknown,
               double max_range, int8_t* result, float* ends3, long long* visited, cudaStream_t st, uint64_t* launches);

// Edits (DESIGN.md §4b'''''''').  Synchronous.  The box loop per axis: c = res * floor(p / res) + res / 2, points from
// (c - s/2) + 0.001 while <= (c + s/2) - 0.001 in steps of res (double), each cast to float and keyed; invalid keys skipped.
// setLogOddsBoundingBox of n boxes (double triples; finite, sizes >= 0, checked by the caller) in call order: every voxel a
// loop point keys becomes known with L_max (occupied[i] != 0) or L_min.  LS_ERR_ARG when an axis has more than 2^17 points,
// LS_ERR_NOMEM before any allocation when the call's bricks and those in use exceed 2^29, or when the map cannot grow; the
// known voxels and their values are unchanged after any error (*why says why).  *voxels_set: loop points with a valid key.
int set_boxes(Map& m, const Params& P, const double* centres3, const double* sizes3, const int8_t* occupied, int n,
              long long* voxels_set, long long* new_known, const char** why, cudaStream_t st, uint64_t* launches);
// resetMap: no known voxel and no brick; the capacity stays.
int clear(Map& m, cudaStream_t st);
// getOccupiedPointcloudInBoundingBox: per loop point of the box (x outer, z inner) whose voxel is in `which` (LS_OCC_*),
// its packed key, log-odds and voxel centre {x, y, z, 1}, in loop order.  *n: their number; LS_ERR_ARG without a copy when
// it exceeds cap, or when an axis has more than 2^17 points or the box more than 2^31 - 1.  Outputs may be NULL.
int box_voxels(Map& m, const Params& P, const double center3[3], const double size3[3], int which, uint64_t* keys,
               float* log_odds, float* centres4, long long cap, long long* n, cudaStream_t st, uint64_t* launches);
// The smallest and largest known key per axis; *empty when no voxel is known.
int key_bounds(Map& m, int kmin[3], int kmax[3], bool* empty, cudaStream_t st, uint64_t* launches);

// Euclidean distance map of a box of the map (ls_distance.cu; DESIGN.md §4b''''''''').  The grid covers keys kmin ...
// kmin + size - 1 per axis, cell (x, y, z) at (z * size[1] + y) * size[0] + x.  The field is val[0] (the squared distance in
// cells, M where no obstacle is within it) and site[0] (the obstacle's cell index, -1 when none).  The other buffers are
// scratch: the obstacle grid (one byte per cell), val[1] / site[1] between the passes and the per-column stacks.
struct DistanceField {
  ls::Buffer<unsigned char> grid;
  ls::Buffer<int> val[2], site[2];
  ls::Buffer<uint2> stack;
  ls::Buffer<unsigned long long> cnt_dev;
  ls::PinnedBuffer<unsigned long long> cnt_host;
  ls::Buffer<char> qbuf;  // query staging, grown by doubling
  int kmin[3] = {0, 0, 0}, size[3] = {0, 0, 0};
  long long cells = 0, obstacles = 0;
  double res = 0.0, inv = 0.0;
  int M = 0;
};
// Every buffer of a field of `cells` cells, all or nothing: after LS_ERR_NOMEM every buffer is empty.
int distance_reserve(DistanceField& f, long long cells);
// The field of the map's known voxels inside f's box (kmin, size, cells and M set by the caller, buffers reserved): an
// obstacle is an occupied voxel (v >= l_occ), and with unknown_occ every unknown cell too.  Reads the map only.  Synchronous;
// sets f.obstacles.
int distance_update(DistanceField& f, const Map& m, float l_occ, bool unknown_occ, cudaStream_t st, uint64_t* launches);
// One thread per point (host float triples): distance [m], squared distance in cells and the obstacle's voxel centre, each
// output may be NULL; -1 / -1 / NaN for a point whose key is invalid or outside the box (*outside counts them), NaN obstacle
// centres where the cell has no obstacle.  Synchronous.
int distance_query(DistanceField& f, const float* pts3, int n, float* dist, int* sq, float* obst3, long long* outside,
                   cudaStream_t st, uint64_t* launches);
// The whole field in cell order (each output may be NULL): squared distances, obstacles as packed keys (all ones when none).
int distance_download(DistanceField& f, int* sq, uint64_t* keys, cudaStream_t st, uint64_t* launches);
size_t distance_bytes(const DistanceField& f);

// Change detection (ls_changes.cu).  Both read the map only and are synchronous.
// The map's state now (P.res, P.l_occ) becomes c.base.  On an error c.base is as it was.
int capture_baseline(Changes& c, const Map& m, const Params& P, cudaStream_t st, uint64_t* launches);
// The voxels whose state (LS_CELL_*) differs from c.base's, by ascending packed key: keys, states now and then, centres
// {x, y, z, 1} (at P.res when known now, at c.base.res otherwise), each output may be NULL.  *n: their number;
// LS_ERR_ARG without a copy when it exceeds cap.
int diff_changes(Changes& c, const Map& m, const Params& P, uint64_t* keys, int8_t* status, int8_t* previous, float* centres4,
                 long long cap, long long* n, cudaStream_t st, uint64_t* launches);
void release_changes(Changes& c);
size_t changes_bytes(const Changes& c);

// Box status and robot collision (ls_collision.cu; DESIGN.md §4b''''''''''').  Both read the map only, stage in m.qbuf
// and are synchronous; *visited: the voxel states read.  LS_ERR_ARG, before any result, for a size that is negative or
// not finite, an axis of more than 2^17 loop points in a box whose centre has a valid key, or boxes spanning more than
// 2^36 (box, brick) items in all.
// getCellStatusBoundingBox per box (double triples): LS_CELL_*.  n <= 0 launches nothing.
int box_status(Map& m, const Params& P, const double* centres3, const double* sizes3, int n, int8_t* status,
               long long* visited, cudaStream_t st, uint64_t* launches);
// checkPathForCollisionsWithRobot per path: the robot box robot3 at positions3[offsets[p] ... offsets[p + 1]) (offsets
// checked by the caller: non-decreasing from 0, at most 2^31 - 1 poses); first[p] the first colliding pose's index
// within its path, -1 when none.  A pose collides when its status is occupied, or not free with unknown_occ.
int check_paths(Map& m, const Params& P, const double* positions3, const int64_t* offsets, int n_paths,
                const double robot3[3], int unknown_occ, int64_t* first, long long* visited, cudaStream_t st,
                uint64_t* launches);

}  // namespace lso
