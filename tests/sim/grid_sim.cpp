// CPU simulation of the CUDA grid build + exact NN query (test tool; not a product path).
//
// Compiles laser_slam_b200/csrc/ls_grid.cuh for the host (-ffp-contract=off) and builds the same
// two-level structure (+ occupancy pyramid) the build kernels produce, so the query logic (loop bounds, pruning margins,
// tie-break, seeding) can be checked against brute force here, where there is no GPU.  The CUDA
// kernels are still checked on the GPU by tests/test_gpu_*.py; this only shortens the debug loop.
#define LS_SIM_COUNTERS 1
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <vector>

#include "../../laser_slam_b200/csrc/ls_grid.cuh"

thread_local long long ls::ls_sim_cand = 0, ls::ls_sim_entries = 0, ls::ls_sim_steps = 0;

namespace {
struct SimGrid {
  ls::Grid g;
  std::vector<ls::Entry> top, tab1;
  std::vector<float4> pts;
  std::vector<unsigned long long> pyr, topmask;
};

void build(SimGrid& S, const float* refc3, int m, float cell, int max_cells, int split) {
  float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (int i = 0; i < m; ++i)
    for (int a = 0; a < 3; ++a) {
      lo[a] = std::min(lo[a], refc3[3 * i + a]);
      hi[a] = std::max(hi[a], refc3[3 * i + a]);
    }
  if (m == 0) { lo[0] = lo[1] = lo[2] = 0; hi[0] = hi[1] = hi[2] = 0; }
  ls::grid_setup(S.g, lo, hi, cell, max_cells, split, m);
  const ls::Grid& g = S.g;
  struct Key { int c0, f1, idx; };
  std::vector<Key> keys(m);
  std::vector<int> cnt0(g.n_cells0, 0);
  for (int i = 0; i < m; ++i) {
    keys[i] = {ls::top_index(g, refc3[3 * i], refc3[3 * i + 1], refc3[3 * i + 2]), -1, i};
    cnt0[keys[i].c0]++;
  }
  std::vector<int> tabidx0(g.n_cells0, -1);
  int n1 = 0;
  for (int c = 0; c < g.n_cells0; ++c)
    if (cnt0[c] > g.leaf_split) tabidx0[c] = n1++;
  std::vector<int> cnt1((size_t)n1 * LS_FB3, 0);
  for (int i = 0; i < m; ++i) {
    const int t = tabidx0[keys[i].c0];
    if (t < 0) continue;
    float lx, ly, lz;
    ls::top_origin(g, keys[i].c0, lx, ly, lz);
    keys[i].f1 = ls::sub_index(refc3[3 * i], refc3[3 * i + 1], refc3[3 * i + 2], lx, ly, lz, g.inv1);
    cnt1[(size_t)t * LS_FB3 + keys[i].f1]++;
  }
  std::sort(keys.begin(), keys.end(), [](const Key& a, const Key& b) {
    if (a.c0 != b.c0) return a.c0 < b.c0;
    if (a.f1 != b.f1) return a.f1 < b.f1;
    return a.idx > b.idx;  // deliberately NOT index order: the GPU scatter order is arbitrary
  });
  S.pts.resize(m);
  for (int i = 0; i < m; ++i) {
    const int id = keys[i].idx;
    float4 p; p.x = refc3[3 * id]; p.y = refc3[3 * id + 1]; p.z = refc3[3 * id + 2]; p.w = ls::i2f(id);
    S.pts[i] = p;
  }
  S.top.assign(g.n_cells0, ls::Entry{0, 0});
  S.tab1.assign((size_t)n1 * LS_FB3, ls::Entry{0, 0});
  uint32_t run = 0;
  for (int c = 0; c < g.n_cells0; ++c) {
    S.top[c].start = run;
    if (tabidx0[c] < 0) {
      S.top[c].meta = cnt0[c];
      run += cnt0[c];
      continue;
    }
    S.top[c].meta = ~tabidx0[c];
    for (int f = 0; f < LS_FB3; ++f) {
      const size_t k = (size_t)tabidx0[c] * LS_FB3 + f;
      S.tab1[k].start = run;
      S.tab1[k].meta = cnt1[k];
      run += cnt1[k];
    }
  }
  S.g.n_tab1 = n1;
  S.topmask.assign(g.n_cells0, 0ull);
  for (int c = 0; c < g.n_cells0; ++c)
    if (tabidx0[c] >= 0)
      for (int f = 0; f < LS_FB3; ++f)
        if (cnt1[(size_t)tabidx0[c] * LS_FB3 + f] > 0) S.topmask[c] |= 1ull << (f / LS_FB);
  // occupancy pyramid
  S.pyr.assign(g.n_pyr_cells, 0ull);
  for (int l = 1; l <= g.n_pyr; ++l) {
    const int* pd = g.pdim[l];
    const int* cd = g.pdim[l - 1];
    for (int z = 0; z < pd[2]; ++z)
      for (int y = 0; y < pd[1]; ++y)
        for (int x = 0; x < pd[0]; ++x) {
          unsigned long long mask = 0;
          for (int bit = 0; bit < 64; ++bit) {
            const int cx = 4 * x + (bit & 3), cy = 4 * y + ((bit >> 2) & 3), cz = 4 * z + (bit >> 4);
            if (cx >= cd[0] || cy >= cd[1] || cz >= cd[2]) continue;
            const size_t ci = ((size_t)cz * cd[1] + cy) * cd[0] + cx;
            const bool occ = (l == 1) ? (S.top[ci].meta != 0) : (S.pyr[g.poff[l - 1] + ci] != 0ull);
            if (occ) mask |= 1ull << bit;
          }
          S.pyr[g.poff[l] + ((size_t)z * pd[1] + y) * pd[0] + x] = mask;
        }
  }
}
}  // namespace

extern "C" {
// Exact NN of n queries (stride 3) over the centred reference (stride 3).  warm: optional previous
// match ORIGINAL indices (-1 = cold).  stats (optional, 4 doubles): mean candidates, mean entry
// loads, max candidates, number of fine tables, H0, number of level-0 cells.
void sim_nn(const float* q3, int n, const float* refc3, int m, float cell, int max_cells, int split,
            const int32_t* warm_ids, int32_t* ids, float* d2, double* stats, int32_t* per_query_cand,
            int32_t* per_query_entries, float cap_d2) {
  SimGrid S;
  build(S, refc3, m, cell, max_cells, split);
  std::vector<int> pos_of(m);
  for (int i = 0; i < m; ++i) pos_of[ls::f2i(S.pts[i].w)] = i;
  ls::GridView v{S.top.data(), S.tab1.data(), S.pts.data(), S.pyr.data(), S.topmask.data()};
  long long cand = 0, ent = 0, cmax = 0;
  for (int i = 0; i < n; ++i) {
    ls::ls_sim_cand = 0;
    ls::ls_sim_entries = 0;
    ls::ls_sim_steps = 0;
    const int warm = (warm_ids && warm_ids[i] >= 0) ? pos_of[warm_ids[i]] : -1;
    const ls::Best b = ls::nn_search(S.g, v, q3[3 * i], q3[3 * i + 1], q3[3 * i + 2], warm, cap_d2);
    ids[i] = b.idx;
    d2[i] = b.d2;
    if (per_query_cand) per_query_cand[i] = (int32_t)ls::ls_sim_cand;
    if (per_query_entries) per_query_entries[i] = (int32_t)(ls::ls_sim_entries | (ls::ls_sim_steps << 16));
    cand += ls::ls_sim_cand;
    ent += ls::ls_sim_entries;
    cmax = std::max(cmax, ls::ls_sim_cand);
  }
  if (stats) {
    stats[0] = n ? (double)cand / n : 0;
    stats[1] = n ? (double)ent / n : 0;
    stats[2] = (double)cmax;
    stats[3] = S.g.n_tab1;
    stats[4] = S.g.H0;
    stats[5] = S.g.n_cells0;
  }
}

// The geometry grid_setup derives from a centred bounding box [lo, hi]: H0 (and the m/leaf_split it is given) go to
// H0_out; out (int32) = dim[3], n_cells0, n_pyr, n_pyr_cells, then pdim[l][3] and poff[l] for l = 0..L, where L (the
// return value) is the deepest pyramid level Grid has room for.
int sim_grid(const float* lo, const float* hi, float cell, int max_cells, int split, int m, float* H0_out,
             int32_t* out) {
  ls::Grid g;
  ls::grid_setup(g, lo, hi, cell, max_cells, split, m);
  const int levels = (int)(sizeof(g.pdim) / sizeof(g.pdim[0])) - 1;
  *H0_out = g.H0;
  int k = 0;
  for (int a = 0; a < 3; ++a) out[k++] = g.dim[a];
  out[k++] = g.n_cells0;
  out[k++] = g.n_pyr;
  out[k++] = g.n_pyr_cells;
  for (int l = 0; l <= levels; ++l) {
    for (int a = 0; a < 3; ++a) out[k++] = l <= g.n_pyr ? g.pdim[l][a] : 0;
    out[k++] = l <= g.n_pyr ? g.poff[l] : 0;
  }
  return levels;
}

// Exact K nearest neighbours (knn_search, the normals' query) of n queries over the centred reference: ids/d2 are n x k,
// ascending by (d2, index); a map with fewer than k points leaves INT_MAX / +inf in the tail.  stats as sim_nn.
void sim_knn(const float* q3, int n, const float* refc3, int m, float cell, int max_cells, int split, int k,
             int32_t* ids, float* d2, double* stats) {
  SimGrid S;
  build(S, refc3, m, cell, max_cells, split);
  ls::GridView v{S.top.data(), S.tab1.data(), S.pts.data(), S.pyr.data(), S.topmask.data()};
  for (int i = 0; i < n; ++i) {
    ls::TopK t;
    ls::knn_search(S.g, v, q3[3 * i], q3[3 * i + 1], q3[3 * i + 2], k, t);
    for (int j = 0; j < k; ++j) {
      ids[(size_t)i * k + j] = t.id[j];
      d2[(size_t)i * k + j] = t.d[j];
    }
  }
  if (stats) {
    stats[3] = S.g.n_tab1;
    stats[4] = S.g.H0;
    stats[5] = S.g.n_cells0;
  }
}

// Certified candidate lists over a sequence of poses: queries rd3 (n x 3) are moved by T_seq[t] (column-major 4x4,
// n_iter of them); iteration t answers every query through vlist_query when its certificate holds and through
// nn_search (+ vlist_build) otherwise, exactly as the ICP kernel's phase A does, and checks each answer against
// nn_search alone.  caps[t] = capped-search radius^2 of iteration t, skin_w/skin_v[t] = motion bound of the last
// step (|rotation vector|, |translation|).  Returns the number of answers that differ (must be 0);
// hits[t] = queries answered from their list, overflow[t] = list builds refused (more than LS_VK points).
int sim_vlists(const float* rd3, int n, const float* refc3, int m, float cell, int max_cells, int split, const float* T_seq,
               int n_iter, const float* caps, const float* skin_w, const float* skin_v, int32_t* hits, int32_t* overflow,
               int32_t* ids_last, float* d2_last) {
  SimGrid S;
  build(S, refc3, m, cell, max_cells, split);
  ls::GridView v{S.top.data(), S.tab1.data(), S.pts.data(), S.pyr.data(), S.topmask.data()};
  std::vector<float4> vq(n, make_float4(0.f, 0.f, 0.f, 0.f)), vpts((size_t)LS_VK * n);
  std::vector<int> warm(n, -1);
  ls::VLists L{vq.data(), vpts.data(), n};
  int bad = 0;
  for (int t = 0; t < n_iter; ++t) {
    const float* T = T_seq + 16 * t;
    int h = 0, of = 0, of_builds = 0;
    for (int i = 0; i < n; ++i) {
      float qx, qy, qz;
      ls::xform_point(T, rd3[3 * i], rd3[3 * i + 1], rd3[3 * i + 2], qx, qy, qz);
      const ls::Best ref = ls::nn_search(S.g, v, qx, qy, qz, warm[i], caps[t]);
      ls::Best b;
      float4 cb = make_float4(0.f, 0.f, 0.f, 0.f);
      if (ls::vlist_query(L, S.pts.data(), i, vq[i], vpts[i], qx, qy, qz, caps[t], b, cb)) {
        ++h;
        if (b.pos >= 0 && (ls::f2i(cb.w) != b.pos || cb.x != S.pts[b.pos].x || cb.y != S.pts[b.pos].y || cb.z != S.pts[b.pos].z)) ++bad;
        if (b.pos >= 0) b.idx = ls::f2i(S.pts[b.pos].w);
        else { b.idx = -1; b.d2 = INFINITY; }
        if (b.pos != ref.pos || b.idx != ref.idx || !(b.d2 == ref.d2)) ++bad;
      } else if (t >= 1) {
        float px, py, pz;  // where the previous iteration had this query
        ls::xform_point(T_seq + 16 * (t - 1), rd3[3 * i], rd3[3 * i + 1], rd3[3 * i + 2], px, py, pz);
        const float motion = std::sqrt(ls::dist2(qx, qy, qz, px, py, pz));
        (void)skin_w; (void)skin_v;
        const float4 before = vq[i];
        ls::vlist_build(S.g, v, L, i, qx, qy, qz, ref.pos >= 0, ref.d2, caps[t], motion);
        if (ls::f2i(vq[i].w) == 0 && (before.x != vq[i].x || ls::f2i(before.w) != 0)) ++of;
        if (before.x != vq[i].x || before.y != vq[i].y || before.w != vq[i].w) ++of_builds;
      }
      if (ref.pos >= 0) warm[i] = ref.pos;
      if (t == n_iter - 1) { ids_last[i] = ref.idx; d2_last[i] = ref.d2; }
    }
    if (hits) hits[t] = h;
    if (overflow) overflow[t] = of | (of_builds << 12);  // low 12 bits: refused builds (saturating use in tests is fine), rest: builds
  }
  return bad;
}
}
