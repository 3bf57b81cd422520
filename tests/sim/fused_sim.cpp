// CPU simulation of phase A's search with candidate-list build in one walk (ls_grid.cuh nn_search_collect), next to
// the build in a walk of its own (vlist_build) -- test and tuning tool, not a product path.
//
// The grid build and the query counters are grid_sim.cpp's: it is compiled into this library as a whole
// (one translation unit; this library is loaded on its own, never together with libgrid_sim.so).
#include "grid_sim.cpp"

extern "C" {
// Certified candidate lists over a sequence of poses: queries rd3 (n x 3) are moved by T_seq[t] (column-major 4x4,
// n_iter of them); iteration t answers every query through vlist_query when its certificate holds and otherwise through
// the search and the list build of phase A -- nn_search_collect (fused != 0, as the ICP kernel does) or nn_search and
// then a second walk for the list (fused == 0, the previous kernel) -- and checks each answer against nn_search alone.
// caps[t] = capped-search radius^2 of iteration t.  Returns the number of answers that differ (must be 0).  Per
// iteration: hits[t] = queries answered from their list, builds[t] = list collections (a radius passed the motion
// gate), refused[t] = collections that found more than LS_VK points (no list), steps[t] = dependent round trips
// (ls_sim_steps) of the searches and builds of the queries that missed their list.
int sim_vlists_paths(const float* rd3, int n, const float* refc3, int m, float cell, int max_cells, int split,
                     const float* T_seq, int n_iter, const float* caps, int fused, int32_t* hits, int32_t* builds,
                     int32_t* refused, int64_t* steps, int32_t* ids_last, float* d2_last) {
  SimGrid S;
  build(S, refc3, m, cell, max_cells, split);
  ls::GridView v{S.top.data(), S.tab1.data(), S.pts.data(), S.pyr.data(), S.topmask.data()};
  std::vector<float4> vq(n, make_float4(0.f, 0.f, 0.f, 0.f)), vpts((size_t)LS_VK * n);
  std::vector<int> warm(n, -1);
  ls::VLists L{vq.data(), vpts.data(), n};
  int bad = 0;
  for (int t = 0; t < n_iter; ++t) {
    const float* T = T_seq + 16 * t;
    int h = 0, nb = 0, nr = 0;
    long long st = 0;
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
      } else {
        const float4 before = vq[i];
        vq[i].w = ls::i2f(-1);  // sentinel: a header the build never writes (its radius is positive)
        const long long s0 = ls::ls_sim_steps;
        if (t == 0) {
          b = ls::nn_search(S.g, v, qx, qy, qz, warm[i], caps[t]);
        } else {
          float px, py, pz;  // where the previous iteration had this query
          ls::xform_point(T_seq + 16 * (t - 1), rd3[3 * i], rd3[3 * i + 1], rd3[3 * i + 2], px, py, pz);
          const float motion = std::sqrt(ls::dist2(qx, qy, qz, px, py, pz));
          if (fused) {
            b = ls::nn_search_collect(S.g, v, L, i, qx, qy, qz, warm[i], caps[t], motion);
          } else {
            b = ls::nn_search(S.g, v, qx, qy, qz, warm[i], caps[t]);
            ls::vlist_build(S.g, v, L, i, qx, qy, qz, b.pos >= 0, b.d2, caps[t], motion);
          }
        }
        st += ls::ls_sim_steps - s0;
        if (ls::f2i(vq[i].w) == -1) {
          vq[i] = before;  // no build: the old list stays
        } else {
          ++nb;
          if (ls::f2i(vq[i].w) == 0) ++nr;
        }
        if (b.pos != ref.pos || b.idx != ref.idx || !(b.d2 == ref.d2)) ++bad;
      }
      if (ref.pos >= 0) warm[i] = ref.pos;
      if (t == n_iter - 1) { ids_last[i] = ref.idx; d2_last[i] = ref.d2; }
    }
    if (hits) hits[t] = h;
    if (builds) builds[t] = nb;
    if (refused) refused[t] = nr;
    if (steps) steps[t] = st;
  }
  return bad;
}

// One phase-A search with list build per query, against the plain search: for each query i (warm_ids[i] = original
// index of the warm start, -1: seeded), nn_search_collect(.., caps[i], motion[i]) returns ids/d2/pos and list i
// (vq: n x 4 floats, vpts: LS_VK planes of n x 4, candidate .w = ORIGINAL index here), nn_search returns
// ref_ids/ref_d2/ref_pos.  rv[i] = the list radius vlist_radius gives for the search's first candidate (0: no list).
// Returns LS_VK.
int sim_search_collect(const float* q3, int n, const float* refc3, int m, float cell, int max_cells, int split,
                       const int32_t* warm_ids, const float* caps, const float* motion, int32_t* ids, float* d2,
                       int32_t* pos, int32_t* ref_ids, float* ref_d2, int32_t* ref_pos, float* vq_out, float* vpts_out,
                       float* rv) {
  SimGrid S;
  build(S, refc3, m, cell, max_cells, split);
  std::vector<int> pos_of(m);
  for (int i = 0; i < m; ++i) pos_of[ls::f2i(S.pts[i].w)] = i;
  ls::GridView v{S.top.data(), S.tab1.data(), S.pts.data(), S.pyr.data(), S.topmask.data()};
  std::vector<float4> vq(n, make_float4(0.f, 0.f, 0.f, 0.f)), vpts((size_t)LS_VK * n, make_float4(0.f, 0.f, 0.f, 0.f));
  ls::VLists L{vq.data(), vpts.data(), n};
  for (int i = 0; i < n; ++i) {
    const float qx = q3[3 * i], qy = q3[3 * i + 1], qz = q3[3 * i + 2];
    const int warm = (warm_ids[i] >= 0 && m > 0) ? pos_of[warm_ids[i]] : -1;
    const ls::Best r = ls::nn_search(S.g, v, qx, qy, qz, warm, caps[i]);
    const ls::Best b = ls::nn_search_collect(S.g, v, L, i, qx, qy, qz, warm, caps[i], motion[i]);
    ids[i] = b.idx; d2[i] = b.d2; pos[i] = b.pos;
    ref_ids[i] = r.idx; ref_d2[i] = r.d2; ref_pos[i] = r.pos;
    // the first candidate, as nn_search_collect takes it
    ls::Best f;
    f.d2 = caps[i]; f.idx = INT_MAX; f.pos = -1;
    if (m > 0) {
      if (warm >= 0) ls::consider(S.pts.data(), warm, qx, qy, qz, f);
      else ls::seed_query(S.g, v, qx, qy, qz, f);
    }
    rv[i] = m > 0 ? ls::vlist_radius(f.pos >= 0, f.d2, caps[i], motion[i]) : 0.0f;
  }
  for (int i = 0; i < n; ++i) {
    const float4 h = vq[i];
    vq_out[4 * i] = h.x; vq_out[4 * i + 1] = h.y; vq_out[4 * i + 2] = h.z; vq_out[4 * i + 3] = h.w;
  }
  for (size_t k = 0; k < (size_t)LS_VK * n; ++k) {
    float4 c = vpts[k];
    const int p = ls::f2i(c.w);
    if (ls::f2i(vq[k % n].w) != 0 && (int)(k / n) < (int)(ls::f2i(vq[k % n].w) & 15)) c.w = ls::i2f(ls::f2i(S.pts[p].w));
    vpts_out[4 * k] = c.x; vpts_out[4 * k + 1] = c.y; vpts_out[4 * k + 2] = c.z; vpts_out[4 * k + 3] = c.w;
  }
  return LS_VK;
}
}
