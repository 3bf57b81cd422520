// GPU-resident spatial hash of the local map and the exact nearest-neighbour query over it.
//
// Replaces libnabo's kd-tree behind libpointmatcher's KDTreeMatcher{knn 1, epsilon 0} (reference
// laser_slam/configurations/icp_default.yaml:9-12, executed inside icp_.compute at reference
// laser_slam/src/laser_track.cpp:496).  Result contract (oracle/icp_oracle.cpp, SURVEY.md §8c):
//   id  = argmin_j (d2(q, p_j), j) lexicographic  -> lowest reference index wins exact ties
//   d2  = fl(fl(fl(dx*dx) + fl(dy*dy)) + fl(dz*dz)), float32, no FMA
//
// Structure: a two-level sparse voxel grid under an occupancy pyramid.  The hash of a point is its lattice
// cell -- a perfect hash over the map's bounding box, so a lookup is one indexed load, never a probe sequence:
//   level 0  dense array of cells of edge H0 over the bounding box                (Entry top[nx*ny*nz])
//   level 1  a cell holding more than `leaf_split` points owns ONE direct table of LS_FB^3 fine cells of
//            edge H0/LS_FB (LS_FB = 8: 12.5 cm at H0 = 1 m)
//   above    occupancy pyramid: 64-bit child masks at edges H0*4^l, at most LS_PYR_LEVELS levels, up to a single
//            root or a row of top cells (empty-space skipping for wide balls, greedy seed for cold queries)
// Points are stored sorted by (level-0 cell, fine cell), x fastest, as float4 {x, y, z, original index bits}:
// every cell is one contiguous range and a row of x-adjacent fine cells is one contiguous candidate run.
// Why two levels with a wide table (round 1 went through a three-level 4x4x4 design first): the query is
// latency bound on DEPENDENT loads; top entry -> row entries (all independent) -> candidates is three round
// trips, where the 4-ary hierarchy needed one more per sub-cell of every level.
//
// Exactness: the query is a ball query around a real candidate (the previous iteration's match, or a seed found
// by descending the grid), radius sqrt(best).  Loop bounds come from the same monotone float cell-coordinate
// function that binned the points, so they are a superset of the cells a closer point could be in; per-cell
// pruning uses a geometric lower bound widened by `margin` and is only taken when strictly greater than the
// current best, so ties are never pruned.
//
// This header is also compiled for the host by tests/sim (CPU simulation of the query against brute force).
// The product never runs it on the CPU.
#pragma once
#include <cfloat>
#include <climits>
#include <cstring>

#include <vector_types.h>
#include <vector_functions.h>

#include "ls_math.cuh"

#define LS_FB 8  // fine cells per level-0 cell edge (12.5 cm at H0 = 1 m); a table's 8x8 rows fill GridView::topmask
#define LS_FB3 (LS_FB * LS_FB * LS_FB)
// occupancy pyramid levels above level 0, at most.  A top cell covers 4^7 = 16384 level-0 cells per axis, so the top
// level of a map longer than that along one axis (up to 2^22 cells: the device caps max_cells there) holds several
// cells; pyramid_query and seed_query walk all of them.
#define LS_PYR_LEVELS 7

namespace ls {

struct Entry {
  uint32_t start;  // first sorted position of the cell's points
  int32_t meta;    // >= 0: leaf holding `meta` points;  < 0: internal, child table index = ~meta
};

struct Grid {
  float org[3];  // lower corner of the level-0 lattice, centred coordinates
  float H0, H1;      // H1 = H0 / LS_FB
  float inv0, inv1;
  int dim[3];
  int n_cells0;
  float margin;     // absolute slack (metres) covering float rounding of cell boundaries
  float mu[3];      // reference mean (float32) subtracted from the map
  int m;            // number of map points
  int leaf_split;   // a cell with more points than this is subdivided
  int n_tab1;
  int overflow;     // set if a table pool was exhausted (cells then stay leaves: slower, still exact)
  // occupancy pyramid above level 0: level l (1..n_pyr) has cells of edge H0*4^l, each a 64-bit mask
  // of its non-empty 4x4x4 children; the top level is a single cell unless an axis spans more than 4^LS_PYR_LEVELS
  // level-0 cells.
  int n_pyr;
  int pdim[LS_PYR_LEVELS + 1][3];   // pdim[0] == dim
  int poff[LS_PYR_LEVELS + 1];      // offset of level l's masks in GridView::pyr (poff[0] unused)
  int n_pyr_cells;
};

struct GridView {
  const Entry* top;
  const Entry* tab1;  // fine tables, LS_FB3 entries each (all leaves)
  const float4* pts;  // sorted {x,y,z,idx}
  const unsigned long long* pyr;  // occupancy masks, levels 1..n_pyr
  // per level-0 cell that owns a fine table: bit (z*LS_FB + y) set iff row (z, y) of the table holds a point (64
  // rows).  Surfaces leave most rows of a table empty; the mask -- fetched together with the cell's entry, same
  // index -- lets the ball query skip them without touching their entries.  Meaningless for other cells.
  const unsigned long long* topmask;
};

// Accumulator of the traversal.  `bound()` is the squared distance beyond which a candidate cannot matter
// (cells are pruned against it), `offer()` takes one candidate.  Best = 1-NN with the lowest-index tie-break.
struct Best {
  float d2;
  int idx;  // original reference index
  int pos;  // sorted position
  LS_HD float bound() const { return d2; }
  LS_HD void offer(float d, int i, int p) {
    if (d < d2 || (d == d2 && i < idx)) {
      d2 = d;
      idx = i;
      pos = p;
    }
  }
  LS_HD void offer_pt(float d, const float4& c, int p);
};

// K nearest (K <= LS_KNN_MAX at run time), ascending by (d2, index); a candidate offered twice is kept once.
#define LS_KNN_MAX 16
struct TopK {
  float d[LS_KNN_MAX];
  int id[LS_KNN_MAX];
  int k;
  float cap;  // only candidates with d2 <= cap are of interest in this round
  LS_HD void reset(int kk) {
    k = kk;
    cap = INFINITY;
    for (int j = 0; j < LS_KNN_MAX; ++j) { d[j] = INFINITY; id[j] = INT_MAX; }
  }
  LS_HD float bound() const { return fminf(d[k - 1], cap); }
  LS_HD void offer(float dist, int i, int) {
    if (dist > cap || !(dist < d[k - 1] || (dist == d[k - 1] && i < id[k - 1]))) return;
    for (int j = 0; j < k; ++j)
      if (id[j] == i) return;  // already listed (the balls of successive rounds overlap)
    int j = k - 1;
    while (j > 0 && (dist < d[j - 1] || (dist == d[j - 1] && i < id[j - 1]))) {
      d[j] = d[j - 1];
      id[j] = id[j - 1];
      --j;
    }
    d[j] = dist;
    id[j] = i;
  }
  LS_HD void offer_pt(float dist, const float4& c, int p);
};

// tests/sim instruments the query (candidates examined, table entries loaded) to tune H0/leaf_split
#if defined(LS_SIM_COUNTERS) && !defined(__CUDA_ARCH__)
extern thread_local long long ls_sim_cand, ls_sim_entries, ls_sim_steps;
#define LS_CNT_CAND() (++ls_sim_cand)
#define LS_CNT_ENTRY() (++ls_sim_entries)
#define LS_CNT_STEP() (++ls_sim_steps)   /* one dependent round trip to memory */
#else
#define LS_CNT_CAND() ((void)0)
#define LS_CNT_ENTRY() ((void)0)
#define LS_CNT_STEP() ((void)0)
#endif

#if defined(__CUDA_ARCH__)
LS_HD float4 ld_pt(const float4* p) { return __ldg(p); }
LS_HD Entry ld_entry(const Entry* e) {
  const int2 v = __ldg(reinterpret_cast<const int2*>(e));
  Entry r;
  r.start = (uint32_t)v.x;
  r.meta = v.y;
  return r;
}
LS_HD int f2i(float f) { return __float_as_int(f); }
LS_HD float i2f(int i) { return __int_as_float(i); }
LS_HD float4 ld_state4(const float4* p) { return __ldcg(p); }   // per-query state crosses CTAs: L2, never L1
LS_HD void st_state4(float4* p, const float4 v) { __stcg(p, v); }
LS_HD unsigned long long ld_mask(const unsigned long long* p) { return __ldg(p); }
LS_HD unsigned long long ld_rows(const unsigned long long* p) { return __ldg(p); }
LS_HD int ctz64(unsigned long long m) { return __ffsll((long long)m) - 1; }
#else
LS_HD float4 ld_pt(const float4* p) { LS_CNT_CAND(); return *p; }
LS_HD Entry ld_entry(const Entry* e) { LS_CNT_ENTRY(); return *e; }
LS_HD int f2i(float f) { int i; std::memcpy(&i, &f, 4); return i; }
LS_HD float i2f(int i) { float f; std::memcpy(&f, &i, 4); return f; }
LS_HD float4 ld_state4(const float4* p) { return *p; }
LS_HD void st_state4(float4* p, const float4 v) { *p = v; }
LS_HD unsigned long long ld_mask(const unsigned long long* p) { LS_CNT_ENTRY(); return *p; }
LS_HD unsigned long long ld_rows(const unsigned long long* p) { return *p; }
LS_HD int ctz64(unsigned long long m) { return __builtin_ctzll(m); }
#endif

// Monotone (non-decreasing in v) cell coordinate functions; the SAME functions bin the map points
// at build time and bound the query loops.
LS_HD int coord_top(float v, float o, float inv, int n) {
  float t = floorf((v - o) * inv);
  t = fminf(fmaxf(t, 0.0f), (float)(n - 1));
  return (int)t;
}
LS_HD int coord_sub(float v, float lo, float inv) {
  float t = floorf((v - lo) * inv);
  t = fminf(fmaxf(t, 0.0f), (float)(LS_FB - 1));
  return (int)t;
}
LS_HD float cell_lo(float o, int c, float H) { return o + (float)c * H; }

// distance from q to the slab [lo - m, hi + m] (0 inside)
LS_HD float gap(float q, float lo, float hi, float m) {
  const float a = (lo - m) - q;
  const float b = q - (hi + m);
  return fmaxf(0.0f, fmaxf(a, b));
}

// prune iff lower_bound * kShrink > best: kShrink absorbs the relative rounding of the bound itself
#define LS_SHRINK 0.999999f

LS_HD float ball_radius(float best_d2, float margin) { return sqrtf(best_d2) * 1.000001f + margin; }

// The candidate test (for Best: branch-free selects rather than a data-dependent branch per candidate).
LS_HD void Best::offer_pt(float d, const float4& c, int p) { offer(d, f2i(c.w), p); }
LS_HD void TopK::offer_pt(float dist, const float4& c, int p) { offer(dist, f2i(c.w), p); }
template <class Acc>
LS_HD void consider_pt(const float4 p, int pos, float qx, float qy, float qz, Acc& b) {
  b.offer_pt(dist2(qx, qy, qz, p.x, p.y, p.z), p, pos);
}
template <class Acc>
LS_HD void consider(const float4* pts, int pos, float qx, float qy, float qz, Acc& b) {
  consider_pt(ld_pt(pts + pos), pos, qx, qy, qz, b);
}

// candidates are independent loads: issue four before touching any (memory-level parallelism).
template <class Acc>
LS_HD void scan_range(const float4* pts, uint32_t a, uint32_t e, float qx, float qy, float qz, Acc& b) {
  uint32_t pos = a;
  for (; pos + 4 <= e; pos += 4) {
    LS_CNT_STEP();
    const float4 p0 = ld_pt(pts + pos), p1 = ld_pt(pts + pos + 1), p2 = ld_pt(pts + pos + 2), p3 = ld_pt(pts + pos + 3);
    consider_pt(p0, (int)pos, qx, qy, qz, b);
    consider_pt(p1, (int)pos + 1, qx, qy, qz, b);
    consider_pt(p2, (int)pos + 2, qx, qy, qz, b);
    consider_pt(p3, (int)pos + 3, qx, qy, qz, b);
  }
  if (pos < e) LS_CNT_STEP();
  for (; pos < e; ++pos) consider(pts, (int)pos, qx, qy, qz, b);
}

// ---- ball query inside one fine table (all entries are leaves) ---------------------------------------
// Points are sorted x-fastest, so for a row (z, y) the fine cells x0..x1 are ONE contiguous run
// [start(z,y,x0), end(z,y,x1)): two entry loads, then a stream of candidates.
template <class Acc>
LS_HD void visit_fine(const Grid& g, const Entry* tab, unsigned long long rows, float lox, float loy, float loz,
                      const float4* pts, float qx, float qy, float qz, Acc& b) {
  const float R = ball_radius(b.bound(), g.margin);
  const int x0 = coord_sub(qx - R, lox, g.inv1), x1 = coord_sub(qx + R, lox, g.inv1);
  const int y0 = coord_sub(qy - R, loy, g.inv1), y1 = coord_sub(qy + R, loy, g.inv1);
  const int z0 = coord_sub(qz - R, loz, g.inv1), z1 = coord_sub(qz + R, loz, g.inv1);
  for (int z = z0; z <= z1; ++z) {
    const float gz = gap(qz, cell_lo(loz, z, g.H1), cell_lo(loz, z + 1, g.H1), g.margin);
    const float gz2 = gz * gz;
    if (gz2 * LS_SHRINK > b.bound()) continue;
    const Entry* row = tab + (z * LS_FB + y0) * LS_FB;
    for (int y = y0; y <= y1; ++y, row += LS_FB) {
      if (!((rows >> (z * LS_FB + y)) & 1ull)) continue;  // empty row
      const float gy = gap(qy, cell_lo(loy, y, g.H1), cell_lo(loy, y + 1, g.H1), g.margin);
      const float lb = gy * gy + gz2;
      if (lb * LS_SHRINK > b.bound()) continue;
      LS_CNT_STEP();
      const Entry e0 = ld_entry(row + x0);
      const Entry e1 = ld_entry(row + x1);
      scan_range(pts, e0.start, e1.start + (uint32_t)e1.meta, qx, qy, qz, b);
    }
  }
}

// one level-0 cell (leaf scan or fine table)
template <class Acc>
LS_HD void visit_top_entry(const Grid& g, const GridView& v, const Entry e, unsigned long long rows, float cx, float cy,
                           float cz, float qx, float qy, float qz, Acc& b) {
  if (e.meta > 0) {
    scan_range(v.pts, e.start, e.start + (uint32_t)e.meta, qx, qy, qz, b);
  } else if (e.meta < 0) {
    visit_fine(g, v.tab1 + (size_t)(~e.meta) * LS_FB3, rows, cx, cy, cz, v.pts, qx, qy, qz, b);
  }
}
template <class Acc>
LS_HD void visit_top_cell(const Grid& g, const GridView& v, int x, int y, int z, float cx, float cy, float cz, float qx,
                          float qy, float qz, Acc& b) {
  LS_CNT_STEP();
  const size_t ci = ((size_t)z * g.dim[1] + y) * g.dim[0] + x;
  const Entry e = ld_entry(v.top + ci);
  const unsigned long long rows = ld_rows(v.topmask + ci);  // independent of the entry: one round trip for both
  visit_top_entry(g, v, e, rows, cx, cy, cz, qx, qy, qz, b);
}

// ---- large balls: depth-first walk of the occupancy pyramid (empty space costs one mask load per
// 64 cells instead of one entry load per cell) -------------------------------------------------------
template <class Acc>
LS_HDN void pyramid_query(const Grid& g, const GridView& v, float qx, float qy, float qz, Acc& b) {
  int lvl[LS_PYR_LEVELS + 1], bx[LS_PYR_LEVELS + 1], by[LS_PYR_LEVELS + 1], bz[LS_PYR_LEVELS + 1];
  unsigned long long mk[LS_PYR_LEVELS + 1];
  const int* td = g.pdim[g.n_pyr];
  const int n_top = td[0] * td[1] * td[2];  // 1 unless an axis spans more than 4^LS_PYR_LEVELS level-0 cells
  for (int t = 0; t < n_top; ++t) {
    int sp = 0;
    lvl[0] = g.n_pyr;
    bx[0] = (t % td[0]) * 4;
    by[0] = ((t / td[0]) % td[1]) * 4;
    bz[0] = (t / (td[0] * td[1])) * 4;
    mk[0] = ld_mask(v.pyr + g.poff[g.n_pyr] + t);
    while (sp >= 0) {
      if (mk[sp] == 0ull) { --sp; continue; }
      const int bit = ctz64(mk[sp]);
      mk[sp] &= mk[sp] - 1ull;
      LS_CNT_STEP();
      const int cl = lvl[sp] - 1;  // level of the child cell
      const int cx = bx[sp] + (bit & 3), cy = by[sp] + ((bit >> 2) & 3), cz = bz[sp] + (bit >> 4);
      const float Hc = g.H0 * (float)(1 << (2 * cl));
      const float lx = cell_lo(g.org[0], cx, Hc), ly = cell_lo(g.org[1], cy, Hc), lz = cell_lo(g.org[2], cz, Hc);
      const float gx = gap(qx, lx, cell_lo(g.org[0], cx + 1, Hc), g.margin);
      const float gy = gap(qy, ly, cell_lo(g.org[1], cy + 1, Hc), g.margin);
      const float gz = gap(qz, lz, cell_lo(g.org[2], cz + 1, Hc), g.margin);
      const float lb = gx * gx + (gy * gy + gz * gz);
      if (lb * LS_SHRINK > b.bound()) continue;
      if (cl == 0) {
        visit_top_cell(g, v, cx, cy, cz, lx, ly, lz, qx, qy, qz, b);
      } else {
        ++sp;
        lvl[sp] = cl;
        bx[sp] = cx * 4; by[sp] = cy * 4; bz[sp] = cz * 4;
        mk[sp] = ld_mask(v.pyr + g.poff[cl] + ((size_t)cz * g.pdim[cl][1] + cy) * g.pdim[cl][0] + cx);
      }
    }
  }
}

// ---- ball query, level 0 -----------------------------------------------------------------------
template <class Acc>
LS_HD void ball_query(const Grid& g, const GridView& v, float qx, float qy, float qz, Acc& b) {
  const float R = ball_radius(b.bound(), g.margin);
  const int x0 = coord_top(qx - R, g.org[0], g.inv0, g.dim[0]), x1 = coord_top(qx + R, g.org[0], g.inv0, g.dim[0]);
  const int y0 = coord_top(qy - R, g.org[1], g.inv0, g.dim[1]), y1 = coord_top(qy + R, g.org[1], g.inv0, g.dim[1]);
  const int z0 = coord_top(qz - R, g.org[2], g.inv0, g.dim[2]), z1 = coord_top(qz + R, g.org[2], g.inv0, g.dim[2]);
  if ((x1 - x0 + 1) * (y1 - y0 + 1) * (z1 - z0 + 1) > 27 && g.n_pyr > 0) {
    pyramid_query(g, v, qx, qy, qz, b);
    return;
  }
  for (int z = z0; z <= z1; ++z) {
    const float cz = cell_lo(g.org[2], z, g.H0);
    const float gz = gap(qz, cz, cell_lo(g.org[2], z + 1, g.H0), g.margin);
    const float gz2 = gz * gz;
    if (gz2 * LS_SHRINK > b.bound()) continue;
    for (int y = y0; y <= y1; ++y) {
      const float cy = cell_lo(g.org[1], y, g.H0);
      const float gy = gap(qy, cy, cell_lo(g.org[1], y + 1, g.H0), g.margin);
      const float lbyz = gy * gy + gz2;
      if (lbyz * LS_SHRINK > b.bound()) continue;
      for (int x = x0; x <= x1; ++x) {
        const float cx = cell_lo(g.org[0], x, g.H0);
        const float gx = gap(qx, cx, cell_lo(g.org[0], x + 1, g.H0), g.margin);
        const float lb = gx * gx + lbyz;
        if (lb * LS_SHRINK > b.bound()) continue;
        visit_top_cell(g, v, x, y, z, cx, cy, cz, qx, qy, qz, b);
      }
    }
  }
}

// ---- seed: any real candidate close to q (first iteration only; later iterations warm-start) -----
LS_HDN void seed_query(const Grid& g, const GridView& v, float qx, float qy, float qz, Best& b) {
  const int cx = coord_top(qx, g.org[0], g.inv0, g.dim[0]);
  const int cy = coord_top(qy, g.org[1], g.inv0, g.dim[1]);
  const int cz = coord_top(qz, g.org[2], g.inv0, g.dim[2]);
  const Entry e = ld_entry(v.top + ((size_t)cz * g.dim[1] + cy) * g.dim[0] + cx);
  if (e.meta == 0) {
    // empty level-0 cell: greedy descent of the occupancy pyramid towards the nearest occupied child
    // at every level; the first point of the level-0 cell reached is a real (if loose) candidate.
    int X = 0, Y = 0, Z = 0;
    const int* td = g.pdim[g.n_pyr];
    const int n_top = td[0] * td[1] * td[2];
    if (n_top > 1) {  // several top cells (an axis spans more than 4^LS_PYR_LEVELS cells): start in the nearest occupied one
      const float Ht = g.H0 * (float)(1 << (2 * g.n_pyr));
      float best_lb = INFINITY;
      for (int t = 0; t < n_top; ++t) {
        if (ld_mask(v.pyr + g.poff[g.n_pyr] + t) == 0ull) continue;
        const int tx = t % td[0], ty = (t / td[0]) % td[1], tz = t / (td[0] * td[1]);
        const float gx = gap(qx, cell_lo(g.org[0], tx, Ht), cell_lo(g.org[0], tx + 1, Ht), 0.f);
        const float gy = gap(qy, cell_lo(g.org[1], ty, Ht), cell_lo(g.org[1], ty + 1, Ht), 0.f);
        const float gz = gap(qz, cell_lo(g.org[2], tz, Ht), cell_lo(g.org[2], tz + 1, Ht), 0.f);
        const float lb = gx * gx + (gy * gy + gz * gz);
        if (lb < best_lb) { best_lb = lb; X = tx; Y = ty; Z = tz; }
      }
    }
    for (int l = g.n_pyr; l >= 1; --l) {
      unsigned long long mask = ld_mask(v.pyr + g.poff[l] + ((size_t)Z * g.pdim[l][1] + Y) * g.pdim[l][0] + X);
      const float Hc = g.H0 * (float)(1 << (2 * (l - 1)));
      float best_lb = INFINITY;
      int best_bit = -1;
      while (mask) {
        const int bit = ctz64(mask);
        mask &= mask - 1ull;
        const int ccx = X * 4 + (bit & 3), ccy = Y * 4 + ((bit >> 2) & 3), ccz = Z * 4 + (bit >> 4);
        const float gx = gap(qx, cell_lo(g.org[0], ccx, Hc), cell_lo(g.org[0], ccx + 1, Hc), 0.f);
        const float gy = gap(qy, cell_lo(g.org[1], ccy, Hc), cell_lo(g.org[1], ccy + 1, Hc), 0.f);
        const float gz = gap(qz, cell_lo(g.org[2], ccz, Hc), cell_lo(g.org[2], ccz + 1, Hc), 0.f);
        const float lb = gx * gx + (gy * gy + gz * gz);
        if (lb < best_lb) { best_lb = lb; best_bit = bit; }
      }
      if (best_bit < 0) return;  // empty map
      X = X * 4 + (best_bit & 3);
      Y = Y * 4 + ((best_bit >> 2) & 3);
      Z = Z * 4 + (best_bit >> 4);
    }
    const Entry s0 = ld_entry(v.top + ((size_t)Z * g.dim[1] + Y) * g.dim[0] + X);
    if (s0.meta != 0) consider(v.pts, (int)s0.start, qx, qy, qz, b);
    return;
  }
  if (e.meta > 0) { scan_range(v.pts, e.start, e.start + (uint32_t)e.meta, qx, qy, qz, b); return; }
  const float lox = cell_lo(g.org[0], cx, g.H0), loy = cell_lo(g.org[1], cy, g.H0), loz = cell_lo(g.org[2], cz, g.H0);
  const int fx = coord_sub(qx, lox, g.inv1), fy = coord_sub(qy, loy, g.inv1), fz = coord_sub(qz, loz, g.inv1);
  const Entry* tab = v.tab1 + (size_t)(~e.meta) * LS_FB3;
  const Entry e1 = ld_entry(tab + (fz * LS_FB + fy) * LS_FB + fx);
  if (e1.meta != 0) { scan_range(v.pts, e1.start, e1.start + (uint32_t)e1.meta, qx, qy, qz, b); return; }
  // empty home cell: the 3x3 rows around it (x-run of three cells each) almost always hold a close point
  const int xa = fx > 0 ? fx - 1 : 0, xb = fx < LS_FB - 1 ? fx + 1 : LS_FB - 1;
  for (int z = (fz > 0 ? fz - 1 : 0); z <= (fz < LS_FB - 1 ? fz + 1 : LS_FB - 1); ++z)
    for (int y = (fy > 0 ? fy - 1 : 0); y <= (fy < LS_FB - 1 ? fy + 1 : LS_FB - 1); ++y) {
      const Entry r0 = ld_entry(tab + (z * LS_FB + y) * LS_FB + xa);
      const Entry r1 = ld_entry(tab + (z * LS_FB + y) * LS_FB + xb);
      scan_range(v.pts, r0.start, r1.start + (uint32_t)r1.meta, qx, qy, qz, b);
    }
  if (b.pos < 0) consider(v.pts, (int)e.start, qx, qy, qz, b);  // still nothing: any point of the level-0 cell
}

// Exact 1-NN within a squared-distance cap.  warm_pos: sorted position of the previous iteration's
// match, or -1.  cap_d2 = +inf gives the unbounded search of KDTreeMatcher{maxDist: inf}.  With a
// finite cap the result is the exact nearest neighbour whenever its d2 <= cap_d2, and "not found"
// (idx -1, pos -1, d2 +inf) otherwise -- callers use caps that provably do not change what the
// trimmed outlier filter keeps (ls_kernels.cuh, phase A).
LS_HD Best nn_search(const Grid& g, const GridView& v, float qx, float qy, float qz, int warm_pos, float cap_d2) {
  Best b;
  b.d2 = cap_d2;
  b.idx = INT_MAX;
  b.pos = -1;
  if (g.m <= 0) { b.idx = -1; b.d2 = INFINITY; return b; }
  if (warm_pos >= 0) consider(v.pts, warm_pos, qx, qy, qz, b);
  else seed_query(g, v, qx, qy, qz, b);  // candidates beyond the cap are simply not accepted
  ball_query(g, v, qx, qy, qz, b);
  if (b.pos < 0) { b.idx = -1; b.d2 = INFINITY; }
  return b;
}

// ---- certified candidate lists ("Verlet lists") ------------------------------------------------------------------
// Between two ICP iterations a query moves by far less than the distance to its match, so the search result rarely
// changes -- but "rarely" is not "never", and the contract is the EXACT nearest neighbour every iteration.  A list
// makes the repeat provable: during a full search at position q0 the kernel also records EVERY map point within
// R_v = d * ratio (capped by d + skin) of q0, d being the distance of the search's first candidate, an upper bound of
// the match distance (nn_search_collect).  At a later position q (moved by delta = |q - q0|) any
// point NOT in the list is farther than R_v - delta from q, hence: if the best listed candidate lies within
// R_c = R_v - delta (minus rounding slack) it is the exact nearest neighbour -- ties included, since every point at
// that distance is listed too; and if nothing lies within sqrt(cap) <= R_c the capped search provably finds nothing.
// Otherwise the list is refused and the full search runs (and rebuilds the list).  The certificate only ever
// replaces a search by its own proven result: correspondences are bit-identical with or without lists.
//
// Layout (per query i of n, in the kernel's rank order): vq[i] = {q0.x, q0.y, q0.z, bits}, bits = R_v with its low
// 4 mantissa bits replaced by the candidate count (R_v is thereby rounded DOWN: conservative); bits == 0: no list.
// vpts[k*n + i] = candidate k as {x, y, z, sorted position} -- structure of arrays, so a warp streams 512
// contiguous bytes per k.  The original index (tie-break) is fetched from the sorted map only when two candidates
// are exactly equidistant.
#ifndef LS_VK
#define LS_VK 8  // candidates per list; a ball holding more is not listed
#endif
static_assert(LS_VK <= 15, "the list header keeps the candidate count in 4 bits");
// tuning knobs of vlist_radius (tests/sim sweeps them; results never depend on them)
#ifndef LS_VL_ABS
#define LS_VL_ABS 0.0f   // floor of the list margin [m]
#endif
#ifndef LS_VL_REL
#define LS_VL_REL 0.5f   // cap of the list margin relative to the match distance
#endif
#ifndef LS_VL_SKIN
#define LS_VL_SKIN 4.0f  // margin wanted = skin * (how far the last step moved the query)
#endif
#ifndef LS_VL_GATE
#define LS_VL_GATE 1.0f  // build only if motion * gate <= margin
#endif
struct VLists {
  float4* vq;
  float4* vpts;
  int n;  // stride between candidate planes
};

// All points within sqrt(r2) of the query, at most LS_VK of them: one more and the collection gives up (r2 turns
// negative, which prunes every remaining cell and rejects every remaining candidate).
struct Collector {
  float r2;
  int cnt;
  float4* out;
  int stride;
  LS_HD float bound() const { return r2; }
  LS_HD void offer_pt(float d, const float4& c, int p) {
    if (d <= r2) {
      if (cnt < LS_VK) st_state4(out + (size_t)cnt * stride, make_float4(c.x, c.y, c.z, i2f(p)));
      else r2 = -1.0f;
      ++cnt;
    }
  }
};

// Try to answer the capped query (qx,qy,qz) from list i, whose header `v` = vq[i] and first candidate `c0` =
// vpts[i] the caller has already loaded (both addresses are known up front, so the common case -- a one-candidate
// list -- costs a single round trip to memory; a longer list costs one more, its other planes being loaded together).
// true: `b` is exactly what nn_search(.., cap_d2) returns (b.pos < 0: nothing within the cap; b.idx is NOT filled in)
// and cbest = the match's {x, y, z, sorted position}.  false: no valid certificate, run the search.
LS_HD bool vlist_query(const VLists& L, const float4* pts, int i, const float4 v, const float4 c0, float qx, float qy,
                       float qz, float cap_d2, Best& b, float4& cbest) {
  const unsigned int bits = (unsigned int)f2i(v.w);
  if (bits == 0u) return false;
  const int cnt = (int)(bits & 15u);
  const float Rv = i2f((int)(bits & ~15u));
  // rounding slack: fl(d2) carries < 4 ulp relative error, sqrtf is correctly rounded; 4e-6 dwarfs both
  const float Rc = Rv * 0.999996f - sqrtf(dist2(qx, qy, qz, v.x, v.y, v.z)) * 1.000004f;
  if (!(Rc > 0.0f)) return false;
  b.d2 = cap_d2;
  b.idx = INT_MAX;
  b.pos = -1;
  auto take = [&](const float4 c) {  // candidates in ascending k: the order decides nothing but ties
    const float d = dist2(qx, qy, qz, c.x, c.y, c.z);
    const int cpos = f2i(c.w);
    if (d < b.d2) {
      b.d2 = d;
      b.pos = cpos;
      cbest = c;
    } else if (d == b.d2) {
      // exact tie (or d == cap): lowest original index wins, as in Best::offer; indices live in the sorted map
      if (b.pos < 0 || f2i(ld_pt(pts + cpos).w) < f2i(ld_pt(pts + b.pos).w)) {
        b.pos = cpos;
        cbest = c;
      }
    }
  };
  if (cnt > 0) take(c0);  // cnt == 0: nothing within R_v, plane 0 holds no candidate of this list
  // The other planes are independent loads: issue four before comparing any (fixed slots, as in scan_range).  Seven
  // slots, the whole list in one group, measured no faster on the H100 (DESIGN.md §7).
  for (int k0 = 1; k0 < cnt; k0 += 4) {
    float4 cs[4];
#pragma unroll
    for (int u = 0; u < 4; ++u)  // every slot assigned: a slot left unwritten put the array in local memory
      cs[u] = k0 + u < cnt ? ld_state4(L.vpts + (size_t)(k0 + u) * L.n + i) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int u = 0; u < 4; ++u)
      if (k0 + u < cnt) take(cs[u]);
  }
  // b.d2 == cap_d2 when nothing was accepted: then the certificate must cover the whole cap
  return b.d2 * 1.00001f <= Rc * Rc;
}

// The radius of the list to build at a query whose match lies within sqrt(found_d2) (found) -- or of which nothing is
// known inside cap_d2 (!found) -- or 0: no list, it would not pay off.  `motion` bounds how far the last ICP step moved
// this query; steps shrink geometrically, so a list is only worth its collection when its margin (R_v minus the match
// distance) covers about twice that.  A list that is not rebuilt is left as it is: it remains a true statement about
// its own q0.  Any R_v gives a valid certificate (every point within it is listed), so `found_d2` may be any upper
// bound of the match distance.
LS_HD float vlist_radius(bool found, float found_d2, float cap_d2, float motion) {
  float Rv;
  if (found) {
    const float want = sqrtf(found_d2);
    const float margin = fmaxf(want * LS_VL_REL, LS_VL_ABS) + 1e-4f;
    if (!(motion * LS_VL_GATE <= margin)) return 0.0f;
    Rv = want + fminf(margin, fmaxf(0.002f, LS_VL_SKIN * motion));
  } else {
    const float want = sqrtf(cap_d2);  // the cap itself moves a little between iterations: 5 % head room
    if (!(motion <= want * 0.125f)) return 0.0f;
    Rv = want * 1.05f + fminf(want * 0.25f, fmaxf(0.002f, 4.0f * motion));
  }
  return Rv < 3.0e38f ? Rv : 0.0f;
}

// The list header of a collection of radius Rv at (qx,qy,qz) that saw `cnt` points within it.  Every point with
// fl(d2) <= fl(Rv*Rv) is recorded; the stored radius is rounded down twice (1 ulp for the square's rounding, then the
// count bits).  More than LS_VK points: no list.
LS_HD void vlist_head(const VLists& L, int i, float qx, float qy, float qz, float Rv, int cnt) {
  float4 head = make_float4(qx, qy, qz, 0.0f);
  if (cnt <= LS_VK) head.w = i2f((int)((((unsigned int)f2i(Rv * 0.9999999f)) & ~15u) | (unsigned int)cnt));
  st_state4(L.vq + i, head);
}

// The list build in a walk of its own after a search whose answer was `found_d2` (or nothing within cap_d2).  The
// kernel collects in the search's walk instead (nn_search_collect); tests/sim replays this as the reference it compares
// against.
LS_HD void vlist_build(const Grid& g, const GridView& v, const VLists& L, int i, float qx, float qy, float qz, bool found,
                       float found_d2, float cap_d2, float motion) {
  const float Rv = vlist_radius(found, found_d2, cap_d2, motion);
  if (!(Rv > 0.0f)) return;
  Collector c;
  c.r2 = Rv * Rv;
  c.cnt = 0;
  c.out = L.vpts + i;
  c.stride = L.n;
  ball_query(g, v, qx, qy, qz, c);
  vlist_head(L, i, qx, qy, qz, Rv, c.cnt);
}

// The search and the list's collection in one walk: `best` is exactly nn_search's accumulator, `list` collects every
// point within its radius.  The walk covers the larger of the two balls while the list is collecting; once it
// overflows, or when no list is wanted (list.r2 < 0), only the search's ball is left to walk.
struct SearchCollect {
  Best best;
  Collector list;
  LS_HD float bound() const { return fmaxf(best.d2, list.r2); }
  LS_HD void offer_pt(float d, const float4& c, int p) {
    best.offer_pt(d, c, p);
    list.offer_pt(d, c, p);
  }
};

// nn_search(.., warm_pos, cap_d2) that also rebuilds list i at (qx,qy,qz) when that can pay off (vlist_radius).  The
// list radius is fixed before the walk from the first candidate -- the warm start, or the seed -- whose distance bounds
// the match's; walking the search's cells a second time for the list would double the dependent round trips.
LS_HD Best nn_search_collect(const Grid& g, const GridView& v, const VLists& L, int i, float qx, float qy, float qz,
                             int warm_pos, float cap_d2, float motion) {
  SearchCollect s;
  Best& b = s.best;
  b.d2 = cap_d2;
  b.idx = INT_MAX;
  b.pos = -1;
  if (g.m <= 0) { b.idx = -1; b.d2 = INFINITY; return b; }
  // the first candidate goes to the search only: the walk offers it again, and the list must see each point once
  if (warm_pos >= 0) consider(v.pts, warm_pos, qx, qy, qz, b);
  else seed_query(g, v, qx, qy, qz, b);
  const float Rv = vlist_radius(b.pos >= 0, b.d2, cap_d2, motion);
  // No list wanted: r2 < 0 collects nothing and leaves the search's own bound.  The same walk either way, so that the
  // lanes of a warp that build a list and those that do not walk together instead of one group after the other.
  s.list.r2 = Rv > 0.0f ? Rv * Rv : -1.0f;
  s.list.cnt = 0;
  s.list.out = L.vpts + i;
  s.list.stride = L.n;
  ball_query(g, v, qx, qy, qz, s);
  if (Rv > 0.0f) vlist_head(L, i, qx, qy, qz, Rv, s.list.cnt);
  if (b.pos < 0) { b.idx = -1; b.d2 = INFINITY; }
  return b;
}

// Exact K nearest neighbours (ties: lower index first) by verified expanding balls: a round searches the ball of
// radius R exactly (pruned by the running K-th distance); if K points lie inside it they are the K nearest,
// otherwise R doubles.  Fewer than K points in the whole map leaves the tail of the list at +inf / INT_MAX.
LS_HDN void knn_search(const Grid& g, const GridView& v, float qx, float qy, float qz, int k, TopK& t) {
  t.reset(k);
  if (g.m <= 0) return;
  const float extent = g.H0 * (float)(g.dim[0] + g.dim[1] + g.dim[2]) + 1.0f;
  float R = g.H1;
  for (int round = 0; round < 64; ++round) {
    t.cap = R * R;
    ball_query(g, v, qx, qy, qz, t);
    if (t.d[k - 1] <= t.cap) break;  // K points inside the ball: exact
    // the ball already covered every cell (query assumed within ~extent of the map): nothing more to find
    if (R > extent + fabsf(qx - g.org[0]) + fabsf(qy - g.org[1]) + fabsf(qz - g.org[2])) break;
    R = R * 2.0f;
  }
}

// Cell keys used by the build (same functions => same membership as the query assumes).
LS_HD int top_index(const Grid& g, float x, float y, float z) {
  const int cx = coord_top(x, g.org[0], g.inv0, g.dim[0]);
  const int cy = coord_top(y, g.org[1], g.inv0, g.dim[1]);
  const int cz = coord_top(z, g.org[2], g.inv0, g.dim[2]);
  return (cz * g.dim[1] + cy) * g.dim[0] + cx;
}
LS_HD void top_origin(const Grid& g, int c0, float& lox, float& loy, float& loz) {
  const int cx = c0 % g.dim[0];
  const int cy = (c0 / g.dim[0]) % g.dim[1];
  const int cz = c0 / (g.dim[0] * g.dim[1]);
  lox = cell_lo(g.org[0], cx, g.H0);
  loy = cell_lo(g.org[1], cy, g.H0);
  loz = cell_lo(g.org[2], cz, g.H0);
}
LS_HD int sub_index(float x, float y, float z, float lox, float loy, float loz, float inv) {
  return (coord_sub(z, loz, inv) * LS_FB + coord_sub(y, loy, inv)) * LS_FB + coord_sub(x, lox, inv);
}

// Grid geometry from the centred bounding box (single thread on the device; host in tests/sim).
LS_HDN void grid_setup(Grid& g, const float* lo, const float* hi, float cell_size, int max_cells, int leaf_split,
                       int m) {
  float H = cell_size > 0.f ? cell_size : 2.0f;
  float ext[3], emax = 0.f, oabs = 0.f;
  for (int a = 0; a < 3; ++a) {
    ext[a] = hi[a] - lo[a];
    if (!(ext[a] >= 0.f)) ext[a] = 0.f;
    emax = fmaxf(emax, ext[a]);
    oabs = fmaxf(oabs, fmaxf(fabsf(lo[a]), fabsf(hi[a])));
  }
  // grow H (powers of two) until the dense level-0 array fits the budget.  The cells are counted with the float
  // expression that sets `dim` below, so n_cells0 <= max_cells holds exactly (for a cell size that is not a power of
  // two, floor(ext / H) in double can be one less than floorf(ext * (1 / H)) in float).
  for (int it = 0; it < 40; ++it) {
    const float inv = 1.0f / H;
    double cells = 1.0;
    for (int a = 0; a < 3; ++a) cells *= (double)floorf(ext[a] * inv) + 1.0;
    if (cells <= (double)max_cells) break;
    H = H * 2.0f;
  }
  g.H0 = H;
  g.H1 = H / (float)LS_FB;  // LS_FB is a power of two: exact
  g.inv0 = 1.0f / g.H0;
  g.inv1 = 1.0f / g.H1;
  int n = 1;
  for (int a = 0; a < 3; ++a) {
    g.org[a] = lo[a];
    int d = (int)floorf(ext[a] * g.inv0) + 1;
    if (d < 1) d = 1;
    g.dim[a] = d;
    n *= d;
  }
  g.n_cells0 = n;
  g.margin = (oabs + emax + H) * 1.9073486328125e-06f;  // 2^-19 of the coordinate magnitude
  g.m = m;
  g.leaf_split = leaf_split > 0 ? leaf_split : 32;
  g.n_tab1 = 0;
  g.overflow = 0;
  for (int a = 0; a < 3; ++a) g.pdim[0][a] = g.dim[a];
  g.poff[0] = 0;
  int off = 0, l = 0;
  do {
    ++l;
    for (int a = 0; a < 3; ++a) g.pdim[l][a] = (g.pdim[l - 1][a] + 3) / 4;
    g.poff[l] = off;
    off += g.pdim[l][0] * g.pdim[l][1] * g.pdim[l][2];
  } while ((g.pdim[l][0] > 1 || g.pdim[l][1] > 1 || g.pdim[l][2] > 1) && l < LS_PYR_LEVELS);
  g.n_pyr = l;
  g.n_pyr_cells = off;
}

}  // namespace ls
