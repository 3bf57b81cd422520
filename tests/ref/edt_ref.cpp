// Reference of the distance map (test infrastructure only; the rules are DESIGN.md §4b''''''''').  Three parts, sequential:
//   edt_obstacles  the obstacle grid of a box from the known voxels (packed keys, float log-odds), L_occ and the mode
//   edt_transform  an exact separable EDT: Felzenszwalb-Huttenlocher lower envelopes along x, then y, then z, in int64 and
//                  uncapped, with the envelope's breakpoints kept as exact fractions.  A breakpoint belongs to the lower site,
//                  so each pass takes the least value first and the lower coordinate second.  The cap is applied at the end
//   edt_query      the query rule
#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>
#include <vector>

namespace {

constexpr int64_t kInf = std::numeric_limits<int64_t>::max();

struct Frac {  // num / den, den > 0
  int64_t num, den;
};
bool less_eq(const Frac& a, const Frac& b) { return (__int128)a.num * b.den <= (__int128)b.num * a.den; }
bool less_than_int(const Frac& a, int64_t x) { return (__int128)a.num < (__int128)x * a.den; }

// One line: f[i] (kInf = no site), lab[i] the label its site carries.  Writes the lower envelope's value and label.
// v: the envelope's sites; z[k] (k >= 1): where site v[k] starts to be strictly below v[k - 1] (v[0] starts at -infinity).
void envelope(std::vector<int64_t>& f, std::vector<int32_t>& lab, std::vector<int>& v, std::vector<Frac>& z) {
  const int n = (int)f.size();
  int k = -1;
  for (int q = 0; q < n; ++q) {
    if (f[q] == kInf) continue;
    if (k < 0) {
      k = 0;
      v[0] = q;
      continue;
    }
    for (;;) {
      const int p = v[k];
      const Frac s{(f[q] + (int64_t)q * q) - (f[p] + (int64_t)p * p), 2 * (int64_t)(q - p)};
      if (k > 0 && less_eq(s, z[k])) {  // v[k] is nowhere strictly below both neighbours
        --k;
        continue;
      }
      ++k;
      v[k] = q;
      z[k] = s;
      break;
    }
  }
  std::vector<int64_t> out(n, kInf);
  std::vector<int32_t> olab(n, -1);
  if (k >= 0) {
    const int top = k;
    k = 0;
    for (int x = 0; x < n; ++x) {
      while (k < top && less_than_int(z[k + 1], x)) ++k;
      const int64_t d = (int64_t)(x - v[k]);
      out[x] = d * d + f[v[k]];
      olab[x] = lab[v[k]];
    }
  }
  f.swap(out);
  lab.swap(olab);
}

}  // namespace

extern "C" {

// grid: size[0] * size[1] * size[2] bytes, cell (x, y, z) at (z * size[1] + y) * size[0] + x; 1 = obstacle.
void edt_obstacles(const uint64_t* keys, const float* log_odds, int64_t n, float l_occ, const int* kmin, const int* size,
                   int unknown_occ, uint8_t* grid) {
  const int64_t cells = (int64_t)size[0] * size[1] * size[2];
  std::memset(grid, unknown_occ ? 1 : 0, (size_t)cells);
  for (int64_t i = 0; i < n; ++i) {
    int c[3];
    bool in = true;
    for (int a = 0; a < 3; ++a) {
      c[a] = (int)((keys[i] >> (16 * a)) & 0xffff) - kmin[a];
      in = in && c[a] >= 0 && c[a] < size[a];
    }
    if (!in) continue;
    const bool occ = log_odds[i] >= l_occ;
    grid[((int64_t)c[2] * size[1] + c[1]) * size[0] + c[0]] = occ ? 1 : 0;
  }
}

// s_out: per cell the squared distance in cells, M when above M; site_out: the obstacle's cell index, -1 when none.
void edt_transform(const uint8_t* grid, const int* size, int64_t M, int32_t* s_out, int32_t* site_out) {
  const int64_t sx = size[0], sy = size[1], sz = size[2], cells = sx * sy * sz;
  std::vector<int64_t> val(cells);
  std::vector<int32_t> lab(cells);
  for (int64_t i = 0; i < cells; ++i) val[i] = grid[i] ? 0 : kInf, lab[i] = grid[i] ? (int32_t)i : -1;
  const int64_t step[3] = {1, sx, sx * sy};
  for (int a = 0; a < 3; ++a) {
    const int n = size[a];
    std::vector<int64_t> f(n);
    std::vector<int32_t> l(n);
    std::vector<int> v(n);
    std::vector<Frac> z(n + 1);
    for (int64_t zc = 0; zc < sz; ++zc)
      for (int64_t yc = 0; yc < sy; ++yc)
        for (int64_t xc = 0; xc < sx; ++xc) {
          const int64_t c[3] = {xc, yc, zc};
          if (c[a] != 0) continue;  // one line per start cell on this axis
          const int64_t base = xc + yc * sx + zc * sx * sy;
          for (int i = 0; i < n; ++i) f[i] = val[base + i * step[a]], l[i] = lab[base + i * step[a]];
          envelope(f, l, v, z);
          for (int i = 0; i < n; ++i) val[base + i * step[a]] = f[i], lab[base + i * step[a]] = l[i];
        }
  }
  for (int64_t i = 0; i < cells; ++i) {
    const bool keep = val[i] <= M;
    s_out[i] = (int32_t)(keep ? val[i] : M);
    site_out[i] = keep ? lab[i] : -1;
  }
}

// The query rule over a field of edt_transform: float points keyed floor((double)c * (1/res)) + 32768.
void edt_query(const int32_t* s, const int32_t* site, const int* kmin, const int* size, double res, const float* pts3,
               int64_t n, float* dist, int32_t* sq, float* obst3) {
  const double inv = 1.0 / res;
  const float nan = std::numeric_limits<float>::quiet_NaN();
  for (int64_t i = 0; i < n; ++i) {
    int c[3];
    bool in = true;
    for (int a = 0; a < 3; ++a) {
      const double f = std::floor((double)pts3[3 * i + a] * inv);
      if (!(f >= -32768.0 && f < 32768.0)) {
        in = false;
        break;
      }
      c[a] = (int)f + 32768 - kmin[a];
      in = in && c[a] >= 0 && c[a] < size[a];
    }
    float* o = obst3 + 3 * i;
    if (!in) {
      dist[i] = -1.0f, sq[i] = -1, o[0] = o[1] = o[2] = nan;
      continue;
    }
    const int64_t cell = ((int64_t)c[2] * size[1] + c[1]) * size[0] + c[0];
    sq[i] = s[cell];
    dist[i] = (float)((double)(float)std::sqrt((double)s[cell]) * res);
    const int32_t w = site[cell];
    if (w < 0) {
      o[0] = o[1] = o[2] = nan;
      continue;
    }
    const int w3[3] = {w % size[0], (w / size[0]) % size[1], w / size[0] / size[1]};
    for (int a = 0; a < 3; ++a) o[a] = (float)(((double)(kmin[a] + w3[a] - 32768) + 0.5) * res);
  }
}

}  // extern "C"
