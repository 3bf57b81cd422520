// Occupancy map oracle (test infrastructure only): laser_to_octomap's insertion loop restated sequentially from the rules
// of oracle/OCCUPANCY.md.  A sorted map of packed voxel key -> float log-odds (two sorted vectors), per-scan free /
// occupied key sets (sorted, de-duplicated), one update per touched voxel per scan.  Built with -ffp-contract=off: every
// float / double operation is rounded on its own, in the order the rules spell out.
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <set>
#include <vector>

namespace {

const int64_t kKeyMax = 32768;  // octomap's tree_max_val: 16-level keys in [0, 65535]

struct Params {
  double res, inv, max_range;
  float l_hit, l_miss, l_min, l_max, l_occ;
};

float logodds(double p) { return (float)std::log(p / (1.0 - p)); }

// floor(c * (1/res)) + 32768, valid iff in [0, 65535]
bool key_of(const Params& P, float c, int* k) {
  const double s = std::floor((double)c * P.inv);
  if (!(s >= -(double)kKeyMax && s < (double)kKeyMax)) return false;
  *k = (int)s + (int)kKeyMax;
  return true;
}
bool key3(const Params& P, const float p[3], int k[3]) {
  return key_of(P, p[0], &k[0]) && key_of(P, p[1], &k[1]) && key_of(P, p[2], &k[2]);
}
uint64_t pack(const int k[3]) { return (uint64_t)k[0] | ((uint64_t)k[1] << 16) | ((uint64_t)k[2] << 32); }

// |v|: squares and sums in float, the root in double
double norm3(const float v[3]) {
  float a = v[0] * v[0], b = v[1] * v[1], c = v[2] * v[2];
  float s = a + b;
  s = s + c;
  return std::sqrt((double)s);
}

// The free cells of one ray (octomap's computeRayKeys).  Returns false (no cells) when either end key is invalid.
bool ray_keys(const Params& P, const float o[3], const float e[3], std::vector<uint64_t>* out) {
  out->clear();
  int ko[3], ke[3];
  if (!key3(P, o, ko) || !key3(P, e, ke)) return false;
  if (ko[0] == ke[0] && ko[1] == ke[1] && ko[2] == ke[2]) return true;
  out->push_back(pack(ko));
  float dir[3] = {e[0] - o[0], e[1] - o[1], e[2] - o[2]};
  const float length = (float)norm3(dir);
  for (int i = 0; i < 3; ++i) dir[i] = dir[i] / length;
  int step[3], cur[3] = {ko[0], ko[1], ko[2]};
  double tmax[3], tdelta[3];
  for (int i = 0; i < 3; ++i) {
    step[i] = dir[i] > 0.0f ? 1 : (dir[i] < 0.0f ? -1 : 0);
    if (step[i] != 0) {
      double border = ((double)(cur[i] - (int)kKeyMax) + 0.5) * P.res;
      border += (double)(float)((double)step[i] * P.res * 0.5);
      tmax[i] = (border - (double)o[i]) / (double)dir[i];
      tdelta[i] = P.res / (double)std::fabs(dir[i]);
    } else {
      tmax[i] = DBL_MAX;
      tdelta[i] = DBL_MAX;
    }
  }
  for (;;) {
    int dim;
    if (tmax[0] < tmax[1]) dim = tmax[0] < tmax[2] ? 0 : 2;
    else dim = tmax[1] < tmax[2] ? 1 : 2;
    cur[dim] += step[dim];
    tmax[dim] += tdelta[dim];
    if (cur[0] == ke[0] && cur[1] == ke[1] && cur[2] == ke[2]) break;
    if (cur[dim] < 0 || cur[dim] > 65535) break;
    const double dist = std::fmin(std::fmin(tmax[0], tmax[1]), tmax[2]);
    if (dist > (double)length) break;
    out->push_back(pack(cur));
  }
  return true;
}

struct Occ {
  Params P;
  std::vector<uint64_t> keys;  // known voxels, ascending packed key
  std::vector<float> vals;
};

}  // namespace

extern "C" {

// prm: resolution, prob_hit, prob_miss, clamp_min, clamp_max, occupancy_threshold, max_range
void* occo_create(const double* prm) {
  Occ* m = new Occ();
  m->P.res = prm[0];
  m->P.inv = 1.0 / prm[0];
  m->P.l_hit = logodds(prm[1]);
  m->P.l_miss = logodds(prm[2]);
  m->P.l_min = logodds(prm[3]);
  m->P.l_max = logodds(prm[4]);
  m->P.l_occ = logodds(prm[5]);
  m->P.max_range = prm[6];
  return m;
}

void occo_destroy(void* h) { delete static_cast<Occ*>(h); }

// One scan: pts4 (n points, x y z w) moved by T (column-major float32, xform_point order; an exact identity copies).
// stats: rays cast, points without a ray, free updates, occupied updates, known voxels after the scan.
void occo_insert(void* h, const float* pts4, int n, const float* T, int64_t* stats) {
  Occ* m = static_cast<Occ*>(h);
  const Params& P = m->P;
  bool identity = true;
  for (int i = 0; i < 16; ++i) identity = identity && T[i] == ((i % 5 == 0) ? 1.f : 0.f);
  const float o[3] = {T[12], T[13], T[14]};
  std::vector<uint64_t> free_cells;
  std::set<uint64_t> occ_cells;
  std::vector<uint64_t> ray;
  int64_t cast = 0, skipped = 0;
  for (int i = 0; i < n; ++i) {
    const float* q = pts4 + 4 * (size_t)i;
    float p[3];
    if (identity) {
      p[0] = q[0], p[1] = q[1], p[2] = q[2];
    } else {
      for (int r = 0; r < 3; ++r) {
        float a = T[r] * q[0], b = T[4 + r] * q[1], c = T[8 + r] * q[2];
        float s = a + b;
        s = s + c;
        p[r] = s + T[12 + r];
      }
    }
    if (!std::isfinite(p[0]) || !std::isfinite(p[1]) || !std::isfinite(p[2])) {
      ++skipped;
      continue;
    }
    int kp[3];
    const bool valid = key3(P, p, kp);
    if (valid && occ_cells.count(pack(kp))) {  // already checked
      ++skipped;
      continue;
    }
    ++cast;
    const float d[3] = {p[0] - o[0], p[1] - o[1], p[2] - o[2]};
    const double len = norm3(d);
    if (P.max_range < 0.0 || len <= P.max_range) {
      if (ray_keys(P, o, p, &ray)) free_cells.insert(free_cells.end(), ray.begin(), ray.end());
      if (valid) occ_cells.insert(pack(kp));
    } else {
      const float fl = (float)len, fr = (float)P.max_range;
      float e[3];
      for (int r = 0; r < 3; ++r) {
        const float u = d[r] / fl;
        const float w = u * fr;
        e[r] = o[r] + w;
      }
      if (ray_keys(P, o, e, &ray)) free_cells.insert(free_cells.end(), ray.begin(), ray.end());
    }
  }
  std::sort(free_cells.begin(), free_cells.end());
  free_cells.erase(std::unique(free_cells.begin(), free_cells.end()), free_cells.end());
  // touched voxels in key order: occupied wins over free
  std::vector<std::pair<uint64_t, float> > upd;
  upd.reserve(free_cells.size() + occ_cells.size());
  int64_t n_free = 0, n_occ = (int64_t)occ_cells.size();
  {
    auto f = free_cells.begin();
    auto o = occ_cells.begin();
    while (f != free_cells.end() || o != occ_cells.end()) {
      if (o != occ_cells.end() && (f == free_cells.end() || *o <= *f)) {
        if (f != free_cells.end() && *f == *o) ++f;
        upd.emplace_back(*o++, P.l_hit);
      } else {
        upd.emplace_back(*f++, P.l_miss);
        ++n_free;
      }
    }
  }
  // merge into the map: v = clamp(v + l), a new voxel starting from 0
  std::vector<uint64_t> keys;
  std::vector<float> vals;
  keys.reserve(m->keys.size() + upd.size());
  vals.reserve(m->keys.size() + upd.size());
  size_t a = 0, b = 0;
  while (a < m->keys.size() || b < upd.size()) {
    if (b == upd.size() || (a < m->keys.size() && m->keys[a] < upd[b].first)) {
      keys.push_back(m->keys[a]);
      vals.push_back(m->vals[a++]);
      continue;
    }
    float v = 0.0f;
    if (a < m->keys.size() && m->keys[a] == upd[b].first) v = m->vals[a++];
    v = v + upd[b].second;
    if (v < P.l_min) v = P.l_min;
    if (v > P.l_max) v = P.l_max;
    keys.push_back(upd[b].first);
    vals.push_back(v);
    ++b;
  }
  m->keys.swap(keys);
  m->vals.swap(vals);
  if (stats) {
    stats[0] = cast;
    stats[1] = skipped;
    stats[2] = n_free;
    stats[3] = n_occ;
    stats[4] = (int64_t)m->keys.size();
  }
}

// which: 1 known, 2 occupied (known and log-odds >= the threshold).  Writes min(count, cap) voxels in ascending key
// order; returns the count.
int64_t occo_download(void* h, int which, uint64_t* keys, float* log_odds, int64_t cap) {
  Occ* m = static_cast<Occ*>(h);
  int64_t k = 0;
  for (size_t j = 0; j < m->keys.size(); ++j) {
    if (which == 2 && !(m->vals[j] >= m->P.l_occ)) continue;
    if (k < cap) {
      if (keys) keys[k] = m->keys[j];
      if (log_odds) log_odds[k] = m->vals[j];
    }
    ++k;
  }
  return k;
}

// The free cells of one ray from o to e at resolution res (cap keys at most); -1 when an end key is invalid.
int64_t occo_ray_keys(double res, const float* o, const float* e, uint64_t* out, int64_t cap) {
  Params P{};
  P.res = res;
  P.inv = 1.0 / res;
  std::vector<uint64_t> ray;
  if (!ray_keys(P, o, e, &ray)) return -1;
  for (size_t i = 0; i < ray.size() && (int64_t)i < cap; ++i) out[i] = ray[i];
  return (int64_t)ray.size();
}

// (float)log(p / (1 - p)), the log-odds both implementations use
float occo_logodds(double p) { return logodds(p); }

}  // extern "C"
