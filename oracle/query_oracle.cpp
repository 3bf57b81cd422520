// Query oracle (test infrastructure only): volumetric_mapping's WorldBase queries and octomap's castRay restated
// sequentially from oracle/QUERIES.md over an occupancy map's known voxels (ascending packed keys and their log-odds, as
// occo_download gives them).  It is built from occupancy_oracle.cpp itself, so keys, the norm and computeRayKeys are
// the insert oracle's own code; built with the same flags (-ffp-contract=off).
#include "occupancy_oracle.cpp"

#include <cstring>

namespace {

const int kFree = 0, kOccupied = 1, kUnknown = 2;                         // LS_CELL_*
const int kInvalid = 0, kHit = 1, kRayUnknown = 2, kMaxRange = 3, kKeyBound = 4;  // LS_RAY_*
const uint64_t kNone = ~0ull;

float nan_value() {
  const uint32_t bits = 0x7fc00000u;
  float f;
  std::memcpy(&f, &bits, sizeof f);
  return f;
}

struct Known {
  Params P;
  const uint64_t* keys;
  const float* vals;
  int64_t n;
  int64_t visited = 0;

  // LS_CELL_* of voxel k (binary search over the known keys); *v its log-odds when known
  int state(const int k[3], float* v = nullptr) {
    ++visited;
    const uint64_t key = pack(k);
    const uint64_t* it = std::lower_bound(keys, keys + n, key);
    if (it == keys + n || *it != key) return kUnknown;
    const float x = vals[it - keys];
    if (v) *v = x;
    return x >= P.l_occ ? kOccupied : kFree;
  }
};

Known known_of(const double* prm, const uint64_t* keys, const float* vals, int64_t n) {
  Known K{};
  K.P.res = prm[0];
  K.P.inv = 1.0 / prm[0];
  K.P.l_occ = logodds(prm[5]);
  K.keys = keys;
  K.vals = vals;
  K.n = n;
  return K;
}

// octomap's search(double x, double y, double z): the key of the double coordinate
bool key_of_double(const Params& P, double c, int* k) {
  const double s = std::floor(c * P.inv);
  if (!(s >= -(double)kKeyMax && s < (double)kKeyMax)) return false;
  *k = (int)s + (int)kKeyMax;
  return true;
}

// getLineStatus / getVisibility from s to e (float)
int line(Known& K, const float s[3], const float e[3], int stop_at_unknown, uint64_t* first) {
  std::vector<uint64_t> ray;
  *first = kNone;
  ray_keys(K.P, s, e, &ray);
  for (uint64_t key : ray) {
    const int k[3] = {(int)(key & 0xffff), (int)((key >> 16) & 0xffff), (int)((key >> 32) & 0xffff)};
    const int st = K.state(k);
    if (st == kOccupied || (st == kUnknown && stop_at_unknown)) {
      *first = key;
      return st;
    }
  }
  return kFree;
}

float centre(const Params& P, int k) { return (float)(((double)(k - (int)kKeyMax) + 0.5) * P.res); }

// octomap's castRay
int cast_ray(Known& K, const float o[3], const float d[3], int ignore_unknown, double max_range, float end[3]) {
  const Params& P = K.P;
  int k[3];
  if (!key3(P, o, k)) return kInvalid;
  const int s0 = K.state(k);
  if (s0 == kOccupied || (s0 == kUnknown && !ignore_unknown)) {
    for (int a = 0; a < 3; ++a) end[a] = centre(P, k[a]);
    return s0 == kOccupied ? kHit : kRayUnknown;
  }
  float dir[3] = {d[0], d[1], d[2]};
  const double len = norm3(dir);
  if (len > 0.0) {
    const float fl = (float)len;
    for (int a = 0; a < 3; ++a) dir[a] = dir[a] / fl;
  }
  int step[3];
  double tmax[3], tdelta[3];
  for (int i = 0; i < 3; ++i) {
    step[i] = dir[i] > 0.0f ? 1 : (dir[i] < 0.0f ? -1 : 0);
    if (step[i] != 0) {
      double border = ((double)(k[i] - (int)kKeyMax) + 0.5) * P.res;
      border += (double)step[i] * P.res * 0.5;  // castRay keeps the half step in double
      tmax[i] = (border - (double)o[i]) / (double)dir[i];
      tdelta[i] = P.res / (double)std::fabs(dir[i]);
    } else {
      tmax[i] = DBL_MAX;
      tdelta[i] = DBL_MAX;
    }
  }
  if (step[0] == 0 && step[1] == 0 && step[2] == 0) return kInvalid;
  const bool range = max_range > 0.0;
  const double range_sq = max_range * max_range;
  for (;;) {
    int dim;
    if (tmax[0] < tmax[1]) dim = tmax[0] < tmax[2] ? 0 : 2;
    else dim = tmax[1] < tmax[2] ? 1 : 2;
    if ((step[dim] < 0 && k[dim] == 0) || (step[dim] > 0 && k[dim] == 65535)) {
      for (int a = 0; a < 3; ++a) end[a] = centre(P, k[a]);
      return kKeyBound;
    }
    k[dim] += step[dim];
    tmax[dim] += tdelta[dim];
    for (int a = 0; a < 3; ++a) end[a] = centre(P, k[a]);
    if (range) {
      double dist = 0.0;
      for (int a = 0; a < 3; ++a) {
        const float x = end[a] - o[a];
        dist += (double)(x * x);
      }
      if (dist > range_sq) return kMaxRange;
    }
    const int s = K.state(k);
    if (s == kOccupied) return kHit;
    if (s == kUnknown && !ignore_unknown) return kRayUnknown;
  }
}

}  // namespace

extern "C" {

// prm as occo_create (only the resolution and the occupancy threshold are read); keys ascending.  Returns keys visited.
int64_t occo_cell_status(const double* prm, const uint64_t* keys, const float* vals, int64_t nk, const double* pts3, int n,
                         int8_t* status, float* log_odds) {
  Known K = known_of(prm, keys, vals, nk);
  for (int i = 0; i < n; ++i) {
    int k[3];
    int st = kUnknown;
    float v = nan_value();
    if (key_of_double(K.P, pts3[3 * i], &k[0]) && key_of_double(K.P, pts3[3 * i + 1], &k[1]) &&
        key_of_double(K.P, pts3[3 * i + 2], &k[2])) {
      st = K.state(k, &v);
      if (st == kUnknown) v = nan_value();
    }
    status[i] = (int8_t)st;
    if (log_odds) log_odds[i] = v;
  }
  return K.visited;
}

// Plain lines (box3 NULL) or getLineStatusBoundingBox's loop (box3: the box size).  Returns keys visited.
int64_t occo_line_status(const double* prm, const uint64_t* keys, const float* vals, int64_t nk, const double* s3,
                         const double* e3, int n, const double* box3, int stop_at_unknown, int8_t* status, uint64_t* first) {
  Known K = known_of(prm, keys, vals, nk);
  for (int i = 0; i < n; ++i) {
    uint64_t fk = kNone;
    int st = kFree;
    if (!box3) {
      const float s[3] = {(float)s3[3 * i], (float)s3[3 * i + 1], (float)s3[3 * i + 2]};
      const float e[3] = {(float)e3[3 * i], (float)e3[3 * i + 1], (float)e3[3 * i + 2]};
      st = line(K, s, e, stop_at_unknown, &fk);
    } else {
      double disc[3], half[3];
      for (int a = 0; a < 3; ++a) {
        disc[a] = box3[a] / std::ceil((box3[a] + 0.001) / K.P.res);
        if (disc[a] <= 0.0) disc[a] = 1.0;
        half[a] = box3[a] * 0.5;
      }
      for (double x = -half[0]; x <= half[0] && st == kFree; x += disc[0]) {
        for (double y = -half[1]; y <= half[1] && st == kFree; y += disc[1]) {
          for (double z = -half[2]; z <= half[2] && st == kFree; z += disc[2]) {
            const double off[3] = {x, y, z};
            float s[3], e[3];
            for (int a = 0; a < 3; ++a) {
              s[a] = (float)(s3[3 * i + a] + off[a]);
              e[a] = (float)(e3[3 * i + a] + off[a]);
            }
            st = line(K, s, e, stop_at_unknown, &fk);
          }
        }
      }
    }
    status[i] = (int8_t)st;
    if (first) first[i] = fk;
  }
  return K.visited;
}

// castRay per ray (float triples); ends3 NaN for an invalid ray.  Returns keys visited.
int64_t occo_cast_rays(const double* prm, const uint64_t* keys, const float* vals, int64_t nk, const float* o3, const float* d3,
                       int n, int ignore_unknown, double max_range, int8_t* result, float* ends3) {
  Known K = known_of(prm, keys, vals, nk);
  for (int i = 0; i < n; ++i) {
    float e[3] = {nan_value(), nan_value(), nan_value()};
    const int r = cast_ray(K, o3 + 3 * i, d3 + 3 * i, ignore_unknown, max_range, e);
    if (r == kInvalid) e[0] = e[1] = e[2] = nan_value();
    result[i] = (int8_t)r;
    if (ends3)
      for (int a = 0; a < 3; ++a) ends3[3 * i + a] = e[a];
  }
  return K.visited;
}

}  // extern "C"
