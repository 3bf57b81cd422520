// laser_slam::DistanceMap over ls_distance_map_* (include/laser_slam/distance_map.hpp).
#include "laser_slam/distance_map.hpp"

#include <mutex>
#include <stdexcept>
#include <string>

namespace laser_slam {

namespace {
void throwOnError(ls_ctx* ctx, int rc, const char* what) {
  if (rc < 0) throw std::runtime_error(std::string(what) + ": " + ls_b200_last_error(ctx));
}
}  // namespace

constexpr float DistanceMap::distanceValue_Error;
constexpr int DistanceMap::distanceInCellsValue_Error;

DistanceMap::DistanceMap(float maxdist, OccupancyMap& map, const kindr::minimal::Position& bbx_min,
                         const kindr::minimal::Position& bbx_max, bool treat_unknown_as_occupied)
    : map_(map), ctx_(map.ctx_) {
  ls_distance_map_params p;
  p.max_dist = maxdist;
  for (int a = 0; a < 3; ++a) p.bbx_min[a] = (float)bbx_min[a], p.bbx_max[a] = (float)bbx_max[a];
  p.treat_unknown_as_occupied = treat_unknown_as_occupied ? 1 : 0;
  throwOnError(ctx_, ls_distance_map_create(ctx_, &p, &dm_), "ls_distance_map_create");
}

DistanceMap::~DistanceMap() { ls_distance_map_destroy(dm_); }

void DistanceMap::update(ls_distance_map_stats* stats) {
  ls_distance_map_stats st;
  {
    std::lock_guard<std::mutex> lock(map_.mutex_);
    throwOnError(ctx_, ls_distance_map_update(dm_, map_.map_, &st), "ls_distance_map_update");
  }
  max_dist_ = st.max_dist;
  max_sqdist_cells_ = st.max_sqdist_cells;
  if (stats) *stats = st;
}

void DistanceMap::getDistances(const std::vector<kindr::minimal::Position>& points, std::vector<float>* distances,
                               std::vector<int>* squared_distances_in_cells,
                               std::vector<kindr::minimal::Position>* closest) const {
  const size_t n = points.size();
  std::vector<float> p(3 * n), d(n > 0 ? n : 1), o(3 * (n > 0 ? n : 1));
  std::vector<int32_t> s(n > 0 ? n : 1);
  for (size_t i = 0; i < n; ++i)
    for (int a = 0; a < 3; ++a) p[3 * i + a] = (float)points[i][a];
  throwOnError(ctx_,
               ls_distance_map_query(dm_, p.data(), (int)n, distances ? d.data() : NULL,
                                     squared_distances_in_cells ? s.data() : NULL, closest ? o.data() : NULL, NULL),
               "ls_distance_map_query");
  if (distances) distances->assign(d.begin(), d.begin() + (std::ptrdiff_t)n);
  if (squared_distances_in_cells) squared_distances_in_cells->assign(s.begin(), s.begin() + (std::ptrdiff_t)n);
  if (closest) {
    closest->resize(n);
    for (size_t i = 0; i < n; ++i) (*closest)[i] = kindr::minimal::Position{o[3 * i], o[3 * i + 1], o[3 * i + 2]};
  }
}

float DistanceMap::getDistance(const kindr::minimal::Position& p) const {
  std::vector<float> d;
  getDistances(std::vector<kindr::minimal::Position>{p}, &d);
  return d[0];
}

void DistanceMap::getDistanceAndClosestObstacle(const kindr::minimal::Position& p, float& dist,
                                                kindr::minimal::Position& closest) const {
  std::vector<float> d;
  std::vector<kindr::minimal::Position> c;
  getDistances(std::vector<kindr::minimal::Position>{p}, &d, NULL, &c);
  dist = d[0];
  closest = c[0];
}

int DistanceMap::getSquaredDistanceInCells(const kindr::minimal::Position& p) const {
  std::vector<int> s;
  getDistances(std::vector<kindr::minimal::Position>{p}, NULL, &s);
  return s[0];
}

}  // namespace laser_slam
