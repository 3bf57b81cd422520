// laser_slam::OccupancyMap over ls_occupancy_* (include/laser_slam/occupancy_map.hpp).
#include "laser_slam/occupancy_map.hpp"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <stdexcept>
#include <string>
#include <tuple>

namespace laser_slam {

namespace {
void throwOnError(ls_ctx* ctx, int rc, const char* what) {
  if (rc < 0) throw std::runtime_error(std::string(what) + ": " + ls_b200_last_error(ctx));
}
}  // namespace

OccupancyMap::OccupancyMap(const OccupancyMapParams& params, IncrementalEstimator& estimator)
    : params_(params), estimator_(estimator), ctx_(estimator.trackContext()) {
  ls_occupancy_params p;
  ls_occupancy_default_params(&p);
  p.resolution = params.resolution;
  p.prob_hit = params.probability_hit;
  p.prob_miss = params.probability_miss;
  p.clamp_min = params.clamping_thres_min;
  p.clamp_max = params.clamping_thres_max;
  p.occupancy_threshold = params.occupancy_thres;
  p.max_range = params.sensor_max_range;
  p.initial_capacity = params.initial_capacity_bricks;
  throwOnError(ctx_, ls_occupancy_create(ctx_, &p, &map_), "ls_occupancy_create");
}

OccupancyMap::~OccupancyMap() { ls_occupancy_destroy(map_); }

void OccupancyMap::insertScan(const LaserTrack& laser_track, const Time& time_ns, ls_occupancy_stats* stats) {
  std::lock_guard<std::mutex> lock(mutex_);
  Trajectory trajectory;
  laser_track.getTrajectory(&trajectory);
  const PointMatcher::TransformationParameters T =
      PointMatcher::TransformationParameters::cast(trajectory.at(time_ns).getTransformationMatrix());
  const uint64_t id = laser_track.residentScanAtTime(time_ns);
  throwOnError(ctx_, ls_occupancy_insert_scan(map_, laser_track.ring(), id, T.data(), stats), "ls_occupancy_insert_scan");
}

size_t OccupancyMap::insertLaserTracks() {
  std::vector<std::shared_ptr<LaserTrack> > tracks = estimator_.getAllLaserTracks();
  std::vector<std::tuple<Time, size_t, size_t> > order;  // (time, track, scan)
  for (size_t k = 0; k < tracks.size(); ++k) {
    const std::vector<LaserScan>& scans = tracks[k]->getLaserScans();
    for (size_t j = 0; j < scans.size(); ++j) order.emplace_back(scans[j].time_ns, k, j);
  }
  std::sort(order.begin(), order.end());
  bool zero_added = false;
  size_t inserted = 0;
  for (const auto& e : order) {
    const Time t = std::get<0>(e);
    if (t == 0u) {
      if (zero_added) continue;
      zero_added = true;
    }
    insertScan(*tracks[std::get<1>(e)], t);
    ++inserted;
  }
  return inserted;
}

void OccupancyMap::download(int which, std::vector<uint64_t>* keys, std::vector<float>* log_odds,
                            std::vector<float>* centres4) const {
  std::lock_guard<std::mutex> lock(mutex_);
  int64_t n = 0;
  throwOnError(ctx_, ls_occupancy_size(map_, which, &n), "ls_occupancy_size");
  const size_t m = (size_t)(n > 0 ? n : 1);
  if (keys) keys->resize(m);
  if (log_odds) log_odds->resize(m);
  if (centres4) centres4->resize(4 * m);
  int64_t got = 0;
  throwOnError(ctx_,
               ls_occupancy_download(map_, which, keys ? keys->data() : NULL, log_odds ? log_odds->data() : NULL,
                                     centres4 ? centres4->data() : NULL, n, &got),
               "ls_occupancy_download");
  if (keys) keys->resize((size_t)got);
  if (log_odds) log_odds->resize((size_t)got);
  if (centres4) centres4->resize(4 * (size_t)got);
}

void OccupancyMap::getOccupiedCloud(DataPoints* cloud) const {
  if (cloud == NULL) throw std::invalid_argument("null output");
  std::vector<float> c;
  download(LS_OCC_OCCUPIED, NULL, NULL, &c);
  *cloud = DataPoints::fromArrays(c.data(), NULL, c.size() / 4);
}

bool OccupancyMap::writeBinary(const std::string& filename) {
  std::lock_guard<std::mutex> lock(mutex_);
  const int rc = ls_occupancy_write_octomap(map_, filename.c_str(), NULL);
  if (rc == LS_ERR_ARG) return false;
  throwOnError(ctx_, rc, "ls_occupancy_write_octomap");
  return true;
}

bool OccupancyMap::readBinary(const std::string& filename) {
  std::lock_guard<std::mutex> lock(mutex_);
  ls_octomap_read_stats stats;
  const int rc = ls_occupancy_read_octomap(map_, filename.c_str(), &stats);
  if (rc == LS_ERR_ARG || rc == LS_ERR_NOMEM) return false;
  throwOnError(ctx_, rc, "ls_occupancy_read_octomap");
  params_.resolution = stats.resolution;
  return true;
}

bool OccupancyMap::write(const std::string& filename) {
  std::lock_guard<std::mutex> lock(mutex_);
  const int rc = ls_occupancy_write_octomap_full(map_, filename.c_str(), NULL);
  if (rc == LS_ERR_ARG) return false;
  throwOnError(ctx_, rc, "ls_occupancy_write_octomap_full");
  return true;
}

bool OccupancyMap::read(const std::string& filename) {
  std::lock_guard<std::mutex> lock(mutex_);
  ls_octomap_read_stats stats;
  const int rc = ls_occupancy_read_octomap_full(map_, filename.c_str(), &stats);
  if (rc == LS_ERR_ARG || rc == LS_ERR_NOMEM) return false;
  throwOnError(ctx_, rc, "ls_occupancy_read_octomap_full");
  params_.resolution = stats.resolution;
  return true;
}

void OccupancyMap::writeData(std::vector<uint8_t>* payload, int64_t* nodes) {
  if (payload == NULL || nodes == NULL) throw std::invalid_argument("null output");
  std::lock_guard<std::mutex> lock(mutex_);
  ls_full_octree_stats st;
  throwOnError(ctx_, ls_occupancy_build_full_octree(map_, &st), "ls_occupancy_build_full_octree");
  payload->resize((size_t)st.payload_bytes);
  throwOnError(ctx_, ls_occupancy_download_full_octree(map_, payload->data(), st.payload_bytes),
               "ls_occupancy_download_full_octree");
  *nodes = st.nodes;
}

bool OccupancyMap::readData(const std::vector<uint8_t>& payload, int64_t nodes, double resolution) {
  std::lock_guard<std::mutex> lock(mutex_);
  ls_octomap_read_stats stats;
  const int rc = ls_occupancy_read_full_octree(map_, payload.empty() ? NULL : payload.data(), (int64_t)payload.size(), nodes,
                                               resolution, &stats);
  if (rc == LS_ERR_ARG || rc == LS_ERR_NOMEM) return false;
  throwOnError(ctx_, rc, "ls_occupancy_read_full_octree");
  params_.resolution = stats.resolution;
  return true;
}

void OccupancyMap::getOccupiedLeafCloud(DataPoints* cloud) {
  if (cloud == NULL) throw std::invalid_argument("null output");
  std::lock_guard<std::mutex> lock(mutex_);
  ls_octree_stats st;
  throwOnError(ctx_, ls_occupancy_build_octree(map_, &st), "ls_occupancy_build_octree");
  std::vector<uint8_t> payload((size_t)(st.payload_bytes > 0 ? st.payload_bytes : 1));
  std::vector<float> c(4 * (size_t)(st.occupied_leaves > 0 ? st.occupied_leaves : 1));
  throwOnError(ctx_,
               ls_occupancy_download_octree(map_, payload.data(), st.payload_bytes, c.data(), NULL, st.occupied_leaves),
               "ls_occupancy_download_octree");
  *cloud = DataPoints::fromArrays(c.data(), NULL, (size_t)st.occupied_leaves);
}

void OccupancyMap::getVoxels(int which, std::vector<uint64_t>* keys, std::vector<float>* log_odds) const {
  download(which, keys, log_odds, NULL);
}

// ---- leaf boxes and marker cubes ------------------------------------------------------------------------------------
void OccupancyMap::boxes(int which, const kindr::minimal::Position* region_min, const kindr::minimal::Position* region_max,
                         BoxVector* out) const {
  if (out == NULL) throw std::invalid_argument("null output");
  std::lock_guard<std::mutex> lock(mutex_);
  ls_leaf_stats st;
  throwOnError(ctx_, ls_occupancy_build_leaves(map_, region_min ? region_min->data() : NULL,
                                               region_max ? region_max->data() : NULL, &st),
               "ls_occupancy_build_leaves");
  const int64_t n = which == LS_LEAVES_FREE ? st.free_leaves : st.occupied_leaves;
  const size_t m = (size_t)(n > 0 ? n : 1);
  std::vector<float> c(4 * m);
  std::vector<uint8_t> depth(m);
  std::vector<int8_t> state(m);
  int64_t got = 0;
  throwOnError(ctx_, ls_occupancy_download_leaves(map_, which, c.data(), depth.data(), state.data(), n, &got),
               "ls_occupancy_download_leaves");
  out->clear();
  out->reserve((size_t)got);
  for (int64_t i = 0; i < got; ++i)
    out->emplace_back(kindr::minimal::Position{c[4 * i], c[4 * i + 1], c[4 * i + 2]},
                      params_.resolution * std::ldexp(1.0, 16 - depth[(size_t)i]));
}

void OccupancyMap::getAllFreeBoxes(BoxVector* free_boxes) const { boxes(LS_LEAVES_FREE, NULL, NULL, free_boxes); }

void OccupancyMap::getAllOccupiedBoxes(BoxVector* occupied_boxes) const {
  boxes(LS_LEAVES_OCCUPIED, NULL, NULL, occupied_boxes);
}

void OccupancyMap::getAllFreeBoxes(const kindr::minimal::Position& region_min, const kindr::minimal::Position& region_max,
                                   BoxVector* free_boxes) const {
  boxes(LS_LEAVES_FREE, &region_min, &region_max, free_boxes);
}

void OccupancyMap::getAllOccupiedBoxes(const kindr::minimal::Position& region_min,
                                       const kindr::minimal::Position& region_max, BoxVector* occupied_boxes) const {
  boxes(LS_LEAVES_OCCUPIED, &region_min, &region_max, occupied_boxes);
}

void OccupancyMap::generateMarkerArray(double min_z, double max_z, double color_factor,
                                       std::vector<CubeList>* occupied_nodes, std::vector<CubeList>* free_nodes) const {
  if (occupied_nodes == NULL || free_nodes == NULL) throw std::invalid_argument("null output");
  std::lock_guard<std::mutex> lock(mutex_);
  ls_leaf_stats st;
  throwOnError(ctx_, ls_occupancy_build_leaves(map_, NULL, NULL, &st), "ls_occupancy_build_leaves");
  const int64_t n = st.free_leaves + st.occupied_leaves;
  const size_t m = (size_t)(n > 0 ? n : 1);
  std::vector<float> c(4 * m), rgba(4 * m);
  int64_t occ[18], fre[18], got = 0;
  throwOnError(ctx_, ls_occupancy_marker_cubes(map_, min_z, max_z, color_factor, c.data(), rgba.data(), occ, fre, n, &got),
               "ls_occupancy_marker_cubes");
  occupied_nodes->assign(17, CubeList());
  free_nodes->assign(17, CubeList());
  for (int d = 0; d < 17; ++d) {
    CubeList& o = (*occupied_nodes)[(size_t)d];
    CubeList& f = (*free_nodes)[(size_t)d];
    o.size = f.size = params_.resolution * std::ldexp(1.0, 16 - d);
    for (int64_t i = occ[d]; i < occ[d + 1]; ++i) {
      o.points.push_back(kindr::minimal::Position{c[4 * i], c[4 * i + 1], c[4 * i + 2]});
      o.colors.push_back(std::array<float, 4>{rgba[4 * i], rgba[4 * i + 1], rgba[4 * i + 2], rgba[4 * i + 3]});
    }
    for (int64_t i = fre[d]; i < fre[d + 1]; ++i) f.points.push_back(kindr::minimal::Position{c[4 * i], c[4 * i + 1], c[4 * i + 2]});
  }
}

// ---- 2D projection -------------------------------------------------------------------------------------------------
void OccupancyMap::getProjectedMap(const ProjectedMapParams& params, ProjectedMap* map) const {
  if (map == NULL) throw std::invalid_argument("null output");
  std::lock_guard<std::mutex> lock(mutex_);
  ls_grid_info info;
  throwOnError(ctx_,
               ls_occupancy_build_projection(map_, params.occupancy_min_z, params.occupancy_max_z, params.min_x_size,
                                             params.min_y_size, &info),
               "ls_occupancy_build_projection");
  map->width = (uint32_t)info.width;
  map->height = (uint32_t)info.height;
  map->resolution = info.resolution;
  map->origin_x = info.origin_x;
  map->origin_y = info.origin_y;
  map->data.resize((size_t)(info.width * info.height));
  throwOnError(ctx_, ls_occupancy_download_projection(map_, map->data.data(), (int64_t)map->data.size()),
               "ls_occupancy_download_projection");
}

bool OccupancyMap::saveProjectedMap(const std::string& stem, const ProjectedMapParams& params) const {
  ProjectedMap m;
  getProjectedMap(params, &m);
  // map_saver: the message's float32 resolution; rows from the top (j = height - 1) down
  const float res = (float)m.resolution;
  const std::string image = stem + ".pgm";
  FILE* out = std::fopen(image.c_str(), "wb");
  if (!out) return false;
  std::fprintf(out, "P5\n# CREATOR: map_saver.cpp %.3f m/pix\n%d %d\n255\n", res, (int)m.width, (int)m.height);
  for (uint32_t y = 0; y < m.height; ++y)
    for (uint32_t x = 0; x < m.width; ++x) {
      const int8_t v = m.data[(size_t)x + (size_t)(m.height - y - 1) * m.width];
      std::fputc(v == 0 ? 254 : v == 100 ? 0 : 205, out);
    }
  bool ok = std::fclose(out) == 0;
  FILE* yaml = std::fopen((stem + ".yaml").c_str(), "w");
  if (!yaml) return false;
  std::fprintf(yaml, "image: %s\nresolution: %f\norigin: [%f, %f, %f]\nnegate: 0\noccupied_thresh: 0.65\nfree_thresh: 0.196\n\n",
               image.c_str(), res, m.origin_x, m.origin_y, 0.0);
  ok = std::fclose(yaml) == 0 && ok;
  return ok;
}

// ---- queries ------------------------------------------------------------------------------------------------------
OccupancyMap::CellStatus OccupancyMap::cellStatus(const kindr::minimal::Position& point, float* log_odds) const {
  std::lock_guard<std::mutex> lock(mutex_);
  int8_t st = LS_CELL_UNKNOWN;
  throwOnError(ctx_, ls_occupancy_cell_status(map_, point.data(), 1, &st, log_odds, NULL), "ls_occupancy_cell_status");
  return static_cast<CellStatus>(st);
}

OccupancyMap::CellStatus OccupancyMap::getCellStatusPoint(const kindr::minimal::Position& point) const {
  return cellStatus(point, NULL);
}

OccupancyMap::CellStatus OccupancyMap::getCellProbabilityPoint(const kindr::minimal::Position& point,
                                                               double* probability) const {
  float v = 0.f;
  const CellStatus st = cellStatus(point, &v);
  if (probability) *probability = st == CellStatus::kUnknown ? -1.0 : 1.0 - 1.0 / (1.0 + std::exp((double)v));
  return st;
}

OccupancyMap::CellStatus OccupancyMap::getLineStatus(const kindr::minimal::Position& start,
                                                     const kindr::minimal::Position& end) const {
  return getVisibility(start, end, true);
}

OccupancyMap::CellStatus OccupancyMap::getVisibility(const kindr::minimal::Position& view_point,
                                                     const kindr::minimal::Position& voxel_to_test,
                                                     bool stop_at_unknown_cell) const {
  std::vector<CellStatus> st;
  getLineStatus(std::vector<kindr::minimal::Position>{view_point}, std::vector<kindr::minimal::Position>{voxel_to_test}, &st,
                stop_at_unknown_cell);
  return st[0];
}

OccupancyMap::CellStatus OccupancyMap::getLineStatusBoundingBox(const kindr::minimal::Position& start,
                                                                const kindr::minimal::Position& end,
                                                                const kindr::minimal::Position& bounding_box_size) const {
  std::vector<CellStatus> st;
  getLineStatus(std::vector<kindr::minimal::Position>{start}, std::vector<kindr::minimal::Position>{end}, &st, true,
                &bounding_box_size);
  return st[0];
}

bool OccupancyMap::castRay(const kindr::minimal::Position& origin, const kindr::minimal::Position& direction,
                           kindr::minimal::Position* end, bool ignore_unknown, double max_range) const {
  std::vector<int> r;
  std::vector<kindr::minimal::Position> e;
  castRays(std::vector<kindr::minimal::Position>{origin}, std::vector<kindr::minimal::Position>{direction}, &r, &e,
           ignore_unknown, max_range);
  if (end && r[0] != LS_RAY_INVALID) *end = e[0];
  return r[0] == LS_RAY_HIT;
}

void OccupancyMap::getLineStatus(const std::vector<kindr::minimal::Position>& starts,
                                 const std::vector<kindr::minimal::Position>& ends, std::vector<CellStatus>* status,
                                 bool stop_at_unknown_cell, const kindr::minimal::Position* bounding_box_size,
                                 std::vector<uint64_t>* first_keys) const {
  if (status == NULL) throw std::invalid_argument("null output");
  if (starts.size() != ends.size()) throw std::invalid_argument("starts and ends differ in length");
  const size_t n = starts.size();
  std::vector<double> s(3 * n), e(3 * n);
  for (size_t i = 0; i < n; ++i)
    for (int a = 0; a < 3; ++a) s[3 * i + a] = starts[i][a], e[3 * i + a] = ends[i][a];
  std::vector<int8_t> st(n > 0 ? n : 1);
  if (first_keys) first_keys->resize(n);
  std::lock_guard<std::mutex> lock(mutex_);
  throwOnError(ctx_,
               ls_occupancy_line_status(map_, s.data(), e.data(), (int)n, bounding_box_size ? bounding_box_size->data() : NULL,
                                        stop_at_unknown_cell ? 1 : 0, st.data(), first_keys ? first_keys->data() : NULL, NULL),
               "ls_occupancy_line_status");
  status->resize(n);
  for (size_t i = 0; i < n; ++i) (*status)[i] = static_cast<CellStatus>(st[i]);
}

void OccupancyMap::castRays(const std::vector<kindr::minimal::Position>& origins,
                            const std::vector<kindr::minimal::Position>& directions, std::vector<int>* results,
                            std::vector<kindr::minimal::Position>* ends, bool ignore_unknown, double max_range) const {
  if (results == NULL) throw std::invalid_argument("null output");
  if (origins.size() != directions.size()) throw std::invalid_argument("origins and directions differ in length");
  const size_t n = origins.size();
  std::vector<float> o(3 * n), d(3 * n), e(3 * (n > 0 ? n : 1));
  for (size_t i = 0; i < n; ++i)
    for (int a = 0; a < 3; ++a) o[3 * i + a] = (float)origins[i][a], d[3 * i + a] = (float)directions[i][a];
  std::vector<int8_t> r(n > 0 ? n : 1);
  {
    std::lock_guard<std::mutex> lock(mutex_);
    throwOnError(ctx_,
                 ls_occupancy_cast_rays(map_, o.data(), d.data(), (int)n, ignore_unknown ? 1 : 0, max_range, r.data(), e.data(),
                                        NULL),
                 "ls_occupancy_cast_rays");
  }
  results->assign(r.begin(), r.begin() + (std::ptrdiff_t)n);
  if (ends) {
    ends->resize(n);
    for (size_t i = 0; i < n; ++i) (*ends)[i] = kindr::minimal::Position{e[3 * i], e[3 * i + 1], e[3 * i + 2]};
  }
}

// ---- box status and robot collision --------------------------------------------------------------------------------
OccupancyMap::CellStatus OccupancyMap::getCellStatusBoundingBox(const kindr::minimal::Position& point,
                                                                const kindr::minimal::Position& bounding_box_size) const {
  std::vector<CellStatus> st;
  getCellStatusBoundingBox(std::vector<kindr::minimal::Position>{point}, std::vector<kindr::minimal::Position>{bounding_box_size},
                           &st);
  return st[0];
}

void OccupancyMap::getCellStatusBoundingBox(const std::vector<kindr::minimal::Position>& points,
                                            const std::vector<kindr::minimal::Position>& bounding_box_sizes,
                                            std::vector<CellStatus>* statuses) const {
  if (statuses == NULL) throw std::invalid_argument("null output");
  if (points.size() != bounding_box_sizes.size()) throw std::invalid_argument("points and sizes differ in length");
  const size_t n = points.size();
  std::vector<double> c(3 * n), s(3 * n);
  for (size_t i = 0; i < n; ++i)
    for (int a = 0; a < 3; ++a) c[3 * i + a] = points[i][a], s[3 * i + a] = bounding_box_sizes[i][a];
  std::vector<int8_t> st(n > 0 ? n : 1);
  {
    std::lock_guard<std::mutex> lock(mutex_);
    throwOnError(ctx_, ls_occupancy_box_status(map_, c.data(), s.data(), (int)n, st.data(), NULL), "ls_occupancy_box_status");
  }
  statuses->resize(n);
  for (size_t i = 0; i < n; ++i) (*statuses)[i] = static_cast<CellStatus>(st[i]);
}

void OccupancyMap::setRobotSize(const kindr::minimal::Position& robot_size) {
  std::lock_guard<std::mutex> lock(mutex_);
  robot_size_ = robot_size;
}

kindr::minimal::Position OccupancyMap::getRobotSize() const {
  std::lock_guard<std::mutex> lock(mutex_);
  return robot_size_;
}

bool OccupancyMap::checkCollisionWithRobot(const kindr::minimal::Position& robot_position) const {
  return checkPathForCollisionsWithRobot(std::vector<kindr::minimal::Position>{robot_position}, NULL);
}

bool OccupancyMap::checkPathForCollisionsWithRobot(const std::vector<kindr::minimal::Position>& robot_positions,
                                                   size_t* collision_index) const {
  std::vector<int64_t> first;
  checkPathsForCollisionsWithRobot(std::vector<std::vector<kindr::minimal::Position> >{robot_positions}, &first);
  if (first[0] < 0) return false;
  if (collision_index) *collision_index = (size_t)first[0];
  return true;
}

void OccupancyMap::checkPathsForCollisionsWithRobot(const std::vector<std::vector<kindr::minimal::Position> >& paths,
                                                    std::vector<int64_t>* first_collisions) const {
  if (first_collisions == NULL) throw std::invalid_argument("null output");
  std::vector<int64_t> offsets(1, 0);
  std::vector<double> pos;
  for (const auto& path : paths) {
    for (const auto& p : path)
      for (int a = 0; a < 3; ++a) pos.push_back(p[a]);
    offsets.push_back(offsets.back() + (int64_t)path.size());
  }
  first_collisions->assign(paths.size(), -1);
  std::lock_guard<std::mutex> lock(mutex_);
  throwOnError(ctx_,
               ls_occupancy_check_paths(map_, pos.empty() ? NULL : pos.data(), offsets.data(), (int)paths.size(),
                                        robot_size_.data(), params_.treat_unknown_as_occupied ? 1 : 0,
                                        first_collisions->empty() ? NULL : first_collisions->data(), NULL),
               "ls_occupancy_check_paths");
}

// ---- edits ---------------------------------------------------------------------------------------------------------
void OccupancyMap::setFree(const kindr::minimal::Position& position, const kindr::minimal::Position& bounding_box_size) {
  setBoxes({position}, {bounding_box_size}, {false});
}

void OccupancyMap::setOccupied(const kindr::minimal::Position& position, const kindr::minimal::Position& bounding_box_size) {
  setBoxes({position}, {bounding_box_size}, {true});
}

void OccupancyMap::setBoxes(const std::vector<kindr::minimal::Position>& positions,
                            const std::vector<kindr::minimal::Position>& bounding_box_sizes, const std::vector<bool>& occupied,
                            ls_occupancy_edit_stats* stats) {
  const size_t n = positions.size();
  if (bounding_box_sizes.size() != n || occupied.size() != n)
    throw std::invalid_argument("positions, sizes and occupied flags differ in length");
  std::vector<double> c(3 * n), s(3 * n);
  std::vector<int8_t> o(n > 0 ? n : 1);
  for (size_t i = 0; i < n; ++i) {
    for (int a = 0; a < 3; ++a) c[3 * i + a] = positions[i][a], s[3 * i + a] = bounding_box_sizes[i][a];
    o[i] = occupied[i] ? 1 : 0;
  }
  std::lock_guard<std::mutex> lock(mutex_);
  throwOnError(ctx_, ls_occupancy_set_boxes(map_, c.data(), s.data(), o.data(), (int)n, stats), "ls_occupancy_set_boxes");
}

void OccupancyMap::resetMap() {
  std::lock_guard<std::mutex> lock(mutex_);
  throwOnError(ctx_, ls_occupancy_clear(map_), "ls_occupancy_clear");
}

void OccupancyMap::getOccupiedPointcloudInBoundingBox(const kindr::minimal::Position& center,
                                                      const kindr::minimal::Position& bounding_box_size,
                                                      DataPoints* output_cloud) const {
  if (output_cloud == NULL) throw std::invalid_argument("null output");
  std::lock_guard<std::mutex> lock(mutex_);
  int64_t n = 0;
  int rc = ls_occupancy_box_voxels(map_, center.data(), bounding_box_size.data(), LS_OCC_OCCUPIED, NULL, NULL, NULL, 0, &n);
  if (!(rc == LS_ERR_ARG && n > 0)) throwOnError(ctx_, rc, "ls_occupancy_box_voxels");
  std::vector<float> c(4 * (size_t)(n > 0 ? n : 1));
  if (n > 0)
    throwOnError(ctx_, ls_occupancy_box_voxels(map_, center.data(), bounding_box_size.data(), LS_OCC_OCCUPIED, NULL, NULL,
                                               c.data(), n, &n),
                 "ls_occupancy_box_voxels");
  *output_cloud = DataPoints::fromArrays(c.data(), NULL, (size_t)n);
}

void OccupancyMap::getMapBounds(kindr::minimal::Position* min_bound, kindr::minimal::Position* max_bound) const {
  if (min_bound == NULL || max_bound == NULL) throw std::invalid_argument("null output");
  std::lock_guard<std::mutex> lock(mutex_);
  throwOnError(ctx_, ls_occupancy_bounds(map_, min_bound->data(), max_bound->data()), "ls_occupancy_bounds");
}

kindr::minimal::Position OccupancyMap::getMapSize() const {
  kindr::minimal::Position lo, hi;
  getMapBounds(&lo, &hi);
  return kindr::minimal::Position{hi[0] - lo[0], hi[1] - lo[1], hi[2] - lo[2]};
}

kindr::minimal::Position OccupancyMap::getMapCenter() const {
  kindr::minimal::Position lo, hi;
  getMapBounds(&lo, &hi);
  kindr::minimal::Position c;
  for (int a = 0; a < 3; ++a) c[a] = lo[a] + (hi[a] - lo[a]) / 2.0;
  return c;
}

// ---- change detection ----------------------------------------------------------------------------------------------
void OccupancyMap::enableChangeDetection(bool enable) {
  std::lock_guard<std::mutex> lock(mutex_);
  throwOnError(ctx_, ls_occupancy_track_changes(map_, enable ? 1 : 0), "ls_occupancy_track_changes");
  change_detection_ = enable;
}

bool OccupancyMap::isChangeDetectionEnabled() const {
  std::lock_guard<std::mutex> lock(mutex_);
  return change_detection_;
}

void OccupancyMap::resetChangeDetection() {
  std::lock_guard<std::mutex> lock(mutex_);
  if (change_detection_) throwOnError(ctx_, ls_occupancy_track_changes(map_, 1), "ls_occupancy_track_changes");
}

size_t OccupancyMap::changes(std::vector<uint64_t>* keys, std::vector<int8_t>* status, std::vector<int8_t>* previous,
                             std::vector<float>* centres4, bool reset) const {
  std::lock_guard<std::mutex> lock(mutex_);
  if (!change_detection_) {
    if (keys) keys->clear();
    if (status) status->clear();
    if (previous) previous->clear();
    if (centres4) centres4->clear();
    return 0;
  }
  // the count (with cap 0 a reset happens only when nothing changed), then the copy and the reset
  int64_t n = 0;
  const int rc = ls_occupancy_changes(map_, NULL, NULL, NULL, NULL, 0, &n, reset ? 1 : 0, NULL);
  if (!(rc == LS_ERR_ARG && n > 0)) throwOnError(ctx_, rc, "ls_occupancy_changes");
  if (n == 0 || !(keys || status || previous || centres4)) return (size_t)n;
  const size_t m = (size_t)n;
  if (keys) keys->resize(m);
  if (status) status->resize(m);
  if (previous) previous->resize(m);
  if (centres4) centres4->resize(4 * m);
  throwOnError(ctx_,
               ls_occupancy_changes(map_, keys ? keys->data() : NULL, status ? status->data() : NULL,
                                    previous ? previous->data() : NULL, centres4 ? centres4->data() : NULL, n, &n,
                                    reset ? 1 : 0, NULL),
               "ls_occupancy_changes");
  return m;
}

size_t OccupancyMap::numChangesDetected() const { return changes(NULL, NULL, NULL, NULL, false); }

void OccupancyMap::getChangedKeys(std::vector<uint64_t>* keys, std::vector<int8_t>* status,
                                  std::vector<int8_t>* previous) const {
  if (keys == NULL || status == NULL || previous == NULL) throw std::invalid_argument("null output");
  changes(keys, status, previous, NULL, false);
}

void OccupancyMap::getChangedPoints(std::vector<kindr::minimal::Position>* changed_points,
                                    std::vector<bool>* changed_states) {
  if (changed_points == NULL || changed_states == NULL) throw std::invalid_argument("null output");
  std::vector<int8_t> status;
  std::vector<float> c;
  const size_t n = changes(NULL, &status, NULL, &c, true);
  changed_points->resize(n);
  changed_states->resize(n);
  for (size_t i = 0; i < n; ++i) {
    (*changed_points)[i] = kindr::minimal::Position{c[4 * i], c[4 * i + 1], c[4 * i + 2]};
    (*changed_states)[i] = status[i] == LS_CELL_OCCUPIED;
  }
}

}  // namespace laser_slam
