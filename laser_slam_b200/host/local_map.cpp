// laser_slam::LocalMap over ls_local_map_* (include/laser_slam/local_map.hpp).
#include "laser_slam/local_map.hpp"

#include <stdexcept>
#include <string>

namespace laser_slam {

namespace {
void throwOnError(ls_ctx* ctx, int rc, const char* what) {
  if (rc < 0) throw std::runtime_error(std::string(what) + ": " + ls_b200_last_error(ctx));
}
PointMatcher::TransformationParameters toFloatMatrix(const SE3& T) {
  return PointMatcher::TransformationParameters::cast(T.getTransformationMatrix());
}
}  // namespace

LocalMap::LocalMap(const LocalMapParams& params, const LaserTrack& laser_track) : params_(params), laser_track_(laser_track) {
  ls_local_map_params p{};
  p.distance_to_consider_fixed = params.distance_to_consider_fixed;
  p.separate_distant_map = params.separate_distant_map ? 1 : 0;
  p.voxel_size_m = params.voxel_size_m;
  p.minimum_point_number_per_voxel = params.minimum_point_number_per_voxel;
  p.remove_ground_from_local_map = params.remove_ground_from_local_map ? 1 : 0;
  p.ground_distance_to_robot_center_m = params.ground_distance_to_robot_center_m;
  throwOnError(laser_track.context(), ls_local_map_create(laser_track.context(), &p, &map_), "ls_local_map_create");
}

LocalMap::~LocalMap() { ls_local_map_destroy(map_); }

void LocalMap::addScan() {
  if (!params_.create_filtered_map) return;  // reference :236
  std::lock_guard<std::recursive_mutex> lock(mutex_);
  // getLocalCloudInWorldFrame(getMaxTime()) (reference :195-197): the scan's pose, corrected, as laser_track.cpp does
  const Time t = laser_track_.getMaxTime();
  PointMatcher::TransformationParameters T = toFloatMatrix(laser_track_.evaluate(t));
  correctTransformationMatrix(&T);
  const uint64_t id = laser_track_.residentScanAtTime(t);
  const double robot_z = laser_track_.getCurrentPose().T_w.getPosition()[2];  // reference :222
  int n = 0;
  throwOnError(laser_track_.context(), ls_local_map_add_scan(map_, laser_track_.ring(), id, T.data(), robot_z, &n),
               "ls_local_map_add_scan");
}

void LocalMap::getFilteredMap(DataPoints* filtered_map) {
  if (filtered_map == NULL) throw std::invalid_argument("null output");
  std::lock_guard<std::recursive_mutex> lock(mutex_);
  const SE3::Position p = laser_track_.getCurrentPose().T_w.getPosition();
  const double center[3] = {(double)(float)p[0], (double)(float)p[1], (double)(float)p[2]};  // a PclPoint (:418-421)
  int n = 0;
  throwOnError(laser_track_.context(), ls_local_map_filter(map_, center, &n), "ls_local_map_filter");
  download(LS_LM_FILTERED_MAP, filtered_map);
}

void LocalMap::getLocalMapFiltered(DataPoints* out) const { download(LS_LM_LOCAL_FILTERED, out); }
void LocalMap::getLocalMap(DataPoints* out) const { download(LS_LM_LOCAL, out); }
void LocalMap::getDistantMap(DataPoints* out) const { download(LS_LM_DISTANT, out); }

void LocalMap::download(int which, DataPoints* out) const {
  if (out == NULL) throw std::invalid_argument("null output");
  std::lock_guard<std::recursive_mutex> lock(mutex_);
  const int n = ls_local_map_size(map_, which);
  throwOnError(laser_track_.context(), n, "ls_local_map_size");
  std::vector<float> feat(4 * (size_t)(n > 0 ? n : 1));
  int got = 0;
  throwOnError(laser_track_.context(), ls_local_map_download(map_, which, feat.data(), n, &got), "ls_local_map_download");
  *out = DataPoints::fromArrays(feat.data(), NULL, (size_t)got);
}

std::vector<DataPoints> LocalMap::getQueuedPoints() {
  std::lock_guard<std::recursive_mutex> lock(mutex_);
  const int n = ls_local_map_size(map_, LS_LM_QUEUE);
  throwOnError(laser_track_.context(), n, "ls_local_map_size");
  std::vector<float> feat(4 * (size_t)(n > 0 ? n : 1));
  std::vector<int> offsets((size_t)n + 2);  // every queued cloud holds at least one point
  int k = 0;
  throwOnError(laser_track_.context(), ls_local_map_take_queue(map_, feat.data(), n, offsets.data(), n + 1, &k),
               "ls_local_map_take_queue");
  std::vector<DataPoints> clouds;
  for (int j = 0; j < k; ++j)
    clouds.push_back(DataPoints::fromArrays(feat.data() + 4 * (size_t)offsets[j], NULL, (size_t)(offsets[j + 1] - offsets[j])));
  return clouds;
}

void LocalMap::updateLocalMap(const SE3& last_pose_before_update, const Time last_pose_before_update_timestamp_ns) {
  std::lock_guard<std::recursive_mutex> lock(mutex_);
  Trajectory new_trajectory;
  laser_track_.getTrajectory(&new_trajectory);
  const SE3 new_last_pose = new_trajectory.at(last_pose_before_update_timestamp_ns);
  // cast to float, not corrected (reference :529-530)
  PointMatcher::TransformationParameters T = toFloatMatrix(new_last_pose * last_pose_before_update.inverse());
  throwOnError(laser_track_.context(), ls_local_map_transform(map_, T.data()), "ls_local_map_transform");
}

void LocalMap::clearLocalMap() {
  std::lock_guard<std::recursive_mutex> lock(mutex_);
  throwOnError(laser_track_.context(), ls_local_map_clear(map_), "ls_local_map_clear");
}

}  // namespace laser_slam
