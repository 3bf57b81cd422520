// LocalMap -- the map maintenance of LaserSlamWorker (reference laser_slam_ros/src/laser_slam_worker.cpp:195-246,
// 407-540) without ROS, over the resident local map of the C ABI (ls_local_map_*, include/ls_b200.h): the worker's
// local_map_, local_map_filtered_, distant_map_ and local_map_queue_ stay on the device next to the track's scan ring.
// Each method takes the pose, the centre or the transform from the track, as the worker does.  Clouds are features-only
// DataPoints ({x, y, z, 1} per point); PCL is not used.
#ifndef LASER_SLAM_LOCAL_MAP_HPP_
#define LASER_SLAM_LOCAL_MAP_HPP_

#include <mutex>
#include <vector>

#include "laser_slam/common.hpp"
#include "laser_slam/laser_track.hpp"

namespace laser_slam {

// The map fields of LaserSlamWorkerParams (reference laser_slam_ros/include/laser_slam_ros/common.hpp:20-31), same names.
struct LocalMapParams {
  double distance_to_consider_fixed = 20.0;
  bool separate_distant_map = false;
  bool create_filtered_map = true;
  double voxel_size_m = 0.1;
  int minimum_point_number_per_voxel = 0;
  bool remove_ground_from_local_map = false;
  double ground_distance_to_robot_center_m = 1.0;
};

class LocalMap {
 public:
  // The map lives on the track's context and reads its scans from the track's ring (its own or its estimator's); the
  // track must outlive the map.
  LocalMap(const LocalMapParams& params, const LaserTrack& laser_track);
  ~LocalMap();
  LocalMap(const LocalMap&) = delete;
  LocalMap& operator=(const LocalMap&) = delete;

  // scanCallback's map part (:195-246): the track's newest scan in the world frame, ground removed against the current
  // pose, appended and queued.  Nothing is added when create_filtered_map is false.
  void addScan();
  // getFilteredMap (:415-488) around the track's current position.
  void getFilteredMap(DataPoints* filtered_map);
  // getLocalMapFiltered (:490-494).
  void getLocalMapFiltered(DataPoints* local_map_filtered) const;
  // getQueuedPoints (:407-412): the queued clouds in order; the queue is empty afterwards.
  std::vector<DataPoints> getQueuedPoints();
  // updateLocalMap (:522-540): local_map_ and local_map_filtered_ moved by (new pose * pose before update^-1) at that
  // time; distant_map_ and the queue are not moved, as in the reference.
  void updateLocalMap(const SE3& last_pose_before_update, const Time last_pose_before_update_timestamp_ns);
  // clearLocalMap (:496-506): distant_map_ and the queue stay.
  void clearLocalMap();
  // (new) the other members, for tests and publishing
  void getLocalMap(DataPoints* local_map) const;
  void getDistantMap(DataPoints* distant_map) const;

 private:
  void download(int which, DataPoints* out) const;

  LocalMapParams params_;
  const LaserTrack& laser_track_;
  ls_local_map* map_ = nullptr;
  // one mutex where the worker holds local_map_mutex_ and local_map_filtered_mutex_: every call changes or reads both
  mutable std::recursive_mutex mutex_;
};

}  // namespace laser_slam

#endif  // LASER_SLAM_LOCAL_MAP_HPP_
