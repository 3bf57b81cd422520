// OccupancyMap -- laser_to_octomap (reference laser_slam_tools/src/laser_to_octomap.cpp) without ROS: every scan of every
// track of an estimator inserted at its pose into an occupancy map, over the resident map of the C ABI (ls_occupancy_*,
// include/ls_b200.h).  writeBinary saves the map as octomap's pruned binary tree (.bt), the file laser_to_octomap writes;
// getOccupiedLeafCloud gives what octomap_to_point_cloud exports from it (the occupied leaves' centres), getOccupiedCloud
// every occupied voxel's centre at the finest resolution.  The rules are oracle/OCCUPANCY.md and, for the tree,
// oracle/OCTREE.md.
#ifndef LASER_SLAM_OCCUPANCY_MAP_HPP_
#define LASER_SLAM_OCCUPANCY_MAP_HPP_

#include <cstdint>
#include <mutex>
#include <string>
#include <vector>

#include "laser_slam/common.hpp"
#include "laser_slam/incremental_estimator.hpp"
#include "laser_slam/laser_track.hpp"

namespace laser_slam {

// laser_to_octomap's defaults (:18-21) and volumetric_mapping's clamping and threshold.
struct OccupancyMapParams {
  double resolution = 0.075;
  double probability_hit = 0.9;
  double probability_miss = 0.4;
  double clamping_thres_min = 0.12;
  double clamping_thres_max = 0.97;
  double occupancy_thres = 0.7;
  double sensor_max_range = 20.0;  // < 0: unlimited
  int initial_capacity_bricks = 0;  // 8x8x8-voxel bricks to start with; <= 0: the library's default
};

class OccupancyMap {
 public:
  // The map lives on the estimator's track context and reads the scans from its tracks' ring; the estimator must outlive
  // the map.
  OccupancyMap(const OccupancyMapParams& params, IncrementalEstimator& estimator);
  ~OccupancyMap();
  OccupancyMap(const OccupancyMap&) = delete;
  OccupancyMap& operator=(const OccupancyMap&) = delete;

  // One scan of `laser_track` at its trajectory pose (cast to float, not corrected, as getLaserTracksServiceCall sends it,
  // reference laser_slam_worker.cpp:279-283).  The scan is uploaded again if the ring evicted it.
  void insertScan(const LaserTrack& laser_track, const Time& time_ns, ls_occupancy_stats* stats = NULL);
  // laser_to_octomap's loop: every scan of every track by time (ties by track, then by scan), every time-0 scan after the
  // first dropped (reference laser_slam_worker.cpp:297-311).  Returns the scans inserted.
  size_t insertLaserTracks();
  // The occupied voxels' centres, features only ({x, y, z, 1}), by ascending voxel key.
  void getOccupiedCloud(DataPoints* cloud) const;
  // octomap's OcTree::writeBinary: the map's max-likelihood states, pruned, as a .bt file (ls_occupancy_write_octomap).
  // Returns false when the file cannot be written.
  bool writeBinary(const std::string& filename);
  // The occupied leaves of the pruned tree in octomap's leaf order, features only ({x, y, z, 1}): what
  // octomap_to_point_cloud writes from writeBinary's file.
  void getOccupiedLeafCloud(DataPoints* cloud);
  // (new) LS_OCC_KNOWN or LS_OCC_OCCUPIED voxels: packed keys and log-odds, by ascending key.
  void getVoxels(int which, std::vector<uint64_t>* keys, std::vector<float>* log_odds) const;

 private:
  void download(int which, std::vector<uint64_t>* keys, std::vector<float>* log_odds, std::vector<float>* centres4) const;

  OccupancyMapParams params_;
  IncrementalEstimator& estimator_;
  ls_ctx* ctx_ = nullptr;
  ls_occupancy* map_ = nullptr;
  mutable std::mutex mutex_;
};

}  // namespace laser_slam

#endif  // LASER_SLAM_OCCUPANCY_MAP_HPP_
