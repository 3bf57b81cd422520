// DistanceMap -- octomap's DynamicEDTOctomap (dynamicEDT3D) over the device occupancy map (ls_distance_map_*,
// include/ls_b200.h): the Euclidean distance of every finest cell of a box to its nearest obstacle, capped at maxdist, and
// that obstacle.  update() recomputes the whole field on the device from the map's current state; the queries read the
// last update only.  The rules are DESIGN.md §4b'''''''''.  Unlike DynamicEDT3D the transform is exact and is not
// incremental: every update recomputes it in full.
#ifndef LASER_SLAM_DISTANCE_MAP_HPP_
#define LASER_SLAM_DISTANCE_MAP_HPP_

#include <cstdint>
#include <vector>

#include "laser_slam/occupancy_map.hpp"

namespace laser_slam {

class DistanceMap {
 public:
  static constexpr float distanceValue_Error = -1.0f;
  static constexpr int distanceInCellsValue_Error = -1;

  // The map must outlive the distance map.  Throws std::runtime_error on refused parameters (maxdist not finite or <= 0, a
  // corner not finite, bbx_min > bbx_max on an axis).
  DistanceMap(float maxdist, OccupancyMap& map, const kindr::minimal::Position& bbx_min,
              const kindr::minimal::Position& bbx_max, bool treat_unknown_as_occupied);
  ~DistanceMap();
  DistanceMap(const DistanceMap&) = delete;
  DistanceMap& operator=(const DistanceMap&) = delete;

  // The field of the map as it is now, read under the map's mutex.  stats may be NULL.  Throws on an error (the box then
  // has more than 2^30 cells, a corner has no key at the map's resolution, or maxdist is more than 46340 cells).
  void update(ls_distance_map_stats* stats = NULL);

  // distanceValue_Error outside the box; the capped distance where no obstacle is within maxdist.
  float getDistance(const kindr::minimal::Position& p) const;
  // closest: the obstacle's voxel centre (NaN where none is within maxdist); dist: as getDistance.
  void getDistanceAndClosestObstacle(const kindr::minimal::Position& p, float& dist, kindr::minimal::Position& closest) const;
  // distanceInCellsValue_Error outside the box.
  int getSquaredDistanceInCells(const kindr::minimal::Position& p) const;
  // (float)(m * res) and m * m of the last update, m = (int)(maxdist / res + 1).
  float getMaxDist() const { return max_dist_; }
  int getSquaredMaxDistCells() const { return max_sqdist_cells_; }

  // Batches: one device call for all points; any output may be NULL.
  void getDistances(const std::vector<kindr::minimal::Position>& points, std::vector<float>* distances,
                    std::vector<int>* squared_distances_in_cells = NULL,
                    std::vector<kindr::minimal::Position>* closest = NULL) const;

 private:
  OccupancyMap& map_;
  ls_ctx* ctx_ = nullptr;
  ls_distance_map* dm_ = nullptr;
  float max_dist_ = 0.f;
  int max_sqdist_cells_ = 0;
};

}  // namespace laser_slam

#endif  // LASER_SLAM_DISTANCE_MAP_HPP_
