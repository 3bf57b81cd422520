// OccupancyMap -- laser_to_octomap (reference laser_slam_tools/src/laser_to_octomap.cpp) without ROS: every scan of every
// track of an estimator inserted at its pose into an occupancy map, over the resident map of the C ABI (ls_occupancy_*,
// include/ls_b200.h).  writeBinary saves the map as octomap's pruned binary tree (.bt), the file laser_to_octomap writes;
// getOccupiedLeafCloud gives what octomap_to_point_cloud exports from it (the occupied leaves' centres), getOccupiedCloud
// every occupied voxel's centre at the finest resolution.  The rules are oracle/OCCUPANCY.md and, for the tree,
// oracle/OCTREE.md.
#ifndef LASER_SLAM_OCCUPANCY_MAP_HPP_
#define LASER_SLAM_OCCUPANCY_MAP_HPP_

#include <array>
#include <cstdint>
#include <limits>
#include <mutex>
#include <string>
#include <utility>
#include <vector>

#include "laser_slam/common.hpp"
#include "laser_slam/incremental_estimator.hpp"
#include "laser_slam/laser_track.hpp"

namespace laser_slam {

class DistanceMap;

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
  // volumetric_mapping's: robot collision checks count unknown space as a collision (recalled, unverified).  The status
  // calls report unknown either way.
  bool treat_unknown_as_occupied = true;
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
  // octomap's OcTree::readBinary: the .bt file replaces the map, its resolution becomes the map's, free leaves load as
  // clamping_thres_min and occupied ones as clamping_thres_max (ls_occupancy_read_octomap).  Returns false, with the map
  // unchanged, when the file cannot be read, is malformed or covers more than the map can hold.
  bool readBinary(const std::string& filename);
  // octomap's OcTree::write: every node's float log-odds, pruned by value, as a .ot file (ls_occupancy_write_octomap_full),
  // so a saved map resumes mapping exactly.  Returns false when the file cannot be written.
  bool write(const std::string& filename);
  // octomap's AbstractOcTree::read of a .ot file: it replaces the map, its resolution becomes the map's and every leaf's
  // voxels take its value verbatim (ls_occupancy_read_octomap_full).  Returns false, with the map unchanged, when the file
  // cannot be read, is malformed or covers more than the map can hold.
  bool read(const std::string& filename);
  // The full tree's payload (what getOctomapFullMsg carries as data) and its node count.
  void writeData(std::vector<uint8_t>* payload, int64_t* nodes);
  // setOctomapFromFullMsg: a full-tree payload of `nodes` nodes at `resolution` replaces the map, as read().  Returns false,
  // with the map unchanged, when it is refused.
  bool readData(const std::vector<uint8_t>& payload, int64_t nodes, double resolution);
  // The occupied leaves of the pruned tree in octomap's leaf order, features only ({x, y, z, 1}): what
  // octomap_to_point_cloud writes from writeBinary's file.
  void getOccupiedLeafCloud(DataPoints* cloud);
  // (new) LS_OCC_KNOWN or LS_OCC_OCCUPIED voxels: packed keys and log-odds, by ascending key.
  void getVoxels(int which, std::vector<uint64_t>* keys, std::vector<float>* log_odds) const;

  // ---- queries: volumetric_mapping's WorldBase and octomap's castRay on the device map (ls_occupancy_cell_status /
  // _line_status / _cast_rays; rules in oracle/QUERIES.md).  Each single query is a device call of one; the batched
  // overloads are the intended use.
  enum class CellStatus { kFree = LS_CELL_FREE, kOccupied = LS_CELL_OCCUPIED, kUnknown = LS_CELL_UNKNOWN };

  CellStatus getCellStatusPoint(const kindr::minimal::Position& point) const;
  // octomap's probability 1 - 1 / (1 + exp(v)) of the voxel's log-odds, -1 when unknown.
  CellStatus getCellProbabilityPoint(const kindr::minimal::Position& point, double* probability) const;
  CellStatus getLineStatus(const kindr::minimal::Position& start, const kindr::minimal::Position& end) const;
  CellStatus getVisibility(const kindr::minimal::Position& view_point, const kindr::minimal::Position& voxel_to_test,
                           bool stop_at_unknown_cell) const;
  CellStatus getLineStatusBoundingBox(const kindr::minimal::Position& start, const kindr::minimal::Position& end,
                                      const kindr::minimal::Position& bounding_box_size) const;
  // octomap's castRay: true on a hit; *end (may be NULL) the centre of the voxel the ray stopped in (left alone for an
  // invalid ray).  max_range <= 0: none.
  bool castRay(const kindr::minimal::Position& origin, const kindr::minimal::Position& direction,
               kindr::minimal::Position* end, bool ignore_unknown = false, double max_range = -1.0) const;
  // Batches: one status per segment (bounding_box_size NULL: getLineStatus / getVisibility); first_keys may be NULL.
  void getLineStatus(const std::vector<kindr::minimal::Position>& starts, const std::vector<kindr::minimal::Position>& ends,
                     std::vector<CellStatus>* status, bool stop_at_unknown_cell = true,
                     const kindr::minimal::Position* bounding_box_size = NULL, std::vector<uint64_t>* first_keys = NULL) const;
  // One LS_RAY_* result and end per ray.
  void castRays(const std::vector<kindr::minimal::Position>& origins, const std::vector<kindr::minimal::Position>& directions,
                std::vector<int>* results, std::vector<kindr::minimal::Position>* ends, bool ignore_unknown = false,
                double max_range = -1.0) const;

  // ---- box status and robot collision: volumetric_mapping's getCellStatusBoundingBox and robot calls on the device map
  // (ls_occupancy_box_status / _check_paths; rules in DESIGN.md §4b''''''''''').  The robot is an axis-aligned box of
  // getRobotSize() (zero until set) at each position; a pose collides when its box is occupied, or, with
  // treat_unknown_as_occupied, when it is not free.
  CellStatus getCellStatusBoundingBox(const kindr::minimal::Position& point,
                                      const kindr::minimal::Position& bounding_box_size) const;
  // (new) One status per box.
  void getCellStatusBoundingBox(const std::vector<kindr::minimal::Position>& points,
                                const std::vector<kindr::minimal::Position>& bounding_box_sizes,
                                std::vector<CellStatus>* statuses) const;
  void setRobotSize(const kindr::minimal::Position& robot_size);
  kindr::minimal::Position getRobotSize() const;
  bool checkCollisionWithRobot(const kindr::minimal::Position& robot_position) const;
  // True when a pose collides; *collision_index (may be NULL) the first one.
  bool checkPathForCollisionsWithRobot(const std::vector<kindr::minimal::Position>& robot_positions,
                                       size_t* collision_index) const;
  // (new) Per path the first colliding pose's index, -1 when none (an empty path included).
  void checkPathsForCollisionsWithRobot(const std::vector<std::vector<kindr::minimal::Position> >& paths,
                                        std::vector<int64_t>* first_collisions) const;

  // ---- edits: volumetric_mapping's WorldBase map calls on the device map (ls_occupancy_set_boxes / _clear / _box_voxels /
  // _bounds; rules in DESIGN.md §4b'''''''').  Errors throw, as every call here.
  // setFree / setOccupied: every voxel the box's loop reaches becomes known with clamping_thres_min / _max.
  void setFree(const kindr::minimal::Position& position, const kindr::minimal::Position& bounding_box_size);
  void setOccupied(const kindr::minimal::Position& position, const kindr::minimal::Position& bounding_box_size);
  // (new) Both in one call, in order: the last box covering a voxel decides it.  stats may be NULL.
  void setBoxes(const std::vector<kindr::minimal::Position>& positions,
                const std::vector<kindr::minimal::Position>& bounding_box_sizes, const std::vector<bool>& occupied,
                ls_occupancy_edit_stats* stats = NULL);
  // resetMap: no known voxel; the parameters and the device memory stay.
  void resetMap();
  // The occupied voxels the box's loop reaches, in loop order, as their centres ({x, y, z, 1}).
  void getOccupiedPointcloudInBoundingBox(const kindr::minimal::Position& center,
                                          const kindr::minimal::Position& bounding_box_size, DataPoints* output_cloud) const;
  // getMetricMin / getMetricMax over the known voxels (zeros when none), their difference and midpoint.
  void getMapBounds(kindr::minimal::Position* min_bound, kindr::minimal::Position* max_bound) const;
  kindr::minimal::Position getMapSize() const;
  kindr::minimal::Position getMapCenter() const;

  // ---- leaf boxes and marker cubes: volumetric_mapping's getAllFreeBoxes / getAllOccupiedBoxes and generateMarkerArray on
  // the device map (ls_occupancy_build_leaves / _download_leaves / _marker_cubes; rules in DESIGN.md §4b'''''''''''').  A box
  // is a leaf of the value-pruned tree (octomap's tree in memory, not the .bt file's), as (centre, edge), in octomap's leaf
  // order.
  typedef std::vector<std::pair<kindr::minimal::Position, double> > BoxVector;
  void getAllFreeBoxes(BoxVector* free_boxes) const;
  void getAllOccupiedBoxes(BoxVector* occupied_boxes) const;
  // (new) Only the leaves whose key cube meets the box [region_min, region_max] (metres, each corner keyed and clamped to
  // the key range); a region that is not finite or is inverted throws.
  void getAllFreeBoxes(const kindr::minimal::Position& region_min, const kindr::minimal::Position& region_max,
                       BoxVector* free_boxes) const;
  void getAllOccupiedBoxes(const kindr::minimal::Position& region_min, const kindr::minimal::Position& region_max,
                           BoxVector* occupied_boxes) const;
  // One of generateMarkerArray's cube lists: the cube edge of its depth, the cubes' centres and, for occupied cubes, one
  // colour {r, g, b, a} per cube (free lists carry none: the marker's own colour is set by the caller).
  struct CubeList {
    double size;
    std::vector<kindr::minimal::Position> points;
    std::vector<std::array<float, 4> > colors;
  };
  // One list per depth 0..16 for the occupied leaves, coloured by height (octomap_server's heightMapColor over min_z ...
  // max_z, times color_factor), and for the free ones.  min_z < max_z, all finite, or it throws.
  void generateMarkerArray(double min_z, double max_z, double color_factor, std::vector<CubeList>* occupied_nodes,
                           std::vector<CubeList>* free_nodes) const;

  // ---- 2D projection: octomap_server's projected_map and map_saver on the device map (ls_occupancy_build_projection /
  // _download_projection; rules in DESIGN.md §4b''''''''''''').  octomap_server's occupancy_min_z / occupancy_max_z (NaN
  // throws, infinities allowed) and min_x_size / min_y_size (finite, >= 0, or it throws).
  struct ProjectedMapParams {
    double occupancy_min_z = -std::numeric_limits<double>::infinity();
    double occupancy_max_z = std::numeric_limits<double>::infinity();
    double min_x_size = 0.0, min_y_size = 0.0;
  };
  // A nav_msgs/OccupancyGrid's content: cell (i, j) is data[j * width + i], -1 unknown, 0 free, 100 occupied; origin is the
  // lower corner of cell (0, 0) (z and yaw 0).
  struct ProjectedMap {
    uint32_t width = 0, height = 0;
    double resolution = 0.0, origin_x = 0.0, origin_y = 0.0;
    std::vector<int8_t> data;
  };
  void getProjectedMap(const ProjectedMapParams& params, ProjectedMap* map) const;
  // The projection written as map_saver writes it: stem + ".pgm" and stem + ".yaml".  False when a file cannot be written.
  bool saveProjectedMap(const std::string& stem, const ProjectedMapParams& params) const;

  // ---- change detection: octomap's calls and volumetric_mapping's getChangedPoints on the device map
  // (ls_occupancy_track_changes / _changes; rules in DESIGN.md §4b'''''''''').  A change is a voxel whose state (free,
  // occupied, unknown) differs from its state at the last enable or reset.
  // true takes the map as it is now as the baseline (again when enabled); false turns tracking off.
  void enableChangeDetection(bool enable);
  bool isChangeDetectionEnabled() const;
  // The map as it is now becomes the baseline; nothing while tracking is off.
  void resetChangeDetection();
  // 0 while tracking is off.
  size_t numChangesDetected() const;
  // (new) The changed voxels by ascending key: packed keys, LS_CELL_* now and at the baseline; empty while tracking is off.
  void getChangedKeys(std::vector<uint64_t>* keys, std::vector<int8_t>* status, std::vector<int8_t>* previous) const;
  // The changed voxels' centres and whether each is occupied now, by ascending key, then resetChangeDetection; empty
  // while tracking is off.
  void getChangedPoints(std::vector<kindr::minimal::Position>* changed_points, std::vector<bool>* changed_states);

 private:
  friend class DistanceMap;  // reads map_ under mutex_ in its update (include/laser_slam/distance_map.hpp)

  CellStatus cellStatus(const kindr::minimal::Position& point, float* log_odds) const;
  // Under mutex_: the leaves of LS_LEAVES_FREE or LS_LEAVES_OCCUPIED, of the region when region_min is not NULL.
  void boxes(int which, const kindr::minimal::Position* region_min, const kindr::minimal::Position* region_max,
             BoxVector* out) const;
  void download(int which, std::vector<uint64_t>* keys, std::vector<float>* log_odds, std::vector<float>* centres4) const;
  // Under mutex_: the changes (each output may be NULL), then a reset when `reset`.  Returns their number.
  size_t changes(std::vector<uint64_t>* keys, std::vector<int8_t>* status, std::vector<int8_t>* previous,
                 std::vector<float>* centres4, bool reset) const;

  OccupancyMapParams params_;
  IncrementalEstimator& estimator_;
  ls_ctx* ctx_ = nullptr;
  ls_occupancy* map_ = nullptr;
  bool change_detection_ = false;
  kindr::minimal::Position robot_size_{0.0, 0.0, 0.0};
  mutable std::mutex mutex_;
};

}  // namespace laser_slam

#endif  // LASER_SLAM_OCCUPANCY_MAP_HPP_
