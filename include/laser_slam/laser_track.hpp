// LaserTrack -- public interface of reference laser_slam/include/laser_slam/laser_track.hpp:17-236, implemented
// over the C ABI of include/ls_b200.h: scans live in a device ring (ls_map_*), the scan-to-sub-map ICP is
// ls_icp_register_submap, factors are ls_factor records.
#ifndef LASER_SLAM_LASER_TRACK_HPP_
#define LASER_SLAM_LASER_TRACK_HPP_

#include <map>
#include <mutex>
#include <string>
#include <vector>

#include "laser_slam/common.hpp"
#include "laser_slam/parameters.hpp"

namespace laser_slam {

class LaserTrack {
 public:
  explicit LaserTrack(const LaserTrackParams& parameters, unsigned int laser_track_id = 0u);
  // (new) a track hosted by an IncrementalEstimator: context and scan ring belong to the estimator and are shared by
  // all of its tracks, so that their registrations can be served by ONE batched launch (ls_icp_register_submap_batch).
  LaserTrack(const LaserTrackParams& parameters, unsigned int laser_track_id, ls_ctx* shared_ctx, ls_map** shared_ring,
             int* shared_ring_capacity, int* shared_ring_max_pts, int ring_slots_per_track);
  ~LaserTrack();
  LaserTrack(const LaserTrack&) = delete;
  LaserTrack& operator=(const LaserTrack&) = delete;

  void processPose(const Pose& pose);
  void processLaserScan(const LaserScan& scan);
  void processPoseAndLaserScan(const Pose& pose, const LaserScan& in_scan,
                               gtsam::NonlinearFactorGraph* newFactors = NULL, gtsam::Values* newValues = NULL,
                               bool* is_prior = NULL);

  void getLastPointCloud(DataPoints* out_point_cloud) const;
  void getPointCloudOfTimeInterval(const std::pair<Time, Time>& times_ns, DataPoints* out_point_cloud) const;
  void getLocalCloudInWorldFrame(const Time& timestamp, DataPoints* out_point_cloud) const;
  const std::vector<LaserScan>& getLaserScans() const;
  void getTrajectory(Trajectory* trajectory) const;
  void getOdometryTrajectory(Trajectory* out_trajectory) const;
  void getCovariances(std::vector<Covariance>* out_covariances) const;
  Pose getCurrentPose() const;
  Pose getPreviousPose() const;
  Time getMinTime() const;
  Time getMaxTime() const;
  void getLaserScansTimes(std::vector<Time>* out_times_ns) const;

  void appendPriorFactors(const curves::Time& prior_time_ns, gtsam::NonlinearFactorGraph* graph) const;
  void appendOdometryFactors(const curves::Time& optimization_min_time_ns, const curves::Time& optimization_max_time_ns,
                             gtsam::noiseModel::Base::shared_ptr noise_model, gtsam::NonlinearFactorGraph* graph) const;
  void appendICPFactors(const curves::Time& optimization_min_time_ns, const curves::Time& optimization_max_time_ns,
                        gtsam::noiseModel::Base::shared_ptr noise_model, gtsam::NonlinearFactorGraph* graph) const;
  void appendLoopClosureFactors(const curves::Time& optimization_min_time_ns, const curves::Time& optimization_max_time_ns,
                                gtsam::noiseModel::Base::shared_ptr noise_model, gtsam::NonlinearFactorGraph* graph) const;

  void initializeGTSAMValues(const gtsam::KeySet& keys, gtsam::Values* values) const;
  void updateFromGTSAMValues(const gtsam::Values& values);
  // gtsam::Marginals(factor_graph, values).marginalCovariance(key) for every node of the trajectory
  // (reference laser_track.cpp:421-429): one device pass (ls_pg_marginals) instead of one elimination per key
  void updateCovariancesFromGTSAMValues(const gtsam::NonlinearFactorGraph& factor_graph, const gtsam::Values& values);
  void printTrajectory() const;

  size_t getNumScans() const;
  Pose findNearestPose(const Time& timestamp_ns) const;
  void buildSubMapAroundTime(const curves::Time& time_ns, const unsigned int sub_maps_radius, DataPoints* submap_out) const;
  // The same sub-map left on the device: its scans are pushed into a new ring of `ctx` (caller destroys it with
  // ls_map_destroy) and described by (ids, 16 floats per part), ready for ls_icp_register_submaps.
  void stageSubMapAroundTime(const curves::Time& time_ns, const unsigned int sub_maps_radius, ls_ctx* ctx, ls_map** ring_out,
                             std::vector<uint64_t>* ids_out, std::vector<float>* T_parts_out) const;
  gtsam::Expression<SE3> getValueExpression(const curves::Time& time_ns) const;  // leaf expression of the node at time_ns
  Key getValueKey(const curves::Time& time_ns) const;                            // its key
  SE3 evaluate(const curves::Time& time_ns) const;
  void getScanMatchingTimes(std::map<Time, double>* scan_matching_times) const;
  void saveTrajectory(const std::string& filename) const;

  // (new) processPoseAndLaserScan in two halves around the registration, so that a host of several tracks can run the
  // registrations of one step as a batch: begin...() does everything up to and including the staging of the
  // scan-to-sub-map problem (reference laser_track.cpp:122-206, 466-491) and describes it in `pending` (active == false:
  // first scan of the track, or ICP factors disabled); the caller registers it -- alone through ls_icp_register_submap
  // or together with other tracks' problems -- and hands the outcome to end...(), which stores the RelativePose and
  // emits factors and values (reference :493-519, 208-230).
  struct PendingIcp {
    bool active = false;
    uint64_t reading_id = 0;
    std::vector<uint64_t> part_ids;
    std::vector<float> T_parts;  // 16 floats per part
    PointMatcher::TransformationParameters T0;
    RelativePose icp_transformation;
    // (internal) carried from begin to end
    RelativePose relative_measurement;
    Key scan_key = 0;
    Time scan_time_ns = 0;
    bool first = false;
    Pose pose;
    double t_start_ms = 0.0;
  };
  void beginPoseAndLaserScan(const Pose& pose, const LaserScan& in_scan, PendingIcp* pending);
  // (new) A hint: upload a scan that WILL be passed to processPoseAndLaserScan / beginPoseAndLaserScan (recognised by its
  // time stamp) now, e.g. while the previous scan is still being registered.  Without it the upload happens inside the
  // scan's own call.  Never changes a result.
  void prefetchLaserScan(const LaserScan& scan);
  void endPoseAndLaserScan(PendingIcp* pending, int rc, const float* T_out16, const ls_icp_stats* stats,
                           gtsam::NonlinearFactorGraph* newFactors, gtsam::Values* newValues, bool* is_prior);
  const ls_icp_params& icpParams() const { return icp_params_; }

  // (new) ICP results and run statistics, for tests and the bench
  const RelativePoseVector& getIcpTransformations() const { return icp_transformations_; }
  const ls_icp_stats& getLastIcpStats() const { return last_icp_stats_; }
  ls_ctx* context() const { return ctx_; }
  // (new) the device copy of the scan at time_ns (scanIndexAtTime): its id in ring(), uploaded again if it was evicted.
  // What a resident local map (include/laser_slam/local_map.hpp) reads instead of the host cloud.
  uint64_t residentScanAtTime(const curves::Time& time_ns) const;
  const ls_map* ring() const { return *map_p_; }
  unsigned int id() const { return laser_track_id_; }

 private:
  struct Node { SE3 value; Key key; };
  gtsam::ExpressionFactor<SE3> makeRelativeMeasurementFactor(const RelativePose& relative_pose_measurement,
                                                             gtsam::noiseModel::Base::shared_ptr noise_model,
                                                             const bool fix_first_node = false) const;
  gtsam::ExpressionFactor<SE3> makeMeasurementFactor(const Pose& pose_measurement, gtsam::noiseModel::Base::shared_ptr noise_model) const;
  void stageLocalScanToSubMap(PendingIcp* pending);
  void finishLocalScanToSubMap(const PendingIcp& pending, int rc, const float* T_out16);
  void ensureRing(size_t max_pts) const;  // the ring is a device cache of laser_scans_ (reached through map_p_)
  const Pose& findPose(const Time& timestamp_ns) const;
  Pose& findPose(const Time& timestamp_ns);
  Key extendTrajectory(const Time& timestamp_ns, const SE3& value);
  size_t scanIndexAtTime(const curves::Time& time_ns) const;
  uint64_t residentScan(size_t index) const;  // device id of laser_scans_[index], uploading it if it was evicted
  uint64_t uploadScan(const DataPoints& cloud) const;
  // the input filters on the device (ls_map_push_scan_filtered) into the ring; *filtered = the slot's cloud, downloaded
  int pushFiltered(const DataPoints& raw, uint64_t* id, DataPoints* filtered);
  void describeSubMapAroundTime(const curves::Time& time_ns, const unsigned int sub_maps_radius, std::vector<size_t>* scan_indices,
                                std::vector<PointMatcher::TransformationParameters>* Ts) const;
  void assembleSubMap(const std::vector<size_t>& scan_indices, const std::vector<PointMatcher::TransformationParameters>& Ts,
                      DataPoints* out) const;

  unsigned int laser_track_id_;
  PoseVector pose_measurements_;
  RelativePoseVector odometry_measurements_, icp_transformations_, loop_closures_;
  std::vector<LaserScan> laser_scans_;
  std::map<Time, Node> trajectory_;  // curves::DiscreteSE3Curve: time -> (value, key)
  mutable std::recursive_mutex full_laser_track_mutex_;
  std::vector<Covariance> covariances_;
  gtsam::noiseModel::Base::shared_ptr prior_noise_model_, odometry_noise_model_, icp_noise_model_;
  std::map<Time, double> scan_matching_times_;
  LaserTrackParams params_;
  ls_icp_params icp_params_;
  std::vector<ls_point_filter> input_filters_;  // icp_input_filters_file (reference :24-30); empty: scans are stored as given
  ls_icp_stats last_icp_stats_;
  // device side
  ls_ctx* ctx_ = nullptr;
  bool owns_ctx_ = true;
  // the ring: the track's own, or the host's (then these point into the IncrementalEstimator)
  ls_map* own_map_ = nullptr;
  int own_capacity_ = 0, own_max_pts_ = 0;
  ls_map** map_p_ = &own_map_;
  int* map_capacity_p_ = &own_capacity_;
  int* map_max_pts_p_ = &own_max_pts_;
  int ring_slots_per_track_ = 0;  // shared ring: slots every track may count on
  mutable std::map<size_t, uint64_t> resident_;  // scan index -> device scan id
  std::map<Time, std::pair<uint64_t, LaserScan> > prefetched_;  // time stamp -> (device scan id, the scan: keeps its storage alive)
  static constexpr double kDistanceBetweenPriorPoses_m = 100.0;
};

}  // namespace laser_slam

#endif  // LASER_SLAM_LASER_TRACK_HPP_
