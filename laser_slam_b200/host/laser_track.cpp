// LaserTrack over the ls_b200 C ABI.  Control flow follows reference laser_slam/src/laser_track.cpp (cited per
// function); the heavy steps call include/ls_b200.h instead of libpointmatcher:
//   laser_scans_ copies + RigidTransformation::compute + concatenate  ->  ls_map_push_scan / device assembly
//   icp_.compute                                                       ->  ls_icp_register_submap
//   input_filters_.apply(scan) (:81, :146)                             ->  ls_map_push_scan_filtered
// The input filters of icp_input_filters_file run on the device straight into the scan's ring slot; the track keeps the
// filtered cloud (downloaded once), as the reference stores the filtered scan.  Without filters -- or without a normal
// filter among them -- scans must arrive with a "normals" descriptor.
#include "laser_slam/laser_track.hpp"

#include <atomic>
#include <chrono>
#include <cstdio>
#include <fstream>
#include <sstream>
#include <stdexcept>

namespace laser_slam {

namespace {

#define LS_CHECK(cond, msg)                                             \
  do {                                                                  \
    if (!(cond)) throw std::logic_error(std::string("CHECK failed: ") + (msg)); \
  } while (0)

std::atomic<uint64_t> g_key_counter{1};

std::string readFile(const std::string& path) {
  std::ifstream ifs(path.c_str());
  if (!ifs.good()) return std::string();
  std::stringstream ss;
  ss << ifs.rdbuf();
  return ss.str();
}

PointMatcher::TransformationParameters toFloatMatrix(const SE3& T) {
  return PointMatcher::TransformationParameters::cast(T.getTransformationMatrix());
}

void throwOnError(ls_ctx* ctx, int rc, const char* what) {
  if (rc < 0) throw std::runtime_error(std::string(what) + ": " + ls_b200_last_error(ctx));
}

}  // namespace

// reference laser_track.cpp:10-65
LaserTrack::LaserTrack(const LaserTrackParams& parameters, unsigned int laser_track_id)
    : LaserTrack(parameters, laser_track_id, nullptr, nullptr, nullptr, nullptr, 0) {}

LaserTrack::LaserTrack(const LaserTrackParams& parameters, unsigned int laser_track_id, ls_ctx* shared_ctx, ls_map** shared_ring,
                       int* shared_ring_capacity, int* shared_ring_max_pts, int ring_slots_per_track)
    : laser_track_id_(laser_track_id), params_(parameters) {
  // ICP chain: the YAML the reference hands to icp_.loadFromYaml, or libpointmatcher's setDefault() values
  // (SURVEY.md Appendix A.7) when the file cannot be opened (reference :14-21).
  ls_icp_default_params(&icp_params_);
  const std::string yaml = readFile(params_.icp_configuration_file);
  if (!yaml.empty()) {
    if (ls_icp_params_from_yaml(yaml.c_str(), &icp_params_) != LS_OK)
      throw std::runtime_error("unsupported ICP chain in " + params_.icp_configuration_file);
  } else {
    icp_params_.trim_ratio = 0.85f;
    icp_params_.min_diff_rot = 0.001f;
    icp_params_.min_diff_trans = 0.001f;
    icp_params_.smooth_length = 3;
  }
  // reference :24-30 is fatal when the input-filter file cannot be opened; an empty name means "no filters".
  if (!params_.icp_input_filters_file.empty()) {
    if (!std::ifstream(params_.icp_input_filters_file.c_str()).good())
      throw std::runtime_error("Could not open ICP input filters configuration file.");
    const std::string text = readFile(params_.icp_input_filters_file);
    int n = 0;
    if (ls_point_filters_from_yaml(text.c_str(), nullptr, 0, &n) != LS_OK ||
        (input_filters_.resize((size_t)n), ls_point_filters_from_yaml(text.c_str(), input_filters_.data(), n, &n)) != LS_OK)
      throw std::runtime_error("unsupported input filter #" + std::to_string(n) + " in " + params_.icp_input_filters_file);
  }
  // noise models (reference :36-64)
  using namespace gtsam::noiseModel;
  odometry_noise_model_ = Diagonal::Sigmas(params_.odometry_noise_model);
  if (params_.add_m_estimator_on_odom) odometry_noise_model_ = Robust::Create(mEstimator::Cauchy::Create(1), odometry_noise_model_);
  icp_noise_model_ = Diagonal::Sigmas(params_.icp_noise_model);
  if (params_.add_m_estimator_on_icp) icp_noise_model_ = Robust::Create(mEstimator::Cauchy::Create(1), icp_noise_model_);
  prior_noise_model_ = Diagonal::Sigmas(std::array<double, 6>{{1e-7, 1e-7, 1e-7, 1e-7, 1e-7, 1e-7}});
  std::memset(&last_icp_stats_, 0, sizeof(last_icp_stats_));
  if (shared_ctx) {
    ctx_ = shared_ctx;
    owns_ctx_ = false;
    map_p_ = shared_ring;
    map_capacity_p_ = shared_ring_capacity;
    map_max_pts_p_ = shared_ring_max_pts;
    ring_slots_per_track_ = ring_slots_per_track;
  } else {
    const int rc = ls_b200_init(params_.cuda_device, &ctx_);
    if (rc != LS_OK) throw std::runtime_error("ls_b200_init failed: no usable CUDA device (no CPU fallback)");
  }
}

LaserTrack::~LaserTrack() {
  if (own_map_) ls_map_destroy(own_map_);
  if (ctx_ && owns_ctx_) ls_b200_destroy(ctx_);
}

// reference :67-73
void LaserTrack::processPose(const Pose& pose) {
  std::lock_guard<std::recursive_mutex> lock(full_laser_track_mutex_);
  pose_measurements_.push_back(pose);
}

// reference :75-120 (older twin of processPoseAndLaserScan without factor output)
void LaserTrack::processLaserScan(const LaserScan& in_scan) {
  std::lock_guard<std::recursive_mutex> lock(full_laser_track_mutex_);
  const Pose pose = findPose(in_scan.time_ns);  // registered earlier through processPose
  for (auto it = pose_measurements_.begin(); it != pose_measurements_.end(); ++it)
    if (it->time_ns == in_scan.time_ns) { pose_measurements_.erase(it); break; }  // re-appended just below
  processPoseAndLaserScan(pose, in_scan, NULL, NULL, NULL);
}

// reference :122-231
void LaserTrack::processPoseAndLaserScan(const Pose& pose, const LaserScan& in_scan, gtsam::NonlinearFactorGraph* newFactors,
                                         gtsam::Values* newValues, bool* is_prior) {
  std::lock_guard<std::recursive_mutex> lock(full_laser_track_mutex_);
  if (newFactors != NULL) LS_CHECK(newFactors->empty(), "newFactors must be empty on entry");
  PendingIcp pending;
  beginPoseAndLaserScan(pose, in_scan, &pending);
  int rc = LS_OK;
  PointMatcher::TransformationParameters icp_solution = pending.T0;
  ls_icp_stats stats;
  std::memset(&stats, 0, sizeof(stats));
  if (pending.active)  // icp_.compute(reading, sub_map, T0) (reference :496)
    rc = ls_icp_register_submap(ctx_, &icp_params_, *map_p_, pending.reading_id, (int)pending.part_ids.size(),
                                pending.part_ids.data(), pending.T_parts.data(), pending.T0.data(), icp_solution.data(), &stats,
                                NULL, NULL, NULL);
  endPoseAndLaserScan(&pending, rc, icp_solution.data(), &stats, newFactors, newValues, is_prior);
}

// reference :122-206 and, through computeICPTransformations (:460-464), localScanToSubMap up to the ICP call (:466-491)
void LaserTrack::beginPoseAndLaserScan(const Pose& pose, const LaserScan& in_scan, PendingIcp* pending) {
  std::lock_guard<std::recursive_mutex> lock(full_laser_track_mutex_);
  LS_CHECK(pending != NULL, "null pending");
  *pending = PendingIcp();
  pending->t_start_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count();
  const bool filtered = !input_filters_.empty();
  auto pf = prefetched_.find(in_scan.time_ns);
  // the input filters (reference :146) before anything is stored; the normals check comes after them
  LaserScan stored;
  uint64_t filtered_id = 0;
  if (filtered && pf == prefetched_.end()) {
    stored.time_ns = in_scan.time_ns;
    stored.key = in_scan.key;
    throwOnError(ctx_, pushFiltered(in_scan.scan, &filtered_id, &stored.scan), "ls_map_push_scan_filtered");
  }
  LS_CHECK(filtered || in_scan.scan.descriptorExists("normals"), "scans must carry a 'normals' descriptor");
  pending->pose = pose;
  laser_scans_.push_back(filtered_id ? stored : in_scan);  // the one copy the track keeps (the reference copies twice, :143 and :197)
  LaserScan& scan = laser_scans_.back();
  pose_measurements_.push_back(pose);
  if (filtered_id) resident_[laser_scans_.size() - 1u] = filtered_id;
  if (pf != prefetched_.end()) {  // already on the device (prefetchLaserScan); share the storage that upload reads from
    const bool resident = *map_p_ && ls_map_scan_size(*map_p_, pf->second.first) >= 0;
    if (resident || filtered) scan.scan = pf->second.second.scan;  // a filtered hint holds the chain's output either way
    if (resident) resident_[laser_scans_.size() - 1u] = pf->second.first;
    prefetched_.erase(pf);
  }

  if (trajectory_.empty()) {
    pending->first = true;
    scan.key = extendTrajectory(scan.time_ns, findPose(scan.time_ns).T_w);
    findPose(scan.time_ns).key = scan.key;
    pending->scan_key = scan.key;
    pending->scan_time_ns = scan.time_ns;
    return;
  }
  const Time t_last = trajectory_.rbegin()->first;
  const SE3 last_pose_measurement = findPose(t_last).T_w;
  const SE3 new_pose_measurement = findPose(scan.time_ns).T_w;
  RelativePose& relative_measurement = pending->relative_measurement;
  relative_measurement.T_a_b = last_pose_measurement.inverse() * new_pose_measurement;
  relative_measurement.time_a_ns = t_last;
  relative_measurement.key_a = findPose(t_last).key;
  relative_measurement.time_b_ns = scan.time_ns;
  relative_measurement.track_id_a = relative_measurement.track_id_b = laser_track_id_;
  // extend the trajectory by odometry (reference :192)
  scan.key = extendTrajectory(scan.time_ns, trajectory_.rbegin()->second.value * relative_measurement.T_a_b);
  findPose(scan.time_ns).key = scan.key;
  pending->scan_key = scan.key;
  pending->scan_time_ns = scan.time_ns;
  relative_measurement.key_b = scan.key;
  odometry_measurements_.push_back(relative_measurement);
  if (params_.use_icp_factors && getNumScans() > 1u) stageLocalScanToSubMap(pending);  // computeICPTransformations (:460-464)
}

// reference :493-519 (rest of localScanToSubMap) and :208-230 (factor and value emission)
void LaserTrack::endPoseAndLaserScan(PendingIcp* pending, int rc, const float* T_out16, const ls_icp_stats* stats,
                                     gtsam::NonlinearFactorGraph* newFactors, gtsam::Values* newValues, bool* is_prior) {
  std::lock_guard<std::recursive_mutex> lock(full_laser_track_mutex_);
  LS_CHECK(pending != NULL, "null pending");
  if (newFactors != NULL) LS_CHECK(newFactors->empty(), "newFactors must be empty on entry");
  if (newValues != NULL) newValues->clear();
  struct { Key key; Time time_ns; } scan{pending->scan_key, pending->scan_time_ns};
  if (pending->first) {
    if (newFactors != NULL) {
      Pose prior_pose = pending->pose;
      prior_pose.key = scan.key;
      prior_pose.time_ns = scan.time_ns;
      if (params_.force_priors)  // reference :165-169
        prior_pose.T_w = SE3(SO3(1.0, 0.0, 0.0, 0.0), SE3::Position{0.0, kDistanceBetweenPriorPoses_m * laser_track_id_, 0.0});
      newFactors->push_back(makeMeasurementFactor(prior_pose, prior_noise_model_));
    }
    if (is_prior != NULL) *is_prior = true;
  } else {
    if (pending->active) {
      if (stats) last_icp_stats_ = *stats;
      finishLocalScanToSubMap(*pending, rc, T_out16);
    }
    const double now_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count();
    scan_matching_times_.emplace(scan.time_ns, now_ms - pending->t_start_ms);
    if (newFactors != NULL) {
      if (params_.use_odom_factors) newFactors->push_back(makeRelativeMeasurementFactor(pending->relative_measurement, odometry_noise_model_));
      if (params_.use_icp_factors && !icp_transformations_.empty())
        newFactors->push_back(makeRelativeMeasurementFactor(icp_transformations_.back(), icp_noise_model_));
    }
    if (is_prior != NULL) *is_prior = false;
  }
  if (newValues != NULL) newValues->insert(scan.key, pending->pose.T_w);  // reference :228-230
}

void LaserTrack::getLastPointCloud(DataPoints* out_point_cloud) const {  // stub in the reference too (:233-237)
  LS_CHECK(out_point_cloud != NULL, "null output");
}
void LaserTrack::getPointCloudOfTimeInterval(const std::pair<Time, Time>&, DataPoints* out_point_cloud) const {
  LS_CHECK(out_point_cloud != NULL, "null output");
  *out_point_cloud = DataPoints();  // reference :239-245
}

// reference :247-266
void LaserTrack::getLocalCloudInWorldFrame(const Time& timestamp_ns, DataPoints* out_point_cloud) const {
  std::lock_guard<std::recursive_mutex> lock(full_laser_track_mutex_);
  LS_CHECK(out_point_cloud != NULL, "null output");
  const size_t idx = scanIndexAtTime(timestamp_ns);
  PointMatcher::TransformationParameters T = toFloatMatrix(evaluate(timestamp_ns));
  correctTransformationMatrix(&T);
  assembleSubMap({idx}, {T}, out_point_cloud);
}

void LaserTrack::getTrajectory(Trajectory* trajectory) const {
  std::lock_guard<std::recursive_mutex> lock(full_laser_track_mutex_);
  LS_CHECK(trajectory != NULL, "null output");
  trajectory->clear();
  for (const auto& kv : trajectory_) trajectory->emplace(kv.first, kv.second.value);
}
const std::vector<LaserScan>& LaserTrack::getLaserScans() const { return laser_scans_; }
void LaserTrack::getCovariances(std::vector<Covariance>* out) const {
  LS_CHECK(out != NULL, "null output");
  *out = covariances_;
}
Pose LaserTrack::getCurrentPose() const {
  std::lock_guard<std::recursive_mutex> lock(full_laser_track_mutex_);
  Pose p;
  if (!trajectory_.empty()) {
    p.time_ns = trajectory_.rbegin()->first;
    p.T_w = trajectory_.rbegin()->second.value;
    p.key = trajectory_.rbegin()->second.key;
  }
  return p;
}
Pose LaserTrack::getPreviousPose() const {
  std::lock_guard<std::recursive_mutex> lock(full_laser_track_mutex_);
  Pose p;
  if (trajectory_.size() > 1u) {
    auto it = trajectory_.rbegin();
    ++it;
    p.time_ns = it->first;
    p.T_w = it->second.value;
    p.key = it->second.key;
  }
  return p;
}
void LaserTrack::getOdometryTrajectory(Trajectory* trajectory) const {
  std::lock_guard<std::recursive_mutex> lock(full_laser_track_mutex_);
  LS_CHECK(trajectory != NULL, "null output");
  trajectory->clear();
  for (const auto& pose : pose_measurements_) trajectory->emplace(pose.time_ns, pose.T_w);
}
Time LaserTrack::getMinTime() const {
  std::lock_guard<std::recursive_mutex> lock(full_laser_track_mutex_);
  LS_CHECK(!trajectory_.empty(), "empty trajectory");
  return trajectory_.begin()->first;
}
Time LaserTrack::getMaxTime() const {
  std::lock_guard<std::recursive_mutex> lock(full_laser_track_mutex_);
  LS_CHECK(!trajectory_.empty(), "empty trajectory");
  return trajectory_.rbegin()->first;
}
void LaserTrack::getLaserScansTimes(std::vector<curves::Time>* out_times_ns) const {
  std::lock_guard<std::recursive_mutex> lock(full_laser_track_mutex_);
  LS_CHECK(out_times_ns != NULL, "null output");
  out_times_ns->clear();
  for (const auto& s : laser_scans_) out_times_ns->push_back(s.time_ns);
}
size_t LaserTrack::getNumScans() const {
  std::lock_guard<std::recursive_mutex> lock(full_laser_track_mutex_);
  return laser_scans_.size();
}

// reference :339-344 (curves::DiscreteSE3Curve::addPriorFactors: prior at the node value)
void LaserTrack::appendPriorFactors(const Time& prior_time_ns, gtsam::NonlinearFactorGraph* graph) const {
  std::lock_guard<std::recursive_mutex> lock(full_laser_track_mutex_);
  LS_CHECK(graph != NULL, "null graph");
  auto it = trajectory_.find(prior_time_ns);
  LS_CHECK(it != trajectory_.end(), "no trajectory node at the prior time");
  Pose p;
  p.T_w = it->second.value;
  p.time_ns = prior_time_ns;
  p.key = it->second.key;
  graph->push_back(makeMeasurementFactor(p, prior_noise_model_));
}
// reference :346-361
void LaserTrack::appendOdometryFactors(const Time& tmin, const Time& tmax, gtsam::noiseModel::Base::shared_ptr noise,
                                       gtsam::NonlinearFactorGraph* graph) const {
  std::lock_guard<std::recursive_mutex> lock(full_laser_track_mutex_);
  LS_CHECK(graph != NULL, "null graph");
  for (const auto& m : odometry_measurements_)
    if (m.time_a_ns >= tmin && m.time_b_ns <= tmax) graph->push_back(makeRelativeMeasurementFactor(m, noise));
}
namespace {
template <typename MakeFn>
void appendWindowed(const RelativePoseVector& v, const Time& tmin, const Time& tmax, gtsam::NonlinearFactorGraph* graph, MakeFn make) {
  for (const auto& m : v) {
    if (m.time_b_ns >= tmin && m.time_b_ns <= tmax) {  // second node inside the window
      const bool a_inside = m.time_a_ns >= tmin && m.time_a_ns <= tmax;
      graph->push_back(make(m, !a_inside));  // first node outside -> frozen (fix_first_node)
    }
  }
}
}  // namespace
// reference :363-384
void LaserTrack::appendICPFactors(const Time& tmin, const Time& tmax, gtsam::noiseModel::Base::shared_ptr noise,
                                  gtsam::NonlinearFactorGraph* graph) const {
  std::lock_guard<std::recursive_mutex> lock(full_laser_track_mutex_);
  LS_CHECK(graph != NULL, "null graph");
  appendWindowed(icp_transformations_, tmin, tmax, graph,
                 [&](const RelativePose& m, bool fix) { return makeRelativeMeasurementFactor(m, noise, fix); });
}
// reference :386-409
void LaserTrack::appendLoopClosureFactors(const Time& tmin, const Time& tmax, gtsam::noiseModel::Base::shared_ptr noise,
                                          gtsam::NonlinearFactorGraph* graph) const {
  std::lock_guard<std::recursive_mutex> lock(full_laser_track_mutex_);
  LS_CHECK(graph != NULL, "null graph");
  appendWindowed(loop_closures_, tmin, tmax, graph,
                 [&](const RelativePose& m, bool fix) { return makeRelativeMeasurementFactor(m, noise, fix); });
}

// reference :411-419
void LaserTrack::initializeGTSAMValues(const gtsam::KeySet& keys, gtsam::Values* values) const {
  std::lock_guard<std::recursive_mutex> lock(full_laser_track_mutex_);
  LS_CHECK(values != NULL, "null values");
  for (const auto& kv : trajectory_)
    if (keys.count(kv.second.key) && !values->exists(kv.second.key)) values->insert(kv.second.key, kv.second.value);
}
void LaserTrack::updateFromGTSAMValues(const gtsam::Values& values) {
  std::lock_guard<std::recursive_mutex> lock(full_laser_track_mutex_);
  for (auto& kv : trajectory_)
    if (values.exists(kv.second.key)) kv.second.value = values.at(kv.second.key);
}

// reference :421-429
void LaserTrack::updateCovariancesFromGTSAMValues(const gtsam::NonlinearFactorGraph& factor_graph, const gtsam::Values& values) {
  std::lock_guard<std::recursive_mutex> lock(full_laser_track_mutex_);
  gtsam::Marginals marginals(factor_graph, values);
  std::vector<Key> keys;
  for (const auto& kv : trajectory_)
    if (values.exists(kv.second.key)) keys.push_back(kv.second.key);
  const std::vector<gtsam::Marginals::Matrix6> cov = marginals.marginalCovariances(keys);
  covariances_.clear();
  for (const auto& c : cov) covariances_.push_back(Covariance(c.begin(), c.end()));
}

void LaserTrack::printTrajectory() const {  // reference laser_track.hpp:114-117 (trajectory_.print)
  std::lock_guard<std::recursive_mutex> lock(full_laser_track_mutex_);
  std::printf("Laser track trajectory (%zu nodes)\n", trajectory_.size());
  for (const auto& kv : trajectory_) {
    const SE3::Position& t = kv.second.value.getPosition();
    const SO3& q = kv.second.value.getRotation();
    std::printf("  t = %lld ns  key %llu  p = [%.6f %.6f %.6f]  q = [%.6f %.6f %.6f %.6f]\n", (long long)kv.first,
                (unsigned long long)kv.second.key, t[0], t[1], t[2], q.w(), q.x(), q.y(), q.z());
  }
}

// reference :431-451: T_a_b expression = inverse(T_w_a) * T_w_b with T_w_a a leaf or, when the first node is frozen, a constant
gtsam::ExpressionFactor<SE3> LaserTrack::makeRelativeMeasurementFactor(const RelativePose& relative_pose_measurement,
                                                                       gtsam::noiseModel::Base::shared_ptr noise_model,
                                                                       const bool fix_first_node) const {
  using gtsam::Expression;
  Expression<SE3> T_w_b(relative_pose_measurement.key_b);
  Expression<SE3> T_w_a(relative_pose_measurement.key_a);
  if (fix_first_node) T_w_a = Expression<SE3>(evaluate(relative_pose_measurement.time_a_ns));  // constant (reference :440-444)
  Expression<SE3> T_a_w(kindr::minimal::inverse(T_w_a));
  Expression<SE3> relative(kindr::minimal::compose(T_a_w, T_w_b));
  return gtsam::ExpressionFactor<SE3>(noise_model, relative_pose_measurement.T_a_b, relative);
}
// reference :453-458
gtsam::ExpressionFactor<SE3> LaserTrack::makeMeasurementFactor(const Pose& pose_measurement,
                                                               gtsam::noiseModel::Base::shared_ptr noise_model) const {
  gtsam::Expression<SE3> T_w(getValueKey(pose_measurement.time_ns));
  return gtsam::ExpressionFactor<SE3>(noise_model, pose_measurement.T_w, T_w);
}

uint64_t LaserTrack::residentScan(size_t index) const {
  auto it = resident_.find(index);
  if (it != resident_.end() && ls_map_scan_size(*map_p_, it->second) >= 0) return it->second;
  const uint64_t id = uploadScan(laser_scans_[index].scan);
  resident_[index] = id;
  return id;
}

uint64_t LaserTrack::residentScanAtTime(const curves::Time& time_ns) const {
  std::lock_guard<std::recursive_mutex> lock(full_laser_track_mutex_);
  const size_t index = scanIndexAtTime(time_ns);
  // the ring exists from the first registration on; a reader of the first scan creates it, sized as the staging does
  const size_t n = laser_scans_.size();
  size_t max_pts = 0;
  for (size_t i = (n > 16 ? n - 16 : 0); i < n; ++i) max_pts = std::max(max_pts, laser_scans_[i].scan.getNbPoints());
  ensureRing(max_pts);
  return residentScan(index);
}

uint64_t LaserTrack::uploadScan(const DataPoints& c) const {
  const int off = c.descriptorOffset("normals");
  LS_CHECK(off >= 0, "scan without normals");
  uint64_t id = 0;
  // A scan whose storage is pinned goes up asynchronously straight from where it lies (the track keeps the scan, so the
  // memory outlives the upload; the registration orders itself behind it); any other is staged by ls_map_push_scan.
  const float* fp = c.features.data();
  const float* np = c.descriptors.data() + off;
  const bool direct = c.descriptorDim >= 3 && c.descriptorDim <= 8 && ls_host_is_pinned(fp) == 1 && ls_host_is_pinned(np) == 1;
  const int rc = direct ? ls_map_push_scan_async(*map_p_, fp, np, (int)c.descriptorDim, (int)c.getNbPoints(), &id)
                        : ls_map_push_scan(*map_p_, fp, np, (int)c.descriptorDim, (int)c.getNbPoints(), &id);
  throwOnError(ctx_, rc, "ls_map_push_scan");
  return id;
}

// A filtered scan goes through the chain on the device into a fresh slot of the ring; the ring's slots hold a whole raw
// scan, so the chain's output always fits.  Returns the C ABI's code (LS_ERR_STATE: the context is busy with a batch).
int LaserTrack::pushFiltered(const DataPoints& raw, uint64_t* id, DataPoints* filtered) {
  const size_t n = raw.getNbPoints();
  ensureRing(n);
  const int off = raw.descriptorOffset("normals");
  int kept = 0;
  int rc = ls_map_push_scan_filtered(*map_p_, input_filters_.data(), (int)input_filters_.size(), raw.features.data(),
                                     off >= 0 ? raw.descriptors.data() + off : NULL, (int)raw.descriptorDim, (int)n, id, &kept);
  if (rc != LS_OK) return rc;
  // the track's copy is the slot's cloud, bit for bit (ls_map_assemble of the one scan, identity: copied verbatim)
  std::vector<float> feat(4 * std::max<size_t>(1, (size_t)kept)), nrm(3 * std::max<size_t>(1, (size_t)kept));
  const PointMatcher::TransformationParameters I;
  int m = 0;
  if (kept > 0 && (rc = ls_map_assemble(ctx_, *map_p_, 1, id, I.data(), feat.data(), nrm.data(), &m)) != LS_OK) return rc;
  *filtered = DataPoints::fromArrays(feat.data(), nrm.data(), (size_t)m);
  return LS_OK;
}

void LaserTrack::prefetchLaserScan(const LaserScan& scan) {
  std::lock_guard<std::recursive_mutex> lock(full_laser_track_mutex_);
  const bool filtered = !input_filters_.empty();
  if (!params_.use_icp_factors || scan.scan.getNbPoints() == 0 || (!filtered && !scan.scan.descriptorExists("normals"))) return;
  if (prefetched_.count(scan.time_ns)) return;
  if (!*map_p_ || (int)scan.scan.getNbPoints() > *map_max_pts_p_) return;  // no ring yet, or it would have to grow: not now
  if (prefetched_.size() >= 2) {  // hints that were never followed up
    ls_map_sync(*map_p_);         // their uploads may still be reading the storage about to be released
    prefetched_.erase(prefetched_.begin());
  }
  if (filtered) {
    // the chain needs the context's workspace: while a batch is in flight (between beginPosesAndLaserScans and
    // endPosesAndLaserScans) the hint is dropped and the scan is filtered in its own call
    LaserScan f;
    f.time_ns = scan.time_ns;
    f.key = scan.key;
    uint64_t id = 0;
    const int rc = pushFiltered(scan.scan, &id, &f.scan);
    if (rc == LS_ERR_STATE) return;
    throwOnError(ctx_, rc, "ls_map_push_scan_filtered");
    prefetched_[scan.time_ns] = std::make_pair(id, f);
    return;
  }
  std::pair<uint64_t, LaserScan>& slot = prefetched_[scan.time_ns];
  slot.second = scan;  // shares the storage (copy-on-write)
  slot.first = uploadScan(slot.second.scan);
}

// device ring large enough for the sub-map + the reading; (re)created when a larger scan shows up.  A track of its own
// keeps nscan_in_sub_map + 3 slots; a hosted track shares its host's ring (ring_slots_per_track_ slots per track).
void LaserTrack::ensureRing(size_t max_pts) const {
  const int want_cap = owns_ctx_ ? std::max(8, params_.nscan_in_sub_map + 3) : *map_capacity_p_;
  if (!*map_p_ || (int)max_pts > *map_max_pts_p_ || want_cap > *map_capacity_p_) {
    LS_CHECK(owns_ctx_ || !*map_p_, "a scan larger than the shared ring's slots arrived (the host sizes the ring from the first scans)");
    if (*map_p_) ls_map_destroy(*map_p_);
    *map_p_ = nullptr;
    resident_.clear();
    *map_max_pts_p_ = (int)(max_pts + max_pts / 4 + 1024);
    *map_capacity_p_ = std::max(want_cap, 8);
    throwOnError(ctx_, ls_map_create(ctx_, *map_capacity_p_, *map_max_pts_p_, map_p_), "ls_map_create");
  }
}

// reference :466-491: the sub-map, the initial guess, the uploads -- everything before icp_.compute
void LaserTrack::stageLocalScanToSubMap(PendingIcp* pending) {
  const size_t n = laser_scans_.size();
  const LaserScan& last_scan = laser_scans_[n - 1u];
  RelativePose& icp_transformation = pending->icp_transformation;
  icp_transformation.time_b_ns = last_scan.time_ns;
  icp_transformation.time_a_ns = laser_scans_[n - 2u].time_ns;
  icp_transformation.track_id_a = icp_transformation.track_id_b = laser_track_id_;

  size_t max_pts = 0;
  for (size_t i = (n > 16 ? n - 16 : 0); i < n; ++i) max_pts = std::max(max_pts, laser_scans_[i].scan.getNbPoints());
  ensureRing(max_pts);

  // the last (nscan_in_sub_map - 1) scans expressed in the frame of the second-last scan (reference :474-486)
  const SE3 T_w_to_second_last_scan = evaluate(laser_scans_[n - 2u].time_ns);
  std::vector<size_t> part_index{n - 2u};
  std::vector<PointMatcher::TransformationParameters> part_T(1);  // identity: scan n-2 verbatim (:476)
  const size_t n_prev = std::min(n - 2u, size_t(params_.nscan_in_sub_map > 0 ? params_.nscan_in_sub_map - 1 : 0));
  for (size_t i = 0u; i < n_prev; ++i) {
    const size_t idx = n - 3u - i;
    PointMatcher::TransformationParameters T = toFloatMatrix(T_w_to_second_last_scan.inverse() * evaluate(laser_scans_[idx].time_ns));
    correctTransformationMatrix(&T);
    part_index.push_back(idx);
    part_T.push_back(T);
  }
  // initial guess from the trajectory (reference :488-491)
  const SE3 initial_guess = evaluate(icp_transformation.time_a_ns).inverse() * evaluate(icp_transformation.time_b_ns);
  pending->T0 = toFloatMatrix(initial_guess);

  // upload what is not resident yet (normally only the newest scan), reading last so it cannot evict a part
  pending->part_ids.clear();
  for (size_t idx : part_index) pending->part_ids.push_back(residentScan(idx));
  pending->reading_id = residentScan(n - 1u);
  for (size_t k = 0; k < part_index.size(); ++k) pending->part_ids[k] = residentScan(part_index[k]);
  pending->T_parts.clear();
  for (const auto& T : part_T) pending->T_parts.insert(pending->T_parts.end(), T.data(), T.data() + 16);
  pending->active = true;
}

// reference :493-519: ConvergenceError keeps the initial guess; the result becomes a RelativePose
void LaserTrack::finishLocalScanToSubMap(const PendingIcp& pending, int rc, const float* T_out16) {
  PointMatcher::TransformationParameters icp_solution = pending.T0;
  if (rc == LS_ERR_CONVERGENCE) {
    // PointMatcher::ConvergenceError is swallowed: keep the initial guess (reference :495-502)
  } else {
    throwOnError(ctx_, rc, "ls_icp_register_submap");
    std::memcpy(icp_solution.data(), T_out16, 16 * sizeof(float));
  }
  RelativePose icp_transformation = pending.icp_transformation;
  icp_transformation.T_a_b = convertTransformationMatrixToSE3(icp_solution);
  icp_transformation.key_a = findPose(icp_transformation.time_a_ns).key;
  icp_transformation.key_b = findPose(icp_transformation.time_b_ns).key;
  icp_transformations_.push_back(icp_transformation);
}

// reference :521-555 (reverse linear scan for an exact time stamp)
const Pose& LaserTrack::findPose(const Time& timestamp_ns) const {
  LS_CHECK(!pose_measurements_.empty(), "Cannot register the scan as no pose was registered.");
  for (auto it = pose_measurements_.rbegin(); it != pose_measurements_.rend(); ++it)
    if (it->time_ns == timestamp_ns) return *it;
  throw std::logic_error("CHECK failed: The requested time does not exist in the pose measurements.");
}
Pose& LaserTrack::findPose(const Time& timestamp_ns) {
  return const_cast<Pose&>(static_cast<const LaserTrack*>(this)->findPose(timestamp_ns));
}
// reference :557-571
Pose LaserTrack::findNearestPose(const Time& timestamp_ns) const {
  std::lock_guard<std::recursive_mutex> lock(full_laser_track_mutex_);
  Pose pose;
  pose.time_ns = timestamp_ns;
  pose.T_w = evaluate(timestamp_ns);
  pose.key = Key();
  return pose;
}
// reference :573-582; keys are unique across tracks (mincurves' process-wide key generator) and carry the track id
Key LaserTrack::extendTrajectory(const Time& timestamp_ns, const SE3& value) {
  LS_CHECK(trajectory_.empty() || timestamp_ns > trajectory_.rbegin()->first, "trajectory must be extended forward in time");
  const Key key = ((Key)laser_track_id_ << 48) | (g_key_counter.fetch_add(1) & 0xFFFFFFFFFFFFull);
  trajectory_.emplace(timestamp_ns, Node{value, key});
  return key;
}
size_t LaserTrack::scanIndexAtTime(const curves::Time& time_ns) const {  // reference :584-600
  for (size_t i = 0; i < laser_scans_.size(); ++i)
    if (laser_scans_[i].time_ns == time_ns) return i;
  throw std::logic_error("CHECK failed: Could not find the scan.");
}
gtsam::Expression<SE3> LaserTrack::getValueExpression(const curves::Time& time_ns) const {
  return gtsam::Expression<SE3>(getValueKey(time_ns));  // exact node times only, as every caller in laser_slam uses it
}
Key LaserTrack::getValueKey(const curves::Time& time_ns) const {
  std::lock_guard<std::recursive_mutex> lock(full_laser_track_mutex_);
  auto it = trajectory_.find(time_ns);
  LS_CHECK(it != trajectory_.end(), "no trajectory node at that time");
  return it->second.key;
}
SE3 LaserTrack::evaluate(const curves::Time& time_ns) const {
  std::lock_guard<std::recursive_mutex> lock(full_laser_track_mutex_);
  auto it = trajectory_.find(time_ns);
  LS_CHECK(it != trajectory_.end(), "no trajectory node at that time (only exact node times are evaluated)");
  return it->second.value;
}
void LaserTrack::getScanMatchingTimes(std::map<Time, double>* out) const {
  LS_CHECK(out != NULL, "null output");
  *out = scan_matching_times_;
}
void LaserTrack::saveTrajectory(const std::string& filename) const {  // curves::saveCurveTimesAndValues
  std::lock_guard<std::recursive_mutex> lock(full_laser_track_mutex_);
  std::ofstream out(filename.c_str());
  out.precision(17);
  for (const auto& kv : trajectory_) {
    double a[7];
    kv.second.value.toArray7(a);
    out << kv.first << "," << a[4] << "," << a[5] << "," << a[6] << "," << a[0] << "," << a[1] << "," << a[2] << "," << a[3] << "\n";
  }
}

void LaserTrack::assembleSubMap(const std::vector<size_t>& scan_indices,
                                const std::vector<PointMatcher::TransformationParameters>& Ts, DataPoints* out) const {
  LS_CHECK(!scan_indices.empty() && scan_indices.size() == Ts.size(), "bad sub-map description");
  // a private ring sized for this request (loop-closure sub-maps can be wider than the rolling window)
  size_t max_pts = 0, total = 0;
  for (size_t idx : scan_indices) {
    max_pts = std::max(max_pts, laser_scans_[idx].scan.getNbPoints());
    total += laser_scans_[idx].scan.getNbPoints();
  }
  ls_map* tmp = nullptr;
  throwOnError(ctx_, ls_map_create(ctx_, (int)std::max<size_t>(2, scan_indices.size()), (int)std::max<size_t>(1, max_pts), &tmp),
               "ls_map_create");
  std::vector<uint64_t> ids;
  std::vector<float> T_flat;
  try {
    for (size_t k = 0; k < scan_indices.size(); ++k) {
      const DataPoints& c = laser_scans_[scan_indices[k]].scan;
      const int off = c.descriptorOffset("normals");
      LS_CHECK(off >= 0, "scan without normals");
      uint64_t id = 0;
      throwOnError(ctx_, ls_map_push_scan(tmp, c.features.data(), c.descriptors.data() + off, (int)c.descriptorDim,
                                          (int)c.getNbPoints(), &id), "ls_map_push_scan");
      ids.push_back(id);
      T_flat.insert(T_flat.end(), Ts[k].data(), Ts[k].data() + 16);
    }
    std::vector<float> feat(4 * std::max<size_t>(1, total)), nrm(3 * std::max<size_t>(1, total));
    int m = 0;
    throwOnError(ctx_, ls_map_assemble(ctx_, tmp, (int)ids.size(), ids.data(), T_flat.data(), feat.data(), nrm.data(), &m),
                 "ls_map_assemble");
    *out = DataPoints::fromArrays(feat.data(), nrm.data(), (size_t)m);
  } catch (...) {
    ls_map_destroy(tmp);
    throw;
  }
  ls_map_destroy(tmp);
}

// reference :602-651: the centre scan verbatim, then up to `radius` scans before it (decreasing time stamps) and after
// it (increasing), each re-expressed in the centre scan's frame
void LaserTrack::describeSubMapAroundTime(const curves::Time& time_ns, const unsigned int sub_maps_radius,
                                          std::vector<size_t>* scan_indices,
                                          std::vector<PointMatcher::TransformationParameters>* Ts) const {
  const SE3 T_w_a = evaluate(time_ns);
  const size_t centre = scanIndexAtTime(time_ns);
  scan_indices->assign(1, centre);
  Ts->assign(1, PointMatcher::TransformationParameters());
  auto add = [&](size_t i) {
    PointMatcher::TransformationParameters T = toFloatMatrix(T_w_a.inverse() * evaluate(laser_scans_[i].time_ns));
    correctTransformationMatrix(&T);
    scan_indices->push_back(i);
    Ts->push_back(T);
  };
  for (unsigned int i = 1; i <= sub_maps_radius && centre >= i; ++i) add(centre - i);
  for (unsigned int i = 1; i <= sub_maps_radius && centre + i < laser_scans_.size(); ++i) add(centre + i);
}

void LaserTrack::buildSubMapAroundTime(const curves::Time& time_ns, const unsigned int sub_maps_radius, DataPoints* submap_out) const {
  std::lock_guard<std::recursive_mutex> lock(full_laser_track_mutex_);
  LS_CHECK(submap_out != NULL, "null output");
  std::vector<size_t> idx;
  std::vector<PointMatcher::TransformationParameters> Ts;
  describeSubMapAroundTime(time_ns, sub_maps_radius, &idx, &Ts);
  assembleSubMap(idx, Ts, submap_out);
}

void LaserTrack::stageSubMapAroundTime(const curves::Time& time_ns, const unsigned int sub_maps_radius, ls_ctx* ctx,
                                       ls_map** ring_out, std::vector<uint64_t>* ids_out, std::vector<float>* T_parts_out) const {
  std::lock_guard<std::recursive_mutex> lock(full_laser_track_mutex_);
  LS_CHECK(ctx != NULL && ring_out != NULL && ids_out != NULL && T_parts_out != NULL, "null argument");
  std::vector<size_t> idx;
  std::vector<PointMatcher::TransformationParameters> Ts;
  describeSubMapAroundTime(time_ns, sub_maps_radius, &idx, &Ts);
  size_t max_pts = 1;
  for (size_t i : idx) max_pts = std::max(max_pts, laser_scans_[i].scan.getNbPoints());
  ls_map* ring = nullptr;
  throwOnError(ctx, ls_map_create(ctx, (int)std::max<size_t>(2, idx.size()), (int)max_pts, &ring), "ls_map_create");
  ids_out->clear();
  T_parts_out->clear();
  try {
    for (size_t k = 0; k < idx.size(); ++k) {
      const DataPoints& c = laser_scans_[idx[k]].scan;
      const int off = c.descriptorOffset("normals");
      LS_CHECK(off >= 0, "scan without normals");
      uint64_t id = 0;
      throwOnError(ctx, ls_map_push_scan(ring, c.features.data(), c.descriptors.data() + off, (int)c.descriptorDim,
                                         (int)c.getNbPoints(), &id), "ls_map_push_scan");
      ids_out->push_back(id);
      T_parts_out->insert(T_parts_out->end(), Ts[k].data(), Ts[k].data() + 16);
    }
  } catch (...) {
    ls_map_destroy(ring);
    throw;
  }
  *ring_out = ring;
}

}  // namespace laser_slam
