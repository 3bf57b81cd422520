// IncrementalEstimator over the ls_b200 C ABI.  Control flow follows reference
// laser_slam/src/incremental_estimator.cpp (cited per function); gtsam::ISAM2 is replaced by the device pose
// graph (ls_pg_*): every update runs three Gauss-Newton iterations over the whole graph, mirroring
// isam2_.update(new) + update() + update() (reference :156-159, :258-262, :272-289).
#include "laser_slam/incremental_estimator.hpp"

#include <algorithm>
#include <fstream>
#include <sstream>
#include <stdexcept>

namespace laser_slam {

namespace {
#define LS_CHECK(cond, msg)                                             \
  do {                                                                  \
    if (!(cond)) throw std::logic_error(std::string("CHECK failed: ") + (msg)); \
  } while (0)
}  // namespace

// reference :12-61
IncrementalEstimator::IncrementalEstimator(const EstimatorParams& parameters, unsigned int n_laser_slam_workers)
    : n_laser_slam_workers_(n_laser_slam_workers), params_(parameters) {
  std::memset(&last_stats_, 0, sizeof(last_stats_));
  if (ls_pg_create(params_.laser_track_params.cuda_device, &graph_) != LS_OK)
    throw std::runtime_error("ls_pg_create failed: no usable CUDA device (no CPU fallback)");
  // all tracks live on one device context and share one scan ring (every track may count on nscan_in_sub_map + 4
  // slots), so that processPosesAndLaserScans can register them in one batched launch
  if (ls_b200_init(params_.laser_track_params.cuda_device, &track_ctx_) != LS_OK)
    throw std::runtime_error("ls_b200_init failed: no usable CUDA device (no CPU fallback)");
  const int slots = std::max(8, params_.laser_track_params.nscan_in_sub_map + 4);
  track_ring_capacity_ = slots * (int)std::max(1u, n_laser_slam_workers_);
  for (unsigned int i = 0u; i < n_laser_slam_workers_; ++i)
    laser_tracks_.push_back(std::make_shared<LaserTrack>(params_.laser_track_params, i, track_ctx_, &track_ring_,
                                                         &track_ring_capacity_, &track_ring_max_pts_, slots));
  using namespace gtsam::noiseModel;
  loop_closure_noise_model_ = Diagonal::Sigmas(params_.loop_closure_noise_model);
  if (params_.add_m_estimator_on_loop_closures)
    loop_closure_noise_model_ = Robust::Create(mEstimator::Cauchy::Create(1), loop_closure_noise_model_);
  first_association_noise_model_ = Diagonal::Sigmas(std::array<double, 6>{{0.05, 0.05, 0.05, 0.015, 0.015, 0.015}});  // reference :40-48
  // same chain as the lidar odometry (reference :50-60)
  ls_icp_default_params(&icp_params_);
  std::ifstream ifs(params_.laser_track_params.icp_configuration_file.c_str());
  if (ifs.good()) {
    std::stringstream ss;
    ss << ifs.rdbuf();
    if (ls_icp_params_from_yaml(ss.str().c_str(), &icp_params_) != LS_OK) throw std::runtime_error("unsupported ICP chain");
  } else {
    icp_params_.trim_ratio = 0.85f;
    icp_params_.min_diff_trans = 0.001f;
    icp_params_.smooth_length = 3;
  }
}

IncrementalEstimator::~IncrementalEstimator() {
  laser_tracks_.clear();
  if (track_ring_) ls_map_destroy(track_ring_);
  if (track_ctx_) ls_b200_destroy(track_ctx_);
  if (icp_ctx_) ls_b200_destroy(icp_ctx_);
  if (graph_) ls_pg_destroy(graph_);
}

// (new) the scan callbacks of several workers, registrations batched (see the header)
void IncrementalEstimator::processPosesAndLaserScans(const std::vector<unsigned int>& worker_ids, const std::vector<Pose>& poses,
                                                     const std::vector<LaserScan>& scans,
                                                     std::vector<gtsam::NonlinearFactorGraph>* new_factors,
                                                     std::vector<gtsam::Values>* new_values, std::vector<bool>* is_prior) {
  std::lock_guard<std::recursive_mutex> lock(full_class_mutex_);
  LS_CHECK(new_factors != NULL && new_values != NULL && is_prior != NULL, "null output");
  beginPosesAndLaserScans(worker_ids, poses, scans);
  endPosesAndLaserScans(new_factors, new_values, is_prior);
}

void IncrementalEstimator::beginPosesAndLaserScans(const std::vector<unsigned int>& worker_ids, const std::vector<Pose>& poses,
                                                   const std::vector<LaserScan>& scans) {
  std::lock_guard<std::recursive_mutex> lock(full_class_mutex_);
  LS_CHECK(!step_.open, "beginPosesAndLaserScans: the previous step has not been ended");
  const size_t n = worker_ids.size();
  LS_CHECK(poses.size() == n && scans.size() == n, "one pose and one scan per worker");
  step_ = PendingStep();
  step_.worker_ids = worker_ids;
  step_.pending.resize(n);
  for (size_t i = 0; i < n; ++i) {
    LS_CHECK(worker_ids[i] < laser_tracks_.size(), "bad worker id");
    for (size_t j = 0; j < i; ++j) LS_CHECK(worker_ids[j] != worker_ids[i], "a worker may appear once per step");
    laser_tracks_[worker_ids[i]]->beginPoseAndLaserScan(poses[i], scans[i], &step_.pending[i]);
    if (step_.pending[i].active) step_.active.push_back(i);
  }
  step_.open = true;
  // a scan uploaded by a later track may have evicted an earlier track's scan from the shared ring only if the ring
  // were too small for one step: it holds nscan_in_sub_map + 4 slots per track
  const std::vector<size_t>& active = step_.active;
  step_.T_outs.assign(16 * std::max<size_t>(active.size(), 1), 0.f);
  step_.stats.assign(std::max<size_t>(active.size(), 1), ls_icp_stats());
  step_.statuses.assign(std::max<size_t>(active.size(), 1), LS_OK);
  constexpr size_t kMaxBatch = 160;  // ls_icp_register_submap_batch's limit
  for (size_t b0 = 0; b0 < active.size(); b0 += kMaxBatch) {
    const size_t nb = std::min(kMaxBatch, active.size() - b0);
    std::vector<uint64_t> reading_ids, part_ids;
    std::vector<int> n_parts;
    std::vector<float> T_parts, T0s;
    for (size_t k = 0; k < nb; ++k) {
      const LaserTrack::PendingIcp& p = step_.pending[active[b0 + k]];
      reading_ids.push_back(p.reading_id);
      n_parts.push_back((int)p.part_ids.size());
      part_ids.insert(part_ids.end(), p.part_ids.begin(), p.part_ids.end());
      T_parts.insert(T_parts.end(), p.T_parts.begin(), p.T_parts.end());
      T0s.insert(T0s.end(), p.T0.data(), p.T0.data() + 16);
    }
    const ls_icp_params& prm = laser_tracks_[worker_ids[active[b0]]]->icpParams();
    int rc;
    if (active.size() <= kMaxBatch) {  // the usual case: one launch, left in flight until endPosesAndLaserScans
      std::memcpy(step_.T_outs.data(), T0s.data(), sizeof(float) * T0s.size());
      rc = ls_icp_register_submap_batch_begin(track_ctx_, &prm, track_ring_, (int)nb, reading_ids.data(), n_parts.data(),
                                              part_ids.data(), T_parts.data(), T0s.data());
      step_.inflight = rc == LS_OK;
    } else {
      rc = ls_icp_register_submap_batch(track_ctx_, &prm, track_ring_, (int)nb, reading_ids.data(), n_parts.data(), part_ids.data(),
                                        T_parts.data(), T0s.data(), step_.T_outs.data() + 16 * b0, step_.stats.data() + b0,
                                        step_.statuses.data() + b0);
    }
    if (rc < 0) {
      step_.open = false;
      throw std::runtime_error(std::string("ls_icp_register_submap_batch: ") + ls_b200_last_error(track_ctx_));
    }
  }
}

void IncrementalEstimator::endPosesAndLaserScans(std::vector<gtsam::NonlinearFactorGraph>* new_factors,
                                                 std::vector<gtsam::Values>* new_values, std::vector<bool>* is_prior) {
  std::lock_guard<std::recursive_mutex> lock(full_class_mutex_);
  LS_CHECK(step_.open, "endPosesAndLaserScans without beginPosesAndLaserScans");
  LS_CHECK(new_factors != NULL && new_values != NULL && is_prior != NULL, "null output");
  step_.open = false;
  if (step_.inflight) {
    step_.inflight = false;
    const int rc = ls_icp_register_submap_batch_end(track_ctx_, step_.T_outs.data(), step_.stats.data(), step_.statuses.data());
    if (rc < 0) throw std::runtime_error(std::string("ls_icp_register_submap_batch_end: ") + ls_b200_last_error(track_ctx_));
  }
  const size_t n = step_.worker_ids.size();
  new_factors->assign(n, gtsam::NonlinearFactorGraph());
  new_values->assign(n, gtsam::Values());
  is_prior->assign(n, false);
  size_t a = 0;
  for (size_t i = 0; i < n; ++i) {
    bool prior = false;
    LaserTrack& track = *laser_tracks_[step_.worker_ids[i]];
    if (step_.pending[i].active) {
      track.endPoseAndLaserScan(&step_.pending[i], step_.statuses[a], step_.T_outs.data() + 16 * a, &step_.stats[a],
                                &(*new_factors)[i], &(*new_values)[i], &prior);
      ++a;
    } else {
      track.endPoseAndLaserScan(&step_.pending[i], LS_OK, NULL, NULL, &(*new_factors)[i], &(*new_values)[i], &prior);
    }
    (*is_prior)[i] = prior;
  }
}

void IncrementalEstimator::prefetchLaserScans(const std::vector<unsigned int>& worker_ids, const std::vector<LaserScan>& scans) {
  std::lock_guard<std::recursive_mutex> lock(full_class_mutex_);
  LS_CHECK(worker_ids.size() == scans.size(), "one scan per worker");
  for (size_t i = 0; i < worker_ids.size(); ++i) {
    LS_CHECK(worker_ids[i] < laser_tracks_.size(), "bad worker id");
    laser_tracks_[worker_ids[i]]->prefetchLaserScan(scans[i]);
  }
}

// reference :63-149
void IncrementalEstimator::processLoopClosure(const RelativePose& loop_closure) {
  std::lock_guard<std::recursive_mutex> lock(full_class_mutex_);
  LS_CHECK(loop_closure.track_id_a < laser_tracks_.size() && loop_closure.track_id_b < laser_tracks_.size(), "bad track id");
  LaserTrack& track_a = *laser_tracks_[loop_closure.track_id_a];
  LaserTrack& track_b = *laser_tracks_[loop_closure.track_id_b];
  if (loop_closure.track_id_a == loop_closure.track_id_b)
    LS_CHECK(loop_closure.time_a_ns < loop_closure.time_b_ns, "Loop closure has invalid time.");
  LS_CHECK(loop_closure.time_a_ns >= track_a.getMinTime() && loop_closure.time_a_ns <= track_a.getMaxTime(), "Loop closure has invalid time.");
  LS_CHECK(loop_closure.time_b_ns >= track_b.getMinTime() && loop_closure.time_b_ns <= track_b.getMaxTime(), "Loop closure has invalid time.");

  RelativePose updated = loop_closure;
  // world-frame correction -> relative pose of the two nodes (reference :78-87)
  const SE3 T_w_a = track_a.evaluate(loop_closure.time_a_ns);
  const SE3 T_w_b = track_b.evaluate(loop_closure.time_b_ns);
  updated.T_a_b = T_w_a.inverse() * loop_closure.T_a_b * T_w_b;

  if (params_.do_icp_step_on_loop_closures) {  // reference :89-115; a ConvergenceError propagates here
    const PointMatcher::TransformationParameters initial_guess =
        PointMatcher::TransformationParameters::cast(updated.T_a_b.getTransformationMatrix());
    if (!icp_ctx_ && ls_b200_init(params_.laser_track_params.cuda_device, &icp_ctx_) != LS_OK)
      throw std::runtime_error("ls_b200_init failed");
    // both sub-maps are assembled on the device (ls_icp_register_submaps): the scans go up once, nothing comes back
    // but the 4x4
    ls_map *ring_a = nullptr, *ring_b = nullptr;
    std::vector<uint64_t> ids_a, ids_b;
    std::vector<float> T_a, T_b;
    PointMatcher::TransformationParameters icp_solution;
    int rc = LS_OK;
    try {
      track_a.stageSubMapAroundTime(loop_closure.time_a_ns, params_.loop_closures_sub_maps_radius, icp_ctx_, &ring_a, &ids_a, &T_a);
      track_b.stageSubMapAroundTime(loop_closure.time_b_ns, params_.loop_closures_sub_maps_radius, icp_ctx_, &ring_b, &ids_b, &T_b);
      rc = ls_icp_register_submaps(icp_ctx_, &icp_params_, ring_a, (int)ids_a.size(), ids_a.data(), T_a.data(), ring_b,
                                   (int)ids_b.size(), ids_b.data(), T_b.data(), initial_guess.data(), icp_solution.data(), NULL);
    } catch (...) {
      if (ring_a) ls_map_destroy(ring_a);
      if (ring_b) ls_map_destroy(ring_b);
      throw;
    }
    ls_map_destroy(ring_a);
    ls_map_destroy(ring_b);
    if (rc == LS_ERR_CONVERGENCE) throw PointMatcher::ConvergenceError(ls_b200_last_error(icp_ctx_));
    if (rc != LS_OK) throw std::runtime_error(std::string("ls_icp_register_submaps: ") + ls_b200_last_error(icp_ctx_));
    updated.T_a_b = convertTransformationMatrixToSE3(icp_solution);
  }

  // loop-closure factor, once with the loop-closure noise and once with the looser "first association" noise
  // (reference :117-133)
  // reference :117-125: ExpressionFactor over inverse(T_w_a) * T_w_b, both trajectory leaves
  auto make = [&](const gtsam::noiseModel::Base::shared_ptr& noise) {
    using gtsam::Expression;
    Expression<SE3> T_w_b(track_b.getValueExpression(updated.time_b_ns));
    Expression<SE3> T_w_a(track_a.getValueExpression(updated.time_a_ns));
    Expression<SE3> T_a_w(kindr::minimal::inverse(T_w_a));
    Expression<SE3> relative(kindr::minimal::compose(T_a_w, T_w_b));
    return gtsam::ExpressionFactor<SE3>(noise, updated.T_a_b, relative);
  };
  gtsam::NonlinearFactorGraph new_factors, new_associations_factors;
  new_factors.push_back(make(loop_closure_noise_model_));
  new_associations_factors.push_back(make(first_association_noise_model_));

  std::vector<unsigned int> affected_worker_ids{loop_closure.track_id_a, loop_closure.track_id_b};
  gtsam::Values new_values;
  const gtsam::Values result = estimateAndRemove(new_factors, new_associations_factors, new_values, affected_worker_ids,
                                                 updated.time_b_ns);
  for (auto& track : laser_tracks_) track->updateFromGTSAMValues(result);  // reference :145-147
}

Pose IncrementalEstimator::getCurrentPose(unsigned int laser_track_id) const {
  std::lock_guard<std::recursive_mutex> lock(full_class_mutex_);
  return laser_tracks_.at(laser_track_id)->getCurrentPose();
}

gtsam::Values IncrementalEstimator::updateGraph(const gtsam::NonlinearFactorGraph& factors, const gtsam::Values& values,
                                                const std::vector<uint64_t>& remove, std::vector<uint64_t>* new_indices) {
  auto fail = [&](const char* what) { throw std::runtime_error(std::string(what) + ": " + ls_pg_last_error(graph_)); };
  if (!values.empty()) {
    std::vector<uint64_t> keys;
    std::vector<uint32_t> tracks;
    std::vector<double> poses;
    for (const auto& kv : values) {
      keys.push_back(kv.first);
      tracks.push_back((uint32_t)(kv.first >> 48));  // keys carry the track id (LaserTrack::extendTrajectory)
      double a[7];
      kv.second.toArray7(a);
      poses.insert(poses.end(), a, a + 7);
    }
    if (ls_pg_add_poses(graph_, keys.data(), tracks.data(), poses.data(), (int)keys.size()) != LS_OK) fail("ls_pg_add_poses");
  }
  if (!remove.empty() && ls_pg_remove_factors(graph_, remove.data(), (int)remove.size()) != LS_OK) fail("ls_pg_remove_factors");
  std::vector<uint64_t> idx(factors.size());
  if (!factors.empty() && ls_pg_add_factors(graph_, factors.factors().data(), (int)factors.size(), idx.data()) != LS_OK)
    fail("ls_pg_add_factors");
  if (new_indices) *new_indices = idx;
  const int rc = ls_pg_optimize(graph_, 3, &last_stats_);
  if (rc != LS_OK) fail("ls_pg_optimize");
  int n = 0;
  ls_pg_get_poses(graph_, NULL, NULL, &n);
  std::vector<uint64_t> keys(n);
  std::vector<double> poses(7 * (size_t)n);
  ls_pg_get_poses(graph_, keys.data(), poses.data(), &n);
  gtsam::Values result;  // isam2_.calculateEstimate(): every value
  for (int i = 0; i < n; ++i) result.insert(keys[i], SE3::fromArray7(&poses[7 * (size_t)i]));
  return result;
}

// reference :151-163
gtsam::Values IncrementalEstimator::estimate(const gtsam::NonlinearFactorGraph& new_factors, const gtsam::Values& new_values,
                                             laser_slam::Time) {
  std::lock_guard<std::recursive_mutex> lock(full_class_mutex_);
  return updateGraph(new_factors, new_values, {}, nullptr);
}

// reference :165-266
gtsam::Values IncrementalEstimator::estimateAndRemove(const gtsam::NonlinearFactorGraph& new_factors,
                                                      const gtsam::NonlinearFactorGraph& new_associations_factors,
                                                      const gtsam::Values& new_values,
                                                      const std::vector<unsigned int>& affected_worker_ids, laser_slam::Time) {
  std::lock_guard<std::recursive_mutex> lock(full_class_mutex_);
  LS_CHECK(affected_worker_ids.size() == 2u, "exactly two affected workers");
  std::vector<uint64_t> factor_indices_to_remove;
  const unsigned int first = affected_worker_ids[0], second = affected_worker_ids[1];
  if (first != second) {
    int g_first = -1, g_second = -1;
    for (size_t g = 0; g < linked_workers_.size(); ++g) {
      if (std::find(linked_workers_[g].begin(), linked_workers_[g].end(), first) != linked_workers_[g].end()) g_first = (int)g;
      if (std::find(linked_workers_[g].begin(), linked_workers_[g].end(), second) != linked_workers_[g].end()) g_second = (int)g;
    }
    LS_CHECK(g_first >= 0 && g_second >= 0, "both workers must have registered a prior before they are linked");
    if (g_first != g_second) {
      // keep the group holding worker 0, dissolve the other one and drop its prior (reference :208-237)
      const bool first_has_zero = std::find(linked_workers_[g_first].begin(), linked_workers_[g_first].end(), 0u) != linked_workers_[g_first].end();
      const int keep = first_has_zero ? g_first : g_second, drop = first_has_zero ? g_second : g_first;
      for (unsigned int worker_id : linked_workers_[drop]) {
        auto it = factor_indices_to_remove_.find(worker_id);
        if (it != factor_indices_to_remove_.end()) {
          factor_indices_to_remove.push_back(it->second);
          factor_indices_to_remove_.erase(it);
        }
        linked_workers_[keep].push_back(worker_id);
      }
      LS_CHECK(factor_indices_to_remove.size() == 1u, "exactly one prior to remove");
      linked_workers_.erase(linked_workers_.begin() + drop);
    }
  }
  // a removed prior means this is the first association of two groups: use the looser factor (reference :251-256)
  const gtsam::NonlinearFactorGraph& to_add = factor_indices_to_remove.empty() ? new_factors : new_associations_factors;
  return updateGraph(to_add, new_values, factor_indices_to_remove, nullptr);
}

// reference :268-291
gtsam::Values IncrementalEstimator::registerPrior(const gtsam::NonlinearFactorGraph& new_factors, const gtsam::Values& new_values,
                                                  const unsigned int worker_id) {
  std::lock_guard<std::recursive_mutex> lock(full_class_mutex_);
  std::vector<uint64_t> idx;
  const gtsam::Values result = updateGraph(new_factors, new_values, {}, &idx);
  LS_CHECK(idx.size() == 1u, "registerPrior expects exactly one new factor");
  if (worker_id > 0u) factor_indices_to_remove_.insert(std::make_pair(worker_id, (size_t)idx[0]));
  linked_workers_.push_back(std::vector<unsigned int>{worker_id});
  return result;
}

std::shared_ptr<LaserTrack> IncrementalEstimator::getLaserTrack(unsigned int laser_track_id) {
  std::lock_guard<std::recursive_mutex> lock(full_class_mutex_);
  LS_CHECK(laser_track_id < laser_tracks_.size(), "bad laser track id");
  return laser_tracks_[laser_track_id];
}
std::vector<std::shared_ptr<LaserTrack> > IncrementalEstimator::getAllLaserTracks() {
  std::lock_guard<std::recursive_mutex> lock(full_class_mutex_);
  return laser_tracks_;
}

}  // namespace laser_slam
