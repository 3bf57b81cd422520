// C hooks over the C++ host layer so that tests (ctypes) can drive LaserTrack / IncrementalEstimator exactly the
// way the ROS worker does (reference laser_slam_ros/src/laser_slam_worker.cpp:124-173): processPoseAndLaserScan,
// then registerPrior or estimate, then updateFromGTSAMValues.  Not part of the drop-in boundary.
#include <algorithm>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "laser_slam/incremental_estimator.hpp"
#include "laser_slam/local_map.hpp"
#include "laser_slam/distance_map.hpp"
#include "laser_slam/occupancy_map.hpp"
#include "laser_slam/velodyne_assembler.hpp"

using namespace laser_slam;

namespace {
struct Handle {
  std::unique_ptr<IncrementalEstimator> est;
  std::string err;
  std::vector<unsigned int> step_ids;   // the step between lsh_begin_batch and lsh_end_batch
  std::vector<int64_t> step_times;
};
LaserScan make_scan(const float* feat4, const float* normals3, int n, int64_t time_ns, bool view) {
  LaserScan s;
  s.scan = view ? DataPoints::viewOfArrays(feat4, normals3, (size_t)n) : DataPoints::fromArrays(feat4, normals3, (size_t)n);
  s.time_ns = time_ns;
  return s;
}
template <typename F>
int guarded(Handle* h, F f) {
  try {
    return f();
  } catch (const laser_slam::PointMatcher::ConvergenceError& e) {
    h->err = e.what();
    return LS_ERR_CONVERGENCE;
  } catch (const std::exception& e) {
    h->err = e.what();
    return LS_ERR_STATE;
  }
}
}  // namespace

extern "C" {

void* lsh_create(int n_workers, int nscan_in_sub_map, int use_icp_factors, int use_odom_factors, int robust_icp, int device,
                 int do_icp_step_on_loop_closures, int loop_closures_sub_maps_radius, const char* icp_yaml_path,
                 const char* icp_input_filters_path, char* err, int errlen) {
  try {
    EstimatorParams p;
    p.laser_track_params.nscan_in_sub_map = nscan_in_sub_map;
    p.laser_track_params.use_icp_factors = use_icp_factors != 0;
    p.laser_track_params.use_odom_factors = use_odom_factors != 0;
    p.laser_track_params.add_m_estimator_on_icp = robust_icp != 0;
    p.laser_track_params.cuda_device = device;
    p.laser_track_params.icp_configuration_file = icp_yaml_path ? icp_yaml_path : "";
    p.laser_track_params.icp_input_filters_file = icp_input_filters_path ? icp_input_filters_path : "";
    p.do_icp_step_on_loop_closures = do_icp_step_on_loop_closures != 0;
    p.loop_closures_sub_maps_radius = loop_closures_sub_maps_radius;
    Handle* h = new Handle();
    h->est.reset(new IncrementalEstimator(p, (unsigned int)n_workers));
    return h;
  } catch (const std::exception& e) {
    if (err && errlen > 0) std::strncpy(err, e.what(), (size_t)errlen - 1), err[errlen - 1] = 0;
    return nullptr;
  }
}

void lsh_destroy(void* hv) { delete static_cast<Handle*>(hv); }
const char* lsh_last_error(void* hv) { return static_cast<Handle*>(hv)->err.c_str(); }

// One scan callback.  pose7 = odometry pose T_w (qw,qx,qy,qz,tx,ty,tz); normals3 may be NULL (raw scan: the track's
// input filters must then make the normals).  out_icp7 (may be NULL) receives the ICP
// T_a_b of this step (identity for the first scan); out_stats (may be NULL) the device-side ICP statistics.
int lsh_step(void* hv, int worker, int64_t time_ns, const double* pose7, const float* feat4, const float* normals3, int n,
             double* out_icp7, ls_icp_stats* out_stats) {
  Handle* h = static_cast<Handle*>(hv);
  return guarded(h, [&]() {
    std::shared_ptr<LaserTrack> track = h->est->getLaserTrack((unsigned int)worker);
    Pose pose;
    pose.T_w = SE3::fromArray7(pose7);
    pose.time_ns = time_ns;
    LaserScan scan;
    scan.scan = DataPoints::fromArrays(feat4, normals3, (size_t)n);
    scan.time_ns = time_ns;
    gtsam::NonlinearFactorGraph new_factors;
    gtsam::Values new_values;
    bool is_prior = false;
    track->processPoseAndLaserScan(pose, scan, &new_factors, &new_values, &is_prior);
    gtsam::Values result = is_prior ? h->est->registerPrior(new_factors, new_values, (unsigned int)worker)
                                    : h->est->estimate(new_factors, new_values, time_ns);
    track->updateFromGTSAMValues(result);
    if (out_icp7) {
      SE3 T;
      if (!track->getIcpTransformations().empty() && !is_prior) T = track->getIcpTransformations().back().T_a_b;
      T.toArray7(out_icp7);
    }
    if (out_stats) *out_stats = track->getLastIcpStats();
    return LS_OK;
  });
}

// The scan callbacks of `n_workers` workers at once (IncrementalEstimator::processPosesAndLaserScans: one batched
// launch for all registrations), each followed by registerPrior / estimate and updateFromGTSAMValues exactly as
// lsh_step does.  pose7: 7 doubles per worker; feat4 / normals3: per-worker host pointers; n: points per worker.
// out_icp7 (may be NULL): 7 doubles per worker.  with_estimator == 0 skips the pose-graph update (odometry only).
int lsh_step_batch(void* hv, int n_workers, const int* workers, const int64_t* times_ns, const double* pose7, const float* const* feat4,
                   const float* const* normals3, const int* n, int with_estimator, double* out_icp7, ls_icp_stats* out_stats) {
  // with_estimator bit 1 (value 2): the DataPoints are VIEWS of the caller's arrays (DataPoints::viewOfArrays), which
  // must then stay valid for the life of the estimator -- the tracks keep every scan.  Otherwise they are copies.
  const bool views = (with_estimator & 2) != 0;
  with_estimator &= 1;
  Handle* h = static_cast<Handle*>(hv);
  return guarded(h, [&]() {
    std::vector<unsigned int> ids;
    std::vector<Pose> poses((size_t)n_workers);
    std::vector<LaserScan> scans((size_t)n_workers);
    for (int i = 0; i < n_workers; ++i) {
      ids.push_back((unsigned int)workers[i]);
      poses[i].T_w = SE3::fromArray7(pose7 + 7 * (size_t)i);
      poses[i].time_ns = times_ns[i];
      scans[i].scan = views ? DataPoints::viewOfArrays(feat4[i], normals3[i], (size_t)n[i]) : DataPoints::fromArrays(feat4[i], normals3[i], (size_t)n[i]);
      scans[i].time_ns = times_ns[i];
    }
    std::vector<gtsam::NonlinearFactorGraph> nf;
    std::vector<gtsam::Values> nv;
    std::vector<bool> prior;
    h->est->processPosesAndLaserScans(ids, poses, scans, &nf, &nv, &prior);
    for (int i = 0; i < n_workers; ++i) {
      std::shared_ptr<LaserTrack> track = h->est->getLaserTrack(ids[i]);
      if (with_estimator) {
        gtsam::Values result = prior[i] ? h->est->registerPrior(nf[i], nv[i], ids[i]) : h->est->estimate(nf[i], nv[i], times_ns[i]);
        track->updateFromGTSAMValues(result);
      }
      if (out_icp7) {
        SE3 T;
        if (!track->getIcpTransformations().empty() && !prior[i]) T = track->getIcpTransformations().back().T_a_b;
        T.toArray7(out_icp7 + 7 * (size_t)i);
      }
      if (out_stats) out_stats[i] = track->getLastIcpStats();
    }
    return LS_OK;
  });
}

// lsh_step_batch in two halves (IncrementalEstimator::beginPosesAndLaserScans / endPosesAndLaserScans) with the prefetch
// hint in between.  flags bit 1 (value 2): DataPoints are views of the caller's arrays.
int lsh_begin_batch(void* hv, int n_workers, const int* workers, const int64_t* times_ns, const double* pose7, const float* const* feat4,
                    const float* const* normals3, const int* n, int flags) {
  Handle* h = static_cast<Handle*>(hv);
  return guarded(h, [&]() {
    std::vector<Pose> poses((size_t)n_workers);
    std::vector<LaserScan> scans((size_t)n_workers);
    h->step_ids.clear();
    h->step_times.assign(times_ns, times_ns + n_workers);
    for (int i = 0; i < n_workers; ++i) {
      h->step_ids.push_back((unsigned int)workers[i]);
      poses[i].T_w = SE3::fromArray7(pose7 + 7 * (size_t)i);
      poses[i].time_ns = times_ns[i];
      scans[i] = make_scan(feat4[i], normals3[i], n[i], times_ns[i], (flags & 2) != 0);
    }
    h->est->beginPosesAndLaserScans(h->step_ids, poses, scans);
    return LS_OK;
  });
}

int lsh_prefetch(void* hv, int n_workers, const int* workers, const int64_t* times_ns, const float* const* feat4,
                 const float* const* normals3, const int* n, int flags) {
  Handle* h = static_cast<Handle*>(hv);
  return guarded(h, [&]() {
    std::vector<unsigned int> ids;
    std::vector<LaserScan> scans((size_t)n_workers);
    for (int i = 0; i < n_workers; ++i) {
      ids.push_back((unsigned int)workers[i]);
      scans[i] = make_scan(feat4[i], normals3[i], n[i], times_ns[i], (flags & 2) != 0);
    }
    h->est->prefetchLaserScans(ids, scans);
    return LS_OK;
  });
}

int lsh_end_batch(void* hv, int with_estimator, double* out_icp7, ls_icp_stats* out_stats) {
  Handle* h = static_cast<Handle*>(hv);
  return guarded(h, [&]() {
    std::vector<gtsam::NonlinearFactorGraph> nf;
    std::vector<gtsam::Values> nv;
    std::vector<bool> prior;
    h->est->endPosesAndLaserScans(&nf, &nv, &prior);
    for (size_t i = 0; i < h->step_ids.size(); ++i) {
      std::shared_ptr<LaserTrack> track = h->est->getLaserTrack(h->step_ids[i]);
      if (with_estimator & 1) {
        gtsam::Values result = prior[i] ? h->est->registerPrior(nf[i], nv[i], h->step_ids[i]) : h->est->estimate(nf[i], nv[i], h->step_times[i]);
        track->updateFromGTSAMValues(result);
      }
      if (out_icp7) {
        SE3 T;
        if (!track->getIcpTransformations().empty() && !prior[i]) T = track->getIcpTransformations().back().T_a_b;
        T.toArray7(out_icp7 + 7 * i);
      }
      if (out_stats) out_stats[i] = track->getLastIcpStats();
    }
    return LS_OK;
  });
}

int lsh_loop_closure(void* hv, int track_a, int64_t time_a, int track_b, int64_t time_b, const double* w_T_a_b7) {
  Handle* h = static_cast<Handle*>(hv);
  return guarded(h, [&]() {
    RelativePose lc;
    lc.T_a_b = SE3::fromArray7(w_T_a_b7);
    lc.time_a_ns = time_a;
    lc.time_b_ns = time_b;
    lc.track_id_a = (unsigned int)track_a;
    lc.track_id_b = (unsigned int)track_b;
    h->est->processLoopClosure(lc);
    return LS_OK;
  });
}

// Trajectory of one track: times and poses (7 doubles each); returns the number of nodes (<= cap written).
int lsh_trajectory(void* hv, int worker, int64_t* times, double* poses7, int cap) {
  Handle* h = static_cast<Handle*>(hv);
  return guarded(h, [&]() {
    Trajectory traj;
    h->est->getLaserTrack((unsigned int)worker)->getTrajectory(&traj);
    int i = 0;
    for (const auto& kv : traj) {
      if (i < cap) {
        if (times) times[i] = kv.first;
        if (poses7) kv.second.toArray7(poses7 + 7 * (size_t)i);
      }
      ++i;
    }
    return i;
  });
}

int lsh_num_scans(void* hv, int worker) {
  Handle* h = static_cast<Handle*>(hv);
  return guarded(h, [&]() { return (int)h->est->getLaserTrack((unsigned int)worker)->getNumScans(); });
}

// LaserTrack::buildSubMapAroundTime; returns the number of points (features4 / normals3 sized by the caller).
int lsh_build_submap(void* hv, int worker, int64_t time_ns, int radius, float* features4, float* normals3, int cap_points) {
  Handle* h = static_cast<Handle*>(hv);
  return guarded(h, [&]() {
    DataPoints sub;
    h->est->getLaserTrack((unsigned int)worker)->buildSubMapAroundTime(time_ns, (unsigned int)radius, &sub);
    const int m = (int)sub.getNbPoints();
    if (m <= cap_points) {
      std::memcpy(features4, sub.features.data(), sizeof(float) * 4 * (size_t)m);
      if (normals3) std::memcpy(normals3, sub.descriptors.data(), sizeof(float) * 3 * (size_t)m);
    }
    return m;
  });
}

// ---- laser_slam::LocalMap (include/laser_slam/local_map.hpp) on one worker's track, for the tests.  Destroy it before
// the estimator: the map lives on the estimator's context.
}  // extern "C"

namespace {
struct LocalMapHandle {
  std::shared_ptr<LaserTrack> track;
  std::unique_ptr<LocalMap> map;
  DataPoints filtered;                 // what the last lsh_local_map_filter returned
  std::vector<DataPoints> queue;       // what the last lsh_local_map_take_queue took
  std::string err;
};
int copy_cloud(const DataPoints& d, float* out4, int cap) {
  const int n = (int)d.getNbPoints();
  if (out4 && n <= cap) std::memcpy(out4, d.features.data(), sizeof(float) * 4 * (size_t)n);
  return n;
}
template <typename F>
int guarded_lm(LocalMapHandle* h, F f) {
  try {
    return f();
  } catch (const std::exception& e) {
    h->err = e.what();
    return LS_ERR_STATE;
  }
}
}  // namespace

extern "C" {

void* lsh_local_map_create(void* hv, int worker, double distance_to_consider_fixed, int separate_distant_map,
                           int create_filtered_map, double voxel_size_m, int minimum_point_number_per_voxel,
                           int remove_ground_from_local_map, double ground_distance_to_robot_center_m, char* err, int errlen) {
  try {
    LocalMapParams p;
    p.distance_to_consider_fixed = distance_to_consider_fixed;
    p.separate_distant_map = separate_distant_map != 0;
    p.create_filtered_map = create_filtered_map != 0;
    p.voxel_size_m = voxel_size_m;
    p.minimum_point_number_per_voxel = minimum_point_number_per_voxel;
    p.remove_ground_from_local_map = remove_ground_from_local_map != 0;
    p.ground_distance_to_robot_center_m = ground_distance_to_robot_center_m;
    LocalMapHandle* h = new LocalMapHandle();
    h->track = static_cast<Handle*>(hv)->est->getLaserTrack((unsigned int)worker);
    h->map.reset(new LocalMap(p, *h->track));
    return h;
  } catch (const std::exception& e) {
    if (err && errlen > 0) std::strncpy(err, e.what(), (size_t)errlen - 1), err[errlen - 1] = 0;
    return nullptr;
  }
}
void lsh_local_map_destroy(void* lv) { delete static_cast<LocalMapHandle*>(lv); }
const char* lsh_local_map_last_error(void* lv) { return static_cast<LocalMapHandle*>(lv)->err.c_str(); }

int lsh_local_map_add_scan(void* lv) {
  LocalMapHandle* h = static_cast<LocalMapHandle*>(lv);
  return guarded_lm(h, [&]() { h->map->addScan(); return LS_OK; });
}
// getFilteredMap; returns its number of points (read it with lsh_local_map_get(LS_LM_FILTERED_MAP))
int lsh_local_map_filter(void* lv) {
  LocalMapHandle* h = static_cast<LocalMapHandle*>(lv);
  return guarded_lm(h, [&]() { h->map->getFilteredMap(&h->filtered); return (int)h->filtered.getNbPoints(); });
}
// LS_LM_LOCAL / _LOCAL_FILTERED / _DISTANT / _FILTERED_MAP: returns the number of points, written to out4 if <= cap
int lsh_local_map_get(void* lv, int which, float* out4, int cap) {
  LocalMapHandle* h = static_cast<LocalMapHandle*>(lv);
  return guarded_lm(h, [&]() {
    DataPoints d;
    if (which == LS_LM_LOCAL) h->map->getLocalMap(&d);
    else if (which == LS_LM_LOCAL_FILTERED) h->map->getLocalMapFiltered(&d);
    else if (which == LS_LM_DISTANT) h->map->getDistantMap(&d);
    else if (which == LS_LM_FILTERED_MAP) d = h->filtered;
    else return LS_ERR_ARG;
    return copy_cloud(d, out4, cap);
  });
}
// getQueuedPoints; returns the number of clouds taken (read cloud k with lsh_local_map_queued)
int lsh_local_map_take_queue(void* lv) {
  LocalMapHandle* h = static_cast<LocalMapHandle*>(lv);
  return guarded_lm(h, [&]() { h->queue = h->map->getQueuedPoints(); return (int)h->queue.size(); });
}
int lsh_local_map_queued(void* lv, int k, float* out4, int cap) {
  LocalMapHandle* h = static_cast<LocalMapHandle*>(lv);
  if (k < 0 || k >= (int)h->queue.size()) return LS_ERR_ARG;
  return copy_cloud(h->queue[(size_t)k], out4, cap);
}
int lsh_local_map_update(void* lv, const double* last_pose_before_update7, int64_t time_ns) {
  LocalMapHandle* h = static_cast<LocalMapHandle*>(lv);
  return guarded_lm(h, [&]() { h->map->updateLocalMap(SE3::fromArray7(last_pose_before_update7), time_ns); return LS_OK; });
}
int lsh_local_map_clear(void* lv) {
  LocalMapHandle* h = static_cast<LocalMapHandle*>(lv);
  return guarded_lm(h, [&]() { h->map->clearLocalMap(); return LS_OK; });
}

// ---- laser_slam::VelodyneAssembler (include/laser_slam/velodyne_assembler.hpp) for the tests
void* lsh_assembler_create(const float* T_sensor_base16, int naive, int device) {
  VelodyneAssembler::Matrix4 T;
  if (T_sensor_base16) std::memcpy(T.data(), T_sensor_base16, 16 * sizeof(float));
  return new VelodyneAssembler(T, naive != 0, device);
}
void lsh_assembler_destroy(void* a) { delete static_cast<VelodyneAssembler*>(a); }
// returns 1 when a revolution was completed by this packet (out4 then holds *m_out points, at most cap), 0 if not, < 0 on error
int lsh_assembler_add_packet(void* av, const float* pts4, int n, const float* T_fixed_base16, int64_t stamp_ns, float* out4, int cap,
                             int* m_out, int64_t* stamp_out) {
  try {
    VelodyneAssembler* a = static_cast<VelodyneAssembler*>(av);
    VelodyneAssembler::Matrix4 T;
    std::memcpy(T.data(), T_fixed_base16, 16 * sizeof(float));
    DataPoints in = DataPoints::viewOfArrays(pts4, NULL, (size_t)n), rev;
    Time st = 0;
    if (!a->addPacket(in, T, (Time)stamp_ns, &rev, &st)) return 0;
    const int m = (int)rev.getNbPoints();
    if (m > cap) return LS_ERR_ARG;
    std::memcpy(out4, static_cast<const DataPoints&>(rev).features.data(), sizeof(float) * 4 * (size_t)m);
    *m_out = m;
    if (stamp_out) *stamp_out = (int64_t)st;
    return 1;
  } catch (const std::exception&) {
    return LS_ERR_STATE;
  }
}

// ---- laser_slam::OccupancyMap (include/laser_slam/occupancy_map.hpp) on an estimator, for the tests.  Destroy it before
// the estimator.  prm: resolution, hit, miss, clamp min, clamp max, occupancy threshold, max range, treat unknown as
// occupied (0 or 1).
struct OccupancyHandle {
  std::unique_ptr<OccupancyMap> map;
  std::string err;
  OccupancyMap::ProjectedMap projected;  // the last getProjectedMap, held for lsh_occupancy_projected_cells
};

void* lsh_occupancy_create(void* hv, const double* prm, int initial_capacity_bricks, char* err, int errlen) {
  try {
    OccupancyMapParams p;
    p.resolution = prm[0];
    p.probability_hit = prm[1];
    p.probability_miss = prm[2];
    p.clamping_thres_min = prm[3];
    p.clamping_thres_max = prm[4];
    p.occupancy_thres = prm[5];
    p.sensor_max_range = prm[6];
    p.initial_capacity_bricks = initial_capacity_bricks;
    p.treat_unknown_as_occupied = prm[7] != 0.0;
    OccupancyHandle* h = new OccupancyHandle();
    h->map.reset(new OccupancyMap(p, *static_cast<Handle*>(hv)->est));
    return h;
  } catch (const std::exception& e) {
    if (err && errlen > 0) std::strncpy(err, e.what(), (size_t)errlen - 1), err[errlen - 1] = 0;
    return nullptr;
  }
}
void lsh_occupancy_destroy(void* ov) { delete static_cast<OccupancyHandle*>(ov); }
const char* lsh_occupancy_last_error(void* ov) { return static_cast<OccupancyHandle*>(ov)->err.c_str(); }

// insertLaserTracks; returns the scans inserted
int lsh_occupancy_insert_laser_tracks(void* ov) {
  OccupancyHandle* h = static_cast<OccupancyHandle*>(ov);
  try {
    return (int)h->map->insertLaserTracks();
  } catch (const std::exception& e) {
    h->err = e.what();
    return LS_ERR_STATE;
  }
}

// getVoxels (keys / log_odds may be NULL: count only); returns the number of voxels, written when it is <= cap
int64_t lsh_occupancy_voxels(void* ov, int which, uint64_t* keys, float* log_odds, int64_t cap) {
  OccupancyHandle* h = static_cast<OccupancyHandle*>(ov);
  try {
    std::vector<uint64_t> k;
    std::vector<float> v;
    h->map->getVoxels(which, &k, &v);
    const int64_t n = (int64_t)k.size();
    if (keys && log_odds && n <= cap) {
      std::memcpy(keys, k.data(), sizeof(uint64_t) * (size_t)n);
      std::memcpy(log_odds, v.data(), sizeof(float) * (size_t)n);
    }
    return n;
  } catch (const std::exception& e) {
    h->err = e.what();
    return LS_ERR_STATE;
  }
}

// getOccupiedCloud; returns its number of points, written when it is <= cap
int lsh_occupancy_occupied_cloud(void* ov, float* out4, int cap) {
  OccupancyHandle* h = static_cast<OccupancyHandle*>(ov);
  try {
    DataPoints d;
    h->map->getOccupiedCloud(&d);
    const int n = (int)d.getNbPoints();
    if (out4 && n <= cap) std::memcpy(out4, static_cast<const DataPoints&>(d).features.data(), sizeof(float) * 4 * (size_t)n);
    return n;
  } catch (const std::exception& e) {
    h->err = e.what();
    return LS_ERR_STATE;
  }
}

// writeBinary; 0 on success, LS_ERR_ARG when the file cannot be written
int lsh_occupancy_write_binary(void* ov, const char* path) {
  OccupancyHandle* h = static_cast<OccupancyHandle*>(ov);
  try {
    return h->map->writeBinary(path) ? 0 : LS_ERR_ARG;
  } catch (const std::exception& e) {
    h->err = e.what();
    return LS_ERR_STATE;
  }
}

// readBinary; 0 on success, LS_ERR_ARG when it returns false
int lsh_occupancy_read_binary(void* ov, const char* path) {
  OccupancyHandle* h = static_cast<OccupancyHandle*>(ov);
  try {
    return h->map->readBinary(path) ? 0 : LS_ERR_ARG;
  } catch (const std::exception& e) {
    h->err = e.what();
    return LS_ERR_STATE;
  }
}

// write (.ot); 0 on success, LS_ERR_ARG when the file cannot be written
int lsh_occupancy_write_full(void* ov, const char* path) {
  OccupancyHandle* h = static_cast<OccupancyHandle*>(ov);
  try {
    return h->map->write(path) ? 0 : LS_ERR_ARG;
  } catch (const std::exception& e) {
    h->err = e.what();
    return LS_ERR_STATE;
  }
}

// read (.ot); 0 on success, LS_ERR_ARG when it returns false
int lsh_occupancy_read_full(void* ov, const char* path) {
  OccupancyHandle* h = static_cast<OccupancyHandle*>(ov);
  try {
    return h->map->read(path) ? 0 : LS_ERR_ARG;
  } catch (const std::exception& e) {
    h->err = e.what();
    return LS_ERR_STATE;
  }
}

// writeData: the payload's size (0: empty map; nothing copied when it exceeds cap) and node count; LS_ERR_STATE on error
int64_t lsh_occupancy_write_full_data(void* ov, uint8_t* out, int64_t cap, int64_t* nodes) {
  OccupancyHandle* h = static_cast<OccupancyHandle*>(ov);
  try {
    std::vector<uint8_t> payload;
    h->map->writeData(&payload, nodes);
    if ((int64_t)payload.size() <= cap && !payload.empty()) std::memcpy(out, payload.data(), payload.size());
    return (int64_t)payload.size();
  } catch (const std::exception& e) {
    h->err = e.what();
    return LS_ERR_STATE;
  }
}

// readData; 0 on success, LS_ERR_ARG when it returns false
int lsh_occupancy_read_full_data(void* ov, const uint8_t* payload, int64_t bytes, int64_t nodes, double resolution) {
  OccupancyHandle* h = static_cast<OccupancyHandle*>(ov);
  try {
    return h->map->readData(std::vector<uint8_t>(payload, payload + bytes), nodes, resolution) ? 0 : LS_ERR_ARG;
  } catch (const std::exception& e) {
    h->err = e.what();
    return LS_ERR_STATE;
  }
}

// getCellProbabilityPoint per point (single queries): status and probability; 0 or LS_ERR_STATE
int lsh_occupancy_cell_status(void* ov, const double* pts3, int n, int8_t* status, double* probability) {
  OccupancyHandle* h = static_cast<OccupancyHandle*>(ov);
  try {
    for (int i = 0; i < n; ++i) {
      const kindr::minimal::Position p{pts3[3 * i], pts3[3 * i + 1], pts3[3 * i + 2]};
      status[i] = (int8_t)h->map->getCellProbabilityPoint(p, &probability[i]);
      if (h->map->getCellStatusPoint(p) != static_cast<OccupancyMap::CellStatus>(status[i]))
        throw std::runtime_error("getCellStatusPoint and getCellProbabilityPoint disagree");
    }
    return 0;
  } catch (const std::exception& e) {
    h->err = e.what();
    return LS_ERR_STATE;
  }
}

// Line status per segment: single = 1 calls getLineStatus (stop_at_unknown 1, no box), getVisibility or
// getLineStatusBoundingBox (box3 set) once per segment; single = 0 the batched overload, which also gives first_keys.
int lsh_occupancy_line_status(void* ov, const double* s3, const double* e3, int n, const double* box3, int stop_at_unknown,
                              int single, int8_t* status, uint64_t* first_keys) {
  OccupancyHandle* h = static_cast<OccupancyHandle*>(ov);
  try {
    std::vector<kindr::minimal::Position> s(n), e(n);
    for (int i = 0; i < n; ++i)
      s[i] = {s3[3 * i], s3[3 * i + 1], s3[3 * i + 2]}, e[i] = {e3[3 * i], e3[3 * i + 1], e3[3 * i + 2]};
    const kindr::minimal::Position box = box3 ? kindr::minimal::Position{box3[0], box3[1], box3[2]} : kindr::minimal::Position{};
    if (single) {
      for (int i = 0; i < n; ++i) {
        OccupancyMap::CellStatus c;
        if (box3) c = h->map->getLineStatusBoundingBox(s[i], e[i], box);
        else if (stop_at_unknown) c = h->map->getLineStatus(s[i], e[i]);
        else c = h->map->getVisibility(s[i], e[i], false);
        status[i] = (int8_t)c;
      }
      return 0;
    }
    std::vector<OccupancyMap::CellStatus> st;
    std::vector<uint64_t> fk;
    h->map->getLineStatus(s, e, &st, stop_at_unknown != 0, box3 ? &box : NULL, &fk);
    for (int i = 0; i < n; ++i) status[i] = (int8_t)st[(size_t)i], first_keys[i] = fk[(size_t)i];
    return 0;
  } catch (const std::exception& e) {
    h->err = e.what();
    return LS_ERR_STATE;
  }
}

// castRay per ray (single = 1: the bool overload, results 1 for a hit and 0 otherwise) or castRays (single = 0: LS_RAY_*);
// ends3 as the C++ layer returns them (left at the input's values where it leaves *end alone).
int lsh_occupancy_cast_rays(void* ov, const double* o3, const double* d3, int n, int ignore_unknown, double max_range,
                            int single, int* results, double* ends3) {
  OccupancyHandle* h = static_cast<OccupancyHandle*>(ov);
  try {
    std::vector<kindr::minimal::Position> o(n), d(n), e;
    for (int i = 0; i < n; ++i)
      o[i] = {o3[3 * i], o3[3 * i + 1], o3[3 * i + 2]}, d[i] = {d3[3 * i], d3[3 * i + 1], d3[3 * i + 2]};
    if (single) {
      for (int i = 0; i < n; ++i) {
        kindr::minimal::Position end{ends3[3 * i], ends3[3 * i + 1], ends3[3 * i + 2]};
        results[i] = h->map->castRay(o[i], d[i], &end, ignore_unknown != 0, max_range) ? 1 : 0;
        for (int a = 0; a < 3; ++a) ends3[3 * i + a] = end[a];
      }
      return 0;
    }
    std::vector<int> r;
    h->map->castRays(o, d, &r, &e, ignore_unknown != 0, max_range);
    for (int i = 0; i < n; ++i) {
      results[i] = r[(size_t)i];
      for (int a = 0; a < 3; ++a) ends3[3 * i + a] = e[(size_t)i][a];
    }
    return 0;
  } catch (const std::exception& e) {
    h->err = e.what();
    return LS_ERR_STATE;
  }
}

// getOccupiedLeafCloud; returns its number of points, written when it is <= cap
int lsh_occupancy_occupied_leaf_cloud(void* ov, float* out4, int cap) {
  OccupancyHandle* h = static_cast<OccupancyHandle*>(ov);
  try {
    DataPoints d;
    h->map->getOccupiedLeafCloud(&d);
    const int n = (int)d.getNbPoints();
    if (out4 && n <= cap) std::memcpy(out4, static_cast<const DataPoints&>(d).features.data(), sizeof(float) * 4 * (size_t)n);
    return n;
  } catch (const std::exception& e) {
    h->err = e.what();
    return LS_ERR_STATE;
  }
}

// Edits.  single = 1: setFree / setOccupied once per box, else one setBoxes call; stats (voxels_set, new_known, known voxels)
// of the batched call.  0 or LS_ERR_STATE.
int lsh_occupancy_set_boxes(void* ov, const double* c3, const double* s3, const int8_t* occupied, int n, int single,
                            int64_t* stats3) {
  OccupancyHandle* h = static_cast<OccupancyHandle*>(ov);
  try {
    std::vector<kindr::minimal::Position> c(n), s(n);
    std::vector<bool> o(n);
    for (int i = 0; i < n; ++i)
      c[i] = {c3[3 * i], c3[3 * i + 1], c3[3 * i + 2]}, s[i] = {s3[3 * i], s3[3 * i + 1], s3[3 * i + 2]}, o[i] = occupied[i] != 0;
    if (single) {
      for (int i = 0; i < n; ++i) o[i] ? h->map->setOccupied(c[i], s[i]) : h->map->setFree(c[i], s[i]);
      return 0;
    }
    ls_occupancy_edit_stats st;
    h->map->setBoxes(c, s, o, &st);
    stats3[0] = st.voxels_set, stats3[1] = st.new_known, stats3[2] = st.known_voxels;
    return 0;
  } catch (const std::exception& e) {
    h->err = e.what();
    return LS_ERR_STATE;
  }
}

int lsh_occupancy_reset(void* ov) {
  OccupancyHandle* h = static_cast<OccupancyHandle*>(ov);
  try {
    h->map->resetMap();
    return 0;
  } catch (const std::exception& e) {
    h->err = e.what();
    return LS_ERR_STATE;
  }
}

// getOccupiedPointcloudInBoundingBox; returns its number of points, written when it is <= cap
int lsh_occupancy_box_cloud(void* ov, const double* c3, const double* s3, float* out4, int cap) {
  OccupancyHandle* h = static_cast<OccupancyHandle*>(ov);
  try {
    DataPoints d;
    h->map->getOccupiedPointcloudInBoundingBox({c3[0], c3[1], c3[2]}, {s3[0], s3[1], s3[2]}, &d);
    const int n = (int)d.getNbPoints();
    if (out4 && n <= cap) std::memcpy(out4, static_cast<const DataPoints&>(d).features.data(), sizeof(float) * 4 * (size_t)n);
    return n;
  } catch (const std::exception& e) {
    h->err = e.what();
    return LS_ERR_STATE;
  }
}

// getMapBounds, getMapSize and getMapCenter: out12 = min, max, size, centre
int lsh_occupancy_bounds(void* ov, double* out12) {
  OccupancyHandle* h = static_cast<OccupancyHandle*>(ov);
  try {
    kindr::minimal::Position lo, hi;
    h->map->getMapBounds(&lo, &hi);
    const kindr::minimal::Position size = h->map->getMapSize(), centre = h->map->getMapCenter();
    for (int a = 0; a < 3; ++a) out12[a] = lo[a], out12[3 + a] = hi[a], out12[6 + a] = size[a], out12[9 + a] = centre[a];
    return 0;
  } catch (const std::exception& e) {
    h->err = e.what();
    return LS_ERR_STATE;
  }
}
// Change detection.  enableChangeDetection (enable >= 0) or resetChangeDetection (enable < 0); returns
// isChangeDetectionEnabled, or LS_ERR_STATE.
int lsh_occupancy_track_changes(void* ov, int enable) {
  OccupancyHandle* h = static_cast<OccupancyHandle*>(ov);
  try {
    if (enable < 0) h->map->resetChangeDetection();
    else h->map->enableChangeDetection(enable != 0);
    return h->map->isChangeDetectionEnabled() ? 1 : 0;
  } catch (const std::exception& e) {
    h->err = e.what();
    return LS_ERR_STATE;
  }
}

// numChangesDetected, then (when keys is not NULL and it is <= cap) getChangedKeys; returns the count or LS_ERR_STATE
int64_t lsh_occupancy_changed_keys(void* ov, uint64_t* keys, int8_t* status, int8_t* previous, int64_t cap) {
  OccupancyHandle* h = static_cast<OccupancyHandle*>(ov);
  try {
    const int64_t n = (int64_t)h->map->numChangesDetected();
    if (!keys || n > cap) return n;
    std::vector<uint64_t> k;
    std::vector<int8_t> s, p;
    h->map->getChangedKeys(&k, &s, &p);
    if ((int64_t)k.size() != n) throw std::runtime_error("numChangesDetected and getChangedKeys disagree");
    for (int64_t i = 0; i < n; ++i) keys[i] = k[(size_t)i], status[i] = s[(size_t)i], previous[i] = p[(size_t)i];
    return n;
  } catch (const std::exception& e) {
    h->err = e.what();
    return LS_ERR_STATE;
  }
}

// getChangedPoints (which resets); returns its number of points, the first min(n, cap) written: centres and occupied
int64_t lsh_occupancy_changed_points(void* ov, double* pts3, uint8_t* occupied, int64_t cap) {
  OccupancyHandle* h = static_cast<OccupancyHandle*>(ov);
  try {
    std::vector<kindr::minimal::Position> p;
    std::vector<bool> s;
    h->map->getChangedPoints(&p, &s);
    const int64_t n = (int64_t)p.size();
    for (int64_t i = 0; i < n && i < cap; ++i) {
      for (int a = 0; a < 3; ++a) pts3[3 * i + a] = p[(size_t)i][a];
      occupied[i] = s[(size_t)i] ? 1 : 0;
    }
    return n;
  } catch (const std::exception& e) {
    h->err = e.what();
    return LS_ERR_STATE;
  }
}

// getAllFreeBoxes (occupied = 0) or getAllOccupiedBoxes, of the region when min3 is not NULL; returns the number of boxes,
// the first min(n, cap) written: centres and edges.  LS_ERR_STATE on an error
int64_t lsh_occupancy_boxes(void* ov, int occupied, const double* min3, const double* max3, double* centres3, double* edges,
                            int64_t cap) {
  OccupancyHandle* h = static_cast<OccupancyHandle*>(ov);
  try {
    if (!min3 != !max3) throw std::invalid_argument("a region needs both corners");
    OccupancyMap::BoxVector b;
    if (min3) {
      const kindr::minimal::Position lo{min3[0], min3[1], min3[2]}, hi{max3[0], max3[1], max3[2]};
      occupied ? h->map->getAllOccupiedBoxes(lo, hi, &b) : h->map->getAllFreeBoxes(lo, hi, &b);
    } else {
      occupied ? h->map->getAllOccupiedBoxes(&b) : h->map->getAllFreeBoxes(&b);
    }
    const int64_t n = (int64_t)b.size();
    for (int64_t i = 0; i < n && i < cap; ++i) {
      for (int a = 0; a < 3; ++a) centres3[3 * i + a] = b[(size_t)i].first[a];
      edges[i] = b[(size_t)i].second;
    }
    return n;
  } catch (const std::exception& e) {
    h->err = e.what();
    return LS_ERR_STATE;
  }
}

// generateMarkerArray; returns the number of cubes, the first min(n, cap) written in list order (occupied depths 0..16,
// then free depths 0..16): centres, colours (occupied cubes only, rgba4 holds cap of them), and per list its size and
// length (sizes34, counts34).  LS_ERR_STATE on an error
int64_t lsh_occupancy_marker_array(void* ov, double min_z, double max_z, double color_factor, double* centres3, float* rgba4,
                                   double* sizes34, int64_t* counts34, int64_t cap) {
  OccupancyHandle* h = static_cast<OccupancyHandle*>(ov);
  try {
    std::vector<OccupancyMap::CubeList> lists[2];
    h->map->generateMarkerArray(min_z, max_z, color_factor, &lists[0], &lists[1]);
    int64_t n = 0, k = 0;
    for (int part = 0; part < 2; ++part)
      for (size_t d = 0; d < lists[part].size(); ++d, ++k) {
        const OccupancyMap::CubeList& l = lists[part][d];
        sizes34[k] = l.size, counts34[k] = (int64_t)l.points.size();
        for (size_t i = 0; i < l.points.size(); ++i, ++n) {
          if (n >= cap) continue;
          for (int a = 0; a < 3; ++a) centres3[3 * n + a] = l.points[i][a];
          if (part == 0)
            for (int a = 0; a < 4; ++a) rgba4[4 * n + a] = l.colors[i][(size_t)a];
        }
      }
    return n;
  } catch (const std::exception& e) {
    h->err = e.what();
    return LS_ERR_STATE;
  }
}

// getProjectedMap of the band (min_z, max_z) padded to min_x_size x min_y_size, kept in the handle; returns width * height
// and geo5 = {width, height, resolution, origin x, origin y}.  LS_ERR_STATE on an error
int64_t lsh_occupancy_projected_map(void* ov, double min_z, double max_z, double min_x_size, double min_y_size, double* geo5) {
  OccupancyHandle* h = static_cast<OccupancyHandle*>(ov);
  try {
    OccupancyMap::ProjectedMapParams p;
    p.occupancy_min_z = min_z, p.occupancy_max_z = max_z, p.min_x_size = min_x_size, p.min_y_size = min_y_size;
    h->map->getProjectedMap(p, &h->projected);
    const OccupancyMap::ProjectedMap& m = h->projected;
    geo5[0] = m.width, geo5[1] = m.height, geo5[2] = m.resolution, geo5[3] = m.origin_x, geo5[4] = m.origin_y;
    return (int64_t)m.data.size();
  } catch (const std::exception& e) {
    h->err = e.what();
    return LS_ERR_STATE;
  }
}

// The cells of the last lsh_occupancy_projected_map, written when they fit in cap; returns their number
int64_t lsh_occupancy_projected_cells(void* ov, int8_t* data, int64_t cap) {
  const OccupancyHandle* h = static_cast<const OccupancyHandle*>(ov);
  const int64_t n = (int64_t)h->projected.data.size();
  if (n <= cap) std::copy(h->projected.data.begin(), h->projected.data.end(), data);
  return n;
}

// saveProjectedMap: 1 written, 0 a file could not be written, LS_ERR_STATE on an error
int lsh_occupancy_save_projected_map(void* ov, const char* stem, double min_z, double max_z, double min_x_size,
                                     double min_y_size) {
  OccupancyHandle* h = static_cast<OccupancyHandle*>(ov);
  try {
    OccupancyMap::ProjectedMapParams p;
    p.occupancy_min_z = min_z, p.occupancy_max_z = max_z, p.min_x_size = min_x_size, p.min_y_size = min_y_size;
    return h->map->saveProjectedMap(stem, p) ? 1 : 0;
  } catch (const std::exception& e) {
    h->err = e.what();
    return LS_ERR_STATE;
  }
}

// Box status.  single = 1: getCellStatusBoundingBox once per box, else the batched overload.  0 or LS_ERR_STATE
int lsh_occupancy_box_status(void* ov, const double* c3, const double* s3, int n, int single, int8_t* status) {
  OccupancyHandle* h = static_cast<OccupancyHandle*>(ov);
  try {
    std::vector<kindr::minimal::Position> c(n), s(n);
    for (int i = 0; i < n; ++i) c[i] = {c3[3 * i], c3[3 * i + 1], c3[3 * i + 2]}, s[i] = {s3[3 * i], s3[3 * i + 1], s3[3 * i + 2]};
    if (single) {
      for (int i = 0; i < n; ++i) status[i] = (int8_t)h->map->getCellStatusBoundingBox(c[i], s[i]);
      return 0;
    }
    std::vector<OccupancyMap::CellStatus> st;
    h->map->getCellStatusBoundingBox(c, s, &st);
    for (int i = 0; i < n; ++i) status[i] = (int8_t)st[(size_t)i];
    return 0;
  } catch (const std::exception& e) {
    h->err = e.what();
    return LS_ERR_STATE;
  }
}

// Robot collision after setRobotSize(robot3) (getRobotSize must return it).  single = 1: checkPathForCollisionsWithRobot
// per path (first[p] its collision_index, -1 when false; a path of one pose also through checkCollisionWithRobot, which
// must agree); single = 0: checkPathsForCollisionsWithRobot.  0 or LS_ERR_STATE
int lsh_occupancy_check_paths(void* ov, const double* p3, const int64_t* offsets, int n_paths, const double* robot3,
                              int single, int64_t* first) {
  OccupancyHandle* h = static_cast<OccupancyHandle*>(ov);
  try {
    const kindr::minimal::Position r{robot3[0], robot3[1], robot3[2]};
    h->map->setRobotSize(r);
    const kindr::minimal::Position got = h->map->getRobotSize();
    if (!(got[0] == r[0] && got[1] == r[1] && got[2] == r[2])) throw std::runtime_error("getRobotSize differs");
    std::vector<std::vector<kindr::minimal::Position> > paths((size_t)n_paths);
    for (int p = 0; p < n_paths; ++p)
      for (int64_t i = offsets[p]; i < offsets[p + 1]; ++i) paths[(size_t)p].push_back({p3[3 * i], p3[3 * i + 1], p3[3 * i + 2]});
    if (single) {
      for (int p = 0; p < n_paths; ++p) {
        size_t idx = 0;
        const bool hit = h->map->checkPathForCollisionsWithRobot(paths[(size_t)p], &idx);
        first[p] = hit ? (int64_t)idx : -1;
        if (paths[(size_t)p].size() == 1 && h->map->checkCollisionWithRobot(paths[(size_t)p][0]) != hit)
          throw std::runtime_error("checkCollisionWithRobot and checkPathForCollisionsWithRobot disagree");
      }
      return 0;
    }
    std::vector<int64_t> f;
    h->map->checkPathsForCollisionsWithRobot(paths, &f);
    for (int p = 0; p < n_paths; ++p) first[p] = f[(size_t)p];
    return 0;
  } catch (const std::exception& e) {
    h->err = e.what();
    return LS_ERR_STATE;
  }
}

// ---- laser_slam::DistanceMap (include/laser_slam/distance_map.hpp) on an OccupancyMap handle, for the tests.  Destroy it
// before the occupancy map.  box6: bbx_min, bbx_max.
struct DistanceHandle {
  std::unique_ptr<DistanceMap> map;
  std::string err;
};

void* lsh_distance_create(void* ov, float maxdist, const double* box6, int unknown_occ, char* err, int errlen) {
  try {
    DistanceHandle* h = new DistanceHandle();
    h->map.reset(new DistanceMap(maxdist, *static_cast<OccupancyHandle*>(ov)->map, {box6[0], box6[1], box6[2]},
                                 {box6[3], box6[4], box6[5]}, unknown_occ != 0));
    return h;
  } catch (const std::exception& e) {
    if (err && errlen > 0) std::strncpy(err, e.what(), (size_t)errlen - 1), err[errlen - 1] = 0;
    return nullptr;
  }
}
void lsh_distance_destroy(void* dv) { delete static_cast<DistanceHandle*>(dv); }
const char* lsh_distance_last_error(void* dv) { return static_cast<DistanceHandle*>(dv)->err.c_str(); }

// update; out2: getMaxDist, getSquaredMaxDistCells.  0 or LS_ERR_STATE
int lsh_distance_update(void* dv, double* out2) {
  DistanceHandle* h = static_cast<DistanceHandle*>(dv);
  try {
    h->map->update();
    out2[0] = h->map->getMaxDist(), out2[1] = h->map->getSquaredMaxDistCells();
    return 0;
  } catch (const std::exception& e) {
    h->err = e.what();
    return LS_ERR_STATE;
  }
}

// single = 1: getDistance, getDistanceAndClosestObstacle and getSquaredDistanceInCells once per point (the two distances
// must agree); single = 0: the batched getDistances.  closest3 as the C++ layer returns it.  0 or LS_ERR_STATE
int lsh_distance_query(void* dv, const double* pts3, int n, int single, float* dist, int* sq, double* closest3) {
  DistanceHandle* h = static_cast<DistanceHandle*>(dv);
  try {
    std::vector<kindr::minimal::Position> p(n);
    for (int i = 0; i < n; ++i) p[i] = {pts3[3 * i], pts3[3 * i + 1], pts3[3 * i + 2]};
    if (single) {
      for (int i = 0; i < n; ++i) {
        kindr::minimal::Position c;
        h->map->getDistanceAndClosestObstacle(p[i], dist[i], c);
        const float d = h->map->getDistance(p[i]);
        if (!(d == dist[i])) throw std::runtime_error("getDistance and getDistanceAndClosestObstacle disagree");
        sq[i] = h->map->getSquaredDistanceInCells(p[i]);
        for (int a = 0; a < 3; ++a) closest3[3 * i + a] = c[a];
      }
      return 0;
    }
    std::vector<float> d;
    std::vector<int> s;
    std::vector<kindr::minimal::Position> c;
    h->map->getDistances(p, &d, &s, &c);
    for (int i = 0; i < n; ++i) {
      dist[i] = d[(size_t)i], sq[i] = s[(size_t)i];
      for (int a = 0; a < 3; ++a) closest3[3 * i + a] = c[(size_t)i][a];
    }
    return 0;
  } catch (const std::exception& e) {
    h->err = e.what();
    return LS_ERR_STATE;
  }
}
}  // extern "C"
