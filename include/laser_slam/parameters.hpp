// Same fields as reference laser_slam/include/laser_slam/parameters.hpp:8-34
// (Eigen::Matrix<double,6,1> -> std::array<double,6>; Eigen is absent here).
#ifndef LASER_SLAM_PARAMETERS_HPP_
#define LASER_SLAM_PARAMETERS_HPP_

#include <array>
#include <string>

namespace laser_slam {

struct LaserTrackParams {
  std::array<double, 6> odometry_noise_model{{0.005, 0.005, 0.005, 0.0015, 0.0015, 0.0015}};
  std::array<double, 6> icp_noise_model{{0.005, 0.005, 0.005, 0.0015, 0.0015, 0.0015}};
  bool add_m_estimator_on_odom = false;
  bool add_m_estimator_on_icp = true;

  std::string icp_configuration_file;   // libpointmatcher chain YAML; unreadable -> icp_default.yaml values
  std::string icp_input_filters_file;   // DataPointsFilters YAML run on every scan on the device; without a normal filter
                                        // in it (or without the file) scans must carry normals
  bool use_icp_factors = true;
  bool use_odom_factors = true;
  int nscan_in_sub_map = 4;
  bool save_icp_results = false;

  bool force_priors = false;

  int cuda_device = 0;                  // (new) device the track's context lives on
};

struct EstimatorParams {
  std::array<double, 6> loop_closure_noise_model{{0.005, 0.005, 0.005, 0.0015, 0.0015, 0.0015}};
  bool add_m_estimator_on_loop_closures = false;

  bool do_icp_step_on_loop_closures = false;
  int loop_closures_sub_maps_radius = 3;

  LaserTrackParams laser_track_params;
};

}  // namespace laser_slam

#endif  // LASER_SLAM_PARAMETERS_HPP_
