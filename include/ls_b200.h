/* ls_b200.h -- C ABI of the H100-native laser_slam hot path (libls_b200.so).
 *
 * Plain C, plain pointers and sizes; no torch / CUDA types cross this boundary.  Each entry point
 * names the reference interface it replaces (paths relative to the reference repo root).
 *
 * Conventions
 *   - Clouds use the libpointmatcher DataPoints memory layout the reference passes around
 *     (laser_slam/include/laser_slam/common.hpp:14-15,113-120): `features` is a column-major
 *     4xN float matrix, i.e. N consecutive {x, y, z, 1} quadruples; a `normals` descriptor is read
 *     through (pointer, stride-in-floats) so a DxN descriptor block can be passed without copying.
 *   - 4x4 transforms are 16 floats, column-major (PointMatcher::TransformationParameters::data()).
 *   - Host buffers are owned by the caller and only read/written during the call.  Device memory
 *     is owned by the library (ls_ctx / ls_map) and freed by the matching *_destroy.
 *   - Return value: 0 ok; > 0 algorithmic condition (LS_ERR_CONVERGENCE maps to
 *     PointMatcher::ConvergenceError, which laser_slam/src/laser_track.cpp:495-502 catches and
 *     turns into "keep the initial guess"; laser_slam/src/incremental_estimator.cpp:108 lets it
 *     propagate); < 0 argument / CUDA / resource error.  There is no CPU fallback: without a usable
 *     CUDA device ls_b200_init fails with LS_ERR_CUDA.
 *   - Calls on one ls_ctx are serialised by the caller (the reference holds
 *     full_laser_track_mutex_ / full_class_mutex_ around them); distinct contexts are independent
 *     (own stream, own buffers).  Calls are synchronous: results are on the host at return.
 */
#ifndef LS_B200_H_
#define LS_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LS_OK 0
#define LS_ERR_CONVERGENCE 1 /* no point to minimise / NaN  -> PointMatcher::ConvergenceError */
#define LS_ERR_ARG (-1)
#define LS_ERR_CUDA (-2)
#define LS_ERR_NOMEM (-3)
#define LS_ERR_STATE (-4)
#define LS_ERR_NCCL (-5)

typedef struct ls_ctx ls_ctx;
typedef struct ls_map ls_map;

/* ICP chain parameters = the subset of laser_slam/configurations/icp_default.yaml the path uses. */
typedef struct ls_icp_params {
  int max_iterations;   /* CounterTransformationChecker.maxIterationCount      yaml:22-23 */
  float trim_ratio;     /* TrimmedDistOutlierFilter.ratio                      yaml:14-16 */
  int use_differential; /* DifferentialTransformationChecker present           yaml:24-27 */
  float min_diff_rot;   /* minDiffRotErr [rad] */
  float min_diff_trans; /* minDiffTransErr [m] */
  int smooth_length;    /* smoothLength (<= 15) */
  /* spatial-hash tuning (no reference counterpart; results do not depend on these) */
  float cell_size;      /* level-0 cell edge [m]; <= 0 -> 1.0 */
  int leaf_split;       /* subdivide cells holding more points; <= 0 -> 32 (min 16) */
  int max_cells;        /* cap on level-0 cells; <= 0 -> 4194304 */
  /* The DataPointsFilters sections of the chain (icp_default.yaml:1-7).  ls_icp_params_from_yaml reports them here; the
   * registration entry points do NOT apply them -- they take clouds as given, normals included -- the caller does, with
   * ls_keep_point / ls_estimate_normals (what PointMatcher::ICP::compute in include/laser_slam_compat/compat.hpp does). */
  float reading_sampling_prob;    /* readingDataPointsFilters: RandomSamplingDataPointsFilter.prob; 1 = absent */
  int reference_normals_knn;      /* referenceDataPointsFilters: (Sampling)SurfaceNormalDataPointsFilter.knn; 0 = absent */
  float reference_sampling_ratio; /* its ratio (SamplingSurfaceNormal keeps that fraction); 1 = absent */
  int unapplied_modules;          /* YAML modules present that the registration itself does not run (the filter sections above) */
} ls_icp_params;

typedef struct ls_icp_stats {
  int iterations;       /* ICP iterations executed */
  int converged;        /* stopped by the differential checker */
  int max_iter_reached; /* stopped by the counter (flag, not an error) */
  int last_kept;        /* matches with weight 1 in the last iteration */
  float last_limit;     /* trimmed squared-distance limit of the last iteration */
  float used_ratio;     /* last_kept / n (libpointmatcher pointUsedRatio) */
  float device_ms;      /* CUDA-event time of the device work of this call */
  float build_ms;       /* of which: sub-map assembly + spatial-hash build */
  int grid_cells;       /* level-0 cells */
  int grid_tables;      /* fine (8x8x8) tables allocated */
  int grid_overflow;    /* 1 if a table pool overflowed (slower, still exact) */
  float icp_ms;         /* CUDA-event duration of the persistent ICP kernel launch (shared by a batch) */
} ls_icp_stats;

/* ---- context ------------------------------------------------------------------------------- */
int ls_b200_init(int device, ls_ctx** out);
void ls_b200_destroy(ls_ctx* ctx);
const char* ls_b200_last_error(const ls_ctx* ctx); /* text of the last failure on this context */
int ls_b200_version(void);
/* Cap the number of CTAs the persistent ICP kernel of this context may occupy (0 = all that can be co-resident, the
 * default).  Two contexts that each take half of the device run their cooperative launches side by side, so the map build
 * and host-side staging of one overlap the ICP iterations of the other (bench.py drives two such contexts). */
int ls_b200_set_icp_cta_budget(ls_ctx* ctx, int ctas);
/* The budget in force.  A launch of B problems gives each max(1, budget / B) CTAs (fewer for a small reading), so it
 * stays within the budget unless B exceeds it: then every problem still gets one CTA and the launch uses B. */
int ls_b200_icp_cta_budget(const ls_ctx* ctx);
/* Number of this library's kernel launches issued on the context so far (bench "gpu_launches"). */
uint64_t ls_b200_launch_count(const ls_ctx* ctx);

/* icp_.setDefault()-like defaults, but with the values of icp_default.yaml:9-27
 * (replaces PointMatcher::ICP::loadFromYaml at laser_slam/src/laser_track.cpp:14-21). */
void ls_icp_default_params(ls_icp_params* p);
/* Parse the keys of icp_default.yaml this path honours out of a YAML text; unsupported matcher / minimiser / outlier
 * filter names return LS_ERR_ARG; reading / reference DataPointsFilters are reported in the params (see the struct:
 * `unapplied_modules` counts them) because they run upstream of the registration; inspector / logger are ignored. */
int ls_icp_params_from_yaml(const char* yaml_text, ls_icp_params* p);

/* Deterministic stand-in for RandomSamplingDataPointsFilter's `rand() / RAND_MAX < prob`
 * (laser_slam/configurations/icp_default.yaml:1-3; libpointmatcher draws from the process-global libc generator, which is
 * not reproducible): point `index` of a cloud is kept iff hash32(index, salt) < prob * 2^32, a counter-based rule that
 * host, device and oracle evaluate identically.  Returns 1 (keep) or 0. */
int ls_keep_point(uint32_t index, uint32_t salt, float prob);

/* ---- one-shot registration ----------------------------------------------------------------------
 * Replaces PointMatcher::ICP::compute(reading, reference, T0) at
 *   laser_slam/src/laser_track.cpp:496              (scan -> sub-map)
 *   laser_slam/src/incremental_estimator.cpp:108    (sub-map b -> sub-map a on loop closure)
 * reading: 4xN features; reference: 4xM features + normals.  T_out = T_ref<-reading.
 * On LS_ERR_CONVERGENCE T_out == T0.  opt_ids / opt_d2 (may be NULL, length n) receive the
 * correspondence indices (into the reference, -1 = none) and squared distances of the LAST
 * iteration; opt_T_iter_hist (may be NULL, max_iterations*16 floats) the accumulated T_iter after
 * every iteration (centred frame). */
int ls_icp_register(ls_ctx* ctx, const ls_icp_params* prm, const float* reading4, int n,
                    const float* ref4, const float* ref_normals, int normals_stride, int m,
                    const float T0[16], float T_out[16], ls_icp_stats* stats, int32_t* opt_ids,
                    float* opt_d2, float* opt_T_iter_hist);

/* KDTreeMatcher-level entry (icp_default.yaml:9-12): nearest reference point of T0*reading for
 * every reading point, with the reference centred exactly as ICP::compute does.  ids index the
 * reference as given; d2 are squared float32 distances. */
int ls_nn_query(ls_ctx* ctx, const ls_icp_params* prm, const float* reading4, int n, const float* ref4,
                int m, const float T0[16], int32_t* ids, float* d2);

/* RigidTransformation::compute (laser_slam/src/laser_track.cpp:265,485,508,511,630,643):
 * out = T * features, normals rotated by the 3x3 block.  normals/out_normals may be NULL. */
int ls_transform_cloud(ls_ctx* ctx, const float T[16], const float* in4, const float* normals,
                       int normals_stride, int n, float* out4, float* out_normals3);
/* RigidTransformation::checkParameters / correctParameters as used by
 * correctTransformationMatrix (laser_slam/include/laser_slam/common.hpp:136-149).  Host-side. */
int ls_check_rigid(const float T[16]);
void ls_correct_rigid(const float T_in[16], float T_out[16]);

/* ---- device-resident rolling map ------------------------------------------------------------------
 * Replaces LaserTrack::laser_scans_ + the per-scan copy/transform/concatenate loop of
 * LaserTrack::localScanToSubMap (laser_slam/src/laser_track.cpp:466-486) and
 * LaserTrack::buildSubMapAroundTime (laser_track.cpp:602-651): scans are uploaded once, kept in
 * their own sensor frame, and sub-maps are assembled on the device. */
int ls_map_create(ls_ctx* ctx, int capacity_scans, int max_pts_per_scan, ls_map** out);
void ls_map_destroy(ls_map* map);
/* Upload one scan; returns its id through *scan_id (ids grow monotonically; the scan stays
 * addressable until `capacity_scans` newer scans have been pushed). */
int ls_map_push_scan(ls_map* map, const float* features4, const float* normals, int normals_stride, int n,
                     uint64_t* scan_id);
/* The same, enqueued on the map's own upload stream; returns at once.  The host buffers must stay valid (pinned
 * memory, or the copies are synchronous after all) until ls_map_sync() or until a registration that uses the scan
 * has returned.  Registrations wait for exactly the uploads they depend on, so the next scan can go up while the
 * current one is being registered (the reference copies every scan twice on the host before its ICP starts,
 * laser_track.cpp:143,197).  3 <= normals_stride <= 8. */
int ls_map_push_scan_async(ls_map* map, const float* features4, const float* normals, int normals_stride, int n,
                           uint64_t* scan_id);
/* 1 if `p` points into page-locked (pinned) host memory known to the CUDA driver, 0 if not, < 0 on error.  The host
 * layer uses it to pick ls_map_push_scan_async (no staging copy) for DataPoints whose storage is pinned. */
int ls_host_is_pinned(const void* p);
int ls_map_sync(ls_map* map); /* wait for every asynchronous upload of this map */
int ls_map_scan_size(const ls_map* map, uint64_t scan_id); /* points, or <0 if evicted/unknown */

/* Surface normals on the device (SURVEY.md §8 row f1): replaces the SurfaceNormal / SamplingSurfaceNormal
 * DataPointsFilters the reference applies to every input scan and to the sub-map
 * (laser_slam/configurations/icp_default.yaml:5-7, laser_slam/src/laser_track.cpp:27,146).  For every point: exact
 * `knn` nearest neighbours (self included), covariance, eigenvector of the smallest eigenvalue, flipped towards the
 * sensor (origin of the scan frame).  Points with fewer than 3 neighbours get a zero normal.  3 <= knn <= 16.
 * Unlike the reference's filter this one is deterministic (no rand()-based sub-sampling). */
int ls_estimate_normals(ls_ctx* ctx, const float* features4, int n, int knn, float* out_normals3);
/* ls_map_push_scan for clouds that arrive without normals: they are estimated on the device into the slot. */
int ls_map_push_scan_estimate_normals(ls_map* map, const float* features4, int n, int knn, uint64_t* scan_id);

/* Scan -> sub-map registration on resident data.  The reference is the concatenation, in order,
 * of scans part_ids[0..n_parts) each transformed by T_parts[16*p..] (float32, already passed
 * through correctTransformationMatrix by the caller; an exact identity matrix copies the scan
 * verbatim as laser_track.cpp:476 does).  Reading = scan reading_id, untransformed.
 * Correspondence ids index that concatenation. */
int ls_icp_register_submap(ls_ctx* ctx, const ls_icp_params* prm, const ls_map* map, uint64_t reading_id,
                           int n_parts, const uint64_t* part_ids, const float* T_parts, const float T0[16],
                           float T_out[16], ls_icp_stats* stats, int32_t* opt_ids, float* opt_d2,
                           float* opt_T_iter_hist);

/* `batch` independent scan -> sub-map registrations in ONE cooperative launch (several LaserTracks hosted on one
 * GPU: the reference's n_laser_slam_workers tracks, laser_slam/src/incremental_estimator.cpp:22-26).  Problem b
 * uses reading_ids[b], its n_parts[b] parts follow each other in part_ids / T_parts (16 floats per part),
 * T0s / T_outs hold 16 floats per problem, statuses[b] is LS_OK or LS_ERR_CONVERGENCE (then T_out == T0).
 * Results are bit-identical to separate ls_icp_register_submap calls.  1 <= batch <= 160.  A problem whose reading or
 * sub-map is empty is left out of the launch and gets LS_ERR_CONVERGENCE, T_out == T0 and zeroed stats, as its single
 * call would; the other problems run unchanged.  If every problem is empty nothing is launched. */
int ls_icp_register_submap_batch(ls_ctx* ctx, const ls_icp_params* prm, const ls_map* map, int batch,
                                 const uint64_t* reading_ids, const int* n_parts, const uint64_t* part_ids,
                                 const float* T_parts, const float* T0s, float* T_outs, ls_icp_stats* stats,
                                 int* statuses);
/* The same in two halves.  begin() stages every problem and launches; end() waits and fetches the results (same
 * T_outs / stats / statuses as above).  In between the host is free -- typically to post the next scans with
 * ls_map_push_scan_async -- but every other call that needs the context's workspaces returns LS_ERR_STATE. */
int ls_icp_register_submap_batch_begin(ls_ctx* ctx, const ls_icp_params* prm, const ls_map* map, int batch,
                                       const uint64_t* reading_ids, const int* n_parts, const uint64_t* part_ids,
                                       const float* T_parts, const float* T0s);
int ls_icp_register_submap_batch_end(ls_ctx* ctx, float* T_outs, ls_icp_stats* stats, int* statuses);

/* ---- one registration sharded by queries over the GPUs of a node (SURVEY.md 8 e-2) -------------------------
 * The scan-matching of LaserTrack::processPoseAndLaserScan (laser_slam/src/laser_track.cpp:196-292) for ONE scan,
 * with the reading split over the GPUs of a node (one process / context per GPU, at most 8).  Every shard pushes the
 * same scans into its own map and makes the same call; per iteration each GPU stores its partial trimmed-select
 * histograms and normal-equation sums into a slot of every peer's exchange buffer over NVLink (CUDA IPC mapping), from
 * inside the persistent kernel.  The result is bit-identical to ls_icp_register_submap on every shard.
 *
 * Setup, once: every shard calls ls_shard_exchange_create (allocates its buffer, returns 64 handle bytes); the handles
 * are gathered in rank order by any means (torch.distributed all_gather, a pipe ...) and passed to
 * ls_shard_exchange_connect on every shard.  After that ls_icp_register_submap_sharded is a COLLECTIVE: every shard
 * makes the same sequence of calls with the same arguments.  A shard that does not show up trips the kernel's watchdog
 * on the others (the launch fails after 8 s; it does not hang).  Close only after every shard is done (the peers store
 * into the buffer). */
#define LS_IPC_HANDLE_BYTES 64
int ls_shard_exchange_create(ls_ctx* ctx, int shard_rank, int shard_count, unsigned char handle[LS_IPC_HANDLE_BYTES]);
int ls_shard_exchange_connect(ls_ctx* ctx, const unsigned char* handles /* shard_count x LS_IPC_HANDLE_BYTES, rank order */);
void ls_shard_exchange_close(ls_ctx* ctx);
int ls_icp_register_submap_sharded(ls_ctx* ctx, const ls_icp_params* prm, const ls_map* map, uint64_t reading_id,
                                   int n_parts, const uint64_t* part_ids, const float* T_parts, const float T0[16],
                                   float T_out[16], ls_icp_stats* stats);

/* Sub-map <-> sub-map registration on resident data: the loop-closure ICP of
 * IncrementalEstimator::processLoopClosure (laser_slam/src/incremental_estimator.cpp:90-115) without the two
 * buildSubMapAroundTime clouds (laser_slam/src/laser_track.cpp:602-651) visiting the host.  Reference = parts of
 * ref_map (normals included), reading = parts of reading_map, each part transformed by its T (an exact identity
 * copies the scan verbatim); the two maps may be the same object.  T_out maps reading coordinates into reference
 * coordinates.  Bit-identical to ls_map_assemble of both sides followed by ls_icp_register. */
int ls_icp_register_submaps(ls_ctx* ctx, const ls_icp_params* prm, const ls_map* ref_map, int n_ref_parts,
                            const uint64_t* ref_part_ids, const float* T_ref_parts, const ls_map* reading_map,
                            int n_reading_parts, const uint64_t* reading_part_ids, const float* T_reading_parts,
                            const float T0[16], float T_out[16], ls_icp_stats* stats);

/* Assemble a sub-map and download it (LaserTrack::buildSubMapAroundTime,
 * LaserTrack::getLocalCloudInWorldFrame laser_track.cpp:247-266).  out4: 4*M floats,
 * out_normals3: 3*M floats (may be NULL); returns M through *m_out. */
int ls_map_assemble(ls_ctx* ctx, const ls_map* map, int n_parts, const uint64_t* part_ids,
                    const float* T_parts, float* out4, float* out_normals3, int* m_out);

/* ---- input side and map maintenance (SURVEY.md §8 row f4) ---------------------------------------------------
 * The steps laser_slam_ros runs on the CPU either side of the registration, on the device.  Host buffers in and out;
 * `device` selects the GPU (no context needed).
 *   ls_ingest_pointcloud2   sensor_msgs/PointCloud2 payload -> DataPoints features: x, y, z floats at byte offsets
 *                           off_* inside records of point_step bytes -> {x, y, z, 1}
 *                           (laser_slam_ros/src/laser_slam_worker.cpp:125, pcl::fromROSMsg + conversion)
 *   ls_filter_cylinder      applyCylindricalFilter (laser_slam_ros/include/laser_slam_ros/common.hpp:194-223, used by
 *                           LaserSlamWorker::getFilteredMap, laser_slam_worker.cpp:415-488): keeps the points inside
 *                           (remove_points_inside == 0: d_xy^2 <= r^2 and |dz| <= h/2) or outside (>= on either) the
 *                           cylinder, in input order; out4 holds up to n points, *n_out the number kept
 *   ls_voxel_grid           pcl::VoxelGrid as getFilteredMap uses it (laser_slam_worker.cpp:434-441): one centroid per
 *                           occupied voxel of edge leaf_size, voxels in ascending cell-index order (x fastest); the
 *                           centroid is the exact mean of the voxel's points (fixed-point sums), rounded once
 *   ls_deskew_revolution    the point arithmetic of the Velodyne assembler
 *                           (sensor_drivers/velodyne_assembler/src/velodyne_assembler_ros.cpp:57-143): the packets of one
 *                           revolution, concatenated (packet k = points [packet_offsets[k], packet_offsets[k+1])), each
 *                           transformed by its T_packets[k] (column-major 4x4: sensor at the packet's time -> sensor at the
 *                           revolution's start, :124-130) and then all by T_final (start -> last packet, :107-108), as two
 *                           float32 transforms like the reference; an exact identity copies verbatim.  The wrap detection
 *                           and the composition of the transforms stay on the host:
 *                           include/laser_slam/velodyne_assembler.hpp */
int ls_ingest_pointcloud2(int device, const void* data, int point_step, int off_x, int off_y, int off_z, int n, float* out4);
int ls_filter_cylinder(int device, const float* in4, int n, const double center[3], double radius_m, double height_m,
                       int remove_points_inside, float* out4, int* n_out);
int ls_voxel_grid(int device, const float* in4, int n, const float leaf_size[3], float* out4, int* n_out);
int ls_deskew_revolution(int device, const float* points4, const int* packet_offsets, int n_packets, const float* T_packets,
                         const float T_final[16], float* out4);

/* ---- resident local map: the map maintenance of LaserSlamWorker (laser_slam_ros/src/laser_slam_worker.cpp) ------------
 * The worker's local_map_, local_map_filtered_, distant_map_ and local_map_queue_ kept on the device next to a ring, so the
 * scans reach the map and the map reaches the filters without crossing PCIe.  Only counts return to the host until a
 * cloud is downloaded.  The rules (oracle/LOCAL_MAP.md):
 *   ls_local_map_add_scan    scanCallback (:195-246): the slot's scan moved by T_w_scan (float32, the ls_map_assemble
 *                            arithmetic; an exact identity copies it verbatim); with remove_ground_from_local_map a point is
 *                            kept iff (double)z > robot_z - ground_distance_to_robot_center_m; input order kept; the cloud is
 *                            appended to LOCAL and queued as one cloud, unless nothing is left (then neither)
 *   ls_local_map_filter      getFilteredMap (:415-488): snapshot = LOCAL; LOCAL := the snapshot inside the cylinder around
 *                            `center` of radius distance_to_consider_fixed and height 40 (ls_filter_cylinder's <= rule);
 *                            with separate_distant_map, v = voxel grid of the SNAPSHOT (ls_voxel_grid's rule, voxels with
 *                            fewer than minimum_point_number_per_voxel points dropped), LOCAL_FILTERED := inside(v) (<=),
 *                            DISTANT += outside(v) (>=; a centroid on the boundary lands in both), FILTERED_MAP =
 *                            LOCAL_FILTERED ++ DISTANT; without it FILTERED_MAP = the snapshot and LOCAL_FILTERED is kept
 *   ls_local_map_transform   updateLocalMap (:522-540): LOCAL and LOCAL_FILTERED moved by T in place (float32, no
 *                            correctTransformationMatrix); DISTANT and the queue are not moved, as in the reference
 *   ls_local_map_clear       clearLocalMap (:496-506): empties LOCAL and LOCAL_FILTERED; DISTANT and the queue stay
 *   ls_local_map_take_queue  getQueuedPoints (:407-412): the queued clouds in order (cloud k = points
 *                            [cloud_offsets[k], cloud_offsets[k+1])), then the queue is empty
 * FILTERED_MAP is the cloud the last ls_local_map_filter returned; it is kept as a value, unaffected by later calls.
 * The local map has its own stream and device buffers (grown geometrically, never per call) and uses none of the context's
 * workspaces, so its calls are legal between ls_icp_register_submap_batch_begin and _end.  Calls are synchronous.  Errors:
 * LS_ERR_STATE for a scan no longer in the ring, LS_ERR_ARG for a ring on another device, a too-small buffer or bad
 * parameters, LS_ERR_NOMEM when a buffer cannot grow; the map is unchanged after any error.  The voxel grid refuses a
 * snapshot whose cell index space reaches 9e18 (LS_ERR_ARG) like ls_voxel_grid; it does not fall back to the unfiltered
 * cloud as pcl::VoxelGrid does past INT32_MAX cells. */
#define LS_LM_LOCAL 0          /* local_map_ */
#define LS_LM_LOCAL_FILTERED 1 /* local_map_filtered_ */
#define LS_LM_DISTANT 2        /* distant_map_ */
#define LS_LM_FILTERED_MAP 3   /* what the last ls_local_map_filter returned */
#define LS_LM_QUEUE 4          /* local_map_queue_, all clouds concatenated */

typedef struct ls_local_map ls_local_map;
typedef struct ls_local_map_params { /* LaserSlamWorkerParams (laser_slam_ros/include/laser_slam_ros/common.hpp:20-31) */
  double distance_to_consider_fixed;        /* cylinder radius [m], >= 0 */
  int separate_distant_map;
  double voxel_size_m;                      /* leaf [m], > 0 (used with separate_distant_map) */
  int minimum_point_number_per_voxel;       /* >= 0; 0 and 1 keep every voxel */
  int remove_ground_from_local_map;
  double ground_distance_to_robot_center_m;
  int initial_capacity_points;              /* first size of every buffer; <= 0: 262144 */
} ls_local_map_params;

int ls_local_map_create(ls_ctx* ctx, const ls_local_map_params* params, ls_local_map** out);
void ls_local_map_destroy(ls_local_map* lm);
/* T_w_scan: the track's pose at the scan's time after correctTransformationMatrix (LaserTrack::getLocalCloudInWorldFrame);
 * robot_z: the current pose's z.  *n_added = points appended (0: nothing appended or queued). */
int ls_local_map_add_scan(ls_local_map* lm, const ls_map* ring, uint64_t scan_id, const float T_w_scan[16], double robot_z,
                          int* n_added);
/* center: the current pose's position (rounded to float32 by the caller, as the reference's PclPoint does). */
int ls_local_map_filter(ls_local_map* lm, const double center[3], int* n_filtered_map);
int ls_local_map_size(const ls_local_map* lm, int which); /* points in LS_LM_*, < 0 on a bad argument */
/* cap: points out4 can hold (4 floats each); LS_ERR_ARG without a copy if the cloud is larger. */
int ls_local_map_download(const ls_local_map* lm, int which, float* out4, int cap, int* n);
int ls_local_map_take_queue(ls_local_map* lm, float* out4, int cap_points, int* cloud_offsets, int cap_clouds, int* n_clouds);
int ls_local_map_transform(ls_local_map* lm, const float T[16]);
int ls_local_map_clear(ls_local_map* lm);

/* ---- resident occupancy map: laser_to_octomap's insertion loop (laser_slam_tools/src/laser_to_octomap.cpp) ------------
 * Every scan of a trajectory inserted at its pose into a voxel map of float log-odds, the job volumetric_mapping's
 * OctomapManager does for the tool on one CPU thread.  The rules (oracle/OCCUPANCY.md):
 *   points      the slot's scan moved by T_w_scan (float32, the ls_map_assemble arithmetic; an exact identity copies it);
 *               the ray origin is T_w_scan's translation column; a point with a non-finite coordinate casts no ray
 *   keys        floor(c * (1/resolution)) + 32768 per axis in double, valid iff in [0, 65535]; packed kx | ky<<16 | kz<<32;
 *               a voxel's centre is (float)((k - 32768 + 0.5) * resolution)
 *   one ray     within max_range (or max_range < 0): free cells = the DDA keys from the origin to the point, the point's key
 *               occupied if valid; beyond it: free cells only, to origin + dir * max_range.  The DDA is octomap's
 *               computeRayKeys (origin key and every key stepped into before the end key; none when an end key is invalid
 *               or both ends share a key)
 *   one scan    a point whose endpoint key an earlier in-range point of the scan already has casts no ray; occupied wins
 *               over free; each touched voxel gets one update v = clamp(v + L_hit or L_miss, L_min, L_max) (float32,
 *               starting from 0) and becomes known.  A voxel is occupied iff known and v >= L_occ
 * L = (float)log(p / (1 - p)) of the probabilities below, computed on the host in double.  Scans apply in call order.
 * The map has its own stream and device buffers and uses none of the context's workspaces, so its calls are legal between
 * ls_icp_register_submap_batch_begin and _end.  Calls are synchronous; per insert only counters return to the host.
 * Errors: LS_ERR_STATE for a scan no longer in the ring, LS_ERR_ARG for a ring on another device, a too-small buffer or bad
 * parameters, LS_ERR_NOMEM when the map cannot grow; the known voxels and their log-odds are unchanged after any error. */
#define LS_OCC_KNOWN 1    /* every voxel that has had an update */
#define LS_OCC_OCCUPIED 2 /* known voxels with log-odds >= the occupancy threshold */

typedef struct ls_occupancy ls_occupancy;
typedef struct ls_occupancy_params {
  double resolution;          /* voxel edge [m], > 0 (laser_to_octomap: 0.075) */
  double prob_hit;            /* 0.9 */
  double prob_miss;           /* 0.4 */
  double clamp_min;           /* 0.12 */
  double clamp_max;           /* 0.97 */
  double occupancy_threshold; /* 0.7 */
  double max_range;           /* [m]; < 0: unlimited (laser_to_octomap: 20) */
  int initial_capacity;       /* bricks of 8x8x8 voxels the map starts with; <= 0: 32768.  It grows by doubling */
} ls_occupancy_params;

typedef struct ls_occupancy_stats {
  int64_t rays_cast;        /* points that cast a ray */
  int64_t rays_skipped;     /* points that did not: non-finite, or an endpoint key already occupied in this scan */
  int64_t free_updates;     /* voxels updated as free by this scan */
  int64_t occupied_updates; /* voxels updated as occupied by this scan */
  int64_t known_voxels;     /* known voxels of the map after the scan */
  int64_t bricks;           /* bricks in use */
  int64_t device_bytes;     /* device memory the map holds */
  float device_ms;          /* the insert on the map's stream */
} ls_occupancy_stats;

void ls_occupancy_default_params(ls_occupancy_params* out);
int ls_occupancy_create(ls_ctx* ctx, const ls_occupancy_params* params, ls_occupancy** out);
void ls_occupancy_destroy(ls_occupancy* om);
/* T_w_scan: the scan's pose (float32, column-major), not corrected.  stats may be NULL. */
int ls_occupancy_insert_scan(ls_occupancy* om, const ls_map* ring, uint64_t scan_id, const float T_w_scan[16],
                             ls_occupancy_stats* stats);
int ls_occupancy_size(ls_occupancy* om, int which, int64_t* n); /* voxels in LS_OCC_* */
/* The voxels of LS_OCC_* by ascending packed key (x fastest): keys, log-odds and centres {x, y, z, 1}; any output may be
 * NULL.  cap: voxels the outputs can hold; LS_ERR_ARG without a copy if there are more. */
int ls_occupancy_download(ls_occupancy* om, int which, uint64_t* keys, float* log_odds, float* centres4, int64_t cap,
                          int64_t* n);

/* The map as octomap's pruned binary tree, what OcTree::writeBinary saves (toMaxLikelihood, prune, writeBinaryConst) and
 * octomap_to_point_cloud reads back (reference laser_slam_tools/src/octomap_to_point_cloud.cpp).  The rules
 * (oracle/OCTREE.md):
 *   states      a known voxel is occupied iff v >= L_occ, else free; a node exists iff a voxel below it is known
 *   tree        depth 16 over the keys; child i of a node at depth d is bx | by<<1 | bz<<2, b = key bit 15-d per axis.  A node
 *               at depth 1..15 is a leaf iff its 8 children exist, are leaves and share a state (bottom-up; the root stays)
 *   payload     the inner nodes in pre-order (children 0..7), 2 bytes each: byte 0 covers children 0-3, byte 1 children 4-7;
 *               bit pair (2(i%4), 2(i%4)+1) is 00 unknown, 10 free leaf, 01 occupied leaf, 11 inner
 *   leaves      the occupied leaves in the same pre-order, centre (float)((floor((kc - 32768) / 2^s) + 0.5) * res * 2^s) per
 *               axis in double (octomap's keyToCoord(key, depth)), s = 16 - depth, kc the node's centre key
 * The build reads the map only and runs on its stream; an insert afterwards invalidates it, and a download then returns
 * LS_ERR_STATE.  Legal between ls_icp_register_submap_batch_begin and _end like every ls_occupancy_* call. */
typedef struct ls_octree_stats {
  int64_t nodes;           /* every node, root and leaves included (the .bt file's size line); 0 for an empty map */
  int64_t payload_bytes;   /* 2 per inner node */
  int64_t occupied_leaves;
  float device_ms;         /* the build on the map's stream */
} ls_octree_stats;

int ls_occupancy_build_octree(ls_occupancy* om, ls_octree_stats* stats);
/* The last build's payload and, each when not NULL, its occupied leaves' centres {x, y, z, 1} and depths (1..16).  payload_cap:
 * bytes payload can hold; leaf_cap: leaves centres4 and depths can hold; LS_ERR_ARG without a copy if either is too small. */
int ls_occupancy_download_octree(ls_occupancy* om, uint8_t* payload, int64_t payload_cap, float* centres4, uint8_t* depths,
                                 int64_t leaf_cap);
/* The whole .bt file at `path`: octomap's three comment lines, "id OcTree", "size <nodes>", "res <resolution as %g>", "data",
 * then the payload.  Builds the tree unless the last build is current.  stats may be NULL. */
int ls_occupancy_write_octomap(ls_occupancy* om, const char* path, ls_octree_stats* stats);

/* octomap's OcTree::readBinary into the map (DESIGN.md §4b'''''').  A read replaces the map: the file's
 * resolution becomes the map's (hit, miss, clamps, threshold and max range stay), and every voxel below a free leaf becomes
 * known with L_min (the clamp_min log-odds), below an occupied leaf with L_max; the rest is unknown.  Unpruned files and
 * inner nodes without children are accepted.  With clamp_min < occupancy_threshold <= clamp_max (the defaults) writing the
 * loaded map gives the file's bytes again.  The parse and the expansion run on the device, on the map's stream; the call
 * is synchronous, invalidates the last octree build on success and is legal between ls_icp_register_submap_batch_begin and
 * _end.  Errors: LS_ERR_ARG for a bad header, a truncated payload, an inner node at depth 16, a size that does not count
 * the payload's nodes or a resolution that is not finite and > 0 (bytes after the tree are ignored); LS_ERR_NOMEM, before
 * the map grows, when the file covers more bricks than the map can index (2^29), or when it cannot grow.  The map, its
 * resolution and a current octree build are unchanged after any error. */
typedef struct ls_octomap_read_stats {
  int64_t nodes, inner_nodes, free_leaves, occupied_leaves;
  int64_t known_voxels, bricks; /* of the map after the read */
  double resolution;            /* the map's resolution after the read */
  float device_ms;              /* the read on the map's stream, the payload's upload included */
} ls_octomap_read_stats;
/* payload: the bytes after "data\n" (payload_bytes of them; NULL when 0); nodes: the header's size (>= 0).  stats may be
 * NULL. */
int ls_occupancy_read_octree(ls_occupancy* om, const uint8_t* payload, int64_t payload_bytes, int64_t nodes,
                             double resolution, ls_octomap_read_stats* stats);
/* The whole .bt file at `path`: its header is parsed on the host as laser_slam_b200.read_octomap parses it, then as above. */
int ls_occupancy_read_octomap(ls_occupancy* om, const char* path, ls_octomap_read_stats* stats);

/* The map as octomap's full tree, what OcTree::write saves (the .ot file) and the data of a full octomap message
 * (getOctomapFullMsg): every node's float log-odds, so a saved map resumes mapping exactly (DESIGN.md §4b').  Rules:
 *   tree        as the .bt tree (depth 16, child i = bx | by<<1 | bz<<2); a node exists iff a known voxel lies below it
 *   pruning     a node at depth 1..15 is a leaf iff its 8 children exist, are leaves and their log-odds compare equal as
 *               floats (+0.0 == -0.0); bottom-up and maximal, the root stays.  The collapsed leaf keeps child 0's bits
 *   inner       an inner node holds its largest child's value (a strict > scan over children 0..7: the earliest wins ties)
 *   payload     every node in pre-order (children 0..7), 5 bytes each: its value as float32 little-endian, then a byte whose
 *               bit i is set iff child i exists
 * The build reads the map only, runs on its stream and is cached apart from the .bt build: neither build invalidates the
 * other; an insert or a successful read invalidates both, and a download then returns LS_ERR_STATE.  Legal between
 * ls_icp_register_submap_batch_begin and _end like every ls_occupancy_* call. */
typedef struct ls_full_octree_stats {
  int64_t nodes;          /* every node, root and leaves included (the .ot file's size line); 0 for an empty map */
  int64_t leaves;
  int64_t payload_bytes;  /* 5 per node */
  float device_ms;        /* the build on the map's stream */
} ls_full_octree_stats;

int ls_occupancy_build_full_octree(ls_occupancy* om, ls_full_octree_stats* stats);
/* The last full build's payload; LS_ERR_ARG without a copy when payload_cap is below its size. */
int ls_occupancy_download_full_octree(ls_occupancy* om, uint8_t* payload, int64_t payload_cap);
/* The whole .ot file at `path`: "# Octomap OcTree file", octomap's two further comment lines, "id OcTree", "size <nodes>",
 * "res <resolution as %g>", "data", then the payload.  Builds the full tree unless the last full build is current.  stats may
 * be NULL. */
int ls_occupancy_write_octomap_full(ls_occupancy* om, const char* path, ls_full_octree_stats* stats);

/* octomap's readData of a full tree into the map (setOctomapFromFullMsg; AbstractOcTree::read for a file).  A read
 * replaces the map: the file's resolution becomes the map's, and every voxel below a leaf becomes known with the leaf's
 * value verbatim (no clamp: the next insert clamps as usual); stored inner values are not used.  Unpruned files are
 * accepted.  Read then write gives the bytes of any file this library wrote, and the map's .bt equals the original's.  The
 * parse and the expansion run on the device, on the map's stream; the call is synchronous and legal between
 * ls_icp_register_submap_batch_begin and _end.  Errors: LS_ERR_ARG for a bad header (first line, id other than OcTree), a
 * truncated payload, a node at depth 16 with children, a size other than the nodes parsed, a leaf value that is NaN or
 * infinite, or a resolution that is not finite and > 0 (bytes after the tree are ignored); LS_ERR_NOMEM, before the map
 * grows, when the file covers more than 2^29 bricks or the map cannot grow.  After any error the map, its resolution and
 * both cached builds are unchanged.  stats (may be NULL): nodes, inner_nodes = nodes with children, free and occupied
 * leaves classified by the map's occupancy threshold. */
int ls_occupancy_read_full_octree(ls_occupancy* om, const uint8_t* payload, int64_t payload_bytes, int64_t nodes,
                                  double resolution, ls_octomap_read_stats* stats);
/* The whole .ot file at `path`: its header is parsed on the host as laser_slam_b200.read_octomap_full parses it, then as
 * above. */
int ls_occupancy_read_octomap_full(ls_occupancy* om, const char* path, ls_octomap_read_stats* stats);

/* The map's leaves as boxes: volumetric_mapping's getAllFreeBoxes / getAllOccupiedBoxes and generateMarkerArray's cube lists
 * (DESIGN.md §4b'''''''''''').  Rules:
 *   tree        the leaves of the value-pruned tree the .ot build writes (octomap's tree in memory), not the .bt file's
 *               max-likelihood tree, so occupied leaves can be finer than ls_occupancy_download_octree's; for a map read
 *               from a .bt file the two coincide
 *   state       LS_CELL_OCCUPIED iff the leaf's log-odds >= L_occ, else LS_CELL_FREE
 *   order       octomap's leaf iterator: pre-order, children 0..7
 *   box         depth d (1..16), centre keyToCoord(key, d) per axis as the .bt leaves above (float), edge res * 2^(16-d)
 *   region      region_min3 / region_max3 in metres, keyed as the map's points in double (floor(c * (1/res)) + 32768) and
 *               clamped to [0, 65535]: a leaf is listed iff its key cube [k0, k0 + 2^(16-d)) meets [key(min), key(max)] on
 *               every axis.  Both NULL: every leaf
 *   cubes       the listed leaves ordered by state (occupied first), then depth 0..16, then the leaf order.  An occupied
 *               cube's colour is octomap_server's heightMapColor(h), h = (1 - min(max((z - min_z) / (max_z - min_z), 0), 1))
 *               * color_factor, z the float centre's z widened to double, all in double and cast to float once, alpha 1
 * ls_occupancy_build_leaves lists the leaves (building the .ot tree first unless its cached build is current; neither
 * cached build is invalidated, and their outputs do not change).  Only the counts come back; the list stays on the device
 * until an insert, edit, read or reset of the map invalidates it, and a download then returns LS_ERR_STATE.  Calls run on
 * the map's stream, are synchronous, never change the map and are legal between ls_icp_register_submap_batch_begin and
 * _end.  Errors: LS_ERR_ARG for a region that is not finite, inverted (min > max on an axis) or given by one pointer only,
 * bad `which`, NULL n, cap < 0, a NULL output with cap > 0, more leaves than cap (*n then holds their number, nothing is
 * copied), or colour arguments that are not finite, have min_z >= max_z or a difference that overflows; LS_ERR_NOMEM when the list cannot grow.  A
 * refused call leaves the map, both cached builds and the last list as they were. */
#define LS_LEAVES_FREE 1
#define LS_LEAVES_OCCUPIED 2
#define LS_LEAVES_ALL 3
typedef struct ls_leaf_stats {
  int64_t free_leaves, occupied_leaves;           /* listed leaves */
  int64_t free_by_depth[17], occupied_by_depth[17]; /* listed leaves per depth 0..16 */
  float device_ms;                                /* the call on the map's stream, a .ot build it needed included */
} ls_leaf_stats;
/* stats may be NULL. */
int ls_occupancy_build_leaves(ls_occupancy* om, const double* region_min3, const double* region_max3, ls_leaf_stats* stats);
/* which: LS_LEAVES_*; per listed leaf of that state, in leaf order: centre {x, y, z, 1}, depth and state LS_CELL_*.  *n always
 * set, so cap = 0 asks for the count. */
int ls_occupancy_download_leaves(ls_occupancy* om, int which, float* centres4, uint8_t* depths, int8_t* states, int64_t cap,
                                 int64_t* n);
/* The cube lists of the last list: centres4 holds *n cubes {x, y, z, 1} in the cube order, the occupied cubes of depth d at
 * [occupied_offsets[d], occupied_offsets[d + 1]) and the free ones at [free_offsets[d], free_offsets[d + 1]) (so
 * occupied_offsets[17] = free_offsets[0]); colors4 {r, g, b, a} per occupied cube.  Offsets and *n always set; cap: cubes
 * centres4 can hold. */
int ls_occupancy_marker_cubes(ls_occupancy* om, double min_z, double max_z, double color_factor, float* centres4,
                              float* colors4, int64_t occupied_offsets[18], int64_t free_offsets[18], int64_t cap, int64_t* n);

/* The map projected onto a 2D occupancy grid: octomap_server's projected_map (nav_msgs/OccupancyGrid) at m_maxTreeDepth = 16
 * with a complete projection (DESIGN.md §4b''''''''''''').  Rules:
 *   tree        the leaves of the .bt tree (toMaxLikelihood + prune, what ls_occupancy_write_octomap writes); every leaf is
 *               free or occupied.  A map with no known voxel gives a 0 x 0 grid
 *   bounds      octomap's calcMinMax over those leaves, in double: per axis the least centre - size/2 and the largest
 *               (centre - size/2) + size, centre keyToCoord(key, d) and size res * 2^(16-d).  Unlike ls_occupancy_bounds,
 *               which takes depth-16 leaves, a coarse leaf counts whole
 *   padding     min x = min(min x, -min_size_x/2), max x = max(max x, min_size_x/2), the same in y
 *   keys        paddedMinKey / paddedMaxKey = coordToKeyChecked of the padded corners as float points (z too)
 *   geometry    width = paddedMaxKey.x - paddedMinKey.x + 1, height likewise in y, resolution = res, origin =
 *               (float)keyToCoord(paddedMinKey) - res/2 in x and y (z and yaw 0).  Cell (i, j) is data[j * width + i]
 *   band        a leaf takes part iff z + size/2 > min_z && z - size/2 < max_z, z = keyToCoord(key, d).z in double
 *   paint       a taking-part leaf at depth d fills its 2^(16-d) x 2^(16-d) cells from (key.x - paddedMinKey.x, key.y -
 *               paddedMinKey.y): an occupied leaf writes 100, a free one 0 where the cell is still -1; every cell starts
 *               at -1.  So a cell is 100 if any occupied leaf covers it, else 0 if any free leaf does, else -1
 * ls_occupancy_build_projection builds the .bt tree first unless its cached build is current (neither cached build is
 * invalidated, and their outputs do not change), projects it and sets *info; the grid stays on the device until an insert,
 * edit, read or reset of the map invalidates it, and a download then returns LS_ERR_STATE.  Calls run on the map's stream,
 * are synchronous, never change the map and are legal between ls_icp_register_submap_batch_begin and _end.  Errors:
 * LS_ERR_ARG for NULL info, a NaN min_z or max_z (infinities are allowed), a min_size that is negative, NaN or infinite, a
 * padded corner outside the key space, a grid of more than 2^31 - 1 cells, a NULL data with cap > 0 or cap < width *
 * height (nothing is copied); LS_ERR_NOMEM when the grid cannot be allocated.  A refused call leaves the map, both cached
 * builds, the leaf list and the last projection as they were. */
typedef struct ls_grid_info {
  int64_t width, height;      /* cells along x and y; 0 x 0 for a map with no known voxel */
  double resolution;          /* the map's resolution [m] (the message's float32 field holds it rounded) */
  double origin_x, origin_y;  /* the lower corner of cell (0, 0) [m] */
  int64_t unknown_cells, free_cells, occupied_cells; /* cells of -1, 0 and 100 */
  float device_ms;            /* the call on the map's stream, a .bt build it needed included */
} ls_grid_info;
int ls_occupancy_build_projection(ls_occupancy* om, double min_z, double max_z, double min_size_x, double min_size_y,
                                  ls_grid_info* info);
/* The last projection's width * height cells (-1, 0 or 100), row j at data[j * width]. */
int ls_occupancy_download_projection(ls_occupancy* om, int8_t* data, int64_t cap);

/* Queries of the map: volumetric_mapping's WorldBase (getCellStatusPoint, getLineStatus, getVisibility,
 * getLineStatusBoundingBox) and octomap's castRay, batched, one device thread per query.  The rules (oracle/QUERIES.md):
 *   cell        the key of the double point (octomap's search(x, y, z): floor(c * (1/resolution)) + 32768, no float cast);
 *               unknown when the key is invalid (non-finite included) or the voxel is not known, occupied when known and
 *               v >= L_occ, else free.  log_odds: v, or NaN (0x7fc00000) when unknown
 *   line        the keys of computeRayKeys((float)start, (float)end) (as one ray of the insert: origin key first, the end
 *               key never, none when an end key is invalid or both share a key), walked in order up to the first occupied
 *               key or, when stop_at_unknown, the first unknown one; that key's state and packed key, else free and all
 *               ones.  getLineStatus is stop_at_unknown = 1; getVisibility takes it as its flag.  So a segment whose ends
 *               share a key, or whose end key is invalid, is free, and the end voxel is never checked
 *   box         box3 = the box size (finite, >= 0 per axis).  disc = size / ceil((size + 0.001) / resolution) (1.0 if
 *               <= 0); offsets x = -size/2; x <= size/2; x += disc, in double, y inside x and z innermost; line i runs
 *               from start + offset_i to end + offset_i (added in double, then cast to float).  The result is that of the
 *               first line in loop order that is not free, else free
 *   ray         castRay(origin, direction, end, ignore_unknown, max_range) on float triples: LS_RAY_INVALID for an origin
 *               with an invalid key or a zero direction (end NaN); an occupied origin voxel is a hit, an unknown one (not
 *               ignored) LS_RAY_UNKNOWN, both at the origin voxel's centre; then octomap's DDA from the normalised
 *               direction (border half step in double), stopping with LS_RAY_KEY_BOUND before a step out of [0, 65535],
 *               LS_RAY_MAX_RANGE when max_range > 0 and the new centre is farther (sum of float squares in double > max_range^2),
 *               LS_RAY_HIT on an occupied voxel, LS_RAY_UNKNOWN on an unknown one unless ignored.  ends3: the centre of the
 *               voxel the result names
 * A query reads the map only, on the map's stream, and is synchronous; only the outputs and a counter return.  Legal between
 * ls_icp_register_submap_batch_begin and _end.  n = 0 is LS_OK without a launch.  Errors: LS_ERR_ARG for n < 0, a NULL
 * required buffer, a negative or non-finite box size or more than 2^31 - 1 box lines in the call; LS_ERR_NOMEM when the
 * staging cannot grow.  The map is unchanged after any call. */
#define LS_CELL_FREE 0
#define LS_CELL_OCCUPIED 1
#define LS_CELL_UNKNOWN 2
#define LS_RAY_INVALID 0
#define LS_RAY_HIT 1
#define LS_RAY_UNKNOWN 2
#define LS_RAY_MAX_RANGE 3
#define LS_RAY_KEY_BOUND 4

typedef struct ls_occupancy_query_stats {
  int64_t keys_visited; /* voxel states the kernels read */
  float device_ms;      /* the call on the map's stream, copies included */
} ls_occupancy_query_stats;

/* points3: n double triples.  log_odds and stats may be NULL. */
int ls_occupancy_cell_status(ls_occupancy* om, const double* points3, int n, int8_t* status, float* log_odds,
                             ls_occupancy_query_stats* stats);
/* starts3 / ends3: n double triples; box3: NULL for plain lines.  first_keys and stats may be NULL. */
int ls_occupancy_line_status(ls_occupancy* om, const double* starts3, const double* ends3, int n, const double* box3,
                             int stop_at_unknown, int8_t* status, uint64_t* first_keys, ls_occupancy_query_stats* stats);
/* origins3 / directions3: n float triples; max_range <= 0 (or NaN): none.  ends3 and stats may be NULL. */
int ls_occupancy_cast_rays(ls_occupancy* om, const float* origins3, const float* directions3, int n, int ignore_unknown,
                           double max_range, int8_t* result, float* ends3, ls_occupancy_query_stats* stats);

/* Box status and robot collision: volumetric_mapping's getCellStatusBoundingBox, checkCollisionWithRobot and
 * checkPathForCollisionsWithRobot, batched (DESIGN.md §4b''''''''''').  Per box (centre p, size s, double triples):
 *   1  the centre's state by the cell rule above (double key); when it is not free, that is the box's status
 *   2  the float centre (float)p with an invalid key: unknown
 *   3  corners bmin = (float)(p - s/2), bmax = (float)(p + s/2) per axis
 *   4  occupied pass, only when both corners have valid keys: every known voxel with keys between key(bmin) and key(bmax)
 *      on all axes whose cube c +- res/2 (c = ((double)(k - 32768) + 0.5) * res) is not wholly outside [bmin, bmax] on an
 *      axis; an occupied one makes the box occupied
 *   5  unknown pass: per axis x = bmin; x <= bmax; x += res in double (y inside x, z innermost), each point cast to float
 *      and keyed; an invalid key or a voxel that is not known makes the box unknown
 *   6  otherwise free.  Occupied beats unknown beats free, so the order of the work does not matter
 * A pose collides when its box (the robot's size at the position) is occupied, or with unknown_as_occupied when it is not
 * free.  Path p is positions3[offsets[p] ... offsets[p + 1]); its result is the first colliding pose's index within the
 * path, or -1 (an empty path included).  checkCollisionWithRobot is a path of one pose.
 * Calls read the map only, on the map's stream, are synchronous and are legal between ls_icp_register_submap_batch_begin
 * and _end; n = 0 (n_paths = 0) is LS_OK without a launch.  keys_visited counts the centres and the voxel states the
 * passes read (it depends on the scheduling).  Errors, before any result: LS_ERR_ARG for n < 0, a NULL required array, a
 * size that is negative or not finite (the robot size even when every path is empty), more than 2^17 loop points on an
 * axis of a box whose centre has a valid key, boxes that span more than 2^36 (box, brick) items in all (per box with a
 * valid centre, the product over the axes of the 8-voxel bricks its passes touch, whatever the map holds), path offsets
 * that are not non-decreasing from 0, or more than 2^31 - 1 poses; LS_ERR_NOMEM when the staging cannot grow.  A centre that is NaN or infinite is not refused: it is unknown by step 1. */
/* getCellStatusBoundingBox per box: centres3 / sizes3 n double triples; status LS_CELL_*.  stats may be NULL. */
int ls_occupancy_box_status(ls_occupancy* om, const double* centres3, const double* sizes3, int n, int8_t* status,
                            ls_occupancy_query_stats* stats);
/* checkPathForCollisionsWithRobot per path: path p is positions3[offsets[p] .. offsets[p+1]); first_collision[p] the
 * first colliding pose's index within its path, -1 when none.  stats may be NULL. */
int ls_occupancy_check_paths(ls_occupancy* om, const double* positions3, const int64_t* offsets, int n_paths,
                             const double robot_size3[3], int unknown_as_occupied, int64_t* first_collision,
                             ls_occupancy_query_stats* stats);

/* Edits of the map: volumetric_mapping's setFree / setOccupied (OctomapWorld::setLogOddsBoundingBox, the set-box-occupancy
 * service), resetMap, getOccupiedPointcloudInBoundingBox and the extent getMapBounds reads (DESIGN.md §4b'''''''').  Rules:
 *   box loop    per axis in double: c = res * floor(p / res) + res / 2 (a division), then x = (c - s/2) + 0.001; x <=
 *               (c + s/2) - 0.001; x += res, y inside x and z innermost; each point is cast to float and keyed as above
 *               (floor(c * (1/resolution)) + 32768); a point with an invalid key is skipped.  A size of 0 covers nothing
 *   set         every voxel a loop point keys becomes known with L_min (setFree) or L_max (setOccupied); later inserts update
 *               it as usual.  Boxes apply in call order: the last box covering a voxel decides its value
 *   reset       no known voxel, no brick; resolution, parameters and device memory stay (device_bytes is unchanged).  An
 *               insert afterwards equals the same insert into a new map
 *   box voxels  per loop point (in loop order, repeats kept) whose voxel is occupied (LS_OCC_OCCUPIED) or known
 *               (LS_OCC_KNOWN): its packed key, log-odds and voxel centre {x, y, z, 1}
 *   bounds      per axis over the known keys: min = (double)centre(kmin) - res/2, max = ((double)centre(kmax) - res/2) + res,
 *               centre(k) the float voxel centre; all zeros for a map without known voxels
 * Calls run on the map's stream, are synchronous and are legal between ls_icp_register_submap_batch_begin and _end.  A
 * successful set or reset invalidates both cached tree builds.  Errors: LS_ERR_ARG for n < 0, a NULL array, a centre or
 * size that is not finite, a negative size, a box axis of more than 2^17 loop points (or a box of more than 2^31 - 1 for
 * box voxels); LS_ERR_NOMEM, before anything is allocated, when the bricks a set covers and those in use exceed 2^29, or
 * when the map cannot grow.  Every box is checked before any work, so one bad box refuses the whole call; after any error
 * the known voxels, their values and both cached builds are unchanged. */
typedef struct ls_occupancy_edit_stats {
  int64_t voxels_set;   /* loop points with a valid key, summed over the boxes (repeats counted) */
  int64_t new_known;    /* voxels that became known */
  int64_t known_voxels, bricks, device_bytes; /* of the map after the call */
  float device_ms;      /* the call on the map's stream */
} ls_occupancy_edit_stats;
/* n boxes: centres3 / sizes3 double triples; occupied[i] 0 = setFree, otherwise setOccupied.  stats may be NULL. */
int ls_occupancy_set_boxes(ls_occupancy* om, const double* centres3, const double* sizes3, const int8_t* occupied, int n,
                           ls_occupancy_edit_stats* stats);
int ls_occupancy_clear(ls_occupancy* om);
/* which: LS_OCC_KNOWN / LS_OCC_OCCUPIED; outputs may be NULL; *n always set; LS_ERR_ARG without a copy when *n > cap, so
 * cap = 0 asks for the count. */
int ls_occupancy_box_voxels(ls_occupancy* om, const double center3[3], const double size3[3], int which, uint64_t* keys,
                            float* log_odds, float* centres4, int64_t cap, int64_t* n);
int ls_occupancy_bounds(ls_occupancy* om, double min3[3], double max3[3]);

/* Change detection: octomap's enableChangeDetection / changedKeysBegin / numChangesDetected / resetChangeDetection, as
 * volumetric_mapping's getChangedPoints reads them, kept as a diff against a baseline (DESIGN.md §4b'''''''''').  Rules:
 *   state     per voxel: LS_CELL_UNKNOWN, LS_CELL_FREE (known, v < L_occ) or LS_CELL_OCCUPIED (known, v >= L_occ)
 *   baseline  the state of every voxel known when tracking was enabled or last reset, stored by brick key (not by pool
 *             index), with the map's resolution then
 *   changed   a voxel whose state now differs from its state at the baseline: one known now and unknown then (octomap's
 *             `true`), one whose occupied state differs (an odd number of flips; an even number leaves nothing), and one
 *             known then and unknown now (only ls_occupancy_clear or a .bt / .ot read does that).  A log-odds change that
 *             keeps the state is not a change.  The result does not depend on the order of the updates since the baseline,
 *             so inserts, edits and reads run exactly as without tracking
 *   outputs   per changed voxel, by ascending packed key: the key, the state now (status) and then (previous), LS_CELL_*,
 *             and the voxel centre {x, y, z, 1}: (float)(((double)(k - 32768) + 0.5) * res) per axis, res the map's
 *             resolution for a voxel known now and the baseline's for one unknown now
 *   reset     reset != 0 makes the map as it is now the new baseline after a successful copy (getChangedPoints followed by
 *             resetChangeDetection); a refused call does not reset
 * ls_occupancy_track_changes(om, 1) takes a fresh baseline (again when tracking is on); (om, 0) turns tracking off and
 * frees the baseline.  Calls run on the map's stream, are synchronous, never change the map and are legal between
 * ls_icp_register_submap_batch_begin and _end.  Errors: LS_ERR_STATE from ls_occupancy_changes while tracking is off;
 * LS_ERR_ARG, without a copy and without a reset, for a NULL n, cap < 0 or more changes than cap (so cap = 0 asks for the
 * count); LS_ERR_NOMEM when the baseline or the scratch cannot grow.  After any error the baseline, the tracking state and
 * the map are as they were. */
typedef struct ls_occupancy_change_stats {
  int64_t bricks_compared; /* the map's bricks plus the baseline's, each read once per pass */
  int64_t changed;         /* voxels changed (= *n) */
  int64_t baseline_bricks; /* bricks of the baseline after the call */
  int64_t device_bytes;    /* device memory change detection holds: baselines and scratch */
  float device_ms;         /* the call on the map's stream, the reset's capture included */
} ls_occupancy_change_stats;
int ls_occupancy_track_changes(ls_occupancy* om, int enable);
/* keys, status, previous, centres4 and stats may be NULL; *n always set. */
int ls_occupancy_changes(ls_occupancy* om, uint64_t* keys, int8_t* status, int8_t* previous, float* centres4, int64_t cap,
                         int64_t* n, int reset, ls_occupancy_change_stats* stats);

/* Euclidean distance map of the occupancy map: octomap's DynamicEDTOctomap(maxdist, octree, bbxMin, bbxMax,
 * treatUnknownAsOccupied) over the finest cells of a box, recomputed in full on the device at every update and queried in
 * batches (DESIGN.md §4b''''''''').  Rules:
 *   box         each corner keyed as the map's points: k = floor((double)c * (1/res)) + 32768 per axis.  The grid covers keys
 *               kmin ... kmax per axis, both included; cell (x, y, z) is key kmin + (x, y, z); x fastest, then y, then z
 *   obstacles   a cell inside the box whose voxel is occupied (known, v >= L_occ); with treat_unknown_as_occupied, every
 *               unknown cell too.  Voxels outside the box do not count
 *   cap         m = (int)((double)max_dist / res + 1.0), M = m * m; max_dist (getMaxDist) = (float)(m * res)
 *   field       per cell s = the squared distance in cells to the nearest obstacle (dx^2 + dy^2 + dz^2).  s <= M: s and that
 *               obstacle; otherwise M and no obstacle (also when the box has none).  An obstacle cell has s = 0 and is its own
 *   ties        among obstacles at the least s, the smallest packed key (smallest z, then y, then x)
 *   queries     float triples keyed as the corners.  distance = (float)((double)(float)sqrt((double)s) * res), sqdist = s,
 *               obstacle = its voxel centre (float)(((double)(k - 32768) + 0.5) * res) per axis, NaN when the cell has none.
 *               A point whose key is invalid (non-finite included) or outside the box: -1.0f, -1 and NaN
 *   snapshot    the field is the map as of the last successful update; the box, the resolution, L_occ and M are taken from
 *               the map then.  Queries and downloads before the first update return LS_ERR_STATE
 * Unlike DynamicEDT3D, which propagates obstacles through the 26-neighbourhood with a priority queue and updates from
 * octomap's change detection, the transform is exact and recomputed in full.  The handle has its own stream and buffers and
 * uses none of the context's workspaces, so every call is legal between ls_icp_register_submap_batch_begin and _end.  Calls
 * are synchronous and never change the occupancy map.  Errors: LS_ERR_ARG, checked before any work and leaving the previous
 * field intact, for max_dist not finite or <= 0, m > 46340, a corner that is not finite or has an invalid key, bbx_min >
 * bbx_max on an axis, more than 2^30 cells, n < 0, a NULL required array, a map on another device or a too-small buffer;
 * LS_ERR_NOMEM when the field's buffers cannot grow, after which the handle has no field. */
typedef struct ls_distance_map ls_distance_map;
typedef struct ls_distance_map_params {
  float max_dist;                 /* [m], finite and > 0 */
  float bbx_min[3], bbx_max[3];   /* the box's corners [m] */
  int treat_unknown_as_occupied;
} ls_distance_map_params;

typedef struct ls_distance_map_stats {
  int32_t min_key[3];        /* kmin */
  int32_t size[3];           /* cells per axis */
  int64_t cells;
  int64_t obstacles;         /* obstacle cells in the box */
  double resolution;         /* the map's at the update */
  int32_t max_sqdist_cells;  /* M */
  float max_dist;            /* getMaxDist */
  int64_t device_bytes;      /* device memory the handle holds */
  float device_ms;           /* the update on the handle's stream */
} ls_distance_map_stats;

typedef struct ls_distance_map_query_stats {
  int64_t outside;  /* points with an invalid key or outside the box */
  float device_ms;  /* the call on the handle's stream, copies included */
} ls_distance_map_query_stats;

int ls_distance_map_create(ls_ctx* ctx, const ls_distance_map_params* params, ls_distance_map** out);
void ls_distance_map_destroy(ls_distance_map* dm);
/* The field of om's current state.  stats may be NULL. */
int ls_distance_map_update(ls_distance_map* dm, ls_occupancy* om, ls_distance_map_stats* stats);
/* points3: n float triples.  distance, sqdist_cells, obstacles3 (n float triples) and stats may be NULL. */
int ls_distance_map_query(ls_distance_map* dm, const float* points3, int n, float* distance, int32_t* sqdist_cells,
                          float* obstacles3, ls_distance_map_query_stats* stats);
/* The whole field in layout order: s per cell and its obstacle's packed key (all ones when none); either output may be NULL.
 * *n always set to the cells (after an update); LS_ERR_ARG without a copy when cap_cells is below it. */
int ls_distance_map_download(ls_distance_map* dm, int32_t* sqdist, uint64_t* obstacle_keys, int64_t cap_cells, int64_t* n);

/* ---- per-scan input filters (reference laser_slam/src/laser_track.cpp:24-30 loads them from
 * LaserTrackParams::icp_input_filters_file, :81 and :146 apply them to every scan before it is stored) ----------------
 * A chain is an array of ls_point_filter records applied in order; each filter sees the cloud the previous one produced,
 * every compaction keeps the input order and normals travel with their points.  The rules (oracle/INPUT_FILTERS.md):
 *   LS_PF_REMOVE_NAN          drop a point whose x, y or z is NaN (+-inf is left to the distance filters)
 *   LS_PF_MAX_DIST            dim -1: keep iff (x*x + y*y) + z*z < dist*dist (float32, each operation rounded);
 *                             dim 0/1/2: keep iff |coord| < dist
 *   LS_PF_MIN_DIST            the same with >
 *   LS_PF_BOUNDING_BOX        inside iff box[2a] < coord_a < box[2a+1] on all three axes; keeps the outside points
 *                             (remove_inside != 0) or the inside ones
 *   LS_PF_RANDOM_SAMPLING     keep iff ls_keep_point(i, 0x7e11, prob), i = index in the cloud entering the filter
 *   LS_PF_FIX_STEP_SAMPLING   keep iff i % step == 0
 *   LS_PF_VOXEL_GRID          ls_voxel_grid's centroids with edge leaf[3]; normals, when present, are averaged the same
 *                             exact way (not renormalised)
 *   LS_PF_SURFACE_NORMAL      normals as ls_estimate_normals with knn clamped to [3, 16]
 *   LS_PF_SAMPLING_SURFACE_NORMAL  the same, then keep iff ls_keep_point(i, 0x5a17, prob) */
#define LS_PF_REMOVE_NAN 1
#define LS_PF_MAX_DIST 2
#define LS_PF_MIN_DIST 3
#define LS_PF_BOUNDING_BOX 4
#define LS_PF_RANDOM_SAMPLING 5
#define LS_PF_FIX_STEP_SAMPLING 6
#define LS_PF_VOXEL_GRID 7
#define LS_PF_SURFACE_NORMAL 8
#define LS_PF_SAMPLING_SURFACE_NORMAL 9

typedef struct ls_point_filter {
  int32_t type;          /* LS_PF_* */
  int32_t dim;           /* Max/MinDist: -1 = distance to the origin, 0/1/2 = one axis */
  int32_t knn;           /* (Sampling)SurfaceNormal */
  int32_t step;          /* FixStepSampling: startStep */
  int32_t remove_inside; /* BoundingBox */
  int32_t reserved;
  float dist;            /* maxDist / minDist */
  float prob;            /* RandomSampling: prob; SamplingSurfaceNormal: ratio */
  float box[6];          /* BoundingBox: xMin, xMax, yMin, yMax, zMin, zMax */
  float leaf[3];         /* VoxelGrid: vSizeX, vSizeY, vSizeZ */
  float reserved_f;
} ls_point_filter;

/* Parse a libpointmatcher DataPointsFilters YAML list (`- NameDataPointsFilter:` followed by `key: value` lines, or
 * `{key: value, ...}` on the same line).  Host code: needs no GPU.  Absent keys take libpointmatcher's defaults except
 * knn 10, prob 1 and ratio 1, which keep the values PointMatcher::DataPointsFilters used before (oracle/INPUT_FILTERS.md).  out
 * may be NULL (count only).  On success *n_out = number of filters.  LS_ERR_ARG for a filter this path does not run
 * (any other name), a key value it cannot honour (FixStep endStep != startStep or stepMult != 1, VoxelGrid useCentroid 0,
 * ...) or more filters than `capacity`; *n_out is then the index of the offending filter. */
int ls_point_filters_from_yaml(const char* yaml_text, ls_point_filter* out, int capacity, int* n_out);
/* Run a chain on the device: host cloud in (normals through (pointer, stride) as ls_map_push_scan; may be NULL), host
 * cloud out.  out4 holds up to n points, out_normals3 (may be NULL) 3 floats per point; *n_out = points kept.  Asking
 * for out_normals3 when neither the input nor a normal filter provides normals returns LS_ERR_ARG. */
int ls_filter_cloud(ls_ctx* ctx, const ls_point_filter* filters, int n_filters, const float* in4, const float* normals,
                    int normals_stride, int n, float* out4, float* out_normals3, int* n_out);
/* Push a raw scan through a chain into the next ring slot: one upload, the whole chain on the device, the result in the
 * slot (synchronous, like ls_map_push_scan_estimate_normals).  The chain must leave normals (given, or a normal filter)
 * and at most max_pts_per_scan points; otherwise LS_ERR_ARG and no slot is taken.  A chain that keeps nothing stores an
 * empty scan (*n_kept 0; a registration with it as the reading or as its whole sub-map returns LS_ERR_CONVERGENCE,
 * also as one problem of a batch). */
int ls_map_push_scan_filtered(ls_map* map, const ls_point_filter* filters, int n_filters, const float* in4, const float* normals,
                              int normals_stride, int n, uint64_t* scan_id, int* n_kept);

/* ---- pose graph ------------------------------------------------------------------------------------
 * Replaces gtsam::ISAM2 as IncrementalEstimator uses it (laser_slam/src/incremental_estimator.cpp:17-20,
 * 151-163 estimate, 165-266 estimateAndRemove, 268-291 registerPrior).  Poses are 7 doubles
 * {qw,qx,qy,qz,tx,ty,tz}; a factor is what LaserTrack::makeMeasurementFactor /
 * makeRelativeMeasurementFactor build (laser_slam/src/laser_track.cpp:431-458):
 *   LS_FACTOR_PRIOR    error = Local(meas, T(key_a))
 *   LS_FACTOR_BETWEEN  error = Local(meas, T(key_a)^-1 * T(key_b)); fix_a != 0 freezes node a at fixed_a
 * whitened by sigma[6] ([translation x3; rotation x3], gtsam::noiseModel::Diagonal::Sigmas); robust != 0
 * wraps it in Robust(Cauchy(1)) (laser_track.cpp:37-64, incremental_estimator.cpp:29-48). */
#define LS_FACTOR_PRIOR 0
#define LS_FACTOR_BETWEEN 1

typedef struct ls_pg ls_pg;

typedef struct ls_factor {
  int32_t type;
  int32_t robust;
  int32_t fix_a;
  int32_t reserved;
  uint64_t key_a, key_b; /* prior: key_a (key_b ignored) */
  double meas[7];
  double sigma[6];
  double fixed_a[7];
} ls_factor;

typedef struct ls_pg_stats {
  int iterations, n_poses, n_factors, n_border; /* n_border = factors outside the per-track chains */
  double cost_first, cost_last;                 /* robust cost at the first / last linearisation point */
  double last_step_max;                         /* max |component| of the last update */
  float device_ms;
} ls_pg_stats;

int ls_pg_create(int device, ls_pg** out);
void ls_pg_destroy(ls_pg* pg);
const char* ls_pg_last_error(const ls_pg* pg);
uint64_t ls_pg_launch_count(const ls_pg* pg);
int ls_pg_num_poses(const ls_pg* pg);
int ls_pg_num_factors(const ls_pg* pg);
/* gtsam::Values::insert for new nodes; within one track_id the insertion order is the time order
 * (curves::DiscreteSE3Curve::extend, laser_track.cpp:573-582).  track_ids may be NULL (all track 0). */
int ls_pg_add_poses(ls_pg* pg, const uint64_t* keys, const uint32_t* track_ids, const double* poses7, int n);
int ls_pg_set_poses(ls_pg* pg, const uint64_t* keys, const double* poses7, int n);
/* isam2.update(newFactors, ...): out_indices (may be NULL) receives ISAM2Result::newFactorsIndices. */
int ls_pg_add_factors(ls_pg* pg, const ls_factor* factors, int n, uint64_t* out_indices);
/* isam2.update(..., removeFactorIndices) (incremental_estimator.cpp:258). */
int ls_pg_remove_factors(ls_pg* pg, const uint64_t* indices, int n);
/* gn_iters Gauss-Newton iterations over the whole graph on the device (3 = one estimate() call:
 * update(new) + update() + update(), incremental_estimator.cpp:156-159). */
int ls_pg_optimize(ls_pg* pg, int gn_iters, ls_pg_stats* stats);
/* gtsam::Marginals(graph, values).marginalCovariance(key) for each of keys[0..n)
 * (LaserTrack::updateCovariancesFromGTSAMValues, laser_slam/src/laser_track.cpp:421-429): the 6x6 block of the inverse
 * Gauss-Newton Hessian at the CURRENT estimate (robust factors at their current Cauchy weights), tangent order
 * [translation; rotation], row-major, 36 doubles per key. */
int ls_pg_marginals(ls_pg* pg, const uint64_t* keys, int n, double* out_cov36);
/* isam2.calculateEstimate(): all keys and poses (either pointer may be NULL); *n = number of poses. */
int ls_pg_get_poses(const ls_pg* pg, uint64_t* out_keys, double* out_poses7, int* n);

/* ---- multi-GPU -----------------------------------------------------------------------------------------
 * The path shards by independent tracks, one per GPU (the reference's n_laser_slam_workers LaserTracks,
 * laser_slam/src/incremental_estimator.cpp:22-26); the only exchange is one 32-byte record per rank per step
 * so that every rank can feed the shared estimator: a single ncclAllGather over NVLink.  NCCL is resolved at
 * run time (dlopen), so single-GPU users need no NCCL at all. */
typedef struct ls_comm ls_comm;

typedef struct ls_pose_record {
  float delta[6];  /* translation x3, rotation vector x3 of the step's T_a_b */
  int32_t status;  /* return code of the registration that produced it */
  int32_t key;     /* caller-defined (e.g. scan counter) */
} ls_pose_record;  /* 32 bytes */

int ls_comm_unique_id(void* id128);                       /* rank 0: ncclGetUniqueId -> 128 bytes to broadcast */
int ls_comm_init(int device, int rank, int nranks, const void* id128, ls_comm** out);
void ls_comm_destroy(ls_comm* comm);
const char* ls_comm_last_error(const ls_comm* comm);
/* all[nranks] <- every rank's record (rank order). */
int ls_comm_allgather_pose_records(ls_comm* comm, const ls_pose_record* mine, ls_pose_record* all);
/* The same in two halves: begin() only enqueues (copy in, ncclAllGather, copy out) on the communicator's stream
 * and returns; end() waits for it.  A track posts its step's record and collects it before posting the next one,
 * so the slowest rank of a step no longer stalls the others on the host (the estimator consumes the factors
 * asynchronously anyway, reference incremental_estimator.cpp:151-163).  One exchange in flight at a time
 * (LS_ERR_STATE otherwise). */
int ls_comm_allgather_pose_records_begin(ls_comm* comm, const ls_pose_record* mine);
int ls_comm_allgather_pose_records_end(ls_comm* comm, ls_pose_record* all);

#ifdef __cplusplus
}
#endif
#endif /* LS_B200_H_ */
