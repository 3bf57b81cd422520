"""ORACLE -- test infrastructure only.  Restatement of LaserSlamWorker's local-map maintenance (reference
laser_slam_ros/src/laser_slam_worker.cpp) without ROS: the rules of ls_local_map_* (include/ls_b200.h), stated in
oracle/LOCAL_MAP.md, on top of the oracle's filter_cylinder, voxel_grid rule and float32 transforms."""
import numpy as np

import oracle

HEIGHT_M = 40.0   # getFilteredMap's cylinder height, hard-coded in the reference (:428-429, :459-463)


def _empty():
    return np.zeros((0, 4), np.float32)


def voxel_grid(pts4, leaf_size, min_points=0):
    """oracle.voxel_grid (float32 floor(p * (1/leaf)), 64-bit cell index, ascending cells, exact fixed-point centroid rounded
    once) with pcl::VoxelGrid's minimum point number per voxel [upstream]: a voxel is kept iff it holds at least
    `min_points` points; 0 and 1 keep every voxel, so oracle.voxel_grid's output is returned as it is."""
    out = oracle.voxel_grid(pts4, leaf_size)
    if min_points <= 1 or len(out) == 0:
        return out
    # the points per voxel, in the same ascending cell order as oracle.voxel_grid's output
    p = np.asarray(pts4, np.float32).reshape(-1, 4)
    inv = (np.float32(1.0) / np.broadcast_to(np.asarray(leaf_size, np.float32), (3,))).astype(np.float32)
    ijk = np.floor(p[np.isfinite(p[:, :3]).all(1), :3] * inv[None, :]).astype(np.int64)
    dim = ijk.max(0) - ijk.min(0) + 1
    c = ijk - ijk.min(0)
    _, cnt = np.unique(c[:, 0] + c[:, 1] * dim[0] + c[:, 2] * dim[0] * dim[1], return_counts=True)
    return out[cnt >= min_points].copy()


def transform_points(T, pts4):
    """updateLocalMap's move: the xform_point order, no identity shortcut (pcl::transformPointCloud moves every point)."""
    p = np.asarray(pts4, np.float32).reshape(-1, 4)
    return oracle.transform_points(T, p) if len(p) else _empty()


class LocalMap:
    """local_map_, local_map_filtered_, distant_map_ and local_map_queue_ of LaserSlamWorker with the methods that change
    them (scanCallback's map part, getFilteredMap, updateLocalMap, clearLocalMap, getQueuedPoints)."""

    def __init__(self, distance_to_consider_fixed=20.0, separate_distant_map=True, voxel_size_m=0.1,
                 minimum_point_number_per_voxel=0, remove_ground_from_local_map=False, ground_distance_to_robot_center_m=1.0):
        self.distance_to_consider_fixed = float(distance_to_consider_fixed)
        self.separate_distant_map = bool(separate_distant_map)
        self.voxel_size_m = float(voxel_size_m)
        self.minimum_point_number_per_voxel = int(minimum_point_number_per_voxel)
        self.remove_ground_from_local_map = bool(remove_ground_from_local_map)
        self.ground_distance_to_robot_center_m = float(ground_distance_to_robot_center_m)
        self.local_map = _empty()
        self.local_map_filtered = _empty()
        self.distant_map = _empty()
        self.queue = []

    def add_scan(self, scan4, T_w_scan, robot_z):
        """scanCallback (:195-246): the scan in the world frame (float32, an exact identity copies it), ground points
        ((double)z <= robot_z - ground distance) removed, appended and queued unless nothing is left.  Returns the count."""
        cloud = oracle._xform_points(T_w_scan, np.asarray(scan4, np.float32).reshape(-1, 4))
        if self.remove_ground_from_local_map:
            z_min = float(robot_z) - self.ground_distance_to_robot_center_m
            cloud = cloud[cloud[:, 2].astype(np.float64) > z_min]
        if len(cloud) == 0:
            return 0
        self.local_map = np.concatenate([self.local_map, cloud])
        self.queue.append(cloud.copy())
        return len(cloud)

    def get_filtered_map(self, center):
        """getFilteredMap (:415-488).  `center` is rounded to float32 (the reference stores it in a PclPoint)."""
        c = np.asarray(center, np.float32).astype(np.float64)
        r = self.distance_to_consider_fixed
        snapshot = self.local_map
        self.local_map = oracle.filter_cylinder(snapshot, c, r, HEIGHT_M)
        if not self.separate_distant_map:
            return snapshot.copy()
        v = voxel_grid(snapshot, self.voxel_size_m, self.minimum_point_number_per_voxel)
        self.local_map_filtered = oracle.filter_cylinder(v, c, r, HEIGHT_M)
        self.distant_map = np.concatenate([self.distant_map, oracle.filter_cylinder(v, c, r, HEIGHT_M, remove_points_inside=True)])
        return np.concatenate([self.local_map_filtered, self.distant_map])

    def update_local_map(self, T):
        """updateLocalMap (:522-540): local_map_ and local_map_filtered_ moved by T; distant_map_ and the queue are not."""
        self.local_map = transform_points(T, self.local_map)
        self.local_map_filtered = transform_points(T, self.local_map_filtered)

    def clear_local_map(self):
        """clearLocalMap (:496-506): distant_map_ and the queue stay."""
        self.local_map = _empty()
        self.local_map_filtered = _empty()

    def get_queued_points(self):
        """getQueuedPoints (:407-412): the queue, swapped out."""
        q, self.queue = self.queue, []
        return q
