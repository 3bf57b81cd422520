"""Reference of the 2D projection (test infrastructure only; DESIGN.md §4b''''''''''''').  bt_leaves() walks a .bt payload
(octomap's writeBinary bytes) in pre-order, as octomap_server's iterator visits the tree it loads; project() restates
handlePreNodeTraversal and update2DMap at m_maxTreeDepth = 16 with a complete projection, elementwise over the leaves."""
import math

import numpy as np


def bt_leaves(payload):
    """Every leaf of a .bt payload in pre-order (children 0..7): first-voxel keys (n,3) int64, depths uint8 and occupied
    bool."""
    keys, depths, occ = [], [], []
    pos = 0
    stack = [(3, 0, 0, 0, 0)] if len(payload) else []  # bit pair, depth, first-voxel key
    while stack:
        bits, d, kx, ky, kz = stack.pop()
        if bits != 3:
            keys.append((kx, ky, kz))
            depths.append(d)
            occ.append(bits == 2)
            continue
        m = payload[pos] | (payload[pos + 1] << 8)
        pos += 2
        sh = 15 - d
        for i in range(7, -1, -1):
            b = (m >> (2 * i)) & 3
            if b:
                stack.append((b, d + 1, kx | ((i & 1) << sh), ky | (((i >> 1) & 1) << sh), kz | (((i >> 2) & 1) << sh)))
    assert pos == len(payload), "bytes after the tree"
    return np.array(keys, np.int64).reshape(-1, 3), np.array(depths, np.uint8), np.array(occ, bool)


def key_to_coord(k, depth):
    """octomap's keyToCoord(key, depth) of one axis in double, before the resolution: (floor(...) + 0.5) * 2^(16-d)."""
    s = 16 - depth
    kc = k + ((1 << (s - 1)) if s > 0 else 0)
    scale = float(1 << s)
    return math.floor((kc - 32768.0) / scale) + 0.5, scale


def centre(k, depth, res):
    c, scale = key_to_coord(k, depth)
    return c * (res * scale)


def coord_key_checked(c, res):
    """octomap's coordToKeyChecked of a double coordinate: floor(c * (1/res)) + 32768, None outside [0, 65535]."""
    s = math.floor(c * (1.0 / res)) if math.isfinite(c * (1.0 / res)) else None
    if s is None or not (-32768 <= s < 32768):
        return None
    return s + 32768


class Refused(ValueError):
    pass


def project(leaves, res, min_z=-math.inf, max_z=math.inf, min_size_x=0.0, min_size_y=0.0):
    """octomap_server's projected map of .bt leaves (bt_leaves()'s triple): (grid int8 (height, width), info dict of
    width, height, resolution, origin_x, origin_y and unknown / free / occupied cell counts).  Raises Refused where the
    device call returns LS_ERR_ARG."""
    if math.isnan(min_z) or math.isnan(max_z):
        raise Refused("NaN band")
    for s in (min_size_x, min_size_y):
        if not math.isfinite(s) or s < 0.0:
            raise Refused("bad minimum size")
    keys, depths, occ = leaves
    if len(depths) == 0:
        return np.zeros((0, 0), np.int8), dict(width=0, height=0, resolution=res, origin_x=0.0, origin_y=0.0,
                                               unknown=0, free=0, occupied=0)
    # calcMinMax over the leaves, in double (elementwise, each operation as the scalar centre() rounds it)
    k = np.asarray(keys, np.int64)
    s = 16 - np.asarray(depths, np.int64)
    scale = np.left_shift(1, s).astype(np.float64)
    kc = k + np.where(s > 0, np.left_shift(1, np.maximum(s - 1, 0)), 0)[:, None]
    c = (np.floor((kc.astype(np.float64) - 32768.0) / scale[:, None]) + 0.5) * (res * scale)[:, None]
    size = res * scale
    half = size / 2.0
    low = c - half[:, None]
    lo = [float(low[:, a].min()) for a in range(3)]
    hi = [float((low[:, a] + size).max()) for a in range(3)]
    # padding (std::min(a, b) is b < a ? b : a), then the corners as float points, keyed
    hx, hy = 0.5 * min_size_x, 0.5 * min_size_y
    pmin = [-hx if -hx < lo[0] else lo[0], -hy if -hy < lo[1] else lo[1], lo[2]]
    pmax = [hx if hi[0] < hx else hi[0], hy if hi[1] < hy else hi[1], hi[2]]
    kmin = [coord_key_checked(float(np.float32(x)), res) for x in pmin]
    kmax = [coord_key_checked(float(np.float32(x)), res) for x in pmax]
    if None in kmin or None in kmax:
        raise Refused("padded corner outside the key space")
    width, height = kmax[0] - kmin[0] + 1, kmax[1] - kmin[1] + 1
    if width * height > 0x7fffffff:
        raise Refused("more than 2^31 - 1 cells")
    # the band, then update2DMap: free leaves first, then occupied ones, so occupied wins and free fills only unknown cells
    z = c[:, 2]
    take = (z + half > min_z) & (z - half < max_z)
    grid = np.full((height, width), -1, np.int8)
    x0, y0 = k[:, 0] - kmin[0], k[:, 1] - kmin[1]
    occ = np.asarray(occ, bool)
    for value, sel in ((0, take & ~occ), (100, take & occ)):
        for side in np.unique(s[sel]):
            m = sel & (s == side)
            n = 1 << int(side)
            if n <= 64:  # every cell of every such leaf at once
                off = np.arange(n)
                ys = (y0[m][:, None, None] + off[None, :, None]).repeat(n, 2).ravel()
                xs = (x0[m][:, None, None] + off[None, None, :]).repeat(n, 1).ravel()
                grid[ys, xs] = np.maximum(grid[ys, xs], value)
            else:
                for a, b in zip(x0[m], y0[m]):
                    cells = grid[b:b + n, a:a + n]
                    np.maximum(cells, value, out=cells)
    ox = float(np.float32(centre(kmin[0], 16, res))) - res * 0.5
    oy = float(np.float32(centre(kmin[1], 16, res))) - res * 0.5
    return grid, dict(width=width, height=height, resolution=res, origin_x=ox, origin_y=oy,
                      unknown=int((grid == -1).sum()), free=int((grid == 0).sum()), occupied=int((grid == 100).sum()))


def per_voxel(keys, occupied, res, min_z, max_z, kmin_xy, shape):
    """An independent projection for the checks: every known voxel (keys (n,3), occupied bool) whose z extent meets the
    band marks its column, occupied over free, on a grid whose cell (0, 0) is key kmin_xy."""
    grid = np.full(shape, -1, np.int8)
    k = np.asarray(keys, np.int64).reshape(-1, 3)
    z = ((k[:, 2] - 32768).astype(np.float64) + 0.5) * res
    band = (z + res / 2.0 > min_z) & (z - res / 2.0 < max_z)
    x, y = k[:, 0] - kmin_xy[0], k[:, 1] - kmin_xy[1]
    f = band & ~np.asarray(occupied, bool)
    grid[y[f], x[f]] = 0
    o = band & np.asarray(occupied, bool)
    grid[y[o], x[o]] = 100
    return grid


def map_saver_bytes(grid, resolution, origin_x, origin_y, image):
    """map_saver's two files of a grid, derived from its fprintf / fputc calls: (.pgm bytes, .yaml text)."""
    res = float(np.float32(resolution))
    height, width = grid.shape
    head = ("P5\n# CREATOR: map_saver.cpp %.3f m/pix\n%d %d\n255\n" % (res, width, height)).encode()
    body = bytearray()
    for y in range(height):
        for x in range(width):
            v = int(grid[height - y - 1, x])
            body.append(254 if v == 0 else 0 if v == 100 else 205)
    yaml = ("image: %s\nresolution: %f\norigin: [%f, %f, %f]\nnegate: 0\noccupied_thresh: 0.65\nfree_thresh: 0.196\n\n"
            % (image, res, origin_x, origin_y, 0.0))
    return head + bytes(body), yaml
