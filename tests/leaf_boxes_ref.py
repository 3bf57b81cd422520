"""Reference of the leaf boxes and marker cubes (test infrastructure only; DESIGN.md §4b'''''''''''').  walk() lists
the leaves of a .ot payload (octomap's writeData bytes) in pre-order, as octomap's leaf iterator visits the tree in
memory; the region rule and generateMarkerArray's height colour are restated in scalar Python."""
import math

import numpy as np

CELL_FREE, CELL_OCCUPIED = 0, 1


def walk(payload):
    """Every leaf of a .ot payload in pre-order (children 0..7): first-voxel keys (n,3) int64, depths uint8 and log-odds
    float32."""
    keys, depths, values = [], [], []
    view = memoryview(bytes(payload))
    pos = 0
    stack = [(0, 0, 0, 0)] if len(view) else []
    while stack:
        d, kx, ky, kz = stack.pop()
        v = np.frombuffer(view[pos:pos + 4], "<f4")[0]
        m = view[pos + 4]
        pos += 5
        if not m:
            keys.append((kx, ky, kz))
            depths.append(d)
            values.append(v)
            continue
        sh = 15 - d
        for i in range(7, -1, -1):  # pushed 7 ... 0, so popped in child order
            if (m >> i) & 1:
                stack.append((d + 1, kx | ((i & 1) << sh), ky | (((i >> 1) & 1) << sh), kz | (((i >> 2) & 1) << sh)))
    assert pos == len(view), "bytes after the tree"
    return (np.array(keys, np.int64).reshape(-1, 3), np.array(depths, np.uint8), np.array(values, np.float32))


def key_to_coord(k, depth, res):
    """octomap's keyToCoord(key, depth) of one axis, as a float."""
    s = 16 - depth
    kc = k + ((1 << (s - 1)) if s > 0 else 0)
    scale = float(1 << s)
    return np.float32((math.floor((kc - 32768.0) / scale) + 0.5) * (res * scale))


def leaves(payload, res, l_occ):
    """The leaf boxes of a .ot payload: dict of keys (n,3), depths, values, centres (n,3) float32, states int8 (occupied iff
    value >= l_occ) and edges float64, in leaf order."""
    keys, depths, values = walk(payload)
    cen = np.array([[key_to_coord(int(k[a]), int(d), res) for a in range(3)] for k, d in zip(keys, depths)],
                   np.float32).reshape(-1, 3)
    states = np.where(values >= np.float32(l_occ), CELL_OCCUPIED, CELL_FREE).astype(np.int8)
    edges = np.array([res * 2.0 ** (16 - int(d)) for d in depths], np.float64)
    return dict(keys=keys, depths=depths, values=values, centres=cen, states=states, edges=edges)


def corner_key(c, res):
    """The key of a region corner: floor(c * (1/res)) + 32768 in double, clamped to [0, 65535]."""
    k = math.floor(c * (1.0 / res)) + 32768
    return min(max(k, 0), 65535)


def meets(k0, depth, kmin, kmax):
    """Whether the key cube [k0, k0 + 2^(16-depth)) meets [kmin, kmax] on every axis."""
    side = 1 << (16 - depth)
    return all(k0[a] <= kmax[a] and k0[a] + side - 1 >= kmin[a] for a in range(3))


def select(lv, region, res):
    """The leaves of `lv` (leaves()'s dict) a region (min (3,), max (3,)) in metres lists; region None: all."""
    if region is None:
        return dict(lv)
    kmin = [corner_key(float(region[0][a]), res) for a in range(3)]
    kmax = [corner_key(float(region[1][a]), res) for a in range(3)]
    keep = np.array([meets([int(x) for x in k], int(d), kmin, kmax) for k, d in zip(lv["keys"], lv["depths"])], bool)
    return {name: a[keep] if len(keep) else a[:0] for name, a in lv.items()}


def height_map_color(h):
    """octomap_server's heightMapColor(h): (r, g, b, a) as float32, computed in double."""
    s = v = 1.0
    h -= math.floor(h)
    h *= 6
    i = math.floor(h)
    f = h - i
    if not (i & 1):
        f = 1 - f
    m = v * (1 - s)
    n = v * (1 - s * f)
    rgb = {0: (v, n, m), 6: (v, n, m), 1: (n, v, m), 2: (m, v, n), 3: (m, n, v), 4: (n, m, v), 5: (v, m, n)}.get(i, (1, .5, .5))
    return tuple(np.float32(x) for x in rgb) + (np.float32(1.0),)


def cube_color(z, min_z, max_z, color_factor):
    """generateMarkerArray's colour of an occupied cube whose float centre has height z."""
    x = (float(np.float32(z)) - min_z) / (max_z - min_z)
    x = 0.0 if x < 0.0 else x  # std::max(x, 0.0)
    x = 1.0 if 1.0 < x else x  # std::min(x, 1.0)
    return height_map_color((1.0 - x) * color_factor)


def marker_cubes(lv, min_z, max_z, color_factor):
    """generateMarkerArray of the leaves `lv`: per state ("occupied", "free") 17 lists (depth 0..16) of leaf indices in leaf
    order, and the colours (n_occupied, 4) float32 of the occupied cubes in cube order."""
    out = {"occupied": [[] for _ in range(17)], "free": [[] for _ in range(17)]}
    for i, (d, s) in enumerate(zip(lv["depths"], lv["states"])):
        out["occupied" if s == CELL_OCCUPIED else "free"][int(d)].append(i)
    colors = [cube_color(lv["centres"][i][2], min_z, max_z, color_factor) for lst in out["occupied"] for i in lst]
    return out, np.array(colors, np.float32).reshape(-1, 4)
