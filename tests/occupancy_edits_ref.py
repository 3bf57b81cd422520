"""Reference of the occupancy map's edits (test infrastructure only): volumetric_mapping's setLogOddsBoundingBox, resetMap,
getOccupiedPointcloudInBoundingBox and the map's extent restated in pure Python and numpy from DESIGN.md §4b''''''''.
Python floats are IEEE doubles and np.float32 is the float cast, so every step rounds as the device's does.  A map is a
dict {packed key: np.float32 log-odds}."""
import math

import numpy as np

K0 = 32768
MAX_AXIS_POINTS = 1 << 17


def key_of(x, res):
    """OCCUPANCY.md's key of the float coordinate x: floor(x * (1/res)) + 32768, None when outside [0, 65535]."""
    f = math.floor(float(x) * (1.0 / res))
    return f + K0 if -K0 <= f < K0 else None


def axis_points(p, s, res):
    """One axis of the box loop around p of size s: its points (doubles), in loop order."""
    c = res * math.floor(p / res) + res / 2.0
    lo, hi = (c - s / 2) + 0.001, (c + s / 2) - 0.001
    out = []
    x = lo
    while x <= hi:
        if len(out) == MAX_AXIS_POINTS:
            raise ValueError("more than 2^17 loop points on an axis")
        out.append(x)
        x += res
    return out


def axis_keys(p, s, res):
    """The valid keys of one axis's points, each cast to float first, in loop order (ascending, repeats kept)."""
    ks = (key_of(np.float32(x), res) for x in axis_points(p, s, res))
    return [k for k in ks if k is not None]


def pack(kx, ky, kz):
    return kx | (ky << 16) | (kz << 32)


def box_keys(center, size, res):
    """The packed key of every loop point of the box with a valid key: x outer, z inner (the separable loop)."""
    ax = [axis_keys(center[a], size[a], res) for a in range(3)]
    return [pack(x, y, z) for x in ax[0] for y in ax[1] for z in ax[2]]


class Edits:
    """The edits at one resolution and sensor model on a map {packed key: float32}."""

    def __init__(self, res, l_min, l_max, l_occ):
        self.res, self.l_min, self.l_max, self.l_occ = res, np.float32(l_min), np.float32(l_max), np.float32(l_occ)

    def set_boxes(self, vox, centres, sizes, occupied):
        """setFree / setOccupied of each box in order on `vox` (changed in place): the last box covering a voxel decides.
        Returns the loop points set and the voxels that became known."""
        set_n, before = 0, len(vox)
        for c, s, o in zip(centres, sizes, occupied):
            v = self.l_max if o else self.l_min
            for k in box_keys(c, s, self.res):
                vox[k] = v
                set_n += 1
        return set_n, len(vox) - before

    def reset(self, vox):
        """resetMap."""
        vox.clear()

    def crop(self, vox, center, size, which_occupied=True):
        """(keys uint64, log-odds float32, centres (n,4) float32) per loop point whose voxel is occupied (or known)."""
        ks = [k for k in box_keys(center, size, self.res) if k in vox and (not which_occupied or vox[k] >= self.l_occ)]
        keys = np.array(ks, np.uint64)
        lo = np.array([vox[k] for k in ks], np.float32)
        return keys, lo, centres(keys, self.res)

    def bounds(self, vox):
        """(min (3,), max (3,)) as doubles: calcMinMax over depth-16 leaves of the known keys; zeros when empty."""
        if not vox:
            return np.zeros(3), np.zeros(3)
        k = np.array(list(vox), np.uint64)
        lo, hi = np.zeros(3), np.zeros(3)
        for a in range(3):
            ka = (k >> np.uint64(16 * a)) & np.uint64(0xFFFF)
            lo[a] = float(centre(int(ka.min()), self.res)) - self.res / 2.0
            hi[a] = (float(centre(int(ka.max()), self.res)) - self.res / 2.0) + self.res
        return lo, hi


def centre(k, res):
    """octomap's keyToCoord: (float)((k - 32768 + 0.5) * res)."""
    return np.float32(((k - K0) + 0.5) * res)


def centres(keys, res):
    """{x, y, z, 1} voxel centres of packed keys, (n,4) float32."""
    keys = np.asarray(keys, np.uint64)
    out = np.ones((len(keys), 4), np.float32)
    for a in range(3):
        k = ((keys >> np.uint64(16 * a)) & np.uint64(0xFFFF)).astype(np.float64)
        out[:, a] = (((k - K0) + 0.5) * res).astype(np.float32)
    return out


def as_arrays(vox):
    """(ascending packed keys uint64, float32 log-odds) of a map."""
    keys = np.array(sorted(vox), np.uint64)
    return keys, np.array([vox[int(k)] for k in keys], np.float32)


def as_dict(keys, log_odds):
    return {int(k): np.float32(v) for k, v in zip(keys, log_odds)}
