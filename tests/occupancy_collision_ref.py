"""Reference of the occupancy map's box status and robot collision (test infrastructure only): volumetric_mapping's
getCellStatusBoundingBox, checkSinglePoseCollision and checkPathForCollisionsWithRobot restated from DESIGN.md
§4b'''''''''''.  Python floats are IEEE doubles and np.float32 is the float cast, so every step rounds as the device's does.
Two restatements: `box_status` follows steps 1-6 literally over a dict map {packed key: np.float32 log-odds}; `BoxGrid`
answers the same rule over a dense grid of the map's states, for many boxes."""
import math

import numpy as np

K0 = 32768
MAX_AXIS_POINTS = 1 << 17
CELL_FREE, CELL_OCCUPIED, CELL_UNKNOWN = 0, 1, 2
F32 = np.float32


class Refused(ValueError):
    """The call is refused (LS_ERR_ARG)."""


def key_d(x, res):
    """The double rule (octomap's search(x, y, z)): floor(x * (1/res)) + 32768, None when outside [0, 65535] or NaN."""
    f = float(x) * (1.0 / res)
    if not (f == f) or math.isinf(f):
        return None
    f = math.floor(f)
    return f + K0 if -K0 <= f < K0 else None


def key_f(x, res):
    """The float rule: the key of (float)x."""
    return key_d(float(F32(x)), res)


def pack(kx, ky, kz):
    return kx | (ky << 16) | (kz << 32)


def state(vox, k, l_occ):
    v = vox.get(k)
    if v is None:
        return CELL_UNKNOWN
    return CELL_OCCUPIED if v >= F32(l_occ) else CELL_FREE


def check_size(size):
    for s in size:
        if not (s >= 0.0) or math.isinf(s):
            raise Refused("a size is negative or not finite")


def corners(p, s):
    """Step 3 on one axis: (float)(p - s/2), (float)(p + s/2)."""
    return F32(p - s / 2), F32(p + s / 2)


def loop_points(lo, hi, res):
    """Step 5 on one axis: x = lo; x <= hi; x += res in double.  Refused past 2^17 points."""
    out = []
    x = float(lo)
    while x <= float(hi):
        if len(out) == MAX_AXIS_POINTS:
            raise Refused("more than 2^17 loop points on an axis")
        out.append(x)
        x += res
    return out


MAX_WORK = 1 << 36  # (box, brick) items per call


def axis_bricks(p, s, res):
    """The 8-voxel bricks one axis of a box spans: those of its loop's valid keys and, when both corner keys are valid, of
    the keys passing the cube test.  The call's work is the sum over boxes with a valid centre of the product over axes."""
    lo, hi = corners(p, s)
    keys = [k for k in (key_f(x, res) for x in loop_points(lo, hi, res)) if k is not None]
    kmin, kmax = key_f(lo, res), key_f(hi, res)
    if kmin is not None and kmax is not None:
        keys += [k for k in range(kmin, kmax + 1) if cube_passes(k, lo, hi, res)]
    return (max(keys) >> 3) - (min(keys) >> 3) + 1 if keys else 0


def work_items(centre, size, res):
    if None in [key_d(c, res) for c in centre]:
        return 0
    return int(np.prod([axis_bricks(float(centre[a]), float(size[a]), res) for a in range(3)]))


def check_call(centres, sizes, res):
    """The refusals of a whole call (Refused): a bad size, an axis of more than 2^17 loop points, more than 2^36 items."""
    work, seen = 0, {}
    for c, s in zip(centres, sizes):
        check_size([float(x) for x in s])
        key = (tuple(float(x) for x in c), tuple(float(x) for x in s))
        if key not in seen:  # repeated boxes are counted once and added each time
            seen[key] = work_items(c, s, res)
        work += seen[key]
    if work > MAX_WORK:
        raise Refused("more than 2^36 (box, brick) items")
    return work


def cube_passes(k, lo, hi, res):
    """Step 4's test of key k on one axis: the cube c +- res/2 is not wholly outside [lo, hi]."""
    c = (float(k - K0) + 0.5) * res
    return not (c + res / 2 < float(lo) or c - res / 2 > float(hi))


def box_status(vox, centre, size, res, l_occ, order=None):
    """Steps 1-6 for one box.  order: None, "reverse" or a numpy Generator: the order the keys and points are visited
    (the result must not depend on it)."""
    centre = [float(c) for c in centre]
    size = [float(s) for s in size]
    check_size(size)
    kd = [key_d(c, res) for c in centre]
    if None in kd:
        return CELL_UNKNOWN  # step 1: an invalid key is unknown (no refusal for such a box)
    bmin, bmax = zip(*(corners(centre[a], size[a]) for a in range(3)))
    pts = [loop_points(bmin[a], bmax[a], res) for a in range(3)]  # counted before any result: refusals first
    st = state(vox, pack(*kd), l_occ)
    if st != CELL_FREE:
        return st
    if None in [key_f(c, res) for c in centre]:
        return CELL_UNKNOWN  # step 2
    visit = _order(order)
    kmin, kmax = [key_f(x, res) for x in bmin], [key_f(x, res) for x in bmax]
    if None not in kmin and None not in kmax:  # step 4; the cube test is per axis, so each axis's verdicts once
        keys = [[(k, cube_passes(k, bmin[a], bmax[a], res)) for k in range(kmin[a], kmax[a] + 1)] for a in range(3)]
        for kx, px in visit(keys[0]):
            for ky, py in visit(keys[1]):
                for kz, pz in visit(keys[2]):
                    if px and py and pz and state(vox, pack(kx, ky, kz), l_occ) == CELL_OCCUPIED:
                        return CELL_OCCUPIED
    keys = [[key_f(x, res) for x in pts[a]] for a in range(3)]  # step 5, each point cast to float and keyed
    for kx in visit(keys[0]):
        for ky in visit(keys[1]):
            for kz in visit(keys[2]):
                if kx is None or ky is None or kz is None or pack(kx, ky, kz) not in vox:
                    return CELL_UNKNOWN
    return CELL_FREE


def _order(order):
    if order is None:
        return lambda xs: xs
    if order == "reverse":
        return lambda xs: list(reversed(xs))
    return lambda xs: [xs[i] for i in order.permutation(len(xs))]


def collides(status, unknown_as_occupied):
    """checkSinglePoseCollision."""
    return status != CELL_FREE if unknown_as_occupied else status == CELL_OCCUPIED


def first_collisions(statuses, offsets, unknown_as_occupied):
    """Per path (offsets into the poses' statuses): the first colliding pose's index within the path, or -1."""
    hit = np.array([collides(int(s), unknown_as_occupied) for s in statuses], bool)
    out = np.full(len(offsets) - 1, -1, np.int64)
    for p in range(len(offsets) - 1):
        idx = np.flatnonzero(hit[offsets[p]:offsets[p + 1]])
        if len(idx):
            out[p] = idx[0]
    return out


def check_paths(vox, positions, offsets, robot_size, res, l_occ, unknown_as_occupied):
    st = [box_status(vox, p, robot_size, res, l_occ) for p in positions]
    return first_collisions(st, offsets, unknown_as_occupied)


class BoxGrid:
    """The rule over a dense grid of states: keys lo ... lo + shape - 1 per axis (np.int64 (3,)), every voxel outside the
    grid unknown.  Per box the passes are numpy slices and gathers over the grid, so the grid must cover every key a
    box's passes can reach (see `covering`)."""

    def __init__(self, keys, log_odds, l_occ, lo, shape):
        self.lo = np.asarray(lo, np.int64)
        self.shape = tuple(int(x) for x in shape)
        self.known = np.zeros(self.shape, bool)
        self.occ = np.zeros(self.shape, bool)
        keys = np.asarray(keys, np.uint64)
        k = np.stack([(keys >> np.uint64(16 * a)) & np.uint64(0xffff) for a in range(3)], 1).astype(np.int64) - self.lo
        inside = ((k >= 0) & (k < np.array(self.shape))).all(1)
        k = k[inside]
        self.known[k[:, 0], k[:, 1], k[:, 2]] = True
        self.occ[k[:, 0], k[:, 1], k[:, 2]] = np.asarray(log_odds, F32)[inside] >= F32(l_occ)

    @staticmethod
    def covering(centres, sizes, res, margin=2):
        """(lo, shape) of a grid holding every corner key of the boxes (finite centres), plus a margin."""
        c = np.asarray(centres, np.float64).reshape(-1, 3)
        s = np.broadcast_to(np.asarray(sizes, np.float64).reshape(-1, 3), c.shape)
        with np.errstate(invalid="ignore"):
            f = np.floor(c * (1.0 / res))
            ok = ((f >= -K0) & (f < K0)).all(1)  # a centre with an invalid key is unknown without a pass
        lo = np.floor((c[ok] - s[ok] / 2).astype(F32).astype(np.float64) * (1.0 / res)) + K0 - margin
        hi = np.floor((c[ok] + s[ok] / 2).astype(F32).astype(np.float64) * (1.0 / res)) + K0 + margin
        lo = np.clip(lo.min(0), 0, 65535).astype(np.int64)
        hi = np.clip(hi.max(0), 0, 65535).astype(np.int64)
        return lo, hi - lo + 1

    def _state(self, k):
        g = np.asarray(k, np.int64) - self.lo
        if ((g < 0) | (g >= np.array(self.shape))).any():
            return CELL_UNKNOWN
        if not self.known[tuple(g)]:
            return CELL_UNKNOWN
        return CELL_OCCUPIED if self.occ[tuple(g)] else CELL_FREE

    def status(self, centre, size, res):
        centre = [float(c) for c in centre]
        size = [float(s) for s in size]
        check_size(size)
        kd = [key_d(c, res) for c in centre]
        if None in kd:
            return CELL_UNKNOWN
        bmin, bmax = zip(*(corners(centre[a], size[a]) for a in range(3)))
        loop = []
        for a in range(3):  # the loop's keys as an array (the float rule), -1 for an invalid point
            x = np.array(loop_points(bmin[a], bmax[a], res), np.float64)
            f = np.floor(x.astype(F32).astype(np.float64) * (1.0 / res))
            loop.append(np.where((f >= -K0) & (f < K0), f + K0, -1).astype(np.int64))
        st = self._state(kd)
        if st != CELL_FREE:
            return st
        if None in [key_f(c, res) for c in centre]:
            return CELL_UNKNOWN
        kmin, kmax = [key_f(x, res) for x in bmin], [key_f(x, res) for x in bmax]
        if None not in kmin and None not in kmax:
            sl = []
            for a in range(3):
                q = np.arange(kmin[a], kmax[a] + 1, dtype=np.int64)
                c = ((q - K0).astype(np.float64) + 0.5) * res
                q = q[~((c + res / 2 < float(bmin[a])) | (c - res / 2 > float(bmax[a])))]
                sl.append(q[(q >= self.lo[a]) & (q < self.lo[a] + self.shape[a])] - self.lo[a])
            if all(len(x) for x in sl) and self.occ[np.ix_(*sl)].any():
                return CELL_OCCUPIED
        for a in range(3):
            if (loop[a] < 0).any() or (loop[a] < self.lo[a]).any() or (loop[a] >= self.lo[a] + self.shape[a]).any():
                return CELL_UNKNOWN  # an invalid point, or a voxel outside the grid
        g = [np.unique(loop[a]) - self.lo[a] for a in range(3)]
        return CELL_UNKNOWN if not self.known[np.ix_(*g)].all() else CELL_FREE

    def statuses(self, centres, sizes, res):
        c = np.asarray(centres, np.float64).reshape(-1, 3)
        s = np.broadcast_to(np.asarray(sizes, np.float64).reshape(-1, 3), c.shape)
        return np.array([self.status(c[i], s[i], res) for i in range(len(c))], np.int8)


def as_dict(keys, log_odds):
    return {int(k): F32(v) for k, v in zip(np.asarray(keys, np.uint64), np.asarray(log_odds, F32))}
