"""Reference of the occupancy map's change detection (test infrastructure only), restated twice from DESIGN.md
§4b'''''''''' in pure Python and numpy.  A map is a dict {packed key: np.float32 log-odds}; a voxel's state is
CELL_UNKNOWN when it is not in the dict, else CELL_OCCUPIED when v >= L_occ and CELL_FREE otherwise.
  EventLog  octomap's KeyBoolMap, updated at every leaf update: a voxel just created is set to True; a voxel whose
            occupied state flipped is added with False, or erased when it is there with False (True stays)
  diff      the voxels whose state differs between the baseline and now
Within one insert every voxel gets one update, and an edit's boxes apply in order, so the two agree (the tests check it).
"""
import numpy as np

CELL_FREE, CELL_OCCUPIED, CELL_UNKNOWN = 0, 1, 2
K0 = 32768


def state(vox, key, l_occ):
    v = vox.get(key)
    if v is None:
        return CELL_UNKNOWN
    return CELL_OCCUPIED if np.float32(v) >= np.float32(l_occ) else CELL_FREE


class EventLog:
    """octomap's change detection: {key: True (created since the reset) / False (occupied state flipped)}."""

    def __init__(self, l_occ):
        self.l_occ = np.float32(l_occ)
        self.changed = {}

    def update(self, key, before, after):
        """One leaf update of voxel `key` from log-odds `before` (None: the node is created) to `after`."""
        if before is None:
            self.changed[key] = True
        elif (np.float32(before) >= self.l_occ) != (np.float32(after) >= self.l_occ):
            self._flip(key)

    def apply(self, before_map, after_map):
        """Every update of one step in which each voxel of after_map that differs from before_map was updated once (an
        insert, read from the map before and after it)."""
        for k, v in after_map.items():
            b = before_map.get(k)
            if b is None or np.float32(b).view(np.uint32) != np.float32(v).view(np.uint32):
                self.update(k, b, v)

    def apply_arrays(self, before_keys, before_lo, after_keys, after_lo):
        """apply() on two downloads (ascending keys, float32 log-odds) of a step without deletions, as an insert is: the
        created voxels, then each voxel whose occupied state flipped, in key order (distinct voxels, so any order)."""
        pos = np.searchsorted(before_keys, after_keys)
        pos_c = np.minimum(pos, max(len(before_keys) - 1, 0))
        existed = (pos < len(before_keys)) & (np.asarray(before_keys)[pos_c] == after_keys) if len(before_keys) else \
            np.zeros(len(after_keys), bool)
        self.changed.update(dict.fromkeys(np.asarray(after_keys)[~existed].tolist(), True))
        was = np.asarray(before_lo, np.float32)[pos_c[existed]] >= self.l_occ
        flip = was != (np.asarray(after_lo, np.float32)[existed] >= self.l_occ)
        for k in np.asarray(after_keys)[existed][flip].tolist():
            self._flip(k)

    def _flip(self, key):
        if key not in self.changed:
            self.changed[key] = False
        elif self.changed[key] is False:
            del self.changed[key]

    def reset(self):
        self.changed.clear()

    def result(self, now):
        """(keys uint64, status int8, previous int8) by ascending key: True entries were unknown at the baseline, False
        entries had the other occupied state."""
        keys = sorted(self.changed)
        st = np.array([state(now, k, self.l_occ) for k in keys], np.int8)
        prev = np.array([CELL_UNKNOWN if self.changed[k] else 1 - s for k, s in zip(keys, st)], np.int8)
        return np.array(keys, np.uint64), st, prev

    def result_arrays(self, now_keys, now_lo):
        """result() with the map now as a download (ascending keys, float32 log-odds)."""
        keys = np.array(sorted(self.changed), np.uint64)
        pos = np.minimum(np.searchsorted(now_keys, keys), max(len(now_keys) - 1, 0))
        known = (np.asarray(now_keys)[pos] == keys) if len(now_keys) else np.zeros(len(keys), bool)
        st = np.where(known, np.where(np.asarray(now_lo, np.float32)[pos] >= self.l_occ, CELL_OCCUPIED, CELL_FREE),
                      CELL_UNKNOWN).astype(np.int8)
        created = np.array([self.changed[int(k)] for k in keys], bool)
        prev = np.where(created, CELL_UNKNOWN, 1 - st).astype(np.int8)
        return keys, st, prev


def diff(base, now, l_occ):
    """(keys uint64, status int8, previous int8) of every voxel whose state differs between the maps, by ascending key."""
    keys, st, prev = [], [], []
    for k in sorted(set(base) | set(now)):
        a, b = state(base, k, l_occ), state(now, k, l_occ)
        if a != b:
            keys.append(k), st.append(b), prev.append(a)
    return np.array(keys, np.uint64), np.array(st, np.int8), np.array(prev, np.int8)


def diff_arrays(base_keys, base_lo, now_keys, now_lo, l_occ):
    """diff() of two downloads (ascending keys and float32 log-odds each), vectorised."""
    l_occ = np.float32(l_occ)
    keys = np.union1d(base_keys, now_keys).astype(np.uint64)
    sb = np.full(len(keys), CELL_UNKNOWN, np.int8)
    sn = np.full(len(keys), CELL_UNKNOWN, np.int8)
    sb[np.searchsorted(keys, base_keys)] = np.where(np.asarray(base_lo, np.float32) >= l_occ, CELL_OCCUPIED, CELL_FREE)
    sn[np.searchsorted(keys, now_keys)] = np.where(np.asarray(now_lo, np.float32) >= l_occ, CELL_OCCUPIED, CELL_FREE)
    d = sb != sn
    return keys[d], sn[d], sb[d]


def centres(keys, status, res_now, res_base):
    """{x, y, z, 1} per changed voxel, (n,4) float32: (float)(((double)(k - 32768) + 0.5) * res) per axis, res the map's
    resolution now for a voxel known now and the baseline's for one unknown now."""
    keys = np.asarray(keys, np.uint64)
    res = np.where(np.asarray(status) == CELL_UNKNOWN, float(res_base), float(res_now))
    out = np.ones((len(keys), 4), np.float32)
    for a in range(3):
        k = ((keys >> np.uint64(16 * a)) & np.uint64(0xFFFF)).astype(np.float64)
        out[:, a] = (((k - K0) + 0.5) * res).astype(np.float32)
    return out


def as_dict(keys, log_odds):
    return {int(k): np.float32(v) for k, v in zip(keys, log_odds)}
