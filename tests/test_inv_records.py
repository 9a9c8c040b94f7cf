"""Host logic of the packed inverse lists (no GPU): the 16-byte records + overflow array the small-map lidar reads
(rlca_inv_records_host, the same code rlca_env_set_map runs) hold exactly the lists of inv_off / inv_ent, entry for
entry and in the same order, for every relative cell."""
import ctypes as C

import numpy as np
import pytest

from test_walk_tables import _tables


def _records(range_cells):
    from rl_collision_avoidance_b200 import _lib
    lib = _lib.load()
    nrec, novf = C.c_int32(), C.c_int32()
    rc = lib.rlca_inv_records_host(C.c_float(range_cells), C.byref(nrec), C.byref(novf), None, None)
    if rc != 0:
        return None
    rec = np.zeros((nrec.value, 4), np.uint32)
    ovf = np.zeros(max(novf.value, 1), np.uint16)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    _lib.check(lib.rlca_inv_records_host(C.c_float(range_cells), C.byref(nrec), C.byref(novf), p(rec), p(ovf)))
    return rec, ovf[:novf.value]


# 30: the shipped stage maps (6 m at 0.2 m per cell)
@pytest.mark.parametrize('rc', [1.0, 2.5, 7.5, 16.0, 28.5, 30.0, 31.5])
def test_records_reproduce_the_inverse_lists(built, rc):
    kr, keys, keyslot, off, ent = _tables(rc)
    kdim = 2 * kr + 1
    assert len(keys) <= 255
    packed = _records(rc)
    assert packed is not None
    rec, ovf = packed
    assert rec.shape[0] == kdim * kdim
    n = rec[:, 0] & 0xff
    start = rec[:, 0] >> 8
    np.testing.assert_array_equal(n, np.diff(off))
    # the overflow array is the concatenation of every list's entries from the 7th on, in relative-cell order
    tail = np.maximum(n.astype(np.int64) - 6, 0)
    np.testing.assert_array_equal(start, np.concatenate([[0], np.cumsum(tail)[:-1]]))
    assert len(ovf) == tail.sum()
    halves = np.stack([rec[:, 1:] & 0xffff, rec[:, 1:] >> 16], axis=2).reshape(-1, 6)    # entries 0..5 in order
    for c in range(kdim * kdim):
        want = ent[off[c]:off[c + 1]]
        k = min(int(n[c]), 6)
        got = np.concatenate([halves[c, :k], ovf[start[c]:start[c] + tail[c]]]).astype(np.uint32)
        np.testing.assert_array_equal(got & 0xff, want & 0xffff, err_msg=f'slots of cell {c}')
        np.testing.assert_array_equal(got >> 8, want >> 16, err_msg=f'distances of cell {c}')
        assert not halves[c, k:].any(), f'unused entries of cell {c} are not zero'


def test_ranges_beyond_255_slots_are_refused(built):
    """More than 255 slots do not fit the 8-bit slot field: no records (the lidar keeps inv_off / inv_ent)."""
    for rc in (33.0, 60.0):
        kr, keys, keyslot, off, ent = _tables(rc)
        assert len(keys) > 255
        assert _records(rc) is None
