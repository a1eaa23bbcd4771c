"""The terrain curriculum entry points without a GPU: exported, declared with their argument types, and a null batch refused before
anything touches a device."""
import ctypes as C

import numpy as np

from raisimlib_b200 import capi


def test_entry_points_are_exported_and_typed():
    L = capi.lib()
    for name in ("rsb_batch_set_heightmap_index", "rsb_batch_update_heightmaps"):
        assert name in capi.EXPORTED
        assert hasattr(L, name)
    assert L.rsb_batch_set_heightmap_index.argtypes == [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]
    assert L.rsb_batch_update_heightmaps.argtypes == [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int]


def test_a_null_batch_is_refused():
    L = capi.lib()
    idx, h = np.zeros(4, np.int32), np.zeros((1, 3, 3), np.float32)
    assert L.rsb_batch_set_heightmap_index(None, idx.ctypes.data_as(C.c_void_p), 0, 4, capi.HOST) == -1
    assert b"null batch" in L.rsb_last_error()
    assert L.rsb_batch_update_heightmaps(None, 0, 1, h.ctypes.data_as(C.c_void_p), capi.HOST) == -1
    assert b"null batch" in L.rsb_last_error()
