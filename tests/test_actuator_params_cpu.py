"""The per-environment PD gain and effort limit entry points without a GPU: exported, declared with their argument types, and a null
batch refused before anything touches a device."""
import ctypes as C

from raisimlib_b200 import capi


def test_entry_points_are_exported_and_typed():
    L = capi.lib()
    for name in ("rsb_batch_set_actuator_params", "rsb_batch_clear_actuator_params"):
        assert name in capi.EXPORTED
        assert hasattr(L, name)
    assert L.rsb_batch_set_actuator_params.argtypes == [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]
    assert L.rsb_batch_clear_actuator_params.argtypes == [C.c_void_p]


def test_a_null_batch_is_refused():
    L = capi.lib()
    rows = (C.c_float * 3)(300.0, 4.0, 80.0)
    assert L.rsb_batch_set_actuator_params(None, rows, 0, 1, capi.HOST) == -1
    assert b"null batch" in L.rsb_last_error()
    assert L.rsb_batch_set_actuator_params(None, None, 0, 1, capi.DEVICE) == -1
    assert b"null batch" in L.rsb_last_error()
    assert L.rsb_batch_clear_actuator_params(None) == -1
    assert b"null batch" in L.rsb_last_error()
