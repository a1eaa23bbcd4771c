"""The actuation delay without a GPU: the entry points are exported and typed, a null batch is refused before anything touches a device,
the restatement of tests/actuation_delay_ref.py gives hand-computed answers, and capi.Batch checks shapes and dtypes on the host."""
import ctypes as C

import numpy as np
import pytest

from raisimlib_b200 import capi
from actuation_delay_ref import applied, applied_index


def test_entry_points_are_exported_and_typed():
    L = capi.lib()
    for name in ("rsb_batch_set_actuation_delay", "rsb_batch_clear_actuation_delay"):
        assert name in capi.EXPORTED
        assert hasattr(L, name)
    assert L.rsb_batch_set_actuation_delay.argtypes == [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]
    assert L.rsb_batch_clear_actuation_delay.argtypes == [C.c_void_p]


def test_a_null_batch_is_refused():
    L = capi.lib()
    d = np.zeros(4, np.int32)
    assert L.rsb_batch_set_actuation_delay(None, d.ctypes.data_as(C.c_void_p), 0, 4, capi.HOST) == -1
    assert b"null batch" in L.rsb_last_error()
    assert L.rsb_batch_set_actuation_delay(None, None, 0, 4, capi.DEVICE) == -1
    assert b"null batch" in L.rsb_last_error()
    assert L.rsb_batch_clear_actuation_delay(None) == -1
    assert b"null batch" in L.rsb_last_error()


def test_known_answers():
    # commands 10, 11, 12, ... at sub-steps 0, 1, 2, ...
    c = np.arange(10, 20)
    assert applied(c, 0).tolist() == c.tolist()
    # d = 2: the first command holds for the first d + 1 = 3 sub-steps
    assert applied(c, 2).tolist() == [10, 10, 10, 11, 12, 13, 14, 15, 16, 17]
    # a delay longer than the history: the first command holds
    assert applied(c[:4], 16).tolist() == [10, 10, 10, 10]
    # emptied before sub-step 5 with a new delay 1: sub-step 5 is t = 0 again
    d = [3, 3, 3, 3, 3, 1, 1, 1, 1, 1]
    assert applied(c, d, empty_before={5}).tolist() == [10, 10, 10, 10, 11, 15, 15, 16, 17, 18]
    # emptied with the delay kept (a termination): the shift restarts
    assert applied(c, 1, empty_before={4, 6}).tolist() == [10, 10, 11, 12, 14, 14, 16, 16, 17, 18]
    assert [applied_index(t, 4) for t in range(7)] == [0, 0, 0, 0, 0, 1, 2]


def test_launch_commands_shift_inside_a_control_step():
    """targets that change every 4-sub-step launch; d = 2 puts each new target in the middle of the next control step"""
    per_launch = np.array([1.0, 2.0, 3.0])
    cmd = np.repeat(per_launch, 4)
    assert applied(cmd, 2).tolist() == [1, 1, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3]
    # rows of a command triple shift together
    rows = np.stack([cmd, -cmd, 10 * cmd], axis=1)
    assert applied(rows, 6)[:, 2].tolist() == [10] * 10 + [20, 20]


def _unbound_batch():
    """a capi.Batch that owns no native batch: every call that passes the host-side checks reaches the library with a null batch"""
    b = capi.Batch.__new__(capi.Batch)
    b.h, b.n, b.device = None, 4, 0
    return b


def test_host_side_checks():
    b = _unbound_batch()
    for bad in (np.zeros(4, np.int64), np.zeros(4, np.float32), np.zeros((2, 2), np.int32), [0, 1, 2, 3]):
        with pytest.raises(ValueError, match="delays"):
            b.set_actuation_delay(bad)
    # a well-formed call reaches the library, which refuses the null batch
    with pytest.raises(capi.RsbError, match="null batch"):
        b.set_actuation_delay(np.zeros(4, np.int32))
    with pytest.raises(capi.RsbError, match="null batch"):
        b.set_actuation_delay(None)
    with pytest.raises(capi.RsbError, match="null batch"):
        b.clear_actuation_delay()
    # the torch variant wants a CUDA tensor: a host tensor or an array is refused before the library is called
    torch = pytest.importorskip("torch")
    for bad in (torch.zeros(4, dtype=torch.int32), np.zeros(4, np.int32)):
        with pytest.raises(ValueError, match="delays"):
            b.set_actuation_delay_from(bad)
