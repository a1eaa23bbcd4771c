"""The learned actuator network without a GPU: the entry points are exported and typed, a null batch is refused before anything touches a
device, the float64 restatement of tests/actuator_network_ref.py gives a hand-computed answer and the documented feature order, and
capi.Batch.set_actuator_network checks the shapes of a network on the host."""
import ctypes as C

import numpy as np
import pytest

from raisimlib_b200 import capi
from actuator_network_ref import features, net, shift, softsign, torque

NAMES = ("rsb_batch_set_actuator_network", "rsb_batch_set_actuator_history", "rsb_batch_get_actuator_history")


def test_entry_points_are_exported_and_typed():
    L = capi.lib()
    for name in NAMES:
        assert name in capi.EXPORTED
        assert hasattr(L, name)
    assert L.rsb_batch_set_actuator_network.argtypes == [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]
    assert L.rsb_batch_set_actuator_history.argtypes == [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]
    assert L.rsb_batch_get_actuator_history.argtypes == [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]


def test_a_null_batch_is_refused():
    L = capi.lib()
    dofs, params, rows = (C.c_int32 * 1)(6), (C.c_float * 64)(), (C.c_float * 8)()
    assert L.rsb_batch_set_actuator_network(None, dofs, 1, 1, 1, 2, params) == -1
    assert b"null batch" in L.rsb_last_error()
    assert L.rsb_batch_set_actuator_network(None, None, 0, 0, 0, 0, None) == -1
    assert b"null batch" in L.rsb_last_error()
    for fn in (L.rsb_batch_set_actuator_history, L.rsb_batch_get_actuator_history):
        assert fn(None, rows, 0, 1, capi.HOST) == -1
        assert b"null batch" in L.rsb_last_error()


def test_known_answer_width_two_history_one():
    """x = [e, v] = [1, 2]; hidden a = W1 x + b1 = [1 + 4 + 0.5, -1 + 1 - 1] = [5.5, -1] -> softsign [11/13, -1/2];
    out = 2 * 11/13 - 3 * (-1/2) + 1/4 = 179/52"""
    layers = [(np.array([[1.0, 2.0], [-1.0, 0.5]]), np.array([0.5, -1.0])), (np.array([[2.0, -3.0]]), np.array([0.25]))]
    x = features(np.array([1.0]), np.array([2.0]), np.zeros((1, 2, 0)))
    assert x.tolist() == [[1.0, 2.0]]
    assert net(layers, x)[0] == pytest.approx(179.0 / 52.0, rel=1e-15)
    # tau_ff + net, saturated
    assert torque(layers, np.array([1.0]), np.array([2.0]), np.zeros((1, 2, 0)), 0.5, 100.0)[0] == pytest.approx(0.5 + 179.0 / 52.0)
    assert torque(layers, np.array([1.0]), np.array([2.0]), np.zeros((1, 2, 0)), 0.5, 1.5)[0] == 1.5
    assert torque(layers, np.array([1.0]), np.array([2.0]), np.zeros((1, 2, 0)), -10.0, 1.5)[0] == -1.5


def test_feature_order_by_one_hot_first_layer():
    """hidden unit j copies feature j (one-hot row j of W1); an output one-hot on unit k reads softsign(feature k): the features are
    [e_t, e_{t-1}, e_{t-2}, v_t, v_{t-1}, v_{t-2}] with the history most recent first"""
    H = 3
    e, v = np.array([0.1]), np.array([-0.7])
    hist = np.array([[[0.2, 0.3], [-0.8, -0.9]]])
    want = [0.1, 0.2, 0.3, -0.7, -0.8, -0.9]
    for k in range(2 * H):
        out = np.zeros((1, 2 * H)); out[0, k] = 1.0
        layers = [(np.eye(2 * H), np.zeros(2 * H)), (out, np.zeros(1))]
        assert net(layers, features(e, v, hist))[0] == pytest.approx(softsign(want[k]), rel=1e-15)


def test_history_shift():
    hist = np.arange(12.0).reshape(2, 1, 2, 3)
    new = shift(np.array([[-1.0], [-2.0]]), np.array([[-3.0], [-4.0]]), hist)
    assert new[0, 0].tolist() == [[-1.0, 0.0, 1.0], [-3.0, 3.0, 4.0]]
    assert new[1, 0].tolist() == [[-2.0, 6.0, 7.0], [-4.0, 9.0, 10.0]]
    assert shift(np.zeros(1), np.zeros(1), np.zeros((1, 2, 0))).shape == (1, 2, 0)


class _Tables:
    def tables(self):
        return dict(joint_names=["", "LF_HAA", "LF_HFE"], vidx=np.array([-1, 6, 7]))


def _unbound_batch():
    """a capi.Batch that owns no native batch: every call that passes the host-side checks reaches the library with a null batch"""
    b = capi.Batch.__new__(capi.Batch)
    b.h, b.n, b.model, b.an_shape = None, 4, _Tables(), None
    return b


def _pairs(H, W, L):
    rng = np.random.default_rng(0)
    out, nin = [], 2 * H
    for _ in range(L):
        out.append((rng.standard_normal((W, nin)), rng.standard_normal(W)))
        nin = W
    out.append((rng.standard_normal((1, W)), rng.standard_normal(1)))
    return out


def test_capi_checks_shapes_on_the_host():
    b = _unbound_batch()
    good = _pairs(2, 8, 2)
    with pytest.raises(capi.RsbError, match="null batch"):       # shapes accepted: the library refuses the null batch
        b.set_actuator_network([6, 7], good, history=2)
    with pytest.raises(capi.RsbError, match="null batch"):       # joint names resolve through the model's tables
        b.set_actuator_network(["LF_HAA", "LF_HFE"], good, history=2)
    with pytest.raises(ValueError, match="unknown joints"):
        b.set_actuator_network(["RF_KFE"], good, history=2)
    with pytest.raises(ValueError, match="layer 0"):             # the first layer takes 2 * history features
        b.set_actuator_network([6], good, history=3)
    bad = list(good); bad[1] = (good[1][0][:, :5], good[1][1])
    with pytest.raises(ValueError, match="layer 1"):
        b.set_actuator_network([6], bad, history=2)
    bad = list(good); bad[-1] = (np.ones((2, 8)), np.ones(2))
    with pytest.raises(ValueError, match="layer 2"):             # one output
        b.set_actuator_network([6], bad, history=2)
    bad = list(good); bad[0] = (good[0][0], good[0][1][:3])
    with pytest.raises(ValueError, match="layer 0"):
        b.set_actuator_network([6], bad, history=2)
    with pytest.raises(ValueError, match="at least one hidden layer"):
        b.set_actuator_network([6], good[-1:], history=2)
    with pytest.raises(ValueError, match=r"\(W, b\) pairs"):
        b.set_actuator_network([6], [(np.ones((8, 4)),)], history=2)
    with pytest.raises(ValueError, match="no actuator network"):
        b.actuator_history()
    b.an_shape = (2, 3)
    with pytest.raises(ValueError, match=r"need shape \[n, 2, 2, 2\]"):
        b.set_actuator_history(np.zeros((4, 2, 2, 3), np.float32))


def test_capi_takes_a_torch_sequential_of_linear_and_softsign_only():
    torch = pytest.importorskip("torch")
    nn = torch.nn
    b = _unbound_batch()
    torch.manual_seed(0)
    seq = nn.Sequential(nn.Linear(4, 8), nn.Softsign(), nn.Linear(8, 8), nn.Softsign(), nn.Linear(8, 1))
    pairs = capi._network_layers(seq)
    assert [p[0].shape for p in pairs] == [(8, 4), (8, 8), (1, 8)]
    assert pairs[0][0].tobytes() == seq[0].weight.detach().numpy().tobytes()
    with pytest.raises(capi.RsbError, match="null batch"):
        b.set_actuator_network([6], seq, history=2)
    for bad in (nn.Sequential(nn.Linear(4, 8), nn.Tanh(), nn.Linear(8, 1)),
                nn.Sequential(nn.Linear(4, 8), nn.Softsign()),
                nn.Sequential(nn.Linear(4, 8), nn.Linear(8, 1)),
                nn.Sequential(nn.Linear(4, 8, bias=False), nn.Softsign(), nn.Linear(8, 1))):
        with pytest.raises(ValueError, match="actuator network"):
            b.set_actuator_network([6], bad, history=2)
