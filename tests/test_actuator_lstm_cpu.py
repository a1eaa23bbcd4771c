"""The LSTM actuator network without a GPU: the entry point is exported and typed, a null batch is refused before anything touches a
device, the float64 restatement of tests/actuator_lstm_ref.py gives a hand-computed answer and equals torch.nn.LSTM + nn.Linear, and
capi.Batch.set_actuator_lstm checks a network on the host and passes its parameters on in torch order, byte for byte."""
import ctypes as C
import math

import numpy as np
import pytest

from raisimlib_b200 import capi
from actuator_lstm_ref import count, flat, net, random_lstm, step, torque


def test_entry_point_is_exported_and_typed():
    L = capi.lib()
    assert "rsb_batch_set_actuator_lstm" in capi.EXPORTED
    assert hasattr(L, "rsb_batch_set_actuator_lstm")
    assert L.rsb_batch_set_actuator_lstm.argtypes == [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]


def test_a_null_batch_is_refused():
    L = capi.lib()
    dofs, params = (C.c_int32 * 1)(6), (C.c_float * count(1, 2))()
    assert L.rsb_batch_set_actuator_lstm(None, dofs, 1, 1, 2, params) == -1
    assert b"null batch" in L.rsb_last_error()
    assert L.rsb_batch_set_actuator_lstm(None, None, 0, 0, 0, None) == -1
    assert b"null batch" in L.rsb_last_error()


def _one_unit():
    """layers = hidden = 1, gates i f g o: a_i = e - v / 2, a_f = 2 h - 1, a_g = ln 2, a_o = ln 3; read-out 2 h' + 1/2"""
    wih = np.array([[1.0, -0.5], [0.0, 0.0], [0.0, 0.0], [0.0, 0.0]])
    whh = np.array([[0.0], [2.0], [0.0], [0.0]])
    bih = np.array([0.0, -1.0, 0.0, math.log(3.0)])
    bhh = np.array([0.0, 0.0, math.log(2.0), 0.0])
    return [(wih, whh, bih, bhh)], (np.array([[2.0]]), np.array([0.5]))


def test_known_answer_one_layer_one_unit():
    """x = (1, 2), h = 1/2, c = 1/4: i = f = sigmoid(0) = 1/2, g = tanh(ln 2) = 3/5, o = sigmoid(ln 3) = 3/4;
    c' = 1/2 * 1/4 + 1/2 * 3/5 = 17/40, h' = 3/4 tanh(17/40), net = 2 h' + 1/2"""
    layers, readout = _one_unit()
    state = np.array([[[0.5], [0.25]]])
    y, new = net(layers, readout, np.array([1.0, 2.0]), state)
    h2 = 0.75 * math.tanh(17.0 / 40.0)
    assert new[0, 1, 0] == pytest.approx(17.0 / 40.0, rel=1e-15)
    assert new[0, 0, 0] == pytest.approx(h2, rel=1e-15)
    assert y == pytest.approx(2.0 * h2 + 0.5, rel=1e-15)
    # tau_ff + net, saturated; the state advances whether or not the torque saturates
    t, s2 = torque(layers, readout, np.array([1.0]), np.array([2.0]), state[None], np.array([0.25]), np.array([100.0]))
    assert t[0] == pytest.approx(0.25 + 2.0 * h2 + 0.5, rel=1e-15)
    t, s3 = torque(layers, readout, np.array([1.0]), np.array([2.0]), state[None], np.array([0.25]), np.array([0.5]))
    assert t[0] == 0.5 and (s3 == s2).all()
    t, _ = torque(layers, readout, np.array([1.0]), np.array([2.0]), state[None], np.array([-10.0]), np.array([0.5]))
    assert t[0] == -0.5


@pytest.mark.parametrize("layers", [1, 2, 3, 4])
@pytest.mark.parametrize("hidden", [1, 3, 8, 17, 32])
def test_restatement_equals_torch_lstm(layers, hidden):
    """float64 torch.nn.LSTM + nn.Linear over random sequences, state carried from step to step, against the restatement"""
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(100 * layers + hidden)
    lp, ro = random_lstm(rng, layers, hidden)
    lstm = torch.nn.LSTM(2, hidden, layers).double()
    lin = torch.nn.Linear(hidden, 1).double()
    with torch.no_grad():
        for l, p in enumerate(lp):
            for name, a in zip(("weight_ih", "weight_hh", "bias_ih", "bias_hh"), p):
                getattr(lstm, f"{name}_l{l}").copy_(torch.from_numpy(a.astype(np.float64)))
        lin.weight.copy_(torch.from_numpy(ro[0].astype(np.float64)))
        lin.bias.copy_(torch.from_numpy(ro[1].astype(np.float64)))
    T, B = 12, 5
    xs = rng.standard_normal((T, B, 2)) * np.array([0.3, 2.0])
    h0 = rng.standard_normal((layers, B, hidden)) * 0.5
    c0 = rng.standard_normal((layers, B, hidden)) * 0.5
    with torch.no_grad():
        out, (hT, cT) = lstm(torch.from_numpy(xs), (torch.from_numpy(h0), torch.from_numpy(c0)))
        want = lin(out)[..., 0].numpy()
    state = np.stack([h0, c0], axis=2).transpose(1, 0, 2, 3)      # [B, L, 2, hidden]
    got = np.empty((T, B))
    for t in range(T):
        got[t], state = net(lp, ro, xs[t], state)
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(state[:, :, 0].transpose(1, 0, 2), hT.numpy(), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(state[:, :, 1].transpose(1, 0, 2), cT.numpy(), rtol=1e-12, atol=1e-12)
    # the last layer's h' is what step() hands to the read-out
    h, _ = step(lp, xs[0], np.zeros((B, layers, 2, hidden)))
    assert h.shape == (B, hidden)


class _Tables:
    def tables(self):
        return dict(joint_names=["", "LF_HAA", "LF_HFE"], vidx=np.array([-1, 6, 7]))


def _unbound_batch():
    """a capi.Batch that owns no native batch: every call that passes the host-side checks reaches the library with a null batch"""
    b = capi.Batch.__new__(capi.Batch)
    b.h, b.n, b.model, b.an_shape, b.lstm_shape = None, 4, _Tables(), None, None
    return b


def test_capi_packs_a_torch_lstm_in_state_dict_order_byte_for_byte():
    torch = pytest.importorskip("torch")
    torch.manual_seed(0)
    for batch_first in (False, True):
        lstm = torch.nn.LSTM(2, 8, 2, batch_first=batch_first)
        lin = torch.nn.Linear(8, 1)
        layers, hidden, params = capi._lstm_params(lstm, lin)
        sd = lstm.state_dict()
        want = np.concatenate([sd[f"{k}_l{l}"].numpy().ravel() for l in range(2) for k in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]
                              + [lin.weight.detach().numpy().ravel(), lin.bias.detach().numpy().ravel()])
        assert (layers, hidden) == (2, 8)
        assert params.dtype == np.float32 and params.flags.c_contiguous
        assert params.tobytes() == want.astype(np.float32).tobytes()
        assert len(params) == count(2, 8)
    # numpy arrays in torch order give the same bytes
    lp, ro = random_lstm(np.random.default_rng(1), 3, 5)
    layers, hidden, params = capi._lstm_params(lp, ro)
    assert (layers, hidden) == (3, 5)
    assert params.tobytes() == flat(lp, ro).tobytes()
    with pytest.raises(capi.RsbError, match="null batch"):      # accepted on the host: the library refuses the null batch
        _unbound_batch().set_actuator_lstm(["LF_HAA", 7], lp, ro)


def test_capi_checks_the_network_on_the_host():
    torch = pytest.importorskip("torch")
    nn = torch.nn
    b = _unbound_batch()
    lin = nn.Linear(8, 1)
    for bad, what in ((nn.LSTM(3, 8), "input_size must be 2"), (nn.LSTM(2, 8, bias=False), "bias=True"),
                      (nn.LSTM(2, 8, bidirectional=True), "bidirectional"), (nn.LSTM(2, 8, proj_size=4), "proj_size"),
                      (nn.LSTM(2, 8, 5), r"5 layers outside \[1, 4\]"), (nn.LSTM(2, 33), r"hidden size 33 outside \[1, 32\]")):
        with pytest.raises(ValueError, match=what):
            b.set_actuator_lstm([6], bad, nn.Linear(bad.hidden_size, 1))
    with pytest.raises(ValueError, match="read-out Linear needs a bias"):
        b.set_actuator_lstm([6], nn.LSTM(2, 8), nn.Linear(8, 1, bias=False))
    with pytest.raises(ValueError, match=r"read-out needs weight \(1, 8\)"):
        b.set_actuator_lstm([6], nn.LSTM(2, 8), nn.Linear(8, 2))
    with pytest.raises(ValueError, match=r"read-out needs weight \(1, 8\)"):
        b.set_actuator_lstm([6], nn.LSTM(2, 8), nn.Linear(4, 1))
    with pytest.raises(ValueError, match="unknown joints"):
        b.set_actuator_lstm(["RF_KFE"], nn.LSTM(2, 8), lin)
    lp, ro = random_lstm(np.random.default_rng(2), 2, 8)
    bad = [lp[0], (lp[1][0][:, :5],) + lp[1][1:]]
    with pytest.raises(ValueError, match="layer 1"):
        b.set_actuator_lstm([6], bad, ro)
    with pytest.raises(ValueError, match=r"\(weight_ih, weight_hh, bias_ih, bias_hh\)"):
        b.set_actuator_lstm([6], [lp[0][:3]], ro)
    # the history rows take the LSTM's shape while it is set, the MLP's otherwise
    with pytest.raises(ValueError, match="no actuator network"):
        b.actuator_history()
    b.lstm_shape = (3, 2, 8)
    with pytest.raises(ValueError, match=r"need shape \[n, 3, 2, 2, 8\]"):
        b.set_actuator_history(np.zeros((4, 3, 2, 8), np.float32))
    with pytest.raises(capi.RsbError, match="null batch"):
        b.set_actuator_history(np.zeros((4, 3, 2, 2, 8), np.float32))
