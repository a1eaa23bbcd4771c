"""Float64 restatement of the LSTM actuator network (rsb_batch_set_actuator_lstm): one cell step of every layer, the read-out and the
saturation, as the step kernel computes them for every listed dof at the start of every sub-step.  Parameters are in torch order."""
import numpy as np


def sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def step(layers, x, state):
    """layers [(weight_ih [4h, n_in], weight_hh [4h, h], bias_ih [4h], bias_hh [4h])]; x [..., 2] = (e, v); state [..., L, 2, h] (h then
    c of every layer).  -> (h' of the last layer [..., h], the new state [..., L, 2, h])"""
    inp = np.asarray(x, np.float64)
    state = np.asarray(state, np.float64)
    new = np.empty_like(state)
    for l, (wih, whh, bih, bhh) in enumerate(layers):
        hid = np.asarray(whh).shape[1]
        h, c = state[..., l, 0, :], state[..., l, 1, :]
        a = (inp @ np.asarray(wih, np.float64).T + np.asarray(bih, np.float64)
             + h @ np.asarray(whh, np.float64).T + np.asarray(bhh, np.float64))
        i, f = sigmoid(a[..., :hid]), sigmoid(a[..., hid:2 * hid])
        g, o = np.tanh(a[..., 2 * hid:3 * hid]), sigmoid(a[..., 3 * hid:])
        c2 = f * c + i * g
        h2 = o * np.tanh(c2)
        new[..., l, 0, :], new[..., l, 1, :] = h2, c2
        inp = h2
    return inp, new


def net(layers, readout, x, state):
    """(the read-out w_out . h'_L + b_out [...], the new state)"""
    h, new = step(layers, x, state)
    w, b = readout
    return h @ np.asarray(w, np.float64).reshape(-1) + float(np.asarray(b, np.float64).reshape(-1)[0]), new


def torque(layers, readout, e, v, state, tau_ff, limit):
    """(the applied torque tau_ff + net saturated at +-limit, the new state); e, v [..., n], state [..., n, L, 2, h]"""
    x = np.stack([np.asarray(e, np.float64), np.asarray(v, np.float64)], axis=-1)
    y, new = net(layers, readout, x, state)
    lim = np.asarray(limit, np.float64)
    return np.clip(np.asarray(tau_ff, np.float64) + y, -lim, lim), new


def random_lstm(rng, layers, hidden, in_scale=3.0, out_scale=20.0):
    """a seeded network in torch order: gates ~ U(-1, 1) / sqrt(fan-in) (layer 0 scaled by in_scale, so that errors of a tenth of a
    radian move it), read-out large enough for torques of tens of N m"""
    out = []
    for l in range(layers):
        nin = 2 if l == 0 else hidden
        s = in_scale if l == 0 else 1.0
        out.append((rng.uniform(-1, 1, (4 * hidden, nin)) * s / np.sqrt(nin), rng.uniform(-1, 1, (4 * hidden, hidden)) / np.sqrt(hidden),
                    rng.uniform(-0.3, 0.3, 4 * hidden), rng.uniform(-0.3, 0.3, 4 * hidden)))
    readout = (rng.uniform(-1, 1, (1, hidden)) * out_scale / np.sqrt(hidden), rng.uniform(-1, 1, 1))
    f32 = lambda t: tuple(np.asarray(a, np.float32) for a in t)
    return [f32(p) for p in out], f32(readout)


def flat(layers, readout):
    """the float32 parameters of rsb_batch_set_actuator_lstm, in torch order"""
    return np.concatenate([np.asarray(a, np.float32).ravel() for p in layers for a in p] +
                          [np.asarray(a, np.float32).ravel() for a in readout])


def count(layers, hidden):
    return sum(4 * hidden * ((2 if l == 0 else hidden) + hidden + 2) for l in range(layers)) + hidden + 1
