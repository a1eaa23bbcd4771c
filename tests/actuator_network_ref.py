"""Float64 restatement of the learned actuator network (rsb_batch_set_actuator_network) and of its history shift: what the step kernel
computes for every listed dof at the start of every sub-step."""
import numpy as np


def softsign(x):
    return x / (1.0 + np.abs(x))


def features(e, v, hist):
    """e, v [..., n]: this sub-step's position error (ptarget - q) and velocity; hist [..., n, 2, H - 1]: errors then velocities of the
    last H - 1 sub-steps, most recent first.  -> [..., n, 2H] = [e_t, e_{t-1}, ..., e_{t-H+1}, v_t, v_{t-1}, ..., v_{t-H+1}]"""
    e, v, hist = np.asarray(e, np.float64), np.asarray(v, np.float64), np.asarray(hist, np.float64)
    return np.concatenate([e[..., None], hist[..., 0, :], v[..., None], hist[..., 1, :]], axis=-1)


def net(layers, x):
    """layers [(W, b)] in torch.nn.Linear order (hidden layers with softsign, then the linear output [1, width]); x [..., 2H] -> [...]"""
    h = np.asarray(x, np.float64)
    for W, b in layers[:-1]:
        h = softsign(h @ np.asarray(W, np.float64).T + np.asarray(b, np.float64))
    W, b = layers[-1]
    return (h @ np.asarray(W, np.float64).T + np.asarray(b, np.float64))[..., 0]


def shift(e, v, hist):
    """the history after one sub-step: (e, v) in front, the oldest entry dropped"""
    hist = np.asarray(hist)
    new = np.empty_like(hist)
    if hist.shape[-1] == 0:
        return new
    new[..., 0, 0] = e
    new[..., 1, 0] = v
    new[..., :, 1:] = hist[..., :, :-1]
    return new


def torque(layers, e, v, hist, tau_ff, limit):
    """the applied torque: tau_ff + net, saturated at +-limit"""
    t = np.asarray(tau_ff, np.float64) + net(layers, features(e, v, hist))
    return np.clip(t, -np.asarray(limit, np.float64), np.asarray(limit, np.float64))


def random_layers(rng, history, layers, width, scale=1.0, out_scale=20.0):
    """a seeded network: hidden weights ~ U(-1, 1) * scale / sqrt(fan-in), output weights large enough for torques of tens of N m"""
    out, nin = [], 2 * history
    for _ in range(layers):
        out.append((rng.uniform(-1, 1, (width, nin)) * scale / np.sqrt(nin), rng.uniform(-0.3, 0.3, width)))
        nin = width
    out.append((rng.uniform(-1, 1, (1, width)) * out_scale / np.sqrt(width), rng.uniform(-1.0, 1.0, 1)))
    return [(w.astype(np.float32), b.astype(np.float32)) for w, b in out]
