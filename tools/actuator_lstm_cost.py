#!/usr/bin/env python3
"""What the LSTM actuator network costs the batched step, on tools/feature_cost.py's harness: the same options (--parent-lib,
--configs, --envs, --steps, --warmup, --repeats, --out), the same timing, modes alternated in one process.

    python tools/actuator_lstm_cost.py [--parent-lib PATH] [--configs c3,c4] ...

Modes, all on every joint (12 on config 3, 30 on config 4): `limp` (kp = kd = 0 rows, no network), `mlp` (feature_cost.py's MLP:
history 3, three layers of 32), `lstm8` (2 layers, hidden 8: the ANYmal actuator model's shape), `lstm32` (2 layers, hidden 32).  Every network has a zero read-out, so
every weight is loaded and every gate evaluated at every sub-step while the torque is exactly that of `limp`: each mode's final state
must equal `limp`'s bit for bit, and the differences in time are the cost of evaluating the networks.  With --parent-lib the first mode
also runs on the parent build, as `parent`.
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import feature_cost  # noqa: E402


def zero_readout_lstm(rng, layers, hidden):
    """per-layer (weight_ih, weight_hh, bias_ih, bias_hh) in torch order, dense and random; a zero read-out (net = 0 exactly)"""
    out = []
    for l in range(layers):
        nin = 2 if l == 0 else hidden
        out.append(tuple(a.astype(np.float32) for a in (rng.uniform(-1, 1, (4 * hidden, nin)) / np.sqrt(nin),
                                                         rng.uniform(-1, 1, (4 * hidden, hidden)) / np.sqrt(hidden),
                                                         rng.uniform(-0.3, 0.3, 4 * hidden), rng.uniform(-0.3, 0.3, 4 * hidden))))
    return out, (np.zeros((1, hidden), np.float32), np.zeros(1, np.float32))


def actuator_lstm(bt, mode, wl):
    if mode == "limp":
        rows = np.full((wl.n, bt.nv, 3), -1.0, np.float32)
        rows[:, 6:, :2] = 0.0
        bt.set_actuator_params(rows)
    elif mode == "mlp":
        bt.set_actuator_network(list(range(6, bt.nv)), feature_cost.zero_output_network(np.random.default_rng(0)), feature_cost.HISTORY)
    elif mode.startswith("lstm"):
        bt.set_actuator_lstm(list(range(6, bt.nv)), *zero_readout_lstm(np.random.default_rng(0), 2, int(mode[4:])))


feature_cost.FEATURES["actuator_lstm"] = dict(configs="c3,c4", modes=["limp", "mlp", "lstm8", "lstm32"],
                                              setup=feature_cost.per_mode(actuator_lstm), ref="limp")

if __name__ == "__main__":
    sys.argv[1:1] = ["actuator_lstm"]
    feature_cost.main()
