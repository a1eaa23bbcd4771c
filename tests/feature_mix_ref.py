"""Per-environment composition of the batched step's opt-in features, built from the existing restatements: every environment has its
own float64 (or float32) oracle with its own inertial parameters (body_inertia_ref.tables_with), effort limits, terrain friction per
collision body and height map, and self-collision pairs where they are set (oracle.self_oracle.SelfOracle).  The composition steps one
sub-step at a time and applies, in the step kernel's order:

- the command of the sub-step the actuation delay selects (actuation_delay_ref.applied);
- the actuator network's torque on the listed dofs, from the applied target, and its history shift (actuator_network_ref.torque,
  shift), saturated at the environment's effort limit;
- kp and kd of every dof from the environment's row (an entry < 0 takes the batch value; the base and the network dofs get 0);
- the external wrench of the sub-step, if any.

Each sub-step returns the oracles' debug outputs stacked over the environments, for the contact lists, the applied generalized force
and contact_force_ref.scatter_step."""
import numpy as np

from actuation_delay_ref import applied
from actuator_network_ref import shift, torque
from body_inertia_ref import tables_with
from helpers import effort_limits
from oracle.oracle import Oracle
from oracle.self_oracle import SelfOracle


def dof_q(t):
    """[nv] the gc index of every dof's coordinate (the base dofs: -1)"""
    q = np.full(t["nv"], -1)
    for b in range(1, t["nb"]):
        q[t["vidx"][b]] = t["qidx"][b]
    return q


class MixRef:
    """n environments of the model with tables t.  Every feature is optional (None: off):
    kp, kd [nv]: the batch-level gains (set_pd_gains); rows [n, nv, 3]: set_actuator_params rows; inertia [n, nb, 10]: set_body_inertia
    rows; friction [n, ncoll]: set_contact_friction rows; terrain: ("ground", z) or ("atlas", (x_size, y_size, cx, cy), heights
    [count, ys, xs], map_of_env [n]); pairs: set_self_collision pairs; delay [n]: set_actuation_delay; network: (dofs, layers, H)."""

    def __init__(self, t, n, precision="f64", params=None, kp=None, kd=None, rows=None, inertia=None, friction=None,
                 terrain=("ground", 0.0), pairs=None, delay=None, network=None):
        self.t, self.n = t, n
        nv, nbase = t["nv"], 6 if t["floating"] else 0
        kp0 = np.zeros(nv) if kp is None else np.asarray(kp, np.float64)
        kd0 = np.zeros(nv) if kd is None else np.asarray(kd, np.float64)
        r = np.full((n, nv, 3), -1.0) if rows is None else np.asarray(rows, np.float64)
        self.kp = np.where(r[:, :, 0] >= 0, r[:, :, 0], kp0)
        self.kd = np.where(r[:, :, 1] >= 0, r[:, :, 1], kd0)
        self.lim = np.where(r[:, :, 2] >= 0, r[:, :, 2], effort_limits(t))
        self.kp[:, :nbase] = 0.0; self.kd[:, :nbase] = 0.0
        self.lim[:, :nbase] = 1e30
        self.dofs = None
        if network is not None:
            self.dofs, self.layers, H = np.asarray(network[0]), network[1], network[2]
            self.kp[:, self.dofs] = 0.0; self.kd[:, self.dofs] = 0.0
            self.hist = np.zeros((n, len(self.dofs), 2, H - 1))
            self.dq = dof_q(t)[self.dofs]
        self.delay = None if delay is None else np.array(delay, np.int64)
        self.cmds = []          # the commanded (ptarget, vtarget, tau_ff) of every sub-step
        self.start = np.zeros(n, np.int64)   # per environment: the sub-step its delay history was last emptied before
        self.oracles = []
        for e in range(n):
            te = dict(t)
            if inertia is not None:
                te = tables_with(t, inertia[e, :, 0], inertia[e, :, 1:4], inertia[e, :, 4:10])
            jeff = np.asarray(t["jeffort"], np.float64).copy()
            for b in range(1, t["nb"]):
                jeff[b] = self.lim[e, t["vidx"][b]]
            te["jeffort"] = jeff
            o = (SelfOracle if pairs is not None else Oracle)(te, precision=precision, params=params)
            if pairs is not None:
                o.set_self_collision(pairs)
            if terrain[0] == "ground":
                o.set_ground(terrain[1])
            else:
                (xsz, ysz, cx, cy), H, m = terrain[1], terrain[2], terrain[3]
                o.set_heightmap(H.shape[2], H.shape[1], xsz, ysz, cx, cy, np.asarray(H[m[e]], np.float64))
            if friction is not None:
                for ci in range(t["ncoll"]):
                    if friction[e, ci] >= 0:
                        o.set_collision_friction(ci, float(friction[e, ci]))
            self.oracles.append(o)

    def empty_delay_history(self, envs):
        """what a termination, gym_reset or set_actuation_delay does to the listed environments' command history"""
        self.start[np.asarray(envs, np.int64)] = len(self.cmds)

    def reset_network_history(self, envs):
        self.hist[np.asarray(envs, np.int64)] = 0.0

    def applied_command(self, s):
        """(ptarget [n, nq], vtarget [n, nv], tau_ff [n, nv]) that sub-step s (an index into the recorded commands) applies"""
        if self.delay is None:
            return self.cmds[s]
        out = [np.empty_like(x) for x in self.cmds[s]]
        for e in range(self.n):
            a = self.start[e]
            k = a + applied(np.arange(s + 1 - a), int(self.delay[e]))[-1]
            for i in range(3):
                out[i][e] = self.cmds[k][i][e]
        return out

    def substep(self, gc, gv, pt, vt, tau, ext=None):
        """one sub-step of every environment from (gc, gv) [n, nq] / [n, nv] float64, updated in place, under the commanded rows
        (pt, vt, tau).  ext: (body, force [n, 3] | None, torque [n, 3] | None, point (3) | None) acting in this sub-step.  Returns the
        stacked debug outputs, with "tau_net" [n, len(dofs)] the network torque when there is a network."""
        self.cmds.append(tuple(np.array(x, np.float64) for x in (pt, vt, tau)))
        pa, va, fa = self.applied_command(len(self.cmds) - 1)
        tau_ff = fa.copy()
        tau_net = None
        if self.dofs is not None:
            e_ = pa[:, self.dq] - gc[:, self.dq]
            v_ = gv[:, self.dofs]
            tau_net = torque(self.layers, e_, v_, self.hist, fa[:, self.dofs], self.lim[:, self.dofs])
            self.hist = shift(e_, v_, self.hist)
            tau_ff[:, self.dofs] = tau_net
        outs = []
        for e, o in enumerate(self.oracles):
            a, b = gc[e:e + 1].copy(), gv[e:e + 1].copy()
            x = None
            if ext is not None:
                body, F, T, p = ext
                x = (body, None if F is None else F[e:e + 1], None if T is None else T[e:e + 1], p)
            outs.append(o.step(a, b, tau_ff=tau_ff[e:e + 1], ptarget=pa[e:e + 1], vtarget=va[e:e + 1], kp=self.kp[e], kd=self.kd[e],
                               debug=True, ext=x))
            gc[e], gv[e] = a[0], b[0]
        d = {k: np.concatenate([x[k] for x in outs]) for k in outs[0]}
        d["tau_net"] = tau_net
        return d
