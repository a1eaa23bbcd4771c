"""Reference for the per-body contact forces of a whole launch (rsb_batch_get_body_contact_forces): a numpy restatement on top of
the oracle's per-step debug output, no new oracle code.  The oracle is stepped one sub-step at a time; each sub-step's contacts
(body, pair, normal, contact-frame impulse) become world impulses in the tangent frame of DESIGN.md section 2 and are scattered by
body and sub-step."""
import numpy as np


def tangent_frame(n):
    """t1 = normalise(e_x - (e_x . n) n), e_y instead of e_x when |n_x| >= 0.9; t2 = n x t1.  n [..., 3] -> (t1, t2)"""
    n = np.asarray(n, np.float64)
    e = np.where((np.abs(n[..., 0:1]) >= 0.9), np.array([0.0, 1.0, 0.0]), np.array([1.0, 0.0, 0.0]))
    t1 = e - (e * n).sum(-1, keepdims=True) * n
    t1 = t1 / np.linalg.norm(t1, axis=-1, keepdims=True)
    return t1, np.cross(n, t1)


def world_impulses(d):
    """world impulse of every contact of one oracle step on its first body: [n, K, 3] (zero rows beyond ncontacts)"""
    nrm = np.where((d["c_pt"] >= 0)[..., None], d["c_normal"], np.array([0.0, 0.0, 1.0]))
    t1, t2 = tangent_frame(nrm)
    lam = d["c_lambda"]
    imp = t1 * lam[..., 0:1] + t2 * lam[..., 1:2] + nrm * lam[..., 2:3]
    live = np.arange(d["c_pt"].shape[1])[None, :] < d["ncontacts"][:, None]
    return np.where(live[..., None], imp, 0.0)


def scatter_step(d, bodies):
    """one sub-step: (impulse [n, S, 3] on each listed body, touched [n, S] bool).  A contact acts with +impulse on c_body and, when
    c_pair < 0 (a self contact), with -impulse on body -1 - c_pair."""
    imp = world_impulses(d)
    n, K = d["c_pt"].shape
    live = np.arange(K)[None, :] < d["ncontacts"][:, None]
    out, hit = np.zeros((n, len(bodies), 3)), np.zeros((n, len(bodies)), bool)
    for s, body in enumerate(bodies):
        first = live & (d["c_body"] == body)
        second = live & (d["c_pair"] < 0) & (-1 - d["c_pair"] == body)
        for k in range(K):      # contact-list order
            out[:, s] += np.where(first[:, k, None], imp[:, k], 0.0) - np.where(second[:, k, None], imp[:, k], 0.0)
        hit[:, s] = first.any(1) | second.any(1)
    return out, hit


def step_with_forces(o, gc, gv, substeps, bodies, **kw):
    """`substeps` oracle steps from (gc, gv), updated in place: (force [n, S, 3] = summed impulses / (substeps dt),
    steps_in_contact [n, S], the per-sub-step debug outputs)"""
    n = gc.shape[0]
    acc, steps, dbg = np.zeros((n, len(bodies), 3)), np.zeros((n, len(bodies)), np.int32), []
    for _ in range(substeps):
        d = o.step(gc, gv, n_steps=1, debug=True, **kw)
        imp, hit = scatter_step(d, bodies)
        acc += imp; steps += hit
        dbg.append(d)
    return acc / (substeps * o.params["dt"]), steps, dbg
