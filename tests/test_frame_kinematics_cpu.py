"""The frame-kinematics restatement (tests/frame_ref.py) against central differences of helpers.fk_numpy along
helpers.integrate_gc(gc, dv, +-eps): the velocity of a frame's point and the angular velocity of its body, for the whole gv and for
every unit dv (each Jacobian column), on floating-base models with revolute and prismatic joints and a fixed-base one."""
import os

import numpy as np
import pytest

from conftest import RSC
from helpers import PENDULUM_URDF, MAX32, fk_numpy, integrate_gc, random_state
from frame_ref import frame_kinematics, random_frames
from raisimlib_b200 import capi

EPS = 1e-5


def _vee(W):
    return np.array([W[2, 1] - W[1, 2], W[0, 2] - W[2, 0], W[1, 0] - W[0, 1]]) / 2


def _numeric(t, gc, dv, body, pos):
    """(d/de) of the frame point and the body's rotation vector along gc (+) e dv, by central differences"""
    (Rp, pp, _), (Rm, pm, _) = fk_numpy(t, integrate_gc(t, gc, dv, EPS)), fk_numpy(t, integrate_gc(t, gc, dv, -EPS))
    lin = np.stack([(pp[b] + Rp[b] @ x - pm[b] - Rm[b] @ x) / (2 * EPS) for b, x in zip(body, pos)])
    ang = np.stack([_vee(Rp[b] @ Rm[b].T) / (2 * EPS) for b in body])     # R(+e) R(-e)^T = exp(2 e [w]x) + O(e^3)
    return lin, ang


@pytest.mark.parametrize("src", ["anymal_c_like.urdf", "atlas_like.urdf", pytest.param(MAX32, id="max32"), pytest.param(PENDULUM_URDF, id="pendulum")])
def test_restatement_matches_central_differences(src):
    t = capi.Model(os.path.join(RSC, src) if src.endswith(".urdf") else src).tables()
    rng = np.random.default_rng(3)
    body, pos, rot = random_frames(rng, t["nb"], 12)
    gcs, gvs = random_state(t, rng, 3, vel_scale=1.0, joint_scale=0.5)
    assert (t["jtype"] == 2).any() == (src in (MAX32, PENDULUM_URDF))      # a prismatic joint in the generic models
    for gc, gv in zip(gcs, gvs):
        x, Rf, lin, ang, J = frame_kinematics(t, gc, gv, body, pos, rot)
        R, p, _ = fk_numpy(t, gc)
        assert np.allclose(x, p[body] + np.einsum("fij,fj->fi", R[body], pos), rtol=0, atol=1e-14)
        assert np.allclose(Rf, R[body] @ rot, rtol=0, atol=1e-14)
        nl, na = _numeric(t, gc, gv, body, pos)
        scale = max(np.abs(nl).max(), np.abs(na).max())
        assert np.abs(lin - nl).max() < 1e-7 * scale and np.abs(ang - na).max() < 1e-7 * scale
        for c in range(t["nv"]):
            nl, na = _numeric(t, gc, np.eye(t["nv"])[c], body, pos)
            scale = max(np.abs(J).max(), 1.0)
            assert np.abs(J[:, 0:3, c] - nl).max() < 1e-7 * scale, c
            assert np.abs(J[:, 3:6, c] - na).max() < 1e-7 * scale, c
        # world axes from the poses (what the kernel uses) give the same columns
        x2, _, lin2, ang2, J2 = frame_kinematics(t, gc, gv, body, pos, rot, poses=(R, p))
        assert np.abs(J2 - J).max() < 1e-12 and np.abs(lin2 - lin).max() < 1e-12 and np.abs(ang2 - ang).max() < 1e-12
