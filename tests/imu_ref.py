"""Numpy restatement of the batch's IMU readings (rsb_batch_set_imus / rsb_batch_get_imu_readings) in float64, on the frame kinematics
of tests/frame_ref.py: J_p and J_r from frame_kinematics, Jdot_p v as the central difference of J_p(q (+) eps v) v in eps
(helpers.integrate_gc).  It shares no code with the step kernel's chain recursion.  tests/test_imu_cpu.py pins it with known answers and
finite differences of oracle trajectories; it is the reference of tests/test_gpu_imu.py."""
import numpy as np

from frame_ref import frame_kinematics
from helpers import integrate_gc

EPS = 1e-5      # central-difference step of Jdot_p v [s]: truncation O(EPS^2), rounding ~1e-16 / EPS


def imu_substep(t, gc, gv, gv1, dt, body, pos, rot=None, gravity=(0.0, 0.0, -9.81)):
    """One environment, one sub-step from (gc, gv) to velocity gv1: (f [I, 3], w [I, 3]) in the sensor frames,
    f = R_k^T [J_p (gv1 - gv) / dt + Jdot_p gv - g], w = R_k^T J_r gv1."""
    gc, gv, gv1 = (np.asarray(a, np.float64) for a in (gc, gv, gv1))
    _, Rk, _, _, J = frame_kinematics(t, gc, gv, body, pos, rot)
    jp = lambda e: frame_kinematics(t, integrate_gc(t, gc, gv, e), gv, body, pos, rot)[4][:, 0:3] @ gv
    jdot_v = (jp(EPS) - jp(-EPS)) / (2 * EPS)
    a = J[:, 0:3] @ ((gv1 - gv) / dt) + jdot_v - np.asarray(gravity, np.float64)
    return np.einsum("kji,kj->ki", Rk, a), np.einsum("kji,kj->ki", Rk, J[:, 3:6] @ gv1)


def imu_launch(t, gcs, gvs, dt, body, pos, rot=None, gravity=(0.0, 0.0, -9.81)):
    """One environment, one launch of S sub-steps given its states gcs [S + 1, nq], gvs [S + 1, nv] (the start state, then the state
    after each sub-step): the mean readings (lin_acc [I, 3], ang_vel [I, 3]) over the launch"""
    S = len(gcs) - 1
    out = [imu_substep(t, gcs[s], gvs[s], gvs[s + 1], dt, body, pos, rot, gravity) for s in range(S)]
    return sum(o[0] for o in out) / S, sum(o[1] for o in out) / S


def batch_imu_launch(t, gcs, gvs, dt, body, pos, rot=None, gravity=(0.0, 0.0, -9.81)):
    """imu_launch of every environment: gcs [S + 1, n, nq], gvs [S + 1, n, nv] -> (lin_acc [n, I, 3], ang_vel [n, I, 3])"""
    gcs, gvs = np.asarray(gcs, np.float64), np.asarray(gvs, np.float64)
    out = [imu_launch(t, gcs[:, e], gvs[:, e], dt, body, pos, rot, gravity) for e in range(gcs.shape[1])]
    return np.stack([o[0] for o in out]), np.stack([o[1] for o in out])


def point_acceleration_fd(t, gc, gv, gc1, gv1, dt, body, pos, rot=None):
    """(J_p(q_{s+1}) v_{s+1} - J_p(q_s) v_s) / dt in the sensor frames at q_s: the sensor point's velocity change over one sub-step of a
    trajectory, which the analytic acceleration must match to O(dt)"""
    _, Rk, v0, _, _ = frame_kinematics(t, gc, gv, body, pos, rot)
    v1 = frame_kinematics(t, gc1, gv1, body, pos, rot)[2]
    return np.einsum("kji,kj->ki", Rk, (v1 - v0) / dt)
