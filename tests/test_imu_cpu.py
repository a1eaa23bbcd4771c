"""The reference of the IMU readings (tests/imu_ref.py) pinned on the CPU, float64, before it judges the kernel
(tests/test_gpu_imu.py): known answers, and agreement to O(dt) with the finite difference of the sensor point's velocity along oracle
trajectories."""
import numpy as np

from frame_ref import frame_kinematics
from helpers import PENDULUM_URDF, quat_to_rot
from imu_ref import imu_launch, imu_substep, point_acceleration_fd
from oracle.oracle import Oracle
from oracle.urdf_tables import load_tables
from raisimlib_b200 import capi

G = np.array([0.0, 0.0, -9.81])
DT = 0.0025
ROT = quat_to_rot(np.array([0.9, 0.2, -0.3, 0.25]) / np.linalg.norm([0.9, 0.2, -0.3, 0.25]))


def test_pendulum_at_rest_reads_minus_gravity_in_the_sensor_frame():
    t = load_tables(PENDULUM_URDF)
    rng = np.random.default_rng(0)
    for _ in range(5):
        gc = rng.uniform(-1, 1, t["nq"])
        zero = np.zeros(t["nv"])
        body, pos = [1, 2, 3], rng.uniform(-0.3, 0.3, (3, 3))
        rot = np.stack([ROT, np.eye(3), ROT.T])
        f, w = imu_substep(t, gc, zero, zero, DT, body, pos, rot, G)
        Rk = frame_kinematics(t, gc, zero, body, pos, rot)[1]
        assert np.abs(f - np.einsum("kji,j->ki", Rk, -G)).max() < 1e-12
        assert np.abs(w).max() == 0.0


def test_floating_robot_in_free_fall_reads_zero(anymal_tables):
    """no terrain, no torques, at rest: one oracle sub-step accelerates every body at g, which the sensors do not feel"""
    t = anymal_tables
    gc = np.zeros((1, t["nq"])); gc[0, 2] = 1.0; gc[0, 3:7] = [0.8, 0.3, -0.2, 0.4]; gc[0, 3:7] /= np.linalg.norm(gc[0, 3:7])
    gc[0, 7:] = np.random.default_rng(1).uniform(-0.5, 0.5, t["nq"] - 7)
    gv = np.zeros((1, t["nv"]))
    gc0, gv0 = gc.copy(), gv.copy()
    Oracle(t).step(gc, gv, 1)
    assert np.abs(gv[0, :3] - DT * G).max() < 1e-12
    body, pos = [0, 4, 8, 12], np.random.default_rng(2).uniform(-0.2, 0.2, (4, 3))
    f, w = imu_substep(t, gc0[0], gv0[0], gv[0], DT, body, pos, np.tile(ROT, (4, 1, 1)), G)
    assert np.abs(f).max() < 1e-9 and np.abs(w).max() < 1e-12


def test_link_spinning_at_constant_rate_reads_centripetal_and_rate():
    """zero gravity, the first joint of the pendulum turning at omega about y, the others still: -omega^2 r_perp and omega"""
    t = load_tables(PENDULUM_URDF)
    omega, q = 3.0, 0.7
    gc = np.array([q, 0.0, 0.0]); gv = np.array([omega, 0.0, 0.0])
    pos = np.array([[0.2, 0.05, -0.4]])
    f, w = imu_substep(t, gc, gv, gv, DT, [1], pos, ROT[None], np.zeros(3))
    x, Rk = frame_kinematics(t, gc, gv, [1], pos, ROT[None])[:2]
    axis_point = np.array([0.0, 0.0, 1.0])          # joint j1: origin (0, 0, 1), axis y
    r = x[0] - axis_point
    r_perp = r - r[1] * np.array([0.0, 1.0, 0.0])
    assert np.abs(f[0] - Rk[0].T @ (-omega ** 2 * r_perp)).max() < 1e-8
    assert np.abs(w[0] - Rk[0].T @ np.array([0.0, omega, 0.0])).max() < 1e-12


def test_base_translating_with_pure_dv_reads_dv_over_dt(anymal_tables):
    t = anymal_tables
    gc = np.zeros(t["nq"]); gc[2] = 0.6; gc[3:7] = [0.9, -0.1, 0.3, 0.2]; gc[3:7] /= np.linalg.norm(gc[3:7])
    gv, gv1 = np.zeros(t["nv"]), np.zeros(t["nv"])
    gv1[:3] = [0.01, -0.02, 0.005]
    body, pos = [0, 3, 7], np.array([[0.1, 0.0, 0.05], [0.0, 0.0, 0.0], [-0.05, 0.1, 0.0]])
    f, w = imu_substep(t, gc, gv, gv1, DT, body, pos, None, np.zeros(3))
    Rk = frame_kinematics(t, gc, gv, body, pos)[1]
    assert np.abs(f - np.einsum("kji,j->ki", Rk, gv1[:3] / DT)).max() < 1e-10
    assert np.abs(w).max() == 0.0


def _trajectory(t, gc, gv, steps, dt, kw):
    o = Oracle(t, params=dict(dt=dt))
    gcs, gvs = [gc.copy()], [gv.copy()]
    for _ in range(steps):
        o.step(gc, gv, 1, **kw)
        gcs.append(gc.copy()); gvs.append(gv.copy())
    return np.array(gcs), np.array(gvs)


def _fd_error(t, gc, gv, dt, body, pos, rot, kw):
    """largest |analytic - finite difference| over a 0.05 s trajectory, and the largest analytic value"""
    gcs, gvs = _trajectory(t, gc[None].copy(), gv[None].copy(), int(round(0.05 / dt)), dt, kw)
    err = big = 0.0
    for s in range(len(gcs) - 1):
        f, _ = imu_substep(t, gcs[s, 0], gvs[s, 0], gvs[s + 1, 0], dt, body, pos, rot, G)
        fd = point_acceleration_fd(t, gcs[s, 0], gvs[s, 0], gcs[s + 1, 0], gvs[s + 1, 0], dt, body, pos, rot)
        Rk = frame_kinematics(t, gcs[s, 0], gvs[s, 0], body, pos, rot)[1]
        fd = fd - np.einsum("kji,j->ki", Rk, G)
        err, big = max(err, np.abs(f - fd).max()), max(big, np.abs(f).max())
    return err, big


def test_reading_matches_finite_difference_of_point_velocity_to_order_dt(anymal_tables):
    """a swinging pendulum (revolute, revolute, prismatic with a rotated joint frame) under gravity and a floating quadruped thrown
    spinning without terrain under PD torques: the analytic specific force equals the finite difference of the sensor point's velocity
    (minus gravity) up to a first-order term that halves with dt"""
    rng = np.random.default_rng(3)
    cases = []
    t = load_tables(PENDULUM_URDF)
    cases.append((t, np.array([0.4, -0.6, 0.1]), np.array([1.0, -0.5, 0.3]), [1, 2, 3], rng.uniform(-0.2, 0.2, (3, 3)), {}))
    a = anymal_tables
    gc = np.zeros(a["nq"]); gc[2] = 1.0; gc[3:7] = [0.9, 0.2, -0.1, 0.3]; gc[3:7] /= np.linalg.norm(gc[3:7])
    gc[7:] = rng.uniform(-0.4, 0.4, 12)
    gv = np.r_[0.3, -0.2, 1.0, 1.5, -1.0, 0.8, rng.uniform(-2, 2, 12)]
    kw = dict(ptarget=np.r_[gc[:7], np.zeros(12)], vtarget=np.zeros(18), kp=np.r_[np.zeros(6), 50.0 * np.ones(12)], kd=np.r_[np.zeros(6), 1.0 * np.ones(12)])
    cases.append((a, gc, gv, [0, 3, 8, 12], rng.uniform(-0.1, 0.1, (4, 3)), kw))
    for t, gc, gv, body, pos, kw in cases:
        rot = np.tile(ROT, (len(body), 1, 1))
        e1, big = _fd_error(t, gc, gv, 2e-3, body, pos, rot, kw)
        e2, _ = _fd_error(t, gc, gv, 1e-3, body, pos, rot, kw)
        assert big > 1.0
        assert e1 < 0.05 * big, (e1, big)
        assert 1.6 < e1 / e2 < 2.5, (e1, e2)


def test_launch_mean_is_the_mean_of_the_substeps(anymal_tables):
    t = anymal_tables
    rng = np.random.default_rng(4)
    gc = np.zeros((1, t["nq"])); gc[0, 2] = 1.0; gc[0, 3] = 1.0; gc[0, 7:] = rng.uniform(-0.3, 0.3, 12)
    gv = rng.uniform(-1, 1, (1, t["nv"]))
    gcs, gvs = _trajectory(t, gc, gv, 4, DT, {})
    lin, ang = imu_launch(t, gcs[:, 0], gvs[:, 0], DT, [0, 5], np.zeros((2, 3)))
    subs = [imu_substep(t, gcs[s, 0], gvs[s, 0], gvs[s + 1, 0], DT, [0, 5], np.zeros((2, 3))) for s in range(4)]
    assert np.abs(lin - np.mean([s[0] for s in subs], 0)).max() < 1e-12
    assert np.abs(ang - np.mean([s[1] for s in subs], 0)).max() < 1e-12


def test_the_two_exports_are_declared():
    assert capi.SIGNATURES["rsb_batch_set_imus"] == [capi._P, capi._P, capi._P, capi._P, capi._I]
    assert capi.SIGNATURES["rsb_batch_get_imu_readings"] == [capi._P, capi._I, capi._I, capi._P, capi._P, capi._I]
