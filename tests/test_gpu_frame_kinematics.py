"""Frame kinematics on the GPU (pytest -m gpu): rsb_batch_set_frames, rsb_batch_get_frame_states and rsb_batch_get_frame_jacobians
against the numpy restatement of tests/frame_ref.py, on the poses of every compiled instance's kinematics pass; laziness, launch
count and freedom from side effects; environment slices, host and device buffers; refusals; the pybind module.

Bounds.  Poses: the kinematics pass's bounds (3e-6 on rotations, 5e-6 on positions: tests/test_gpu_parity.py), carried through
p + R pos and R rot.  Velocities and Jacobians: twice what the same restatement makes of them in float32 arithmetic from the batch's
own float32 poses, against the float64 restatement from exact poses, plus 1e-6 -- that run has the two error sources of the kernel,
the float32 pose chain and float32 column arithmetic, and differs from it only in the order of the float32 operations."""
import ctypes
import os

import numpy as np
import pytest

from conftest import RSC
from helpers import ANYMAL_GC0, MAX32, PENDULUM_URDF, launch_config, random_state
from frame_ref import batch_frame_kinematics, link_names, model_frames, random_frames

pytestmark = pytest.mark.gpu

N = 512
FEET = ["base", "LF_FOOT", "RF_FOOT", "LH_FOOT", "RH_FOOT"]
# robot description, compiled instance of the step kernel its kinematics pass runs (0 generic, 1 quadruped, 2 humanoid)
INSTANCES = [pytest.param("anymal_c_like.urdf", 1, id="quadruped"), pytest.param("atlas_like.urdf", 2, id="humanoid"),
             pytest.param(MAX32, 0, id="generic-max32"), pytest.param(PENDULUM_URDF, 0, id="generic-pendulum")]


@pytest.fixture(scope="module")
def capi():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from raisimlib_b200 import capi as c
    return c


def _path(src):
    return os.path.join(RSC, src) if src.endswith(".urdf") else src


def _random_batch(capi, src, n, seed):
    """n random_state environments and every model frame plus 8 random frames: (model, tables, batch, frame names, body, pos, rot)"""
    m = capi.Model(_path(src))
    t = m.tables()
    bt = capi.Batch(m, n)
    rng = np.random.default_rng(seed)
    gc, gv = random_state(t, rng, n, pos_scale=2.0)
    bt.set_state(gc.astype(np.float32), gv.astype(np.float32))
    names = link_names(_path(src))
    fb, fp, fr = model_frames(capi, m, names)
    rb, rp, rr = random_frames(rng, t["nb"], 8)
    return m, t, bt, names, np.r_[fb, rb], np.r_[fp.astype(np.float32), rp], np.r_[fr.astype(np.float32), rr]


def _standing(capi, n, seed):
    """ANYmal-like robots standing on the ground under PD control (contacts on every foot)"""
    m = capi.Model(_path("anymal_c_like.urdf"))
    bt = capi.Batch(m, n)
    bt.set_ground(0.0)
    rng = np.random.default_rng(seed)
    gc = np.tile(ANYMAL_GC0, (n, 1)); gc[:, 2] = 0.55; gc[:, 7:] += rng.uniform(-0.1, 0.1, (n, 12))
    gv = 0.2 * rng.standard_normal((n, 18))
    bt.set_pd_gains(np.r_[np.zeros(6), 300.0 * np.ones(12)], np.r_[np.zeros(6), 8.0 * np.ones(12)])
    bt.set_pd_target(np.tile(ANYMAL_GC0, (n, 1)).astype(np.float32), np.zeros((n, 18), np.float32))
    bt.set_state(gc.astype(np.float32), gv.astype(np.float32))
    return m, m.tables(), bt


def _check(t, bt, body, pos, rot, got, J, label):
    """frame states `got` and Jacobians J of the whole batch against the restatement at the batch's current state"""
    x, Rf, lin, ang = got
    gc, gv = (a.astype(np.float64) for a in bt.get_state())
    R, p = bt.body_poses()
    ref = batch_frame_kinematics(t, gc, gv, body, pos, rot)
    r32 = batch_frame_kinematics(t, gc, gv, body, pos, rot, poses=(R, p), dtype=np.float32)
    tol_x = 5e-6 + 3e-6 * np.abs(pos).sum(1)                           # [F]
    tol_R = 3e-6 * np.abs(rot).sum(1)                                  # [F, 3] column sums
    ex, eR = np.abs(x - ref[0]), np.abs(Rf - ref[1])
    err = lambda a, b: np.abs(a - b).max()
    tol_v = 2 * max(err(r32[2], ref[2]), err(r32[3], ref[3])) + 1e-6
    tol_J = 2 * err(r32[4], ref[4]) + 1e-6
    print(f"{label}: pos {ex.max():.1e}  rot {eR.max():.1e}  vel {max(err(lin, ref[2]), err(ang, ref[3])):.1e} (bound {tol_v:.1e})  "
          f"J {err(J, ref[4]):.1e} (bound {tol_J:.1e})")
    assert (ex <= tol_x[None, :, None]).all() and (eR <= tol_R[None, :, None, :]).all()
    assert err(lin, ref[2]) <= tol_v and err(ang, ref[3]) <= tol_v and err(J, ref[4]) <= tol_J
    # J gv (float64 product of the float32 values) is the returned velocity to float32 rounding of its sum
    Jd, gvd = J.astype(np.float64), gv.astype(np.float32).astype(np.float64)
    Jv, scale = np.einsum("efrc,ec->efr", Jd, gvd), np.einsum("efrc,ec->efr", np.abs(Jd), np.abs(gvd))
    assert (np.abs(Jv - np.concatenate([lin, ang], 2)) <= 1e-6 * scale).all()
    # non-ancestor columns (the reference's zero columns: an ancestor's column has a unit axis in it) are exactly 0
    assert (np.abs(J).max(2)[np.abs(ref[4]).max(2) == 0] == 0).all()


@pytest.mark.parametrize("src,spec", INSTANCES)
def test_frames_match_restatement(capi, monkeypatch, src, spec):
    """every model frame and 8 random frames, 512 random environments: poses, velocities and Jacobians against the restatement;
    frames at a body origin with identity rotation are the body poses bit for bit; set_frames_by_name is set_frames"""
    monkeypatch.delenv("RSB_FORCE_GENERIC", raising=False)
    m, t, bt, names, body, pos, rot = _random_batch(capi, src, N, seed=41)
    assert launch_config(capi, bt)["spec"] == spec
    bt.set_frames(body, pos, rot)
    got, J = bt.frame_states(), bt.frame_jacobians()
    assert J.shape == (N, len(body), 6, t["nv"])
    _check(t, bt, body, pos, rot, got, J, src[:20])
    R, p = bt.body_poses()
    origin = np.where((pos == 0).all(1) & (rot == np.eye(3, dtype=np.float32)).all((1, 2)))[0]
    assert len(origin) >= t["nb"] - 1
    assert np.array_equal(got[0][:, origin].view(np.uint32), p[:, body[origin]].view(np.uint32))
    assert np.array_equal(got[1][:, origin].view(np.uint32), R[:, body[origin]].view(np.uint32))
    bt.set_frames_by_name(names)
    by_name = bt.frame_states()
    for a, b in zip(by_name, got):
        assert np.array_equal(a.view(np.uint32), b[:, :len(names)].view(np.uint32))


def _records(bt):
    ct, cnt = bt.contacts()
    return [ct.tobytes(), cnt, bt.contact_points(), bt.solver_iterations(), bt.solver_status(), bt.solver_residual(), bt.diverged(),
            bt.generalized_force()]


def test_lazy_launch_count_and_no_side_effects(capi):
    """after integrate(4) the getters describe the new state (one kinematics pass, then the frame kernel: 2 launches; 1 while the poses
    are current) and leave the records of the last integrate() bit for bit as they were"""
    m, t, bt = _standing(capi, 256, seed=7)
    body, pos, rot = model_frames(capi, m, FEET)
    pos, rot = pos.astype(np.float32), rot.astype(np.float32)
    bt.set_frames_by_name(FEET)
    bt.integrate(4)
    before = _records(bt)
    assert before[1].sum() > 256
    c0 = bt.launch_count()
    got = bt.frame_states()
    assert bt.launch_count() == c0 + 2
    J = bt.frame_jacobians()
    assert bt.launch_count() == c0 + 3
    for a, b in zip(before, _records(bt)):
        assert np.array_equal(np.asarray(a), np.asarray(b))
    _check(t, bt, body, pos, rot, got, J, "after integrate(4)")
    gc, gv = bt.get_state()
    bt.set_state(gc, 2 * gv)                     # a state written through the API makes the poses stale again
    c1 = bt.launch_count()
    got = bt.frame_states()
    assert bt.launch_count() == c1 + 2
    _check(t, bt, body, pos, rot, got, bt.frame_jacobians(), "after set_state")
    # integrate1() + integrate2(): the step writes the getters' buffers with the poses from before it; the frame getters run the
    # kinematics pass for the stepped state rather than pair those poses with the new velocities
    bt.integrate1()
    bt.integrate2()
    c2 = bt.launch_count()
    got = bt.frame_states()
    assert bt.launch_count() == c2 + 2
    _check(t, bt, body, pos, rot, got, bt.frame_jacobians(), "after integrate1 + integrate2")
    assert bt.launch_count() == c2 + 3


def test_getters_leave_the_trajectory_alone(capi):
    """ten control steps with both getters between each are bit for bit ten control steps without"""
    n = 256
    (_, _, a), (_, _, b) = _standing(capi, n, seed=9), _standing(capi, n, seed=9)
    a.set_frames_by_name(FEET)
    target = np.tile(ANYMAL_GC0, (n, 1)).astype(np.float32)
    for _ in range(10):
        oa = a.control_step(target, 4, np.empty((n, a.ob_dim()), np.float32))
        a.frame_states(); a.frame_jacobians()
        ob = b.control_step(target, 4, np.empty((n, b.ob_dim()), np.float32))
        assert np.array_equal(oa, ob)
    for x, y in zip(a.get_state() + tuple(_records(a)), b.get_state() + tuple(_records(b))):
        assert np.array_equal(np.asarray(x), np.asarray(y))


def test_slices_and_buffers(capi):
    """environment slices equal the full read; torch CUDA outputs equal host outputs bit for bit; NULL outputs are skipped; the
    device forms check dtype, shape, contiguity and device"""
    import torch
    n = 300
    m, t, bt, names, body, pos, rot = _random_batch(capi, "anymal_c_like.urdf", n, seed=13)
    bt.set_frames(body, pos, rot)
    F, nv = len(body), t["nv"]
    full, Jf = bt.frame_states(), bt.frame_jacobians()
    for a, b in zip(bt.frame_states(17, 100), full):
        assert np.array_equal(a, b[17:117])
    assert np.array_equal(bt.frame_jacobians(n - 5, 5), Jf[n - 5:])
    dev = [torch.full((n, F) + s, np.nan, dtype=torch.float32, device="cuda") for s in ((3,), (3, 3), (3,), (3,))]
    jac = torch.full((n, F, 6, nv), np.nan, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()                     # the fills run on torch's stream, the frame kernel on the batch's own
    bt.frame_states_into(*dev)
    bt.frame_jacobians_into(jac)
    bt.sync()
    for d, h in zip(dev, full):
        assert np.array_equal(d.cpu().numpy().view(np.uint32), h.view(np.uint32))
    assert np.array_equal(jac.cpu().numpy().view(np.uint32), Jf.view(np.uint32))
    part = torch.full((100, F, 3), np.nan, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    bt.frame_states_into(lin_vel=part, env_begin=17, env_count=100)
    bt.sync()
    assert np.array_equal(part.cpu().numpy(), full[2][17:117])
    # NULL outputs: skipped, the others written
    L = capi.lib()
    xp, av = np.full((n, F, 3), np.nan, np.float32), np.full((n, F, 3), np.nan, np.float32)
    vp = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    assert L.rsb_batch_get_frame_states(bt.h, 0, n, vp(xp), None, None, vp(av), capi.HOST) == 0
    assert np.array_equal(xp, full[0]) and np.array_equal(av, full[3])
    c0 = bt.launch_count()
    assert L.rsb_batch_get_frame_states(bt.h, 0, n, None, None, None, None, capi.HOST) == 0
    assert bt.launch_count() == c0
    for bad in (torch.zeros((n, F, 3), dtype=torch.float64, device="cuda"), torch.zeros((n, F, 4), device="cuda"),
                torch.zeros((F, n, 3), device="cuda").transpose(0, 1), torch.zeros((n, F, 3))):
        with pytest.raises(ValueError):
            bt.frame_states_into(pos=bad)


def test_refusals_keep_the_frames(capi):
    """each refusal returns RSB_ERR_INVALID and the frames set before it give the same results"""
    n = 64
    m, t, bt, names, body, pos, rot = _random_batch(capi, "atlas_like.urdf", n, seed=17)
    L = capi.lib()
    vp = lambda a: None if a is None else a.ctypes.data_as(ctypes.c_void_p)
    out = [np.empty((n, 70, 9), np.float32) for _ in range(4)]
    jac = np.empty((n, 70, 6, t["nv"]), np.float32)
    states = lambda b, c: L.rsb_batch_get_frame_states(bt.h, b, c, *[vp(o) for o in out], capi.HOST)
    jacobians = lambda b, c, j=jac: L.rsb_batch_get_frame_jacobians(bt.h, b, c, vp(j), capi.HOST)
    assert states(0, n) == -1 and jacobians(0, n) == -1                       # no frames set yet
    bt.set_frames(body, pos, rot)
    ref, ref_j = bt.frame_states(), bt.frame_jacobians()
    many = np.zeros(65, np.int32)
    p65, r65 = np.zeros((65, 3), np.float32), np.tile(np.eye(3, dtype=np.float32), (65, 1, 1))
    refused = [
        L.rsb_batch_set_frames(bt.h, vp(body), vp(pos), vp(rot), -1),
        L.rsb_batch_set_frames(bt.h, vp(many), vp(p65), vp(r65), 65),
        L.rsb_batch_set_frames(bt.h, vp(np.array([0, t["nb"]], np.int32)), vp(pos[:2]), None, 2),
        L.rsb_batch_set_frames(bt.h, vp(np.array([-1], np.int32)), vp(pos[:1]), None, 1),
        L.rsb_batch_set_frames(bt.h, None, vp(pos), None, 3),
        L.rsb_batch_set_frames(bt.h, vp(body), None, None, 3),
        states(-1, 4), states(n - 2, 4), states(0, -1), jacobians(n, 1), jacobians(0, n, None),
    ]
    assert refused == [-1] * len(refused)
    for a, b in zip(bt.frame_states(), ref):                                  # the refusals left the frames as they were
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    assert np.array_equal(bt.frame_jacobians().view(np.uint32), ref_j.view(np.uint32))
    assert L.rsb_batch_set_frames(bt.h, vp(body), vp(pos), None, 0) == 0      # n = 0 clears ...
    assert states(0, n) == -1                                                 # ... and the getters refuse again
    bt.set_frames(body, pos, rot)
    with pytest.raises(capi.RsbError):
        bt.set_frames(np.r_[body, t["nb"]], np.r_[pos, pos[:1]])
    assert bt.nframes == len(body)
    for a, b in zip(bt.frame_states(), ref):
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    assert np.array_equal(bt.frame_jacobians().view(np.uint32), ref_j.view(np.uint32))


def test_pybind_frame_states(capi):
    """_rsb_py.Batch.frame_states / frame_jacobians into torch tensors equal the capi host reads"""
    import torch
    from raisimlib_b200 import _rsb_py
    n = 128
    m, t, bt, names, body, pos, rot = _random_batch(capi, "anymal_c_like.urdf", n, seed=23)
    bt.set_frames(body, pos, rot)
    ref, ref_j = bt.frame_states(), bt.frame_jacobians()
    gc, gv = bt.get_state()
    pb = _rsb_py.Batch(_rsb_py.Model(_path("anymal_c_like.urdf")), n, 0)
    torch.from_dlpack(pb.gc()).copy_(torch.from_numpy(gc).cuda()); torch.from_dlpack(pb.gv()).copy_(torch.from_numpy(gv).cuda())
    torch.cuda.synchronize()
    pb.update_kinematics()                       # the state was written through the device views
    pb.set_frames(body.tolist(), pos.reshape(-1).tolist(), rot.reshape(-1).tolist())
    F = len(body)
    dev = [torch.empty((n, F) + s, dtype=torch.float32, device="cuda") for s in ((3,), (3, 3), (3,), (3,))]
    jac = torch.empty((n, F, 6, t["nv"]), dtype=torch.float32, device="cuda")
    c0 = pb.launch_count
    pb.frame_states(*[d.data_ptr() for d in dev])
    pb.frame_jacobians(jac.data_ptr())
    pb.sync()
    assert pb.launch_count == c0 + 2
    for d, h in zip(dev, ref):
        assert np.array_equal(d.cpu().numpy().view(np.uint32), h.view(np.uint32))
    assert np.array_equal(jac.cpu().numpy().view(np.uint32), ref_j.view(np.uint32))
    pb.frame_states(dev[0].data_ptr(), 0, 0, 0)     # 0 skips an output
    with pytest.raises(RuntimeError):
        pb.set_frames([t["nb"]], [0.0, 0.0, 0.0], [])


def test_batch_on_another_device(capi):
    """a batch on cuda:1 read while cuda:0 is current, with poses stale and current, into device and host buffers, equals the reads made
    with its own device current"""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    m = capi.Model(_path("anymal_c_like.urdf"))
    t = m.tables()
    n = 64
    torch.cuda.set_device(1)
    bt = capi.Batch(m, n, device=1)
    gc, gv = random_state(t, np.random.default_rng(29), n, pos_scale=2.0)
    bt.set_state(gc.astype(np.float32), gv.astype(np.float32))
    bt.set_frames_by_name(FEET)
    ref, ref_j = bt.frame_states(), bt.frame_jacobians()
    bt.set_state(gc.astype(np.float32), gv.astype(np.float32))       # stale again
    torch.cuda.set_device(0)
    jac = torch.empty((n, len(FEET), 6, t["nv"]), device="cuda:1")
    bt.frame_jacobians_into(jac)                                     # stale poses: kinematics pass + frame kernel
    got = bt.frame_states()                                          # current poses, host read: the frame kernel alone
    bt.sync()
    assert np.array_equal(jac.cpu().numpy(), ref_j)
    for a, b in zip(got, ref):
        assert np.array_equal(a, b)
    torch.cuda.set_device(1)
    for a, b in zip(bt.frame_states(), ref):
        assert np.array_equal(a, b)
    torch.cuda.set_device(0)
