"""The host side of the C-ABI on the GPU (run on an H100: pytest -m gpu): `where` is checked before anything is enqueued, and host
transfers of every size through the batch's staging buffer give exactly what device buffers give."""
import ctypes as C
import os

import numpy as np
import pytest

from helpers import ANYMAL_GC0

pytestmark = pytest.mark.gpu

RSC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "raisimlib_b200", "rsc")
SUB = 4


@pytest.fixture(scope="module")
def capi():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from raisimlib_b200 import capi as c
    return c


def _anymal(capi, n, seed):
    """a standing quadruped batch under PD control on flat ground, with frames, contact bodies and the gym task configured"""
    bt = capi.Batch(capi.Model(os.path.join(RSC, "anymal_c_like.urdf")), n)
    bt.set_ground(0.0)
    rng = np.random.default_rng(seed)
    gc = np.tile(ANYMAL_GC0, (n, 1)); gc[:, :2] = rng.uniform(-2, 2, (n, 2)); gc[:, 2] = 0.56
    gc[:, 7:] += rng.uniform(-0.1, 0.1, (n, 12))
    bt.set_state(gc.astype(np.float32), (0.2 * rng.standard_normal((n, 18))).astype(np.float32))
    bt.set_pd_gains(np.r_[np.zeros(6), 300.0 * np.ones(12)], np.r_[np.zeros(6), 8.0 * np.ones(12)])
    bt.set_pd_target(np.tile(ANYMAL_GC0, (n, 1)).astype(np.float32), np.zeros((n, 18), np.float32))
    bt.set_frames([3, 6, 9], np.array([[0.0, 0.0, -0.3], [0.01, 0.0, -0.3], [0.0, 0.02, -0.3]]))
    bt.set_contact_bodies([3, 6, 9, 12])
    bt.gym_configure(ANYMAL_GC0, np.zeros(18), ANYMAL_GC0[7:], 0.6 * np.ones(12), [3, 6, 9, 12])
    return bt


def test_where_is_checked_before_anything_is_enqueued(capi):
    """every entry point that takes `where` refuses a value other than RSB_HOST / RSB_DEVICE with RSB_ERR_INVALID, and leaves the
    batch, its launch count and the caller's buffers as they were, even when the buffers are valid device memory"""
    import torch
    n, BAD = 64, 2
    bt = _anymal(capi, n, seed=3)
    bt.integrate(SUB)
    L, h = capi.lib(), bt.h
    sentinel = 12345.0
    buf = torch.full((1 << 18,), sentinel, dtype=torch.float32, device="cuda")      # larger than any output of these calls
    out = torch.full((1 << 18,), sentinel, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    p, q = C.c_void_p(buf.data_ptr()), C.c_void_p(out.data_ptr())
    calls = {
        "set_state": lambda: L.rsb_batch_set_state(h, p, p, 0, n, BAD),
        "get_state": lambda: L.rsb_batch_get_state(h, p, q, 0, n, BAD),
        "set_pd_target": lambda: L.rsb_batch_set_pd_target(h, p, p, 0, n, BAD),
        "set_generalized_force": lambda: L.rsb_batch_set_generalized_force(h, p, 0, n, BAD),
        "get_generalized_force": lambda: L.rsb_batch_get_generalized_force(h, q, 0, n, BAD),
        "set_external_wrench": lambda: L.rsb_batch_set_external_wrench(h, 1, p, p, None, 0, n, BAD),
        "set_body_inertia": lambda: L.rsb_batch_set_body_inertia(h, p, 0, n, BAD),
        "get_mass_matrix": lambda: L.rsb_batch_get_mass_matrix(h, 0, n, q, BAD),
        "get_nonlinearities": lambda: L.rsb_batch_get_nonlinearities(h, 0, n, q, BAD),
        "get_body_poses": lambda: L.rsb_batch_get_body_poses(h, 0, n, q, q, BAD),
        "get_frame_states": lambda: L.rsb_batch_get_frame_states(h, 0, n, q, q, q, q, BAD),
        "get_frame_jacobians": lambda: L.rsb_batch_get_frame_jacobians(h, 0, n, q, BAD),
        "get_body_contact_forces": lambda: L.rsb_batch_get_body_contact_forces(h, 0, n, q, q, BAD),
        "get_contacts": lambda: L.rsb_batch_get_contacts(h, q, q, 0, n, BAD),
        "get_contact_points": lambda: L.rsb_batch_get_contact_points(h, q, 0, n, BAD),
        "get_solver_iterations": lambda: L.rsb_batch_get_solver_iterations(h, q, 0, n, BAD),
        "get_solver_status": lambda: L.rsb_batch_get_solver_status(h, q, 0, n, BAD),
        "get_solver_residual": lambda: L.rsb_batch_get_solver_residual(h, q, 0, n, BAD),
        "get_diverged": lambda: L.rsb_batch_get_diverged(h, q, 0, n, BAD),
        "observe": lambda: L.rsb_batch_observe(h, q, 0, n, BAD),
        "control_step where_in": lambda: L.rsb_batch_control_step(h, p, p, BAD, SUB, q, capi.DEVICE),
        "control_step where_out": lambda: L.rsb_batch_control_step(h, None, None, capi.DEVICE, SUB, q, BAD),
        "gym_step where_in": lambda: L.rsb_batch_gym_step(h, p, BAD, SUB, q, q, q, capi.DEVICE),
        "gym_step where_out": lambda: L.rsb_batch_gym_step(h, p, capi.DEVICE, SUB, q, q, q, BAD),
    }
    gc0, gv0 = bt.get_state()
    launches = bt.launch_count()
    for name, call in calls.items():
        assert call() == -1, f"{name}: where = {BAD} accepted"
        assert "where" in capi.lib().rsb_last_error().decode(), name
        assert bt.launch_count() == launches, f"{name}: launched"
        gc, gv = bt.get_state()
        assert gc.tobytes() == gc0.tobytes() and gv.tobytes() == gv0.tobytes(), f"{name}: the state changed"
    bt.sync()
    torch.cuda.synchronize()
    assert bool((buf == sentinel).all()) and bool((out == sentinel).all()), "a caller buffer was written"
    # the batch still steps as one that never saw those calls
    ref = _anymal(capi, n, seed=3)
    ref.integrate(SUB)
    for b in (bt, ref):
        b.integrate(SUB)
    assert bt.get_state()[0].tobytes() == ref.get_state()[0].tobytes()


def test_host_transfers_through_staging_equal_device_buffers(capi):
    """one interleaved sequence of host transfers of different sizes -- inertia rows, an external wrench, pageable control-step targets
    and observations, state, frame states and Jacobians, observations and applied forces of sub-ranges -- equals, bit for bit, the same
    sequence with device buffers"""
    import torch
    n = 96
    hb, db = _anymal(capi, n, seed=11), _anymal(capi, n, seed=11)
    od, F, nv = hb.ob_dim(), hb.nframes, hb.nv
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    L = capi.lib()
    rng = np.random.default_rng(12)
    model_rows = hb.model_body_inertia()
    for k in range(3):
        e0, ne = 5 + 7 * k, 40 - 9 * k
        rows = np.tile(model_rows, (ne, 1, 1)); rows[:, 0, 0] *= rng.uniform(0.8, 1.3, ne).astype(np.float32)
        force = rng.normal(0, 30, (n - 2, 3)).astype(np.float32)
        torque = rng.normal(0, 3, (n - 2, 3)).astype(np.float32)
        pt = (np.tile(ANYMAL_GC0, (n, 1)) + rng.uniform(-0.15, 0.15, (n, 19))).astype(np.float32)
        vt = rng.normal(0, 0.1, (n, 18)).astype(np.float32)
        got, want = {}, {}

        hb.set_body_inertia(rows, env_begin=e0)
        hb.set_external_wrench(1, force, torque, env_begin=2)
        got["obs_step"] = hb.control_step(pt, SUB, np.empty((n, od), np.float32), vtarget=vt)
        got["gc"], got["gv"] = hb.get_state(env_begin=3, env_count=50)
        got["frames"] = hb.frame_states()
        got["jac"] = hb.frame_jacobians(env_begin=1, env_count=n - 1)
        got["obs"] = hb.observe(env_begin=7, env_count=30)
        got["tau"] = hb.generalized_force(env_begin=4, env_count=60)

        d_rows, d_force, d_torque, d_pt, d_vt = dev(rows), dev(force), dev(torque), dev(pt), dev(vt)
        o_step, o_gc, o_gv = (torch.empty(s, dtype=torch.float32, device="cuda") for s in ((n, od), (50, 19), (50, 18)))
        o_fr = [torch.empty(s, dtype=torch.float32, device="cuda") for s in ((n, F, 3), (n, F, 3, 3), (n, F, 3), (n, F, 3))]
        o_jac, o_obs, o_tau = (torch.empty(s, dtype=torch.float32, device="cuda") for s in ((n - 1, F, 6, nv), (30, od), (60, nv)))
        torch.cuda.synchronize()
        db.set_body_inertia_from(d_rows, env_begin=e0)
        db.set_external_wrench(1, d_force, d_torque, env_begin=2)
        db.control_step(d_pt, SUB, o_step, vtarget=d_vt)
        db.get_state_into(o_gc, o_gv, env_begin=3, env_count=50)
        db.frame_states_into(*o_fr)
        db.frame_jacobians_into(o_jac, env_begin=1, env_count=n - 1)
        db.observe(o_obs, env_begin=7, env_count=30)
        assert L.rsb_batch_get_generalized_force(db.h, C.c_void_p(o_tau.data_ptr()), 4, 60, capi.DEVICE) == 0
        db.sync()
        want.update(obs_step=o_step, gc=o_gc, gv=o_gv, frames=tuple(o_fr), jac=o_jac, obs=o_obs, tau=o_tau)

        for key in got:
            g = got[key] if isinstance(got[key], tuple) else (got[key],)
            w = want[key] if isinstance(want[key], tuple) else (want[key],)
            for a, b in zip(g, w):
                assert a.tobytes() == b.cpu().numpy().tobytes(), f"round {k}: {key} differs between host and device buffers"
    assert hb.launch_count() == db.launch_count()
