"""Terrain height scans on the GPU (pytest -m gpu): rsb_batch_set_height_scan / rsb_batch_get_height_scan against the float64 restatement
of tests/height_scan_ref.py on the root pose from gc and on the kinematics pass of every compiled instance; exact cases; the terrain
atlas; laziness, launch counts and freedom from side effects; environment slices, host, pinned and device buffers; refusals; the
pybind module and the C++ example.

Bounds.  Sample locations: the kinematics pass's bounds (5e-6 on positions, 3e-6 on rotation entries: tests/test_gpu_parity.py) plus
four float32 roundings of the coordinates, carried through the offset; the heading (R00, R10) / |(R00, R10)| turns an entry error e
into an angle error of at most 2 e / |(R00, R10)|, so samples are compared where that norm is at least 0.05 (a body that points nearly
straight up has no well-defined heading; such samples are counted and reported).  Heights: compared with the float64 surface at the
GPU's own sample location, within the local slope times the float32 rounding of the grid coordinate (4 eps (|x| + |x0| + size) per
axis, doubled) plus 8 eps of the largest height."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT, RSC
from helpers import ANYMAL_GC0, MAX32, fk_numpy, launch_config, random_state
from height_scan_ref import base_grid, sample_xy, surface_height

pytestmark = pytest.mark.gpu

EPS = 2.0 ** -24
HM = dict(xs=513, ys=513, size=51.2, cx=0.3, cy=-0.2)
INSTANCES = [pytest.param("anymal_c_like.urdf", 1, id="quadruped"), pytest.param("atlas_like.urdf", 2, id="humanoid"),
             pytest.param(MAX32, 0, id="generic-max32")]


@pytest.fixture(scope="module")
def capi():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from raisimlib_b200 import capi as c
    return c


def _path(src):
    return os.path.join(RSC, src) if src.endswith(".urdf") else src


def _rough(seed, xs=HM["xs"], ys=HM["ys"], amp=0.10):
    rng = np.random.default_rng(seed)
    return rng.uniform(-amp, amp, (ys, xs)).astype(np.float32)


def _batch(capi, src, n, seed, H=None, pos_scale=20.0):
    m = capi.Model(_path(src))
    t = m.tables()
    bt = capi.Batch(m, n)
    H = _rough(seed) if H is None else H
    bt.set_heightmap(H.shape[1], H.shape[0], HM["size"], HM["size"], HM["cx"], HM["cy"], H)
    gc, gv = random_state(t, np.random.default_rng(seed), n, pos_scale=pos_scale)
    bt.set_state(gc.astype(np.float32), gv.astype(np.float32))
    return m, t, bt, H


def _poses64(t, gc):
    R, p = zip(*[fk_numpy(t, g)[:2] for g in gc.astype(np.float64)])
    return np.stack(R), np.stack(p)


def _height_tol(H, sxy):
    """bound on |height - float64 surface at the sample sxy [..., 2]| for the map H laid out as HM (module docstring)"""
    x0, y0 = HM["cx"] - HM["size"] / 2, HM["cy"] - HM["size"] / 2
    Hd = H.astype(np.float64)
    slope = max(np.abs(np.diff(Hd, axis=1)).max(), np.abs(np.diff(Hd, axis=0)).max(), np.abs(Hd[1:, 1:] - Hd[:-1, :-1]).max()) / (HM["size"] / (H.shape[1] - 1))
    dpos = 4 * EPS * (np.abs(sxy).sum(-1) + abs(x0) + abs(y0) + 2 * HM["size"])
    return 2 * slope * dpos + 8 * EPS * np.abs(Hd).max() + 1e-7


def _check(t, bt, H, body, xy, yaw, label):
    """the scan of the whole batch against the restatement at its current state"""
    h, sxy = bt.height_scan()
    gc = bt.get_state()[0]
    R, p = _poses64(t, gc)
    ref = sample_xy(R, p, body, xy, yaw)
    nrm = np.hypot(R[:, body, 0, 0], R[:, body, 1, 0])
    off = np.abs(xy.astype(np.float64)).sum(1)[None]
    tol_xy = 5e-6 + 8 * EPS * (np.abs(p[:, body, :2]).max(2) + off) + (6e-6 / np.maximum(nrm, 0.05) * off if yaw else 0.0)
    ok = (nrm >= 0.05) if yaw else np.ones_like(nrm, bool)
    exy = np.abs(sxy - ref).max(2)
    tol_h = _height_tol(H, sxy)
    href = surface_height(H, HM["size"], HM["size"], HM["cx"], HM["cy"], sxy[..., 0], sxy[..., 1])
    eh = np.abs(h - href)
    print(f"{label}: xy {exy[ok].max():.1e} (worst / bound {(exy / tol_xy)[ok].max():.2f}; {int((~ok).sum())} samples without a heading)  "
          f"height {eh.max():.1e} (worst / bound {(eh / tol_h).max():.2f})")
    assert (exy[ok] <= np.broadcast_to(tol_xy, exy.shape)[ok]).all()
    assert (~ok).mean() < 0.02
    assert (eh <= tol_h).all()
    return h, sxy


def test_base_points_match_reference(capi, monkeypatch):
    """512 ANYmal-like robots at random poses over the 513 x 513 map (many samples off the map): the 187-point grid, yaw-aligned and
    world-aligned, against the restatement; a base-only list is one launch after a state change and never runs the kinematics pass"""
    monkeypatch.delenv("RSB_FORCE_GENERIC", raising=False)
    m, t, bt, H = _batch(capi, "anymal_c_like.urdf", 512, seed=11, pos_scale=30.0)
    xy = base_grid()
    body = np.zeros(len(xy), np.int32)
    for yaw in (True, False):
        bt.set_height_scan(body, xy, "yaw" if yaw else "world")
        l0 = bt.launch_count()
        _check(t, bt, H, body, xy, yaw, f"base grid {'yaw' if yaw else 'world'}")
        assert bt.launch_count() - l0 == 1
    bt.integrate(4)
    l0 = bt.launch_count()
    bt.height_scan()
    assert bt.launch_count() - l0 == 1


@pytest.mark.parametrize("src,spec", INSTANCES)
def test_body_points_match_reference(capi, monkeypatch, src, spec):
    """points on every body (random offsets, both alignments) on the poses of each compiled instance's kinematics pass"""
    monkeypatch.delenv("RSB_FORCE_GENERIC", raising=False)
    m, t, bt, H = _batch(capi, src, 256, seed=23)
    assert launch_config(capi, bt)["spec"] == spec
    rng = np.random.default_rng(5)
    body = np.repeat(np.arange(t["nb"], dtype=np.int32), 3)
    xy = rng.uniform(-0.6, 0.6, (len(body), 2)).astype(np.float32)
    for yaw in (True, False):
        bt.set_height_scan(body, xy, "yaw" if yaw else "world")
        _check(t, bt, H, body, xy, yaw, f"{src[:16]} {'yaw' if yaw else 'world'}")


def test_exact_cases(capi):
    """ground: exactly its z; a constant map: exactly the constant inside and outside; outside a rough map: the clamped border values;
    a NaN state: NaN heights; a base pitched by 90 degrees: finite heights along the world axes"""
    n = 64
    m, t, bt, H = _batch(capi, "anymal_c_like.urdf", n, seed=3, pos_scale=10.0)
    rng = np.random.default_rng(8)
    xy = rng.uniform(-40, 40, (200, 2)).astype(np.float32)
    body = np.zeros(len(xy), np.int32)
    bt.set_height_scan(body, xy, "yaw")
    bt.set_ground(0.37)
    h, _ = bt.height_scan()
    assert (h == np.float32(0.37)).all()
    bt.set_heightmap(33, 33, 8.0, 8.0, 0.0, 0.0, np.full((33, 33), -0.21, np.float32))
    h, sxy = bt.height_scan()
    assert (h == np.float32(-0.21)).all() and (np.abs(sxy) > 4.0).any() and (np.abs(sxy).max(2) < 4.0).any()
    bt.set_heightmap(H.shape[1], H.shape[0], HM["size"], HM["size"], HM["cx"], HM["cy"], H)
    h, sxy = bt.height_scan()
    half = HM["size"] / 2
    cx_, cy_ = np.clip(sxy[..., 0].astype(np.float64), HM["cx"] - half, HM["cx"] + half), np.clip(sxy[..., 1].astype(np.float64), HM["cy"] - half, HM["cy"] + half)
    out = (cx_ != sxy[..., 0]) | (cy_ != sxy[..., 1])
    assert out.sum() > 1000
    href = surface_height(H, HM["size"], HM["size"], HM["cx"], HM["cy"], cx_, cy_)
    assert (np.abs(h - href) <= _height_tol(H, sxy))[out].all()
    far = np.array([[-1e4, -1e4]], np.float32)
    bt.set_height_scan([0], far, "world")
    assert (bt.height_scan()[0] == H[0, 0]).all()
    gc, gv = bt.get_state()
    gc[5, :3] = np.nan
    gc[6, 3:7] = np.nan
    gc[7, :7] = [1.0, 2.0, 0.5, np.cos(np.pi / 4), 0.0, np.sin(np.pi / 4), 0.0]     # pitched by 90 degrees
    bt.set_state(gc, gv)
    bt.set_height_scan(body, xy, "yaw")
    h, sxy = bt.height_scan()
    assert np.isnan(h[5]).all() and np.isnan(h[6]).all()
    assert np.isfinite(np.delete(h, [5, 6], 0)).all()
    assert np.abs(sxy[7] - (np.array([1.0, 2.0], np.float32) + xy)).max() < 1e-5


def test_terrain_atlas_and_replaced_terrain(capi):
    """environment e's scan is bit for bit that of a one-map batch holding map_of_env[e]; a replaced terrain is read by the next scan"""
    n, count = 96, 3
    maps = np.stack([_rough(40 + k, 129, 129, amp=0.2) for k in range(count)])
    moe = (np.arange(n) * 7 % count).astype(np.int32)
    m, t, bt, _ = _batch(capi, "anymal_c_like.urdf", n, seed=41, H=maps[0], pos_scale=8.0)
    bt.set_heightmaps(HM["size"], HM["size"], HM["cx"], HM["cy"], maps, moe)
    body = np.array([0] * 20 + [3] * 10, np.int32)
    xy = np.random.default_rng(2).uniform(-1, 1, (len(body), 2)).astype(np.float32)
    bt.set_height_scan(body, xy, "yaw")
    h, sxy = bt.height_scan()
    gc, gv = bt.get_state()
    for k in range(count):
        one = capi.Batch(m, n)
        one.set_heightmap(129, 129, HM["size"], HM["size"], HM["cx"], HM["cy"], maps[k])
        one.set_state(gc, gv)
        one.set_height_scan(body, xy, "yaw")
        hk, xk = one.height_scan()
        sel = moe == k
        assert np.array_equal(hk[sel].view(np.uint32), h[sel].view(np.uint32)) and np.array_equal(xk.view(np.uint32), sxy.view(np.uint32))
    bt.set_heightmap(129, 129, HM["size"], HM["size"], HM["cx"], HM["cy"], maps[2] + 1.0)
    h2, _ = bt.height_scan()
    assert np.abs(h2 - surface_height(maps[2] + np.float32(1.0), HM["size"], HM["size"], HM["cx"], HM["cy"], sxy[..., 0], sxy[..., 1])).max() < 1e-4
    bt.clear_terrain()
    with pytest.raises(capi.RsbError, match="no terrain"):
        bt.height_scan()


def _records(bt):
    ct, cnt = bt.contacts()
    return [bt.get_state()[0].tobytes(), bt.get_state()[1].tobytes(), ct.tobytes(), cnt.tobytes(), bt.contact_points().tobytes(),
            bt.solver_iterations().tobytes(), bt.solver_status().tobytes(), bt.solver_residual().tobytes(), bt.diverged().tobytes(),
            bt.generalized_force().tobytes(), bt.body_contact_forces()[0].tobytes()]


def _standing(capi, n, seed, H):
    m = capi.Model(_path("anymal_c_like.urdf"))
    bt = capi.Batch(m, n)
    bt.set_heightmap(H.shape[1], H.shape[0], HM["size"], HM["size"], HM["cx"], HM["cy"], H)
    rng = np.random.default_rng(seed)
    gc = np.tile(ANYMAL_GC0, (n, 1)); gc[:, 2] = 0.56 + 0.1; gc[:, 7:] += rng.uniform(-0.1, 0.1, (n, 12))
    bt.set_pd_gains(np.r_[np.zeros(6), 300.0 * np.ones(12)], np.r_[np.zeros(6), 8.0 * np.ones(12)])
    bt.set_pd_target(np.tile(ANYMAL_GC0, (n, 1)).astype(np.float32), np.zeros((n, 18), np.float32))
    bt.set_state(gc.astype(np.float32), (0.2 * rng.standard_normal((n, 18))).astype(np.float32))
    bt.set_contact_bodies([m.body_index(f"{leg}_FOOT") for leg in ("LF", "RF", "LH", "RH")])
    return m, bt


def test_no_side_effects_and_launch_counts(capi):
    """a root-only list adds exactly one launch, also right after integrate; a list with a foot point adds two after a state change
    (the kinematics pass, then the scan) and then one; after a scan the state, contacts, contact forces and solver outputs are as they
    were, and the next integrate is bit for bit that of a batch that never scanned"""
    n, H = 256, _rough(5, amp=0.05)
    m, a = _standing(capi, n, 9, H)
    _, b = _standing(capi, n, 9, H)
    foot = m.body_index("LF_FOOT")
    xy = base_grid()
    for k in range(3):
        a.integrate(4); b.integrate(4)
        before = _records(a)
        a.set_height_scan(np.zeros(len(xy), np.int32), xy, "yaw")
        a.integrate(4); b.integrate(4)
        l0 = a.launch_count(); a.height_scan(); assert a.launch_count() - l0 == 1
        a.set_height_scan(np.r_[np.zeros(4, np.int32), [foot]], np.zeros((5, 2), np.float32), "world")
        l0 = a.launch_count(); a.height_scan(); assert a.launch_count() - l0 == 2
        l0 = a.launch_count(); a.height_scan(); assert a.launch_count() - l0 == 1
        assert before != _records(a)     # the state moved on
        after = _records(a)
        a.height_scan(); a.height_scan()
        assert after == _records(a)
    a.integrate(4); b.integrate(4)
    assert _records(a) == _records(b)


def test_slices_buffers_and_null_outputs(capi):
    """environment slices, pageable, pinned and device outputs and NULL outputs all give the whole-batch scan's values"""
    import torch
    n = 300
    m, t, bt, H = _batch(capi, "anymal_c_like.urdf", n, seed=17)
    body = np.array([0] * 30 + [6] * 10, np.int32)
    xy = np.random.default_rng(1).uniform(-1, 1, (len(body), 2)).astype(np.float32)
    bt.set_height_scan(body, xy, "yaw")
    h, sxy = bt.height_scan()
    hs, xs = bt.height_scan(100, 57)
    assert np.array_equal(hs.view(np.uint32), h[100:157].view(np.uint32)) and np.array_equal(xs.view(np.uint32), sxy[100:157].view(np.uint32))
    P = len(body)
    ph, pxy = torch.empty((n, P)).pin_memory(), torch.empty((n, P, 2)).pin_memory()
    L = capi.lib()
    assert L.rsb_batch_get_height_scan(bt.h, 0, n, C.c_void_p(ph.data_ptr()), C.c_void_p(pxy.data_ptr()), capi.HOST) == 0
    assert np.array_equal(ph.numpy().view(np.uint32), h.view(np.uint32)) and np.array_equal(pxy.numpy().view(np.uint32), sxy.view(np.uint32))
    dh, dxy = torch.empty((57, P), device="cuda"), torch.empty((57, P, 2), device="cuda")
    bt.height_scan_into(dh, dxy, 100, 57)
    torch.cuda.synchronize()
    assert np.array_equal(dh.cpu().numpy().view(np.uint32), hs.view(np.uint32)) and np.array_equal(dxy.cpu().numpy().view(np.uint32), xs.view(np.uint32))
    only = np.full((n, P), -7.0, np.float32)
    assert L.rsb_batch_get_height_scan(bt.h, 0, n, only.ctypes.data_as(C.c_void_p), None, capi.HOST) == 0
    assert np.array_equal(only.view(np.uint32), h.view(np.uint32))
    bt.height_scan_into(None, dxy, 100, 57)
    l0 = bt.launch_count()
    bt.height_scan_into(None, None)
    assert L.rsb_batch_get_height_scan(bt.h, 0, 0, only.ctypes.data_as(C.c_void_p), None, capi.HOST) == 0
    assert bt.launch_count() == l0
    with pytest.raises(ValueError):
        bt.height_scan_into(torch.empty((n, P + 1), device="cuda"))
    with pytest.raises(ValueError):
        bt.height_scan_into(torch.empty((n, P), dtype=torch.float64, device="cuda"))


def test_refusals_keep_the_previous_list(capi):
    """every refused set_height_scan leaves the previous list working; a bad range or `where` is refused before anything is enqueued"""
    n = 32
    m, t, bt, H = _batch(capi, "anymal_c_like.urdf", n, seed=29)
    L = capi.lib()
    body, xy = np.array([0, 2], np.int32), np.array([[0.1, 0.2], [-0.3, 0.0]], np.float32)
    bt.set_height_scan(body, xy, "yaw")
    good = bt.height_scan()
    bd, pp = body.ctypes.data_as(C.c_void_p), xy.ctypes.data_as(C.c_void_p)
    bad_body = np.array([0, t["nb"]], np.int32)
    nan_xy = np.array([[0.1, np.nan], [0.0, 0.0]], np.float32)
    inf_xy = np.array([[0.1, 0.0], [np.inf, 0.0]], np.float32)
    refused = [(bd, pp, -1, 0), (bd, pp, capi.MAX_SCAN_POINTS + 1, 0), (None, pp, 2, 0), (bd, None, 2, 0), (bd, pp, 2, 2), (bd, pp, 2, -1),
               (bad_body.ctypes.data_as(C.c_void_p), pp, 2, 0), (bd, nan_xy.ctypes.data_as(C.c_void_p), 2, 0), (bd, inf_xy.ctypes.data_as(C.c_void_p), 2, 0)]
    for args in refused:
        assert L.rsb_batch_set_height_scan(bt.h, *args) == -1
        again = bt.height_scan()
        assert all(np.array_equal(a.view(np.uint32), b.view(np.uint32)) for a, b in zip(again, good))
    h = np.empty((n, 2), np.float32)
    l0 = bt.launch_count()
    for env_begin, env_count, where in ((0, n, 2), (0, n, -1), (-1, 2, 0), (n - 1, 2, 0), (0, -1, 0)):
        assert L.rsb_batch_get_height_scan(bt.h, env_begin, env_count, h.ctypes.data_as(C.c_void_p), None, where) == -1
    assert bt.launch_count() == l0
    with pytest.raises(ValueError):
        bt.set_height_scan(body, xy, "roll")
    bt.set_height_scan([], np.zeros((0, 2)), "yaw")
    with pytest.raises(capi.RsbError, match="no height-scan points"):
        bt.height_scan()


def test_pybind_entry(capi):
    """the pybind module's set_height_scan / height_scan write what the ctypes binding reads"""
    import torch
    from raisimlib_b200 import _rsb_py
    n = 128
    path = _path("anymal_c_like.urdf")
    H = _rough(31, 129, 129)
    m, t, bt, _ = _batch(capi, "anymal_c_like.urdf", n, seed=31, H=H, pos_scale=5.0)
    pb = _rsb_py.Batch(_rsb_py.Model(path), n, 0)
    pb.set_ground(0.0)
    bt.set_ground(0.0)
    gc, gv = bt.get_state()
    torch.from_dlpack(pb.gc()).copy_(torch.from_numpy(gc).cuda())
    torch.cuda.synchronize()
    body, xy = [0] * 10, np.random.default_rng(0).uniform(-1, 1, (10, 2)).astype(np.float32)
    pb.set_height_scan(body, xy.reshape(-1).tolist(), "world")
    bt.set_height_scan(body, xy, "world")
    dh, dxy = torch.empty((n, 10), device="cuda"), torch.empty((n, 10, 2), device="cuda")
    pb.height_scan(dh.data_ptr(), dxy.data_ptr())
    pb.sync()
    h, sxy = bt.height_scan()
    assert np.array_equal(dh.cpu().numpy(), h) and np.array_equal(dxy.cpu().numpy(), sxy)
    with pytest.raises(RuntimeError, match="align"):
        pb.set_height_scan(body, xy.reshape(-1).tolist(), "up")


def test_cpp_height_scan_example():
    """the raisim:: facade: a 187-point yaw-aligned base grid in an upstream-shaped observe(), one step launch and one scan launch per
    control step, every height equal to HeightMap::getHeight at the returned sample (examples/height_scan.cpp)"""
    exe = os.path.join(ROOT, "examples", "height_scan")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "examples")])
    out = subprocess.run([exe, os.path.join(RSC, "anymal_c_like.urdf")], capture_output=True, text=True, timeout=600)
    print(out.stdout)
    assert out.returncode == 0, out.stdout + out.stderr
