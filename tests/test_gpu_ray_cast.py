"""Ray casts on the GPU (pytest -m gpu): rsb_batch_set_rays / rsb_batch_get_ray_casts against the float64 restatement of
tests/ray_cast_ref.py on the quadruped, humanoid and generic (max32: every shape type) instances, with a base camera, foot-mounted rings
and a lidar-like pattern in both targets modes; watertightness on cell boundaries, vertices and diagonals; agreement with the height
scan and the ground plane; the terrain atlas and terrain updates; the origin-inside rule; poses, launch counts and freedom from side
effects, also with every per-environment feature on; slices, host, pinned, device and NULL outputs; diverged environments; refusals;
the pybind module and the C++ example.

Bound: on every ray the reference does not call ambiguous, the hit ids are equal and |t - t_ref| <= 1e-4 m + 2e-6 t."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT, RSC
from helpers import ANYMAL_GC0, MAX32, fk_numpy, launch_config, random_state
from ray_cast_ref import MISS, TERRAIN, ray_casts as ref_casts, world_rays
from terrain_contact_ref import Grid, centres

pytestmark = pytest.mark.gpu

HM = dict(xs=257, ys=257, size=25.6, cx=0.3, cy=-0.2)
INSTANCES = [pytest.param("anymal_c_like.urdf", 1, id="quadruped"), pytest.param("atlas_like.urdf", 2, id="humanoid"),
             pytest.param(MAX32, 0, id="generic-max32")]
MAXD = 4.0


@pytest.fixture(scope="module")
def capi():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from raisimlib_b200 import capi as c
    return c


def _path(src):
    return os.path.join(RSC, src) if src.endswith(".urdf") else src


def _rough(seed, xs=HM["xs"], ys=HM["ys"], amp=0.06):
    rng = np.random.default_rng(seed)
    return rng.uniform(-amp, amp, (ys, xs)).astype(np.float32)


def _grid(H):
    return Grid(H.astype(np.float64), HM["size"], HM["size"], HM["cx"], HM["cy"])


def _batch(capi, src, n, seed, H=None, pos_scale=3.0):
    m = capi.Model(_path(src))
    t = m.tables()
    bt = capi.Batch(m, n)
    H = _rough(seed) if H is None else H
    bt.set_heightmap(H.shape[1], H.shape[0], HM["size"], HM["size"], HM["cx"], HM["cy"], H)
    gc, gv = random_state(t, np.random.default_rng(seed), n, pos_scale=pos_scale)
    bt.set_state(gc.astype(np.float32), gv.astype(np.float32))
    return m, t, bt, H


def _pitched_camera(w, h, hfov, pitch_deg, pos):
    """a pinhole camera at pos on the base, its optical axis pitched down by pitch_deg: (origin [R, 3], dir [R, 3])"""
    from raisimlib_b200 import capi
    d = capi.pinhole_rays(w, h, hfov)
    a = math.radians(pitch_deg)
    Ry = np.array([[math.cos(a), 0, math.sin(a)], [0, 1, 0], [-math.sin(a), 0, math.cos(a)]])   # +x turned towards -z
    return np.tile(np.asarray(pos, np.float64), (len(d), 1)), d @ Ry.T


def _patterns(t):
    """(body, origin, dir) of a 16 x 12 base camera, an 8-ray ring on every body that owns a sphere, and a lidar-like 4 x 48 fan"""
    body, origin, dirs = [], [], []
    o, d = _pitched_camera(16, 12, 87.0, 30.0, [0.3, 0.0, 0.05])
    body += [0] * len(d); origin.append(o); dirs.append(d)
    feet = sorted({int(t["cbody"][c]) for c in range(t["ncoll"]) if t["ctype"][c] == 0 and t["cbody"][c] != 0})[:6]
    ang = np.linspace(0, 2 * np.pi, 8, endpoint=False)
    ring = np.stack([np.cos(ang), np.sin(ang), -np.ones(8)], 1)
    for f in feet:
        body += [f] * 8; origin.append(np.zeros((8, 3))); dirs.append(ring)
    el, az = np.radians(np.linspace(-25, -4, 4)), np.linspace(-np.pi, np.pi, 48, endpoint=False)
    E, A = np.meshgrid(el, az, indexing="ij")
    lid = np.stack([np.cos(E) * np.cos(A), np.cos(E) * np.sin(A), np.sin(E)], -1).reshape(-1, 3)
    body += [0] * len(lid); origin.append(np.tile([0.0, 0.0, 0.15], (len(lid), 1))); dirs.append(lid)
    return np.array(body, np.int32), np.concatenate(origin).astype(np.float32), np.concatenate(dirs).astype(np.float32)


def _reference(t, gc, body, origin, dirs, H, robot, maxd=MAXD):
    g = _grid(H)
    out = []
    for e in range(len(gc)):
        R, p, _ = fk_numpy(t, gc[e].astype(np.float64))
        o, d = world_rays(R[None], p[None], body, origin, dirs.astype(np.float64))
        out.append(ref_casts(o[0], d[0], maxd, ("map", g), t if robot else None, R, p))
    return [np.stack(x) for x in zip(*out)]


def _compare(dist, hit, ref, label):
    rd, rh, amb = ref
    ok = ~amb
    print(f"{label}: {amb.mean() * 100:.2f} % ambiguous, {int((rh[ok] == TERRAIN).sum())} terrain hits, {int((rh[ok] >= 0).sum())} robot hits, "
          f"{int((rh[ok] == MISS).sum())} misses")
    assert amb.mean() < 0.02
    bad = ok & (hit != rh)
    assert not bad.any(), f"{label}: {int(bad.sum())} rays with another hit id, e.g. gpu {hit[bad][:5]} ref {rh[bad][:5]} at {rd[bad][:5]} / {dist[bad][:5]}"
    fin = ok & (rh != MISS)
    err = np.abs(dist[fin] - rd[fin])
    tol = 1e-4 + 2e-6 * rd[fin]
    print(f"{label}: worst |t - t_ref| {err.max() if err.size else 0:.2e} (worst / bound {(err / tol).max() if err.size else 0:.2f})")
    assert (err <= tol).all()
    assert np.isinf(dist[ok & (rh == MISS)]).all()


@pytest.mark.parametrize("src,spec", INSTANCES)
def test_accuracy_against_reference(capi, monkeypatch, src, spec):
    """camera, foot rings and lidar fan on random states of each compiled instance, terrain-only and with the robot"""
    monkeypatch.delenv("RSB_FORCE_GENERIC", raising=False)
    n = 8
    m, t, bt, H = _batch(capi, src, n, seed=3)
    assert launch_config(capi, bt)["spec"] == spec
    bt.integrate(3)                                    # a GPU trajectory state
    body, origin, dirs = _patterns(t)
    gc = bt.get_state()[0]
    for targets in ("terrain", "all"):
        bt.set_rays(body, origin, dirs, MAXD, targets)
        dist, hit = bt.ray_casts()
        ref = _reference(t, gc, body, origin, dirs, H, targets == "all")
        _compare(dist, hit, ref, f"{src if src.endswith('.urdf') else 'max32'} {targets}")
        if targets == "terrain":
            assert (hit < 0).all()


def test_watertight_on_boundaries_vertices_and_diagonals(capi):
    """steep rays aimed exactly at cell boundaries, vertices and diagonals (terrain_contact_ref.centres) never miss where the reference
    hits, and agree with it where it is unambiguous"""
    n = 4
    H = _rough(8, amp=0.2)
    m, t, bt, _ = _batch(capi, "anymal_c_like.urdf", n, seed=8, H=H)
    g = _grid(H)
    gc = np.tile(ANYMAL_GC0, (n, 1)); gc[:, 0] = np.arange(n) * 0.5; gc[:, 1] = -0.3; gc[:, 2] = 1.0
    bt.set_state(gc.astype(np.float32), np.zeros((n, 18), np.float32))
    rng = np.random.default_rng(4)
    X, Y = centres(rng, g, 4000)
    inside = (X > g.x0 + 1.0) & (X < g.x0 + (g.xs - 1) * g.dx - 1.0) & (Y > g.y0 + 1.0) & (Y < g.y0 + (g.ys - 1) * g.dy - 1.0)
    X, Y = X[inside][:2048], Y[inside][:2048]
    Z = np.array([g.height(x, y) for x, y in zip(X, Y)])
    # origins 1 m above and up to 1 m to the side of each target: every ray comes down at 45 degrees or steeper
    side = rng.uniform(-1, 1, (len(X), 2)) / math.sqrt(2)
    o_w = np.stack([X + side[:, 0], Y + side[:, 1], Z + 1.0], 1)
    dirs = np.stack([X, Y, Z], 1) - o_w
    body = np.zeros(len(X), np.int32)
    origin = (o_w - gc[0, :3]).astype(np.float32)      # body frame of environment 0 (identity orientation)
    bt.set_rays(body, origin, dirs.astype(np.float32), 3.0, "terrain")
    dist, hit = bt.ray_casts()
    o = origin.astype(np.float64) + gc[0, :3].astype(np.float32).astype(np.float64)
    d = dirs.astype(np.float32).astype(np.float64)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    rd, rh, amb = ref_casts(o, d, 3.0, ("map", g))
    assert (rh == TERRAIN).all()
    missed = hit[0] != TERRAIN
    assert not missed.any(), f"{int(missed.sum())} rays slipped through, e.g. targets {np.stack([X, Y], 1)[missed][:4]}"
    ok = ~amb
    assert (np.abs(dist[0][ok] - rd[ok]) <= 1e-4 + 2e-6 * rd[ok]).all()
    print(f"watertight: {len(X)} rays, {amb.mean() * 100:.2f} % ambiguous")


def test_consistent_with_height_scan_and_ground(capi):
    """a straight-down ray from a base upright at any heading reads o_z - h, h the height scan at the same xy, within 1e-5 m; on a flat
    map it reads what the ground plane reads"""
    n = 64
    m, t, bt, H = _batch(capi, "anymal_c_like.urdf", n, seed=12)
    rng = np.random.default_rng(12)
    gc = np.tile(ANYMAL_GC0, (n, 1)); gc[:, :2] = rng.uniform(-8, 8, (n, 2)); gc[:, 2] = rng.uniform(0.4, 1.5, n)
    psi = rng.uniform(-np.pi, np.pi, n)
    gc[:, 3], gc[:, 6] = np.cos(psi / 2), np.sin(psi / 2)
    bt.set_state(gc.astype(np.float32), np.zeros((n, 18), np.float32))
    xy = rng.uniform(-1, 1, (100, 2)).astype(np.float32)
    body = np.zeros(len(xy), np.int32)
    bt.set_height_scan(body, xy, "yaw")
    h, _ = bt.height_scan()
    bt.set_rays(body, np.c_[xy, np.zeros(len(xy))], np.tile([0, 0, -1.0], (len(xy), 1)), 5.0, "terrain")
    dist, hit = bt.ray_casts()
    oz = bt.get_state()[0][:, 2:3]
    assert (hit == TERRAIN).all()
    assert np.abs(dist - (oz - h)).max() <= 1e-5
    flat = np.full((33, 33), 0.125, np.float32)
    bt.set_heightmap(33, 33, 40.0, 40.0, 0.0, 0.0, flat)
    body, origin, dirs = _patterns(t)
    bt.set_rays(body, origin, dirs, MAXD, "terrain")
    dm, hm = bt.ray_casts()
    bt.set_ground(0.125)
    dg, hg = bt.ray_casts()
    assert np.array_equal(hm, hg)
    fin = hg == TERRAIN
    assert fin.any() and np.abs(dm[fin] - dg[fin]).max() <= 1e-5 * (1 + dg[fin].max())


def test_terrain_atlas_and_updates(capi):
    """environment e sees its own atlas map (bit for bit a batch whose environments all use that map of the atlas), and the new map
    after set_heightmap_index and update_heightmaps; with no terrain every ray misses"""
    n, count = 48, 3
    maps = np.stack([_rough(40 + k, 129, 129, amp=0.2) for k in range(count)])
    moe = (np.arange(n) * 7 % count).astype(np.int32)
    m, t, bt, _ = _batch(capi, "anymal_c_like.urdf", n, seed=41, H=maps[0])
    bt.set_heightmaps(HM["size"], HM["size"], HM["cx"], HM["cy"], maps, moe)
    body, origin, dirs = _patterns(t)
    bt.set_rays(body, origin, dirs, MAXD, "all")
    gc, gv = bt.get_state()

    def one_map(k):
        """a batch whose environments all use map k of the same atlas (the same hmax, so the same clip of every ray)"""
        one = capi.Batch(m, n)
        one.set_heightmaps(HM["size"], HM["size"], HM["cx"], HM["cy"], maps, np.full(n, k, np.int32))
        one.set_state(gc, gv)
        one.set_rays(body, origin, dirs, MAXD, "all")
        return one.ray_casts()

    single = [one_map(k) for k in range(count)]
    d, h = bt.ray_casts()
    for k in range(count):
        sel = moe == k
        assert np.array_equal(d[sel].view(np.uint32), single[k][0][sel].view(np.uint32)) and np.array_equal(h[sel], single[k][1][sel])
    moe2 = (moe + 1) % count
    bt.set_heightmap_index(moe2)
    d, h = bt.ray_casts()
    for k in range(count):
        sel = moe2 == k
        assert np.array_equal(d[sel].view(np.uint32), single[k][0][sel].view(np.uint32))
    bt.update_heightmaps(0, maps[1])
    maps[0] = maps[1]
    single0 = one_map(0)
    d, h = bt.ray_casts()
    sel = moe2 == 0
    assert np.array_equal(d[sel].view(np.uint32), single0[0][sel].view(np.uint32))
    bt.clear_terrain()
    d, h = bt.ray_casts()
    assert not (h == TERRAIN).any()


def test_targets_and_origin_inside(capi):
    """a camera at the centre of the base's collision box sees out of it (never reports the box), and the terrain-only mode never
    reports the robot; with the robot the feet below the base are seen"""
    n = 16
    m, t, bt, H = _batch(capi, "anymal_c_like.urdf", n, seed=5)
    gc = np.tile(ANYMAL_GC0, (n, 1)); gc[:, 0] = np.linspace(-2, 2, n)
    bt.set_state(gc.astype(np.float32), np.zeros((n, 18), np.float32))
    base_box = [c for c in range(t["ncoll"]) if t["cbody"][c] == 0 and t["ctype"][c] == 1][0]
    rng = np.random.default_rng(0)
    dirs = rng.standard_normal((512, 3)); dirs[:, 2] = -np.abs(dirs[:, 2])
    body = np.zeros(len(dirs), np.int32)
    origin = np.tile(np.asarray(t["cpos"][base_box], np.float32), (len(dirs), 1))
    bt.set_rays(body, origin, dirs.astype(np.float32), 3.0, "all")
    d, h = bt.ray_casts()
    assert not (h == base_box).any() and (h == TERRAIN).any() and (h >= 0).any()
    ref = _reference(t, bt.get_state()[0], body, origin, dirs.astype(np.float32), H, True, 3.0)
    _compare(d, h, ref, "inside the base box")
    bt.set_rays(body, origin, dirs.astype(np.float32), 3.0, "terrain")
    d, h = bt.ray_casts()
    assert not (h >= 0).any()


def _records(bt):
    ct, cnt = bt.contacts()
    return [bt.get_state()[0].tobytes(), bt.get_state()[1].tobytes(), ct.tobytes(), cnt.tobytes(), bt.contact_points().tobytes(),
            bt.solver_iterations().tobytes(), bt.solver_status().tobytes(), bt.solver_residual().tobytes(), bt.diverged().tobytes(),
            bt.generalized_force().tobytes(), bt.body_contact_forces()[0].tobytes(), bt.imu_readings()[0].tobytes()]


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
    bt.set_imus([0], np.zeros((1, 3), np.float32))
    return m, bt


def test_poses_launch_counts_and_no_side_effects(capi):
    """a terrain-only base list costs one launch after any step; a list with the robot costs the kinematics pass when it is stale and
    one launch; the casts follow set_state and integrate2; the state, contacts, contact forces, IMU readings and solver outputs are
    unchanged and the next step is bit for bit that of a batch without rays"""
    n, H = 256, _rough(5, amp=0.05)
    m, a = _standing(capi, n, 9, H)
    _, b = _standing(capi, n, 9, H)
    t = m.tables()
    body, origin, dirs = _patterns(t)
    cam = body == 0
    for k in range(3):
        a.integrate(4); b.integrate(4)
        before = _records(a)
        a.set_rays(body[cam], origin[cam], dirs[cam], MAXD, "terrain")
        l0 = a.launch_count(); d1 = a.ray_casts(); assert a.launch_count() - l0 == 1
        a.set_rays(body, origin, dirs, MAXD, "all")
        l0 = a.launch_count(); d2 = a.ray_casts(); assert a.launch_count() - l0 == 2
        l0 = a.launch_count(); d3 = a.ray_casts(); assert a.launch_count() - l0 == 1
        assert all(np.array_equal(x.view(np.uint32), y.view(np.uint32)) for x, y in zip(d2, d3))
        assert before == _records(a)
        a.integrate(4); b.integrate(4)
    # integrate1 / integrate2: the casts describe the state after the step
    a.integrate1(); a.integrate2(); b.integrate1(); b.integrate2()
    d, h = a.ray_casts()
    fresh = capi.Batch(m, n)
    fresh.set_heightmap(H.shape[1], H.shape[0], HM["size"], HM["size"], HM["cx"], HM["cy"], H)
    fresh.set_state(*a.get_state())
    fresh.set_rays(body, origin, dirs, MAXD, "all")
    df, hf = fresh.ray_casts()
    assert np.array_equal(d.view(np.uint32), df.view(np.uint32)) and np.array_equal(h, hf)
    # set_state: the next call sees the new state
    gc, gv = a.get_state()
    gc2 = gc.copy(); gc2[:, 0] += 0.37
    a.set_state(gc2, gv); b.set_state(gc2, gv)
    fresh.set_state(gc2, gv)
    d, h = a.ray_casts(); df, hf = fresh.ray_casts()
    assert np.array_equal(d.view(np.uint32), df.view(np.uint32)) and np.array_equal(h, hf)
    a.integrate(4); b.integrate(4)
    assert _records(a) == _records(b)


@pytest.mark.parametrize("name", ["anymal", "anymal_generic"])
def test_every_per_environment_feature_on_and_the_next_step_is_unchanged(capi, monkeypatch, name):
    """with every per-environment feature on (inertia, actuator and friction rows, a terrain atlas, an actuator network, actuation
    delays, self-collision pairs on the generic instance, contact bodies, frames, a height scan, IMUs and an external wrench), casting
    rays with the robot as a target after each control step leaves every output of the step as it was, and every later step is bit for
    bit that of the same batch without rays"""
    import test_gpu_feature_mix as fm
    from test_gpu_contact_forces import _outputs, _same
    n = 64
    x = fm._inputs(name, "AN+DL", n, seed=4100 + len(name))
    a, b = fm._batch(capi, monkeypatch, x), fm._batch(capi, monkeypatch, x)
    for bt in (a, b):
        bt.set_imus([0, x["t"]["nb"] - 1], np.zeros((2, 3), np.float32))
    t = capi.Model(x["path"]).tables()
    body, origin, dirs = _patterns(t)
    a.set_rays(body, origin, dirs, MAXD, "all")

    def outputs(bt):
        o = _outputs(bt)
        o["hist"] = bt.actuator_history()
        o["f"], o["s"] = bt.body_contact_forces()
        o["imu_lin"], o["imu_ang"] = bt.imu_readings()
        o["fpos"], o["frot"], o["flin"], o["fang"] = bt.frame_states()
        o["scan_h"], o["scan_xy"] = bt.height_scan()
        return o

    hits = 0
    for k in range(fm.STEPS):
        for bt in (a, b):
            fm._command(bt, x, k)
            if k == 0:
                fm._wrench(bt, x)
            bt.integrate(fm.SUB)
        before = outputs(a)
        d, h = a.ray_casts()
        d2, h2 = a.ray_casts()
        assert np.array_equal(d.view(np.uint32), d2.view(np.uint32)) and np.array_equal(h, h2)
        hits += int((h >= 0).sum())
        _same(before, outputs(a), f"{name} control step {k}, after the casts: ")
        _same(outputs(b), outputs(a), f"{name} control step {k}, against the batch without rays: ")
    assert hits > 0


def test_cpp_depth_camera_example():
    """the raisim:: facade: a 32 x 24 camera pitched 30 degrees down in an upstream-shaped observe(), one step launch, one kinematics
    pass and one ray launch per control step, every terrain pixel's hit point on HeightMap::getHeight (examples/depth_camera.cpp)"""
    exe = os.path.join(ROOT, "examples", "depth_camera")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "examples")])
    out = subprocess.run([exe, os.path.join(RSC, "anymal_c_like.urdf")], capture_output=True, text=True, timeout=600)
    print(out.stdout)
    assert out.returncode == 0, out.stdout + out.stderr


def test_interfaces_slices_buffers_nan_and_pybind(capi):
    """environment slices, pageable, pinned and device outputs and NULL outputs give the whole-batch values; repeated calls are bit for
    bit the same; a diverged environment reads NaN with RSB_RAY_MISS; the pybind module writes what the ctypes binding reads"""
    import torch
    from raisimlib_b200 import _rsb_py
    n = 200
    m, t, bt, H = _batch(capi, "anymal_c_like.urdf", n, seed=17)
    gc, gv = bt.get_state()
    gc[7, 0] = np.nan
    bt.set_state(gc, gv)
    body, origin, dirs = _patterns(t)
    R = len(body)
    bt.set_rays(body, origin, dirs, MAXD, "all")
    d, h = bt.ray_casts()
    assert np.isnan(d[7]).all() and (h[7] == MISS).all() and not np.isnan(np.delete(d, 7, 0)).any()
    d2, h2 = bt.ray_casts()
    assert np.array_equal(d.view(np.uint32), d2.view(np.uint32)) and np.array_equal(h, h2)
    ds, hs = bt.ray_casts(100, 57)
    assert np.array_equal(ds.view(np.uint32), d[100:157].view(np.uint32)) and np.array_equal(hs, h[100:157])
    L = capi.lib()
    pd, ph = torch.empty((n, R)).pin_memory(), torch.empty((n, R), dtype=torch.int32).pin_memory()
    assert L.rsb_batch_get_ray_casts(bt.h, 0, n, C.c_void_p(pd.data_ptr()), C.c_void_p(ph.data_ptr()), capi.HOST) == 0
    assert np.array_equal(pd.numpy().view(np.uint32), d.view(np.uint32)) and np.array_equal(ph.numpy(), h)
    dd, dh = torch.empty((57, R), device="cuda"), torch.empty((57, R), dtype=torch.int32, device="cuda")
    bt.ray_casts_into(dd, dh, 100, 57)
    torch.cuda.synchronize()
    assert np.array_equal(dd.cpu().numpy().view(np.uint32), ds.view(np.uint32)) and np.array_equal(dh.cpu().numpy(), hs)
    only = np.full((n, R), -7, np.int32)
    assert L.rsb_batch_get_ray_casts(bt.h, 0, n, None, only.ctypes.data_as(C.c_void_p), capi.HOST) == 0
    assert np.array_equal(only, h)
    l0 = bt.launch_count()
    bt.ray_casts_into(None, None)
    assert L.rsb_batch_get_ray_casts(bt.h, 0, 0, only.ctypes.data_as(C.c_void_p), None, capi.HOST) == 0
    assert bt.launch_count() == l0
    with pytest.raises(ValueError):
        bt.ray_casts_into(torch.empty((n, R + 1), device="cuda"))
    with pytest.raises(ValueError):
        bt.ray_casts_into(None, torch.empty((n, R), device="cuda"))          # hit must be int32
    # pybind
    pb = _rsb_py.Batch(_rsb_py.Model(_path("anymal_c_like.urdf")), n, 0)
    pb.set_ground(0.0)
    bt.set_ground(0.0)
    torch.from_dlpack(pb.gc()).copy_(torch.from_numpy(gc).cuda())
    torch.cuda.synchronize()
    pb.set_rays(body.tolist(), origin.reshape(-1).tolist(), dirs.reshape(-1).tolist(), MAXD, "all")
    pd_, ph_ = torch.empty((n, R), device="cuda"), torch.empty((n, R), dtype=torch.int32, device="cuda")
    pb.ray_casts(pd_.data_ptr(), ph_.data_ptr())
    pb.sync()
    d, h = bt.ray_casts()
    assert np.array_equal(pd_.cpu().numpy().view(np.uint32), d.view(np.uint32)) and np.array_equal(ph_.cpu().numpy(), h)
    with pytest.raises(RuntimeError, match="targets"):
        pb.set_rays(body.tolist(), origin.reshape(-1).tolist(), dirs.reshape(-1).tolist(), MAXD, "robot")


def test_refusals_keep_the_previous_list(capi):
    """every refused set_rays leaves the previous list working; a bad range or `where`, or no rays, is refused before anything is
    enqueued"""
    n = 32
    m, t, bt, H = _batch(capi, "anymal_c_like.urdf", n, seed=29)
    L = capi.lib()
    body = np.array([0, 2], np.int32)
    origin = np.array([[0.1, 0.0, 0.0], [0.0, 0.0, 0.0]], np.float32)
    dirs = np.array([[1.0, 0.0, -1.0], [0.0, 0.0, -1.0]], np.float32)
    with pytest.raises(capi.RsbError, match="no rays"):
        bt.ray_casts()
    bt.set_rays(body, origin, dirs, 3.0, "all")
    good = bt.ray_casts()
    P = lambda a: a.ctypes.data_as(C.c_void_p)
    bad_body = np.array([0, t["nb"]], np.int32)
    neg_body = np.array([-1, 0], np.int32)
    nan_o = origin.copy(); nan_o[1, 2] = np.nan
    inf_d = dirs.copy(); inf_d[0, 0] = np.inf
    tiny_d = dirs.copy(); tiny_d[1] = [1e-7, 0, 0]
    bd, po, pd = P(body), P(origin), P(dirs)
    refused = [(bd, po, pd, -1, 3.0, 1), (bd, po, pd, capi.MAX_RAYS + 1, 3.0, 1), (None, po, pd, 2, 3.0, 1), (bd, None, pd, 2, 3.0, 1),
               (bd, po, None, 2, 3.0, 1), (P(bad_body), po, pd, 2, 3.0, 1), (P(neg_body), po, pd, 2, 3.0, 1), (bd, P(nan_o), pd, 2, 3.0, 1),
               (bd, po, P(inf_d), 2, 3.0, 1), (bd, po, P(tiny_d), 2, 3.0, 1), (bd, po, pd, 2, 0.0, 1), (bd, po, pd, 2, -1.0, 1),
               (bd, po, pd, 2, float("inf"), 1), (bd, po, pd, 2, float("nan"), 1), (bd, po, pd, 2, 3.0, 2), (bd, po, pd, 2, 3.0, -1)]
    for args in refused:
        assert L.rsb_batch_set_rays(bt.h, *args) == -1, args
        again = bt.ray_casts()
        assert all(np.array_equal(a.view(np.uint32), b.view(np.uint32)) for a, b in zip(again, good))
    dist = np.empty((n, 2), np.float32)
    l0 = bt.launch_count()
    for env_begin, env_count, where in ((0, n, 2), (0, n, -1), (-1, 2, 0), (n - 1, 2, 0), (0, -1, 0)):
        assert L.rsb_batch_get_ray_casts(bt.h, env_begin, env_count, P(dist), None, where) == -1
    assert bt.launch_count() == l0
    with pytest.raises(ValueError):
        bt.set_rays(body, origin, dirs, 3.0, "robot")
    # the list survives set-params and terrain calls
    bt.set_params(dt=0.002)
    bt.set_ground(0.0)
    assert bt.ray_casts()[0].shape == (n, 2)
    bt.set_rays([], np.zeros((0, 3)), np.zeros((0, 3)), 3.0)
    with pytest.raises(capi.RsbError, match="no rays"):
        bt.ray_casts()
