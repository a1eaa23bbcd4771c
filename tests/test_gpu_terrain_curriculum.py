"""Terrain curriculum on the GPU (pytest -m gpu): rsb_batch_set_heightmap_index moves environments among the maps of the terrain atlas and
rsb_batch_update_heightmaps overwrites maps in place.  Both must compute exactly what a fresh rsb_batch_set_heightmaps of the resulting
terrain computes: state, contacts, contact points, body contact forces and height scans bit for bit after every step, on the quadruped,
humanoid and generic (max32) instances, from host, pinned and device sources.  Also: float64 oracle parity after moves (the bounds of
tests/test_gpu_parity.py::test_terrain_atlas_matches_oracle, step by step), range isolation, refusals that change nothing, the lifetime
of an assignment, launch counts, the torch and pybind layers and the C++ example."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT, RSC
from helpers import ANYMAL_GC0, MARGIN, MAX32, random_state, setup_batch
from height_scan_ref import base_grid

pytestmark = pytest.mark.gpu

HM = dict(xs=129, ys=97, sx=25.6, sy=19.2, cx=0.3, cy=-0.2)
INSTANCES = [pytest.param("anymal_c_like.urdf", id="quadruped"), pytest.param("atlas_like.urdf", id="humanoid"),
             pytest.param(MAX32, id="generic-max32")]


@pytest.fixture(scope="module")
def capi():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from raisimlib_b200 import capi as c
    return c


def _path(src):
    return os.path.join(RSC, src) if src.endswith(".urdf") else src


def _maps(seed, count=3, amp=0.05):
    rng = np.random.default_rng(seed)
    H = rng.uniform(-amp, amp, (count, HM["ys"], HM["xs"])).astype(np.float32)
    H += np.arange(count, dtype=np.float32)[:, None, None] * np.float32(0.02)
    return H


def _atlas(bt, H, moe):
    bt.set_heightmaps(HM["sx"], HM["sy"], HM["cx"], HM["cy"], H, moe)


def _batch(capi, src, n, seed, H, moe, base_z=0.55, upright=False):
    """a batch on the atlas (H, moe) with contact bodies and a base grid scan, in a random state that touches the terrain, or (upright)
    a level base at base_z with slightly bent joints"""
    m = capi.Model(_path(src))
    t = m.tables()
    bt = capi.Batch(m, n)
    _atlas(bt, H, moe)
    gc, gv = random_state(t, np.random.default_rng(seed), n, pos_scale=8.0, base_z=base_z, joint_scale=0.05 if upright else 0.3)
    if upright:
        gc[:, 3:7] = [1, 0, 0, 0]
    bt.set_state(gc.astype(np.float32), gv.astype(np.float32))
    bt.set_contact_bodies([0, t["nb"] - 1])
    xy = base_grid()
    bt.set_height_scan(np.zeros(len(xy), np.int32), xy, "yaw")
    return m, t, bt


def _records(bt):
    ct, cnt = bt.contacts()
    g, v = bt.get_state()
    f, s = bt.body_contact_forces()
    h, sxy = bt.height_scan()
    return [g.tobytes(), v.tobytes(), ct.tobytes(), cnt.tobytes(), bt.contact_points().tobytes(), f.tobytes(), s.tobytes(), h.tobytes(), sxy.tobytes()]


def _index_call(capi, bt, idx, begin, source):
    """set_heightmap_index of idx for environments [begin, begin + len(idx)) from a pageable, pinned or device source"""
    import torch
    if source == "host":
        bt.set_heightmap_index(idx, begin)
    elif source == "pinned":
        p = torch.from_numpy(idx.astype(np.int32)).pin_memory()
        assert capi.lib().rsb_batch_set_heightmap_index(bt.h, C.c_void_p(p.data_ptr()), begin, len(idx), capi.HOST) == 0
    else:
        bt.set_heightmap_index_from(torch.from_numpy(idx.astype(np.int32)).cuda(), begin)


@pytest.mark.parametrize("src", INSTANCES)
def test_reassignment_is_a_fresh_atlas_bit_for_bit(capi, src):
    """set_heightmap_index on a sub-range after k steps == set_heightmaps with the new assignment after the same k steps"""
    n, H = 320, _maps(3)
    m0 = (np.arange(n) % 3).astype(np.int32)
    m1 = m0.copy(); m1[40:250] = (m0[40:250] + 1 + np.arange(210) % 2) % 3
    for source in ("host", "pinned", "device"):
        _, _, a = _batch(capi, src, n, 5, H, m0)
        _, _, b = _batch(capi, src, n, 5, H, m0)
        for _ in range(3):
            a.integrate(2); b.integrate(2)
            assert _records(a) == _records(b)
        _index_call(capi, a, m1[40:250], 40, source)
        _atlas(b, H, m1)
        assert _records(a) == _records(b)           # the last step's records stay, the scan reads the new maps
        for _ in range(4):
            a.integrate(2); b.integrate(2)
            assert _records(a) == _records(b), source
        assert a.contacts()[1].sum() > 0


@pytest.mark.parametrize("src", INSTANCES)
def test_update_is_a_fresh_atlas_bit_for_bit(capi, src):
    """update_heightmaps == set_heightmaps of the edited atlas; a map raised above the old maximum gives the robots on it contacts,
    which the stage-B cull would drop with the old maximum; a map lowered below it"""
    n, H = 240, _maps(7)
    moe = (np.arange(n) % 3).astype(np.int32)
    E = H.copy(); E[1] += np.float32(1.25); E[2] -= np.float32(0.3)
    _, _, a = _batch(capi, src, n, 9, H, moe, base_z=1.3, upright=True)
    _, _, b = _batch(capi, src, n, 9, H, moe, base_z=1.3, upright=True)
    a.integrate(1); b.integrate(1)
    assert _records(a) == _records(b)
    on1 = moe == 1
    assert (a.contacts()[1][on1] == 0).all()        # high above the old terrain
    a.update_heightmaps(1, E[1:3])
    _atlas(b, E, moe)
    assert _records(a) == _records(b)
    for _ in range(3):
        a.integrate(1); b.integrate(1)
        assert _records(a) == _records(b)
    assert (a.contacts()[1][on1] > 0).mean() > 0.9  # the raised map reaches into them
    # device source, and the single map of set_heightmap is map 0 of a one-map atlas
    import torch
    for bt in (a, b):
        bt.set_heightmap(HM["xs"], HM["ys"], HM["sx"], HM["sy"], HM["cx"], HM["cy"], H[0])
    a.update_heightmaps_from(0, torch.from_numpy(E[1:2]).cuda())
    b.set_heightmap(HM["xs"], HM["ys"], HM["sx"], HM["sy"], HM["cx"], HM["cy"], E[1])
    for _ in range(2):
        a.integrate(1); b.integrate(1)
        assert _records(a) == _records(b)


def test_oracle_parity_after_moves(capi):
    """one float64 oracle per environment on the moved assignment: every one of 20 steps from the GPU's state within the bounds of the
    atlas parity test (contact sets equal away from shallow candidates, median |dv| < 5e-5 over the converged environments)"""
    n = 192
    t, bt, o64, o32, gc, gv, tau = setup_batch(capi, "anymal_c_like.urdf", n, seed=231, terrain="none", base_z=0.42)
    rng = np.random.default_rng(232)
    H = (0.1 * rng.uniform(-1, 1, (3, 49, 65))).astype(np.float32)
    H[1] += 0.05; H[2] -= 0.04
    m0 = (np.arange(n) % 3).astype(np.int32)
    m1 = ((np.arange(n) * 5 + 1) % 3).astype(np.int32)
    bt.set_heightmaps(12.8, 9.6, 0.1, -0.2, H, m0)
    bt.integrate(1)
    bt.set_heightmap_index(m1)
    o64.set_heightmaps(12.8, 9.6, 0.1, -0.2, H.astype(np.float64), m1)
    o32.set_heightmaps(12.8, 9.6, 0.1, -0.2, H.astype(np.float64), m1)
    a, b = [x.astype(np.float64) for x in bt.get_state()]
    touched, worst = 0, []
    for step in range(20):
        bt.set_state(a.astype(np.float32), b.astype(np.float32))
        bt.integrate(1)
        g1, v1 = bt.get_state()
        pts, cnt = bt.contact_points(), bt.contacts()[1]
        d32 = o32.step(a.copy(), b.copy(), tau_ff=tau, debug=True)
        shallow = ((np.abs(d32["c_depth"]) < MARGIN) & (d32["c_pt"] >= 0)).any(1)
        assert ((pts != d32["c_pt"]).any(1) & ~shallow).sum() == 0, step
        d = o64.step(a, b, tau_ff=tau, debug=True)
        conv = (pts == d["c_pt"]).all(1) & (bt.solver_iterations() < 150) & (d["iters"] < 150)
        assert conv.mean() > 0.9, step
        err = np.median(np.abs(v1 - b)[conv].max(1))
        worst.append(err)
        assert err < 5e-5, step
        touched += int(cnt.sum() > 0)
        a, b = g1.astype(np.float64), v1.astype(np.float64)
    print(f"20 steps after moves: median |dv| per step, worst {max(worst):.2e}")
    assert touched == 20


def test_range_isolation(capi):
    """environments outside the range keep their map: their scans and their next steps are those of a batch that never moved anyone"""
    n, H = 256, _maps(11)
    m0 = (np.arange(n) % 3).astype(np.int32)
    _, _, a = _batch(capi, "anymal_c_like.urdf", n, 13, H, m0)
    _, _, b = _batch(capi, "anymal_c_like.urdf", n, 13, H, m0)
    a.integrate(2); b.integrate(2)
    a.set_heightmap_index((m0[100:180] + 1) % 3, 100)
    ha, hb = a.height_scan()[0], b.height_scan()[0]
    out = np.r_[0:100, 180:n]
    assert np.array_equal(ha[out].view(np.uint32), hb[out].view(np.uint32))
    assert (ha[100:180] != hb[100:180]).any(1).all()
    a.integrate(2); b.integrate(2)
    assert np.array_equal(a.get_state()[0][out], b.get_state()[0][out]) and np.array_equal(a.get_state()[1][out], b.get_state()[1][out])
    assert np.array_equal(a.contacts()[0][out].tobytes(), b.contacts()[0][out].tobytes())


def test_refusals_change_nothing(capi):
    """every refused call returns RSB_ERR_INVALID, launches nothing, and the batch goes on bit for bit as one that never made it"""
    n, H = 128, _maps(17)
    m0 = (np.arange(n) % 3).astype(np.int32)
    _, _, a = _batch(capi, "anymal_c_like.urdf", n, 19, H, m0)
    _, _, b = _batch(capi, "anymal_c_like.urdf", n, 19, H, m0)
    a.integrate(2); b.integrate(2)
    L = capi.lib()
    ok_idx = np.zeros(n, np.int32)
    bad_hi, bad_lo = ok_idx.copy(), ok_idx.copy()
    bad_hi[77] = 3; bad_lo[5] = -1
    P = lambda x: x.ctypes.data_as(C.c_void_p)
    nan_map, inf_map = H[:1].copy(), H[:2].copy()
    nan_map[0, 3, 4] = np.nan; inf_map[1, 90, 100] = -np.inf
    l0 = a.launch_count()
    refused = [lambda: L.rsb_batch_set_heightmap_index(a.h, P(bad_hi), 0, n, capi.HOST),
               lambda: L.rsb_batch_set_heightmap_index(a.h, P(bad_lo), 0, n, capi.HOST),
               lambda: L.rsb_batch_set_heightmap_index(None, P(ok_idx), 0, n, capi.HOST),
               lambda: L.rsb_batch_set_heightmap_index(a.h, None, 0, n, capi.HOST),
               lambda: L.rsb_batch_set_heightmap_index(a.h, P(ok_idx), -1, 2, capi.HOST),
               lambda: L.rsb_batch_set_heightmap_index(a.h, P(ok_idx), n - 1, 2, capi.HOST),
               lambda: L.rsb_batch_set_heightmap_index(a.h, P(ok_idx), 0, -1, capi.HOST),
               lambda: L.rsb_batch_set_heightmap_index(a.h, P(ok_idx), 0, n, 2),
               lambda: L.rsb_batch_update_heightmaps(a.h, 0, 1, P(nan_map), capi.HOST),
               lambda: L.rsb_batch_update_heightmaps(a.h, 1, 2, P(inf_map), capi.HOST),
               lambda: L.rsb_batch_update_heightmaps(a.h, 2, 2, P(inf_map), capi.HOST),
               lambda: L.rsb_batch_update_heightmaps(a.h, -1, 1, P(nan_map), capi.HOST),
               lambda: L.rsb_batch_update_heightmaps(a.h, 0, -1, P(nan_map), capi.HOST),
               lambda: L.rsb_batch_update_heightmaps(a.h, 0, 1, None, capi.HOST),
               lambda: L.rsb_batch_update_heightmaps(None, 0, 1, P(H), capi.HOST),
               lambda: L.rsb_batch_update_heightmaps(a.h, 0, 1, P(H), -1)]
    import torch
    refused += [lambda: L.rsb_batch_set_heightmap_index(a.h, C.c_void_p(torch.from_numpy(bad_hi).cuda().data_ptr()), 0, n, capi.DEVICE),
                lambda: L.rsb_batch_update_heightmaps(a.h, 0, 1, C.c_void_p(torch.from_numpy(nan_map).cuda().data_ptr()), capi.DEVICE)]
    for k, call in enumerate(refused):
        assert call() == -1, k
    assert L.rsb_batch_set_heightmap_index(a.h, P(ok_idx), 0, 0, capi.HOST) == 0     # env_count 0: nothing to do
    assert L.rsb_batch_update_heightmaps(a.h, 3, 0, P(H), capi.HOST) == 0
    assert a.launch_count() == l0
    for _ in range(3):
        a.integrate(2); b.integrate(2)
        assert _records(a) == _records(b)
    # no atlas: ground, no terrain, the single map of set_heightmap; update needs a height map
    m = capi.Model(_path("anymal_c_like.urdf"))
    c = capi.Batch(m, 8)
    idx8 = np.zeros(8, np.int32)
    assert L.rsb_batch_set_heightmap_index(c.h, P(idx8), 0, 8, capi.HOST) == -1
    assert L.rsb_batch_update_heightmaps(c.h, 0, 1, P(H), capi.HOST) == -1
    c.set_ground(0.0)
    assert L.rsb_batch_set_heightmap_index(c.h, P(idx8), 0, 8, capi.HOST) == -1
    assert L.rsb_batch_update_heightmaps(c.h, 0, 1, P(H), capi.HOST) == -1
    c.set_heightmap(HM["xs"], HM["ys"], HM["sx"], HM["sy"], HM["cx"], HM["cy"], H[0])
    with pytest.raises(capi.RsbError, match="no terrain atlas"):
        c.set_heightmap_index(idx8)
    with pytest.raises(capi.RsbError, match="not all in"):
        c.update_heightmaps(1, H[0])
    c.update_heightmaps(0, H[1])


def test_lifetime_and_launch_counts(capi):
    """gym resets keep the assignment, set_heightmaps replaces it, clear_terrain and set_ground drop it; neither call adds a launch or
    makes a getter run the kinematics pass"""
    n, H = 96, _maps(23)
    m0 = (np.arange(n) % 3).astype(np.int32)
    m1 = ((np.arange(n) + 2) % 3).astype(np.int32)
    mod, t, a = _batch(capi, "anymal_c_like.urdf", n, 29, H, m0)
    _, _, b = _batch(capi, "anymal_c_like.urdf", n, 29, H, m1)
    a.mass_matrix()
    l0 = a.launch_count()
    a.set_heightmap_index(m1)
    a.update_heightmaps(2, H[2])
    a.mass_matrix(); a.body_poses()
    assert a.launch_count() == l0
    feet = [mod.body_index(f"{leg}_FOOT") for leg in ("LF", "RF", "LH", "RH")]
    for bt in (a, b):
        bt.set_pd_gains(np.r_[np.zeros(6), 300.0 * np.ones(12)], np.r_[np.zeros(6), 8.0 * np.ones(12)])
        bt.gym_configure(ANYMAL_GC0, np.zeros(18), ANYMAL_GC0[7:], 0.3 * np.ones(12), feet)
        bt.gym_reset()
    assert _records(a)[-2:] == _records(b)[-2:]
    act = np.zeros((n, 12), np.float32)
    for _ in range(3):
        for bt in (a, b):
            bt.gym_step(act, 4, np.empty((n, bt.ob_dim()), np.float32), np.empty(n, np.float32), np.empty(n, np.uint8))
        assert _records(a) == _records(b)
    _atlas(a, H, m0); _atlas(b, H, m0)
    assert _records(a) == _records(b)
    a.clear_terrain()
    with pytest.raises(capi.RsbError, match="no terrain atlas"):
        a.set_heightmap_index(m1)
    _atlas(a, H, m0)
    a.set_ground(0.0)
    with pytest.raises(capi.RsbError, match="no terrain atlas"):
        a.set_heightmap_index(m1)


def test_torch_refusals_and_pybind(capi):
    """the torch _from variants check dtype, shape, device and contiguity; the pybind calls take device addresses"""
    import torch
    from raisimlib_b200 import _rsb_py
    n, H = 64, _maps(31)
    m0 = (np.arange(n) % 3).astype(np.int32)
    _, _, a = _batch(capi, "anymal_c_like.urdf", n, 37, H, m0)
    good = torch.zeros(n, dtype=torch.int32, device="cuda")
    for bad in (good.long(), good.reshape(n, 1), good.cpu(), torch.zeros(2 * n, dtype=torch.int32, device="cuda")[::2]):
        with pytest.raises(ValueError):
            a.set_heightmap_index_from(bad)
    hg = torch.from_numpy(H[:1]).cuda()
    for bad in (hg.double(), hg[0], hg.cpu(), torch.zeros((1, HM["xs"], HM["ys"]), device="cuda").transpose(1, 2),
                torch.zeros((1, HM["ys"], HM["xs"] + 1), device="cuda")):
        with pytest.raises(ValueError):
            a.update_heightmaps_from(0, bad)
    a.set_heightmap_index_from(good[:10], 5)
    a.update_heightmaps_from(1, hg)
    # the numpy variant: a map of another resolution or a flat array is refused before the library reads it
    l0 = a.launch_count()
    for bad in (np.zeros((1, 65, 65), np.float32), H[:1].reshape(-1), H[:1, :, :-1], np.zeros((2, 3, HM["ys"], HM["xs"]), np.float32)):
        with pytest.raises(ValueError):
            a.update_heightmaps(0, bad)
    assert a.launch_count() == l0
    # pybind: the same calls from device addresses move and edit the pybind batch's atlas as the ctypes binding does
    path = _path("anymal_c_like.urdf")
    pb = _rsb_py.Batch(_rsb_py.Model(path), n, 0)
    pb.set_heightmaps(3, HM["xs"], HM["ys"], HM["sx"], HM["sy"], HM["cx"], HM["cy"], H.reshape(-1).tolist(), m0.tolist())
    gc = a.get_state()[0]
    torch.from_dlpack(pb.gc()).copy_(torch.from_numpy(gc).cuda())
    torch.cuda.synchronize()
    xy = base_grid()
    pb.set_height_scan([0] * len(xy), xy.reshape(-1).tolist(), "yaw")
    E = H.copy(); E[2] += np.float32(0.25)
    m1 = ((np.arange(n) + 1) % 3).astype(np.int32)
    dm1, dE = torch.from_numpy(m1).cuda(), torch.from_numpy(E[2:3]).cuda()
    pb.set_heightmap_index(dm1.data_ptr(), 0, n)
    pb.update_heightmaps(dE.data_ptr(), 2, 1)
    dh, dxy = torch.empty((n, len(xy)), device="cuda"), torch.empty((n, len(xy), 2), device="cuda")
    pb.height_scan(dh.data_ptr(), dxy.data_ptr())
    pb.sync()
    _atlas(a, E, m1)
    h, _ = a.height_scan()
    assert np.array_equal(dh.cpu().numpy(), h)
    with pytest.raises(RuntimeError, match="height-map index"):
        pb.set_heightmap_index(torch.full((n,), 3, dtype=torch.int32, device="cuda").data_ptr(), 0, n)
    assert pb.launch_count >= 0


def test_cpp_terrain_curriculum_example():
    """the raisim:: facade: per-environment addHeightMap with a curriculum in reset(); every scan height equals the environment's own
    HeightMap::getHeight, one step launch per control step, and moves among existing levels upload no map (examples/terrain_curriculum.cpp)"""
    exe = os.path.join(ROOT, "examples", "terrain_curriculum")
    if not os.path.exists(exe):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "examples")])
    out = subprocess.run([exe, os.path.join(RSC, "anymal_c_like.urdf")], capture_output=True, text=True, timeout=600)
    print(out.stdout)
    assert out.returncode == 0, out.stdout + out.stderr


def _hmax(capi, bt):
    v = C.c_float()
    L = capi.lib()
    L.rsb_internal_terrain_hmax.argtypes = [C.c_void_p, C.c_void_p]
    assert L.rsb_internal_terrain_hmax(bt.h, C.byref(v)) == 0
    return v.value


def test_cull_height_follows_every_update(capi):
    """the stage-B cull height is the exact maximum over all maps after every update, also when the highest map comes down; updates
    from pinned memory; more maps in one call than a grid has rows (65535), on maps of 2 x 2 samples"""
    import torch
    n, H = 96, _maps(41)
    moe = (np.arange(n) % 3).astype(np.int32)
    _, _, a = _batch(capi, "anymal_c_like.urdf", n, 43, H, moe)
    _, _, b = _batch(capi, "anymal_c_like.urdf", n, 43, H, moe)
    assert _hmax(capi, a) == H.max()
    E = H.copy()
    E[2] -= np.float32(0.5)                           # the highest map goes below the others
    a.update_heightmaps(2, E[2])
    assert _hmax(capi, a) == E.max() < H.max()
    E[0] = np.float32(-2.0)                           # every height of a map the same, negative
    pinned = torch.from_numpy(E[0:1].copy()).pin_memory()
    assert capi.lib().rsb_batch_update_heightmaps(a.h, 0, 1, C.c_void_p(pinned.data_ptr()), capi.HOST) == 0
    assert _hmax(capi, a) == E.max()
    _atlas(b, E, moe)
    assert _hmax(capi, b) == _hmax(capi, a)
    for _ in range(3):
        a.integrate(2); b.integrate(2)
        assert _records(a) == _records(b)
    # 70000 maps of 2 x 2: the check kernel strides over the maps beyond the grid's 65535 rows
    count = 70000
    m = capi.Model(_path("anymal_c_like.urdf"))
    c = capi.Batch(m, 4)
    T = np.random.default_rng(5).uniform(-1, 1, (count, 2, 2)).astype(np.float32)
    c.set_heightmaps(2.0, 2.0, 0.0, 0.0, T, np.array([0, 1, count - 2, count - 1], np.int32))
    U = T.copy(); U[1:] *= np.float32(0.5); U[count - 1, 1, 1] = np.float32(3.0)
    c.update_heightmaps(1, U[1:])
    assert _hmax(capi, c) == U.max() == np.float32(3.0)
    U[count - 1, 1, 1] = np.float32(0.25)
    c.update_heightmaps_from(count - 1, torch.from_numpy(U[count - 1:]).cuda())
    assert _hmax(capi, c) == U.max()
    d = capi.Batch(m, 4)
    d.set_heightmaps(2.0, 2.0, 0.0, 0.0, U, np.array([0, 1, count - 2, count - 1], np.int32))
    for bt in (c, d):
        bt.set_height_scan(np.zeros(5, np.int32), np.array([[0.9, 0.9], [-0.9, 0.9], [0.3, -0.7], [-0.5, -0.5], [0.0, 0.0]], np.float32), "world")
    assert np.array_equal(c.height_scan()[0], d.height_scan()[0])
    bad = U[1:].copy(); bad[68000, 0, 1] = np.nan
    with pytest.raises(capi.RsbError, match="map 68001"):
        c.update_heightmaps(1, bad)
    assert _hmax(capi, c) == U.max()


def test_facade_terrain_mirror(tmp_path):
    """the facade's terrain mirror on one batch (tests/cpp/terrain_mirror_check.cpp): environments without terrain of their own share the
    lowest-numbered environment's map (one plain upload for one common map), distinct maps make one atlas, a rebuilt atlas keeps the
    levels nobody is on so that moving back to them is an index move, and a ground in one environment with maps in others is refused"""
    exe = tmp_path / "terrain_mirror_check"
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-Wall", "-I" + os.path.join(ROOT, "include"), "-o", str(exe), os.path.join(ROOT, "tests", "cpp", "terrain_mirror_check.cpp"),
                           "-L" + os.path.join(ROOT, "raisimlib_b200"), "-lrsb", "-Wl,-rpath," + os.path.join(ROOT, "raisimlib_b200"), "-Wl,-rpath,/usr/local/cuda/lib64"])
    out = subprocess.run([str(exe), os.path.join(RSC, "anymal_c_like.urdf")], capture_output=True, text=True, timeout=300)
    print(out.stdout)
    assert out.returncode == 0, out.stdout + out.stderr
