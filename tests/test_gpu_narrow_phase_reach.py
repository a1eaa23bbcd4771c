"""The kernel's height-map narrow phase (integrate1() contact lists) against the exact float64 restatement in
tests/terrain_contact_ref.py, at the shape-to-pitch ratios, map shapes and compiled instances where a search limited to the cells
next to a shape's centre goes wrong (issue: "Test the height-map narrow phase against an exact mesh reference, and search every cell
a collision shape reaches").

Contact lists (candidate indices, in candidate order) must equal the reference's outside a 2e-6 m margin and near-ties (1e-5 m); pair
indices must be one the reference allows.  Depth and normal errors must be no worse than 3x the float32 oracle's own error against the
reference on the same inputs (both are printed).
"""
import os

import numpy as np
import pytest

import terrain_contact_ref as ref
from conftest import RSC
from helpers import ANYMAL_GC0, MAX32, random_state
from oracle.oracle import Oracle
from oracle.urdf_tables import load_tables

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def capi():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from raisimlib_b200 import capi as c
    return c


def _model(urdf):
    return os.path.join(RSC, urdf) if urdf.endswith(".urdf") else urdf


def kernel_lists(capi, urdf, maps, X, Y, cx, cy, gc, map_of_env=None):
    """integrate1() on the state gc (zero velocity and force) over one map, or an atlas maps [count, ys, xs] with map_of_env"""
    n = len(gc)
    t = load_tables(_model(urdf))
    bt = capi.Batch(capi.Model(_model(urdf)), n)
    if map_of_env is None:
        ys, xs = maps.shape
        bt.set_heightmap(xs, ys, X, Y, cx, cy, np.ascontiguousarray(maps, np.float32))
    else:
        bt.set_heightmaps(X, Y, cx, cy, np.ascontiguousarray(maps, np.float32), np.asarray(map_of_env, np.int32))
    bt.set_control_mode(capi.FORCE_AND_TORQUE)
    bt.set_state(gc.astype(np.float32), np.zeros((n, t["nv"]), np.float32))
    bt.set_generalized_force(np.zeros((n, t["nv"]), np.float32))
    bt.integrate1()
    ct, cnt = bt.contacts()
    return bt, (bt.contact_points(), cnt, ct["pair_index"], ct["depth"], ct["normal"])


def oracle32_lists(urdf, maps, X, Y, cx, cy, gc, map_of_env=None):
    t = load_tables(_model(urdf))
    o = Oracle(t, precision="f32")
    if map_of_env is None:
        ys, xs = maps.shape
        o.set_heightmap(xs, ys, X, Y, cx, cy, np.asarray(maps, np.float64))
    else:
        o.set_heightmaps(X, Y, cx, cy, np.asarray(maps, np.float64), np.asarray(map_of_env, np.int32))
    d = o.step(gc.copy(), np.zeros((len(gc), t["nv"])), debug=True)
    return d["c_pt"], d["ncontacts"], d["c_pair"], d["c_depth"], d["c_normal"]


def check(capi, urdf, maps, X, Y, cx, cy, gc, label, min_contacts, map_of_env=None):
    t = load_tables(_model(urdf))
    grids = [ref.Grid(m, X, Y, cx, cy) for m in (maps if map_of_env is not None else [maps])]
    R = [ref.env_contacts(t, gc[e], grids[map_of_env[e]] if map_of_env is not None else grids[0]) for e in range(len(gc))]
    n_ref = sum(len(lst) for lst, amb in R if not amb)
    assert n_ref >= min_contacts, n_ref
    _, got = kernel_lists(capi, urdf, maps, X, Y, cx, cy, gc, map_of_env)
    bad, ed, en, w = ref.compare(R, got, f"{label} kernel")
    assert not bad, f"kernel contact lists differ from the reference in environments {bad[:10]}"
    _, ed32, en32, w32 = ref.compare(R, oracle32_lists(urdf, maps, X, Y, cx, cy, gc, map_of_env), f"{label} f32 oracle")
    # the suite's scale rule: no worse than 3x the float32 oracle's own error (a normal divided by a distance scaled by 1 / distance)
    far = max(abs(cx) + X, abs(cy) + Y)
    floor_d = 2e-7 * (1.0 + far)
    sn, sn32 = en / (1.0 + 1e-2 * w), en32 / (1.0 + 1e-2 * w32)
    print(f"[{label}] depth err kernel {ed.max():.2e} / f32 oracle {ed32.max():.2e}; scaled normal err kernel {sn.max():.2e} / "
          f"f32 oracle {sn32.max():.2e}")
    assert ed.max() <= 3.0 * max(ed32.max(), floor_d)
    assert sn.max() <= 3.0 * max(sn32.max(), 1e-6 * (1.0 + far))
    return got


PITCH = 0.1


@pytest.mark.parametrize("ratio", (0.1, 0.3, 0.5, 0.7, 1.2, 2.5))
def test_sphere_every_radius_to_pitch_ratio(capi, ratio):
    """single spheres (generic instance) on a rough map, centres on cell boundaries, diagonals, the last row / column and off the map"""
    rng = np.random.default_rng(100 + int(ratio * 10))
    xs, ys = 33, 25
    X, Y = (xs - 1) * PITCH, (ys - 1) * PITCH
    H = (0.15 * rng.uniform(-1, 1, (ys, xs))).astype(np.float32)
    r = ratio * PITCH
    g = ref.Grid(H, X, Y, 0.0, 0.0)
    gc = ref.drop_single_shape(rng, g, 512, "sphere", (r,), (-0.3 * r, 0.5 * r))
    check(capi, ref.single_shape_urdf(f'<sphere radius="{r}"/>'), H, X, Y, 0.0, 0.0, gc, f"sphere r/pitch {ratio}", 250)


@pytest.mark.parametrize("reach", (0.8, 1.6, 3.0))
def test_capsule_side_reach(capi, reach):
    """capsules lying nearly flat, reach up to 3 pitches, on non-square cells (0.08 x 0.1 m) of an off-centre map"""
    rng = np.random.default_rng(200 + int(reach * 10))
    xs, ys = 33, 25
    X, Y, cx, cy = (xs - 1) * 0.08, (ys - 1) * 0.1, 0.37, -0.21
    H = (0.08 * rng.uniform(-1, 1, (ys, xs))).astype(np.float32)
    rc = 0.03
    hl = reach * 0.08 - rc
    g = ref.Grid(H, X, Y, cx, cy)
    gc = ref.drop_single_shape(rng, g, 512, "capsule", (rc, hl), (-0.02, 0.06))
    check(capi, ref.single_shape_urdf(f'<capsule radius="{rc}" length="{2 * hl}"/>'), H, X, Y, cx, cy, gc, f"capsule reach {reach}", 250)


@pytest.mark.parametrize("half_x", (0.15, 0.29))
def test_box_face_reach(capi, half_x):
    """trunk-sized boxes on sparse peaks, pitch 0.05 (half extent up to 6 pitches), yawed anywhere and at 45 degrees"""
    rng = np.random.default_rng(300 + int(half_x * 100))
    xs, ys = 41, 37
    p = 0.05
    X, Y = (xs - 1) * p, (ys - 1) * p
    H = np.where(rng.uniform(0, 1, (ys, xs)) < 0.08, rng.uniform(0.02, 0.08, (ys, xs)), 0.0).astype(np.float32)
    h = (half_x, 0.14, 0.09)
    g = ref.Grid(H, X, Y, 0.0, 0.0)
    gc = ref.drop_single_shape(rng, g, 512, "box", h, (-0.06, 0.01))
    check(capi, ref.single_shape_urdf(f'<box size="{2 * h[0]} {2 * h[1]} {2 * h[2]}"/>'), H, X, Y, 0.0, 0.0, gc, f"box {half_x}", 250)


@pytest.mark.parametrize("xs,ys", [(2, 2), (3, 2), (2, 3), (3, 3)])
def test_tiny_maps(capi, xs, ys):
    """maps of 2 or 3 samples a side, where the sphere block is clamped onto the map (xs - 3, ys - 3)"""
    rng = np.random.default_rng(400 + 10 * xs + ys)
    X, Y = (xs - 1) * PITCH, (ys - 1) * 0.13
    H = (0.05 * rng.uniform(-1, 1, (ys, xs))).astype(np.float32)
    g = ref.Grid(H, X, Y, -0.02, 0.04)
    for r in (0.03, 0.08, 0.2):
        gc = ref.drop_single_shape(rng, g, 128, "sphere", (r,), (-0.3 * r, 0.5 * r))
        check(capi, ref.single_shape_urdf(f'<sphere radius="{r}"/>'), H, X, Y, -0.02, 0.04, gc, f"tiny {xs}x{ys} r {r}", 20)


def test_far_from_the_origin(capi):
    """a map around (24.1, -23.7), the corner of the benchmark's 51.2 m map"""
    rng = np.random.default_rng(500)
    xs, ys = 21, 21
    X, Y, cx, cy = 2.0, 2.0, 24.1, -23.7
    H = (0.1 * rng.uniform(-1, 1, (ys, xs))).astype(np.float32)
    g = ref.Grid(H, X, Y, cx, cy)
    for r in (0.05, 0.12, 0.25):
        gc = ref.drop_single_shape(rng, g, 256, "sphere", (r,), (-0.3 * r, 0.5 * r))
        check(capi, ref.single_shape_urdf(f'<sphere radius="{r}"/>'), H, X, Y, cx, cy, gc, f"far r {r}", 100)


def test_atlas_maps_one_and_two(capi):
    """environments on maps 1 and 2 of a three-map atlas (a non-zero offset into the heights), spheres of 1.2 pitches"""
    rng = np.random.default_rng(600)
    xs, ys = 25, 21
    X, Y = (xs - 1) * PITCH, (ys - 1) * PITCH
    maps = (0.15 * rng.uniform(-1, 1, (3, ys, xs))).astype(np.float32)
    r = 0.12
    n = 512
    map_of_env = np.where(np.arange(n) % 2 == 0, 1, 2).astype(np.int32)
    gc = np.zeros((n, 7))
    for m in (1, 2):
        sel = np.where(map_of_env == m)[0]
        gc[sel] = ref.drop_single_shape(rng, ref.Grid(maps[m], X, Y, 0.0, 0.0), len(sel), "sphere", (r,), (-0.3 * r, 0.5 * r))
    check(capi, ref.single_shape_urdf(f'<sphere radius="{r}"/>'), maps, X, Y, 0.0, 0.0, gc, "atlas maps 1, 2", 250, map_of_env)


def bench_like_map(rng, xs, ys, amp):
    """smooth value noise plus fine detail, like the benchmark's terrain"""
    lat = rng.uniform(-1, 1, (ys // 4 + 2, xs // 4 + 2))
    yy, xx = np.meshgrid(np.arange(ys) / 4.0, np.arange(xs) / 4.0, indexing="ij")
    i, j = yy.astype(int), xx.astype(int)
    fy, fx = yy - i, xx - j
    smooth = (lat[i, j] * (1 - fx) * (1 - fy) + lat[i, j + 1] * fx * (1 - fy) + lat[i + 1, j] * (1 - fx) * fy + lat[i + 1, j + 1] * fx * fy)
    return (amp * (0.8 * smooth + 0.2 * rng.uniform(-1, 1, (ys, xs)))).astype(np.float32)


@pytest.mark.parametrize("urdf,pitch,spec", [("anymal_c_like.urdf", 0.1, 1), ("anymal_c_like.urdf", 0.05, 1),
                                              ("atlas_like.urdf", 0.1, 2), ("atlas_like.urdf", 0.05, 2), (MAX32, 0.1, 0)],
                         ids=["anymal-0.1", "anymal-0.05", "atlas-0.1", "atlas-0.05", "max32-0.1"])
def test_robots_dropped_near_the_ground(capi, urdf, pitch, spec):
    """ANYmal on the quadruped instance, Atlas on the humanoid instance, the 64-candidate model (second candidate slot) on the generic
    one, in random orientations with their bases just above a rough map: trunks, hips, heads and limbs on the terrain"""
    from helpers import launch_config
    rng = np.random.default_rng(700 + int(pitch * 100))
    t = load_tables(_model(urdf))
    xs = ys = 61
    X = Y = (xs - 1) * pitch
    H = bench_like_map(rng, xs, ys, 0.1)
    n = 128
    gc, _ = random_state(t, rng, n, pos_scale=0.3 * X, base_z=0.0, joint_scale=0.5)
    g = ref.Grid(H, X, Y, 0.0, 0.0)
    for e in range(n):
        gc[e, 2] = g.height(gc[e, 0], gc[e, 1]) + rng.uniform(0.1, 0.3)
    gc = gc.astype(np.float32).astype(np.float64)
    check(capi, urdf, H, X, Y, 0.0, 0.0, gc, f"{urdf[:12]} pitch {pitch}", 200)
    bt, _ = kernel_lists(capi, urdf, H, X, Y, 0.0, 0.0, gc[:4])
    assert launch_config(capi, bt)["spec"] == spec


def test_gym_terminates_when_the_trunk_lands_on_a_peak(capi):
    """an ANYmal lowered belly-first onto a single peak 0.21 / 0.25 m ahead of its trunk centre (0.1 m map), its feet in the air: the
    trunk's box face touches the peak and the episode ends (the cell range once stopped one cell from the centre: no contact)"""
    path = os.path.join(RSC, "anymal_c_like.urdf")
    t = load_tables(path)
    xs = ys = 41
    H = np.zeros((ys, xs), np.float32); H[20, 23] = 0.8                    # the peak at (0.3, 0)
    m = capi.Model(path)
    n = 2
    bt = capi.Batch(m, n)
    bt.set_heightmap(xs, ys, 4.0, 4.0, 0.0, 0.0, H)
    box = int(np.where(t["pt_type"] == 2)[0][0])
    trunk = t["pt_coll"][box]
    gc = np.tile(ANYMAL_GC0, (n, 1))
    gc[:, 0] = 0.3 - np.array([0.21, 0.25]) - t["cpos"][trunk][0]            # trunk centre 0.21 / 0.25 m behind the peak
    gc[:, 2] = 0.8 + t["csize"][trunk][2] - t["cpos"][trunk][2] - 0.01       # bottom face 1 cm into the peak
    R = [ref.env_contacts(t, gc[e], ref.Grid(H, 4.0, 4.0, 0.0, 0.0)) for e in range(n)]
    for lst, amb in R:                                                       # the reference: the trunk face alone touches
        assert not amb and [c["pt"] for c in lst] == [box] and abs(lst[0]["depth"] - 0.01) < 1e-6
    kp = np.r_[np.zeros(6), 100.0 * np.ones(12)]; kd = np.r_[np.zeros(6), 2.0 * np.ones(12)]
    feet = [m.body_index(f"{leg}_FOOT") for leg in ("LF", "RF", "LH", "RH")]
    bt.set_pd_gains(kp, kd)
    bt.gym_configure(gc[0], np.zeros(18), gc[0, 7:], 0.6 * np.ones(12), feet)
    bt.gym_reset()
    bt.set_state(gc.astype(np.float32), np.zeros((n, 18), np.float32))
    obs = np.empty((n, 34), np.float32); rew = np.empty(n, np.float32); done = np.empty(n, np.uint8)
    bt.gym_step(np.zeros((n, 12), np.float32), 1, obs, rew, done)
    assert done.tolist() == [1, 1]
