"""The ray-cast entry points without a GPU: exported, declared with their argument types, a null batch refused before anything touches a
device; the float64 restatement of tests/ray_cast_ref.py, which the GPU tests compare against, checked on its own against known answers
for the terrain and every shape type, the origin-inside rule and a fine float64 march over rough maps; and the geometry of
capi.pinhole_rays."""
import ctypes as C
import math

import numpy as np
import pytest

from raisimlib_b200 import capi
from ray_cast_ref import CT_BOX, CT_CAPSULE, CT_CYLINDER, CT_SPHERE, MISS, TERRAIN, ground_hit, ray_casts, shape_entry, terrain_hit
from terrain_contact_ref import Grid


def test_entry_points_are_exported_and_typed():
    L = capi.lib()
    for name in ("rsb_batch_set_rays", "rsb_batch_get_ray_casts"):
        assert name in capi.EXPORTED
        assert hasattr(L, name)
    assert L.rsb_batch_set_rays.argtypes == [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_float, C.c_int]
    assert L.rsb_batch_get_ray_casts.argtypes == [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int]
    assert (capi.MAX_RAYS, capi.RAY_MISS, capi.RAY_TERRAIN, capi.RAYS_TERRAIN, capi.RAYS_TERRAIN_AND_ROBOT) == (16384, -1, -2, 0, 1)


def test_a_null_batch_is_refused():
    L = capi.lib()
    body, o, d, dist = (C.c_int32 * 1)(0), (C.c_float * 3)(0, 0, 0), (C.c_float * 3)(1, 0, 0), (C.c_float * 1)()
    assert L.rsb_batch_set_rays(None, body, o, d, 1, 5.0, capi.RAYS_TERRAIN) == -1
    assert b"null batch" in L.rsb_last_error()
    assert L.rsb_batch_get_ray_casts(None, 0, 1, dist, None, capi.HOST) == -1
    assert b"null batch" in L.rsb_last_error()


def _plane_grid(a, b, c, xs=21, ys=17, size=(4.0, 3.0), cx=0.3, cy=-0.2):
    x = cx - 0.5 * size[0] + np.arange(xs) * size[0] / (xs - 1)
    y = cy - 0.5 * size[1] + np.arange(ys) * size[1] / (ys - 1)
    return Grid(a * x[None, :] + b * y[:, None] + c, size[0], size[1], cx, cy)


def _unit(v):
    v = np.asarray(v, np.float64)
    return v / np.linalg.norm(v)


def test_tilted_plane_known_answers():
    """rays onto the plane z = a x + b y + c: the hit is the analytic intersection; rays from below, rays that leave the map first,
    rays pointing up and rays stopped by max_distance miss"""
    a, b, c = 0.2, -0.1, 0.05
    g = _plane_grid(a, b, c)
    rng = np.random.default_rng(1)
    n = np.array([-a, -b, 1.0]) / math.sqrt(a * a + b * b + 1)
    for _ in range(200):
        x, y = rng.uniform(-1.2, 1.6), rng.uniform(-1.2, 0.8)
        o = np.array([x, y, a * x + b * y + c + rng.uniform(0.2, 1.5)])
        d = _unit([rng.uniform(-0.5, 0.5), rng.uniform(-0.5, 0.5), -1.0])
        t_true = ((np.array([0, 0, c]) - o) @ n) / (d @ n)
        q = o + t_true * d
        t, amb = terrain_hit(g, o, d, 10.0)
        if g.on_map(q[0], q[1]) and not g.near_edge(q[0], q[1], 1e-3):
            assert t is not None and abs(t - t_true) < 1e-12 and not amb
        t, _ = terrain_hit(g, o, -d, 10.0)                     # away from the surface
        assert t is None
        below = o.copy(); below[2] = a * x + b * y + c - 0.3
        assert terrain_hit(g, below, d, 10.0)[0] is None       # starts under it and only goes further down
        assert terrain_hit(g, o, d, 0.5 * t_true)[0] is None   # out of range
    o = np.array([0.3, -0.2, 5.0])
    assert terrain_hit(g, o + [10.0, 0, 0], [0, 0, -1.0], 20.0)[0] is None   # off the map: no walls, no floor


def test_flat_map_matches_the_ground_plane():
    g = Grid(np.full((9, 11), 0.25), 2.0, 1.6, 0.0, 0.0)
    rng = np.random.default_rng(2)
    for _ in range(100):
        o = np.array([rng.uniform(-0.8, 0.8), rng.uniform(-0.6, 0.6), rng.uniform(0.3, 2.0)])
        d = _unit([rng.uniform(-0.2, 0.2), rng.uniform(-0.2, 0.2), -1.0])
        tm, _ = terrain_hit(g, o, d, 20.0)
        tg, _ = ground_hit(0.25, o, d, 20.0)
        q = o + tg * d
        if abs(q[0]) < 0.95 and abs(q[1]) < 0.75:
            assert abs(tm - tg) < 1e-12
    assert ground_hit(0.25, np.array([0, 0, 0.1]), np.array([0, 0, 1.0]), 5.0)[0] is None   # from below: never
    assert ground_hit(0.25, np.array([0, 0, 0.1]), np.array([0, 0, -1.0]), 5.0)[0] is None


def test_ray_coming_back_up_through_the_surface():
    """an origin under a ridge: the ray must come up through the surface and go down through it again before it hits"""
    H = np.zeros((3, 41)); H[:, 20] = 1.0                   # a ridge along y at x = 0, 1 m high, 0.1 m pitch
    g = Grid(H, 4.0, 0.2, 0.0, 0.0)
    o = np.array([-0.05, 0.0, 0.2])                          # inside the ridge, under its surface
    t, _ = terrain_hit(g, o, _unit([1.0, 0.0, 0.0]), 5.0)
    assert t is None                                          # leaves through the far slope going up... and stays at z = 0.2 over flat ground
    d = _unit([1.0, 0.0, -0.1])
    t, _ = terrain_hit(g, o, d, 5.0)
    # it comes out of the far slope (z = 10 (0.1 - x)) and then meets the flat ground z = 0
    assert t is not None and abs((o + t * d)[2]) < 1e-12


def test_sphere_known_answers():
    r = 0.3
    o = np.array([-2.0, 0.0, 0.0])
    assert abs(shape_entry(CT_SPHERE, [r, 0, 0], o, _unit([1, 0, 0])) - (2.0 - r)) < 1e-12          # head on
    assert shape_entry(CT_SPHERE, [r, 0, 0], o, _unit([1, 0.2, 0])) is None                          # misses
    t = shape_entry(CT_SPHERE, [r, 0, 0], o, _unit([1, math.tan(math.asin(r / 2.0)) * 0.999, 0]))   # nearly grazing
    assert t is not None and abs(t - math.sqrt(4 - r * r)) < 0.05
    assert shape_entry(CT_SPHERE, [r, 0, 0], o, _unit([1, math.tan(math.asin(r / 2.0)) * 1.001, 0])) is None
    assert shape_entry(CT_SPHERE, [r, 0, 0], o, _unit([-1, 0, 0])) is None                           # behind
    assert shape_entry(CT_SPHERE, [r, 0, 0], np.array([0.1, 0, 0]), _unit([1, 0, 0])) is None        # origin inside
    assert shape_entry(CT_SPHERE, [r, 0, 0], np.array([r, 0, 0]), _unit([-1, 0, 0])) is None         # origin on it


def test_capsule_side_and_cap():
    r, hl = 0.1, 0.3
    size = [r, hl, 0]
    assert abs(shape_entry(CT_CAPSULE, size, np.array([-1.0, 0, 0.2]), _unit([1, 0, 0])) - 0.9) < 1e-12   # side
    assert abs(shape_entry(CT_CAPSULE, size, np.array([0, 0, 2.0]), _unit([0, 0, -1])) - (2.0 - hl - r)) < 1e-12   # end cap
    t = shape_entry(CT_CAPSULE, size, np.array([0.05, 0, 2.0]), _unit([0, 0, -1]))
    assert abs(t - (2.0 - hl - math.sqrt(r * r - 0.05 ** 2))) < 1e-12
    assert shape_entry(CT_CAPSULE, size, np.array([-1.0, 0, 0.45]), _unit([1, 0, 0])) is None         # above the end sphere
    assert shape_entry(CT_CAPSULE, size, np.array([0, 0, 0.35]), _unit([0, 0, 1])) is None            # origin in the end sphere


def test_box_face_and_edge():
    h = [0.2, 0.1, 0.05]
    assert abs(shape_entry(CT_BOX, h, np.array([-1.0, 0.03, 0.01]), _unit([1, 0, 0])) - 0.8) < 1e-12   # face
    d = _unit([1, 1, 0])
    t = shape_entry(CT_BOX, h, np.array([-1.0, -0.9, 0.0]) , d)                                     # through the edge x = -0.2, y = -0.1
    assert t is not None and np.allclose(np.array([-1.0, -0.9, 0.0]) + t * d, [-0.2, -0.1, 0.0], atol=1e-12)
    assert shape_entry(CT_BOX, h, np.array([-1.0, -0.6999, 0.0]), d) is None                         # passes just outside the edge x = -0.2, y = 0.1
    assert shape_entry(CT_BOX, h, np.array([-1.0, -0.7001, 0.0]), d) is not None                     # clips it
    assert shape_entry(CT_BOX, h, np.array([0.0, 0.0, 0.0]), d) is None                              # origin inside: a camera in the base box
    assert shape_entry(CT_BOX, h, np.array([0.2, 0.0, 0.0]), _unit([-1, 0, 0])) is None              # origin on the face


def test_cylinder_side_and_cap():
    r, hl = 0.1, 0.3
    size = [r, hl, 0]
    assert abs(shape_entry(CT_CYLINDER, size, np.array([-1.0, 0, 0.29]), _unit([1, 0, 0])) - 0.9) < 1e-12   # side
    assert abs(shape_entry(CT_CYLINDER, size, np.array([0.05, 0.05, 2.0]), _unit([0, 0, -1])) - 1.7) < 1e-12  # cap
    assert abs(shape_entry(CT_CYLINDER, size, np.array([0.0, 0.0, -2.0]), _unit([0, 0, 1])) - 1.7) < 1e-12   # the other cap
    assert shape_entry(CT_CYLINDER, size, np.array([-1.0, 0, 0.31]), _unit([1, 0, 0])) is None             # above the top cap
    d = _unit([1, 0, -1])
    t = shape_entry(CT_CYLINDER, size, np.array([-0.6, 0, 0.8]), d)                                      # meets the cap's rim region
    q = np.array([-0.6, 0, 0.8]) + t * d
    assert abs(q[2] - hl) < 1e-12 or abs(math.hypot(q[0], q[1]) - r) < 1e-12
    assert shape_entry(CT_CYLINDER, size, np.array([0.0, 0.0, 0.0]), _unit([1, 0, 0])) is None


def test_origin_inside_a_shape_sees_out_of_it():
    """a camera inside the base box of a one-body robot sees the ground, not the box; from outside the box hides the ground"""
    t = dict(ncoll=1, cbody=np.array([0]), ctype=np.array([CT_BOX]), csize=np.array([[0.3, 0.2, 0.1]]), cpos=np.zeros((1, 3)),
             crot=np.eye(3).reshape(1, 9))
    R, p = np.eye(3)[None], np.array([[0.0, 0.0, 0.5]])
    o = np.array([[0.25, 0.0, 0.5], [0.0, 0.0, 0.9]])
    d = np.array([_unit([0.5, 0, -1]), _unit([0, 0, -1])])
    dist, hit, amb = ray_casts(o, d, 5.0, ("ground", 0.0), t, R, p)
    assert hit[0] == TERRAIN and abs(dist[0] - 0.5 / (1 / math.sqrt(1.25))) < 1e-12
    assert hit[1] == 0 and abs(dist[1] - 0.3) < 1e-12
    dist, hit, _ = ray_casts(o, d, 5.0, None, t, R, p)
    assert hit[0] == MISS and np.isinf(dist[0])
    dist, hit, _ = ray_casts(np.array([[np.nan, 0, 0]]), d[:1], 5.0, ("ground", 0.0))
    assert np.isnan(dist[0]) and hit[0] == MISS


def _march(g, o, d, max_distance, step=1e-4):
    """the first t on a float64 march where the ray goes from above the surface (over the map) to below it"""
    ts = np.arange(step, max_distance + step / 2, step)
    P = o[None] + ts[:, None] * d[None]
    gx, gy = (P[:, 0] - g.x0) / g.dx, (P[:, 1] - g.y0) / g.dy
    on = (gx >= 0) & (gx <= g.xs - 1) & (gy >= 0) & (gy <= g.ys - 1)
    ix = np.clip(np.floor(gx), 0, g.xs - 2).astype(int); iy = np.clip(np.floor(gy), 0, g.ys - 2).astype(int)
    fx, fy = gx - ix, gy - iy
    H = g.H
    h00, h10, h01, h11 = H[iy, ix], H[iy, ix + 1], H[iy + 1, ix], H[iy + 1, ix + 1]
    h = np.where(fx >= fy, h00 + (h10 - h00) * fx + (h11 - h10) * fy, h00 + (h11 - h01) * fx + (h01 - h00) * fy)
    above = P[:, 2] - h >= 0
    prev = np.r_[o[2] - h[0] > 0 if on[0] else True, above[:-1]]
    prev_on = np.r_[on[0], on[:-1]]
    k = np.nonzero(on & prev_on & prev & ~above)[0]
    return ts[k[0]] if len(k) else None


def test_first_crossing_agrees_with_a_fine_march():
    """random rays over random rough maps: the reference's first crossing is the first sign change of a 1e-4 m float64 march, within
    one step, wherever the reference calls the ray unambiguous"""
    rng = np.random.default_rng(7)
    checked = 0
    for m in range(4):
        H = rng.uniform(-0.15, 0.15, (31, 41))
        g = Grid(H, 4.0, 3.0, 0.2 * m, -0.1 * m)
        for _ in range(60):
            o = np.array([g.x0 + rng.uniform(0.2, 3.8), g.y0 + rng.uniform(0.2, 2.8), rng.uniform(-0.05, 0.6)])
            d = _unit([rng.uniform(-1, 1), rng.uniform(-1, 1), rng.uniform(-0.8, 0.1)])
            t, amb = terrain_hit(g, o, d, 2.5)
            if amb:
                continue
            tm = _march(g, o, d, 2.5)
            checked += 1
            if t is None:
                assert tm is None
            else:
                assert tm is not None and -1e-9 <= tm - t <= 1e-4 + 1e-9, (t, tm)
    assert checked > 150


def test_pinhole_geometry():
    """pixel centres, the optical axis, square pixels, row-major order from the top-left pixel, and the z-depth of a plane facing the
    camera being constant"""
    W, Hh, hfov = 8, 6, 90.0
    d = capi.pinhole_rays(W, Hh, hfov)
    assert d.shape == (W * Hh, 3) and np.allclose(np.linalg.norm(d, axis=1), 1.0)
    f = 0.5 * W / math.tan(math.radians(hfov) / 2)
    img = d.reshape(Hh, W, 3)
    u = -img[..., 1] / img[..., 0] * f + 0.5 * W      # column of the pixel centre
    v = -img[..., 2] / img[..., 0] * f + 0.5 * Hh     # row
    assert np.allclose(u, np.arange(W)[None] + 0.5) and np.allclose(v, np.arange(Hh)[:, None] + 0.5)
    assert img[0, 0, 1] > 0 and img[0, 0, 2] > 0      # top-left: left (+y) and up (+z)
    assert img[-1, -1, 1] < 0 and img[-1, -1, 2] < 0
    c = capi.pinhole_rays(1, 1, 60.0)
    assert np.allclose(c, [[1.0, 0.0, 0.0]])          # a single pixel looks along the optical axis
    # the outermost pixel centres of a row span the horizontal field of view less half a pixel on each side
    assert abs(math.degrees(math.atan2(img[0, 0, 1], img[0, 0, 0])) - math.degrees(math.atan((0.5 * W - 0.5) / f))) < 1e-9
    # z-depth: distance to the plane x = 2 times dirs[:, 0] is 2 for every pixel
    dist = 2.0 / d[:, 0]
    assert np.allclose(dist * d[:, 0], 2.0)
    with pytest.raises(ValueError):
        capi.pinhole_rays(0, 4, 60.0)
    with pytest.raises(ValueError):
        capi.pinhole_rays(4, 4, 180.0)
