"""The terrain height-scan entry points without a GPU: exported, declared with their argument types, a null batch refused before anything
touches a device; and the float64 restatement of tests/height_scan_ref.py, which the GPU tests compare against, checked on its own: the
triangle surface of a plane is the plane, outside the map the nearest border point, NaN for a diverged sample, and the yaw-aligned
sample pattern turns with the heading and ignores roll and pitch."""
import ctypes as C

import numpy as np

from raisimlib_b200 import capi
from helpers import axis_angle
from height_scan_ref import base_grid, sample_xy, surface_height


def test_entry_points_are_exported_and_typed():
    L = capi.lib()
    for name in ("rsb_batch_set_height_scan", "rsb_batch_get_height_scan"):
        assert name in capi.EXPORTED
        assert hasattr(L, name)
    assert L.rsb_batch_set_height_scan.argtypes == [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    assert L.rsb_batch_get_height_scan.argtypes == [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int]
    assert (capi.SCAN_YAW, capi.SCAN_WORLD, capi.MAX_SCAN_POINTS) == (0, 1, 1024)


def test_a_null_batch_is_refused():
    L = capi.lib()
    body, xy, h = (C.c_int32 * 1)(0), (C.c_float * 2)(0.1, 0.2), (C.c_float * 1)()
    assert L.rsb_batch_set_height_scan(None, body, xy, 1, capi.SCAN_YAW) == -1
    assert b"null batch" in L.rsb_last_error()
    assert L.rsb_batch_get_height_scan(None, 0, 1, h, None, capi.HOST) == -1
    assert b"null batch" in L.rsb_last_error()


def _plane_map(xs, ys, x_size, y_size, cx, cy, a, b, c):
    x = cx - 0.5 * x_size + np.arange(xs) * x_size / (xs - 1)
    y = cy - 0.5 * y_size + np.arange(ys) * y_size / (ys - 1)
    return a * x[None, :] + b * y[:, None] + c


def test_reference_is_exact_on_a_tilted_plane():
    """every sample inside the map of a plane z = a x + b y + c lies on the plane (both triangles of a cell, grid nodes and edges)"""
    xs, ys, sx, sy, cx, cy, a, b, c = 13, 9, 6.0, 4.0, 0.7, -0.4, 0.31, -0.17, 0.05
    H = _plane_map(xs, ys, sx, sy, cx, cy, a, b, c)
    rng = np.random.default_rng(3)
    x = rng.uniform(cx - sx / 2, cx + sx / 2, 2000)
    y = rng.uniform(cy - sy / 2, cy + sy / 2, 2000)
    assert np.abs(surface_height(H, sx, sy, cx, cy, x, y) - (a * x + b * y + c)).max() < 1e-12
    xn = cx - sx / 2 + np.arange(xs) * sx / (xs - 1)
    yn = cy - sy / 2 + np.arange(ys) * sy / (ys - 1)
    X, Y = np.meshgrid(xn, yn)
    assert np.abs(surface_height(H, sx, sy, cx, cy, X, Y) - H).max() < 1e-12


def test_reference_clamps_to_the_border_and_gives_nan_for_diverged_samples():
    """outside the map: the height of the nearest border point (on a plane: the plane at the clamped coordinates); a rough map's
    corners and edges; NaN or inf coordinates give NaN"""
    xs, ys, sx, sy, cx, cy, a, b, c = 13, 9, 6.0, 4.0, 0.7, -0.4, 0.31, -0.17, 0.05
    H = _plane_map(xs, ys, sx, sy, cx, cy, a, b, c)
    rng = np.random.default_rng(4)
    x, y = rng.uniform(-20, 20, 3000), rng.uniform(-20, 20, 3000)
    xc, yc = np.clip(x, cx - sx / 2, cx + sx / 2), np.clip(y, cy - sy / 2, cy + sy / 2)
    assert np.abs(surface_height(H, sx, sy, cx, cy, x, y) - (a * xc + b * yc + c)).max() < 1e-12
    R = rng.uniform(-0.3, 0.3, (ys, xs))
    x0, x1, y0, y1 = cx - sx / 2, cx + sx / 2, cy - sy / 2, cy + sy / 2
    corners = surface_height(R, sx, sy, cx, cy, [x0 - 5, x1 + 5, x0 - 5, x1 + 5], [y0 - 5, y0 - 5, y1 + 5, y1 + 5])
    assert np.array_equal(corners, [R[0, 0], R[0, -1], R[-1, 0], R[-1, -1]])
    xe = rng.uniform(x0, x1, 50)
    assert np.allclose(surface_height(R, sx, sy, cx, cy, xe, y1 + 3.0), surface_height(R, sx, sy, cx, cy, xe, y1), rtol=0, atol=1e-15)
    z = surface_height(R, sx, sy, cx, cy, [np.nan, 0.0, np.inf, -np.inf], [0.0, np.nan, 0.0, 1.0])
    assert np.isnan(z).all()


def test_reference_sample_pattern():
    """yaw alignment: the 187-point grid turns with the heading about the body origin and ignores roll and pitch; a body pitched by 90
    degrees (no heading) keeps the grid along the world axes; world alignment only translates"""
    xy = base_grid()
    assert xy.shape == (187, 2) and np.allclose(xy.min(0), [-0.8, -0.5]) and np.allclose(xy.max(0), [0.8, 0.5])
    psi, roll, pitch = 0.7, 0.3, -0.2
    Rz = axis_angle(np.array([0.0, 0.0, 1.0]), psi)
    Rfull = Rz @ axis_angle(np.array([0.0, 1.0, 0.0]), pitch) @ axis_angle(np.array([1.0, 0.0, 0.0]), roll)
    p = np.array([[[1.0, -2.0, 0.5]]])
    for R in (Rz, Rfull):
        got = sample_xy(R[None, None], p, [0] * len(xy), xy)[0]
        want = p[0, 0, :2] + xy.astype(np.float64) @ Rz[:2, :2].T
        assert np.abs(got - want).max() < 1e-12
    up = axis_angle(np.array([0.0, 1.0, 0.0]), np.pi / 2)
    got = sample_xy(up[None, None], p, [0] * len(xy), xy)[0]
    assert np.abs(got - (p[0, 0, :2] + xy)).max() < 1e-12
    got = sample_xy(Rfull[None, None], p, [0] * len(xy), xy, yaw=False)[0]
    assert np.abs(got - (p[0, 0, :2] + xy)).max() < 1e-12
