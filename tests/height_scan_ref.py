"""Float64 numpy restatement of the terrain height scan (rsb_batch_set_height_scan / rsb_batch_get_height_scan): the sample locations of
body-attached points and the collision surface under them, clamped to the nearest border point outside a height map."""
import numpy as np


def surface_height(H, x_size, y_size, cx, cy, x, y):
    """height of the two-triangles-per-cell surface of the map H [ys, xs] (x fastest) at world (x, y), any shape; outside the map the
    nearest border point (HeightMap::getHeight); a coordinate that is not finite gives NaN"""
    H = np.asarray(H, np.float64)
    ys, xs = H.shape
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    finite = np.isfinite(x) & np.isfinite(y)
    x, y = np.where(finite, x, 0.0), np.where(finite, y, 0.0)
    dx, dy = x_size / (xs - 1), y_size / (ys - 1)
    gx = np.clip((x - (cx - 0.5 * x_size)) / dx, 0.0, xs - 1)
    gy = np.clip((y - (cy - 0.5 * y_size)) / dy, 0.0, ys - 1)
    ix, iy = np.minimum(gx.astype(np.int64), xs - 2), np.minimum(gy.astype(np.int64), ys - 2)
    fx, fy = gx - ix, gy - iy
    h00, h10, h01, h11 = H[iy, ix], H[iy, ix + 1], H[iy + 1, ix], H[iy + 1, ix + 1]
    z = np.where(fx >= fy, h00 + (h10 - h00) * fx + (h11 - h10) * fy, h00 + (h11 - h01) * fx + (h01 - h00) * fy)
    return np.where(finite, z, np.nan)


def sample_xy(R, p, body, xy, yaw=True):
    """world sample locations [n, P, 2] of points on body[P] at horizontal offsets xy [P, 2], from body poses R [n, nb, 3, 3] and
    p [n, nb, 3]: p_xy + Rz(psi) offset with (cos psi, sin psi) = (R00, R10) normalised (psi = 0 below 1e-6), or p_xy + offset"""
    R, p = np.asarray(R, np.float64), np.asarray(p, np.float64)
    body, xy = np.asarray(body), np.asarray(xy, np.float64)
    base = p[:, body, :2]
    if not yaw:
        return base + xy[None]
    c0, c1 = R[:, body, 0, 0], R[:, body, 1, 0]
    nrm = np.hypot(c0, c1)
    flat = nrm < 1e-6
    c = np.where(flat, 1.0, c0 / np.where(flat, 1.0, nrm))
    s = np.where(flat, 0.0, c1 / np.where(flat, 1.0, nrm))
    return base + np.stack([c * xy[None, :, 0] - s * xy[None, :, 1], s * xy[None, :, 0] + c * xy[None, :, 1]], -1)


def base_grid(nx=11, ny=17, x_extent=0.8, y_extent=0.5):
    """the nx x ny horizontal grid of a base-centred scan (legged_gym's 11 x 17 = 187 points: x in [-0.8, 0.8], y in [-0.5, 0.5])"""
    gx, gy = np.meshgrid(np.linspace(-x_extent, x_extent, nx), np.linspace(-y_extent, y_extent, ny), indexing="ij")
    return np.stack([gx.reshape(-1), gy.reshape(-1)], 1).astype(np.float32)
