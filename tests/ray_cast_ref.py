"""Float64 restatement of the ray casts (rsb_batch_set_rays / rsb_batch_get_ray_casts), written from the contract (include/rsb.h,
DESIGN.md section 2).  It shares no code with the kernel: the terrain is every triangle of every cell that the xy bounding box of the
ray segment meets (no cell walk), each hit only when the ray crosses it from its upper side to its lower side; the robot's shapes are
intersected analytically on the poses they are given (helpers.fk_numpy in the tests).

Every ray also gets an `ambiguous` flag: float32 rounding of a pose or of the arithmetic may legitimately change its answer.  It is set
when the ray
  - passes within TOL (1e-4 m) of a surface it does not cross (a shape: the ray hits the shape grown by TOL but not the shape, or the
    shape but not the shape shrunk by TOL, or starts within TOL of its surface; the terrain: the ray's distance to a triangle it does
    not cross falls below TOL somewhere away from the hit, or it comes back up within DIP of where it went down);
  - hits at a grazing angle, |d.n| < GRAZE (on the terrain: on any triangle the ray's path meets within 1e-3 of the hit, since a hit
    on an edge or a diagonal belongs to both faces);
  - has two targets within TOL of each other along it;
  - hits within TOL of max_distance or of the map's outline."""
import math

import numpy as np

MISS, TERRAIN = -1, -2
TOL = 1e-4
GRAZE = 0.02
DIP = 2 * TOL / GRAZE            # a dip shallower than TOL at an incidence of at least GRAZE is shorter than this
CT_SPHERE, CT_BOX, CT_CAPSULE, CT_CYLINDER = 0, 1, 2, 3


def world_rays(R, p, body, origin, dir):
    """world (o [n, R, 3], d [n, R, 3]) of rays on body[R] with body-frame origin [R, 3] and direction [R, 3] (normalised here), from
    body poses R [n, nb, 3, 3] and p [n, nb, 3]"""
    R, p = np.asarray(R, np.float64), np.asarray(p, np.float64)
    body = np.asarray(body)
    u = np.asarray(dir, np.float64)
    u = u / np.linalg.norm(u, axis=1, keepdims=True)
    o = p[:, body] + np.einsum("nrij,rj->nri", R[:, body], np.asarray(origin, np.float64))
    d = np.einsum("nrij,rj->nri", R[:, body], u)
    return o, d


# ---- robot shapes -----------------------------------------------------------------------------------------------------------------

def _sphere(o, d, r):
    """entry t > 0 of the unit ray o + t d into the ball |x| <= r from outside; None when it starts inside or on it, or misses"""
    c = o @ o - r * r
    if c <= 0:
        return None
    b = o @ d
    disc = b * b - c
    if disc < 0 or b >= 0:
        return None
    return -b - math.sqrt(disc)


def _box(o, d, h):
    if np.all(np.abs(o) <= h):
        return None
    tn, tf = 0.0, math.inf
    for k in range(3):
        if d[k] == 0:
            if abs(o[k]) > h[k]:
                return None
            continue
        t0, t1 = (-h[k] - o[k]) / d[k], (h[k] - o[k]) / d[k]
        tn, tf = max(tn, min(t0, t1)), min(tf, max(t0, t1))
    return tn if 0 < tn <= tf else None


def _cyl_side(o, d, r, hl):
    """entry through the side x^2 + y^2 = r^2, |z| <= hl, from outside the infinite cylinder"""
    a = d[0] ** 2 + d[1] ** 2
    c = o[0] ** 2 + o[1] ** 2 - r * r
    if a == 0 or c <= 0:
        return None
    b = o[0] * d[0] + o[1] * d[1]
    disc = b * b - a * c
    if disc < 0 or b >= 0:
        return None
    t = (-b - math.sqrt(disc)) / a
    return t if abs(o[2] + t * d[2]) <= hl else None


def _first(*ts):
    ts = [t for t in ts if t is not None and t > 0]
    return min(ts) if ts else None


def shape_entry(typ, size, o, d, grow=0.0):
    """entry t of the unit ray (o, d), in the shape's local frame, into the shape grown by `grow` (negative: shrunk); None when the origin
    is inside or on it, or the ray does not enter it"""
    o, d = np.asarray(o, np.float64), np.asarray(d, np.float64)
    if typ == CT_SPHERE:
        return _sphere(o, d, size[0] + grow)
    if typ == CT_BOX:
        return _box(o, d, np.asarray(size, np.float64) + grow)
    r, hl = size[0] + grow, size[1]
    if typ == CT_CAPSULE:
        zc = min(max(o[2], -hl), hl)
        if (o[0] ** 2 + o[1] ** 2 + (o[2] - zc) ** 2) <= r * r:
            return None
        return _first(_cyl_side(o, d, r, hl), _sphere(o - [0, 0, hl], d, r), _sphere(o + [0, 0, hl], d, r))
    hl = hl + grow
    if o[0] ** 2 + o[1] ** 2 <= r * r and abs(o[2]) <= hl:
        return None
    caps = []
    for zp in (hl, -hl):
        if d[2] != 0 and (zp - o[2]) * d[2] > 0 and abs(o[2]) > hl and np.sign(o[2]) == np.sign(zp):
            t = (zp - o[2]) / d[2]
            q = o + t * d
            if q[0] ** 2 + q[1] ** 2 <= r * r:
                caps.append(t)
    return _first(_cyl_side(o, d, r, hl), *caps)


def robot_hits(t, R, p, o, d):
    """[(t, collision body, ambiguous)] of one ray (world o, d) against every collision body of the model tables t, on body poses
    R [nb, 3, 3], p [nb, 3]"""
    out = []
    for c in range(t["ncoll"]):
        b = t["cbody"][c]
        Rc = R[b] @ np.asarray(t["crot"][c], np.float64).reshape(3, 3)
        cc = p[b] + R[b] @ np.asarray(t["cpos"][c], np.float64)
        ol, dl = Rc.T @ (o - cc), Rc.T @ d
        size = np.asarray(t["csize"][c], np.float64)
        typ = t["ctype"][c]
        te, tg, ts = shape_entry(typ, size, ol, dl), shape_entry(typ, size, ol, dl, TOL), shape_entry(typ, size, ol, dl, -TOL)
        amb = (te is None) != (tg is None) or (te is None) != (ts is None)
        if te is not None and tg is not None and te - tg > TOL / GRAZE:    # grazing: growing the shape moves the entry far
            amb = True
        if te is not None or amb:
            out.append((te if te is not None else (tg if tg is not None else 0.0), c, amb or te is None))
    return out


# ---- terrain ----------------------------------------------------------------------------------------------------------------------

def terrain_hit(g, o, d, max_distance, zlo=None, zhi=None):
    """(t or None, ambiguous) of one ray against the height map of terrain_contact_ref.Grid g: every triangle of every cell that the xy
    bounding box of the segment o + t d, t in [0, max_distance], meets (the segment first clipped to the z range of the map), hit where
    the ray crosses it downwards (d.n < 0, n the upward normal)"""
    o, d = np.asarray(o, np.float64), np.asarray(d, np.float64)
    zlo = g.H.min() if zlo is None else zlo
    zhi = g.H.max() if zhi is None else zhi
    t0, t1 = 0.0, max_distance
    if d[2] != 0:
        a, b = (zlo - 1e-3 - o[2]) / d[2], (zhi + 1e-3 - o[2]) / d[2]
        t0, t1 = max(t0, min(a, b)), min(t1, max(a, b))
    elif not zlo - 1e-3 <= o[2] <= zhi + 1e-3:
        return None, False
    if t0 > t1:
        return None, False
    A, B = o + t0 * d, o + t1 * d
    cells = g.cells(min(A[0], B[0]), max(A[0], B[0]), min(A[1], B[1]), max(A[1], B[1]))
    if not cells:
        return None, False
    ix, iy = np.array(cells).T
    # the two triangles of every cell: vertices [m, 3, 3]
    X0, Y0 = g.x0 + ix * g.dx, g.y0 + iy * g.dy
    P00 = np.stack([X0, Y0, g.H[iy, ix]], -1); P10 = np.stack([X0 + g.dx, Y0, g.H[iy, ix + 1]], -1)
    P01 = np.stack([X0, Y0 + g.dy, g.H[iy + 1, ix]], -1); P11 = np.stack([X0 + g.dx, Y0 + g.dy, g.H[iy + 1, ix + 1]], -1)
    V = np.concatenate([np.stack([P00, P10, P11], 1), np.stack([P00, P11, P01], 1)])
    n = np.cross(V[:, 1] - V[:, 0], V[:, 2] - V[:, 0])
    n /= np.linalg.norm(n, axis=1, keepdims=True)            # upward: n_z > 0 for both triangles
    # the ray's xy path clipped to each triangle: t interval where the projection is inside (three half-planes, counter-clockwise)
    lo, hi = np.full(len(V), t0), np.full(len(V), t1)
    for k in range(3):
        a, b = V[:, k, :2], V[:, (k + 1) % 3, :2]
        e = b - a
        # inside: cross(e, x - a) >= 0 with x = o + t d
        c0 = e[:, 0] * (o[1] - a[:, 1]) - e[:, 1] * (o[0] - a[:, 0])
        c1 = e[:, 0] * d[1] - e[:, 1] * d[0]
        with np.errstate(divide="ignore", invalid="ignore"):
            tc = -c0 / c1
        lo = np.where(c1 > 0, np.maximum(lo, tc), lo)
        hi = np.where(c1 < 0, np.minimum(hi, tc), hi)
        dead = (c1 == 0) & (c0 < 0)
        hi = np.where(dead, -np.inf, hi)
    live = lo <= hi
    V, n, lo, hi = V[live], n[live], lo[live], hi[live]
    if not len(V):
        return None, False
    # signed distance of the ray to each triangle's plane at both ends of its piece
    fa = np.einsum("mk,mk->m", o + lo[:, None] * d - V[:, 0], n)
    fb = np.einsum("mk,mk->m", o + hi[:, None] * d - V[:, 0], n)
    dn = n @ d
    down = (fa >= 0) & (fb < 0) & (dn < 0)
    with np.errstate(divide="ignore", invalid="ignore"):
        tcross = np.where(dn != 0, lo + fa / np.where(dn != 0, -dn, 1.0), np.inf)
    down &= tcross > 0
    t_hit = tcross[down].min() if down.any() else None
    amb = False
    if t_hit is not None:
        # grazing: on any triangle the ray's path meets near the hit (a hit on an edge or a diagonal belongs to both faces)
        at_hit = (lo <= t_hit + 1e-3) & (hi >= t_hit - 1e-3)
        amb |= bool((np.abs(dn[at_hit]) < GRAZE).any())
        amb |= t_hit > max_distance - TOL
        hp = o + t_hit * d
        amb |= bool(g.near_edge(hp[0], hp[1], TOL))
        up = (fa < 0) & (fb >= 0)
        with np.errstate(divide="ignore", invalid="ignore"):
            tup = np.where(up & (dn != 0), lo + fa / np.where(dn != 0, -dn, 1.0), np.inf)
        amb |= bool(((tup > t_hit) & (tup < t_hit + DIP)).any())
    # near misses: a piece that does not cross its plane but comes within TOL of it, away from the hit
    cross = (fa >= 0) != (fb >= 0)
    near_t = np.where(np.abs(fa) < np.abs(fb), lo, hi)
    near = ~cross & (np.minimum(np.abs(fa), np.abs(fb)) < TOL)
    if t_hit is not None:
        near &= (near_t < t_hit - 1e-3)
    amb |= bool(near.any())
    return t_hit, bool(amb)


def ground_hit(z0, o, d, max_distance):
    o, d = np.asarray(o, np.float64), np.asarray(d, np.float64)
    if d[2] < 0 and o[2] > z0:
        t = (z0 - o[2]) / d[2]
        if t <= max_distance:
            return t, abs(d[2]) < GRAZE or t > max_distance - TOL
        return None, t < max_distance + TOL
    return None, False


def ray_casts(o, d, max_distance, terrain=None, tables=None, R=None, p=None):
    """reference of one environment: o, d [n, 3] world rays; terrain None, ("ground", z0) or ("map", Grid); with tables (model tables),
    R [nb, 3, 3] and p [nb, 3] the robot's collision bodies are targets too.  -> (distance [n], hit [n] int, ambiguous [n] bool)"""
    n = len(o)
    dist, hit, amb = np.full(n, np.inf), np.full(n, MISS, np.int64), np.zeros(n, bool)
    for i in range(n):
        oi, di = o[i], d[i]
        if not (np.isfinite(oi).all() and np.isfinite(di).all()):
            dist[i] = np.nan
            continue
        cands = []
        if terrain is not None:
            th, ta = (ground_hit(terrain[1], oi, di, max_distance) if terrain[0] == "ground"
                      else terrain_hit(terrain[1], oi, di, max_distance))
            amb[i] |= ta
            if th is not None:
                cands.append((th, TERRAIN))
        if tables is not None:
            for tc, c, a in robot_hits(tables, R, p, oi, di):
                amb[i] |= a
                if tc > 0:
                    cands.append((tc, c))
        cands = sorted(c for c in cands if c[0] <= max_distance + TOL)
        amb[i] |= any(abs(c[0] - max_distance) < TOL for c in cands)
        cands = [c for c in cands if c[0] <= max_distance]
        if cands:
            dist[i], hit[i] = cands[0]
            if len(cands) > 1 and cands[1][0] - cands[0][0] < TOL:
                amb[i] = True
    return dist, hit, amb
