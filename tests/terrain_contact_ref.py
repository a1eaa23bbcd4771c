"""Exact float64 restatement of the height-map narrow phase, written from the contract (DESIGN.md section 2, include/rsb.h) for the
tests: every collision candidate against EVERY triangle, edge or vertex of the cells under its horizontal reach, with no limit on the
size of the shape against the grid pitch.  It shares no routine with the oracle or the kernel: the closest point of a triangle is a
projection on its plane followed by the three edge segments (not a walk over Voronoi regions), and the closest points of two segments
come from the interior stationary point and the four clamped boundary problems.

Grid: samples H[iy, ix] at (x0 + ix dx, y0 + iy dy); cell (ix, iy) holds tri 0 = (P00, P10, P11) and tri 1 = (P00, P11, P01);
pair index = 2 (iy (xs - 1) + ix) + tri.  A candidate whose centre (sphere centre, segment midpoint, box centre, point) is off the map
has no contact.

Every contact is a dict: pt, body, pair, depth, n (terrain -> robot), pos, and two entries the comparisons use:
  alts      (pair, normal) of every feature within TIE_TOL of the chosen one, itself included: a float32 pose may pick any of them;
  unpinned  a buried sphere centre whose nearest surface point lies outside the footprint [C +- r]: the contract only says the contact
            is deeper than r.
"""
import math

import numpy as np

KMAX = 8                 # RSB_KMAX: contacts kept per environment
TIE = 1e-6               # the contract's tie width: features within TIE of the best go to the lowest pair index
TIE_TOL = 1e-5           # what the comparisons treat as a near-tie (float32 rounding of a pose moves depths by ~1e-7 m)


class Grid:
    def __init__(self, H, x_size, y_size, cx, cy):
        self.H = np.asarray(H, np.float64)
        self.ys, self.xs = self.H.shape
        self.dx, self.dy = x_size / (self.xs - 1), y_size / (self.ys - 1)
        self.x0, self.y0 = cx - 0.5 * x_size, cy - 0.5 * y_size

    def v(self, ix, iy):
        return np.array([self.x0 + ix * self.dx, self.y0 + iy * self.dy, self.H[iy, ix]])

    def on_map(self, x, y):
        gx, gy = (x - self.x0) / self.dx, (y - self.y0) / self.dy
        return 0.0 <= gx < self.xs - 1 and 0.0 <= gy < self.ys - 1

    def near_edge(self, x, y, tol=1e-5):
        """within tol (m) of the map's outline: float32 rounding of the pose may put the centre on either side"""
        ex, ey = self.x0 + (self.xs - 1) * self.dx, self.y0 + (self.ys - 1) * self.dy
        return (self.x0 - tol <= x <= ex + tol and self.y0 - tol <= y <= ey + tol and
                min(abs(x - self.x0), abs(x - ex), abs(y - self.y0), abs(y - ey)) < tol)

    def cells(self, lox, hix, loy, hiy):
        """cells (ix, iy) whose square meets [lox, hix] x [loy, hiy], iy-major"""
        ix0 = max(math.floor((lox - self.x0) / self.dx), 0); ix1 = min(math.floor((hix - self.x0) / self.dx), self.xs - 2)
        iy0 = max(math.floor((loy - self.y0) / self.dy), 0); iy1 = min(math.floor((hiy - self.y0) / self.dy), self.ys - 2)
        return [(ix, iy) for iy in range(iy0, iy1 + 1) for ix in range(ix0, ix1 + 1)]

    def height(self, x, y):
        """the surface height at (x, y), clamped onto the map"""
        gx = min(max((x - self.x0) / self.dx, 0.0), self.xs - 1 - 1e-9); gy = min(max((y - self.y0) / self.dy, 0.0), self.ys - 1 - 1e-9)
        ix, iy = int(gx), int(gy)
        a, b, c = self.tri(ix, iy, 0 if gx - ix >= gy - iy else 1)
        n = np.cross(b - a, c - a)
        return a[2] - (n[0] * (x - a[0]) + n[1] * (y - a[1])) / n[2]

    def tri(self, ix, iy, t):
        p00, p10, p01, p11 = self.v(ix, iy), self.v(ix + 1, iy), self.v(ix, iy + 1), self.v(ix + 1, iy + 1)
        return (p00, p10, p11) if t == 0 else (p00, p11, p01)

    def pair(self, ix, iy, t):
        return 2 * (iy * (self.xs - 1) + ix) + t


def tri_normal(a, b, c):
    n = np.cross(b - a, c - a)
    n = n / np.linalg.norm(n)
    return n if n[2] >= 0 else -n


def closest_on_segment(p, a, b):
    d = b - a
    s = np.clip(np.dot(p - a, d) / np.dot(d, d), 0.0, 1.0)
    return a + s * d


def closest_on_triangle(p, a, b, c):
    """the plane projection when it falls inside the triangle (barycentric coordinates by area ratios), else the nearest of the
    three edge segments' closest points"""
    n = np.cross(b - a, c - a)
    q = p - np.dot(p - a, n) / np.dot(n, n) * n
    nn = np.dot(n, n)
    wa = np.dot(np.cross(c - b, q - b), n) / nn
    wb = np.dot(np.cross(a - c, q - c), n) / nn
    wc = 1.0 - wa - wb
    if wa >= 0.0 and wb >= 0.0 and wc >= 0.0:
        return q
    cands = [closest_on_segment(p, a, b), closest_on_segment(p, b, c), closest_on_segment(p, c, a)]
    return min(cands, key=lambda x: np.dot(p - x, p - x))


def closest_segments(p1, q1, p2, q2):
    """(s, t) minimising |p1 + s d1 - p2 - t d2| over [0, 1]^2: the interior stationary point if it is inside, else the best of the
    four edges of the square, each a clamped one-dimensional problem"""
    d1, d2, r = q1 - p1, q2 - p2, p1 - p2
    a, b, e = np.dot(d1, d1), np.dot(d1, d2), np.dot(d2, d2)
    c, f = np.dot(d1, r), np.dot(d2, r)
    f2 = lambda s, t: np.dot(r + s * d1 - t * d2, r + s * d1 - t * d2)
    cand = []
    den = a * e - b * b
    if den > 1e-14 * a * e:
        s, t = (b * f - c * e) / den, (a * f - b * c) / den
        if 0.0 <= s <= 1.0 and 0.0 <= t <= 1.0:
            return s, t
    for s in (0.0, 1.0):
        cand.append((s, float(np.clip((b * s + f) / e, 0.0, 1.0))))
    for t in (0.0, 1.0):
        cand.append((float(np.clip((b * t - c) / a, 0.0, 1.0)), t))
    return min(cand, key=lambda st: f2(*st))


def _pick(hits):
    """deepest hit; hits within TIE of it go to the lowest pair index.  alts = (pair, normal) of every hit within TIE_TOL of the deepest:
    a float32 pose may tip the choice to any of them"""
    if not hits:
        return None
    dmax = max(h["depth"] for h in hits)
    best = dict(min((h for h in hits if h["depth"] >= dmax - TIE), key=lambda h: h["pair"]))
    best["alts"] = [(h["pair"], h["n"]) for h in hits if h["depth"] >= dmax - TIE_TOL]
    return best


def point_contact(g, P, rad=0.0):
    """zero-radius point (box corner, cylinder rim point): the triangle directly beneath, depth rad - signed distance to its plane"""
    if not g.on_map(P[0], P[1]):
        return None, 0.0 if g.near_edge(P[0], P[1]) else np.inf
    gx, gy = (P[0] - g.x0) / g.dx, (P[1] - g.y0) / g.dy
    ix, iy = int(gx), int(gy)
    t = 0 if gx - ix >= gy - iy else 1
    a, b, c = g.tri(ix, iy, t)
    n = tri_normal(a, b, c)
    depth = rad - np.dot(P - a, n)
    near = 0.0 if g.near_edge(P[0], P[1]) else abs(depth)
    if not depth > 0.0:
        return None, near
    return dict(pair=g.pair(ix, iy, t), depth=depth, n=n, pos=P - rad * n, alts=[(g.pair(ix, iy, t), n)], unpinned=False), near


def sphere_contact(g, C, r):
    """the closest point of the triangles under the footprint [C +- r]; inside / outside from the triangle beneath the centre"""
    if not g.on_map(C[0], C[1]):
        return None, 0.0 if g.near_edge(C[0], C[1]) else np.inf
    gx, gy = (C[0] - g.x0) / g.dx, (C[1] - g.y0) / g.dy
    ix, iy = int(gx), int(gy)
    tb = 0 if gx - ix >= gy - iy else 1
    a, b, c = g.tri(ix, iy, tb)
    side = np.dot(C - a, tri_normal(a, b, c))
    inside = side < 0.0
    on_edge = g.near_edge(C[0], C[1])
    hits = []
    for (jx, jy) in g.cells(C[0] - r, C[0] + r, C[1] - r, C[1] + r):
        for t in (0, 1):
            a, b, c = g.tri(jx, jy, t)
            v = C - closest_on_triangle(C, a, b, c)
            d = np.linalg.norm(v)
            n = tri_normal(a, b, c) if inside or d <= 1e-9 else v / d
            # ranked by distance: the nearest point decides, above the surface (depth r - d) and under it (depth r + d) alike
            hits.append(dict(pair=g.pair(jx, jy, t), depth=r - d, n=n, d=d))
    best = _pick(hits)
    d = best["d"]
    depth = r + d if inside else r - d
    near = 0.0 if abs(side) < 1e-6 or on_edge else abs(depth)          # a centre on the surface: inside / outside is up to rounding
    if not depth > 0.0:
        return None, near
    return dict(pair=best["pair"], depth=depth, n=best["n"], pos=C - r * best["n"], alts=best["alts"], unpinned=inside and d > r, r=r, d=d), near


def segment_contact(g, A, B, r):
    """the interior of segment A-B swept by r against every cell edge under its bounding box: an edge counts when the segment point
    lies beyond it as seen from each of the cell's triangles on it (convex seen from above) and above the triangle's plane"""
    M = 0.5 * (A + B)
    if not g.on_map(M[0], M[1]):
        return None, 0.0 if g.near_edge(M[0], M[1]) else np.inf
    hits, near = [], 0.0 if g.near_edge(M[0], M[1]) else np.inf
    for (ix, iy) in g.cells(min(A[0], B[0]) - r, max(A[0], B[0]) + r, min(A[1], B[1]) - r, max(A[1], B[1]) + r):
        p00, p10, p01, p11 = g.v(ix, iy), g.v(ix + 1, iy), g.v(ix, iy + 1), g.v(ix + 1, iy + 1)
        n0, n1 = tri_normal(p00, p10, p11), tri_normal(p00, p11, p01)
        # edge, the third vertices of this cell's triangle(s) on it, the triangle whose pair index it carries
        for e0, e1, others, t in ((p00, p10, (p11,), 0), (p10, p11, (p00,), 0), (p00, p11, (p10, p01), 0), (p01, p11, (p00,), 1), (p00, p01, (p11,), 1)):
            s, u = closest_segments(A, B, e0, e1)
            if not (1e-3 < s < 1.0 - 1e-3):
                continue                                            # an end of the segment: the end sphere's business
            v = (A + s * (B - A)) - (e0 + u * (e1 - e0))
            dist = np.linalg.norm(v)
            ed = e1 - e0
            ms = [(o - e0) - np.dot(o - e0, ed) / np.dot(ed, ed) * ed for o in others]
            if not all(np.dot(v, m) < -1e-6 * dist * np.linalg.norm(m) for m in ms):
                continue
            nt = n0 if t == 0 else n1
            if not (np.dot(v, nt) > 0.0 and dist > 1e-9):
                continue
            near = min(near, abs(r - dist))
            if not dist < r:
                continue
            n = v / dist
            hits.append(dict(pair=g.pair(ix, iy, t), depth=r - dist, n=n, pos=(A + s * (B - A)) - r * n, d=dist))
    best = _pick(hits)
    if best is not None:
        best["unpinned"] = False
    return best, near


def box_contact(g, c, R, h):
    """terrain vertices under the box's bounding box that stand proud of their four neighbours and lie inside it, pushed out through
    the nearest face (lowest axis on a tie); the contact normal is the opposite of that face's outward normal"""
    if not g.on_map(c[0], c[1]):
        return None, 0.0 if g.near_edge(c[0], c[1]) else np.inf
    e = np.abs(R) @ h
    ix0 = max(math.floor((c[0] - e[0] - g.x0) / g.dx), 0); ix1 = min(math.floor((c[0] + e[0] - g.x0) / g.dx) + 1, g.xs - 1)
    iy0 = max(math.floor((c[1] - e[1] - g.y0) / g.dy), 0); iy1 = min(math.floor((c[1] + e[1] - g.y0) / g.dy) + 1, g.ys - 1)
    H = g.H
    hits, near = [], 0.0 if g.near_edge(c[0], c[1]) else np.inf
    for iy in range(iy0, iy1 + 1):
        for ix in range(ix0, ix1 + 1):
            hn = 0.25 * (H[iy, max(ix - 1, 0)] + H[iy, min(ix + 1, g.xs - 1)] + H[max(iy - 1, 0), ix] + H[min(iy + 1, g.ys - 1), ix])
            if not H[iy, ix] - hn > 1e-6:
                continue
            V = g.v(ix, iy)
            q = R.T @ (V - c)
            pen = h - np.abs(q)
            near = min(near, abs(pen.min()))
            if not (pen > 0.0).all():
                continue
            ax = int(np.argmin(pen))                                # first minimum: the lowest axis on a tie
            nf = np.zeros(3); nf[ax] = 1.0 if q[ax] >= 0.0 else -1.0
            hits.append(dict(pair=g.pair(min(ix, g.xs - 2), min(iy, g.ys - 2), 0), depth=pen[ax], n=-(R @ nf), pos=V))
    best = _pick(hits)
    if best is not None:
        best["unpinned"] = False
    return best, near


def candidate_contacts(t, R, p, g):
    """every candidate's contact (None: none) for body rotations R [nb, 3, 3] and positions p [nb, 3] of one environment, and the
    smallest |depth| of a feature that touches or nearly touches (a float32 pose may move it across zero)"""
    out, near = [], np.inf
    for k in range(t["npts"]):
        b = int(t["pt_body"][k])
        if b == 0 and not t["floating"]:
            out.append(None); continue
        P = p[b] + R[b] @ t["pt_pos"][k]
        rad, ty = float(t["pt_rad"][k]), int(t["pt_type"][k])
        if ty == 0:
            c, nr = sphere_contact(g, P, rad) if rad > 0.0 else point_contact(g, P)
        elif ty == 1:
            c, nr = segment_contact(g, P, p[b] + R[b] @ t["pt_pos2"][k], rad)
        elif ty == 2:
            ci = int(t["pt_coll"][k])
            c, nr = box_contact(g, p[b] + R[b] @ t["cpos"][ci], R[b] @ t["crot"][ci].reshape(3, 3), t["csize"][ci])
        else:                                                       # cylinder cap: the lowest point of its rim circle
            a = P - (p[b] + R[b] @ t["pt_pos2"][k]); a = a / np.linalg.norm(a)
            dd = np.array([a[2] * a[0], a[2] * a[1], a[2] * a[2] - 1.0])
            dn = np.linalg.norm(dd)
            c, nr = point_contact(g, P + rad / dn * dd) if dn > 1e-6 else (None, np.inf)
        near = min(near, nr)
        if c is not None:
            c.update(pt=k, body=b)
        out.append(c)
    return out, near


def rank(cands, kmax=KMAX):
    """the kmax deepest contacts (ties: lower candidate index), listed in candidate order, and whether the cut at kmax falls between
    two depths within TIE_TOL (then either may be kept)"""
    hits = sorted(sorted([c for c in cands if c is not None], key=lambda c: c["pt"]), key=lambda c: -c["depth"])
    cut_tie = len(hits) > kmax and hits[kmax - 1]["depth"] - hits[kmax]["depth"] < TIE_TOL
    return sorted(hits[:kmax], key=lambda c: c["pt"]), cut_tie


def env_contacts(t, gc, g):
    """(contact list, ambiguous): ambiguous = a feature within MARGIN of touching, or a near-tie at the kmax cut"""
    from helpers import fk_numpy, MARGIN
    R, p, _ = fk_numpy(t, np.asarray(gc, np.float64))
    cands, near = candidate_contacts(t, R, p, g)
    lst, cut_tie = rank(cands)
    return lst, bool(near < MARGIN or cut_tie)


def brute_force_distance(g, C, reach, m=40):
    """smallest distance from C to the surface over the cells within `reach` of it horizontally, every triangle sampled on a
    barycentric grid of m + 1 points per side: pins closest_on_triangle"""
    a, b = np.meshgrid(np.arange(m + 1) / m, np.arange(m + 1) / m)
    keep = a + b <= 1.0 + 1e-12
    a, b = a[keep], b[keep]
    best = np.inf
    for (ix, iy) in g.cells(C[0] - reach, C[0] + reach, C[1] - reach, C[1] + reach):
        for t in (0, 1):
            p0, p1, p2 = g.tri(ix, iy, t)
            pts = p0 + np.outer(a, p1 - p0) + np.outer(b, p2 - p0)
            best = min(best, np.linalg.norm(pts - C, axis=1).min())
    return best


def compare(ref, got, label=""):
    """ref: per environment (contact list, ambiguous) from env_contacts; got: (pts [n, K], cnt [n], pair [n, K], depth [n, K],
    normal [n, K, 3]) of the oracle or the kernel.  Outside the ambiguous environments the candidate lists must be identical, every
    pair index one the reference allows (alts), unpinned contacts deeper than r.  Returns the mismatching environments, the depth and
    normal errors of the compared contacts, and 1 / the distance each normal was divided by (0 for a face normal): a float32 pose
    moves a normal (centre - closest point) / distance by its rounding over that distance."""
    pts, cnt, pair, depth, normal = got
    bad, ed, en, w, skipped, total = [], [0.0], [0.0], [0.0], [], 0
    for e, (lst, amb) in enumerate(ref):
        if amb:
            skipped.append(e)
            continue
        k = int(cnt[e])
        total += len(lst)
        if k != len(lst) or [int(x) for x in pts[e, :k]] != [c["pt"] for c in lst]:
            bad.append(e)
            continue
        for j, c in enumerate(lst):
            if c["unpinned"]:
                if not depth[e, j] > c["r"]:
                    bad.append(e)
                continue
            ok = [a for a in c["alts"] if a[0] == int(pair[e, j])]
            if not ok:
                bad.append(e)
                continue
            ed.append(abs(float(depth[e, j]) - c["depth"]))
            en.append(min(float(np.abs(normal[e, j] - n).max()) for _, n in ok))
            w.append(1.0 / max(c["d"], 1e-4) if "d" in c else 0.0)
    print(f"[{label}] envs {len(ref)} (ambiguous {len(skipped)}), contacts {total}, mismatching envs {len(bad)}, "
          f"depth err {max(ed):.2e}, normal err {max(en):.2e}")
    return bad, np.array(ed), np.array(en), np.array(w)


# ---- test scenes shared by the CPU and GPU tests -------------------------------------------------------------------------------------

def single_shape_urdf(geometry, rpy="0 0 0"):
    return (f'<robot name="one"><link name="b"><inertial><origin xyz="0 0 0"/><mass value="2.0"/><inertia ixx="0.02" ixy="0" ixz="0" '
            f'iyy="0.02" iyz="0" izz="0.02"/></inertial>\n  <collision><origin xyz="0 0 0" rpy="{rpy}"/><geometry>{geometry}</geometry>'
            f'</collision></link></robot>')


def quat(axis, angle):
    a = np.asarray(axis, np.float64); a = a / np.linalg.norm(a)
    return np.r_[np.cos(angle / 2), np.sin(angle / 2) * a]


def qmul(p, q):
    return np.r_[p[0] * q[0] - p[1:] @ q[1:], p[0] * q[1:] + q[0] * p[1:] + np.cross(p[1:], q[1:])]


def centres(rng, g, n):
    """horizontal positions over the whole map with the places where cell arithmetic goes wrong mixed in: on cell boundaries in x and
    in y, on the P00-P11 diagonal of a cell, in the last row and column, and just outside every edge of the map"""
    X = rng.uniform(g.x0, g.x0 + (g.xs - 1) * g.dx, n); Y = rng.uniform(g.y0, g.y0 + (g.ys - 1) * g.dy, n)
    kind = np.arange(n) % 8
    ix = rng.integers(0, g.xs - 1, n); iy = rng.integers(0, g.ys - 1, n)
    f = rng.uniform(0, 1, n)
    X = np.where(kind == 1, g.x0 + ix * g.dx, X)                                      # on a vertical cell boundary
    Y = np.where(kind == 2, g.y0 + iy * g.dy, Y)                                      # on a horizontal one
    X = np.where(kind == 3, g.x0 + (ix + f) * g.dx, X); Y = np.where(kind == 3, g.y0 + (iy + f) * g.dy, Y)   # on the diagonal
    X = np.where(kind == 4, g.x0 + (g.xs - 2 + f) * g.dx, X)                          # last column
    Y = np.where(kind == 5, g.y0 + (g.ys - 2 + f) * g.dy, Y)                          # last row
    out = rng.uniform(1e-4, 0.3, n) * np.where(rng.uniform(0, 1, n) < 0.5, -1.0, 1.0)   # just outside: before the first or after the last
    side = rng.integers(0, 2, n)
    X = np.where((kind == 6) & (side == 0), np.where(out < 0, g.x0 + out * g.dx, g.x0 + (g.xs - 1 + out) * g.dx), X)
    Y = np.where((kind == 6) & (side == 1), np.where(out < 0, g.y0 + out * g.dy, g.y0 + (g.ys - 1 + out) * g.dy), Y)
    return X, Y


def drop_single_shape(rng, g, n, shape, size, lift):
    """poses gc [n, 7] (float32 values) of a single-shape body near the surface: shape sphere (size = r), capsule (r, half length),
    box (half extents); lift = (lo, hi) of the lowest point of the shape over the surface beneath its centre"""
    X, Y = centres(rng, g, n)
    gc = np.zeros((n, 7))
    for e in range(n):
        if shape == "sphere":
            q = quat(rng.standard_normal(3), rng.uniform(0, np.pi)); low = size[0]
        elif shape == "capsule":   # lying roughly flat: the side, not an end, meets the terrain
            q = qmul(quat([0, 0, 1], rng.uniform(-np.pi, np.pi)), quat([0, 1, 0], np.pi / 2 + rng.uniform(-0.25, 0.25)))
            low = size[0]
        else:                       # yaw anywhere (every fourth: exactly 45 degrees), slightly rolled and pitched
            yaw = np.pi / 4 if e % 4 == 0 else rng.uniform(-np.pi, np.pi)
            q = qmul(quat([0, 0, 1], yaw), qmul(quat([1, 0, 0], rng.uniform(-0.15, 0.15)), quat([0, 1, 0], rng.uniform(-0.15, 0.15))))
            low = size[2]
        gc[e, :3] = X[e], Y[e], g.height(X[e], Y[e]) + low + rng.uniform(*lift)
        gc[e, 3:] = q / np.linalg.norm(q)
    return gc.astype(np.float32).astype(np.float64)
