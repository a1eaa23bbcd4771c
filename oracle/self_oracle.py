"""ORACLE python wrapper of the self-collision restatement (ctypes over oracle/liboracle_self.so) -- test infrastructure, NOT
product.  SelfOracle is oracle.Oracle on the library whose Sim also collides enabled pairs of the robot's own collision bodies
(self_collision.hpp); without pairs it computes exactly what Oracle computes.  The same import rules as oracle.oracle hold."""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle import oracle as _o

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "liboracle_self.so")
_SOURCES = ("self_collision_capi.cpp", "self_collision.hpp", "oracle_capi.cpp", "rbd_oracle.hpp", "counting_scalar.hpp")
# the parity build's flags (oracle/Makefile): no FMA contraction, portable ISA, so that the float32 instance evaluates the
# narrow-phase predicates exactly as written
_CXXFLAGS = ["-O3", "-march=x86-64-v3", "-ffp-contract=off", "-fopenmp", "-fPIC", "-std=c++17", "-Wall", "-Wno-unused-variable"]


def build(force=False):
    if force or not os.path.exists(_LIB_PATH) or any(os.path.getmtime(os.path.join(_HERE, f)) > os.path.getmtime(_LIB_PATH) for f in _SOURCES):
        subprocess.check_call(["/usr/bin/g++", *_CXXFLAGS, "-shared", "-o", _LIB_PATH, os.path.join(_HERE, "self_collision_capi.cpp")])
    return _LIB_PATH


def lib():
    if "self" not in _o._libs:
        build()
        L = _o._declare(C.CDLL(_LIB_PATH))
        L.orc_set_self_pairs.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
        L.orc_self_pair_geometry.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 5
        L.orc_self_contact_jacobians.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 4
        _o._libs["self"] = L
    return _o._libs["self"]


class SelfOracle(_o.Oracle):
    """oracle.Oracle with self-collision between enabled pairs of collision bodies"""

    def __init__(self, tables, precision="f64", params=None):
        lib()
        super().__init__(tables, precision=precision, params=params, build="self")

    def set_self_collision(self, pairs, mu=None):
        """enable self-collision between pairs of collision bodies ([n][2] collision-body indices; mu [n] or None = default
        material; an empty list clears them).  Contacts of pair j have candidate index npts + j and pair index -1 - second body."""
        idesc, geo = self_pair_tables(self.t, pairs, mu)
        self.L.orc_set_self_pairs(self.h, len(idesc), idesc.ctypes.data, geo.ctypes.data)

    def self_pair_geometry(self, j, RA, pA, RB, pB):
        """narrow phase of enabled pair j alone, its bodies A, B (the sphere's body first for a sphere-box pair) at the given poses:
        None when the shapes do not overlap, else (depth, normal from the second body to the first, position)"""
        f = lambda a: np.ascontiguousarray(a, np.float64).reshape(-1)
        out = np.zeros(7)
        hit = self.L.orc_self_pair_geometry(self.h, int(j), _o._p(f(RA)), _o._p(f(pA)), _o._p(f(RB)), _o._p(f(pB)), _o._p(out))
        return (out[0], out[1:4], out[4:7]) if hit else None

    def contact_jacobians(self, gc):
        """contact lists of the states gc [n, nq] and their contact Jacobians: (ncontacts [n], candidate ids [n, KMAX],
        Jt [n, nv, 3 KMAX] with column 3 k + (t1, t2, n) of contact k)"""
        gc = np.ascontiguousarray(gc, np.float64)
        n = gc.shape[0]
        cnt, pts, Jt = np.zeros(n, np.int32), np.zeros((n, self.kmax), np.int32), np.zeros((n, self.nv, 3 * self.kmax))
        self.L.orc_self_contact_jacobians(self.h, n, _o._p(gc), cnt.ctypes.data, pts.ctypes.data, _o._p(Jt))
        return cnt, pts, Jt


_SPHERE, _BOX, _CAPSULE, _CYLINDER = 0, 1, 2, 3
_SHAPE_NAMES = {_SPHERE: "sphere", _BOX: "box", _CAPSULE: "capsule", _CYLINDER: "cylinder"}


def self_pair_tables(t, pairs, mu=None):
    """self-collision pairs of collision bodies -> the oracle's pair description (self_collision.hpp SelfPair): idesc [n][6] int32 =
    kind, flip, first body, second body, body A, body B; geo [n][24] = a0, a1, b0, b1, box rotation (9), rA, rB, mu.  Spheres and
    capsules are segments swept by their radius (a sphere: a segment of length 0); a sphere-box pair puts the sphere in A."""
    pairs = np.asarray(pairs, np.int64).reshape(-1, 2)
    mu = np.full(len(pairs), -1.0) if mu is None else np.asarray(mu, np.float64).reshape(-1)
    idesc, geo = np.zeros((len(pairs), 6), np.int32), np.zeros((len(pairs), 24))

    def seg(c):
        p, R, s = t["cpos"][c], t["crot"][c].reshape(3, 3), t["csize"][c]
        if t["ctype"][c] == _SPHERE:
            return p, p, s[0]
        return p - s[1] * R[:, 2], p + s[1] * R[:, 2], s[0]

    for j, (c1, c2) in enumerate(pairs):
        if not (0 <= c1 < t["ncoll"] and 0 <= c2 < t["ncoll"]):
            raise ValueError(f"pair {j}: collision body index out of range")
        ty1, ty2 = int(t["ctype"][c1]), int(t["ctype"][c2])
        b1, b2 = int(t["cbody"][c1]), int(t["cbody"][c2])
        if b1 == b2:
            raise ValueError(f"pair {j}: both collision bodies are on body {b1}")
        if ty1 in (_SPHERE, _CAPSULE) and ty2 in (_SPHERE, _CAPSULE):
            (a0, a1, ra), (g0, g1, rb) = seg(c1), seg(c2)
            idesc[j] = (0, 0, b1, b2, b1, b2)
            geo[j, 0:3], geo[j, 3:6], geo[j, 6:9], geo[j, 9:12], geo[j, 21], geo[j, 22] = a0, a1, g0, g1, ra, rb
            geo[j, 12:21] = np.eye(3).reshape(9)
        elif sorted((ty1, ty2)) == [_SPHERE, _BOX]:
            flip = ty1 == _BOX
            cs, cb = (c2, c1) if flip else (c1, c2)
            idesc[j] = (1, int(flip), b1, b2, int(t["cbody"][cs]), int(t["cbody"][cb]))
            geo[j, 0:3] = geo[j, 3:6] = t["cpos"][cs]
            geo[j, 6:9], geo[j, 9:12], geo[j, 12:21] = t["cpos"][cb], t["csize"][cb], t["crot"][cb].reshape(9)
            geo[j, 21] = t["csize"][cs][0]
        else:
            raise ValueError(f"pair {j}: {_SHAPE_NAMES[ty1]}-{_SHAPE_NAMES[ty2]} self-collision is not supported")
        geo[j, 23] = mu[j]
    return idesc, geo
