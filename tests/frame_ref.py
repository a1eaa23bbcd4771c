"""Numpy restatement of the batch's frame kinematics (rsb_batch_get_frame_states / rsb_batch_get_frame_jacobians) on helpers.fk_numpy:
world pose, velocity and point Jacobian of frames rigidly attached to bodies.  tests/test_frame_kinematics_cpu.py checks it against
central differences of fk_numpy; it is the reference of tests/test_gpu_frame_kinematics.py."""
import ctypes
import os
import xml.etree.ElementTree as ET

import numpy as np

from helpers import fk_numpy, quat_to_rot


def frame_kinematics(t, gc, gv, body, pos, rot=None, poses=None, dtype=np.float64):
    """One environment, F frames on bodies body[F] at pos [F, 3] with orientation rot [F, 3, 3] (None: identity) in the body frame ->
    (x [F, 3], Rf [F, 3, 3], lin [F, 3], ang [F, 3], J [F, 6, nv]): world position and orientation, velocity of the frame's point,
    angular velocity of its body, and J with [lin; ang] = J gv.  Revolute column (a x (x - p_j), a), prismatic (a, 0), floating base
    [I, -[x - p_0]x; 0, I], gv ordered as the batch's.
    poses = (R [nb, 3, 3], p [nb, 3]) replaces fk_numpy's; the world axes are then R_j axis_j (equal to fk_numpy's a_j for both joint
    types: the joint's rotation about its axis leaves the axis in place).  dtype is the arithmetic after the poses."""
    if poses is None:
        R, p, a = fk_numpy(t, gc)
    else:
        R, p = (np.asarray(x, np.float64) for x in poses)
        a = np.einsum("bij,bj->bi", R, np.asarray(t["axis"], np.float64).reshape(-1, 3))
    R, p, a = R.astype(dtype), p.astype(dtype), a.astype(dtype)
    pos = np.asarray(pos, np.float64).reshape(-1, 3).astype(dtype)
    F, nv = len(pos), t["nv"]
    rot = np.tile(np.eye(3), (F, 1, 1)).astype(dtype) if rot is None else np.asarray(rot, np.float64).reshape(F, 3, 3).astype(dtype)
    eye = np.eye(3, dtype=dtype)
    x, Rf, J = np.zeros((F, 3), dtype), np.zeros((F, 3, 3), dtype), np.zeros((F, 6, nv), dtype)
    for f, b in enumerate(body):
        x[f] = p[b] + R[b] @ pos[f]
        Rf[f] = R[b] @ rot[f]
        if t["floating"]:
            J[f, 0:3, 0:3] = eye
            J[f, 0:3, 3:6] = np.cross(eye, x[f] - p[0]).T      # column i: e_i x (x - p_0) = -[x - p_0]x e_i
            J[f, 3:6, 3:6] = eye
        j = b
        while t["parent"][j] >= 0:
            c = t["vidx"][j]
            if t["jtype"][j] == 1:
                J[f, 0:3, c] = np.cross(a[j], x[f] - p[j])
                J[f, 3:6, c] = a[j]
            else:
                J[f, 0:3, c] = a[j]
            j = t["parent"][j]
    vel = J @ np.asarray(gv, np.float64).astype(dtype)
    return x, Rf, vel[:, 0:3], vel[:, 3:6], J


def batch_frame_kinematics(t, gc, gv, body, pos, rot=None, poses=None, dtype=np.float64):
    """frame_kinematics of every environment: gc [n, nq], gv [n, nv], poses = (R [n, nb, 3, 3], p [n, nb, 3]) or None"""
    out = [frame_kinematics(t, gc[e], gv[e], body, pos, rot, None if poses is None else (poses[0][e], poses[1][e]), dtype) for e in range(len(gc))]
    return tuple(np.stack(k) for k in zip(*out))


def link_names(urdf):
    """link names of a URDF file or XML text: the model's frames"""
    root = ET.parse(urdf).getroot() if os.path.exists(urdf) else ET.fromstring(urdf)
    return [ln.get("name") for ln in root.findall("link")]


def model_frames(capi, model, names):
    """(body [F], pos [F, 3], rot [F, 3, 3]) of the named frames as rsb_model_frame gives them"""
    L = capi.lib()
    body, pos, rot = [], np.zeros((len(names), 3)), np.zeros((len(names), 9))
    for k, name in enumerate(names):
        f, b = L.rsb_model_frame_index(model.h, name.encode()), ctypes.c_int()
        assert f >= 0 and L.rsb_model_frame(model.h, f, ctypes.byref(b), pos[k].ctypes.data_as(ctypes.c_void_p), rot[k].ctypes.data_as(ctypes.c_void_p)) == 0
        body.append(b.value)
    return np.array(body, np.int32), pos, rot.reshape(-1, 3, 3)


def random_frames(rng, nb, count):
    """`count` frames on random bodies at random points (within 0.3 m of the body origin) with random orientations, float32 values"""
    body = rng.integers(0, nb, count).astype(np.int32)
    pos = rng.uniform(-0.3, 0.3, (count, 3)).astype(np.float32)
    rot = np.stack([quat_to_rot(q) for q in rng.standard_normal((count, 4))]).astype(np.float32)
    return body, pos, rot
