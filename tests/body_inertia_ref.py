"""Inertial parameters of a body that carries a rigid payload, and the per-environment rows of rsb_batch_set_body_inertia built from
them.  The payload composition is what a URDF loader does when it merges a link on a fixed joint into its parent: masses add, the
centre of mass is the mass-weighted mean, and both inertias are rotated into the body frame and moved to the new centre of mass by
the parallel-axis theorem.  Rows and inertias use the order of rsb_model_tables: mass, com (3), inertia xx xy xz yy yz zz."""
import numpy as np


def sym(i6):
    xx, xy, xz, yy, yz, zz = i6
    return np.array([[xx, xy, xz], [xy, yy, yz], [xz, yz, zz]], dtype=np.float64)


def unsym(I):
    return np.array([I[0, 0], I[0, 1], I[0, 2], I[1, 1], I[1, 2], I[2, 2]])


def shift(I, m, d):
    """inertia about a point at offset d from the centre of mass of a body of mass m whose inertia about that centre is I"""
    d = np.asarray(d, np.float64)
    return I + m * (d @ d * np.eye(3) - np.outer(d, d))


def add_payload(mass, com, inertia6, pm, ppos, pinertia6=(0, 0, 0, 0, 0, 0), prot=np.eye(3)):
    """(mass, com, inertia6) of a body plus a payload of mass pm whose centre of mass sits at ppos (body frame) and whose inertia
    about that centre is pinertia6 in a frame rotated by prot against the body frame"""
    m = mass + pm
    c = (mass * np.asarray(com, np.float64) + pm * np.asarray(ppos, np.float64)) / m
    Ip = prot @ sym(pinertia6) @ prot.T
    I = shift(sym(inertia6), mass, np.asarray(com) - c) + shift(Ip, pm, np.asarray(ppos) - c)
    return m, c, unsym(I)


def tables_with(t, mass, com, inertia):
    """a copy of the tables dict t with other inertial parameters (for oracle.Oracle)"""
    u = dict(t)
    u["mass"], u["com"], u["inertia"] = np.asarray(mass, np.float64).copy(), np.asarray(com, np.float64).copy(), np.asarray(inertia, np.float64).copy()
    return u


def rows_of(mass, com, inertia):
    """[nb, 10] float32 row block of rsb_batch_set_body_inertia"""
    return np.concatenate([np.asarray(mass)[:, None], com, inertia], axis=1).astype(np.float32)


def random_rotation(rng):
    q = rng.standard_normal(4)
    w, x, y, z = q / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def randomized(t, rng):
    """one parameter set of the GPU parity tests: every mass x U(0.7, 1.3), every centre of mass moved by up to 2 cm per axis, every
    inertia rescaled by U(0.7, 1.3) and turned by a random rotation (stays symmetric positive definite).  Returns (mass, com, inertia)
    rounded to float32, so that the oracle and the batch integrate the same numbers."""
    nb = t["nb"]
    mass = t["mass"] * rng.uniform(0.7, 1.3, nb)
    com = t["com"] + rng.uniform(-0.02, 0.02, (nb, 3))
    inertia = np.empty((nb, 6))
    for b in range(nb):
        R = random_rotation(rng)
        inertia[b] = unsym(rng.uniform(0.7, 1.3) * (R @ sym(t["inertia"][b]) @ R.T))
    r = rows_of(mass, com, inertia).astype(np.float64)
    return r[:, 0], r[:, 1:4], r[:, 4:10]
