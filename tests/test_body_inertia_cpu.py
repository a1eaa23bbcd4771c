"""Per-environment inertial parameters pinned on the CPU before the GPU tests rely on them: the payload composition of
tests/body_inertia_ref.py against the URDF loaders' own merge of a link on a fixed joint, and the float64 oracle built from modified
tables against known answers for every parameter set."""
import os

import numpy as np
import pytest

from body_inertia_ref import add_payload, randomized, sym, tables_with
from conftest import RSC
from helpers import SPHERE_URDF
from oracle.oracle import Oracle
from oracle.urdf_tables import load_tables, rpy_to_rot
from raisimlib_b200 import capi

G, DT = 9.81, 0.0025

BASE = ("<link name='base'><inertial><origin xyz='0.01 -0.02 0.03' rpy='0.1 0.2 0.3'/><mass value='7.5'/>"
        "<inertia ixx='0.10' ixy='0.004' ixz='-0.002' iyy='0.20' iyz='0.003' izz='0.25'/></inertial></link>")
PAYLOAD = ("<link name='payload'><inertial><origin xyz='{cx} {cy} {cz}' rpy='{cr} {cp} {cyaw}'/><mass value='{m}'/>"
           "<inertia ixx='{ixx}' ixy='0' ixz='0' iyy='{iyy}' iyz='0' izz='{izz}'/></inertial></link>"
           "<joint name='mount' type='fixed'><parent link='base'/><child link='payload'/><origin xyz='{jx} {jy} {jz}' rpy='{jr} {jp} {jyaw}'/></joint>")


@pytest.mark.parametrize("seed", range(4))
def test_payload_composition_equals_the_loaders_merge_of_a_fixed_link(seed):
    """a payload (mass, centre of mass, inertia in a turned frame) mounted on a base link through a fixed joint: both loaders merge
    the two links into one body, and add_payload on the base alone gives the same mass, centre of mass and inertia"""
    rng = np.random.default_rng(seed)
    p = dict(m=rng.uniform(0.5, 10.0), cx=rng.uniform(-0.1, 0.1), cy=rng.uniform(-0.1, 0.1), cz=rng.uniform(-0.1, 0.1),
             cr=rng.uniform(-1, 1), cp=rng.uniform(-1, 1), cyaw=rng.uniform(-1, 1), ixx=rng.uniform(0.01, 0.1), iyy=rng.uniform(0.01, 0.1),
             izz=rng.uniform(0.01, 0.1), jx=rng.uniform(-0.3, 0.3), jy=rng.uniform(-0.3, 0.3), jz=rng.uniform(-0.3, 0.3),
             jr=rng.uniform(-1, 1), jp=rng.uniform(-1, 1), jyaw=rng.uniform(-1, 1))
    alone = load_tables(f"<robot name='r'>{BASE}</robot>")
    merged_urdf = f"<robot name='r'>{BASE}{PAYLOAD.format(**p)}</robot>"
    Rj = rpy_to_rot([p["jr"], p["jp"], p["jyaw"]])
    pos = np.array([p["jx"], p["jy"], p["jz"]]) + Rj @ np.array([p["cx"], p["cy"], p["cz"]])
    m, c, I = add_payload(alone["mass"][0], alone["com"][0], alone["inertia"][0], p["m"], pos, (p["ixx"], 0, 0, p["iyy"], 0, p["izz"]),
                          Rj @ rpy_to_rot([p["cr"], p["cp"], p["cyaw"]]))
    for merged in (load_tables(merged_urdf), capi.Model(merged_urdf).tables()):
        assert merged["nb"] == 1
        assert abs(merged["mass"][0] - m) < 1e-12
        assert np.abs(merged["com"][0] - c).max() < 1e-12
        assert np.abs(merged["inertia"][0] - I).max() < 1e-12


def test_randomized_parameters_stay_physical(anymal_tables):
    t = anymal_tables
    rng = np.random.default_rng(3)
    for _ in range(16):
        mass, com, inertia = randomized(t, rng)
        assert (mass >= 0.7 * t["mass"] * (1 - 1e-6)).all() and (mass <= 1.3 * t["mass"] * (1 + 1e-6)).all()
        assert np.abs(com - t["com"]).max() <= 0.02 + 1e-6
        for b in range(t["nb"]):
            w = np.linalg.eigvalsh(sym(inertia[b]))
            w0 = np.linalg.eigvalsh(sym(t["inertia"][b]))
            assert w.min() > 0
            assert 0.7 * w0.sum() * (1 - 1e-5) <= w.sum() <= 1.3 * w0.sum() * (1 + 1e-5)


@pytest.mark.parametrize("m", [0.3, 2.0, 17.0])
def test_resting_sphere_carries_its_own_weight(m):
    """normal impulse of a sphere resting on the plane: m g dt, whatever its mass"""
    t = load_tables(SPHERE_URDF)
    u = tables_with(t, [m], t["com"], t["inertia"] * m / t["mass"][0])
    o = Oracle(u); o.set_ground(0.0)
    gc = np.array([[0, 0, 0.0999, 1, 0, 0, 0.0]]); gv = np.zeros((1, 6))
    d = o.step(gc, gv, debug=True)
    assert d["ncontacts"][0] == 1
    assert abs(d["c_lambda"][0, 0, 2] - m * G * DT) < 1e-9 * m * G * DT


def test_free_fall_does_not_depend_on_the_inertial_parameters(anymal_tables):
    """a robot in the air with its joints still falls as a rigid body at g for every parameter set"""
    t = anymal_tables
    rng = np.random.default_rng(7)
    gc0 = np.zeros(t["nq"]); gc0[2] = 3.0; gc0[3] = 1.0
    gc0[7:] = rng.uniform(-0.3, 0.3, t["nq"] - 7)
    ends = []
    for _ in range(4):
        mass, com, inertia = randomized(t, rng)
        o = Oracle(tables_with(t, mass, com, inertia))
        gc, gv = gc0[None].copy(), np.zeros((1, t["nv"]))
        o.step(gc, gv, n_steps=40)
        ends.append(gc[0])
        assert np.abs(gv[0, 2] + 40 * G * DT) < 1e-9
        assert np.abs(gv[0, 6:]).max() < 1e-9 and np.abs(gv[0, :2]).max() < 1e-9 and np.abs(gv[0, 3:6]).max() < 1e-9
    for e in ends[1:]:
        assert np.abs(e - ends[0]).max() < 1e-9
