"""Shared test helpers: independent numpy restatements used to pin the oracle (SURVEY.md 4(3)), the test models, and the
batch / oracle set-up the GPU parity tests share."""
import os
import xml.etree.ElementTree as ET

import numpy as np

MARGIN = 2e-6          # metres; contact candidates shallower than this are excluded from index parity
THRESH = 1e-6          # solver threshold used on both sides

ANYMAL_GC0 = np.array([0, 0, 0.60, 1, 0, 0, 0, 0.03, 0.4, -0.8, -0.03, 0.4, -0.8, 0.03, -0.4, 0.8, -0.03, -0.4, 0.8], dtype=np.float64)

PENDULUM_URDF = """<robot name="pend">
  <link name="world"/>
  <link name="l1"><inertial><origin xyz="0 0 -0.5"/><mass value="2.0"/><inertia ixx="0.1" ixy="0" ixz="0" iyy="0.1" iyz="0" izz="0.01"/></inertial></link>
  <joint name="j1" type="revolute"><parent link="world"/><child link="l1"/><origin xyz="0 0 1.0"/><axis xyz="0 1 0"/></joint>
  <link name="l2"><inertial><origin xyz="0 0 -0.3"/><mass value="1.0"/><inertia ixx="0.03" ixy="0" ixz="0" iyy="0.03" iyz="0" izz="0.005"/></inertial></link>
  <joint name="j2" type="revolute"><parent link="l1"/><child link="l2"/><origin xyz="0 0.1 -1.0"/><axis xyz="0 1 0"/></joint>
  <link name="l3"><inertial><origin xyz="0.1 0 0"/><mass value="0.5"/><inertia ixx="0.01" ixy="0.001" ixz="0" iyy="0.02" iyz="0" izz="0.02"/></inertial></link>
  <joint name="j3" type="prismatic"><parent link="l2"/><child link="l3"/><origin xyz="0 0 -0.6" rpy="0.3 0.2 0.1"/><axis xyz="1 0 0"/></joint>
</robot>"""

SPHERE_URDF = """<robot name="ball">
  <link name="ball"><inertial><origin xyz="0 0 0"/><mass value="2.0"/><inertia ixx="0.008" ixy="0" ixz="0" iyy="0.008" iyz="0" izz="0.008"/></inertial>
  <collision><origin xyz="0 0 0"/><geometry><sphere radius="0.1"/></geometry></collision></link>
</robot>"""

BOX_URDF = """<robot name="box">
  <link name="box"><inertial><origin xyz="0 0 0"/><mass value="3.0"/><inertia ixx="0.02" ixy="0" ixz="0" iyy="0.03" iyz="0" izz="0.04"/></inertial>
  <collision><origin xyz="0 0 0"/><geometry><box size="0.4 0.3 0.2"/></geometry></collision></link>
</robot>"""


def quat_to_rot(q):
    w, x, y, z = q / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def axis_angle(a, q):
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(q) * K + (1 - np.cos(q)) * K @ K


def skew(v):
    return np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]])


def fk_numpy(t, gc):
    """Independent FK: returns R[nb,3,3], p[nb,3], world joint axes a[nb,3]."""
    nb = t["nb"]
    R, p, a = np.zeros((nb, 3, 3)), np.zeros((nb, 3)), np.zeros((nb, 3))
    for i in range(nb):
        pr = t["parent"][i]
        if pr < 0:
            if t["floating"]:
                R[i], p[i] = quat_to_rot(gc[3:7]), gc[0:3]
            else:
                R[i], p[i] = t["jrot"][i].reshape(3, 3), t["jpos"][i]
            continue
        Rj = R[pr] @ t["jrot"][i].reshape(3, 3)
        a[i] = Rj @ t["axis"][i]
        p[i] = p[pr] + R[pr] @ t["jpos"][i]
        q = gc[t["qidx"][i]]
        if t["jtype"][i] == 1:
            R[i] = Rj @ axis_angle(t["axis"][i], q)
        else:
            R[i] = Rj
            p[i] = p[i] + q * a[i]
    return R, p, a


def body_jacobians(t, gc):
    """Per body: Jv (COM linear velocity) and Jw (angular velocity), each [3,nv]; the textbook
    M = sum_b m Jv^T Jv + Jw^T (R I R^T) Jw identity, independent of the oracle's CRBA."""
    R, p, a = fk_numpy(t, gc)
    nb, nv = t["nb"], t["nv"]
    out = []
    for b in range(nb):
        c = p[b] + R[b] @ t["com"][b]
        Jv, Jw = np.zeros((3, nv)), np.zeros((3, nv))
        if t["floating"]:
            Jv[:, 0:3] = np.eye(3)
            Jv[:, 3:6] = -skew(c - p[0])
            Jw[:, 3:6] = np.eye(3)
        j = b
        while t["parent"][j] >= 0:
            vi = t["vidx"][j]
            if t["jtype"][j] == 1:
                Jv[:, vi] = np.cross(a[j], c - p[j])
                Jw[:, vi] = a[j]
            else:
                Jv[:, vi] = a[j]
            j = t["parent"][j]
        out.append((Jv, Jw, R[b], c))
    return out


def mass_matrix_numpy(t, gc):
    M = np.zeros((t["nv"], t["nv"]))
    for b, (Jv, Jw, Rb, c) in enumerate(body_jacobians(t, gc)):
        I6 = t["inertia"][b]
        I = np.array([[I6[0], I6[1], I6[2]], [I6[1], I6[3], I6[4]], [I6[2], I6[4], I6[5]]])
        M += t["mass"][b] * Jv.T @ Jv + Jw.T @ (Rb @ I @ Rb.T) @ Jw
    return M


def potential_energy(t, gc, g=9.81):
    R, p, _ = fk_numpy(t, gc)
    return sum(t["mass"][b] * g * (p[b] + R[b] @ t["com"][b])[2] for b in range(t["nb"]))


def integrate_gc(t, gc, dv, eps):
    """gc (+) eps*dv with the oracle's conventions (world-frame base angular velocity)."""
    out = gc.copy()
    if t["floating"]:
        out[0:3] += eps * dv[0:3]
        w = dv[3:6] * eps
        ang = np.linalg.norm(w)
        if ang > 0:
            dq = np.r_[np.cos(ang / 2), np.sin(ang / 2) * w / ang]
        else:
            dq = np.array([1.0, 0, 0, 0])
        q = gc[3:7]
        out[3:7] = np.array([dq[0] * q[0] - dq[1:] @ q[1:], *(dq[0] * q[1:] + q[0] * dq[1:] + np.cross(dq[1:], q[1:]))])
    for i in range(1, t["nb"]):
        out[t["qidx"][i]] += eps * dv[t["vidx"][i]]
    return out


def random_state(t, rng, n, pos_scale=0.0, vel_scale=1.0, joint_scale=0.5, base_z=0.6):
    gc = np.zeros((n, t["nq"])); gv = vel_scale * rng.standard_normal((n, t["nv"]))
    if t["floating"]:
        gc[:, 0:2] = pos_scale * rng.uniform(-1, 1, (n, 2))
        gc[:, 2] = base_z
        q = rng.standard_normal((n, 4)); q /= np.linalg.norm(q, axis=1, keepdims=True)
        gc[:, 3:7] = q
        gc[:, 7:] = joint_scale * rng.uniform(-1, 1, (n, t["nq"] - 7))
    else:
        gc[:] = joint_scale * rng.uniform(-1, 1, (n, t["nq"]))
    return gc, gv

# a link set as real robot descriptions have it: visuals, meshes, cylinders, gazebo / transmission tags
REALISTIC_URDF = """<?xml version="1.0" ?>
<!-- generated by xacro -->
<robot name="mini" xmlns:xacro="http://www.ros.org/wiki/xacro">
  <material name="grey"><color rgba="0.5 0.5 0.5 1"/></material>
  <link name="trunk">
    <visual><origin xyz="0 0 0" rpy="0 0 0"/><geometry><mesh filename="package://x/meshes/trunk.dae" scale="1 1 1"/></geometry><material name="grey"/></visual>
    <collision><geometry><box size="0.4 0.2 0.1"/></geometry></collision>
    <collision><geometry><mesh filename="package://x/meshes/trunk_col.stl"/></geometry></collision>
    <inertial><origin xyz="0.01 0 0"/><mass value="5"/><inertia ixx="0.02" ixy="0" ixz="0" iyy="0.06" iyz="0" izz="0.07"/></inertial>
  </link>
  <link name="imu_link"/>
  <joint name="imu_joint" type="fixed"><parent link="trunk"/><child link="imu_link"/><origin rpy="0 0 0" xyz="0 0 0.05"/></joint>
  <link name="leg">
    <visual><geometry><cylinder length="0.3" radius="0.02"/></geometry></visual>
    <collision><origin xyz="0 0 -0.15" rpy="0 0 0"/><geometry><cylinder length="0.3" radius="0.025"/></geometry></collision>
    <inertial><origin xyz="0 0 -0.15"/><mass value="0.8"/><inertia ixx="0.006" ixy="0" ixz="0" iyy="0.006" iyz="0" izz="0.0003"/></inertial>
  </link>
  <joint name="hip" type="continuous"><parent link="trunk"/><child link="leg"/><origin xyz="0.15 0.1 0"/><axis xyz="0 1 0"/>
    <dynamics damping="0.0" friction="0.0"/><limit effort="30" velocity="20"/></joint>
  <transmission name="t"><type>transmission_interface/SimpleTransmission</type><joint name="hip"><hardwareInterface>hardware_interface/EffortJointInterface</hardwareInterface></joint></transmission>
  <gazebo reference="leg"><mu1>0.8</mu1><self_collide>1</self_collide></gazebo>
</robot>"""


# ---------------------------------------------------------------------------------------------------------------------------------
# Test models for the compiled instances of the step kernel (batch.cu dispatch_spec): which instance a model takes depends on its
# dimensions (nb, nq, nv, floating base, tree depth, dof-tree depth), its parent table, and whether it has more than 32 contact
# candidates (two candidate slots per lane).  Each model below is built to reach one instance, or one bound of the loader.

_RSC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "raisimlib_b200", "rsc")


def _anymal_tree():
    return ET.parse(os.path.join(_RSC, "anymal_c_like.urdf")).getroot()


def _anymal_variant(feet_only=False, prismatic_knees=False):
    root = _anymal_tree()
    if feet_only:                       # the ANYmal-like tree with the four foot spheres as its only collision bodies
        for link in root.findall("link"):
            if not link.get("name").endswith("_FOOT"):
                for c in link.findall("collision"):
                    link.remove(c)
    if prismatic_knees:                 # KFE joints slide along the shank instead of turning: jtype 2 inside the compiled chains
        for j in root.findall("joint"):
            if j.get("name").endswith("_KFE"):
                j.set("type", "prismatic")
                j.find("axis").set("xyz", "0 0 1")
                lim = j.find("limit")
                lim.set("lower", "-0.12"); lim.set("upper", "0.12"); lim.set("effort", "300")
    return ET.tostring(root, encoding="unicode")


def _urdf(name, links, joints):
    """links: (name, mass, com, (ixx, iyy, izz), [collision geometry xml, xyz, rpy]); joints: (name, type, parent, child, xyz, rpy,
    axis, (lower, upper, effort) or None)"""
    s = f'<robot name="{name}">\n'
    for ln, m, com, I, colls in links:
        s += (f'  <link name="{ln}"><inertial><origin xyz="{com[0]} {com[1]} {com[2]}"/><mass value="{m}"/>'
              f'<inertia ixx="{I[0]}" ixy="0" ixz="0" iyy="{I[1]}" iyz="0" izz="{I[2]}"/></inertial>\n')
        for g, xyz, rpy in colls:
            s += f'    <collision><origin xyz="{xyz[0]} {xyz[1]} {xyz[2]}" rpy="{rpy[0]} {rpy[1]} {rpy[2]}"/><geometry>{g}</geometry></collision>\n'
        s += '  </link>\n'
    for jn, jt, par, ch, xyz, rpy, ax, lim in joints:
        s += (f'  <joint name="{jn}" type="{jt}"><parent link="{par}"/><child link="{ch}"/>'
              f'<origin xyz="{xyz[0]} {xyz[1]} {xyz[2]}" rpy="{rpy[0]} {rpy[1]} {rpy[2]}"/><axis xyz="{ax[0]} {ax[1]} {ax[2]}"/>')
        if lim is not None:
            s += f'<limit lower="{lim[0]}" upper="{lim[1]}" effort="{lim[2]}" velocity="10"/>'
        s += '</joint>\n'
    return s + '</robot>\n'


_Z3 = (0, 0, 0)


def _quad_branched():
    """The quadruped's dimensions (nb 13, nq 19, nv 18, floating, depth 3, dof depth 8) in a different tree: the left front hip
    carries two children and the right hind leg has no shank, so the compiled 4 x 3-chain arithmetic does not apply."""
    links = [("base", 25.0, (0, 0, 0.02), (0.22, 0.86, 0.93), [('<box size="0.58 0.28 0.18"/>', _Z3, _Z3)])]
    joints = []
    for leg, fx, fy, kids in (("LF", 1, 1, 3), ("RF", 1, -1, 2), ("LH", -1, 1, 2), ("RH", -1, -1, 1)):
        links.append((f"{leg}_HIP", 2.0, (fx * 0.05, 0, 0), (0.0034, 0.0041, 0.004), []))
        joints.append((f"{leg}_HAA", "revolute", "base", f"{leg}_HIP", (fx * 0.3, fy * 0.1, 0), _Z3, (1, 0, 0), (-0.72, 0.49, 80)))
        links.append((f"{leg}_THIGH", 3.0, (0, fy * 0.04, -0.12), (0.024, 0.023, 0.0045), []))
        joints.append((f"{leg}_HFE", "revolute", f"{leg}_HIP", f"{leg}_THIGH", (fx * 0.06, fy * 0.08, 0), _Z3, (0, 1, 0), (-3, 3, 80)))
        if kids >= 2:
            links.append((f"{leg}_SHANK", 0.85, (0, 0, -0.15), (0.006, 0.006, 0.0005), [('<sphere radius="0.03"/>', (0, 0, -0.3), _Z3)]))
            joints.append((f"{leg}_KFE", "revolute", f"{leg}_THIGH", f"{leg}_SHANK", (0, fy * 0.1, -0.285), _Z3, (0, 1, 0), (-3, 3, 80)))
        if kids >= 3:           # second child of the hip
            links.append((f"{leg}_ARM", 0.5, (0.05, 0, 0), (0.001, 0.002, 0.002), [('<sphere radius="0.04"/>', (0.1, 0, 0), _Z3)]))
            joints.append((f"{leg}_ARM_J", "revolute", f"{leg}_HIP", f"{leg}_ARM", (0.05, 0, 0.05), _Z3, (0, 0, 1), (-1, 1, 40)))
    return _urdf("quad_branched", links, joints)


def _hexapod():
    """Floating base and six 3-joint legs: nb 19 (more than 16 bodies), exactly 32 contact candidates (one slot per lane)."""
    links = [("base", 10.0, (0, 0, 0), (0.09, 0.3, 0.37), [('<box size="0.6 0.3 0.12"/>', _Z3, _Z3)])]     # 8 corners + 1 face
    joints = []
    for i, (x, s) in enumerate(((0.25, 1), (0.0, 1), (-0.25, 1), (0.25, -1), (0.0, -1), (-0.25, -1))):
        links.append((f"coxa{i}", 0.5, (0, s * 0.03, 0), (0.0005, 0.0004, 0.0005),
                      [('<sphere radius="0.04"/>', (0, s * 0.03, 0), _Z3)] if i < 5 else []))
        joints.append((f"yaw{i}", "revolute", "base", f"coxa{i}", (x, s * 0.15, 0), _Z3, (0, 0, 1), (-0.6, 0.6, 40)))
        links.append((f"femur{i}", 0.8, (0, s * 0.08, 0), (0.002, 0.0004, 0.002),
                      [('<capsule radius="0.03" length="0.12"/>', (0, s * 0.08, 0), (1.5707963267948966, 0, 0))] if i < 4 else []))
        joints.append((f"lift{i}", "revolute", f"coxa{i}", f"femur{i}", (0, s * 0.06, 0), _Z3, (1, 0, 0), (-1.2, 1.2, 40)))
        links.append((f"tibia{i}", 0.3, (0, s * 0.01, -0.1), (0.001, 0.001, 0.0002), [('<sphere radius="0.025"/>', (0, s * 0.02, -0.2), _Z3)]))
        joints.append((f"knee{i}", "revolute", f"femur{i}", f"tibia{i}", (0, s * 0.16, 0), _Z3, (1, 0, 0), (-2.0, 0.3, 30)))
    return _urdf("hexapod", links, joints)


def _max32():
    """Every bound the loader accepts: nb 32 (one body per lane), nv 37 (> 32 dofs), depth 6, exactly 64 contact candidates of every
    type (spheres, capsules, box corners and faces, cylinder rims), a prismatic joint, position and effort limits on every joint.
    A floating star: five 6-link chains lying in the base plane (link 1 turns about the base normal), and a mast carrying a cylinder."""
    links = [("base", 15.0, (0, 0, 0), (0.22, 0.33, 0.5), [('<box size="0.5 0.4 0.15"/>', _Z3, _Z3)])]
    joints = [("mast_j", "revolute", "base", "mast", (0, 0, 0.1), _Z3, (0, 0, 1), (-1.0, 1.0, 20))]
    links.append(("mast", 1.0, (0, 0, 0.1), (0.004, 0.004, 0.001), [('<cylinder radius="0.05" length="0.2"/>', (0, 0, 0.1), _Z3)]))
    axes = [(0, 0, 1), (0, 1, 0), (1, 0, 0), (0, 1, 0), (1, 0, 0), (0, 1, 0)]
    cap = ('<capsule radius="0.03" length="0.06"/>', (0.05, 0, 0), (0, 1.5707963267948966, 0))       # along the link
    for c in range(5):
        phi = 2 * np.pi * c / 5
        parent = "base"
        for k in range(6):
            ln = f"c{c}_l{k + 1}"
            colls = []
            if k == 1 or (k == 2 and c in (1, 3, 4)):
                colls.append(cap)
            if k in (3, 5) or (k == 4 and c == 2):
                colls.append(('<sphere radius="0.04"/>', (0.1, 0, 0), _Z3))
            if k == 5 and c == 0:
                colls.append(('<box size="0.06 0.04 0.03"/>', (0.05, 0, 0), _Z3))
            links.append((ln, 0.6 - 0.07 * k, (0.05, 0, 0), (0.0004, 0.001, 0.001), colls))
            xyz = (0.28 * np.cos(phi), 0.22 * np.sin(phi), 0) if k == 0 else (0.1, 0, 0)
            rpy = (0, 0, phi) if k == 0 else _Z3
            prismatic = c == 2 and k == 3
            joints.append((f"c{c}_j{k + 1}", "prismatic" if prismatic else "revolute", parent, ln, xyz, rpy, (1, 0, 0) if prismatic else axes[k],
                           (-0.05, 0.05, 200) if prismatic else (-0.5, 0.5, 15 + 5 * (k % 3))))
            parent = ln
    return _urdf("max32", links, joints)


QUAD_FEET = _anymal_variant(feet_only=True)
QUAD_PRISMATIC = _anymal_variant(prismatic_knees=True)
QUAD_BRANCHED = _quad_branched()
HEXAPOD = _hexapod()
MAX32 = _max32()


# ---------------------------------------------------------------------------------------------------------------------------------
# GPU batch and oracles on the same seeded inputs

def setup_batch(capi, urdf, n, seed, terrain="ground", base_z=0.45, vel=0.5, tau_scale=20.0, params=None, joint_scale=0.5):
    from oracle.oracle import Oracle
    from oracle.urdf_tables import load_tables
    path = os.path.join(_RSC, urdf) if urdf.endswith(".urdf") else urdf
    t = load_tables(path)
    m = capi.Model(path)
    bt = capi.Batch(m, n)
    rng = np.random.default_rng(seed)
    gc, gv = random_state(t, rng, n, vel_scale=vel, base_z=base_z, pos_scale=2.0, joint_scale=joint_scale)
    tau = rng.uniform(-tau_scale, tau_scale, (n, t["nv"]))
    if t["floating"]:
        tau[:, :6] = 0
    prm = dict(threshold=THRESH)     # everything else at the library defaults = what bench.py runs (accelerated sweeps, stagnation
                                     # window 8 with the compliant fallback); tests of the plain published method pass accel_m=0, stall_window=0
    prm.update(params or {})
    o64, o32 = Oracle(t, params=prm), Oracle(t, precision="f32", params=prm)
    bt.set_params(**{k: v for k, v in prm.items() if k not in ("gx", "gy", "gz")})
    if any(k in prm for k in ("gx", "gy", "gz")):
        bt.set_params(gravity=(prm.get("gx", 0.0), prm.get("gy", 0.0), prm.get("gz", -9.81)))
    if terrain == "ground":
        for o in (o64, o32):
            o.set_ground(0.0)
        bt.set_ground(0.0)
    elif terrain == "hm":
        xs, ys = 65, 49
        H = (0.1 * rng.uniform(-1, 1, (ys, xs))).astype(np.float32)
        for o in (o64, o32):
            o.set_heightmap(xs, ys, 12.8, 9.6, 0.1, -0.2, H.astype(np.float64))
        bt.set_heightmap(xs, ys, 12.8, 9.6, 0.1, -0.2, H)
    gc32, gv32, tau32 = gc.astype(np.float32), gv.astype(np.float32), tau.astype(np.float32)
    bt.set_control_mode(capi.FORCE_AND_TORQUE)
    bt.set_state(gc32, gv32)
    bt.set_generalized_force(tau32)
    return t, bt, o64, o32, gc32.astype(np.float64), gv32.astype(np.float64), tau32.astype(np.float64)


# Contact row bias on: ERP pushes penetrations and joint-limit violations out, restitution reflects approach speeds beyond
# rest_threshold.  The tests that run with it check that the threshold splits the contacts (normal_speeds).
ROW_BIAS = dict(erp=0.02, restitution=0.4, rest_threshold=0.2)


def normal_speeds(t, gc, gv, d):
    """J_n v of every terrain contact of the oracle's debug output d at the state (gc, gv) it stepped from (nan elsewhere): the approach
    speed that the restitution switch compares with -rest_threshold"""
    n, K = d["c_pt"].shape
    out = np.full((n, K), np.nan)
    for e in range(n):
        R, p, a = fk_numpy(t, gc[e])
        for k in range(d["ncontacts"][e]):
            if d["c_pair"][e, k] < 0:
                continue
            x = d["c_pos"][e, k]
            v = gv[e, 0:3] + np.cross(gv[e, 3:6], x - p[0]) if t["floating"] else np.zeros(3)
            j = d["c_body"][e, k]
            while t["parent"][j] >= 0:
                v = v + gv[e, t["vidx"][j]] * (np.cross(a[j], x - p[j]) if t["jtype"][j] == 1 else a[j])
                j = t["parent"][j]
            out[e, k] = d["c_normal"][e, k] @ v
    return out


def check_restitution_split(vn, rest_threshold):
    """the restitution switch is taken for some contacts and not for others, and no approach speed lies so close to the threshold that
    float32 rounding of the state could flip the switch"""
    vn = vn[np.isfinite(vn)]
    print(f"approach speeds beyond the restitution threshold: {int((vn < -rest_threshold).sum())} of {vn.size}, closest "
          f"{np.abs(vn + rest_threshold).min():.1e} m/s")
    assert (vn < -rest_threshold).sum() > 10 and (vn > -rest_threshold).sum() > 10
    assert np.abs(vn + rest_threshold).min() > 1e-4


def index_parity(pts_gpu, cnt_gpu, d_ref, label):
    """bit-exact contact lists, excluding environments that hold a candidate inside the margin."""
    n = len(cnt_gpu)
    shallow = (np.abs(d_ref["c_depth"]) < MARGIN) & (d_ref["c_pt"] >= 0)
    ok_env = ~shallow.any(1)
    excluded = int((~ok_env).sum())
    mism = (pts_gpu != d_ref["c_pt"]).any(1) | (cnt_gpu != d_ref["ncontacts"])
    # an environment may only mismatch if it has a margin candidate in the reference ...
    hard = mism & ok_env
    # ... or a candidate that the reference rejected by less than the margin (not recorded): allow
    # those only if the contact COUNT differs by the extra near-zero candidates
    print(f"[{label}] envs={n} contacts={int(cnt_gpu.sum())} margin-excluded envs={excluded} mismatching={int(mism.sum())}")
    return hard


def launch_config(capi, bt):
    """the step kernel's launch as pick_config chose it: warps per CTA, CTAs, compiled instance (spec 0 generic, 1 quadruped,
    2 humanoid) and candidate slots per lane"""
    import ctypes
    L = capi.lib()
    L.rsb_internal_launch_config.argtypes = [ctypes.c_void_p] * 3
    L.rsb_internal_launch_instance.argtypes = [ctypes.c_void_p] * 3
    v = [ctypes.c_int() for _ in range(4)]
    assert L.rsb_internal_launch_config(bt.h, ctypes.byref(v[0]), ctypes.byref(v[1])) == 0
    assert L.rsb_internal_launch_instance(bt.h, ctypes.byref(v[2]), ctypes.byref(v[3])) == 0
    return dict(zip(("wpc", "grid", "spec", "slots"), [x.value for x in v]))


# ---------------------------------------------------------------------------------------------------------------------------------
# Every compiled instance of the step kernel: the models that reach each one, and a batch of robots landing under stiff PD

OPTIONS = (28, 16, 14, 8, 4, 1)          # warps per CTA, as pick_config offers them
# name, robot description, RSB_FORCE_GENERIC, (spec, slots) it must run, base height, nominal joint positions
_Q = ANYMAL_GC0[7:]
_QP = np.where(np.arange(12) % 3 == 2, 0.0, _Q)          # prismatic knees at the middle of their travel
CASES = {
    "quad_feet": (QUAD_FEET, False, (1, 1), 0.56, _Q),
    "anymal": ("anymal_c_like.urdf", False, (1, 2), 0.56, _Q),
    "quad_prismatic": (QUAD_PRISMATIC, False, (1, 2), 0.62, _QP),
    "quad_branched": (QUAD_BRANCHED, False, (0, 1), 0.6, None),
    "atlas": ("atlas_like.urdf", False, (2, 2), 0.95, None),
    "hexapod": (HEXAPOD, False, (0, 1), 0.22, None),
    "max32": (MAX32, False, (0, 2), 0.1, None),
    "anymal_generic": ("anymal_c_like.urdf", True, (0, 2), 0.56, _Q),
    "atlas_generic": ("atlas_like.urdf", True, (0, 2), 0.95, None),
}
# warps per CTA whose CTA (model block + one workspace per warp) fits in the 227 KB of shared memory of an H100
FITS = {
    "quad_feet": OPTIONS, "anymal": OPTIONS, "quad_prismatic": OPTIONS, "quad_branched": OPTIONS, "anymal_generic": OPTIONS,
    "hexapod": (16, 14, 8, 4, 1),
    "atlas": (16, 14, 8, 4, 1), "atlas_generic": (16, 14, 8, 4, 1),
    "max32": (16, 14, 8, 4, 1),
}


def _nominal(name, t):
    urdf, generic, inst, base_z, q = CASES[name]
    gc0 = np.zeros(t["nq"]); gc0[2] = base_z; gc0[3] = 1.0
    if q is not None:
        gc0[7:] = q
    return gc0


def _state(name, t, n, rng):
    """upright robots with a small random tilt, jittered joints and velocities, spread over the terrain; in every environment two
    joints of short travel (less than 3 rad or m between the stops) start up to 5 cm or 0.05 rad past a stop"""
    gc0 = _nominal(name, t)
    gc = np.tile(gc0, (n, 1))
    gc[:, :2] = rng.uniform(-2, 2, (n, 2))
    q = np.c_[np.ones(n), 0.08 * rng.standard_normal((n, 3))]; q /= np.linalg.norm(q, axis=1, keepdims=True)
    gc[:, 3:7] = q
    gc[:, 7:] += rng.uniform(-0.15, 0.15, (n, t["nq"] - 7))
    short = np.where((t["jlimit"][1:, 1] - t["jlimit"][1:, 0]) < 3.0)[0] + 1
    for e in range(n):
        for body in rng.choice(short, 2, replace=False):
            lo, hi = t["jlimit"][body]
            gc[e, t["qidx"][body]] = hi + rng.uniform(0.01, 0.05) if rng.uniform() < 0.5 else lo - rng.uniform(0.01, 0.05)
    gv = 0.3 * rng.standard_normal((n, t["nv"]))
    return gc.astype(np.float32).astype(np.float64), gv.astype(np.float32).astype(np.float64)


def _pd(t, n, gc0, rng):
    """stiff PD towards targets up to 0.6 rad / m off the nominal pose: joints run into their stops and their actuators' effort limits"""
    kp = np.r_[np.zeros(6), 300.0 * np.ones(t["nv"] - 6)]; kd = np.r_[np.zeros(6), 4.0 * np.ones(t["nv"] - 6)]
    pt = np.tile(gc0, (n, 1)); pt[:, 7:] += rng.uniform(-0.6, 0.6, (n, t["nq"] - 7))
    prismatic = t["jtype"][1:] == 2
    pt[:, 7:][:, prismatic] = np.tile(gc0[7:][prismatic], (n, 1)) + rng.uniform(-0.2, 0.2, (n, prismatic.sum()))
    return kp, kd, pt.astype(np.float32)


def _batch(capi, monkeypatch, name, n, terrain, seed, wpc=None, params=None):
    urdf, generic, inst, base_z, q = CASES[name]
    monkeypatch.setenv("RSB_FORCE_GENERIC", "1" if generic else "0")
    if wpc is None:
        monkeypatch.delenv("RSB_FORCE_WPC", raising=False)
    else:
        monkeypatch.setenv("RSB_FORCE_WPC", str(wpc))
    t, bt, o64, o32, _, _, _ = setup_batch(capi, urdf, n, seed, terrain=terrain, tau_scale=0.0, params=params)
    cfg = launch_config(capi, bt)
    assert (cfg["spec"], cfg["slots"]) == inst, f"{name}: runs instance {cfg}, expected (spec, slots) = {inst}"
    rng = np.random.default_rng(seed + 1)
    gc, gv = _state(name, t, n, rng)
    kp, kd, pt = _pd(t, n, _nominal(name, t), rng)
    bt.set_state(gc.astype(np.float32), gv.astype(np.float32))
    bt.set_control_mode(capi.PD_PLUS_FEEDFORWARD_TORQUE)
    bt.set_generalized_force(np.zeros((n, t["nv"]), np.float32))
    bt.set_pd_gains(kp, kd)
    bt.set_pd_target(pt, np.zeros((n, t["nv"]), np.float32))
    return t, bt, o64, o32, gc, gv, kp, kd, pt, cfg


def effort_limits(t):
    """[nv] URDF effort limit of every dof in the batch's gv order (the base: unlimited)"""
    lim = np.full(t["nv"], 1e30)
    for b in range(1, t["nb"]):
        lim[t["vidx"][b]] = t["jeffort"][b]
    return lim


def _at_effort_limit(t, tau_applied):
    lim = np.array([t["jeffort"][i] for i in range(1, t["nb"])])
    return np.abs(np.abs(tau_applied[:, 6:]) - lim[None, :]) < 1e-9 * lim[None, :]


def _row(name, cfg, n, K, cr, extra):
    T = cfg["wpc"] * cfg["grid"]
    rounds = -(-n // T)
    fill = (n - (rounds - 1) * T) / T
    print(f"| {name:15s} | spec {cfg['spec']} | slots {cfg['slots']} | WPC {cfg['wpc']:2d} | grid {cfg['grid']:3d} | rounds {rounds:2d} | "
          f"last round {100 * fill:5.1f} % | K {K:.2f} | CR max {cr if cr >= 0 else '-':>2} | {extra}")


def step_and_trajectory(capi, monkeypatch, name, terrain, seed, params=None, n=256, near_threshold="refuse", converged=0.88, flips=0):
    """one step (contact lists, state, impulses, complementarity, actuators at their effort limits) and 10 steps (state) of CASES[name]
    against the oracle, PD targets on, joints at their stops and actuators at their effort limits.  params: rsb_params fields (gx, gy,
    gz for gravity) on both sides; dt, mu and joint_limits set the bounds and the edges the run must reach.  With restitution on
    (restitution and rest_threshold > 0) the threshold must split the approach speeds; an approach speed within 1e-4 m/s of it fails
    the run (near_threshold="refuse") or leaves its environment out of the one-step comparison ("exclude").  converged: the least share
    of environments whose solves converge on both sides with equal contact lists (the one-step comparison's sample).  flips: environments
    left out of the 10-step quantiles, the worst ones -- on the rough map index parity allows one contact list per step to differ on a
    tie, and a robot whose contact set changed one step apart from the oracle's follows another trajectory from there.
    Returns a dict of the run's figures for the caller's table."""
    prm = dict(params or {})
    dt, mu, limits = prm.get("dt", 0.0025), prm.get("mu", 0.8), prm.get("joint_limits", 1)
    t, bt, o64, o32, gc, gv, kp, kd, pt, cfg = _batch(capi, monkeypatch, name, n, terrain, seed=seed, params=prm)
    ptd, vt = pt.astype(np.float64), np.zeros((n, t["nv"]))
    bt.integrate(1)
    g1, v1 = bt.get_state(); ct, cnt = bt.contacts(); pts = bt.contact_points(); st = bt.solver_status(); ta = bt.generalized_force()
    a, b = gc.copy(), gv.copy()
    d = o64.step(a, b, ptarget=ptd, vtarget=vt, kp=kp, kd=kd, debug=True)
    c, e_ = gc.copy(), gv.copy()
    d32 = o32.step(c, e_, ptarget=ptd, vtarget=vt, kp=kp, kd=kd, debug=True)
    assert np.isfinite(g1).all() and np.isfinite(v1).all()
    # the edges this test is meant to reach: contacts, joint-limit rows (none with joint_limits = 0), saturated actuators
    sat_ref = _at_effort_limit(t, d["tau_applied"])
    assert cnt.sum() > n // 4 and sat_ref.any()
    assert d["nlimits"].sum() > 0 if limits else d["nlimits"].sum() == 0
    # the effort-limit switch (its threshold moves with dt) takes the oracle's side on every actuator not within rounding of it
    lim = np.array([t["jeffort"][i] for i in range(1, t["nb"])])
    sat_gpu = np.abs(np.abs(ta[:, 6:].astype(np.float64)) - lim[None, :]) < 1e-6 * lim[None, :]
    assert (sat_gpu == sat_ref).mean() > 0.999, f"{int((sat_gpu != sat_ref).sum())} actuators switched differently"
    near = np.zeros(n, bool)
    if prm.get("restitution", 0.0) > 0 and prm.get("rest_threshold", 0.01) > 0:
        vn = normal_speeds(t, gc, gv, d)
        if near_threshold == "refuse":
            check_restitution_split(vn, prm["rest_threshold"])
        else:
            w = vn[np.isfinite(vn)]
            assert (w < -prm["rest_threshold"]).sum() > 10 and (w > -prm["rest_threshold"]).sum() > 10
            near = (np.abs(np.nan_to_num(vn, nan=1e9) + prm["rest_threshold"]) < 1e-4).any(1)
    hard = index_parity(pts, cnt, d32, f"{name} {terrain}")
    # on the rough map two triangles sharing an edge can tie to 1e-6 m under different rounding
    # (test_heightmap_narrow_phase_matches_oracle_on_rough_terrain): at most one environment in 256
    assert hard.sum() <= (0 if terrain == "ground" else 1), f"contact lists differ in envs {np.where(hard)[0][:10]}"
    same = (pts == d["c_pt"]).all(1)
    conv = same & (st == 0) & (d["status"] == 0) & ~near
    ev = np.abs(v1 - b)[conv]; eq = np.abs(g1 - a)[conv]; e32 = np.abs(e_ - b)[conv]
    scale_v = 1.0 + np.abs(b[conv])
    live = conv[:, None] & (d["c_pt"] >= 0)
    ln_gpu = np.einsum("ekj,ekj->ek", ct["impulse"], ct["normal"])
    en = np.abs(ln_gpu - d["c_lambda"][:, :, 2])[live]
    lam_scale = max(1.0, np.abs(d["c_lambda"][:, :, 2][live]).max()) if live.any() else 1.0
    # 10 control steps from the start state
    bt.integrate(9)
    gN, _ = bt.get_state()
    o64.step(a, b, n_steps=9, ptarget=ptd, vtarget=vt, kp=kp, kd=kd)
    o32.step(c, e_, n_steps=9, ptarget=ptd, vtarget=vt, kp=kp, kd=kd)
    e = np.sort(np.abs(gN - a).max(1))[:n - flips]; ef = np.abs(c - a).max(1)
    print(f"   {name} {terrain}: oracle limit rows {np.bincount(d['nlimits'], minlength=5).tolist()}, dofs at their effort limit "
          f"{int(sat_ref.sum())}")
    cr = int((3 * d["ncontacts"] + d["nlimits"]).max())
    _row(name, cfg, n, cnt.mean(), cr, f"{terrain:6s} | converged {100 * conv.mean():.0f} % | 1 step: gv err median {np.median(ev.max(1)):.1e} "
         f"(f32 oracle {np.median(e32.max(1)):.1e}), normal impulse p99 {np.quantile(en, .99) if en.size else 0:.1e} | 10 steps: gc err median "
         f"{np.median(e):.1e} p90 {np.quantile(e, .9):.1e} p99 {np.quantile(e, .99):.1e} (f32 oracle p99 {np.quantile(ef, .99):.1e})")
    assert conv.mean() > converged
    assert np.median(ev.max(1)) < max(2e-5, 3 * np.median(e32.max(1)))
    assert np.max(ev / scale_v) < max(5e-3, 3 * np.max(e32 / scale_v))
    assert eq.max() < 5e-3 * dt * (1.0 + np.abs(b[conv]).max()) + 2e-6
    assert en.size == 0 or np.quantile(en, 0.99) < 1e-4 * lam_scale
    # Signorini and Coulomb on the GPU result itself, with the friction in force
    on = np.arange(ct["impulse"].shape[1])[None, :] < cnt[:, None]
    assert (ln_gpu[on] >= -1e-6).all()
    lt = np.linalg.norm(ct["impulse"] - ln_gpu[:, :, None] * ct["normal"], axis=2)
    assert (lt[on] <= mu * ln_gpu[on] + 1e-4 * (1 + ln_gpu[on])).all()
    assert np.isfinite(gN).all() and flips <= n // 25
    # positions drift from the oracle's in proportion to the step: the absolute floors are those of the default dt, 0.0025
    grow = max(1.0, dt / 0.0025)
    assert np.median(e) < 2e-5 * grow and np.median(e) < 5 * np.median(ef) + 1e-6
    assert np.quantile(e, 0.9) < max(1e-4 * grow, 5 * np.quantile(ef, 0.9))
    assert np.quantile(e, 0.99) < max(5e-3 * grow, 5 * np.quantile(ef, 0.99))
    return dict(t=t, bt=bt, d=d, ct=ct, cnt=cnt, pts=pts, st=st, conv=conv, ln_gpu=ln_gpu, lt=lt, on=on)
