"""CPU-side checks of the product: the C-ABI library loads, exports every symbol include/rsb.h declares,
and its URDF loader agrees table-by-table with the oracle's independent Python restatement."""
import os
import re
import ctypes
import numpy as np
import pytest

from conftest import ROOT, RSC
from raisimlib_b200 import capi
from oracle.urdf_tables import load_tables
from helpers import PENDULUM_URDF, BOX_URDF, REALISTIC_URDF, QUAD_FEET, QUAD_PRISMATIC, QUAD_BRANCHED, HEXAPOD, MAX32


def _declared_symbols():
    src = open(os.path.join(ROOT, "include", "rsb.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(rsb_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    L = capi.lib()
    names = _declared_symbols()
    assert len(names) >= 40
    for n in names:
        assert hasattr(L, n), f"{n} declared in include/rsb.h but not exported by librsb.so"
    assert sorted(capi.EXPORTED) == names


def test_struct_layouts_match_header():
    assert ctypes.sizeof(capi.Contact) == 48       # 12 words, SURVEY 8d algorithmic-bytes formula
    assert ctypes.sizeof(capi.Params) == 4 * 19      # rsb_params: 16 words of round 1 + accel_m, accel_start, stall_reg


def test_set_params_refuses_non_finite_fields_before_the_batch():
    """every non-finite float field of rsb_params is refused by name, before the batch is looked at; a valid set reaches the
    null-batch check"""
    L = capi.lib()
    p = capi.Params()
    assert L.rsb_params_default(ctypes.byref(p)) == 0
    assert L.rsb_batch_set_params(None, ctypes.byref(p)) == -1 and "null argument" in L.rsb_last_error().decode()
    fields = ["dt", "erp", "alpha_init", "alpha_min", "alpha_decay", "threshold", "mu", "restitution", "rest_threshold", "stall_ratio", "stall_reg"]
    for f in fields + [f"gravity[{i}]" for i in range(3)]:
        for v in (float("nan"), float("inf"), float("-inf")):
            q = capi.Params.from_buffer_copy(bytes(p))
            if f.startswith("gravity"):
                q.gravity[int(f[8])] = v
            else:
                setattr(q, f, v)
            assert L.rsb_batch_set_params(None, ctypes.byref(q)) == -1
            assert L.rsb_last_error().decode() == f"params: {f} is not finite", (f, v)


@pytest.mark.parametrize("src", ["anymal_c_like.urdf", "atlas_like.urdf", PENDULUM_URDF, BOX_URDF, REALISTIC_URDF,
                                 pytest.param(QUAD_FEET, id="quad_feet"), pytest.param(QUAD_PRISMATIC, id="quad_prismatic"),
                                 pytest.param(QUAD_BRANCHED, id="quad_branched"), pytest.param(HEXAPOD, id="hexapod"), pytest.param(MAX32, id="max32")])
def test_model_tables_match_python_restatement(src):
    path = os.path.join(RSC, src) if src.endswith(".urdf") else src
    a = capi.Model(path).tables()
    b = load_tables(path)
    for k in ("nb", "nq", "nv", "floating", "ncoll", "npts"):
        assert a[k] == b[k], k
    for k in ("parent", "jtype", "qidx", "vidx", "depth", "cbody", "ctype", "pt_body", "pt_coll", "pt_feat", "pt_type"):
        assert (a[k] == b[k]).all(), k
    for k in ("jpos", "jrot", "axis", "mass", "com", "inertia", "jlimit", "csize", "cpos", "crot", "pt_pos", "pt_rad", "pt_pos2", "jeffort"):
        assert np.allclose(a[k], b[k], rtol=1e-13, atol=1e-15), k
    assert a["body_names"] == b["body_names"] and a["joint_names"] == b["joint_names"]


def test_model_errors_are_reported_not_thrown():
    with pytest.raises(capi.RsbError, match="cannot open"):
        capi.Model("/nonexistent/robot.urdf")
    with pytest.raises(capi.RsbError, match="mismatched"):
        capi.Model("<robot><link name='a'></robot>")
    with pytest.raises(capi.RsbError, match="unsupported joint type"):
        capi.Model("<robot><link name='a'/><link name='b'><inertial><mass value='1'/><inertia ixx='1' iyy='1' izz='1'/></inertial></link>"
                   "<joint name='j' type='planar'><parent link='a'/><child link='b'/></joint></robot>")


def test_body_index_resolves_merged_links():
    m = capi.Model(os.path.join(RSC, "anymal_c_like.urdf"))
    assert m.body_index("base") == 0
    assert m.body_index("LF_SHANK") == 3
    assert m.body_index("LF_FOOT") == 3            # merged through the fixed joint
    with pytest.raises(capi.RsbError):
        m.body_index("nope")


def test_no_gpu_means_loud_failure():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    m = capi.Model(os.path.join(RSC, "anymal_c_like.urdf"))
    with pytest.raises(capi.RsbError, match="no CPU fallback"):
        capi.Batch(m, 4)


def test_argument_validation_without_gpu():
    """empty / negative sizes and null handles are rejected with a message, never a crash (no GPU needed)"""
    import ctypes as C
    L = capi.lib()
    m = capi.Model(os.path.join(RSC, "anymal_c_like.urdf"))
    h = C.c_void_p()
    assert L.rsb_batch_create(m.h, 0, 0, C.byref(h)) < 0 and b"bad arguments" in L.rsb_last_error()
    assert L.rsb_batch_create(m.h, -5, 0, C.byref(h)) < 0
    assert L.rsb_batch_create(None, 4, 0, C.byref(h)) < 0
    assert L.rsb_batch_integrate(None, 1) < 0
    assert L.rsb_batch_num_envs(None) == 0
    assert L.rsb_model_body_index(None, b"x") < 0
    p = capi.Params()
    assert L.rsb_params_default(C.byref(p)) == 0
    assert abs(p.dt - 0.0025) < 1e-9 and p.max_iter == 150 and p.stall_window == 8 and abs(p.mu - 0.8) < 1e-7 and p.accel_m == 2 and p.accel_start == 6 and abs(p.stall_reg - 0.02) < 1e-8


def test_too_many_bodies_is_reported():
    links = "".join(f"<link name='l{i}'><inertial><mass value='1'/><inertia ixx='1' iyy='1' izz='1'/></inertial></link>" for i in range(40))
    joints = "".join(f"<joint name='j{i}' type='revolute'><parent link='l{i}'/><child link='l{i+1}'/><axis xyz='0 0 1'/></joint>" for i in range(39))
    with pytest.raises(capi.RsbError, match="more than 32 movable bodies"):
        capi.Model(f"<robot name='chain'>{links}{joints}</robot>")


def test_realistic_description_features():
    """visual / mesh / gazebo / transmission tags are skipped, a massless fixed link merges, a cylinder yields 8 rim points"""
    t = capi.Model(REALISTIC_URDF).tables()
    assert (t["nb"], t["nq"], t["nv"]) == (2, 8, 7)
    assert t["ncoll"] == 2 and list(t["ctype"]) == [1, 3]          # box + cylinder; the mesh collision body is skipped
    assert t["npts"] == 16 + 1 + 3                                  # 8 box corners + 8 rim samples, then the box-face feature and the cylinder's axis segment + 2 rim features
    assert list(t["pt_type"]) == [0] * 16 + [2, 1, 3, 3]
    rim = t["pt_pos"][8:16]
    assert np.allclose(np.hypot(rim[:, 0], rim[:, 1]), 0.025) and np.allclose(sorted(set(np.round(rim[:, 2], 6))), [-0.3, 0.0])
    assert t["jlimit"][1, 0] < -1e29                               # continuous joint: no limits


def test_terrain_generator_properties():
    """raisim::TerrainProperties analogue: deterministic per seed, bounded by the octave sum, frequency and steps honoured"""
    a = capi.generate_terrain(seed=7); b = capi.generate_terrain(seed=7); c = capi.generate_terrain(seed=8)
    assert a.shape == (129, 129) and np.array_equal(a, b) and not np.array_equal(a, c)
    assert np.abs(a).max() <= 0.5 * (1 + 0.25 + 0.0625) and a.std() > 0.02
    rough = capi.generate_terrain(seed=7, frequency=1.0)
    assert np.abs(np.diff(rough, axis=1)).mean() > 2 * np.abs(np.diff(a, axis=1)).mean()     # higher frequency, steeper
    st = capi.generate_terrain(seed=7, step_size=0.05)
    assert np.allclose(st / 0.05, np.round(st / 0.05), atol=1e-4)
    off = capi.generate_terrain(seed=7, height_offset=1.5)
    assert np.allclose(off - a, 1.5, atol=1e-6)


def test_heightmap_text_and_png_loaders(tmp_path):
    """N3: World::addHeightMap(file ...) front ends -- host code, no GPU needed"""
    from PIL import Image
    rng = np.random.default_rng(9)
    xs, ys = 37, 23
    H = rng.uniform(-0.3, 0.4, (ys, xs)).astype(np.float32)
    txt = tmp_path / "hm.txt"
    with open(txt, "w") as f:
        f.write(f"{xs} {ys} 7.4 4.6\n")
        for row in H:
            f.write(" ".join(f"{v:.9g}" for v in row) + "\n")
    got, sx, sy = capi.read_heightmap_text(str(txt))
    assert got.shape == (ys, xs) and (sx, sy) == (7.4, 4.6) and np.array_equal(got, H)
    # 16-bit grey, 8-bit grey, RGB and RGBA (first channel), with a smooth image so that PNG's adaptive filters are all used
    yy, xx = np.mgrid[0:ys, 0:xs]
    smooth = (np.sin(xx / 5.0) * np.cos(yy / 3.0) * 0.5 + 0.5)
    img16 = (smooth * 60000 + rng.integers(0, 300, (ys, xs))).astype(np.uint16)
    p16 = tmp_path / "hm16.png"; Image.fromarray(img16).save(p16)
    got = capi.read_heightmap_png(str(p16), 1e-4, -2.0)
    assert got.shape == (ys, xs) and np.allclose(got, img16.astype(np.float64) * 1e-4 - 2.0, atol=1e-6)
    img8 = (smooth * 250).astype(np.uint8)
    p8 = tmp_path / "hm8.png"; Image.fromarray(img8).save(p8)
    assert np.array_equal(capi.read_heightmap_png(str(p8)), img8.astype(np.float32))
    rgb = np.stack([img8, 255 - img8, img8 // 2], -1)
    prgb = tmp_path / "hmrgb.png"; Image.fromarray(rgb).save(prgb)
    assert np.array_equal(capi.read_heightmap_png(str(prgb), 0.5, 1.0), img8.astype(np.float32) * 0.5 + 1.0)
    rgba = np.concatenate([rgb, np.full((ys, xs, 1), 200, np.uint8)], -1)
    prgba = tmp_path / "hmrgba.png"; Image.fromarray(rgba).save(prgba)
    assert np.array_equal(capi.read_heightmap_png(str(prgba)), img8.astype(np.float32))
    # errors are reported, not thrown
    bad = tmp_path / "bad.png"; bad.write_bytes(b"not a png at all, just text that is long enough to pass the size check....")
    with pytest.raises(RuntimeError, match="not a PNG"):
        capi.read_heightmap_png(str(bad))
    short = tmp_path / "short.txt"; short.write_text("4 4 1.0 1.0\n0 0 0\n")
    with pytest.raises(RuntimeError, match="heights found"):
        capi.read_heightmap_text(str(short))
    with pytest.raises(RuntimeError, match="cannot open"):
        capi.read_heightmap_text(str(tmp_path / "missing.txt"))


@pytest.mark.parametrize("src", ["anymal_c_like.urdf", "atlas_like.urdf"])
def test_binary_model_cache_round_trip(src, tmp_path):
    """N2: rsb_model_save / rsb_model_load reproduce every table bit for bit; damaged files are reported"""
    m = capi.Model(os.path.join(RSC, src))
    path = str(tmp_path / "model.rsbm")
    m.save(path)
    m2 = capi.Model(path, cache=True)
    a, b = m.tables(), m2.tables()
    assert a.keys() == b.keys()
    for k in a:
        assert (np.array_equal(a[k], b[k]) if isinstance(a[k], np.ndarray) else a[k] == b[k]), k
    assert (m.nq, m.nv, m.nb, m.ncoll, m.npts) == (m2.nq, m2.nv, m2.nb, m2.ncoll, m2.npts)
    foot = "LF_FOOT" if "anymal" in src else m.tables()["body_names"][-1]
    assert m.body_index(foot) == m2.body_index(foot)
    blob = open(path, "rb").read()
    bad = tmp_path / "trunc.rsbm"; bad.write_bytes(blob[: len(blob) // 2])
    with pytest.raises(capi.RsbError, match="truncated|corrupt|inconsistent"):
        capi.Model(str(bad), cache=True)
    bad2 = tmp_path / "magic.rsbm"; bad2.write_bytes(b"XXXX" + blob[4:])
    with pytest.raises(capi.RsbError, match="not a model cache"):
        capi.Model(str(bad2), cache=True)
    with pytest.raises(capi.RsbError, match="cannot open"):
        capi.Model(str(tmp_path / "missing.rsbm"), cache=True)


def test_product_never_touches_the_oracle():
    """the oracle is test infrastructure: nothing under raisimlib_b200/, include/, examples/ or tools/ may import, link or call it"""
    import re
    bad = []
    for top in ("raisimlib_b200", "include", "examples", "tools"):
        for root, _dirs, files in os.walk(os.path.join(ROOT, top)):
            for f in files:
                if not f.endswith((".py", ".cu", ".cuh", ".cpp", ".hpp", ".h", "Makefile")):
                    continue
                txt = open(os.path.join(root, f), errors="ignore").read()
                if re.search(r"^\s*(from|import)\s+oracle\b|liboracle|-loracle|#\s*include[^\n]*oracle|orc_[a-z_]+\(", txt, re.M):
                    bad.append(os.path.relpath(os.path.join(root, f), ROOT))
    assert not bad, bad


def test_pybind_module_loads_and_fails_loudly_without_gpu():
    """N4: the pybind11 + DLPack module (raisimlib_b200/_rsb_py) imports on a CPU-only machine, parses a model, and refuses to
    create a batch without a GPU (no CPU fallback)"""
    import torch
    from raisimlib_b200 import _rsb_py
    m = _rsb_py.Model(os.path.join(RSC, "anymal_c_like.urdf"))
    with pytest.raises(RuntimeError, match="cannot open"):
        _rsb_py.Model("/nonexistent.urdf")
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError, match="no CPU fallback"):
            _rsb_py.Batch(m, 4, 0)


def test_mesh_collision_becomes_its_bounding_box(tmp_path):
    """N2 mesh -> primitive fallback: a <mesh> collision whose file can be read (binary / ASCII STL, OBJ; package:// or relative path,
    <mesh scale>) is replaced by its axis-aligned bounding box in the collision frame; an unreadable one is skipped as before"""
    import struct
    tris = [((0, 0, 0), (0.4, 0, 0), (0, 0.2, 0)), ((0.4, 0.2, 0.1), (0.4, 0, 0), (0, 0.2, 0)), ((-0.1, 0, 0.05), (0, 0, 0), (0, 0.2, 0.1))]
    (tmp_path / "meshes").mkdir()
    with open(tmp_path / "meshes" / "part.stl", "wb") as f:
        f.write(b"binary stl".ljust(80, b" ")); f.write(struct.pack("<I", len(tris)))
        for t3 in tris:
            f.write(struct.pack("<3f", 0, 0, 1))
            for v in t3:
                f.write(struct.pack("<3f", *v))
            f.write(struct.pack("<H", 0))
    with open(tmp_path / "meshes" / "part.obj", "w") as f:
        f.write("# obj\n" + "".join(f"v {x} {y} {z}\n" for t3 in tris for (x, y, z) in t3) + "f 1 2 3\n")
    urdf = tmp_path / "robot.urdf"
    urdf.write_text(f"""<robot name="m"><link name="b"><inertial><mass value="1"/><inertia ixx="0.01" iyy="0.01" izz="0.01"/></inertial>
      <collision><origin xyz="0 0 0.5"/><geometry><mesh filename="package://some_pkg/meshes/part.stl" scale="2 1 1"/></geometry></collision>
      <collision><geometry><mesh filename="meshes/part.obj"/></geometry></collision>
      <collision><geometry><mesh filename="package://some_pkg/meshes/missing.dae"/></geometry></collision></link></robot>""")
    t = capi.Model(str(urdf)).tables()
    assert t["ncoll"] == 2 and list(t["ctype"]) == [1, 1]                                       # two boxes, the unreadable mesh skipped
    assert np.allclose(t["csize"][0], [0.5, 0.1, 0.05]) and np.allclose(t["cpos"][0], [0.3, 0.1, 0.55])   # x scaled by 2: [-0.2, 0.8] x [0, 0.2] x [0, 0.1]
    assert np.allclose(t["csize"][1], [0.25, 0.1, 0.05]) and np.allclose(t["cpos"][1], [0.15, 0.1, 0.05])
    assert t["npts"] == 2 * 8 + 2                                                                # corners + one box-face candidate each


def test_facade_host_pieces(tmp_path):
    """host-only pieces of the C++ facade (no GPU): HeightMap::getHeight against a numpy restatement of the collision surface on a random
    map (cell interiors, both triangles of a cell, grid nodes), Ground, the math helpers, the contact frame, loud failure without a robot"""
    import subprocess
    exe = tmp_path / "facade_host_check"
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-Wall", "-I" + os.path.join(ROOT, "include"), "-o", str(exe), os.path.join(ROOT, "tests", "cpp", "facade_host_check.cpp"),
                           "-L" + os.path.join(ROOT, "raisimlib_b200"), "-lrsb", "-Wl,-rpath," + os.path.join(ROOT, "raisimlib_b200"), "-Wl,-rpath,/usr/local/cuda/lib64"])
    rng = np.random.default_rng(77)
    xs, ys, sx, sy, cx, cy = 9, 7, 4.0, 2.4, 0.3, -0.2
    H = rng.uniform(-0.2, 0.2, (ys, xs))
    np.savetxt(tmp_path / "h.txt", H.reshape(-1))
    dx, dy = sx / (xs - 1), sy / (ys - 1)
    x0, y0 = cx - sx / 2, cy - sy / 2
    q = np.c_[rng.uniform(x0, x0 + sx, 400), rng.uniform(y0, y0 + sy, 400)]
    nodes = np.array([(x0 + i * dx, y0 + j * dy) for j in range(ys) for i in range(xs)])
    q = np.r_[q, nodes[: len(nodes) - xs][np.arange(len(nodes) - xs) % xs != xs - 1]]          # interior nodes (the oracle has no cell beyond the last row / column)
    np.savetxt(tmp_path / "q.txt", q)
    out = subprocess.run([str(exe), str(xs), str(ys), str(sx), str(sy), str(cx), str(cy), str(tmp_path / "h.txt"), str(tmp_path / "q.txt")],
                         capture_output=True, text=True, timeout=60)
    assert out.returncode == 0, out.stdout + out.stderr
    lines = out.stdout.split()
    got = np.array([float(v) for v in lines[: len(q)]])
    # numpy restatement of the two-triangles-per-cell surface (DESIGN.md section 2: cell split along P00-P11, tri 0 where fx >= fy)
    gx, gy = (q[:, 0] - x0) / dx, (q[:, 1] - y0) / dy
    ix, iy = np.minimum(gx.astype(int), xs - 2), np.minimum(gy.astype(int), ys - 2)
    fx, fy = gx - ix, gy - iy
    h00, h10, h01, h11 = H[iy, ix], H[iy, ix + 1], H[iy + 1, ix], H[iy + 1, ix + 1]
    surf = np.where(fx >= fy, h00 + (h10 - h00) * fx + (h11 - h10) * fy, h00 + (h11 - h01) * fx + (h01 - h00) * fy)
    assert np.abs(got - surf).max() < 1e-12
    assert "self-checks ok" in out.stdout
