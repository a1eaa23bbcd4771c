"""ctypes binding of the C-ABI in include/rsb.h (raisimlib_b200/librsb.so).

Thin by design: the product is the CUDA library; Python only drives it from tests and bench.py.
There is NO CPU fallback -- if librsb.so is missing or no GPU is visible the calls fail loudly.
"""
import ctypes as C
import os
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
# RSB_LIB_PATH loads another build of the library instead, such as the parent commit's in an A/B cost comparison
# (tools/feature_cost.py --parent-lib); calls that build does not export are left unbound
_OTHER_BUILD = os.environ.get("RSB_LIB_PATH")
LIB_PATH = _OTHER_BUILD or os.path.join(_HERE, "librsb.so")
KMAX = 8
HOST, DEVICE = 0, 1
FORCE_AND_TORQUE, PD_PLUS_FEEDFORWARD_TORQUE = 0, 1
SCAN_YAW, SCAN_WORLD = 0, 1
MAX_SCAN_POINTS = 1024
MAX_RAYS = 16384
RAY_MISS, RAY_TERRAIN = -1, -2           # hit ids of ray_casts() besides a collision-body index
RAYS_TERRAIN, RAYS_TERRAIN_AND_ROBOT = 0, 1
ACTUATION_DELAY_MAX = 16   # RSB_MAX_ACTUATION_DELAY: sub-steps


class RsbError(RuntimeError):
    pass


class Params(C.Structure):
    _fields_ = [("dt", C.c_float), ("gravity", C.c_float * 3), ("erp", C.c_float), ("alpha_init", C.c_float),
                ("alpha_min", C.c_float), ("alpha_decay", C.c_float), ("max_iter", C.c_int), ("threshold", C.c_float),
                ("mu", C.c_float), ("restitution", C.c_float), ("rest_threshold", C.c_float),
                ("stall_window", C.c_int), ("stall_ratio", C.c_float), ("joint_limits", C.c_int),
                ("accel_m", C.c_int), ("accel_start", C.c_int), ("stall_reg", C.c_float)]


class Contact(C.Structure):
    _fields_ = [("local_body", C.c_int32), ("pair_index", C.c_int32), ("position", C.c_float * 3),
                ("normal", C.c_float * 3), ("impulse", C.c_float * 3), ("depth", C.c_float)]


CONTACT_DTYPE = np.dtype([("local_body", np.int32), ("pair_index", np.int32), ("position", np.float32, 3),
                          ("normal", np.float32, 3), ("impulse", np.float32, 3), ("depth", np.float32)])
assert CONTACT_DTYPE.itemsize == C.sizeof(Contact) == 48


class ModelTables(C.Structure):
    _fields_ = ([(n, C.c_int) for n in ("nb", "nq", "nv", "floating", "ncoll", "npts")] +
                [(n, C.POINTER(C.c_int)) for n in ("parent", "jtype", "qidx", "vidx", "depth")] +
                [(n, C.POINTER(C.c_double)) for n in ("jpos", "jrot", "axis", "mass", "com", "inertia", "jlimit")] +
                [(n, C.POINTER(C.c_int)) for n in ("cbody", "ctype")] +
                [(n, C.POINTER(C.c_double)) for n in ("csize", "cpos", "crot")] +
                [(n, C.POINTER(C.c_int)) for n in ("pt_body", "pt_coll", "pt_feat")] +
                [(n, C.POINTER(C.c_double)) for n in ("pt_pos", "pt_rad")] +
                [("pt_type", C.POINTER(C.c_int)), ("pt_pos2", C.POINTER(C.c_double)), ("jeffort", C.POINTER(C.c_double))])


class TerrainProperties(C.Structure):
    _fields_ = [("x_samples", C.c_int), ("y_samples", C.c_int), ("x_size", C.c_double), ("y_size", C.c_double), ("frequency", C.c_double),
                ("z_scale", C.c_double), ("fractal_octaves", C.c_int), ("fractal_lacunarity", C.c_double), ("fractal_gain", C.c_double),
                ("step_size", C.c_double), ("height_offset", C.c_double), ("seed", C.c_uint32)]


def generate_terrain(x_samples=129, y_samples=129, x_size=12.8, y_size=12.8, frequency=0.2, z_scale=0.5, fractal_octaves=3,
                     fractal_lacunarity=2.0, fractal_gain=0.25, step_size=0.0, height_offset=0.0, seed=1):
    """raisim::TerrainProperties -> heights [y_samples, x_samples] float32 (host)"""
    p = TerrainProperties(x_samples, y_samples, x_size, y_size, frequency, z_scale, fractal_octaves, fractal_lacunarity, fractal_gain,
                          step_size, height_offset, seed)
    out = np.empty((y_samples, x_samples), np.float32)
    _ck(lib().rsb_terrain_generate(C.byref(p), out.ctypes.data_as(C.c_void_p)))
    return out


def pinhole_rays(width, height, hfov_deg):
    """unit directions [height * width, 3] float64 of a pinhole camera's rays through the pixel centres, row-major from the top-left
    pixel, in the camera frame: optical axis +x, image right -y, image down -z.  The vertical field of view follows from the square
    pixels: tan(vfov / 2) = tan(hfov / 2) * height / width.  With ray_casts() distances d [.., height * width] the z-depth image (distance
    along the optical axis) is d * dirs[:, 0]."""
    if width < 1 or height < 1 or not 0.0 < hfov_deg < 180.0:
        raise ValueError(f"pinhole_rays: need width, height >= 1 and 0 < hfov_deg < 180, got {width}, {height}, {hfov_deg}")
    f = 0.5 * width / np.tan(np.radians(hfov_deg) / 2)      # focal length in pixels
    u = np.arange(width) + 0.5 - 0.5 * width                 # pixel centre right of the axis
    v = np.arange(height) + 0.5 - 0.5 * height               # pixel centre below the axis
    V, U = np.meshgrid(v, u, indexing="ij")
    d = np.stack([np.full(U.shape, f), -U, -V], -1).reshape(-1, 3)
    return d / np.linalg.norm(d, axis=1, keepdims=True)


def read_heightmap_text(path):
    """World::addHeightMap(raisimHeightMapFileName, ...): -> (heights [ys, xs] float32, x_size, y_size)"""
    xs, ys, sx, sy = C.c_int(), C.c_int(), C.c_double(), C.c_double()
    L = lib()
    _ck(L.rsb_heightmap_read_text(path.encode(), C.byref(xs), C.byref(ys), C.byref(sx), C.byref(sy), None, 0))
    out = np.empty((ys.value, xs.value), np.float32)
    _ck(L.rsb_heightmap_read_text(path.encode(), C.byref(xs), C.byref(ys), C.byref(sx), C.byref(sy), out.ctypes.data_as(C.c_void_p), out.size))
    return out, sx.value, sy.value


def read_heightmap_png(path, height_scale=1.0, height_offset=0.0):
    """World::addHeightMap(pngFileName, cx, cy, xSize, ySize, heightScale, heightOffset): -> heights [ys, xs] float32"""
    xs, ys = C.c_int(), C.c_int()
    L = lib()
    _ck(L.rsb_heightmap_read_png(path.encode(), height_scale, height_offset, C.byref(xs), C.byref(ys), None, 0))
    out = np.empty((ys.value, xs.value), np.float32)
    _ck(L.rsb_heightmap_read_png(path.encode(), height_scale, height_offset, C.byref(xs), C.byref(ys), out.ctypes.data_as(C.c_void_p), out.size))
    return out


class DeviceView(C.Structure):
    _fields_ = ([(n, C.c_int) for n in ("num_envs", "nq", "nv", "gc_stride", "gv_stride")] +
                [(n, C.c_void_p) for n in ("gc", "gv", "tau_ff", "ptarget", "vtarget", "ncontacts", "contacts")])


_P, _I, _F, _S = C.c_void_p, C.c_int, C.c_float, C.c_char_p

# Every function include/rsb.h declares: symbol -> argtypes, or (argtypes, restype) where it does not return int
SIGNATURES = {
    "rsb_last_error": ([], _S),
    "rsb_version": [],
    "rsb_params_default": [C.POINTER(Params)],
    "rsb_model_create_from_urdf": [_S, C.POINTER(_P)],
    "rsb_model_load": [_S, _P],
    "rsb_model_save": [_P, _S],
    "rsb_model_collision_index": [_P, _S],
    "rsb_model_destroy": [_P],
    "rsb_model_dims": [_P] + [C.POINTER(_I)] * 5,
    "rsb_model_get_tables": [_P, C.POINTER(ModelTables)],
    "rsb_model_body_index": [_P, _S],
    "rsb_model_body_name": ([_P, _I], _S),
    "rsb_model_joint_name": ([_P, _I], _S),
    "rsb_model_frame_index": [_P, _S],
    "rsb_model_frame": [_P, _I, C.POINTER(_I), _P, _P],
    "rsb_batch_create": [_P, _I, _I, C.POINTER(_P)],
    "rsb_batch_destroy": [_P],
    "rsb_batch_set_stream": [_P, _P],
    "rsb_batch_sync": [_P],
    "rsb_batch_num_envs": [_P],
    "rsb_batch_set_ground": [_P, _F],
    "rsb_batch_set_heightmap": [_P, _I, _I, _F, _F, _F, _F, _P],
    "rsb_batch_set_heightmaps": [_P, _I, _I, _I, _F, _F, _F, _F, _P, _P],
    "rsb_batch_set_heightmap_index": [_P, _P, _I, _I, _I],
    "rsb_batch_update_heightmaps": [_P, _I, _I, _P, _I],
    "rsb_batch_clear_terrain": [_P],
    "rsb_batch_set_collision_friction": [_P, _I, _F],
    "rsb_batch_set_self_collision": [_P, _P, _I, _P],
    "rsb_batch_set_params": [_P, C.POINTER(Params)],
    "rsb_batch_get_params": [_P, C.POINTER(Params)],
    "rsb_batch_set_state": [_P, _P, _P, _I, _I, _I],
    "rsb_batch_get_state": [_P, _P, _P, _I, _I, _I],
    "rsb_batch_set_pd_target": [_P, _P, _P, _I, _I, _I],
    "rsb_batch_set_pd_gains": [_P, _P, _P],
    "rsb_batch_set_generalized_force": [_P, _P, _I, _I, _I],
    "rsb_batch_get_generalized_force": [_P, _P, _I, _I, _I],
    "rsb_batch_set_control_mode": [_P, _I],
    "rsb_batch_set_external_wrench": [_P, _I, _P, _P, _P, _I, _I, _I],
    "rsb_batch_bind_pd_target": [_P, _P, _I],
    "rsb_batch_set_body_inertia": [_P, _P, _I, _I, _I],
    "rsb_batch_clear_body_inertia": [_P],
    "rsb_batch_set_contact_friction": [_P, _P, _I, _I, _I],
    "rsb_batch_clear_contact_friction": [_P],
    "rsb_batch_set_actuator_params": [_P, _P, _I, _I, _I],
    "rsb_batch_clear_actuator_params": [_P],
    "rsb_batch_set_actuator_network": [_P, _P, _I, _I, _I, _I, _P],
    "rsb_batch_set_actuator_history": [_P, _P, _I, _I, _I],
    "rsb_batch_get_actuator_history": [_P, _P, _I, _I, _I],
    "rsb_batch_set_actuator_lstm": [_P, _P, _I, _I, _I, _P],
    "rsb_batch_set_actuation_delay": [_P, _P, _I, _I, _I],
    "rsb_batch_clear_actuation_delay": [_P],
    "rsb_batch_integrate1": [_P],
    "rsb_batch_integrate2": [_P],
    "rsb_batch_integrate": [_P, _I],
    "rsb_batch_get_mass_matrix": [_P, _I, _I, _P, _I],
    "rsb_batch_get_nonlinearities": [_P, _I, _I, _P, _I],
    "rsb_batch_get_body_poses": [_P, _I, _I, _P, _P, _I],
    "rsb_batch_get_contacts": [_P, _P, _P, _I, _I, _I],
    "rsb_batch_get_contact_points": [_P, _P, _I, _I, _I],
    "rsb_batch_get_solver_iterations": [_P, _P, _I, _I, _I],
    "rsb_batch_get_diverged": [_P, _P, _I, _I, _I],
    "rsb_batch_get_solver_residual": [_P, _P, _I, _I, _I],
    "rsb_batch_get_solver_status": [_P, _P, _I, _I, _I],
    "rsb_batch_update_kinematics": [_P],
    "rsb_batch_device_ptrs": [_P, C.POINTER(DeviceView)],
    "rsb_batch_launch_count": ([_P], C.c_int64),
    "rsb_batch_set_frames": [_P, _P, _P, _P, _I],
    "rsb_batch_get_frame_states": [_P, _I, _I] + [_P] * 4 + [_I],
    "rsb_batch_get_frame_jacobians": [_P, _I, _I, _P, _I],
    "rsb_batch_set_contact_bodies": [_P, _P, _I],
    "rsb_batch_get_body_contact_forces": [_P, _I, _I, _P, _P, _I],
    "rsb_batch_set_imus": [_P, _P, _P, _P, _I],
    "rsb_batch_get_imu_readings": [_P, _I, _I, _P, _P, _I],
    "rsb_batch_set_height_scan": [_P, _P, _P, _I, _I],
    "rsb_batch_get_height_scan": [_P, _I, _I, _P, _P, _I],
    "rsb_batch_set_rays": [_P, _P, _P, _P, _I, _F, _I],
    "rsb_batch_get_ray_casts": [_P, _I, _I, _P, _P, _I],
    "rsb_batch_ob_dim": [_P],
    "rsb_batch_observe": [_P, _P, _I, _I, _I],
    "rsb_batch_control_step": [_P, _P, _P, _I, _I, _P, _I],
    "rsb_batch_gym_configure": [_P] + [_P] * 5 + [_I, _F, _F, _F],
    "rsb_batch_gym_reset": [_P],
    "rsb_batch_gym_step": [_P, _P, _I, _I, _P, _P, _P, _I],
    "rsb_peer_buffer_create": [_I, C.c_size_t, C.POINTER(_P), _P],
    "rsb_peer_buffer_open": [_I, _P, C.POINTER(_P)],
    "rsb_peer_buffer_close": [_P],
    "rsb_peer_buffer_destroy": [_P],
    "rsb_batch_set_observation_peers": [_P, _I, _I, _P, _P],
    "rsb_batch_wait_observation_peers": [_P, C.POINTER(_I)],
    "rsb_comm_init": [C.POINTER(_P), _I, C.POINTER(_P)],
    "rsb_comm_allgather_obs": [_P, C.POINTER(_P)],
    "rsb_comm_destroy": [_P],
    "rsb_terrain_generate": [C.POINTER(TerrainProperties), _P],
    "rsb_heightmap_read_text": [_S, _P, _P, _P, _P, _P, _I],
    "rsb_heightmap_read_png": [_S, C.c_double, C.c_double, _P, _P, _P, _I],
}
EXPORTED = list(SIGNATURES)

_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            # not a fallback: the same CUDA library, compiled on the spot when the prebuilt one did not travel
            import subprocess
            try:
                subprocess.check_call(["make", "-C", os.path.join(_HERE, "csrc")], stdout=subprocess.DEVNULL)
            except Exception as e:
                raise RsbError(f"{LIB_PATH} is missing and could not be built ({e}): run `python -c 'import __graft_entry__ as g; g.build()'` (no CPU fallback exists)")
        L = C.CDLL(LIB_PATH)
        for name, sig in SIGNATURES.items():
            if not hasattr(L, name):
                if LIB_PATH == _OTHER_BUILD:
                    continue          # an older build: calling what it lacks raises AttributeError
                raise RsbError(f"{LIB_PATH} does not export {name}: rebuild it")
            f = getattr(L, name)
            f.argtypes, f.restype = sig if isinstance(sig, tuple) else (sig, C.c_int)
        _lib = L
    return _lib


def _ck(rc):
    if rc < 0:
        raise RsbError(lib().rsb_last_error().decode())
    return rc


def _ptr(a):
    """numpy array -> host pointer; torch CUDA tensor -> device pointer; int -> raw pointer."""
    if a is None:
        return None, HOST
    if isinstance(a, np.ndarray):
        assert a.flags.c_contiguous
        return a.ctypes.data_as(C.c_void_p), HOST
    if hasattr(a, "data_ptr"):
        assert a.is_contiguous()
        return C.c_void_p(a.data_ptr()), (DEVICE if a.is_cuda else HOST)
    raise TypeError(type(a))


def _network_layers(layers):
    """[(W, b)] float32 numpy pairs of an actuator network given as such pairs or as a torch.nn.Sequential of Linear and Softsign"""
    if hasattr(layers, "named_children") and hasattr(layers, "__iter__"):
        mods = list(layers)
        kinds = [type(m).__name__ for m in mods]
        ok = len(mods) % 2 == 1 and all(k == ("Linear" if i % 2 == 0 else "Softsign") for i, k in enumerate(kinds))
        if not ok:
            raise ValueError(f"actuator network: a Sequential must be Linear, Softsign, ..., Linear; got {kinds}")
        pairs = []
        for m in mods[::2]:
            if m.bias is None:
                raise ValueError("actuator network: every Linear needs a bias")
            pairs.append((m.weight.detach().cpu().numpy(), m.bias.detach().cpu().numpy()))
        layers = pairs
    out = []
    for p in layers:
        if len(p) != 2:
            raise ValueError("actuator network: layers must be (W, b) pairs")
        out.append((np.asarray(p[0], np.float32), np.asarray(p[1], np.float32)))
    return out


ACTNET_MAX_LAYERS, ACTNET_MAX_WIDTH = 4, 32     # RSB_ACTNET_MAX_LAYERS, RSB_ACTNET_MAX_WIDTH of include/rsb.h


def _lstm_params(lstm, readout):
    """(layers, hidden, float32 parameters in the order of rsb_batch_set_actuator_lstm) of an LSTM actuator network.  lstm: a
    torch.nn.LSTM, or a list of per-layer (weight_ih, weight_hh, bias_ih, bias_hh) arrays in torch order; readout: a
    torch.nn.Linear(hidden, 1) or a (weight [1, hidden], bias [1]) pair"""
    if hasattr(lstm, "all_weights") and hasattr(lstm, "hidden_size"):
        if lstm.input_size != 2:
            raise ValueError(f"set_actuator_lstm: the LSTM's input_size must be 2 (position error, velocity), got {lstm.input_size}")
        if not lstm.bias:
            raise ValueError("set_actuator_lstm: the LSTM needs its biases (bias=True)")
        if lstm.bidirectional:
            raise ValueError("set_actuator_lstm: a bidirectional LSTM cannot run one step at a time")
        if getattr(lstm, "proj_size", 0) > 0:
            raise ValueError("set_actuator_lstm: a projected LSTM (proj_size > 0) is not supported")
        sd = lstm.state_dict()
        lstm = [tuple(sd[f"{k}_l{l}"].detach().cpu().numpy() for k in ("weight_ih", "weight_hh", "bias_ih", "bias_hh"))
                for l in range(lstm.num_layers)]
    layers = [tuple(np.asarray(a, np.float32) for a in p) for p in lstm]
    if any(len(p) != 4 for p in layers):
        raise ValueError("set_actuator_lstm: every layer needs (weight_ih, weight_hh, bias_ih, bias_hh)")
    if not 1 <= len(layers) <= ACTNET_MAX_LAYERS:
        raise ValueError(f"set_actuator_lstm: {len(layers)} layers outside [1, {ACTNET_MAX_LAYERS}]")
    hidden = layers[0][1].shape[1] if layers[0][1].ndim == 2 else -1
    if not 1 <= hidden <= ACTNET_MAX_WIDTH:
        raise ValueError(f"set_actuator_lstm: hidden size {hidden} outside [1, {ACTNET_MAX_WIDTH}]")
    for l, (wih, whh, bih, bhh) in enumerate(layers):
        nin = 2 if l == 0 else hidden
        want = ((4 * hidden, nin), (4 * hidden, hidden), (4 * hidden,), (4 * hidden,))
        got = (wih.shape, whh.shape, bih.shape, bhh.shape)
        if got != want:
            raise ValueError(f"set_actuator_lstm: layer {l}: need weight_ih, weight_hh, bias_ih, bias_hh of shapes {want}, got {got}")
    if hasattr(readout, "weight") and hasattr(readout, "in_features"):
        if readout.bias is None:
            raise ValueError("set_actuator_lstm: the read-out Linear needs a bias")
        readout = (readout.weight.detach().cpu().numpy(), readout.bias.detach().cpu().numpy())
    if len(readout) != 2:
        raise ValueError("set_actuator_lstm: the read-out must be a Linear or a (weight, bias) pair")
    wo, bo = (np.asarray(a, np.float32) for a in readout)
    if wo.shape != (1, hidden) or bo.shape != (1,):
        raise ValueError(f"set_actuator_lstm: the read-out needs weight (1, {hidden}) and bias (1,), got {wo.shape} and {bo.shape}")
    params = np.concatenate([a.ravel() for p in layers for a in p] + [wo.ravel(), bo.ravel()])
    return len(layers), hidden, np.ascontiguousarray(params, np.float32)


class Model:
    def __init__(self, path_or_xml, cache=False):
        """URDF path / XML text, or (cache=True) a binary model cache written by Model.save()"""
        h = C.c_void_p()
        if cache:
            _ck(lib().rsb_model_load(path_or_xml.encode(), C.byref(h)))
        else:
            _ck(lib().rsb_model_create_from_urdf(path_or_xml.encode(), C.byref(h)))
        self.h = h
        d = [C.c_int() for _ in range(5)]
        _ck(lib().rsb_model_dims(h, *[C.byref(x) for x in d]))
        self.nq, self.nv, self.nb, self.ncoll, self.npts = [x.value for x in d]

    def collision_index(self, name):
        return _ck(lib().rsb_model_collision_index(self.h, name.encode()))

    def save(self, path):
        _ck(lib().rsb_model_save(self.h, path.encode()))

    def __del__(self):
        if getattr(self, "h", None) and lib is not None and _lib is not None:     # at interpreter shutdown the module globals may be gone already
            _lib.rsb_model_destroy(self.h)
            self.h = None

    def tables(self):
        t = ModelTables()
        _ck(lib().rsb_model_get_tables(self.h, C.byref(t)))
        nb, nc, npt = t.nb, t.ncoll, t.npts
        arr = lambda p, n, dt: np.ctypeslib.as_array(p, shape=(n,)).astype(dt).copy() if n > 0 else np.zeros(0, dt)
        out = dict(nb=nb, nq=t.nq, nv=t.nv, floating=t.floating, ncoll=nc, npts=npt)
        for k in ("parent", "jtype", "qidx", "vidx", "depth"):
            out[k] = arr(getattr(t, k), nb, np.int32)
        for k, w in (("jpos", 3), ("jrot", 9), ("axis", 3), ("mass", 1), ("com", 3), ("inertia", 6), ("jlimit", 2)):
            a = arr(getattr(t, k), nb * w, np.float64)
            out[k] = a.reshape(nb, w) if w > 1 else a
        for k in ("cbody", "ctype"):
            out[k] = arr(getattr(t, k), nc, np.int32)
        for k, w in (("csize", 3), ("cpos", 3), ("crot", 9)):
            out[k] = arr(getattr(t, k), nc * w, np.float64).reshape(nc, w)
        for k in ("pt_body", "pt_coll", "pt_feat"):
            out[k] = arr(getattr(t, k), npt, np.int32)
        out["pt_pos"] = arr(t.pt_pos, npt * 3, np.float64).reshape(npt, 3)
        out["pt_rad"] = arr(t.pt_rad, npt, np.float64)
        out["pt_type"] = arr(t.pt_type, npt, np.int32)
        out["pt_pos2"] = arr(t.pt_pos2, npt * 3, np.float64).reshape(npt, 3)
        out["jeffort"] = arr(t.jeffort, nb, np.float64)
        out["body_names"] = [lib().rsb_model_body_name(self.h, i).decode() for i in range(nb)]
        out["joint_names"] = [lib().rsb_model_joint_name(self.h, i).decode() for i in range(nb)]
        return out

    def body_index(self, name):
        return _ck(lib().rsb_model_body_index(self.h, name.encode()))


class Batch:
    """N environments of one model on one GPU; mirrors World/ArticulatedSystem calls batch-wide."""

    def __init__(self, model, num_envs, device=0):
        self.model = model
        h = C.c_void_p()
        _ck(lib().rsb_batch_create(model.h, num_envs, device, C.byref(h)))
        self.h, self.n, self.nq, self.nv, self.nb = h, num_envs, model.nq, model.nv, model.nb
        self.device, self.nframes, self.ncontact_bodies, self.nscan, self.nimus, self.nrays = device, 0, 0, 0, 0, 0
        self.hm_shape = None                 # (ys, xs) of the height map(s) set through this object
        self.an_shape = None                 # (listed dofs, history) of the actuator network set through this object
        self.lstm_shape = None               # (listed dofs, layers, hidden) of the LSTM actuator network set through this object

    def __del__(self):
        if getattr(self, "h", None) and lib is not None and _lib is not None:
            _lib.rsb_batch_destroy(self.h)
            self.h = None

    def _count(self, env_begin, env_count):
        """environments in [env_begin, env_begin + env_count); env_count None: to the end of the batch"""
        return self.n - env_begin if env_count is None else env_count

    def _read(self, fn, row_shape, dtype, env_begin, env_count, range_first=False):
        """a getter that fills host rows [n, *row_shape]: fn(batch, out, env_begin, n, HOST), or fn(batch, env_begin, n, out, HOST)
        with range_first"""
        n = self._count(env_begin, env_count)
        out = np.empty((n,) + row_shape, dtype)
        p = out.ctypes.data_as(C.c_void_p)
        _ck(fn(self.h, env_begin, n, p, HOST) if range_first else fn(self.h, p, env_begin, n, HOST))
        return out

    # world set-up
    def set_stream(self, stream_ptr):
        _ck(lib().rsb_batch_set_stream(self.h, C.c_void_p(stream_ptr)))

    def sync(self):
        _ck(lib().rsb_batch_sync(self.h))

    def set_ground(self, z=0.0):
        _ck(lib().rsb_batch_set_ground(self.h, z))

    def set_heightmap(self, xs, ys, x_size, y_size, cx, cy, heights):
        hh = np.ascontiguousarray(heights, dtype=np.float32).reshape(-1)
        assert hh.size == xs * ys
        _ck(lib().rsb_batch_set_heightmap(self.h, xs, ys, x_size, y_size, cx, cy, hh.ctypes.data_as(C.c_void_p)))
        self.hm_shape = (ys, xs)

    def set_heightmaps(self, x_size, y_size, cx, cy, heights, map_of_env):
        """terrain atlas: heights [count, ys, xs] float32, map_of_env [n] int32 -> one height map per environment"""
        h = np.ascontiguousarray(heights, np.float32)
        count, ys, xs = h.shape
        m = np.ascontiguousarray(map_of_env, np.int32)
        assert m.shape == (self.n,)
        _ck(lib().rsb_batch_set_heightmaps(self.h, count, xs, ys, x_size, y_size, cx, cy, h.ctypes.data_as(C.c_void_p), m.ctypes.data_as(C.c_void_p)))
        self.hm_shape = (ys, xs)

    def set_heightmap_index(self, map_of_env, env_begin=0, env_count=None):
        """terrain curriculum: environments [env_begin, env_begin + n) collide with the atlas maps map_of_env [n] (numpy int32) from the
        next launch on; no map is uploaded.  env_count defaults to len(map_of_env).  A refused call changes nothing."""
        m = np.ascontiguousarray(map_of_env, np.int32).reshape(-1)
        n = len(m) if env_count is None else env_count
        if n > len(m):
            raise ValueError(f"set_heightmap_index: {n} environments, {len(m)} indices")
        _ck(lib().rsb_batch_set_heightmap_index(self.h, m.ctypes.data_as(C.c_void_p), env_begin, n, HOST))

    def set_heightmap_index_from(self, map_of_env, env_begin=0):
        """set_heightmap_index() from a contiguous int32 torch tensor [n] on the batch's device, checked there"""
        n = map_of_env.shape[0] if hasattr(map_of_env, "shape") and len(map_of_env.shape) > 0 else -1
        _ck(lib().rsb_batch_set_heightmap_index(self.h, self._device_out(map_of_env, (n,), "map_of_env", "int32"), env_begin, n, DEVICE))

    def update_heightmaps(self, first, heights):
        """overwrite maps first .. first + count - 1 of the terrain in place with heights [count, ys, xs] (numpy float32; [ys, xs]: one
        map), the map shape being that of the terrain set by set_heightmap / set_heightmaps.  Every height must be finite; a refused
        call changes nothing."""
        if self.hm_shape is None:
            raise ValueError("update_heightmaps: no height map set through this object")
        h = np.ascontiguousarray(heights, np.float32)
        if h.ndim == 2:
            h = h[None]
        if h.ndim != 3 or h.shape[1:] != self.hm_shape:
            raise ValueError(f"update_heightmaps: need heights [count, {self.hm_shape[0]}, {self.hm_shape[1]}], got shape {h.shape}")
        _ck(lib().rsb_batch_update_heightmaps(self.h, first, h.shape[0], h.ctypes.data_as(C.c_void_p), HOST))

    def update_heightmaps_from(self, first, heights):
        """update_heightmaps() from a contiguous float32 torch tensor [count, ys, xs] on the batch's device, checked there; the map
        shape is that of the terrain set by set_heightmap / set_heightmaps"""
        if self.hm_shape is None:
            raise ValueError("update_heightmaps_from: no height map set through this object")
        n = heights.shape[0] if hasattr(heights, "shape") and len(heights.shape) > 0 else -1
        _ck(lib().rsb_batch_update_heightmaps(self.h, first, n, self._device_out(heights, (n,) + self.hm_shape, "heights"), DEVICE))

    def clear_terrain(self):
        _ck(lib().rsb_batch_clear_terrain(self.h))

    def set_collision_friction(self, collision_body, mu):
        _ck(lib().rsb_batch_set_collision_friction(self.h, collision_body, mu))

    def set_self_collision(self, pairs, mu=None):
        """enable self-collision between pairs of collision bodies ([n, 2] indices, or collision-body names "LINK/k"); mu [n] per-pair
        friction (None: the default material).  An empty list clears the pairs.  Pair j's contacts have candidate index npts + j and
        pair_index -1 - second body."""
        rows = [[self.model.collision_index(c) if isinstance(c, str) else int(c) for c in p] for p in pairs]
        pp = np.ascontiguousarray(np.asarray(rows, np.int32).reshape(-1, 2))
        m = None if mu is None else np.ascontiguousarray(np.broadcast_to(np.asarray(mu, np.float32), (len(pp),)))
        _ck(lib().rsb_batch_set_self_collision(self.h, pp.ctypes.data_as(C.c_void_p), len(pp),
                                               None if m is None else m.ctypes.data_as(C.c_void_p)))

    def get_params(self):
        p = Params()
        _ck(lib().rsb_batch_get_params(self.h, C.byref(p)))
        return p

    def set_params(self, **kw):
        p = self.get_params()
        for k, v in kw.items():
            if k == "gravity":
                p.gravity[0], p.gravity[1], p.gravity[2] = v
            else:
                setattr(p, k, v)
        _ck(lib().rsb_batch_set_params(self.h, C.byref(p)))

    # state / actuation
    def set_state(self, gc=None, gv=None, env_begin=0, env_count=None):
        n = self._count(env_begin, env_count)
        pg, w1 = _ptr(gc); pv, w2 = _ptr(gv)
        _ck(lib().rsb_batch_set_state(self.h, pg, pv, env_begin, n, w1 if gc is not None else w2))

    def get_state(self, env_begin=0, env_count=None):
        n = self._count(env_begin, env_count)
        gc, gv = np.empty((n, self.nq), np.float32), np.empty((n, self.nv), np.float32)
        _ck(lib().rsb_batch_get_state(self.h, gc.ctypes.data_as(C.c_void_p), gv.ctypes.data_as(C.c_void_p), env_begin, n, HOST))
        return gc, gv

    def get_state_into(self, gc, gv, env_begin=0, env_count=None):
        n = self._count(env_begin, env_count)
        pg, w1 = _ptr(gc); pv, w2 = _ptr(gv)
        _ck(lib().rsb_batch_get_state(self.h, pg, pv, env_begin, n, w1 if gc is not None else w2))

    def set_pd_gains(self, kp, kd):
        kp = np.ascontiguousarray(np.broadcast_to(np.asarray(kp, np.float32), (self.nv,)))
        kd = np.ascontiguousarray(np.broadcast_to(np.asarray(kd, np.float32), (self.nv,)))
        _ck(lib().rsb_batch_set_pd_gains(self.h, kp.ctypes.data_as(C.c_void_p), kd.ctypes.data_as(C.c_void_p)))

    def set_pd_target(self, ptarget=None, vtarget=None, env_begin=0, env_count=None):
        n = self._count(env_begin, env_count)
        pp, w1 = _ptr(ptarget); pv, w2 = _ptr(vtarget)
        _ck(lib().rsb_batch_set_pd_target(self.h, pp, pv, env_begin, n, w1 if ptarget is not None else w2))

    def bind_pd_target(self, ptarget_dev, row_stride=None):
        """zero-copy: the kernel reads PD-target rows from this device tensor (None unbinds)"""
        if ptarget_dev is None:
            _ck(lib().rsb_batch_bind_pd_target(self.h, None, 0)); return
        assert ptarget_dev.is_cuda and ptarget_dev.is_contiguous()
        self._bound = ptarget_dev        # keep alive
        _ck(lib().rsb_batch_bind_pd_target(self.h, C.c_void_p(ptarget_dev.data_ptr()), row_stride or ptarget_dev.shape[-1]))

    def set_generalized_force(self, tau, env_begin=0, env_count=None):
        n = self._count(env_begin, env_count)
        p, w = _ptr(tau)
        _ck(lib().rsb_batch_set_generalized_force(self.h, p, env_begin, n, w))

    def generalized_force(self, env_begin=0, env_count=None):
        return self._read(lib().rsb_batch_get_generalized_force, (self.nv,), np.float32, env_begin, env_count)

    def set_control_mode(self, mode):
        _ck(lib().rsb_batch_set_control_mode(self.h, mode))

    # hot path
    def integrate1(self):
        _ck(lib().rsb_batch_integrate1(self.h))

    def integrate2(self):
        _ck(lib().rsb_batch_integrate2(self.h))

    def integrate(self, substeps=1):
        _ck(lib().rsb_batch_integrate(self.h, substeps))

    # read-backs
    def mass_matrix(self, env_begin=0, env_count=None):
        return self._read(lib().rsb_batch_get_mass_matrix, (self.nv, self.nv), np.float32, env_begin, env_count, range_first=True)

    def nonlinearities(self, env_begin=0, env_count=None):
        return self._read(lib().rsb_batch_get_nonlinearities, (self.nv,), np.float32, env_begin, env_count, range_first=True)

    def body_poses(self, env_begin=0, env_count=None):
        n = self._count(env_begin, env_count)
        R, p = np.empty((n, self.nb, 3, 3), np.float32), np.empty((n, self.nb, 3), np.float32)
        _ck(lib().rsb_batch_get_body_poses(self.h, env_begin, n, R.ctypes.data_as(C.c_void_p), p.ctypes.data_as(C.c_void_p), HOST))
        return R, p

    def contacts(self, env_begin=0, env_count=None):
        n = self._count(env_begin, env_count)
        out = np.empty((n, KMAX), CONTACT_DTYPE)
        cnt = np.empty(n, np.int32)
        _ck(lib().rsb_batch_get_contacts(self.h, out.ctypes.data_as(C.c_void_p), cnt.ctypes.data_as(C.c_void_p), env_begin, n, HOST))
        return out, cnt

    def contact_points(self, env_begin=0, env_count=None):
        return self._read(lib().rsb_batch_get_contact_points, (KMAX,), np.int32, env_begin, env_count)

    def solver_iterations(self, env_begin=0, env_count=None):
        return self._read(lib().rsb_batch_get_solver_iterations, (), np.int32, env_begin, env_count)

    def solver_residual(self, env_begin=0, env_count=None):
        """largest impulse update of the last Gauss-Seidel sweep of every environment (< threshold: converged)"""
        return self._read(lib().rsb_batch_get_solver_residual, (), np.float32, env_begin, env_count)

    def solver_status(self, env_begin=0, env_count=None):
        """0 converged, 1 converged on the compliant contact set (stall_reg), 2 stalled, 3 max_iter -- of the last solve"""
        return self._read(lib().rsb_batch_get_solver_status, (), np.int32, env_begin, env_count)

    def update_kinematics(self):
        _ck(lib().rsb_batch_update_kinematics(self.h))

    # frame kinematics
    def set_frames(self, body, pos, rot=None):
        """frames rigidly attached to bodies, shared by all environments: body [F] indices, pos [F, 3] and rot [F, 3, 3] (None:
        identity) in the body frame.  An empty list clears them; a refused call keeps the frames set before."""
        bd = np.ascontiguousarray(body, np.int32).reshape(-1)
        p = np.ascontiguousarray(pos, np.float32).reshape(-1, 3)
        r = None if rot is None else np.ascontiguousarray(rot, np.float32).reshape(-1, 9)
        if len(p) != len(bd) or (r is not None and len(r) != len(bd)):
            raise ValueError(f"set_frames: {len(bd)} bodies, {len(p)} positions, {'no' if r is None else len(r)} rotations")
        _ck(lib().rsb_batch_set_frames(self.h, bd.ctypes.data_as(C.c_void_p), p.ctypes.data_as(C.c_void_p),
                                       None if r is None else r.ctypes.data_as(C.c_void_p), len(bd)))
        self.nframes = len(bd)

    def set_frames_by_name(self, names):
        """the URDF link frames (or joint names) `names`, as rsb_model_frame gives them"""
        L = lib()
        body, pos, rot = [], np.zeros((len(names), 3)), np.zeros((len(names), 9))
        for k, name in enumerate(names):
            f, b = _ck(L.rsb_model_frame_index(self.model.h, name.encode())), C.c_int()
            _ck(L.rsb_model_frame(self.model.h, f, C.byref(b), pos[k].ctypes.data_as(C.c_void_p), rot[k].ctypes.data_as(C.c_void_p)))
            body.append(b.value)
        self.set_frames(body, pos, rot)

    def frame_states(self, env_begin=0, env_count=None):
        """world-frame (pos [n, F, 3], rot [n, F, 3, 3], lin_vel [n, F, 3], ang_vel [n, F, 3]) of the frames at the current state"""
        n = self._count(env_begin, env_count)
        out = (np.empty((n, self.nframes, 3), np.float32), np.empty((n, self.nframes, 3, 3), np.float32),
               np.empty((n, self.nframes, 3), np.float32), np.empty((n, self.nframes, 3), np.float32))
        _ck(lib().rsb_batch_get_frame_states(self.h, env_begin, n, *[a.ctypes.data_as(C.c_void_p) for a in out], HOST))
        return out

    def frame_jacobians(self, env_begin=0, env_count=None):
        """[n, F, 6, nv]: rows 0-2 the frame point's velocity, rows 3-5 its body's angular velocity per unit gv"""
        return self._read(lib().rsb_batch_get_frame_jacobians, (self.nframes, 6, self.nv), np.float32, env_begin, env_count, range_first=True)

    def _device_out(self, t, shape, name, dtype="float32"):
        """device address of a caller-given output tensor (None: skip it)"""
        if t is None:
            return None
        import torch
        if not isinstance(t, torch.Tensor) or not t.is_cuda or t.device.index != self.device:
            raise ValueError(f"{name}: need a torch tensor on cuda:{self.device}")
        if t.dtype != getattr(torch, dtype) or tuple(t.shape) != shape or not t.is_contiguous():
            raise ValueError(f"{name}: need a contiguous {dtype} tensor of shape {shape}, got {t.dtype} {tuple(t.shape)}")
        return C.c_void_p(t.data_ptr())

    def frame_states_into(self, pos=None, rot=None, lin_vel=None, ang_vel=None, env_begin=0, env_count=None):
        """frame_states() written into torch CUDA tensors (None skips one), in the batch's stream order"""
        n, F = self._count(env_begin, env_count), self.nframes
        ptrs = [self._device_out(pos, (n, F, 3), "pos"), self._device_out(rot, (n, F, 3, 3), "rot"),
                self._device_out(lin_vel, (n, F, 3), "lin_vel"), self._device_out(ang_vel, (n, F, 3), "ang_vel")]
        _ck(lib().rsb_batch_get_frame_states(self.h, env_begin, n, *ptrs, DEVICE))

    def frame_jacobians_into(self, jac, env_begin=0, env_count=None):
        """frame_jacobians() written into a torch CUDA tensor [n, F, 6, nv], in the batch's stream order"""
        n = self._count(env_begin, env_count)
        _ck(lib().rsb_batch_get_frame_jacobians(self.h, env_begin, n, self._device_out(jac, (n, self.nframes, 6, self.nv), "jac"), DEVICE))

    # contact forces per body over a whole launch
    def set_contact_bodies(self, bodies):
        """bodies [S] (at most 32 body indices, shared by all environments) whose mean contact force and sub-steps in contact every
        launch that advances the state gathers over all its sub-steps.  An empty list clears them; a refused call keeps the list
        set before."""
        bd = np.ascontiguousarray(bodies, np.int32).reshape(-1)
        _ck(lib().rsb_batch_set_contact_bodies(self.h, bd.ctypes.data_as(C.c_void_p), len(bd)))
        self.ncontact_bodies = len(bd)

    def set_contact_bodies_by_name(self, names):
        self.set_contact_bodies([self.model.body_index(n) for n in names])

    def body_contact_forces(self, env_begin=0, env_count=None):
        """(force [n, S, 3] float32: world-frame mean contact force on each listed body over the last advancing launch;
        steps [n, S] int32: its sub-steps in which the body had a contact)"""
        n = self._count(env_begin, env_count)
        force, steps = np.empty((n, self.ncontact_bodies, 3), np.float32), np.empty((n, self.ncontact_bodies), np.int32)
        _ck(lib().rsb_batch_get_body_contact_forces(self.h, env_begin, n, force.ctypes.data_as(C.c_void_p), steps.ctypes.data_as(C.c_void_p), HOST))
        return force, steps

    def body_contact_forces_into(self, force=None, steps=None, env_begin=0, env_count=None):
        """body_contact_forces() copied into torch CUDA tensors (float32 / int32; None skips one), in the batch's stream order: no launch"""
        n, S = self._count(env_begin, env_count), self.ncontact_bodies
        _ck(lib().rsb_batch_get_body_contact_forces(self.h, env_begin, n, self._device_out(force, (n, S, 3), "force"),
                                                    self._device_out(steps, (n, S), "steps", "int32"), DEVICE))

    # IMU readings over a whole launch
    def set_imus(self, body, pos, rot=None):
        """IMU sensors shared by all environments (at most 8): sensor k hangs on body[k] at pos[k] [3] with orientation rot[k] [3, 3]
        (None: identity), both in the body frame.  Every launch that advances the state gathers their mean specific force and angular
        rate over all its sub-steps.  An empty list clears them; a refused call keeps the sensors set before."""
        bd = np.ascontiguousarray(body, np.int32).reshape(-1)
        p = np.ascontiguousarray(pos, np.float32).reshape(-1, 3)
        r = None if rot is None else np.ascontiguousarray(rot, np.float32).reshape(-1, 9)
        if len(p) != len(bd) or (r is not None and len(r) != len(bd)):
            raise ValueError(f"set_imus: {len(bd)} bodies, {len(p)} positions, {'no' if r is None else len(r)} rotations")
        _ck(lib().rsb_batch_set_imus(self.h, bd.ctypes.data_as(C.c_void_p), p.ctypes.data_as(C.c_void_p),
                                     None if r is None else r.ctypes.data_as(C.c_void_p), len(bd)))
        self.nimus = len(bd)

    def set_imus_by_frame(self, names):
        """IMUs at the URDF link frames (or joint names) `names`, as rsb_model_frame gives them"""
        L = lib()
        body, pos, rot = [], np.zeros((len(names), 3)), np.zeros((len(names), 9))
        for k, name in enumerate(names):
            f, b = _ck(L.rsb_model_frame_index(self.model.h, name.encode())), C.c_int()
            _ck(L.rsb_model_frame(self.model.h, f, C.byref(b), pos[k].ctypes.data_as(C.c_void_p), rot[k].ctypes.data_as(C.c_void_p)))
            body.append(b.value)
        self.set_imus(body, pos, rot)

    def imu_readings(self, env_begin=0, env_count=None):
        """(lin_acc [n, I, 3], ang_vel [n, I, 3]) float32 in the sensor frames: mean specific force [m/s^2] and angular rate [rad/s] over
        the last launch that advanced the state"""
        n = self._count(env_begin, env_count)
        lin, ang = np.empty((n, self.nimus, 3), np.float32), np.empty((n, self.nimus, 3), np.float32)
        _ck(lib().rsb_batch_get_imu_readings(self.h, env_begin, n, lin.ctypes.data_as(C.c_void_p), ang.ctypes.data_as(C.c_void_p), HOST))
        return lin, ang

    def imu_readings_into(self, lin_acc=None, ang_vel=None, env_begin=0, env_count=None):
        """imu_readings() copied into torch CUDA float32 tensors [n, I, 3] (None skips one), in the batch's stream order: no launch"""
        n, I = self._count(env_begin, env_count), self.nimus
        _ck(lib().rsb_batch_get_imu_readings(self.h, env_begin, n, self._device_out(lin_acc, (n, I, 3), "lin_acc"),
                                             self._device_out(ang_vel, (n, I, 3), "ang_vel"), DEVICE))

    # terrain height scans
    def set_height_scan(self, body, xy, align="yaw"):
        """sample points shared by all environments: point i hangs on body[i] at the horizontal offset xy[i] = (dx, dy); align "yaw"
        turns the offsets with the body's heading, "world" keeps them along the world axes.  An empty list clears them; a refused
        call keeps the points set before."""
        modes = {"yaw": SCAN_YAW, "world": SCAN_WORLD}
        if align not in modes:
            raise ValueError(f"set_height_scan: align must be 'yaw' or 'world', got {align!r}")
        bd = np.ascontiguousarray(body, np.int32).reshape(-1)
        p = np.ascontiguousarray(xy, np.float32).reshape(-1, 2)
        if len(p) != len(bd):
            raise ValueError(f"set_height_scan: {len(bd)} bodies, {len(p)} offsets")
        _ck(lib().rsb_batch_set_height_scan(self.h, bd.ctypes.data_as(C.c_void_p), p.ctypes.data_as(C.c_void_p), len(bd), modes[align]))
        self.nscan = len(bd)

    def set_height_scan_by_name(self, names, xy, align="yaw"):
        """set_height_scan() with the bodies given by link name (rsb_model_body_index: a merged link names its body)"""
        self.set_height_scan([self.model.body_index(n) for n in names], xy, align)

    def height_scan(self, env_begin=0, env_count=None):
        """(height [n, P]: world z of the collision surface under every sample, xy [n, P, 2]: the world sample locations) at the
        current state"""
        n = self._count(env_begin, env_count)
        h, xy = np.empty((n, self.nscan), np.float32), np.empty((n, self.nscan, 2), np.float32)
        _ck(lib().rsb_batch_get_height_scan(self.h, env_begin, n, h.ctypes.data_as(C.c_void_p), xy.ctypes.data_as(C.c_void_p), HOST))
        return h, xy

    def height_scan_into(self, height=None, xy=None, env_begin=0, env_count=None):
        """height_scan() written into torch CUDA tensors [n, P] / [n, P, 2] (None skips one), in the batch's stream order"""
        n, P = self._count(env_begin, env_count), self.nscan
        _ck(lib().rsb_batch_get_height_scan(self.h, env_begin, n, self._device_out(height, (n, P), "height"), self._device_out(xy, (n, P, 2), "xy"), DEVICE))

    # ray casts (depth cameras, lidars)
    def set_rays(self, body, origin, dir, max_distance, targets="terrain"):
        """rays shared by all environments: ray i hangs on body[i] with origin[i] [3] and direction dir[i] [3] (any length >= 1e-6,
        normalised here) in the body frame; ray_casts() reports the first hit within max_distance.  targets "terrain" sees the ground
        or height map only, "all" also the robot's own collision bodies (a shape that contains the ray's origin is ignored).  An empty
        list clears them; a refused call keeps the rays set before.  pinhole_rays() gives a camera's directions."""
        modes = {"terrain": RAYS_TERRAIN, "all": RAYS_TERRAIN_AND_ROBOT}
        if targets not in modes:
            raise ValueError(f"set_rays: targets must be 'terrain' or 'all', got {targets!r}")
        bd = np.ascontiguousarray(body, np.int32).reshape(-1)
        o = np.ascontiguousarray(origin, np.float32).reshape(-1, 3)
        d = np.ascontiguousarray(dir, np.float32).reshape(-1, 3)
        if len(o) != len(bd) or len(d) != len(bd):
            raise ValueError(f"set_rays: {len(bd)} bodies, {len(o)} origins, {len(d)} directions")
        _ck(lib().rsb_batch_set_rays(self.h, bd.ctypes.data_as(C.c_void_p), o.ctypes.data_as(C.c_void_p), d.ctypes.data_as(C.c_void_p),
                                     len(bd), max_distance, modes[targets]))
        self.nrays = len(bd)

    def set_rays_by_name(self, names, origin, dir, max_distance, targets="terrain"):
        """set_rays() with the bodies given by link name (rsb_model_body_index: a merged link names its body)"""
        self.set_rays([self.model.body_index(n) for n in names], origin, dir, max_distance, targets)

    def ray_casts(self, env_begin=0, env_count=None):
        """(distance [n, R] float32: the first hit along each ray at the current state, +inf for none, NaN for a diverged
        environment; hit [n, R] int32: RAY_TERRAIN, the collision-body index, or RAY_MISS)"""
        n = self._count(env_begin, env_count)
        dist, hit = np.empty((n, self.nrays), np.float32), np.empty((n, self.nrays), np.int32)
        _ck(lib().rsb_batch_get_ray_casts(self.h, env_begin, n, dist.ctypes.data_as(C.c_void_p), hit.ctypes.data_as(C.c_void_p), HOST))
        return dist, hit

    def ray_casts_into(self, distance=None, hit=None, env_begin=0, env_count=None):
        """ray_casts() written into torch CUDA tensors [n, R] (float32 / int32; None skips one), in the batch's stream order"""
        n, R = self._count(env_begin, env_count), self.nrays
        _ck(lib().rsb_batch_get_ray_casts(self.h, env_begin, n, self._device_out(distance, (n, R), "distance"),
                                          self._device_out(hit, (n, R), "hit", "int32"), DEVICE))

    def diverged(self, env_begin=0, env_count=None):
        return self._read(lib().rsb_batch_get_diverged, (), np.int32, env_begin, env_count)

    def state_tensors(self):
        """zero-copy torch views of the batch state on its GPU: (gc [N, nq], gv [N, nv]) as strided views of the
        padded rows (SURVEY 8f N4).  Writes through these tensors are seen by the next integrate()."""
        import torch
        v = self.device_view()

        class _Raw:
            def __init__(self, ptr, rows, stride):
                self.__cuda_array_interface__ = {"shape": (rows, stride), "typestr": "<f4", "data": (int(ptr), False), "version": 2}

        gc = torch.as_tensor(_Raw(v.gc, v.num_envs, v.gc_stride), device="cuda")[:, :v.nq]
        gv = torch.as_tensor(_Raw(v.gv, v.num_envs, v.gv_stride), device="cuda")[:, :v.nv]
        return gc, gv

    def device_view(self):
        v = DeviceView()
        _ck(lib().rsb_batch_device_ptrs(self.h, C.byref(v)))
        return v

    def launch_count(self):
        return lib().rsb_batch_launch_count(self.h)

    def ob_dim(self):
        return lib().rsb_batch_ob_dim(self.h)

    def set_external_wrench(self, body, force=None, torque=None, point_body=None, env_begin=0, env_count=None):
        """setExternalForce / setExternalTorque: world-frame force / torque rows [n, 3] on `body`, applied at point_body (body
        frame, default = body origin) during the next integrate() / control_step() call only."""
        n = self._count(env_begin, env_count)
        conv = lambda a: a if (a is None or hasattr(a, "data_ptr")) else np.ascontiguousarray(np.broadcast_to(np.asarray(a, np.float32), (n, 3)))
        force, torque = conv(force), conv(torque)
        pf, w1 = _ptr(force); pt_, w2 = _ptr(torque)
        where = w1 if force is not None else w2
        assert force is None or torque is None or w1 == w2
        pp = None if point_body is None else np.ascontiguousarray(point_body, np.float32).ctypes.data_as(C.c_void_p)
        _ck(lib().rsb_batch_set_external_wrench(self.h, int(body), pf, pt_, pp, env_begin, n, where))

    # per-environment inertial parameters
    def model_body_inertia(self):
        """[nb, 10] float32: the model's mass, centre of mass (body frame) and inertia about it (xx xy xz yy yz zz) of every body,
        the rows a batch without per-environment rows integrates and the starting point for set_body_inertia"""
        t = self.model.tables()
        return np.concatenate([t["mass"][:, None], t["com"], t["inertia"]], axis=1).astype(np.float32)

    def set_body_inertia(self, rows, env_begin=0, env_count=None):
        """rows [n, nb, 10] (numpy, see model_body_inertia) for environments [env_begin, env_begin + n); rows None resets env_count
        environments (default: to the end of the batch) to the model's values.  A refused call changes nothing."""
        if rows is None:
            _ck(lib().rsb_batch_set_body_inertia(self.h, None, env_begin, self._count(env_begin, env_count), HOST))
            return
        r = np.ascontiguousarray(rows, np.float32)
        if r.ndim != 3 or r.shape[1:] != (self.nb, 10):
            raise ValueError(f"rows: need shape [n, {self.nb}, 10], got {r.shape}")
        _ck(lib().rsb_batch_set_body_inertia(self.h, r.ctypes.data_as(C.c_void_p), env_begin, r.shape[0], HOST))

    def set_body_inertia_from(self, rows, env_begin=0):
        """set_body_inertia() from a contiguous float32 torch tensor [n, nb, 10] on the batch's device, checked there"""
        n = rows.shape[0] if hasattr(rows, "shape") and len(rows.shape) > 0 else -1
        _ck(lib().rsb_batch_set_body_inertia(self.h, self._device_out(rows, (n, self.nb, 10), "rows"), env_begin, n, DEVICE))

    def clear_body_inertia(self):
        """drop every per-environment row: later steps run as if none had been set"""
        _ck(lib().rsb_batch_clear_body_inertia(self.h))

    # per-environment terrain friction
    def set_contact_friction(self, rows, env_begin=0, env_count=None):
        """rows [n, ncoll] (numpy; collision-body order of the model tables) for environments [env_begin, env_begin + n): an entry
        >= 0 is the friction of that collision body's terrain contacts in that environment, < 0 the batch-level value
        (set_collision_friction, else params mu).  rows None resets env_count environments (default: to the end of the batch) to -1.
        A refused call (NaN or +-inf anywhere) changes nothing."""
        if rows is None:
            _ck(lib().rsb_batch_set_contact_friction(self.h, None, env_begin, self._count(env_begin, env_count), HOST))
            return
        r = np.ascontiguousarray(rows, np.float32)
        if r.ndim != 2 or r.shape[1] != self.model.ncoll:
            raise ValueError(f"rows: need shape [n, {self.model.ncoll}], got {r.shape}")
        _ck(lib().rsb_batch_set_contact_friction(self.h, r.ctypes.data_as(C.c_void_p), env_begin, r.shape[0], HOST))

    def set_contact_friction_from(self, rows, env_begin=0):
        """set_contact_friction() from a contiguous float32 torch tensor [n, ncoll] on the batch's device, checked there"""
        n = rows.shape[0] if hasattr(rows, "shape") and len(rows.shape) > 0 else -1
        _ck(lib().rsb_batch_set_contact_friction(self.h, self._device_out(rows, (n, self.model.ncoll), "rows"), env_begin, n, DEVICE))

    def clear_contact_friction(self):
        """drop every per-environment friction row: later steps run as if none had been set"""
        _ck(lib().rsb_batch_clear_contact_friction(self.h))

    # per-environment PD gains and actuator effort limits
    def set_actuator_params(self, rows, env_begin=0, env_count=None):
        """rows [n, nv, 3] (numpy; the batch's gv order; kp, kd, effort limit per dof) for environments [env_begin, env_begin + n): an
        entry >= 0 replaces the batch-level value of that dof in that environment, < 0 is the batch-level value (set_pd_gains, the
        URDF effort limit); effort +inf is no limit.  The base dofs of a floating robot are ignored.  rows None resets env_count
        environments (default: to the end of the batch) to -1.  A refused call (NaN anywhere, +-inf in kp or kd, -inf in the effort
        limit) changes nothing."""
        if rows is None:
            _ck(lib().rsb_batch_set_actuator_params(self.h, None, env_begin, self._count(env_begin, env_count), HOST))
            return
        r = np.ascontiguousarray(rows, np.float32)
        if r.ndim != 3 or r.shape[1:] != (self.nv, 3):
            raise ValueError(f"rows: need shape [n, {self.nv}, 3], got {r.shape}")
        _ck(lib().rsb_batch_set_actuator_params(self.h, r.ctypes.data_as(C.c_void_p), env_begin, r.shape[0], HOST))

    def set_actuator_params_from(self, rows, env_begin=0):
        """set_actuator_params() from a contiguous float32 torch tensor [n, nv, 3] on the batch's device, checked there"""
        n = rows.shape[0] if hasattr(rows, "shape") and len(rows.shape) > 0 else -1
        _ck(lib().rsb_batch_set_actuator_params(self.h, self._device_out(rows, (n, self.nv, 3), "rows"), env_begin, n, DEVICE))

    def clear_actuator_params(self):
        """drop every per-environment actuator row: later steps run as if none had been set"""
        _ck(lib().rsb_batch_clear_actuator_params(self.h))

    # learned actuator network
    def set_actuator_network(self, dofs_or_joint_names, layers, history):
        """One network for the batch, evaluated by the step kernel at every sub-step for each listed dof (gv indices, or joint names)
        from its last `history` position errors (ptarget - q) and velocities, in place of the PD law of those dofs.  layers: a list of
        (W, b) numpy pairs, torch.nn.Linear order (W [width, 2 * history], b [width], ..., W [1, width], b [1]), or a torch.nn.Sequential
        of Linear and Softsign only (Linear, Softsign, ..., Linear).  Input features: [e_t .. e_{t-H+1}, v_t .. v_{t-H+1}].  An empty
        dof list clears the network.  Every call zeroes all histories; a refused call changes nothing."""
        dofs = self._an_dofs(dofs_or_joint_names, "set_actuator_network")
        if len(dofs) == 0:
            _ck(lib().rsb_batch_set_actuator_network(self.h, None, 0, 0, 0, 0, None))
            self.an_shape = self.lstm_shape = None
            return
        pairs = _network_layers(layers)
        H = int(history)
        if len(pairs) < 2:
            raise ValueError("set_actuator_network: need at least one hidden layer and the output layer")
        width = pairs[0][0].shape[0]
        for l, (w, b) in enumerate(pairs):
            want = (1 if l == len(pairs) - 1 else width, 2 * H if l == 0 else width)
            if w.shape != want or b.shape != (want[0],):
                raise ValueError(f"set_actuator_network: layer {l}: need W {want} and b ({want[0]},), got {w.shape} and {b.shape}")
        params = np.ascontiguousarray(np.concatenate([np.concatenate([w.ravel(), b.ravel()]) for w, b in pairs]), np.float32)
        _ck(lib().rsb_batch_set_actuator_network(self.h, dofs.ctypes.data_as(C.c_void_p), len(dofs), H, len(pairs) - 1, width,
                                                 params.ctypes.data_as(C.c_void_p)))
        self.an_shape, self.lstm_shape = (len(dofs), H), None

    def _an_dofs(self, dofs_or_joint_names, who):
        """int32 gv indices of a dof list given as indices or joint names"""
        names = list(dofs_or_joint_names)
        if any(isinstance(d, str) for d in names):
            t = self.model.tables()
            by_name = {nm: int(t["vidx"][i]) for i, nm in enumerate(t["joint_names"]) if i > 0}
            missing = [d for d in names if isinstance(d, str) and d not in by_name]
            if missing:
                raise ValueError(f"{who}: unknown joints {missing}")
            names = [by_name[d] if isinstance(d, str) else d for d in names]
        return np.ascontiguousarray(names, np.int32).reshape(-1)

    def set_actuator_lstm(self, dofs_or_joint_names, lstm, readout):
        """One LSTM actuator network for the batch, in place of any network set before: at every sub-step the step kernel advances
        the cell of each listed dof (gv indices, or joint names) on x = (ptarget - q, v) and applies tau_ff + readout(h) in place of
        the dof's PD law.  lstm: a torch.nn.LSTM (input_size 2, bias, not bidirectional, no projection; batch_first does not matter)
        or a list of per-layer (weight_ih, weight_hh, bias_ih, bias_hh) arrays in torch order; readout: a torch.nn.Linear(hidden, 1)
        with bias, or a (weight [1, hidden], bias [1]) pair.  An empty dof list clears the network.  Every call zeroes all states; a
        refused call changes nothing."""
        dofs = self._an_dofs(dofs_or_joint_names, "set_actuator_lstm")
        if len(dofs) == 0:
            _ck(lib().rsb_batch_set_actuator_lstm(self.h, None, 0, 0, 0, None))
            self.an_shape = self.lstm_shape = None
            return
        layers, hidden, params = _lstm_params(lstm, readout)
        _ck(lib().rsb_batch_set_actuator_lstm(self.h, dofs.ctypes.data_as(C.c_void_p), len(dofs), layers, hidden,
                                              params.ctypes.data_as(C.c_void_p)))
        self.an_shape, self.lstm_shape = None, (len(dofs), layers, hidden)

    def _an_rows(self):
        if getattr(self, "lstm_shape", None) is not None:
            n, layers, hidden = self.lstm_shape
            return (n, layers, 2, hidden)
        if self.an_shape is None:
            raise ValueError("actuator history: no actuator network set through this object")
        return (self.an_shape[0], 2, self.an_shape[1] - 1)

    def actuator_history(self, env_begin=0, env_count=None):
        """[n, dofs, 2, H - 1] float32: errors then velocities of the last H - 1 sub-steps of every listed dof, most recent first.
        With an LSTM set: [n, dofs, layers, 2, hidden], h then c of every layer.  The same shapes hold for the variants below."""
        return self._read(lib().rsb_batch_get_actuator_history, self._an_rows(), np.float32, env_begin, env_count)

    def actuator_history_into(self, rows, env_begin=0, env_count=None):
        """actuator_history() copied into a torch CUDA tensor [n, dofs, 2, H - 1], in the batch's stream order"""
        n = self._count(env_begin, env_count)
        _ck(lib().rsb_batch_get_actuator_history(self.h, self._device_out(rows, (n,) + self._an_rows(), "rows"), env_begin, n, DEVICE))

    def set_actuator_history(self, rows, env_begin=0, env_count=None):
        """rows [n, dofs, 2, H - 1] (numpy) for environments [env_begin, env_begin + n); rows None zeroes env_count environments
        (default: to the end of the batch).  A refused call (NaN or +-inf anywhere) changes nothing."""
        shape = self._an_rows()
        if rows is None:
            _ck(lib().rsb_batch_set_actuator_history(self.h, None, env_begin, self._count(env_begin, env_count), HOST))
            return
        r = np.ascontiguousarray(rows, np.float32)
        if r.ndim != 1 + len(shape) or r.shape[1:] != shape:
            raise ValueError(f"rows: need shape [n, {', '.join(map(str, shape))}], got {r.shape}")
        _ck(lib().rsb_batch_set_actuator_history(self.h, r.ctypes.data_as(C.c_void_p), env_begin, r.shape[0], HOST))

    def set_actuator_history_from(self, rows, env_begin=0):
        """set_actuator_history() from a contiguous float32 torch tensor [n, dofs, 2, H - 1] on the batch's device, checked there"""
        shape = self._an_rows()
        n = rows.shape[0] if hasattr(rows, "shape") and len(rows.shape) > 0 else -1
        _ck(lib().rsb_batch_set_actuator_history(self.h, self._device_out(rows, (n,) + shape, "rows"), env_begin, n, DEVICE))

    # actuation delay
    def set_actuation_delay(self, delays, env_begin=0):
        """environments [env_begin, env_begin + len(delays)) apply each joint command delays [n] (numpy int32) physics sub-steps late:
        an entry d in [0, ACTUATION_DELAY_MAX] sets the delay and empties the environment's command history, -1 leaves the environment
        as it is.  delays None sets 0 and empties every environment from env_begin on.  A refused call changes nothing."""
        if delays is None:
            _ck(lib().rsb_batch_set_actuation_delay(self.h, None, env_begin, self.n - env_begin, HOST))
            return
        d = np.asarray(delays)
        if d.dtype != np.int32 or d.ndim != 1:
            raise ValueError(f"delays: need a 1-D numpy int32 array, got {d.dtype} of shape {d.shape}")
        d = np.ascontiguousarray(d)
        _ck(lib().rsb_batch_set_actuation_delay(self.h, d.ctypes.data_as(C.c_void_p), env_begin, len(d), HOST))

    def set_actuation_delay_from(self, delays, env_begin=0):
        """set_actuation_delay() from a contiguous int32 torch tensor [n] on the batch's device, checked there: a trainer passes
        torch.where(done, new_delay, -1) without a host round trip"""
        n = delays.shape[0] if hasattr(delays, "shape") and len(delays.shape) == 1 else -1
        _ck(lib().rsb_batch_set_actuation_delay(self.h, self._device_out(delays, (n,), "delays", "int32"), env_begin, n, DEVICE))

    def clear_actuation_delay(self):
        """drop every delay and command history: later steps run as if none had been set"""
        _ck(lib().rsb_batch_clear_actuation_delay(self.h))

    def control_step(self, ptarget, substeps, obs_out, vtarget=None):
        """one RaisimGym control step for the whole batch: targets in, fused sub-steps, observations out"""
        pp, w1 = _ptr(ptarget); pv, _ = _ptr(vtarget); po, w2 = _ptr(obs_out)
        _ck(lib().rsb_batch_control_step(self.h, pp, pv, w1, substeps, po, w2))
        return obs_out

    # RaisimGym task (VectorizedEnvironment)
    def gym_configure(self, gc_init, gv_init, action_mean, action_std, foot_bodies, torque_coeff=-4e-5, forward_vel_coeff=0.3, terminal_reward=-10.0):
        f = lambda a: np.ascontiguousarray(a, np.float32)
        a, b_, c, d = f(gc_init), f(gv_init), f(action_mean), f(action_std)
        fb = np.ascontiguousarray(foot_bodies, np.int32)
        _ck(lib().rsb_batch_gym_configure(self.h, *[x.ctypes.data_as(C.c_void_p) for x in (a, b_, c, d, fb)], len(fb), torque_coeff, forward_vel_coeff, terminal_reward))

    def gym_reset(self):
        _ck(lib().rsb_batch_gym_reset(self.h))

    def gym_step(self, action, substeps, obs, reward, done):
        pa, w1 = _ptr(action); po, w2 = _ptr(obs); pr, _ = _ptr(reward); pd, _ = _ptr(done)
        _ck(lib().rsb_batch_gym_step(self.h, pa, w1, substeps, po, pr, pd, w2))

    def set_observation_peers(self, world, rank, obs_ptrs, flag_ptrs):
        """fused observation all-gather: obs_ptrs [2 * world] / flag_ptrs [world] raw device pointers valid in this process"""
        if world == 0:
            _ck(lib().rsb_batch_set_observation_peers(self.h, 0, 0, None, None)); return
        a = (C.c_void_p * (2 * world))(*[C.c_void_p(int(x)) for x in obs_ptrs])
        f = (C.c_void_p * world)(*[C.c_void_p(int(x)) for x in flag_ptrs])
        _ck(lib().rsb_batch_set_observation_peers(self.h, world, rank, a, f))

    def wait_observation_peers(self):
        """the buffer parity that holds every rank's rows of the last control step (the step's own launch waited for them)"""
        par = C.c_int()
        _ck(lib().rsb_batch_wait_observation_peers(self.h, C.byref(par)))
        return par.value

    def observe(self, out=None, env_begin=0, env_count=None):
        n = self._count(env_begin, env_count)
        if out is None:
            out = np.empty((n, self.ob_dim()), np.float32)
        p, w = _ptr(out)
        _ck(lib().rsb_batch_observe(self.h, p, env_begin, n, w))
        return out
