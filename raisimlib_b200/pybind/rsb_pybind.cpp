// pybind11 module over the C-ABI (SURVEY 8f row N4): the batched device state as DLPack tensors, zero-copy.
// Replaces the numpy path of upstream raisimGymTorch/env/raisim_gym.cpp ([RECALL]; not in the reference snapshot): a PyTorch trainer
// on the same GPU takes `torch.from_dlpack(batch.gc())` and reads / writes the rows the step kernel works on -- no host round trip.
// Only include/rsb.h is used: the module links librsb.so, it contains no CUDA code of its own.
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include <cstdint>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/rsb.h"

namespace py = pybind11;

// ---- DLPack (dlpack.h v0.8 ABI, restated: the header is not vendored here) -------------------------------------------------------
extern "C" {
typedef enum { kDLCPU = 1, kDLCUDA = 2 } DLDeviceType;
typedef struct { int32_t device_type; int32_t device_id; } DLDevice;
typedef struct { uint8_t code; uint8_t bits; uint16_t lanes; } DLDataType;      // code 0 int, 1 uint, 2 float
typedef struct { void* data; DLDevice device; int32_t ndim; DLDataType dtype; int64_t* shape; int64_t* strides; uint64_t byte_offset; } DLTensor;
typedef struct DLManagedTensor { DLTensor dl_tensor; void* manager_ctx; void (*deleter)(struct DLManagedTensor*); } DLManagedTensor;
}

namespace {

void check(int rc, const char* what) {
  if (rc < 0) throw std::runtime_error(std::string(what) + ": " + rsb_last_error());
}

struct ModelHandle {
  rsb_model* m = nullptr;
  explicit ModelHandle(const std::string& urdf) { check(rsb_model_create_from_urdf(urdf.c_str(), &m), "Model"); }
  ~ModelHandle() { if (m) rsb_model_destroy(m); }
};

struct Holder {               // keeps the batch alive as long as a tensor made from it
  std::shared_ptr<void> keep;
  int64_t shape[2], strides[2];
};
void dl_deleter(DLManagedTensor* t) { delete static_cast<Holder*>(t->manager_ctx); delete t; }
void capsule_destructor(PyObject* cap) {
  if (PyCapsule_IsValid(cap, "dltensor")) {     // never consumed: free it ourselves (a consumer renames the capsule to "used_dltensor")
    auto* t = static_cast<DLManagedTensor*>(PyCapsule_GetPointer(cap, "dltensor"));
    if (t && t->deleter) t->deleter(t);
  }
}

class Batch : public std::enable_shared_from_this<Batch> {
 public:
  Batch(std::shared_ptr<ModelHandle> model, int num_envs, int device) : model_(std::move(model)), device_(device) {
    check(rsb_batch_create(model_->m, num_envs, device, &b_), "Batch");
    check(rsb_batch_device_ptrs(b_, &view_), "device_ptrs");
  }
  ~Batch() { if (b_) rsb_batch_destroy(b_); }
  rsb_batch* raw() const { return b_; }

  py::capsule tensor(float* base, int64_t rows, int64_t cols, int64_t row_stride) {
    auto* h = new Holder;
    h->keep = shared_from_this();
    h->shape[0] = rows; h->shape[1] = cols; h->strides[0] = row_stride; h->strides[1] = 1;
    auto* t = new DLManagedTensor;
    t->dl_tensor.data = base;
    t->dl_tensor.device = DLDevice{kDLCUDA, device_};
    t->dl_tensor.ndim = 2;
    t->dl_tensor.dtype = DLDataType{2, 32, 1};
    t->dl_tensor.shape = h->shape; t->dl_tensor.strides = h->strides; t->dl_tensor.byte_offset = 0;
    t->manager_ctx = h; t->deleter = dl_deleter;
    return py::capsule(t, "dltensor", capsule_destructor);
  }
  // zero-copy views of the padded rows the kernel reads and writes: [num_envs, nq | nv], row stride gc_stride | gv_stride
  py::capsule gc() { return tensor(view_.gc, view_.num_envs, view_.nq, view_.gc_stride); }
  py::capsule gv() { return tensor(view_.gv, view_.num_envs, view_.nv, view_.gv_stride); }
  py::capsule tau_ff() { return tensor(view_.tau_ff, view_.num_envs, view_.nv, view_.gv_stride); }
  py::capsule pd_target() { return tensor(view_.ptarget, view_.num_envs, view_.nq, view_.gc_stride); }
  py::capsule pd_velocity_target() { return tensor(view_.vtarget, view_.num_envs, view_.nv, view_.gv_stride); }

  void set_ground(float z) { check(rsb_batch_set_ground(b_, z), "set_ground"); }
  void set_stream(uintptr_t s) { check(rsb_batch_set_stream(b_, reinterpret_cast<void*>(s)), "set_stream"); }
  void set_pd_gains(const std::vector<float>& kp, const std::vector<float>& kd) {
    if ((int)kp.size() != view_.nv || (int)kd.size() != view_.nv) throw std::runtime_error("set_pd_gains: need nv gains");
    check(rsb_batch_set_pd_gains(b_, kp.data(), kd.data()), "set_pd_gains");
  }
  void integrate(int substeps) { check(rsb_batch_integrate(b_, substeps), "integrate"); }
  void update_kinematics() { check(rsb_batch_update_kinematics(b_), "update_kinematics"); }
  void sync() { check(rsb_batch_sync(b_), "sync"); }
  // one control step with everything on the device: obs = DLPack-importable tensor address ([num_envs, ob_dim] float32, contiguous)
  void control_step(uintptr_t ptarget_dev, int substeps, uintptr_t obs_dev) {
    check(rsb_batch_control_step(b_, reinterpret_cast<const float*>(ptarget_dev), nullptr, RSB_DEVICE, substeps, reinterpret_cast<float*>(obs_dev), RSB_DEVICE), "control_step");
  }
  // frames rigidly attached to bodies: body [F], pos [F*3], rot [F*9] row-major in the body frame (empty = identity)
  void set_frames(const std::vector<int32_t>& body, const std::vector<float>& pos, const std::vector<float>& rot) {
    if (pos.size() != 3 * body.size() || (!rot.empty() && rot.size() != 9 * body.size())) throw std::runtime_error("set_frames: need 3 positions and 0 or 9 rotation entries per frame");
    check(rsb_batch_set_frames(b_, body.data(), pos.data(), rot.empty() ? nullptr : rot.data(), (int)body.size()), "set_frames");
  }
  // frame states of every environment into tensor addresses ([num_envs, F, 3 | 9] float32, contiguous); 0 skips an output
  void frame_states(uintptr_t pos_dev, uintptr_t rot_dev, uintptr_t lin_dev, uintptr_t ang_dev) {
    check(rsb_batch_get_frame_states(b_, 0, view_.num_envs, reinterpret_cast<float*>(pos_dev), reinterpret_cast<float*>(rot_dev), reinterpret_cast<float*>(lin_dev),
                                     reinterpret_cast<float*>(ang_dev), RSB_DEVICE), "frame_states");
  }
  // frame Jacobians of every environment into a tensor address ([num_envs, F, 6, nv] float32, contiguous)
  void frame_jacobians(uintptr_t jac_dev) {
    check(rsb_batch_get_frame_jacobians(b_, 0, view_.num_envs, reinterpret_cast<float*>(jac_dev), RSB_DEVICE), "frame_jacobians");
  }
  // bodies whose contact force every stepping launch gathers over all its sub-steps (empty clears)
  void set_contact_bodies(const std::vector<int32_t>& body) { check(rsb_batch_set_contact_bodies(b_, body.data(), (int)body.size()), "set_contact_bodies"); }
  // their mean contact force and sub-steps in contact over the last stepping launch into tensor addresses ([num_envs, S, 3] float32,
  // [num_envs, S] int32, contiguous); 0 skips an output.  A copy in the batch's stream order: no launch
  void body_contact_forces(uintptr_t force_dev, uintptr_t steps_dev) {
    check(rsb_batch_get_body_contact_forces(b_, 0, view_.num_envs, reinterpret_cast<float*>(force_dev), reinterpret_cast<int32_t*>(steps_dev), RSB_DEVICE), "body_contact_forces");
  }
  // IMU sensors shared by all environments: body [I], pos [I*3] and rot [I*9] (empty: identity) in the body frame (empty body clears)
  void set_imus(const std::vector<int32_t>& body, const std::vector<float>& pos, const std::vector<float>& rot) {
    if (pos.size() != 3 * body.size() || (!rot.empty() && rot.size() != 9 * body.size())) throw std::runtime_error("set_imus: need 3 positions and 0 or 9 rotation entries per sensor");
    check(rsb_batch_set_imus(b_, body.data(), pos.data(), rot.empty() ? nullptr : rot.data(), (int)body.size()), "set_imus");
  }
  // their mean specific force and angular rate over the last stepping launch into tensor addresses ([num_envs, I, 3] float32, contiguous,
  // sensor frames); 0 skips an output.  A copy in the batch's stream order: no launch
  void imu_readings(uintptr_t lin_dev, uintptr_t ang_dev) {
    check(rsb_batch_get_imu_readings(b_, 0, view_.num_envs, reinterpret_cast<float*>(lin_dev), reinterpret_cast<float*>(ang_dev), RSB_DEVICE), "imu_readings");
  }
  // terrain height-scan points shared by all environments: body [P], xy [P*2] horizontal offsets, align "yaw" or "world" (empty clears)
  void set_height_scan(const std::vector<int32_t>& body, const std::vector<float>& xy, const std::string& align) {
    if (xy.size() != 2 * body.size()) throw std::runtime_error("set_height_scan: need 2 offset entries per point");
    if (align != "yaw" && align != "world") throw std::runtime_error("set_height_scan: align must be 'yaw' or 'world'");
    check(rsb_batch_set_height_scan(b_, body.data(), xy.data(), (int)body.size(), align == "yaw" ? RSB_SCAN_YAW : RSB_SCAN_WORLD), "set_height_scan");
  }
  // the scan of every environment into tensor addresses ([num_envs, P] and [num_envs, P, 2] float32, contiguous); 0 skips an output
  void height_scan(uintptr_t height_dev, uintptr_t xy_dev) {
    check(rsb_batch_get_height_scan(b_, 0, view_.num_envs, reinterpret_cast<float*>(height_dev), reinterpret_cast<float*>(xy_dev), RSB_DEVICE), "height_scan");
  }
  // per-environment inertial rows [env_count, nb, 10] float32 (mass, com, inertia xx xy xz yy yz zz) from a device address
  void set_body_inertia(uintptr_t rows_dev, int env_begin, int env_count) {
    check(rsb_batch_set_body_inertia(b_, reinterpret_cast<const float*>(rows_dev), env_begin, env_count, RSB_DEVICE), "set_body_inertia");
  }
  // per-environment terrain friction rows [env_count, ncoll] float32 (>= 0: this collision body's friction, < 0: the batch's) from a device address
  void set_contact_friction(uintptr_t rows_dev, int env_begin, int env_count) {
    check(rsb_batch_set_contact_friction(b_, reinterpret_cast<const float*>(rows_dev), env_begin, env_count, RSB_DEVICE), "set_contact_friction");
  }
  // per-environment actuator rows [env_count, nv, 3] float32 (kp, kd, effort limit; >= 0: this dof's own, < 0: the batch's) from a device address
  void set_actuator_params(uintptr_t rows_dev, int env_begin, int env_count) {
    check(rsb_batch_set_actuator_params(b_, reinterpret_cast<const float*>(rows_dev), env_begin, env_count, RSB_DEVICE), "set_actuator_params");
  }
  // learned actuator network: dofs (gv indices), parameters in torch.nn.Linear order (host); an empty dof list clears it
  void set_actuator_network(const std::vector<int32_t>& dofs, int history, int layers, int width, const std::vector<float>& params) {
    if (!dofs.empty()) {   // the library reads exactly this many floats
      const size_t count = (history < 1 || layers < 1 || width < 1) ? 0
                         : size_t(2 * history) * width + width + size_t(layers - 1) * (size_t(width) * width + width) + width + 1;
      if (count == 0 || params.size() != count)
        throw std::runtime_error("set_actuator_network: " + std::to_string(params.size()) + " parameters for history " + std::to_string(history) + ", " +
                                 std::to_string(layers) + " layers of width " + std::to_string(width) + " (need " + std::to_string(count) + ")");
    }
    check(rsb_batch_set_actuator_network(b_, dofs.data(), (int)dofs.size(), history, layers, width, params.data()), "set_actuator_network");
  }
  // its history rows [env_count, dofs, 2, history - 1] float32 at a device address (0: zeroes the range)
  void set_actuator_history(uintptr_t rows_dev, int env_begin, int env_count) {
    check(rsb_batch_set_actuator_history(b_, reinterpret_cast<const float*>(rows_dev), env_begin, env_count, RSB_DEVICE), "set_actuator_history");
  }
  void actuator_history(uintptr_t rows_dev, int env_begin, int env_count) {
    check(rsb_batch_get_actuator_history(b_, reinterpret_cast<float*>(rows_dev), env_begin, env_count, RSB_DEVICE), "actuator_history");
  }
  // terrain atlas: heights [count * ys * xs] and the map of every environment [num_envs], host lists
  void set_heightmaps(int count, int xs, int ys, float x_size, float y_size, float cx, float cy, const std::vector<float>& heights,
                      const std::vector<int32_t>& map_of_env) {
    if ((int64_t)heights.size() != (int64_t)count * xs * ys || (int)map_of_env.size() != view_.num_envs)
      throw std::runtime_error("set_heightmaps: need count * ys * xs heights and one map index per environment");
    check(rsb_batch_set_heightmaps(b_, count, xs, ys, x_size, y_size, cx, cy, heights.data(), map_of_env.data()), "set_heightmaps");
  }
  // terrain curriculum: atlas map index of environments [env_begin, env_begin + env_count) ([env_count] int32) from a device address
  void set_heightmap_index(uintptr_t map_of_env_dev, int env_begin, int env_count) {
    check(rsb_batch_set_heightmap_index(b_, reinterpret_cast<const int32_t*>(map_of_env_dev), env_begin, env_count, RSB_DEVICE), "set_heightmap_index");
  }
  // actuation delays of environments [env_begin, env_begin + env_count) ([env_count] int32, -1: unchanged) from a device address
  // (0: delay 0 and an empty history for the whole range)
  void set_actuation_delay(uintptr_t delays_dev, int env_begin, int env_count) {
    check(rsb_batch_set_actuation_delay(b_, reinterpret_cast<const int32_t*>(delays_dev), env_begin, env_count, RSB_DEVICE), "set_actuation_delay");
  }
  void clear_actuation_delay() { check(rsb_batch_clear_actuation_delay(b_), "clear_actuation_delay"); }
  // maps first .. first + count - 1 of the terrain overwritten with [count, ys, xs] float32 heights from a device address
  void update_heightmaps(uintptr_t heights_dev, int first, int count) {
    check(rsb_batch_update_heightmaps(b_, first, count, reinterpret_cast<const float*>(heights_dev), RSB_DEVICE), "update_heightmaps");
  }
  int num_envs() const { return view_.num_envs; }
  int nq() const { return view_.nq; }
  int nv() const { return view_.nv; }
  int ob_dim() const { return rsb_batch_ob_dim(b_); }
  long launch_count() const { return (long)rsb_batch_launch_count(b_); }

 private:
  std::shared_ptr<ModelHandle> model_;
  rsb_batch* b_ = nullptr;
  rsb_device_view view_{};
  int device_ = 0;
};

}  // namespace

PYBIND11_MODULE(_rsb_py, m) {
  m.doc() = "raisimlib_b200: batched World::integrate() on the GPU, device state as DLPack tensors (zero-copy)";
  py::class_<ModelHandle, std::shared_ptr<ModelHandle>>(m, "Model").def(py::init<const std::string&>(), py::arg("urdf_path_or_xml"));
  py::class_<Batch, std::shared_ptr<Batch>>(m, "Batch")
      .def(py::init<std::shared_ptr<ModelHandle>, int, int>(), py::arg("model"), py::arg("num_envs"), py::arg("device") = 0)
      .def("gc", &Batch::gc, "generalized coordinates [num_envs, nq] as a DLPack capsule (zero-copy view of the batch rows)")
      .def("gv", &Batch::gv)
      .def("tau_ff", &Batch::tau_ff)
      .def("pd_target", &Batch::pd_target)
      .def("pd_velocity_target", &Batch::pd_velocity_target)
      .def("set_ground", &Batch::set_ground)
      .def("set_stream", &Batch::set_stream)
      .def("set_pd_gains", &Batch::set_pd_gains)
      .def("integrate", &Batch::integrate, py::arg("substeps") = 1)
      .def("update_kinematics", &Batch::update_kinematics)
      .def("control_step", &Batch::control_step)
      .def("set_frames", &Batch::set_frames, py::arg("body"), py::arg("pos"), py::arg("rot") = std::vector<float>())
      .def("frame_states", &Batch::frame_states, py::arg("pos_dev"), py::arg("rot_dev"), py::arg("lin_dev"), py::arg("ang_dev"))
      .def("frame_jacobians", &Batch::frame_jacobians, py::arg("jac_dev"))
      .def("set_contact_bodies", &Batch::set_contact_bodies, py::arg("body"))
      .def("body_contact_forces", &Batch::body_contact_forces, py::arg("force_dev"), py::arg("steps_dev"))
      .def("set_imus", &Batch::set_imus, py::arg("body"), py::arg("pos"), py::arg("rot") = std::vector<float>())
      .def("imu_readings", &Batch::imu_readings, py::arg("lin_acc_dev"), py::arg("ang_vel_dev"))
      .def("set_height_scan", &Batch::set_height_scan, py::arg("body"), py::arg("xy"), py::arg("align") = std::string("yaw"))
      .def("height_scan", &Batch::height_scan, py::arg("height_dev"), py::arg("xy_dev"))
      .def("set_body_inertia", &Batch::set_body_inertia, py::arg("rows_dev"), py::arg("env_begin"), py::arg("env_count"))
      .def("set_contact_friction", &Batch::set_contact_friction, py::arg("rows_dev"), py::arg("env_begin"), py::arg("env_count"))
      .def("set_actuator_params", &Batch::set_actuator_params, py::arg("rows_dev"), py::arg("env_begin"), py::arg("env_count"))
      .def("set_actuator_network", &Batch::set_actuator_network, py::arg("dofs"), py::arg("history"), py::arg("layers"), py::arg("width"), py::arg("params"))
      .def("set_actuator_history", &Batch::set_actuator_history, py::arg("rows_dev"), py::arg("env_begin"), py::arg("env_count"))
      .def("actuator_history", &Batch::actuator_history, py::arg("rows_dev"), py::arg("env_begin"), py::arg("env_count"))
      .def("set_heightmaps", &Batch::set_heightmaps, py::arg("count"), py::arg("xs"), py::arg("ys"), py::arg("x_size"), py::arg("y_size"),
           py::arg("cx"), py::arg("cy"), py::arg("heights"), py::arg("map_of_env"))
      .def("set_heightmap_index", &Batch::set_heightmap_index, py::arg("map_of_env_dev"), py::arg("env_begin"), py::arg("env_count"))
      .def("update_heightmaps", &Batch::update_heightmaps, py::arg("heights_dev"), py::arg("first"), py::arg("count"))
      .def("set_actuation_delay", &Batch::set_actuation_delay, py::arg("delays_dev"), py::arg("env_begin"), py::arg("env_count"))
      .def("clear_actuation_delay", &Batch::clear_actuation_delay)
      .def("sync", &Batch::sync)
      .def_property_readonly("num_envs", &Batch::num_envs)
      .def_property_readonly("nq", &Batch::nq)
      .def_property_readonly("nv", &Batch::nv)
      .def_property_readonly("ob_dim", &Batch::ob_dim)
      .def_property_readonly("launch_count", &Batch::launch_count);
}
