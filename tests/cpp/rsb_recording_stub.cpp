// Host-memory stand-in for the C ABI (include/rsb.h) that records what the raisim:: facade asks of the batch: every rsb_batch_* call
// appends one line to rsb_stub_log() -- its name, its scalar arguments (environment range, `where`, sub-steps ...) and an FNV-1a hash of
// every buffer passed in (before the call) or out (after it).  Model queries (tables, names) are host-only and not recorded.
// It is a recorder, not a simulator: getters return what setters stored, rsb_batch_integrate adds 1e-3 * substeps to every coordinate,
// and M, h, poses, contacts, contact forces and height scans are simple functions of the stored state.
// The model: a floating base (body 0) with three revolute joints j1 (body 1, child of 0), j2 (body 2, child of 1), j3 (body 3, child
// of 0); nq = 10, nv = 9, one collision body per body.
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "rsb.h"

std::string& rsb_stub_log() { static std::string s; return s; }

namespace {
const int NB = 4, NQ = 10, NV = 9, NCOLL = 4;
const int kParent[NB] = {-1, 0, 1, 0}, kJtype[NB] = {3, 1, 1, 1}, kQidx[NB] = {0, 7, 8, 9}, kVidx[NB] = {0, 6, 7, 8}, kDepth[NB] = {0, 1, 2, 1};
const double kAxis[NB * 3] = {0, 0, 1, 0, 1, 0, 0, 1, 0, 1, 0, 0};
const double kMass[NB] = {10, 1, 0.5, 1};
const double kCom[NB * 3] = {0, 0, 0, 0.1, 0, 0, 0, 0, -0.1, 0, 0.1, 0};
const double kInertia[NB * 6] = {0.1, 0, 0, 0.2, 0, 0.3, 0.01, 0, 0, 0.01, 0, 0.01, 0.005, 0, 0, 0.005, 0, 0.005, 0.01, 0, 0, 0.01, 0, 0.01};
const double kJlimit[NB * 2] = {-1e30, 1e30, -1, 1, -2, 2, -1.5, 1.5};
const double kJeffort[NB] = {1e30, 40, 30, 1e30};
const int kCbody[NCOLL] = {0, 1, 2, 3};
const char* kBody[NB] = {"base", "l1", "l2", "l3"};
const char* kJoint[NB] = {"root", "j1", "j2", "j3"};

uint64_t fnv(const void* p, size_t bytes) {
  uint64_t h = 1469598103934665603ull;
  const unsigned char* c = static_cast<const unsigned char*>(p);
  for (size_t i = 0; i < bytes; i++) h = (h ^ c[i]) * 1099511628211ull;
  return h;
}
struct Line {
  std::string s;
  explicit Line(const char* name) : s(name) {}
  Line& i(const char* k, long v) { s += " " + std::string(k) + "=" + std::to_string(v); return *this; }
  Line& f(const char* k, double v) { char b[64]; std::snprintf(b, sizeof b, " %s=%.9g", k, v); s += b; return *this; }
  Line& buf(const char* k, const void* p, size_t bytes) {
    char b[64];
    if (p) std::snprintf(b, sizeof b, " %s=%016llx", k, (unsigned long long)fnv(p, bytes)); else std::snprintf(b, sizeof b, " %s=null", k);
    s += b; return *this;
  }
  ~Line() { rsb_stub_log() += s + "\n"; }
};
}  // namespace

struct rsb_model { int unused = 0; };
struct rsb_batch {
  int n;
  rsb_params p{};
  std::vector<float> gc, gv, pt, vt, tau, hist, scan;
  std::vector<int32_t> delay, bodies;
  int64_t launches = 0;
  int histWords = 0, scanPoints = 0, ncb = 0;
  bool terrain = false;
};

extern "C" {
const char* rsb_last_error(void) { return "stub error"; }
int rsb_model_create_from_urdf(const char*, rsb_model** out) { *out = new rsb_model; return 0; }
void rsb_model_destroy(rsb_model* m) { delete m; }
int rsb_model_dims(const rsb_model*, int* nq, int* nv, int* nb, int* ncoll, int* npts) {
  if (nq) *nq = NQ;
  if (nv) *nv = NV;
  if (nb) *nb = NB;
  if (ncoll) *ncoll = NCOLL;
  if (npts) *npts = NCOLL;
  return 0;
}
int rsb_model_get_tables(const rsb_model*, rsb_model_tables* t) {
  std::memset(t, 0, sizeof *t);
  t->nb = NB; t->nq = NQ; t->nv = NV; t->floating = 1; t->ncoll = NCOLL; t->npts = NCOLL;
  t->parent = kParent; t->jtype = kJtype; t->qidx = kQidx; t->vidx = kVidx; t->depth = kDepth;
  t->axis = kAxis; t->mass = kMass; t->com = kCom; t->inertia = kInertia; t->jlimit = kJlimit; t->jeffort = kJeffort; t->cbody = kCbody;
  return 0;
}
int rsb_model_body_index(const rsb_model*, const char* name) { for (int b = 0; b < NB; b++) if (!std::strcmp(name, kBody[b])) return b; return -1; }
const char* rsb_model_body_name(const rsb_model*, int b) { return kBody[b]; }
int rsb_model_collision_index(const rsb_model*, const char* name) {
  for (int b = 0; b < NB; b++) if (std::string(kBody[b]) + "/0" == name) return b;
  return -1;
}
const char* rsb_model_joint_name(const rsb_model*, int b) { return kJoint[b]; }
int rsb_model_frame_index(const rsb_model* m, const char* name) { return rsb_model_body_index(m, name); }
int rsb_model_frame(const rsb_model*, int frame, int* body, double pos[3], double rot[9]) {
  *body = frame;
  for (int k = 0; k < 3; k++) pos[k] = 0.05 * (k + 1);
  for (int k = 0; k < 9; k++) rot[k] = k % 4 == 0 ? 1.0 : 0.0;
  return 0;
}
int rsb_terrain_generate(const rsb_terrain_properties* p, float* h) {
  for (int i = 0; i < p->x_samples * p->y_samples; i++) h[i] = float(0.001 * (i % 17) + p->height_offset);
  return 0;
}
int rsb_heightmap_read_text(const char*, int*, int*, double*, double*, float*, int) { return RSB_ERR_UNSUPPORTED; }
int rsb_heightmap_read_png(const char*, double, double, int*, int*, float*, int) { return RSB_ERR_UNSUPPORTED; }

int rsb_batch_create(const rsb_model*, int n, int, rsb_batch** out) {
  rsb_batch* b = new rsb_batch;
  b->n = n;
  rsb_params_default(&b->p);
  b->gc.assign(size_t(n) * NQ, 0.f); b->gv.assign(size_t(n) * NV, 0.f); b->pt.assign(size_t(n) * NQ, 0.f); b->vt.assign(size_t(n) * NV, 0.f);
  b->tau.assign(size_t(n) * NV, 0.f); b->delay.assign(n, 0);
  for (int e = 0; e < n; e++) b->gc[size_t(e) * NQ + 3] = 1.f;
  *out = b;
  Line("rsb_batch_create").i("n", n);
  return 0;
}
void rsb_batch_destroy(rsb_batch* b) { Line("rsb_batch_destroy"); delete b; }
int rsb_params_default(rsb_params* p) {
  std::memset(p, 0, sizeof *p);
  p->dt = 0.0025f; p->gravity[2] = -9.81f; p->alpha_init = p->alpha_min = p->alpha_decay = 1.f; p->max_iter = 150; p->threshold = 1e-6f; p->mu = 0.8f;
  p->rest_threshold = 0.01f;
  return 0;
}
int rsb_batch_set_params(rsb_batch* b, const rsb_params* p) { Line("rsb_batch_set_params").buf("p", p, sizeof *p); b->p = *p; return 0; }
int rsb_batch_get_params(const rsb_batch* b, rsb_params* p) { *p = b->p; Line("rsb_batch_get_params").buf("p", p, sizeof *p); return 0; }
int rsb_batch_set_ground(rsb_batch* b, float z) { b->terrain = true; Line("rsb_batch_set_ground").f("z", z); return 0; }
int rsb_batch_set_heightmap(rsb_batch* b, int xs, int ys, float sx, float sy, float cx, float cy, const float* h) {
  b->terrain = true;
  Line("rsb_batch_set_heightmap").i("xs", xs).i("ys", ys).f("sx", sx).f("sy", sy).f("cx", cx).f("cy", cy).buf("h", h, sizeof(float) * xs * ys);
  return 0;
}
int rsb_batch_set_heightmaps(rsb_batch* b, int count, int xs, int ys, float sx, float sy, float cx, float cy, const float* h, const int32_t* idx) {
  b->terrain = true;
  Line("rsb_batch_set_heightmaps").i("count", count).i("xs", xs).i("ys", ys).f("sx", sx).f("sy", sy).f("cx", cx).f("cy", cy)
      .buf("h", h, sizeof(float) * count * xs * ys).buf("idx", idx, sizeof(int32_t) * b->n);
  return 0;
}
int rsb_batch_set_heightmap_index(rsb_batch*, const int32_t* idx, int lo, int count, int where) {
  Line("rsb_batch_set_heightmap_index").i("lo", lo).i("count", count).i("where", where).buf("idx", idx, sizeof(int32_t) * count);
  return 0;
}
int rsb_batch_set_collision_friction(rsb_batch*, int c, float mu) { Line("rsb_batch_set_collision_friction").i("body", c).f("mu", mu); return 0; }
int rsb_batch_set_contact_friction(rsb_batch*, const float* rows, int lo, int count, int where) {
  Line("rsb_batch_set_contact_friction").i("lo", lo).i("count", count).i("where", where).buf("rows", rows, sizeof(float) * count * NCOLL);
  return 0;
}
int rsb_batch_set_self_collision(rsb_batch*, const int32_t* pairs, int n, const float* mu) {
  Line("rsb_batch_set_self_collision").i("n", n).buf("pairs", pairs, sizeof(int32_t) * 2 * n).buf("mu", mu, sizeof(float) * n);
  return 0;
}
int rsb_batch_set_state(rsb_batch* b, const float* gc, const float* gv, int lo, int count, int where) {
  Line("rsb_batch_set_state").i("lo", lo).i("count", count).i("where", where).buf("gc", gc, sizeof(float) * count * NQ).buf("gv", gv, sizeof(float) * count * NV);
  if (gc) std::memcpy(&b->gc[size_t(lo) * NQ], gc, sizeof(float) * count * NQ);
  if (gv) std::memcpy(&b->gv[size_t(lo) * NV], gv, sizeof(float) * count * NV);
  return 0;
}
int rsb_batch_get_state(rsb_batch* b, float* gc, float* gv, int lo, int count, int where) {
  if (gc) std::memcpy(gc, &b->gc[size_t(lo) * NQ], sizeof(float) * count * NQ);
  if (gv) std::memcpy(gv, &b->gv[size_t(lo) * NV], sizeof(float) * count * NV);
  Line("rsb_batch_get_state").i("lo", lo).i("count", count).i("where", where).buf("gc", gc, sizeof(float) * count * NQ).buf("gv", gv, sizeof(float) * count * NV);
  return 0;
}
int rsb_batch_set_pd_gains(rsb_batch*, const float* kp, const float* kd) {
  Line("rsb_batch_set_pd_gains").buf("kp", kp, sizeof(float) * NV).buf("kd", kd, sizeof(float) * NV);
  return 0;
}
int rsb_batch_set_pd_target(rsb_batch* b, const float* pt, const float* vt, int lo, int count, int where) {
  Line("rsb_batch_set_pd_target").i("lo", lo).i("count", count).i("where", where).buf("pt", pt, sizeof(float) * count * NQ).buf("vt", vt, sizeof(float) * count * NV);
  if (pt) std::memcpy(&b->pt[size_t(lo) * NQ], pt, sizeof(float) * count * NQ);
  if (vt) std::memcpy(&b->vt[size_t(lo) * NV], vt, sizeof(float) * count * NV);
  return 0;
}
int rsb_batch_set_generalized_force(rsb_batch* b, const float* tau, int lo, int count, int where) {
  Line("rsb_batch_set_generalized_force").i("lo", lo).i("count", count).i("where", where).buf("tau", tau, sizeof(float) * count * NV);
  std::memcpy(&b->tau[size_t(lo) * NV], tau, sizeof(float) * count * NV);
  return 0;
}
int rsb_batch_set_control_mode(rsb_batch*, int mode) { Line("rsb_batch_set_control_mode").i("mode", mode); return 0; }
int rsb_batch_set_external_wrench(rsb_batch*, int body, const float* f, const float* t, const float* p, int lo, int count, int where) {
  Line("rsb_batch_set_external_wrench").i("body", body).i("lo", lo).i("count", count).i("where", where)
      .buf("f", f, sizeof(float) * 3 * count).buf("t", t, sizeof(float) * 3 * count).buf("p", p, sizeof(float) * 3);
  return 0;
}
int rsb_batch_set_body_inertia(rsb_batch*, const float* rows, int lo, int count, int where) {
  Line("rsb_batch_set_body_inertia").i("lo", lo).i("count", count).i("where", where).buf("rows", rows, sizeof(float) * count * NB * 10);
  return 0;
}
int rsb_batch_set_actuator_params(rsb_batch*, const float* rows, int lo, int count, int where) {
  Line("rsb_batch_set_actuator_params").i("lo", lo).i("count", count).i("where", where).buf("rows", rows, sizeof(float) * count * NV * 3);
  return 0;
}
int rsb_batch_set_actuator_network(rsb_batch* b, const int32_t* dofs, int n, int H, int L, int W, const float* params) {
  const size_t count = n ? size_t(2 * H) * W + W + size_t(L - 1) * (size_t(W) * W + W) + W + 1 : 0;
  Line("rsb_batch_set_actuator_network").i("n", n).i("H", H).i("L", L).i("W", W).buf("dofs", dofs, sizeof(int32_t) * n).buf("params", params, sizeof(float) * count);
  b->histWords = n * 2 * (H - 1);
  b->hist.assign(size_t(b->n) * b->histWords, 0.f);
  for (size_t i = 0; i < b->hist.size(); i++) b->hist[i] = 0.25f * float(i % 7);   // so that zeroing rows shows in the hashes
  return 0;
}
int rsb_batch_set_actuator_history(rsb_batch* b, const float* rows, int lo, int count, int where) {
  Line("rsb_batch_set_actuator_history").i("lo", lo).i("count", count).i("where", where).buf("rows", rows, sizeof(float) * count * b->histWords);
  for (size_t i = 0; i < size_t(count) * b->histWords; i++) b->hist[size_t(lo) * b->histWords + i] = rows ? rows[i] : 0.f;
  return 0;
}
int rsb_batch_get_actuator_history(rsb_batch* b, float* rows, int lo, int count, int where) {
  std::memcpy(rows, &b->hist[size_t(lo) * b->histWords], sizeof(float) * count * b->histWords);
  Line("rsb_batch_get_actuator_history").i("lo", lo).i("count", count).i("where", where).buf("rows", rows, sizeof(float) * count * b->histWords);
  return 0;
}
int rsb_batch_set_actuation_delay(rsb_batch*, const int32_t* d, int lo, int count, int where) {
  Line("rsb_batch_set_actuation_delay").i("lo", lo).i("count", count).i("where", where).buf("delays", d, sizeof(int32_t) * count);
  return 0;
}
int rsb_batch_get_generalized_force(rsb_batch* b, float* tau, int lo, int count, int where) {
  for (int i = 0; i < count * NV; i++) tau[i] = b->tau[size_t(lo) * NV + i] + 0.5f * b->gv[size_t(lo) * NV + i];
  Line("rsb_batch_get_generalized_force").i("lo", lo).i("count", count).i("where", where).buf("tau", tau, sizeof(float) * count * NV);
  return 0;
}
int rsb_batch_integrate1(rsb_batch* b) { b->launches++; Line("rsb_batch_integrate1"); return 0; }
int rsb_batch_integrate2(rsb_batch* b) { b->launches++; for (float& q : b->gc) q += 1e-3f; Line("rsb_batch_integrate2"); return 0; }
int rsb_batch_integrate(rsb_batch* b, int substeps) {
  b->launches++;
  for (size_t i = 0; i < b->gc.size(); i++) b->gc[i] += 1e-3f * float(substeps);
  for (size_t i = 0; i < b->gv.size(); i++) b->gv[i] += 2e-3f * float(substeps) * b->pt[(i / NV) * NQ + 1 + i % NV];
  Line("rsb_batch_integrate").i("substeps", substeps);
  return 0;
}
// M = diag(1 + 0.1 i + gc_0) + 0.01 (gc_i + gc_j) off the diagonal, h_i = gv_i + gc_i: both move with the state
int rsb_batch_get_mass_matrix(rsb_batch* b, int lo, int count, float* out, int where) {
  for (int e = lo; e < lo + count; e++)
    for (int i = 0; i < NV; i++)
      for (int j = 0; j < NV; j++) {
        const float* q = &b->gc[size_t(e) * NQ];
        out[(size_t(e - lo) * NV + i) * NV + j] = i == j ? 1.f + 0.1f * float(i) + q[0] : 0.01f * (q[i] + q[j]);
      }
  Line("rsb_batch_get_mass_matrix").i("lo", lo).i("count", count).i("where", where).buf("M", out, sizeof(float) * count * NV * NV);
  return 0;
}
int rsb_batch_get_nonlinearities(rsb_batch* b, int lo, int count, float* out, int where) {
  for (int e = lo; e < lo + count; e++) for (int i = 0; i < NV; i++) out[size_t(e - lo) * NV + i] = b->gv[size_t(e) * NV + i] + b->gc[size_t(e) * NQ + i];
  Line("rsb_batch_get_nonlinearities").i("lo", lo).i("count", count).i("where", where).buf("h", out, sizeof(float) * count * NV);
  return 0;
}
int rsb_batch_get_body_poses(rsb_batch* b, int lo, int count, float* rot, float* pos, int where) {
  for (int e = lo; e < lo + count; e++)
    for (int k = 0; k < NB; k++) {
      const float* q = &b->gc[size_t(e) * NQ];
      float* R = &rot[(size_t(e - lo) * NB + k) * 9];
      for (int r = 0; r < 9; r++) R[r] = r % 4 == 0 ? 1.f : 0.f;
      for (int r = 0; r < 3; r++) pos[(size_t(e - lo) * NB + k) * 3 + r] = q[r] + 0.1f * float(k) * float(r == 2 ? -1 : 1);
    }
  Line("rsb_batch_get_body_poses").i("lo", lo).i("count", count).i("where", where).buf("rot", rot, sizeof(float) * count * NB * 9)
      .buf("pos", pos, sizeof(float) * count * NB * 3);
  return 0;
}
int rsb_batch_get_contacts(rsb_batch* b, rsb_contact* out, int32_t* counts, int lo, int count, int where) {
  std::memset(out, 0, sizeof(rsb_contact) * count * RSB_KMAX);
  for (int e = lo; e < lo + count; e++) {
    counts[e - lo] = 1 + e % 2;
    for (int k = 0; k < counts[e - lo]; k++) {
      rsb_contact& c = out[size_t(e - lo) * RSB_KMAX + k];
      c.local_body = k + 1; c.pair_index = 0; c.normal[2] = 1.f; c.depth = 0.01f;
      for (int r = 0; r < 3; r++) { c.position[r] = b->gc[size_t(e) * NQ + r]; c.impulse[r] = b->gv[size_t(e) * NV + r]; }
    }
  }
  Line("rsb_batch_get_contacts").i("lo", lo).i("count", count).i("where", where).buf("out", out, sizeof(rsb_contact) * count * RSB_KMAX)
      .buf("counts", counts, sizeof(int32_t) * count);
  return 0;
}
int rsb_batch_get_solver_iterations(rsb_batch* b, int32_t* it, int lo, int count, int where) {
  for (int e = 0; e < count; e++) it[e] = int32_t(b->launches + e + lo);
  Line("rsb_batch_get_solver_iterations").i("lo", lo).i("count", count).i("where", where).buf("iters", it, sizeof(int32_t) * count);
  return 0;
}
int rsb_batch_set_contact_bodies(rsb_batch* b, const int32_t* body, int n) {
  b->ncb = n;
  Line("rsb_batch_set_contact_bodies").i("n", n).buf("body", body, sizeof(int32_t) * n);
  return 0;
}
int rsb_batch_get_body_contact_forces(rsb_batch* b, int lo, int count, float* force, int32_t* steps, int where) {
  for (int e = lo; e < lo + count; e++)
    for (int s = 0; s < b->ncb; s++) {
      if (force) for (int r = 0; r < 3; r++) force[(size_t(e - lo) * b->ncb + s) * 3 + r] = b->gc[size_t(e) * NQ + r] * float(s + 1);
      if (steps) steps[size_t(e - lo) * b->ncb + s] = int32_t(b->launches % 5 + s);
    }
  Line("rsb_batch_get_body_contact_forces").i("lo", lo).i("count", count).i("where", where).buf("force", force, sizeof(float) * count * b->ncb * 3)
      .buf("steps", steps, sizeof(int32_t) * count * b->ncb);
  return 0;
}
int rsb_batch_set_height_scan(rsb_batch* b, const int32_t* body, const float* xy, int n, int align) {
  b->scanPoints = n;
  Line("rsb_batch_set_height_scan").i("n", n).i("align", align).buf("body", body, sizeof(int32_t) * n).buf("xy", xy, sizeof(float) * 2 * n);
  return 0;
}
int rsb_batch_get_height_scan(rsb_batch* b, int lo, int count, float* h, float* xy, int where) {
  for (int e = lo; e < lo + count; e++)
    for (int p = 0; p < b->scanPoints; p++) {
      const float* q = &b->gc[size_t(e) * NQ];
      if (h) h[size_t(e - lo) * b->scanPoints + p] = 0.1f * q[0] - 0.2f * q[1] + 0.01f * float(p);
      if (xy) { xy[(size_t(e - lo) * b->scanPoints + p) * 2] = q[0] + float(p); xy[(size_t(e - lo) * b->scanPoints + p) * 2 + 1] = q[1]; }
    }
  Line("rsb_batch_get_height_scan").i("lo", lo).i("count", count).i("where", where).buf("h", h, sizeof(float) * count * b->scanPoints)
      .buf("xy", xy, sizeof(float) * count * b->scanPoints * 2);
  return 0;
}
int64_t rsb_batch_launch_count(const rsb_batch* b) { return b->launches; }
}  // extern "C"
