// C-ABI implementation (include/rsb.h): batch memory, model-constant blob, kernel launches.
// No CPU fallback: every compute entry point launches the sm_90a kernel or fails loudly.
#include <cuda_runtime.h>

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include "model.hpp"
#include "step_kernel.cuh"
#include "aux_kernels.cuh"
#include "ray_cast.cuh"

using namespace rsb;

static thread_local std::string g_err;
static int fail(int code, const std::string& msg) { g_err = msg; return code; }
#define CK(call)                                                                                           \
  do {                                                                                                     \
    cudaError_t e_ = (call);                                                                               \
    if (e_ != cudaSuccess) return fail(RSB_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(e_)); \
  } while (0)

struct rsb_model { Model md; };

// A device allocation of the batch: it grows on demand, never shrinks, and is freed with its owner.  A failed ensure() leaves the
// buffer as it was; a successful one that grows it does not keep the contents.
template <class T>
struct DevBuf {
  void* p = nullptr;
  size_t bytes = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { if (p) cudaFree(p); }
  T* get() const { return static_cast<T*>(p); }
  cudaError_t ensure(size_t need, cudaStream_t s) {
    if (bytes >= need) return cudaSuccess;
    void* q = nullptr;
    cudaError_t e = cudaMalloc(&q, need);
    if (e != cudaSuccess) return e;
    if (p && (e = cudaStreamSynchronize(s)) != cudaSuccess) { cudaFree(q); return e; }   // work enqueued on s may still use the old one
    if (p) cudaFree(p);
    p = q; bytes = need;
    return cudaSuccess;
  }
};

// what the batch's model and overrides decide about the step launch, built whole by rebuild() and taken by the batch only when all of
// it succeeded: the model blob (the kernel's copy is uploaded from this one), the per-warp workspace, the compiled instance and the shape
struct LaunchConfig {
  std::vector<uint32_t> blob;
  BlobHeader hdr{};
  Dims dims{};
  WsLayout ws{};
  int spec = 0;                  // 0 generic, 1 quadruped-12 static dims, 2 humanoid-30 static dims
  int slots = 1;
  int wpc = 0, grid = 0;
  size_t smem_bytes = 0;
};

// the per-batch settings the blob is built from
struct Overrides {
  std::vector<float> kp, kd;         // [nv] PD gains
  std::vector<float> pt_mu;          // [npts] terrain friction of every contact candidate (< 0: default material)
  std::vector<int32_t> self_pairs;   // [n][2] collision bodies of the enabled self-collision pairs (rsb_batch_set_self_collision)
  std::vector<float> self_mu;        // [n] their friction (< 0: default material)
};

// per-environment rows that a step launch reads in place of a batch-level value while `active` (commit_env_rows)
struct EnvRows {
  DevBuf<float> rows;
  bool active = false;
};

struct rsb_batch {
  const rsb_model* model = nullptr;
  int N = 0, device = 0;
  int nq = 0, nv = 0, nb = 0;
  int gc_stride = 0, gv_stride = 0;
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  rsb_params prm{};
  int control_mode = RSB_PD_PLUS_FEEDFORWARD_TORQUE;
  bool pd_set = false;
  const float* pt_bound = nullptr;   // caller-owned device buffer read in place of the internal PD-target rows
  int pt_bound_stride = 0;
  const float* vt_bound = nullptr;   // same for the velocity targets
  int vt_bound_stride = 0;
  // fused observation all-gather over NVLink peer memory (rsb_batch_set_observation_peers)
  int peer_world = 0, peer_rank = 0;
  float* peer_obs[MAX_PEERS][2] = {};     // [peer][buffer parity]: gathered-rows buffers, double-buffered by control step
  unsigned* peer_flag[MAX_PEERS] = {};    // [peer]: arrival counters [world]
  unsigned peer_epoch = 0;                // control steps signalled so far
  DevBuf<unsigned> peer_done;             // device counter of finished CTAs (in-kernel arrival wait)
  bool kin_dirty = true;             // the getters' buffers (M, h, poses) do not describe the current state
  bool kin_prestep = false;          // they were written by a full step (integrate2()) and hold stage A of the state before it
  unsigned* prof = nullptr;          // rsb_internal_set_profile
  unsigned* prof_a = nullptr;        // rsb_internal_set_profile_stage_a
  TerrainDesc ter{};
  DevBuf<float> hmap;
  DevBuf<int> hmap_index;            // terrain atlas: map index per environment
  std::vector<float> hmap_max;       // [maps] largest height of every map while ter.type == 2; ter.hmax is the largest of them
  DevBuf<float> ext;                 // [N][EXT_WORDS] external wrench rows; ext_active: rows hold a wrench for the next launch
  bool ext_active = false;
  // state and solver outputs, allocated and zeroed by rsb_batch_create
  DevBuf<float> gc, gv, tau, pt, vt, tau_applied, resid;
  DevBuf<int> ncontacts, contact_pt, iters, diverged, solver_status;
  DevBuf<rsb_contact> contacts;
  DevBuf<float> dbg_M, dbg_h, dbg_R, dbg_p;   // the getters' M, h and poses (ensure_debug)
  DevBuf<float> stage;               // staging()
  Overrides ovr;
  LaunchConfig cfg;
  DevBuf<uint32_t> blob;
  int64_t launches = 0;
  // RaisimGym task state (rsb_batch_gym_*)
  DevBuf<float> gym_const;           // gc_init | gv_init | action_mean | action_std
  GymConfig gym{};
  bool gym_ready = false;
  DevBuf<float> gym_action, gym_obs, gym_reward;
  DevBuf<unsigned char> gym_done;
  // frames of rsb_batch_set_frames (ftab.nf = 0: none): their table and the model's dof columns, in one device allocation
  FrameTable ftab{};
  DevBuf<int> frame_tab;
  // contact bodies of rsb_batch_set_contact_bodies (none: empty) and the rows the step kernel fills for them, tight for the current
  // list: cf_force [N][S][3], cf_steps [N][S]; allocated once, for RSB_MAX_CONTACT_BODIES
  std::vector<uint8_t> contact_bodies;
  DevBuf<float> cf_force;
  DevBuf<int> cf_steps;
  // IMU sensors of rsb_batch_set_imus (none: empty): body, position and rotation in the body frame as the kernel parameters carry them,
  // and the rows the step kernel fills, tight for the current list: imu_lin, imu_ang [N][I][3]; allocated once, for RSB_MAX_IMUS
  std::vector<uint8_t> imu_body;
  std::vector<float> imu_pos, imu_rot;
  DevBuf<float> imu_lin, imu_ang;
  // points of rsb_batch_set_height_scan (scan.n = 0: none) in one device allocation sized for RSB_MAX_SCAN_POINTS; scan_off_root: a
  // point hangs on a body whose pose comes from the kinematics pass
  ScanTable scan{};
  DevBuf<int> scan_tab;
  bool scan_off_root = false;
  // rays of rsb_batch_set_rays (rays.n = 0: none) and the model's collision bodies, in one device allocation sized for RSB_MAX_RAYS;
  // ray_kin: a ray's pose comes from the kinematics pass
  RayTable rays{};
  DevBuf<float> ray_tab;
  bool ray_kin = false;
  // per-environment rows: inertial ones of rsb_batch_set_body_inertia [N][nb][BI_WORDS], terrain friction of
  // rsb_batch_set_contact_friction [N][ncoll], kp | kd | effort limit of rsb_batch_set_actuator_params [N][3][nv]; row_bad: the verdict
  // of the check a call's rows pass before they replace any of them
  EnvRows body_inertia, contact_friction, actuator;
  DevBuf<int> row_bad;
  // learned actuator network of rsb_batch_set_actuator_network (an_lstm false) or rsb_batch_set_actuator_lstm (an_lstm true; an_dofs
  // empty: none): its parameters as the step kernel reads them (ActNetDesc::params) and the history rows, [N][n][2][H - 1] for the MLP,
  // [N][n][L][2][W] for the LSTM
  std::vector<int32_t> an_dofs;
  bool an_lstm = false;
  int an_H = 0, an_L = 0, an_W = 0;
  DevBuf<float> an_params, an_hist;
  // actuation delays of rsb_batch_set_actuation_delay while delay_active: (delay, sub-steps since the history was emptied) rows [N][2]
  // and the command rings [N][DELAY_SLOTS][3][nv - nbase] (StepArgs::delay_state, delay_ring)
  DevBuf<int> delay_state;
  DevBuf<float> delay_ring;
  bool delay_active = false;
};

static int round_up(int x, int m) { return (x + m - 1) / m * m; }
// the step kernel applies PD laws: PD mode, and gains from rsb_batch_set_pd_gains, per-environment actuator rows or an actuator network
static bool pd_active(const rsb_batch* b) {
  return b->control_mode == RSB_PD_PLUS_FEEDFORWARD_TORQUE && (b->pd_set || b->actuator.active || !b->an_dofs.empty());
}
// words of one environment's actuator history rows (the LSTM's (h, c) of every layer)
static size_t an_hist_words(const rsb_batch* b) {
  return b->an_dofs.size() * 2 * (b->an_lstm ? (size_t)b->an_L * b->an_W : (size_t)std::max(0, b->an_H - 1));
}

// ------------------------------------------------------------------ blob ------------------------
static void build_blob(const Model& md, const Overrides& ov, LaunchConfig& cfg) {
  BlobHeader& H = cfg.hdr;
  // dof tree: a floating base is a chain of 6 dofs; dof order is DFS pre-order so subtrees are contiguous
  const int nv = md.nv;
  std::vector<int> dparent(std::max(1, nv), -1), ddepth(std::max(1, nv), 0), dsub(std::max(1, nv), 1), dbody(std::max(1, nv), 0), bdof(md.nb, -1);
  const int nbase = md.floating ? 6 : 0;
  for (int k = 1; k < nbase; k++) dparent[k] = k - 1;
  if (md.floating) bdof[0] = 5;
  for (int i = 1; i < md.nb; i++) {
    bdof[i] = md.vidx[i]; dbody[md.vidx[i]] = i;
    dparent[md.vidx[i]] = bdof[md.parent[i]];
  }
  int maxdd = 0;
  for (int i = 0; i < nv; i++) { ddepth[i] = dparent[i] >= 0 ? ddepth[dparent[i]] + 1 : 0; maxdd = std::max(maxdd, ddepth[i]); }
  for (int i = nv - 1; i > 0; i--) if (dparent[i] >= 0) dsub[dparent[i]] += dsub[i];
  const int DL = maxdd + 1;
  std::vector<int> lvl(DL + 1, 0), lvldofs, entstart(DL + 1, 0), ent;
  for (int d = 0; d < DL; d++) {
    lvl[d] = (int)lvldofs.size(); entstart[d] = (int)ent.size();
    for (int i = 0; i < nv; i++) if (ddepth[i] == d) { lvldofs.push_back(i); for (int t = 0; t <= d; t++) ent.push_back(i | (t << 8)); }
  }
  lvl[DL] = (int)lvldofs.size(); entstart[DL] = (int)ent.size();
  cfg.dims = Dims{md.nb, md.nq, md.nv, md.floating, md.maxdepth, maxdd};
  const int npairs = (int)ov.self_mu.size();
  H = make_blob_header(cfg.dims, md.npts(), (int)ent.size(), md.ncoll(), npairs);
  {
    bool ident = true;
    for (int i = 1; i < md.nb; i++) for (int k = 0; k < 9; k++) if (std::fabs(md.jrot[9 * i + k] - ((k % 4 == 0) ? 1.0 : 0.0)) > 0.0) ident = false;
    int max_inner = 0;
    for (int i = 1; i < md.nb; i++) max_inner = std::max(max_inner, md.subtree[i] - 1);
    H.flags = (ident ? 1 : 0) | (max_inner << 8);
  }
  const int words = H.words;
  std::vector<uint32_t>& B = cfg.blob;
  B.assign(words, 0u);
  auto F = [&](int o, float v) { std::memcpy(&B[o], &v, 4); };
  auto I = [&](int o, int v) { std::memcpy(&B[o], &v, 4); };
  const int nbp = H.nbp;
  for (int i = 0; i < md.nb; i++) {
    I(H.off_body + BF_PARENT * nbp + i, md.parent[i]); I(H.off_body + BF_JTYPE * nbp + i, md.jtype[i]);
    I(H.off_body + BF_QIDX * nbp + i, md.qidx[i]); I(H.off_body + BF_VIDX * nbp + i, md.vidx[i]);
    I(H.off_body + BF_DEPTH * nbp + i, md.depth[i]); I(H.off_body + BF_SUBTREE * nbp + i, md.subtree[i]);
    for (int k = 0; k < 3; k++) F(H.off_body + (BF_JPOS + k) * nbp + i, (float)md.jpos[3 * i + k]);
    for (int k = 0; k < 9; k++) F(H.off_body + (BF_JROT + k) * nbp + i, (float)md.jrot[9 * i + k]);
    for (int k = 0; k < 3; k++) F(H.off_body + (BF_AXIS + k) * nbp + i, (float)md.axis[3 * i + k]);
    F(H.off_body + BF_MASS * nbp + i, (float)md.mass[i]);
    for (int k = 0; k < 3; k++) F(H.off_body + (BF_COM + k) * nbp + i, (float)md.com[3 * i + k]);
    for (int k = 0; k < 6; k++) F(H.off_body + (BF_INERTIA + k) * nbp + i, (float)md.inertia[6 * i + k]);
    F(H.off_body + BF_LO * nbp + i, (float)std::max(-3.0e38, md.jlimit[2 * i])); F(H.off_body + BF_HI * nbp + i, (float)std::min(3.0e38, md.jlimit[2 * i + 1]));
    // ancestor at depth d (d = 1..depth[i]) stored at anc[(d-1)*nbp + i]
    for (int d = 0; d < std::max(1, md.maxdepth); d++) I(H.off_anc + d * nbp + i, -1);
    for (int j = i; md.parent[j] >= 0; j = md.parent[j]) I(H.off_anc + (md.depth[j] - 1) * nbp + i, j);
  }
  for (int k = 0; k < md.npts(); k++) {
    I(H.off_pts + 0 * H.nptp + k, md.pt_body[k]);
    for (int q = 0; q < 3; q++) F(H.off_pts + (1 + q) * H.nptp + k, (float)md.pt_pos[3 * k + q]);
    F(H.off_pts + 4 * H.nptp + k, (float)md.pt_rad[k]);
    F(H.off_pts + 5 * H.nptp + k, ov.pt_mu[k]);
    I(H.off_pts + 6 * H.nptp + k, md.pt_type[k]);
    for (int q = 0; q < 3; q++) F(H.off_pts + (7 + q) * H.nptp + k, (float)md.pt_pos2[3 * k + q]);
    I(H.off_pts + 10 * H.nptp + k, md.pt_coll[k]);
    // bounding sphere of the candidate for the height cull of stage B: the sphere itself / the rim circle, the whole capsule, the whole box
    double cc[3] = {md.pt_pos[3 * k], md.pt_pos[3 * k + 1], md.pt_pos[3 * k + 2]}, cr = md.pt_rad[k];
    if (md.pt_type[k] == FT_SEGMENT) {
      double hl = 0;
      for (int q = 0; q < 3; q++) { cc[q] = 0.5 * (md.pt_pos[3 * k + q] + md.pt_pos2[3 * k + q]); const double d = md.pt_pos2[3 * k + q] - md.pt_pos[3 * k + q]; hl += d * d; }
      cr = md.pt_rad[k] + 0.5 * std::sqrt(hl);
    } else if (md.pt_type[k] == FT_BOXFACE) {
      const double* sz = &md.csize[3 * md.pt_coll[k]];
      cr = std::sqrt(sz[0] * sz[0] + sz[1] * sz[1] + sz[2] * sz[2]);
    }
    if (bdof[md.pt_body[k]] < 0) cr = -3.0e38;         // welded to the world: cannot collide
    for (int q = 0; q < 3; q++) F(H.off_pts + (11 + q) * H.nptp + k, (float)cc[q]);
    F(H.off_pts + 14 * H.nptp + k, (float)(cr * 1.0001 + 1e-6));   // float32 rounding of the product must never cull a touching candidate
  }
  for (int c = 0; c < md.ncoll(); c++) {   // collision-body table (box features): half extents, body-frame position and rotation
    for (int q = 0; q < 3; q++) { F(H.off_coll + COLL_WORDS * c + q, (float)md.csize[3 * c + q]); F(H.off_coll + COLL_WORDS * c + 3 + q, (float)md.cpos[3 * c + q]); }
    for (int q = 0; q < 9; q++) F(H.off_coll + COLL_WORDS * c + 6 + q, (float)md.crot[9 * c + q]);
  }
  for (int i = 0; i < md.nv; i++) {
    F(H.off_gain + i, ov.kp[i]); F(H.off_gain + H.nvp + i, ov.kd[i]); F(H.off_gain + 2 * H.nvp + i, 3.0e38f);
    I(H.off_dofq + i, -1);
  }
  for (int i = 1; i < md.nb; i++) F(H.off_gain + 2 * H.nvp + md.vidx[i], (float)std::min(md.jeffort[i], 3.0e38));   // actuator effort limit per dof
  for (int i = 1; i < md.nb; i++) I(H.off_dofq + md.vidx[i], md.qidx[i]);
  for (int i = 0; i < nv; i++) {
    I(H.off_ddepth + i, ddepth[i]); I(H.off_dsub + i, dsub[i]); I(H.off_dbody + i, dbody[i]);
    int a = i;
    for (int t = ddepth[i]; t >= 0; t--) { I(H.off_danc + t * H.nvp + i, a); a = dparent[a]; }
  }
  for (int i = 0; i < md.nb; i++) I(H.off_bdof + i, bdof[i]);
  for (int d = 0; d <= DL; d++) { I(H.off_lvl + d, lvl[d]); I(H.off_entstart + d, entstart[d]); }
  for (size_t k = 0; k < lvldofs.size(); k++) I(H.off_lvldofs + (int)k, lvldofs[k]);
  for (size_t k = 0; k < ent.size(); k++) I(H.off_ent + (int)k, ent[k]);
  {   // depth (in the dof tree) of the lowest common ancestor dof of two bodies; -1 when they share none
    int8_t* tab = reinterpret_cast<int8_t*>(&B[H.off_lcad]);
    for (int a = 0; a < md.nb; a++) for (int c = 0; c < md.nb; c++) {
      int x = a, y = c;
      while (x != y) { if (md.depth[x] >= md.depth[y]) x = md.parent[x]; else y = md.parent[y]; }
      tab[a * H.nbp + c] = (int8_t)(bdof[x] >= 0 ? ddepth[bdof[x]] : -1);
    }
  }
  for (int r = 0; r < NROUNDS; r++) {
    double width = 2.0 * M_PI / std::pow((double)NSEC, r);
    for (int k = 0; k <= NSEC; k++) {
      F(H.off_sec + r * SEC_STRIDE + k, (float)std::cos(width * k / NSEC));
      F(H.off_sec + NROUNDS * SEC_STRIDE + r * SEC_STRIDE + k, (float)std::sin(width * k / NSEC));
    }
  }
  for (int j = 0; j < npairs; j++) {   // self-collision pairs (PairField): spheres and capsules as swept segments, sphere-box with the sphere in A
    const int c1 = ov.self_pairs[2 * j], c2 = ov.self_pairs[2 * j + 1];
    const bool box = md.ctype[c1] == CT_BOX || md.ctype[c2] == CT_BOX, flip = md.ctype[c1] == CT_BOX;
    const int ca = flip ? c2 : c1, cb = flip ? c1 : c2;
    const int o = H.off_pair + PAIR_WORDS * j;
    I(o + PR_KIND, box ? 1 : 0); I(o + PR_FLIP, flip ? 1 : 0); I(o + PR_BODY1, md.cbody[c1]); I(o + PR_BODY2, md.cbody[c2]);
    I(o + PR_BA, md.cbody[ca]); I(o + PR_BB, md.cbody[cb]);
    // segment ends in the body frame: centre -/+ half length along the shape's z axis (a sphere: both ends at the centre)
    auto seg = [&](int c, int f0, int f1, double& half) {
      const double* p = &md.cpos[3 * c]; const double* R = &md.crot[9 * c];
      half = md.ctype[c] == CT_CAPSULE ? md.csize[3 * c + 1] : 0.0;
      for (int q = 0; q < 3; q++) { F(o + f0 + q, (float)(p[q] - half * R[3 * q + 2])); F(o + f1 + q, (float)(p[q] + half * R[3 * q + 2])); }
    };
    double ha = 0, hb = 0;
    seg(ca, PR_A0, PR_A1, ha);
    F(o + PR_RA, (float)md.csize[3 * ca]);
    double cull_b;
    if (box) {
      for (int q = 0; q < 3; q++) { F(o + PR_B0 + q, (float)md.cpos[3 * cb + q]); F(o + PR_B1 + q, (float)md.csize[3 * cb + q]); }
      for (int q = 0; q < 9; q++) F(o + PR_BR + q, (float)md.crot[9 * cb + q]);
      F(o + PR_RB, 0.f);
      cull_b = std::sqrt(md.csize[3 * cb] * md.csize[3 * cb] + md.csize[3 * cb + 1] * md.csize[3 * cb + 1] + md.csize[3 * cb + 2] * md.csize[3 * cb + 2]);
    } else {
      seg(cb, PR_B0, PR_B1, hb);
      for (int q = 0; q < 9; q++) F(o + PR_BR + q, q % 4 == 0 ? 1.f : 0.f);
      F(o + PR_RB, (float)md.csize[3 * cb]);
      cull_b = md.csize[3 * cb] + hb;
    }
    F(o + PR_MU, ov.self_mu[j]);
    // bounding spheres of the stage-B cull, widened so that float32 rounding never culls a touching pair
    F(o + PR_CULL_A, (float)((md.csize[3 * ca] + ha) * 1.0001 + 1e-6)); F(o + PR_CULL_B, (float)(cull_b * 1.0001 + 1e-6));
  }
  std::memcpy(B.data(), &H, sizeof(H));
}

// ------------------------------------------------------------------ launches --------------------
template <int WPC, int SLOTS, int SPEC>
static cudaError_t launch_step(const StepArgs& a, int grid, size_t smem, cudaStream_t s) {
  auto kern = a.delay_state ? (a.an.params ? rsb_step_kernel<WPC, SLOTS, SPEC, true, true> : rsb_step_kernel<WPC, SLOTS, SPEC, false, true>)
                            : (a.an.params ? rsb_step_kernel<WPC, SLOTS, SPEC, true, false> : rsb_step_kernel<WPC, SLOTS, SPEC, false, false>);
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  kern<<<grid, WPC * 32, smem, s>>>(a);
  return cudaGetLastError();
}

extern "C" int rsb_batch_ob_dim(const rsb_batch* b);

static int pick_config(const rsb_batch* b, LaunchConfig& c) {
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, b->device));
  // sm_90a code runs on compute capability 9.0 only (arch-specific features are not forward compatible)
  if (prop.major != 9 || prop.minor != 0)
    return fail(RSB_ERR_UNSUPPORTED, "raisimlib_b200 is compiled for sm_90a and needs an H100-class device (compute capability 9.0); found sm_" + std::to_string(prop.major) + std::to_string(prop.minor));
  const size_t budget = prop.sharedMemPerBlockOptin;   // 227 KB on H100
  const size_t blob_bytes = (size_t)c.blob.size() * 4;
  const size_t per_warp = (size_t)c.ws.words * 4;
  const int sms = prop.multiProcessorCount;
  c.slots = b->model->md.npts() > 32 ? 2 : 1;
  // the static instance of the model's dimensions (step_kernel.cuh SPEC_DIMS), if any
  c.spec = SPEC_GENERIC;
  for (int s = SPEC_GENERIC + 1; s < SPEC_COUNT; s++)
    if (c.dims == SPEC_DIMS[s]) c.spec = s;
  // the quadruped instance has the topology compiled in (floating base + 4 serial chains of 3 joints in DFS order): check it
  if (c.spec == SPEC_QUAD) {
    const Model& md = b->model->md;
    for (int leg = 0; leg < 4; leg++)
      for (int j = 0; j < 3; j++) {
        const int body = 1 + 3 * leg + j;
        if (md.parent[body] != (j == 0 ? 0 : body - 1) || md.vidx[body] != 5 + body || md.qidx[body] != 6 + body) c.spec = SPEC_GENERIC;
        if (md.jtype[body] != 1 && md.jtype[body] != 2) c.spec = SPEC_GENERIC;
      }
  }
  if (const char* e = getenv("RSB_FORCE_GENERIC")) if (atoi(e)) c.spec = SPEC_GENERIC;
  if (c.hdr.npairs > 0) c.spec = SPEC_GENERIC;   // self-collision pairs are compiled into the generic instance only
  // Warps per CTA (= resident environments per CTA).  A round of w resident warps per SM costs ~ max(13, w): latency-bound up to a
  // dozen warps, issue-bound beyond.  Choose the option with the smallest rounds x cost, ties to the larger CTA (one sub-step
  // barrier group, one copy of the model block).  On the 132 SMs of an H100, 4096 ANYmal-like environments (7.5 KB workspaces, at
  // most 29 per SM) take two rounds whatever the CTA: 16 (a round of 2112 and one of 1984, each re-aligned at every sub-step:
  // 0.197 ms per control step of 4 sub-steps at 400 W) rather than 28 (a full round and an 11 % one, 0.282 ms), 14 (two CTAs per SM,
  // 0.248 ms) or 8 (four rounds, 0.312 ms); the model ranks 8 above 14 and 28 (52 against 56) and is only checked to pick the
  // fastest, 16.  4096 Atlas-like ones (10.9 KB workspaces): 16 as well (1.41 ms, against 1.68 ms with 14, measured without the
  // sub-step barrier).  One warp per environment: the choice does not change the results (every option that fits, for every compiled instance:
  // tests/test_gpu_instances.py::test_warps_per_cta_bit_identical).
  static const int options[] = {28, 16, 14, 8, 4, 1};
  int best = 0; long best_cost = 0;
  for (int w : options) {
    const size_t cta_bytes = blob_bytes + (size_t)w * per_warp + 1024;
    if (cta_bytes > budget) continue;
    const int ctas = (w == 14 && 2 * cta_bytes <= (size_t)prop.sharedMemPerMultiprocessor) ? 2 : 1;   // 14-warp CTAs are compiled for two per SM
    const long resident = (long)sms * w * ctas;
    const long rounds = (b->N + resident - 1) / resident;
    const long cost = rounds * std::max(13L, (long)w * ctas);
    if (best == 0 || cost < best_cost) { best = w; best_cost = cost; }
  }
  if (const char* e = getenv("RSB_FORCE_WPC")) { int w = atoi(e); if (w == 28 || w == 16 || w == 14 || w == 8 || w == 4 || w == 1) if (blob_bytes + (size_t)w * per_warp + 1024 <= budget) best = w; }
  if (best == 0) return fail(RSB_ERR_UNSUPPORTED, "model too large for one warp's shared-memory workspace");
  c.wpc = best;
  c.grid = std::min((b->N + best - 1) / best, best == 14 ? 2 * sms : sms);
  c.smem_bytes = blob_bytes + (size_t)best * per_warp;
  return RSB_OK;
}

// the launch configuration of overrides `ov`, uploaded on the batch's stream; the batch takes both only when all of it succeeded, so a
// refused or failed call leaves the batch as it was
static int rebuild(rsb_batch* b, Overrides ov) {
  CK(cudaSetDevice(b->device));
  LaunchConfig c;
  build_blob(b->model->md, ov, c);
  c.ws = make_ws_layout(c.dims, c.hdr.npairs);
  int rc = pick_config(b, c); if (rc) return rc;
  CK(b->blob.ensure(c.blob.size() * 4, b->stream));
  CK(cudaMemcpyAsync(b->blob.get(), c.blob.data(), c.blob.size() * 4, cudaMemcpyHostToDevice, b->stream));
  b->ovr = std::move(ov);
  b->cfg = std::move(c);
  return RSB_OK;
}

template <int WPC>
static cudaError_t dispatch_spec(const rsb_batch* b, const StepArgs& a) {
  const LaunchConfig& c = b->cfg;
  if (c.spec == SPEC_QUAD && c.slots == 1) return launch_step<WPC, 1, SPEC_QUAD>(a, c.grid, c.smem_bytes, b->stream);
  if (c.spec == SPEC_QUAD) return launch_step<WPC, 2, SPEC_QUAD>(a, c.grid, c.smem_bytes, b->stream);
  if (c.spec == SPEC_HUMANOID) return launch_step<WPC, 2, SPEC_HUMANOID>(a, c.grid, c.smem_bytes, b->stream);
  if (c.slots == 1) return launch_step<WPC, 1, SPEC_GENERIC>(a, c.grid, c.smem_bytes, b->stream);
  return launch_step<WPC, 2, SPEC_GENERIC>(a, c.grid, c.smem_bytes, b->stream);
}

// what one launch reads or writes besides the batch's own rows and bindings
struct LaunchIO {
  const float* pt = nullptr;     // PD-target rows read in place for this launch only (pinned host rows), stored into the batch's own rows
  const float* vt = nullptr;     // the same for the velocity targets
  float* obs = nullptr;          // observation rows
  bool peers = false;            // ... gathered into the peers' buffers (rsb_batch_set_observation_peers)
  const float* gym_action = nullptr;   // rsb_batch_gym_step: the task fused into the step launch
  float* gym_reward = nullptr;
  unsigned char* gym_done = nullptr;
};

static int do_launch(rsb_batch* b, int substeps, int phase_mask, bool debug, const LaunchIO& io = {}) {
  StepArgs a{};
  a.num_envs = b->N; a.substeps = substeps;
  a.gc_stride = b->gc_stride; a.gv_stride = b->gv_stride;
  a.gc = b->gc.get(); a.gv = b->gv.get(); a.tau = b->tau.get();
  a.use_pd = pd_active(b) ? 1 : 0;
  a.ptarget = b->pt_bound ? b->pt_bound : b->pt.get(); a.pt_stride = b->pt_bound ? b->pt_bound_stride : b->gc_stride;
  a.vtarget = b->vt_bound ? b->vt_bound : b->vt.get(); a.vt_stride = b->vt_bound ? b->vt_bound_stride : b->gv_stride;
  if (io.pt) { a.ptarget = io.pt; a.pt_stride = b->nq; a.pt_store = b->pt.get(); }
  if (io.vt) { a.vtarget = io.vt; a.vt_stride = b->nv; a.vt_store = b->vt.get(); }
  a.prm = b->prm; a.ter = b->ter; a.ws = b->cfg.ws;
  a.blob_words = (int)b->cfg.blob.size(); a.blob = b->blob.get();
  a.tau_applied = b->tau_applied.get();
  if (phase_mask == 0 && !b->contact_bodies.empty()) {   // only a launch that advances the state accumulates (and overwrites) the contact forces
    a.cf_force = b->cf_force.get(); a.cf_steps = b->cf_steps.get(); a.cf_n = (int)b->contact_bodies.size();
    std::memcpy(a.cf_body, b->contact_bodies.data(), b->contact_bodies.size());
  }
  if (phase_mask == 0 && !b->imu_body.empty()) {   // likewise the IMU readings
    a.imu_lin = b->imu_lin.get(); a.imu_ang = b->imu_ang.get(); a.imu_n = (int)b->imu_body.size();
    std::memcpy(a.imu_body, b->imu_body.data(), b->imu_body.size());
    std::memcpy(a.imu_pos, b->imu_pos.data(), b->imu_pos.size() * 4);
    std::memcpy(a.imu_rot, b->imu_rot.data(), b->imu_rot.size() * 4);
  }
  a.ncontacts = b->ncontacts.get(); a.contacts = b->contacts.get(); a.contact_pt = b->contact_pt.get(); a.iters = b->iters.get(); a.diverged = b->diverged.get();
  a.resid = b->resid.get(); a.solver_status = b->solver_status.get();
  if (debug) { a.dbg_M = b->dbg_M.get(); a.dbg_h = b->dbg_h.get(); a.dbg_R = b->dbg_R.get(); a.dbg_p = b->dbg_p.get(); }
  a.phase_mask = phase_mask; a.prof = b->prof; a.prof_a = b->prof_a;
  a.ext = b->ext_active ? b->ext.get() : nullptr;
  a.body_inertia = b->body_inertia.active ? b->body_inertia.rows.get() : nullptr;
  a.contact_friction = b->contact_friction.active ? b->contact_friction.rows.get() : nullptr;
  a.actuator = b->actuator.active ? b->actuator.rows.get() : nullptr;
  if (!b->an_dofs.empty() && a.use_pd) {   // the network and its history act in PD mode only
    a.an.params = b->an_params.get(); a.an.hist = b->an_hist.get();
    a.an.n = (int)b->an_dofs.size(); a.an.H = b->an_H; a.an.L = b->an_L; a.an.W = b->an_W;
    a.an.lstm = b->an_lstm ? 1 : 0; a.an.words = (int)an_hist_words(b);
    for (int s = 0; s < a.an.n; s++) { a.an.dof[s] = (uint8_t)b->an_dofs[s]; a.an.mask |= 1ull << b->an_dofs[s]; }
  }
  if (b->delay_active && phase_mask == 0) { a.delay_state = b->delay_state.get(); a.delay_ring = b->delay_ring.get(); }   // only advancing launches record a command
  a.obs = io.obs; a.ob_dim = rsb_batch_ob_dim(b);
  if (io.gym_action) {   // targets come from the action rows and are kept in the batch's own rows; terminated environments get their reset target there too
    a.gym_action = io.gym_action; a.gym = b->gym; a.gym_reward = io.gym_reward; a.gym_done = io.gym_done;
    a.ptarget = b->pt.get(); a.pt_stride = b->gc_stride; a.pt_store = b->pt.get();
  }
  if (io.peers && b->peer_world > 0 && io.obs && phase_mask == 0) {
    a.peer_world = b->peer_world; a.peer_rank = b->peer_rank;
    for (int p = 0; p < b->peer_world; p++) { a.peer_obs[p] = b->peer_obs[p][b->peer_epoch & 1]; a.peer_flag[p] = b->peer_flag[p]; }
    b->peer_epoch++;
    a.peer_expected = b->peer_epoch * (unsigned)b->cfg.grid; a.peer_done = b->peer_done.get();
  }
  if (phase_mask == 0) {   // every round of warps re-aligns at each sub-step (the kernel counts the warps of the round)
    const char* e = getenv("RSB_SUBSTEP_BARRIER");   // 0 = off, for A/B runs
    a.substep_barrier = e ? atoi(e) != 0 : 1;
    const char* p = getenv("RSB_PAIR_STAGE_A");   // quadruped instance: one warp runs stage A of two environments (0 = off, for A/B runs)
    a.pair_stage_a = p ? atoi(p) : 1;
  }
  cudaError_t e;
  switch (b->cfg.wpc) {
    case 28: e = dispatch_spec<28>(b, a); break;
    case 16: e = dispatch_spec<16>(b, a); break;
    case 14: e = dispatch_spec<14>(b, a); break;
    case 8: e = dispatch_spec<8>(b, a); break;
    case 4: e = dispatch_spec<4>(b, a); break;
    default: e = dispatch_spec<1>(b, a); break;
  }
  if (e != cudaSuccess) return fail(RSB_ERR_CUDA, std::string("step kernel launch: ") + cudaGetErrorString(e));
  b->launches++;
  if (!(phase_mask & PHASE_NO_UPDATE)) { b->kin_dirty = !debug; b->kin_prestep = debug; }   // the state advanced: M, h and poses are stale unless this launch refreshed them
  else if (debug) { b->kin_dirty = false; b->kin_prestep = false; }
  if (phase_mask == 0) b->ext_active = false;   // an external wrench lasts for one integrate() call (upstream semantics)
  return RSB_OK;
}

// The device buffer that host rows pass through on their way to or from the batch.  Every use is on the batch's stream, so stream
// order keeps one use apart from the next; a pointer from here is valid until the next call, which may move the buffer.  It starts
// with room for the rows of any state, target or force copy, so a steady loop of those never grows it.  Null (message set) on failure.
static float* staging(rsb_batch* b, size_t words) {
  const cudaError_t e = b->stage.ensure(std::max(words, (size_t)b->N * 64 + 64) * 4, b->stream);
  if (e != cudaSuccess) { fail(RSB_ERR_CUDA, std::string("staging buffer: ") + cudaGetErrorString(e)); return nullptr; }
  return b->stage.get();
}
// device -> the caller's buffer (where: RSB_HOST / RSB_DEVICE); a host destination has been written when this returns
static int copy_out(rsb_batch* b, void* dst, const void* src, size_t bytes, int where) {
  CK(cudaMemcpyAsync(dst, src, bytes, where == RSB_HOST ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice, b->stream));
  if (where == RSB_HOST) CK(cudaStreamSynchronize(b->stream));
  return RSB_OK;
}
// device-side alias of a pinned, mapped host allocation (cudaHostAlloc / cudaHostRegister / torch pin_memory); null otherwise
static const float* mapped_alias(const void* host) {
  cudaPointerAttributes at{};
  if (cudaPointerGetAttributes(&at, host) != cudaSuccess) { cudaGetLastError(); return nullptr; }
  if (at.type == cudaMemoryTypeHost && at.devicePointer) return static_cast<const float*>(at.devicePointer);
  return nullptr;
}
// rows: tight [n][w] <-> padded [n][stride].  Host buffers go through one CONTIGUOUS PCIe copy into the staging buffer and are
// (un)padded on the device: pitched H2D/D2H copies of 76-byte rows are slow.
static int copy_rows_in(rsb_batch* b, float* dst, int stride, const float* src, int w, int env_begin, int n, int where) {
  if (!src || n == 0) return RSB_OK;
  const float* dsrc = src;
  if (where == RSB_HOST) {
    float* st = staging(b, (size_t)n * w); if (!st) return RSB_ERR_CUDA;
    CK(cudaMemcpyAsync(st, src, (size_t)n * w * 4, cudaMemcpyHostToDevice, b->stream));
    dsrc = st;
  }
  CK(cudaMemcpy2DAsync(dst + (size_t)env_begin * stride, (size_t)stride * 4, dsrc, (size_t)w * 4, (size_t)w * 4, n, cudaMemcpyDeviceToDevice, b->stream));
  return RSB_OK;
}
static int copy_rows_out(rsb_batch* b, float* dst, const float* src, int stride, int w, int env_begin, int n, int where) {
  if (!dst || n == 0) return RSB_OK;
  if (where == RSB_HOST) {
    float* st = staging(b, (size_t)n * w); if (!st) return RSB_ERR_CUDA;
    CK(cudaMemcpy2DAsync(st, (size_t)w * 4, src + (size_t)env_begin * stride, (size_t)stride * 4, (size_t)w * 4, n, cudaMemcpyDeviceToDevice, b->stream));
    CK(cudaMemcpyAsync(dst, st, (size_t)n * w * 4, cudaMemcpyDeviceToHost, b->stream));
  } else {
    CK(cudaMemcpy2DAsync(dst, (size_t)w * 4, src + (size_t)env_begin * stride, (size_t)stride * 4, (size_t)w * 4, n, cudaMemcpyDeviceToDevice, b->stream));
  }
  return RSB_OK;
}
static bool bad_where(int where) { return where != RSB_HOST && where != RSB_DEVICE; }
// the checks of every entry point that copies rows of a range of environments to or from the caller's memory
static int check_range(const rsb_batch* b, int env_begin, int env_count, int where) {
  if (!b) return fail(RSB_ERR_INVALID, "null batch");
  if (env_begin < 0 || env_count < 0 || env_begin + env_count > b->N) return fail(RSB_ERR_INVALID, "environment range out of bounds");
  if (bad_where(where)) return fail(RSB_ERR_INVALID, "`where` must be RSB_HOST or RSB_DEVICE");
  return RSB_OK;
}

// The staging and verdict part of every call that checks the caller's values on the device before any of them is committed
// (commit_env_rows, rsb_batch_set_heightmap_index, rsb_batch_update_heightmaps).  The caller's src_words (host or device memory, 4-byte
// elements) are checked and packed to out_words in the staging buffer by check(out, src, verdict), and the call waits for the verdict.
// A host source is copied into the staging buffer first: behind the checked words, or, with in_place (the check copies element i to
// element i), onto them, so that the buffer grows to out_words only.  verdict[0] stays ROWS_OK when every value is accepted;
// verdict[1 .. extra] start at INT_MIN for what the check gathers with atomicMax.  On success *staged holds the checked words, valid
// until the next use of the staging buffer; a refused value fails the call with RSB_ERR_INVALID and what(verdict[0]).
static constexpr int ROWS_OK = 0x7fffffff;
template <class T, class Check, class What>
static int stage_checked(rsb_batch* b, const T* src, size_t out_words, size_t src_words, int where, bool in_place, int extra, Check check,
                         What what, T** staged, std::vector<int>* verdict = nullptr) {
  static_assert(sizeof(T) == 4, "the staging buffer holds 4-byte words");
  CK(b->row_bad.ensure((size_t)(1 + extra) * 4, b->stream));
  const bool host = where == RSB_HOST;
  float* const stf = staging(b, out_words + (host && !in_place ? src_words : 0)); if (!stf) return RSB_ERR_CUDA;
  T* const st = reinterpret_cast<T*>(stf);
  const T* dsrc = src;
  if (host) {
    T* const to = in_place ? st : st + out_words;
    CK(cudaMemcpyAsync(to, src, src_words * 4, cudaMemcpyHostToDevice, b->stream));
    dsrc = to;
  }
  std::vector<int> v(1 + extra, INT_MIN);
  v[0] = ROWS_OK;
  CK(cudaMemcpyAsync(b->row_bad.get(), v.data(), v.size() * 4, cudaMemcpyHostToDevice, b->stream));
  if (src_words > 0) { check(st, dsrc, b->row_bad.get()); CK(cudaGetLastError()); }
  CK(cudaMemcpyAsync(v.data(), b->row_bad.get(), v.size() * 4, cudaMemcpyDeviceToHost, b->stream));
  CK(cudaStreamSynchronize(b->stream));
  if (v[0] != ROWS_OK) return fail(RSB_ERR_INVALID, what(v[0]));
  *staged = st;
  if (verdict) *verdict = std::move(v);
  return RSB_OK;
}

// The one path by which a call's per-environment rows reach an EnvRows table (rsb_batch_set_body_inertia, set_contact_friction,
// set_actuator_params).
// `dflt` is one environment's row of the table (w words) when nothing overrides it: every environment starts from it at the first commit
// after creation or a clear, and rows == null writes it to the range.  Otherwise the caller's rows (src_w words per environment) are
// checked and packed to w words by check(out, src, env_count, bad) through stage_checked; a refused row changes nothing of the table and
// the call fails with what(verdict).
static std::vector<float> repeat_row(const std::vector<float>& row, size_t n) {
  std::vector<float> r(n * row.size());
  for (size_t e = 0; e < n; e++) std::copy(row.begin(), row.end(), r.begin() + e * row.size());
  return r;
}
template <class Check, class What>
static int commit_env_rows(rsb_batch* b, EnvRows& t, const std::vector<float>& dflt, const float* rows, int env_begin, int env_count, int where,
                           size_t src_w, Check check, What what) {
  int rc = check_range(b, env_begin, env_count, where); if (rc) return rc;
  if (env_count == 0) return RSB_OK;
  CK(cudaSetDevice(b->device));
  const size_t w = dflt.size(), n = (size_t)env_count;
  float* staged = nullptr;
  std::vector<float> reset;
  if (rows) {
    rc = stage_checked(b, rows, n * w, n * src_w, where, false, 0, [&](float* out, const float* src, int* bad) { check(out, src, env_count, bad); },
                       [&](int bad) { return what(bad) + "; no row changed"; }, &staged);
    if (rc) return rc;
  } else {
    reset = repeat_row(dflt, n);
  }
  CK(t.rows.ensure((size_t)b->N * w * 4, b->stream));
  if (!t.active) {
    const std::vector<float> init = repeat_row(dflt, (size_t)b->N);
    CK(cudaMemcpyAsync(t.rows.get(), init.data(), init.size() * 4, cudaMemcpyHostToDevice, b->stream));
    CK(cudaStreamSynchronize(b->stream));   // the pageable source goes out of scope here
  }
  float* const at = t.rows.get() + (size_t)env_begin * w;
  if (staged) CK(cudaMemcpyAsync(at, staged, n * w * 4, cudaMemcpyDeviceToDevice, b->stream));
  else {
    CK(cudaMemcpyAsync(at, reset.data(), reset.size() * 4, cudaMemcpyHostToDevice, b->stream));
    CK(cudaStreamSynchronize(b->stream));
  }
  t.active = true;
  return RSB_OK;
}

extern "C" {

const char* rsb_last_error(void) { return g_err.c_str(); }
int rsb_version(void) { return 100; }

int rsb_params_default(rsb_params* p) {
  if (!p) return fail(RSB_ERR_INVALID, "null params");
  p->dt = 0.0025f; p->gravity[0] = 0.f; p->gravity[1] = 0.f; p->gravity[2] = -9.81f; p->erp = 0.f;
  p->alpha_init = 1.f; p->alpha_min = 1.f; p->alpha_decay = 1.f; p->max_iter = 150; p->threshold = 1e-6f;
  p->mu = 0.8f; p->restitution = 0.f; p->rest_threshold = 0.01f; p->stall_window = 8; p->stall_ratio = 0.5f; p->joint_limits = 1;
  p->accel_m = 2; p->accel_start = 6; p->stall_reg = 0.02f;
  return RSB_OK;
}

// ---- model ---------------------------------------------------------------------------------------
// the limits of the step kernel, checked on every model that enters through the C-ABI
static int adopt_model(Model md, rsb_model** out) {
  if (md.nb > 32) return fail(RSB_ERR_UNSUPPORTED, "more than 32 movable bodies (one lane per body)");
  if (md.npts() > 32 * MAX_PT_SLOTS) return fail(RSB_ERR_UNSUPPORTED, "more than 64 candidate contact points");
  *out = new rsb_model{std::move(md)};
  return RSB_OK;
}
int rsb_model_create_from_urdf(const char* path_or_xml, rsb_model** out) {
  if (!path_or_xml || !out) return fail(RSB_ERR_INVALID, "null argument");
  try { return adopt_model(load_urdf(path_or_xml), out); } catch (const std::exception& e) { return fail(RSB_ERR_PARSE, e.what()); }
}
int rsb_model_save(const rsb_model* m, const char* path) {
  if (!m || !path) return fail(RSB_ERR_INVALID, "null argument");
  try { save_model(m->md, path); return RSB_OK; } catch (const std::exception& e) { return fail(RSB_ERR_PARSE, e.what()); }
}
int rsb_model_load(const char* path, rsb_model** out) {
  if (!path || !out) return fail(RSB_ERR_INVALID, "null argument");
  try { return adopt_model(load_model(path), out); } catch (const std::exception& e) { return fail(RSB_ERR_PARSE, e.what()); }
}
void rsb_model_destroy(rsb_model* m) { delete m; }
int rsb_model_dims(const rsb_model* m, int* nq, int* nv, int* nb, int* ncoll, int* npts) {
  if (!m) return fail(RSB_ERR_INVALID, "null model");
  if (nq) *nq = m->md.nq; if (nv) *nv = m->md.nv; if (nb) *nb = m->md.nb; if (ncoll) *ncoll = m->md.ncoll(); if (npts) *npts = m->md.npts();
  return RSB_OK;
}
int rsb_model_get_tables(const rsb_model* m, rsb_model_tables* t) {
  if (!m || !t) return fail(RSB_ERR_INVALID, "null argument");
  const Model& d = m->md;
  t->nb = d.nb; t->nq = d.nq; t->nv = d.nv; t->floating = d.floating; t->ncoll = d.ncoll(); t->npts = d.npts();
  t->parent = d.parent.data(); t->jtype = d.jtype.data(); t->qidx = d.qidx.data(); t->vidx = d.vidx.data(); t->depth = d.depth.data();
  t->jpos = d.jpos.data(); t->jrot = d.jrot.data(); t->axis = d.axis.data(); t->mass = d.mass.data(); t->com = d.com.data();
  t->inertia = d.inertia.data(); t->jlimit = d.jlimit.data();
  t->cbody = d.cbody.data(); t->ctype = d.ctype.data(); t->csize = d.csize.data(); t->cpos = d.cpos.data(); t->crot = d.crot.data();
  t->pt_body = d.pt_body.data(); t->pt_coll = d.pt_coll.data(); t->pt_feat = d.pt_feat.data(); t->pt_pos = d.pt_pos.data(); t->pt_rad = d.pt_rad.data();
  t->pt_type = d.pt_type.data(); t->pt_pos2 = d.pt_pos2.data(); t->jeffort = d.jeffort.data();
  return RSB_OK;
}
int rsb_model_body_index(const rsb_model* m, const char* name) {
  if (!m || !name) return fail(RSB_ERR_INVALID, "null argument");
  for (int i = 0; i < m->md.nb; i++) if (m->md.body_names[i] == name) return i;
  for (const Frame& f : m->md.frames) if (f.name == name) return f.body;   // a link merged through a fixed joint
  return fail(RSB_ERR_INVALID, std::string("no body named '") + name + "'");
}
// collision bodies are named after the link that carries them, upstream style "LINK/k" for the k-th one ("LINK" = "LINK/0")
int rsb_model_collision_index(const rsb_model* m, const char* name) {
  if (!m || !name) return fail(RSB_ERR_INVALID, "null argument");
  std::string link = name; int which = 0;
  const size_t slash = link.rfind('/');
  if (slash != std::string::npos) { which = std::atoi(link.c_str() + slash + 1); link.resize(slash); }
  int seen = 0;
  for (int c = 0; c < m->md.ncoll(); c++) if (m->md.coll_names[c] == link) { if (seen == which) return c; seen++; }
  return fail(RSB_ERR_INVALID, std::string("no collision body named '") + name + "'");
}
const char* rsb_model_body_name(const rsb_model* m, int body) { return (m && body >= 0 && body < m->md.nb) ? m->md.body_names[body].c_str() : nullptr; }
const char* rsb_model_joint_name(const rsb_model* m, int body) { return (m && body >= 0 && body < m->md.nb) ? m->md.joint_names[body].c_str() : nullptr; }
int rsb_model_frame_index(const rsb_model* m, const char* name) {
  if (!m || !name) return fail(RSB_ERR_INVALID, "null argument");
  for (size_t i = 0; i < m->md.frames.size(); i++) if (m->md.frames[i].name == name) return (int)i;
  for (size_t i = 0; i < m->md.frames.size(); i++) if (!m->md.frames[i].joint.empty() && m->md.frames[i].joint == name) return (int)i;   // joint-name alias
  return fail(RSB_ERR_INVALID, std::string("no frame named '") + name + "'");
}
int rsb_model_frame(const rsb_model* m, int frame, int* body, double pos[3], double rot[9]) {
  if (!m || frame < 0 || frame >= (int)m->md.frames.size()) return fail(RSB_ERR_INVALID, "bad frame index");
  const Frame& f = m->md.frames[frame];
  if (body) *body = f.body;
  if (pos) for (int k = 0; k < 3; k++) pos[k] = f.pos[k];
  if (rot) for (int k = 0; k < 9; k++) rot[k] = f.rot[k];
  return RSB_OK;
}

// ---- batch ---------------------------------------------------------------------------------------
int rsb_batch_create(const rsb_model* m, int num_envs, int device, rsb_batch** out) {
  if (!m || !out || num_envs <= 0) return fail(RSB_ERR_INVALID, "bad arguments to rsb_batch_create");
  int ndev = 0;
  cudaError_t e0 = cudaGetDeviceCount(&ndev);
  if (e0 != cudaSuccess || ndev == 0) return fail(RSB_ERR_CUDA, "no CUDA device: raisimlib_b200 has no CPU fallback");
  if (device < 0 || device >= ndev) return fail(RSB_ERR_INVALID, "device index out of range");
  CK(cudaSetDevice(device));
  rsb_batch* b = new rsb_batch;
  b->model = m; b->N = num_envs; b->device = device;
  const Model& md = m->md;
  b->nq = md.nq; b->nv = md.nv; b->nb = md.nb;
  b->gc_stride = round_up(std::max(1, md.nq), 8); b->gv_stride = round_up(std::max(1, md.nv), 8);   // 32-byte sector-aligned rows
  rsb_params_default(&b->prm);
  cudaError_t e = cudaStreamCreateWithFlags(&b->stream, cudaStreamNonBlocking);
  if (e != cudaSuccess) { delete b; return fail(RSB_ERR_CUDA, std::string("rsb_batch_create: ") + cudaGetErrorString(e)); }
  b->own_stream = true;
  Overrides ov;
  ov.kp.assign(std::max(1, md.nv), 0.f); ov.kd.assign(std::max(1, md.nv), 0.f);
  ov.pt_mu.assign(md.npts(), -1.f);
  const int rc = rebuild(b, std::move(ov));
  if (rc != RSB_OK) { rsb_batch_destroy(b); return rc; }
  const size_t N = (size_t)num_envs;
  auto zeroed = [&](auto& buf, size_t bytes) {
    bytes = std::max<size_t>(bytes, 16);
    if (e == cudaSuccess) e = buf.ensure(bytes, b->stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(buf.get(), 0, bytes, b->stream);
  };
  zeroed(b->gc, N * b->gc_stride * 4); zeroed(b->gv, N * b->gv_stride * 4); zeroed(b->tau, N * b->gv_stride * 4);
  zeroed(b->pt, N * b->gc_stride * 4); zeroed(b->vt, N * b->gv_stride * 4); zeroed(b->tau_applied, N * b->gv_stride * 4);
  zeroed(b->ncontacts, N * 4); zeroed(b->contact_pt, N * KMAX * 4); zeroed(b->iters, N * 4); zeroed(b->diverged, N * 4);
  zeroed(b->resid, N * 4); zeroed(b->solver_status, N * 4); zeroed(b->contacts, N * KMAX * sizeof(rsb_contact));
  if (e == cudaSuccess && md.floating) {   // identity quaternion so that a fresh batch is a valid state
    std::vector<float> q0(N * b->gc_stride, 0.f);
    for (size_t i = 0; i < N; i++) q0[i * b->gc_stride + 3] = 1.f;
    e = cudaMemcpyAsync(b->gc.get(), q0.data(), q0.size() * 4, cudaMemcpyHostToDevice, b->stream);
  }
  if (e == cudaSuccess) e = cudaStreamSynchronize(b->stream);
  if (e != cudaSuccess) { std::string msg = cudaGetErrorString(e); rsb_batch_destroy(b); return fail(RSB_ERR_CUDA, "rsb_batch_create: " + msg); }
  *out = b;
  return RSB_OK;
}

void rsb_batch_destroy(rsb_batch* b) {
  if (!b) return;
  cudaSetDevice(b->device);
  if (b->stream) cudaStreamSynchronize(b->stream);
  if (b->own_stream && b->stream) cudaStreamDestroy(b->stream);
  delete b;   // frees the batch's device buffers
}

int rsb_batch_set_stream(rsb_batch* b, void* s) {
  if (!b) return fail(RSB_ERR_INVALID, "null batch");
  CK(cudaStreamSynchronize(b->stream));
  if (b->own_stream) { cudaStreamDestroy(b->stream); b->own_stream = false; }
  b->stream = (cudaStream_t)s;
  return RSB_OK;
}
int rsb_batch_sync(rsb_batch* b) {
  if (!b) return fail(RSB_ERR_INVALID, "null batch");
  CK(cudaStreamSynchronize(b->stream));
  return RSB_OK;
}
int rsb_batch_num_envs(const rsb_batch* b) { return b ? b->N : 0; }

int rsb_batch_set_ground(rsb_batch* b, float z) {
  if (!b) return fail(RSB_ERR_INVALID, "null batch");
  b->ter = TerrainDesc{}; b->ter.type = 1; b->ter.ground_z = z;
  return RSB_OK;
}
int rsb_batch_clear_terrain(rsb_batch* b) {
  if (!b) return fail(RSB_ERR_INVALID, "null batch");
  b->ter = TerrainDesc{};
  return RSB_OK;
}
// `count` same-sized height maps back to back; map_of_env: the map index of every environment (null: one map that all share)
static int upload_heightmaps(rsb_batch* b, int count, int xs, int ys, float x_size, float y_size, float cx, float cy, const float* h,
                             const int32_t* map_of_env) {
  CK(cudaSetDevice(b->device));
  CK(cudaStreamSynchronize(b->stream));   // no launch still reads the maps overwritten below
  b->ter = TerrainDesc{};               // nothing may point at half-written maps if a step below fails
  const size_t words = (size_t)count * xs * ys;
  CK(b->hmap.ensure(words * 4, b->stream));
  CK(cudaMemcpy(b->hmap.get(), h, words * 4, cudaMemcpyHostToDevice));
  if (map_of_env) {
    CK(b->hmap_index.ensure((size_t)b->N * 4, b->stream));
    CK(cudaMemcpy(b->hmap_index.get(), map_of_env, (size_t)b->N * 4, cudaMemcpyHostToDevice));
  }
  TerrainDesc t{};
  t.type = 2; t.xs = xs; t.ys = ys;
  t.dx = x_size / (float)(xs - 1); t.dy = y_size / (float)(ys - 1); t.inv_dx = 1.0f / t.dx; t.inv_dy = 1.0f / t.dy;
  t.x0 = cx - 0.5f * x_size; t.y0 = cy - 0.5f * y_size;
  t.xmax = (float)(xs - 1); t.ymax = (float)(ys - 1);
  t.h = b->hmap.get(); t.env_map = map_of_env ? b->hmap_index.get() : nullptr; t.map_words = xs * ys;
  b->hmap_max.assign(count, 0.f);
  for (int m = 0; m < count; m++) {
    const float* hm = h + (size_t)m * t.map_words;
    float mx = hm[0];
    for (int i = 1; i < t.map_words; i++) mx = std::max(mx, hm[i]);
    b->hmap_max[m] = mx;
  }
  t.hmax = *std::max_element(b->hmap_max.begin(), b->hmap_max.end());
  b->ter = t;
  return RSB_OK;
}
int rsb_batch_set_heightmap(rsb_batch* b, int xs, int ys, float x_size, float y_size, float cx, float cy, const float* h) {
  if (!b || !h || xs < 2 || ys < 2 || !(x_size > 0) || !(y_size > 0)) return fail(RSB_ERR_INVALID, "bad height map");
  return upload_heightmaps(b, 1, xs, ys, x_size, y_size, cx, cy, h, nullptr);
}
// terrain atlas (SURVEY 8f N3 "per-env distinct terrains"): `count` same-sized height maps back to back and one map
// index per environment; every environment collides with its own map, everything else is as rsb_batch_set_heightmap
int rsb_batch_set_heightmaps(rsb_batch* b, int count, int xs, int ys, float x_size, float y_size, float cx, float cy, const float* h,
                             const int32_t* map_of_env) {
  if (!b || !h || !map_of_env || count < 1 || xs < 2 || ys < 2 || !(x_size > 0) || !(y_size > 0)) return fail(RSB_ERR_INVALID, "bad height-map atlas");
  if ((size_t)count * xs * ys > ((size_t)1 << 30)) return fail(RSB_ERR_INVALID, "height-map atlas too large");
  for (int e = 0; e < b->N; e++) if (map_of_env[e] < 0 || map_of_env[e] >= count) return fail(RSB_ERR_INVALID, "height-map index out of range");
  return upload_heightmaps(b, count, xs, ys, x_size, y_size, cx, cy, h, map_of_env);
}
// terrain curriculum: environments [env_begin, env_begin + env_count) move to other maps of the atlas.  The indices are checked in the
// staging buffer, then copied into the index in stream order: launches enqueued before see the old assignment, later ones the new
int rsb_batch_set_heightmap_index(rsb_batch* b, const int32_t* map_of_env, int env_begin, int env_count, int where) {
  int rc = check_range(b, env_begin, env_count, where); if (rc) return rc;
  if (!map_of_env) return fail(RSB_ERR_INVALID, "height-map index: null index list");
  if (b->ter.type != 2 || !b->ter.env_map) return fail(RSB_ERR_INVALID, "height-map index: no terrain atlas (set one with rsb_batch_set_heightmaps() first)");
  if (env_count == 0) return RSB_OK;
  CK(cudaSetDevice(b->device));
  const int count = (int)b->hmap_max.size();
  int* staged = nullptr;
  auto check = [&](int* out, const int* src, int* bad) {
    const int threads = 256;
    rsb_int_rows_check_kernel<<<(unsigned)((env_count + threads - 1) / threads), threads, 0, b->stream>>>(out, src, env_count, 0, count - 1, bad);
  };
  auto what = [&](int bad) {
    return "height-map index: environment " + std::to_string(env_begin + bad) + " names a map outside [0, " + std::to_string(count) + "); nothing changed";
  };
  rc = stage_checked(b, map_of_env, (size_t)env_count, (size_t)env_count, where, true, 0, check, what, &staged); if (rc) return rc;
  CK(cudaMemcpyAsync(b->hmap_index.get() + env_begin, staged, (size_t)env_count * 4, cudaMemcpyDeviceToDevice, b->stream));
  return RSB_OK;
}
// maps first .. first + count - 1 of the terrain overwritten in place.  The heights are checked, and the largest height of every new map
// found, in the staging buffer before any map changes; the map pointer stays where it is, and the copy follows earlier launches in
// stream order
int rsb_batch_update_heightmaps(rsb_batch* b, int first, int count, const float* heights, int where) {
  if (!b) return fail(RSB_ERR_INVALID, "null batch");
  if (bad_where(where)) return fail(RSB_ERR_INVALID, "`where` must be RSB_HOST or RSB_DEVICE");
  if (!heights) return fail(RSB_ERR_INVALID, "update height maps: null heights");
  if (b->ter.type != 2) return fail(RSB_ERR_INVALID, "update height maps: no height map (set one with rsb_batch_set_heightmap() or rsb_batch_set_heightmaps() first)");
  const int maps = (int)b->hmap_max.size();
  if (first < 0 || count < 0 || first > maps - count)
    return fail(RSB_ERR_INVALID, "update height maps: maps [" + std::to_string(first) + ", " + std::to_string(first) + " + " + std::to_string(count) + ") are not all in the terrain's " + std::to_string(maps));
  if (count == 0) return RSB_OK;
  CK(cudaSetDevice(b->device));
  const int words = b->ter.map_words;
  float* staged = nullptr;
  std::vector<int> verdict;
  auto check = [&](float* out, const float* src, int* v) {
    const int threads = 256, blocks = std::min((words + threads - 1) / threads, 256);
    rsb_heightmap_check_kernel<<<dim3((unsigned)blocks, (unsigned)std::min(count, 65535)), threads, 0, b->stream>>>(out, src, words, count, v, v + 1);
  };
  auto what = [&](int bad) {
    const int m = bad / words, i = bad % words;
    return "update height maps: map " + std::to_string(first + m) + ", sample (" + std::to_string(i % b->ter.xs) + ", " + std::to_string(i / b->ter.xs) + ") is not finite; nothing changed";
  };
  const size_t all = (size_t)count * words;
  int rc = stage_checked(b, heights, all, all, where, true, count, check, what, &staged, &verdict); if (rc) return rc;
  CK(cudaMemcpyAsync(b->hmap.get() + (size_t)first * words, staged, all * 4, cudaMemcpyDeviceToDevice, b->stream));
  for (int m = 0; m < count; m++) {   // every value is finite, so each map has a largest one: back from its ordered-integer image
    const int k = verdict[1 + m], bits = k >= 0 ? k : k ^ 0x7fffffff;
    float mx;
    std::memcpy(&mx, &bits, 4);
    b->hmap_max[first + m] = mx;
  }
  b->ter.hmax = *std::max_element(b->hmap_max.begin(), b->hmap_max.end());
  return RSB_OK;
}
int rsb_batch_set_params(rsb_batch* b, const rsb_params* p) {
  if (!p) return fail(RSB_ERR_INVALID, "null argument");
  // every float field finite, checked before the batch: a non-finite dt, gravity or relaxation factor turns every state into NaN on
  // the next launch, a NaN threshold turns the convergence test off
  const struct { const char* name; float v; } fields[] = {
      {"dt", p->dt}, {"gravity[0]", p->gravity[0]}, {"gravity[1]", p->gravity[1]}, {"gravity[2]", p->gravity[2]}, {"erp", p->erp},
      {"alpha_init", p->alpha_init}, {"alpha_min", p->alpha_min}, {"alpha_decay", p->alpha_decay}, {"threshold", p->threshold},
      {"mu", p->mu}, {"restitution", p->restitution}, {"rest_threshold", p->rest_threshold}, {"stall_ratio", p->stall_ratio},
      {"stall_reg", p->stall_reg}};
  for (const auto& f : fields)
    if (!std::isfinite(f.v)) return fail(RSB_ERR_INVALID, std::string("params: ") + f.name + " is not finite");
  if (!b) return fail(RSB_ERR_INVALID, "null argument");
  if (!(p->dt > 0) || p->max_iter < 1 || !(p->mu >= 0)) return fail(RSB_ERR_INVALID, "invalid params");
  if (p->accel_m != 0 && p->accel_m != 2) return fail(RSB_ERR_INVALID, "accel_m must be 0 (plain sweeps) or 2");
  if (p->accel_m == 2 && p->accel_start < 3) return fail(RSB_ERR_INVALID, "accel_start must be at least 3");
  if (!(p->stall_reg >= 0.f)) return fail(RSB_ERR_INVALID, "stall_reg must be >= 0");
  b->prm = *p;
  return RSB_OK;
}
int rsb_batch_get_params(const rsb_batch* b, rsb_params* p) {
  if (!b || !p) return fail(RSB_ERR_INVALID, "null argument");
  *p = b->prm;
  return RSB_OK;
}

int rsb_batch_set_state(rsb_batch* b, const float* gc, const float* gv, int env_begin, int env_count, int where) {
  int rc = check_range(b, env_begin, env_count, where); if (rc) return rc;
  b->kin_dirty = true;
  rc = copy_rows_in(b, b->gc.get(), b->gc_stride, gc, b->nq, env_begin, env_count, where); if (rc) return rc;
  return copy_rows_in(b, b->gv.get(), b->gv_stride, gv, b->nv, env_begin, env_count, where);
}
int rsb_batch_get_state(rsb_batch* b, float* gc, float* gv, int env_begin, int env_count, int where) {
  int rc = check_range(b, env_begin, env_count, where); if (rc) return rc;
  rc = copy_rows_out(b, gc, b->gc.get(), b->gc_stride, b->nq, env_begin, env_count, where); if (rc) return rc;
  rc = copy_rows_out(b, gv, b->gv.get(), b->gv_stride, b->nv, env_begin, env_count, where); if (rc) return rc;
  if (where == RSB_HOST) CK(cudaStreamSynchronize(b->stream));
  return RSB_OK;
}
int rsb_batch_set_pd_gains(rsb_batch* b, const float* kp, const float* kd) {
  if (!b || !kp || !kd) return fail(RSB_ERR_INVALID, "null argument");
  const Model& md = b->model->md;
  Overrides ov = b->ovr;
  for (int i = 0; i < md.nv; i++) { ov.kp[i] = kp[i]; ov.kd[i] = kd[i]; }
  if (md.floating) for (int i = 0; i < 6; i++) { ov.kp[i] = 0.f; ov.kd[i] = 0.f; }   // the base is not actuated
  const int rc = rebuild(b, std::move(ov)); if (rc) return rc;
  b->pd_set = true;
  return RSB_OK;
}
// friction coefficient of one collision body against the terrain (mu < 0 restores the default material):
// the per-body half of World::setMaterialPairProp / CollisionDefinition::setMaterial
int rsb_batch_set_collision_friction(rsb_batch* b, int collision_body, float mu) {
  if (!b) return fail(RSB_ERR_INVALID, "null batch");
  const Model& md = b->model->md;
  if (collision_body < 0 || collision_body >= md.ncoll()) return fail(RSB_ERR_INVALID, "collision body index out of range");
  Overrides ov = b->ovr;
  for (int k = 0; k < md.npts(); k++) if (md.pt_coll[k] == collision_body) ov.pt_mu[k] = mu;
  return rebuild(b, std::move(ov));
}
// self-collision between explicit pairs of collision bodies (n = 0: none, the default).  Everything is checked before anything changes:
// a refused call leaves the batch as it was.  The pair table goes to the end of the model blob; a batch with pairs runs the generic
// instance of the step kernel (pick_config) with room for the pairs in stage B's hit list and a second column block for stage C.
int rsb_batch_set_self_collision(rsb_batch* b, const int32_t* pairs, int n, const float* mu) {
  if (!b) return fail(RSB_ERR_INVALID, "null batch");
  if (n < 0 || n > MAX_SELF_PAIRS) return fail(RSB_ERR_INVALID, "at most " + std::to_string(MAX_SELF_PAIRS) + " self-collision pairs per batch (got " + std::to_string(n) + ")");
  if (n > 0 && !pairs) return fail(RSB_ERR_INVALID, "null pair list");
  const Model& md = b->model->md;
  static const char* shape[] = {"sphere", "box", "capsule", "cylinder"};
  for (int j = 0; j < n; j++) {
    const int c1 = pairs[2 * j], c2 = pairs[2 * j + 1];
    if (c1 < 0 || c1 >= md.ncoll() || c2 < 0 || c2 >= md.ncoll())
      return fail(RSB_ERR_INVALID, "self-collision pair " + std::to_string(j) + ": collision body index out of range (the model has " + std::to_string(md.ncoll()) + ")");
    if (md.cbody[c1] == md.cbody[c2])
      return fail(RSB_ERR_INVALID, "self-collision pair " + std::to_string(j) + ": collision bodies " + md.coll_names[c1] + " and " + md.coll_names[c2] + " are on the same body");
    const int t1 = md.ctype[c1], t2 = md.ctype[c2];
    const bool round1 = t1 == CT_SPHERE || t1 == CT_CAPSULE, round2 = t2 == CT_SPHERE || t2 == CT_CAPSULE;
    const bool ok = (round1 && round2) || (t1 == CT_SPHERE && t2 == CT_BOX) || (t1 == CT_BOX && t2 == CT_SPHERE);
    if (!ok)
      return fail(RSB_ERR_UNSUPPORTED, "self-collision pair " + std::to_string(j) + " (" + md.coll_names[c1] + ", " + md.coll_names[c2] + "): " + shape[t1] + "-" + shape[t2] +
                                           " is not supported (sphere-sphere, sphere-capsule, capsule-capsule and sphere-box are)");
    if (mu && !(mu[j] < 0.f || mu[j] >= 0.f)) return fail(RSB_ERR_INVALID, "self-collision pair " + std::to_string(j) + ": friction is not a number");
  }
  Overrides ov = b->ovr;
  ov.self_pairs.assign(pairs ? pairs : nullptr, pairs ? pairs + 2 * n : nullptr);
  ov.self_mu.assign(n, -1.f);
  for (int j = 0; j < n && mu; j++) ov.self_mu[j] = mu[j];
  return rebuild(b, std::move(ov));
}

int rsb_batch_set_pd_target(rsb_batch* b, const float* ptarget, const float* vtarget, int env_begin, int env_count, int where) {
  int rc = check_range(b, env_begin, env_count, where); if (rc) return rc;
  if (ptarget) b->pt_bound = nullptr;     // copying targets in ends a zero-copy binding
  rc = copy_rows_in(b, b->pt.get(), b->gc_stride, ptarget, b->nq, env_begin, env_count, where); if (rc) return rc;
  return copy_rows_in(b, b->vt.get(), b->gv_stride, vtarget, b->nv, env_begin, env_count, where);
}
int rsb_batch_bind_pd_target(rsb_batch* b, const float* ptarget_device, int row_stride) {
  if (!b) return fail(RSB_ERR_INVALID, "null batch");
  if (ptarget_device && row_stride < b->nq) return fail(RSB_ERR_INVALID, "row stride smaller than nq");
  b->pt_bound = ptarget_device; b->pt_bound_stride = row_stride;
  return RSB_OK;
}
int rsb_batch_set_generalized_force(rsb_batch* b, const float* tau, int env_begin, int env_count, int where) {
  int rc = check_range(b, env_begin, env_count, where); if (rc) return rc;
  return copy_rows_in(b, b->tau.get(), b->gv_stride, tau, b->nv, env_begin, env_count, where);
}
int rsb_batch_get_generalized_force(rsb_batch* b, float* tau, int env_begin, int env_count, int where) {
  int rc = check_range(b, env_begin, env_count, where); if (rc) return rc;
  rc = copy_rows_out(b, tau, b->tau_applied.get(), b->gv_stride, b->nv, env_begin, env_count, where); if (rc) return rc;
  if (where == RSB_HOST) CK(cudaStreamSynchronize(b->stream));
  return RSB_OK;
}
// ArticulatedSystem::setExternalForce / setExternalTorque for a range of environments: one wrench per environment,
// acting on `body` at `point_body` (body frame; null = body origin), world-frame force / torque rows (null = zero).
// It acts during the next integrate() / control-step call (all of its fused sub-steps) and is cleared afterwards.
int rsb_batch_set_external_wrench(rsb_batch* b, int body, const float* force, const float* torque, const float* point_body, int env_begin, int env_count, int where) {
  int rc = check_range(b, env_begin, env_count, where); if (rc) return rc;
  if (body < 0 || body >= b->nb) return fail(RSB_ERR_INVALID, "external wrench: body index out of range");
  if (env_count == 0) return RSB_OK;
  CK(cudaSetDevice(b->device));
  CK(b->ext.ensure((size_t)b->N * EXT_WORDS * 4, b->stream));
  if (!b->ext_active) {   // rows of an earlier call are stale: body = -1 everywhere
    CK(cudaMemsetAsync(b->ext.get(), 0xff, (size_t)b->N * EXT_WORDS * 4, b->stream));
    b->ext_active = true;
  }
  const float *df = force, *dtq = torque;
  if (where == RSB_HOST && (force || torque)) {
    float* st = staging(b, (size_t)env_count * 6); if (!st) return RSB_ERR_CUDA;   // force rows, then torque rows
    if (force) { CK(cudaMemcpyAsync(st, force, (size_t)env_count * 12, cudaMemcpyHostToDevice, b->stream)); df = st; }
    if (torque) { CK(cudaMemcpyAsync(st + (size_t)env_count * 3, torque, (size_t)env_count * 12, cudaMemcpyHostToDevice, b->stream)); dtq = st + (size_t)env_count * 3; }
  }
  const float px = point_body ? point_body[0] : 0.f, py = point_body ? point_body[1] : 0.f, pz = point_body ? point_body[2] : 0.f;
  const int threads = 128, blocks = (env_count + threads - 1) / threads;
  rsb_ext_pack_kernel<<<blocks, threads, 0, b->stream>>>(b->ext.get() + (size_t)env_begin * EXT_WORDS, body, df, dtq, px, py, pz, env_count);
  CK(cudaGetLastError());
  return RSB_OK;
}
// ---- per-environment inertial parameters (ArticulatedSystem::getMass / getBodyCOM_B / getInertia + updateMassInfo per World upstream) ----
// the model's row of every body, in float32 exactly as build_blob writes BF_MASS / BF_COM / BF_INERTIA
static std::vector<float> model_inertia_row(const Model& md) {
  std::vector<float> r((size_t)md.nb * BI_WORDS, 0.f);
  for (int i = 0; i < md.nb; i++) {
    float* o = &r[(size_t)i * BI_WORDS];
    o[0] = (float)md.mass[i];
    for (int k = 0; k < 3; k++) o[1 + k] = (float)md.com[3 * i + k];
    for (int k = 0; k < 6; k++) o[4 + k] = (float)md.inertia[6 * i + k];
  }
  return r;
}
int rsb_batch_set_body_inertia(rsb_batch* b, const float* rows, int env_begin, int env_count, int where) {
  if (!b) return fail(RSB_ERR_INVALID, "null batch");
  const Model& md = b->model->md;
  auto check = [&](float* out, const float* src, int n, int* bad) {
    const int nrows = n * md.nb, threads = 128;
    rsb_body_inertia_pack_kernel<<<(unsigned)((nrows + threads - 1) / threads), threads, 0, b->stream>>>(out, src, nrows, 1e-6, bad);
  };
  auto what = [&](int bad) {
    static const char* fault[] = {"", "a value that is not finite", "a negative mass", "an inertia that is not symmetric positive semidefinite"};
    const int r = bad / 4, env = env_begin + r / md.nb, body = r % md.nb;
    return "body inertia: environment " + std::to_string(env) + ", body " + std::to_string(body) + " (" + md.body_names[body] + ") has " + fault[bad & 3];
  };
  const int rc = commit_env_rows(b, b->body_inertia, model_inertia_row(md), rows, env_begin, env_count, where, (size_t)md.nb * 10, check, what);
  if (rc == RSB_OK && env_count > 0) b->kin_dirty = true;   // M, h and the poses of the getters describe the new parameters from the next getter on
  return rc;
}
int rsb_batch_clear_body_inertia(rsb_batch* b) {
  if (!b) return fail(RSB_ERR_INVALID, "null batch");
  if (b->body_inertia.active) b->kin_dirty = true;
  b->body_inertia.active = false;
  return RSB_OK;
}
// ---- per-environment terrain friction (World::setMaterialPairProp / setDefaultMaterial / CollisionBody::setMaterial per World
// upstream): -1 is the batch-level value, resolved by the step kernel at every launch; the friction enters no getter, so nothing goes stale
int rsb_batch_set_contact_friction(rsb_batch* b, const float* rows, int env_begin, int env_count, int where) {
  if (!b) return fail(RSB_ERR_INVALID, "null batch");
  const Model& md = b->model->md;
  const int ncoll = md.ncoll();
  auto check = [&](float* out, const float* src, int n, int* bad) {
    const int words = n * ncoll, threads = 128;
    rsb_finite_rows_check_kernel<<<(unsigned)((words + threads - 1) / threads), threads, 0, b->stream>>>(out, src, words, bad);
  };
  auto what = [&](int bad) {
    const int env = env_begin + bad / ncoll, c = bad % ncoll;
    return "contact friction: environment " + std::to_string(env) + ", collision body " + std::to_string(c) + " (" + md.coll_names[c] + ") is not finite";
  };
  return commit_env_rows(b, b->contact_friction, std::vector<float>((size_t)ncoll, -1.f), rows, env_begin, env_count, where, (size_t)ncoll, check, what);
}
int rsb_batch_clear_contact_friction(rsb_batch* b) {
  if (!b) return fail(RSB_ERR_INVALID, "null batch");
  b->contact_friction.active = false;
  return RSB_OK;
}
// ---- per-environment PD gains and actuator effort limits (ArticulatedSystem::setPdGains / setActuationLimits per World upstream):
// -1 is the batch-level value (rsb_batch_set_pd_gains, the URDF effort limit), resolved by the step kernel at every launch; the gains
// enter no getter, so nothing goes stale
int rsb_batch_set_actuator_params(rsb_batch* b, const float* rows, int env_begin, int env_count, int where) {
  if (!b) return fail(RSB_ERR_INVALID, "null batch");
  const Model& md = b->model->md;
  const int nv = md.nv;
  auto check = [&](float* out, const float* src, int n, int* bad) {
    const int threads = 128;
    rsb_actuator_params_check_kernel<<<(unsigned)((n * nv + threads - 1) / threads), threads, 0, b->stream>>>(out, src, n, nv, md.floating ? 6 : 0, bad);
  };
  auto what = [&](int bad) {
    static const char* field[] = {"kp", "kd", "effort limit"};
    static const char* fault[] = {"is NaN or infinite", "is NaN or infinite", "is NaN or -inf"};
    const int r = bad / 3, env = env_begin + r / nv, dof = r % nv;
    return "actuator params: environment " + std::to_string(env) + ", dof " + std::to_string(dof) + ": " + field[bad % 3] + " " + fault[bad % 3];
  };
  return commit_env_rows(b, b->actuator, std::vector<float>((size_t)3 * nv, -1.f), rows, env_begin, env_count, where, (size_t)3 * nv, check, what);
}
int rsb_batch_clear_actuator_params(rsb_batch* b) {
  if (!b) return fail(RSB_ERR_INVALID, "null batch");
  b->actuator.active = false;
  return RSB_OK;
}
// the dof list of an actuator network call: n_dofs in [1, nv], joint dofs only, none twice (who: the message prefix)
static int check_an_dofs(const rsb_batch* b, const int32_t* dofs, int n_dofs, const char* who) {
  const int nv = b->nv, nbase = b->model->md.floating ? 6 : 0;
  if (!dofs) return fail(RSB_ERR_INVALID, std::string(who) + ": null dof list");
  std::vector<char> seen(nv, 0);
  for (int s = 0; s < n_dofs; s++) {
    const int d = dofs[s];
    if (d < nbase || d >= nv) return fail(RSB_ERR_INVALID, std::string(who) + ": dof " + std::to_string(d) + " outside the actuated dofs [" + std::to_string(nbase) + ", " + std::to_string(nv) + ")");
    if (seen[d]) return fail(RSB_ERR_INVALID, std::string(who) + ": dof " + std::to_string(d) + " listed twice");
    seen[d] = 1;
  }
  return RSB_OK;
}
// ---- learned actuator network (one per batch, shared by the listed dofs): checked and repacked on the host, the history on the device
int rsb_batch_set_actuator_network(rsb_batch* b, const int32_t* dofs, int n_dofs, int history, int layers, int width, const float* params) {
  if (!b) return fail(RSB_ERR_INVALID, "null batch");
  const int nv = b->nv;
  if (n_dofs < 0 || n_dofs > nv) return fail(RSB_ERR_INVALID, "actuator network: n_dofs " + std::to_string(n_dofs) + " outside [0, " + std::to_string(nv) + "]");
  if (n_dofs == 0) { b->an_dofs.clear(); return RSB_OK; }
  int rc = check_an_dofs(b, dofs, n_dofs, "actuator network"); if (rc) return rc;
  if (history < 1 || history > RSB_ACTNET_MAX_HISTORY || layers < 1 || layers > RSB_ACTNET_MAX_LAYERS || width < 1 || width > RSB_ACTNET_MAX_WIDTH)
    return fail(RSB_ERR_INVALID, "actuator network: history, layers and width must lie in [1, " + std::to_string(RSB_ACTNET_MAX_HISTORY) + "], [1, " +
                                 std::to_string(RSB_ACTNET_MAX_LAYERS) + "] and [1, " + std::to_string(RSB_ACTNET_MAX_WIDTH) + "]");
  if (!params) return fail(RSB_ERR_INVALID, "actuator network: null parameters");
  const int F = 2 * history, W = width;
  const size_t count = (size_t)W * F + W + (size_t)(layers - 1) * (W * W + W) + W + 1;
  for (size_t k = 0; k < count; k++)
    if (!std::isfinite(params[k])) return fail(RSB_ERR_INVALID, "actuator network: parameter " + std::to_string(k) + " is not finite; nothing changed");
  // torch.nn.Linear order -> ActNetDesc::params: every hidden layer's weights transposed to [n_in][W], then its bias
  std::vector<float> pk(count);
  size_t so = 0;
  for (int l = 0; l < layers; l++) {
    const int nin = l == 0 ? F : W;
    for (int j = 0; j < W; j++) for (int k = 0; k < nin; k++) pk[so + (size_t)k * W + j] = params[so + (size_t)j * nin + k];
    so += (size_t)W * nin;
    for (int j = 0; j < W; j++) pk[so + j] = params[so + j];
    so += W;
  }
  for (size_t k = so; k < count; k++) pk[k] = params[k];   // output weights [W] and bias
  CK(cudaSetDevice(b->device));
  const size_t hist_words = (size_t)b->N * n_dofs * 2 * (history - 1);
  CK(b->an_params.ensure(count * 4, b->stream));
  CK(b->an_hist.ensure(std::max<size_t>(hist_words, 1) * 4, b->stream));
  CK(cudaMemcpyAsync(b->an_params.get(), pk.data(), count * 4, cudaMemcpyHostToDevice, b->stream));
  if (hist_words > 0) CK(cudaMemsetAsync(b->an_hist.get(), 0, hist_words * 4, b->stream));
  CK(cudaStreamSynchronize(b->stream));   // the pageable source goes out of scope here
  b->an_dofs.assign(dofs, dofs + n_dofs);
  b->an_lstm = false;
  b->an_H = history; b->an_L = layers; b->an_W = width;
  return RSB_OK;
}
int rsb_batch_set_actuator_lstm(rsb_batch* b, const int32_t* dofs, int n_dofs, int layers, int hidden, const float* params) {
  if (!b) return fail(RSB_ERR_INVALID, "null batch");
  const int nv = b->nv;
  if (n_dofs < 0 || n_dofs > nv) return fail(RSB_ERR_INVALID, "actuator lstm: n_dofs " + std::to_string(n_dofs) + " outside [0, " + std::to_string(nv) + "]");
  if (n_dofs == 0) { b->an_dofs.clear(); return RSB_OK; }
  int rc = check_an_dofs(b, dofs, n_dofs, "actuator lstm"); if (rc) return rc;
  if (layers < 1 || layers > RSB_ACTNET_MAX_LAYERS || hidden < 1 || hidden > RSB_ACTNET_MAX_WIDTH)
    return fail(RSB_ERR_INVALID, "actuator lstm: layers and hidden must lie in [1, " + std::to_string(RSB_ACTNET_MAX_LAYERS) + "] and [1, " +
                                 std::to_string(RSB_ACTNET_MAX_WIDTH) + "]");
  if (!params) return fail(RSB_ERR_INVALID, "actuator lstm: null parameters");
  const int W = hidden, W4 = 4 * hidden;
  size_t count = (size_t)W + 1, packed = (size_t)W + 1;
  for (int l = 0; l < layers; l++) {
    const int nin = l == 0 ? 2 : W;
    count += (size_t)W4 * (nin + W + 2);
    packed += (size_t)W4 * (nin + W + 1);
  }
  for (size_t k = 0; k < count; k++)
    if (!std::isfinite(params[k])) return fail(RSB_ERR_INVALID, "actuator lstm: parameter " + std::to_string(k) + " is not finite; nothing changed");
  // torch.nn.LSTM order (weight_ih [4W][n_in], weight_hh [4W][W], bias_ih [4W], bias_hh [4W] per layer; read-out [1][W], [1]) ->
  // ActNetDesc::params: per layer [n_in + W][4][W] (row g W + j of torch is gate g of unit j), then bias_ih + bias_hh [4][W]
  std::vector<float> pk(packed);
  size_t so = 0, po = 0;
  for (int l = 0; l < layers; l++) {
    const int nin = l == 0 ? 2 : W;
    const float *wih = params + so, *whh = wih + (size_t)W4 * nin, *bih = whh + (size_t)W4 * W, *bhh = bih + W4;
    for (int r = 0; r < W4; r++) {
      for (int k = 0; k < nin; k++) pk[po + (size_t)k * W4 + r] = wih[(size_t)r * nin + k];
      for (int k = 0; k < W; k++) pk[po + (size_t)(nin + k) * W4 + r] = whh[(size_t)r * W + k];
      pk[po + (size_t)(nin + W) * W4 + r] = bih[r] + bhh[r];
    }
    so += (size_t)W4 * (nin + W + 2);
    po += (size_t)W4 * (nin + W + 1);
  }
  for (int k = 0; k <= W; k++) pk[po + k] = params[so + k];   // read-out weights [W] and bias
  CK(cudaSetDevice(b->device));
  const size_t hist_words = (size_t)b->N * n_dofs * layers * 2 * W;
  CK(b->an_params.ensure(packed * 4, b->stream));
  CK(b->an_hist.ensure(hist_words * 4, b->stream));
  CK(cudaMemcpyAsync(b->an_params.get(), pk.data(), packed * 4, cudaMemcpyHostToDevice, b->stream));
  CK(cudaMemsetAsync(b->an_hist.get(), 0, hist_words * 4, b->stream));
  CK(cudaStreamSynchronize(b->stream));   // the pageable source goes out of scope here
  b->an_dofs.assign(dofs, dofs + n_dofs);
  b->an_lstm = true;
  b->an_H = 0; b->an_L = layers; b->an_W = W;
  return RSB_OK;
}
int rsb_batch_set_actuator_history(rsb_batch* b, const float* rows, int env_begin, int env_count, int where) {
  int rc = check_range(b, env_begin, env_count, where); if (rc) return rc;
  if (b->an_dofs.empty()) return fail(RSB_ERR_INVALID, "actuator history: no actuator network (rsb_batch_set_actuator_network)");
  const size_t w = an_hist_words(b), words = w * env_count;
  if (words == 0) return RSB_OK;
  CK(cudaSetDevice(b->device));
  float* const at = b->an_hist.get() + (size_t)env_begin * w;
  if (!rows) { CK(cudaMemsetAsync(at, 0, words * 4, b->stream)); return RSB_OK; }
  float* staged = nullptr;
  auto check = [&](float* out, const float* src, int* bad) {
    const int threads = 256;
    rsb_finite_rows_check_kernel<<<(unsigned)((words + threads - 1) / threads), threads, 0, b->stream>>>(out, src, (int)words, bad);
  };
  auto what = [&](int bad) {
    return "actuator history: environment " + std::to_string(env_begin + bad / (int)w) + ", word " + std::to_string(bad % (int)w) + " is not finite; nothing changed";
  };
  rc = stage_checked(b, rows, words, words, where, false, 0, check, what, &staged); if (rc) return rc;
  CK(cudaMemcpyAsync(at, staged, words * 4, cudaMemcpyDeviceToDevice, b->stream));
  return RSB_OK;
}
int rsb_batch_get_actuator_history(rsb_batch* b, float* rows, int env_begin, int env_count, int where) {
  int rc = check_range(b, env_begin, env_count, where); if (rc) return rc;
  if (b->an_dofs.empty()) return fail(RSB_ERR_INVALID, "actuator history: no actuator network (rsb_batch_set_actuator_network)");
  const size_t w = an_hist_words(b), words = w * env_count;
  if (words == 0) return RSB_OK;
  if (!rows) return fail(RSB_ERR_INVALID, "actuator history: null rows");
  CK(cudaSetDevice(b->device));
  return copy_out(b, rows, b->an_hist.get() + (size_t)env_begin * w, words * 4, where);
}
// ---- actuation delay: the entries checked in the staging buffer, then committed by a kernel in stream order
int rsb_batch_set_actuation_delay(rsb_batch* b, const int32_t* delays, int env_begin, int env_count, int where) {
  int rc = check_range(b, env_begin, env_count, where); if (rc) return rc;
  if (env_count == 0) return RSB_OK;
  CK(cudaSetDevice(b->device));
  const int threads = 256, blocks = (env_count + threads - 1) / threads;
  int* staged = nullptr;
  if (delays) {
    auto check = [&](int* out, const int* src, int* bad) {
      rsb_int_rows_check_kernel<<<(unsigned)blocks, threads, 0, b->stream>>>(out, src, env_count, -1, RSB_MAX_ACTUATION_DELAY, bad);
    };
    auto what = [&](int bad) {
      return "actuation delay: environment " + std::to_string(env_begin + bad) + ": an entry must be -1 (unchanged) or a delay in [0, " +
             std::to_string(RSB_MAX_ACTUATION_DELAY) + "] sub-steps; nothing changed";
    };
    rc = stage_checked(b, delays, (size_t)env_count, (size_t)env_count, where, true, 0, check, what, &staged); if (rc) return rc;
  }
  const int nj = b->nv - (b->model->md.floating ? 6 : 0);
  CK(b->delay_state.ensure((size_t)b->N * 2 * 4, b->stream));
  CK(b->delay_ring.ensure(std::max<size_t>((size_t)b->N * DELAY_SLOTS * 3 * nj, 1) * 4, b->stream));
  if (!b->delay_active) CK(cudaMemsetAsync(b->delay_state.get(), 0, (size_t)b->N * 2 * 4, b->stream));   // delay 0, history empty
  rsb_actuation_delay_commit_kernel<<<(unsigned)blocks, threads, 0, b->stream>>>(b->delay_state.get() + 2 * (size_t)env_begin, staged, env_count);
  CK(cudaGetLastError());
  b->delay_active = true;
  return RSB_OK;
}
int rsb_batch_clear_actuation_delay(rsb_batch* b) {
  if (!b) return fail(RSB_ERR_INVALID, "null batch");
  b->delay_active = false;
  return RSB_OK;
}
int rsb_batch_set_control_mode(rsb_batch* b, int mode) {
  if (!b || (mode != RSB_FORCE_AND_TORQUE && mode != RSB_PD_PLUS_FEEDFORWARD_TORQUE)) return fail(RSB_ERR_INVALID, "bad control mode");
  b->control_mode = mode;
  return RSB_OK;
}

static int ensure_debug(rsb_batch* b) {
  const size_t N = (size_t)b->N;
  CK(b->dbg_M.ensure(std::max<size_t>(16, N * b->nv * b->nv * 4), b->stream));
  CK(b->dbg_h.ensure(std::max<size_t>(16, N * b->nv * 4), b->stream));
  CK(b->dbg_R.ensure(N * b->nb * 9 * 4, b->stream));
  CK(b->dbg_p.ensure(N * b->nb * 3 * 4, b->stream));
  return RSB_OK;
}

int rsb_batch_integrate1(rsb_batch* b) {
  if (!b) return fail(RSB_ERR_INVALID, "null batch");
  CK(cudaSetDevice(b->device));
  int rc = ensure_debug(b); if (rc) return rc;
  return do_launch(b, 1, PHASE_NO_UPDATE, true);
}
int rsb_batch_update_kinematics(rsb_batch* b) {
  if (!b) return fail(RSB_ERR_INVALID, "null batch");
  CK(cudaSetDevice(b->device));
  int rc = ensure_debug(b); if (rc) return rc;
  return do_launch(b, 1, PHASE_NO_UPDATE | PHASE_KINEMATICS, true);      // stage A + the getters' buffers; contact records of the last integrate() untouched
}
// lazy getters: refresh M, h and the poses when the state changed through this API since they were last computed
static int ensure_kinematics(rsb_batch* b) {
  if (b->dbg_M.get() && !b->kin_dirty) return RSB_OK;
  return rsb_batch_update_kinematics(b);
}
int rsb_batch_integrate2(rsb_batch* b) {
  if (!b) return fail(RSB_ERR_INVALID, "null batch");
  CK(cudaSetDevice(b->device));
  // state is unchanged since integrate1(), so the fused step recomputes stage A-B on-chip and goes on;
  // generalized forces / PD targets set between integrate1() and integrate2() are honoured
  return do_launch(b, 1, 0, b->dbg_M.get() != nullptr);
}
int rsb_batch_integrate(rsb_batch* b, int substeps) {
  if (!b || substeps < 1) return fail(RSB_ERR_INVALID, "bad arguments to rsb_batch_integrate");
  CK(cudaSetDevice(b->device));
  return do_launch(b, substeps, 0, false);
}

int rsb_batch_get_mass_matrix(rsb_batch* b, int env_begin, int env_count, float* out, int where) {
  int rc = check_range(b, env_begin, env_count, where); if (rc) return rc;
  if (!out) return fail(RSB_ERR_INVALID, "null output buffer");
  if (env_count == 0) return RSB_OK;
  rc = ensure_kinematics(b); if (rc) return rc;
  const size_t w = (size_t)b->nv * b->nv;
  return copy_out(b, out, b->dbg_M.get() + env_begin * w, env_count * w * 4, where);
}
int rsb_batch_get_nonlinearities(rsb_batch* b, int env_begin, int env_count, float* out, int where) {
  int rc = check_range(b, env_begin, env_count, where); if (rc) return rc;
  if (!out) return fail(RSB_ERR_INVALID, "null output buffer");
  if (env_count == 0) return RSB_OK;
  rc = ensure_kinematics(b); if (rc) return rc;
  return copy_out(b, out, b->dbg_h.get() + (size_t)env_begin * b->nv, (size_t)env_count * b->nv * 4, where);
}
int rsb_batch_get_body_poses(rsb_batch* b, int env_begin, int env_count, float* rot, float* pos, int where) {
  int rc = check_range(b, env_begin, env_count, where); if (rc) return rc;
  if (env_count == 0) return RSB_OK;
  rc = ensure_kinematics(b); if (rc) return rc;
  rc = rot ? copy_out(b, rot, b->dbg_R.get() + (size_t)env_begin * b->nb * 9, (size_t)env_count * b->nb * 9 * 4, where) : RSB_OK; if (rc) return rc;
  return pos ? copy_out(b, pos, b->dbg_p.get() + (size_t)env_begin * b->nb * 3, (size_t)env_count * b->nb * 3 * 4, where) : RSB_OK;
}

// ---- frame kinematics: pose, velocity and Jacobian of frames rigidly attached to bodies, from the kinematics pass's poses ----------
int rsb_batch_set_frames(rsb_batch* b, const int32_t* body, const float* pos, const float* rot, int n) {
  if (!b) return fail(RSB_ERR_INVALID, "null batch");
  if (n < 0 || n > RSB_MAX_FRAMES) return fail(RSB_ERR_INVALID, "at most " + std::to_string(RSB_MAX_FRAMES) + " frames per batch (got " + std::to_string(n) + ")");
  if (n > 0 && (!body || !pos)) return fail(RSB_ERR_INVALID, "null frame body or position list");
  for (int f = 0; f < n; f++)
    if (body[f] < 0 || body[f] >= b->nb) return fail(RSB_ERR_INVALID, "frame " + std::to_string(f) + ": body index out of range (the model has " + std::to_string(b->nb) + ")");
  if (n == 0) { b->ftab.nf = 0; return RSB_OK; }
  const Model& md = b->model->md;
  const int nb = md.nb, nv = md.nv, F = RSB_MAX_FRAMES;
  // int words: body[F] | flags[F] | dof_body[nv] | dof_kind[nv] | anc[nb] | float words: pos[F][3] | rot[F][9] | dof_axis[nv][3]
  const int o_flags = F, o_dbody = 2 * F, o_dkind = o_dbody + nv, o_anc = o_dkind + nv, o_pos = o_anc + nb, o_rot = o_pos + 3 * F, o_axis = o_rot + 9 * F;
  const int words = o_axis + 3 * nv;
  std::vector<int32_t> W(words, 0);
  auto Fw = [&](int o, float v) { std::memcpy(&W[o], &v, 4); };
  for (int f = 0; f < n; f++) {
    W[f] = body[f];
    int flags = (pos[3 * f] == 0.f && pos[3 * f + 1] == 0.f && pos[3 * f + 2] == 0.f) ? FRAME_AT_ORIGIN : 0;
    bool ident = true;
    for (int k = 0; k < 9; k++) {
      const float r = rot ? rot[9 * f + k] : (k % 4 == 0 ? 1.f : 0.f);
      ident = ident && r == (k % 4 == 0 ? 1.f : 0.f);
      Fw(o_rot + 9 * f + k, r);
    }
    W[o_flags + f] = flags | (ident ? FRAME_IDENTITY : 0);
    for (int k = 0; k < 3; k++) Fw(o_pos + 3 * f + k, pos[3 * f + k]);
  }
  if (md.floating)
    for (int c = 0; c < 6; c++) {   // base: slides along, then turns about, the world axes through the base origin
      W[o_dbody + c] = 0; W[o_dkind + c] = (c < 3 ? JT_PRISMATIC : JT_REVOLUTE) | DOF_WORLD_AXIS;
      Fw(o_axis + 3 * c + c % 3, 1.f);
    }
  for (int i = 1; i < nb; i++) {
    const int c = md.vidx[i];
    W[o_dbody + c] = i; W[o_dkind + c] = md.jtype[i];
    for (int k = 0; k < 3; k++) Fw(o_axis + 3 * c + k, (float)md.axis[3 * i + k]);
  }
  for (int i = 0; i < nb; i++) {
    uint32_t m = 0;
    for (int j = i; j >= 0; j = md.parent[j]) m |= 1u << j;
    W[o_anc + i] = (int32_t)m;
  }
  CK(cudaSetDevice(b->device));
  CK(b->frame_tab.ensure((size_t)words * 4, b->stream));   // sized for RSB_MAX_FRAMES: the layout never moves
  CK(cudaMemcpyAsync(b->frame_tab.get(), W.data(), (size_t)words * 4, cudaMemcpyHostToDevice, b->stream));
  CK(cudaStreamSynchronize(b->stream));
  const int* T = b->frame_tab.get();
  b->ftab = FrameTable{n, nb, nv, T, T + o_flags, (const float*)(T + o_pos), (const float*)(T + o_rot), T + o_dbody, T + o_dkind,
                       (const float*)(T + o_axis), (const unsigned*)(T + o_anc)};
  return RSB_OK;
}
// one launch of rsb_frame_kernel (after the kinematics pass when the poses are stale); out = {pos, rot, lin_vel, ang_vel, jac}
static int frame_outputs(rsb_batch* b, int env_begin, int env_count, float* const out[5], int where) {
  int rc = check_range(b, env_begin, env_count, where); if (rc) return rc;
  if (b->ftab.nf == 0) return fail(RSB_ERR_INVALID, "no frames: call rsb_batch_set_frames() first");
  if (env_count == 0 || !(out[0] || out[1] || out[2] || out[3] || out[4])) return RSB_OK;
  CK(cudaSetDevice(b->device));
  // after integrate2() the getters' buffers hold the poses from before the step: the frame kernel pairs them with the current gv
  rc = b->kin_prestep ? rsb_batch_update_kinematics(b) : ensure_kinematics(b); if (rc) return rc;
  const size_t rows = (size_t)env_count * b->ftab.nf;
  const size_t per[5] = {3, 9, 3, 3, (size_t)6 * b->nv};
  float* dst[5] = {out[0], out[1], out[2], out[3], out[4]};
  if (where == RSB_HOST) {
    size_t need = 0;
    for (int k = 0; k < 5; k++) if (out[k]) need += rows * per[k];
    float* s = staging(b, need); if (!s) return RSB_ERR_CUDA;
    for (int k = 0; k < 5; k++) if (out[k]) { dst[k] = s; s += rows * per[k]; }
  }
  const int threads = 128;
  const unsigned blocks = (unsigned)((rows * 32 + threads - 1) / threads);
  rsb_frame_kernel<<<blocks, threads, 0, b->stream>>>(b->ftab, b->dbg_R.get(), b->dbg_p.get(), b->gv.get(), b->gv_stride, env_begin, env_count, dst[0], dst[1], dst[2], dst[3], dst[4]);
  CK(cudaGetLastError());
  b->launches++;
  if (where != RSB_HOST) return RSB_OK;
  for (int k = 0; k < 5; k++) if (out[k]) { rc = copy_out(b, out[k], dst[k], rows * per[k] * 4, RSB_HOST); if (rc) return rc; }
  return RSB_OK;
}
int rsb_batch_get_frame_states(rsb_batch* b, int env_begin, int env_count, float* pos, float* rot, float* lin_vel, float* ang_vel, int where) {
  float* const out[5] = {pos, rot, lin_vel, ang_vel, nullptr};
  return frame_outputs(b, env_begin, env_count, out, where);
}
int rsb_batch_get_frame_jacobians(rsb_batch* b, int env_begin, int env_count, float* jac, int where) {
  int rc = check_range(b, env_begin, env_count, where); if (rc) return rc;
  if (!jac) return fail(RSB_ERR_INVALID, "null output buffer");
  float* const out[5] = {nullptr, nullptr, nullptr, nullptr, jac};
  return frame_outputs(b, env_begin, env_count, out, where);
}
// ---- contact forces per body over a whole launch: the step kernel accumulates them sub-step by sub-step into the batch's rows --------
int rsb_batch_set_contact_bodies(rsb_batch* b, const int32_t* body, int n) {
  if (!b) return fail(RSB_ERR_INVALID, "null batch");
  if (n < 0 || n > RSB_MAX_CONTACT_BODIES) return fail(RSB_ERR_INVALID, "at most " + std::to_string(RSB_MAX_CONTACT_BODIES) + " contact bodies per batch (got " + std::to_string(n) + ")");
  if (n > 0 && !body) return fail(RSB_ERR_INVALID, "null contact body list");
  for (int s = 0; s < n; s++)
    if (body[s] < 0 || body[s] >= b->nb) return fail(RSB_ERR_INVALID, "contact body " + std::to_string(s) + ": body index out of range (the model has " + std::to_string(b->nb) + ")");
  if (n == 0) { b->contact_bodies.clear(); return RSB_OK; }
  CK(cudaSetDevice(b->device));
  const size_t rows = (size_t)b->N * RSB_MAX_CONTACT_BODIES;
  CK(b->cf_force.ensure(rows * 3 * 4, b->stream));
  CK(b->cf_steps.ensure(rows * 4, b->stream));
  // the rows of a new list read zero until a launch advances the state (in stream order: a step enqueued before this call still wrote the old layout)
  CK(cudaMemsetAsync(b->cf_force.get(), 0, rows * 3 * 4, b->stream));
  CK(cudaMemsetAsync(b->cf_steps.get(), 0, rows * 4, b->stream));
  b->contact_bodies.assign(body, body + n);
  return RSB_OK;
}
int rsb_batch_get_body_contact_forces(rsb_batch* b, int env_begin, int env_count, float* force, int32_t* steps_in_contact, int where) {
  int rc = check_range(b, env_begin, env_count, where); if (rc) return rc;
  if (b->contact_bodies.empty()) return fail(RSB_ERR_INVALID, "no contact bodies: call rsb_batch_set_contact_bodies() first");
  if (env_count == 0) return RSB_OK;
  CK(cudaSetDevice(b->device));
  const size_t S = b->contact_bodies.size();
  rc = force ? copy_out(b, force, b->cf_force.get() + (size_t)env_begin * S * 3, (size_t)env_count * S * 3 * 4, where) : RSB_OK; if (rc) return rc;
  return steps_in_contact ? copy_out(b, steps_in_contact, b->cf_steps.get() + (size_t)env_begin * S, (size_t)env_count * S * 4, where) : RSB_OK;
}
// ---- IMU readings over a whole launch: the step kernel accumulates them sub-step by sub-step into the batch's rows -------------------
int rsb_batch_set_imus(rsb_batch* b, const int32_t* body, const float* pos, const float* rot, int n) {
  if (!b) return fail(RSB_ERR_INVALID, "null batch");
  if (n < 0 || n > RSB_MAX_IMUS) return fail(RSB_ERR_INVALID, "at most " + std::to_string(RSB_MAX_IMUS) + " IMUs per batch (got " + std::to_string(n) + ")");
  if (n > 0 && (!body || !pos)) return fail(RSB_ERR_INVALID, "null IMU body or position list");
  std::vector<float> R(9 * (size_t)n);
  for (int k = 0; k < n; k++) {
    const std::string who = "IMU " + std::to_string(k) + ": ";
    if (body[k] < 0 || body[k] >= b->nb) return fail(RSB_ERR_INVALID, who + "body index out of range (the model has " + std::to_string(b->nb) + ")");
    for (int c = 0; c < 3; c++)
      if (!std::isfinite(pos[3 * k + c])) return fail(RSB_ERR_INVALID, who + "position is not finite");
    for (int c = 0; c < 9; c++) {
      R[9 * k + c] = rot ? rot[9 * k + c] : (c % 4 == 0 ? 1.f : 0.f);
      if (!std::isfinite(R[9 * k + c])) return fail(RSB_ERR_INVALID, who + "rotation is not finite");
    }
    const float* r = &R[9 * k];
    double dev = 0.0;   // largest entry of |R^T R - I|
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++) {
        double e = (i == j) ? -1.0 : 0.0;
        for (int m = 0; m < 3; m++) e += (double)r[3 * m + i] * (double)r[3 * m + j];
        dev = std::max(dev, std::fabs(e));
      }
    const double det = (double)r[0] * ((double)r[4] * r[8] - (double)r[5] * r[7]) - (double)r[1] * ((double)r[3] * r[8] - (double)r[5] * r[6]) +
                       (double)r[2] * ((double)r[3] * r[7] - (double)r[4] * r[6]);
    if (!(dev <= 1e-4) || !(det > 0.0)) return fail(RSB_ERR_INVALID, who + "orientation is not a rotation (|R^T R - I| <= 1e-4 and det R > 0 needed)");
  }
  if (n == 0) { b->imu_body.clear(); b->imu_pos.clear(); b->imu_rot.clear(); return RSB_OK; }
  CK(cudaSetDevice(b->device));
  const size_t words = (size_t)b->N * RSB_MAX_IMUS * 3;
  CK(b->imu_lin.ensure(words * 4, b->stream));
  CK(b->imu_ang.ensure(words * 4, b->stream));
  // the rows of a new list read zero until a launch advances the state (in stream order: a step enqueued before this call still wrote the old layout)
  CK(cudaMemsetAsync(b->imu_lin.get(), 0, words * 4, b->stream));
  CK(cudaMemsetAsync(b->imu_ang.get(), 0, words * 4, b->stream));
  b->imu_body.assign(body, body + n);
  b->imu_pos.assign(pos, pos + 3 * (size_t)n);
  b->imu_rot = R;
  return RSB_OK;
}
int rsb_batch_get_imu_readings(rsb_batch* b, int env_begin, int env_count, float* lin_acc, float* ang_vel, int where) {
  int rc = check_range(b, env_begin, env_count, where); if (rc) return rc;
  if (b->imu_body.empty()) return fail(RSB_ERR_INVALID, "no IMUs: call rsb_batch_set_imus() first");
  if (env_count == 0) return RSB_OK;
  CK(cudaSetDevice(b->device));
  const size_t I = b->imu_body.size();
  rc = lin_acc ? copy_out(b, lin_acc, b->imu_lin.get() + (size_t)env_begin * I * 3, (size_t)env_count * I * 3 * 4, where) : RSB_OK; if (rc) return rc;
  return ang_vel ? copy_out(b, ang_vel, b->imu_ang.get() + (size_t)env_begin * I * 3, (size_t)env_count * I * 3 * 4, where) : RSB_OK;
}
// ---- terrain height scans: the surface height under body-attached sample points, one launch of rsb_height_scan_kernel -------------
int rsb_batch_set_height_scan(rsb_batch* b, const int32_t* body, const float* xy, int n, int align) {
  if (!b) return fail(RSB_ERR_INVALID, "null batch");
  if (n < 0 || n > RSB_MAX_SCAN_POINTS) return fail(RSB_ERR_INVALID, "at most " + std::to_string(RSB_MAX_SCAN_POINTS) + " height-scan points per batch (got " + std::to_string(n) + ")");
  if (n > 0 && (!body || !xy)) return fail(RSB_ERR_INVALID, "null height-scan body or offset list");
  if (align != RSB_SCAN_YAW && align != RSB_SCAN_WORLD) return fail(RSB_ERR_INVALID, "height-scan align must be RSB_SCAN_YAW or RSB_SCAN_WORLD");
  for (int i = 0; i < n; i++) {
    if (body[i] < 0 || body[i] >= b->nb) return fail(RSB_ERR_INVALID, "height-scan point " + std::to_string(i) + ": body index out of range (the model has " + std::to_string(b->nb) + ")");
    if (!std::isfinite(xy[2 * i]) || !std::isfinite(xy[2 * i + 1])) return fail(RSB_ERR_INVALID, "height-scan point " + std::to_string(i) + ": offset is not finite");
  }
  if (n == 0) { b->scan.n = 0; return RSB_OK; }
  const int M = RSB_MAX_SCAN_POINTS;
  std::vector<int32_t> W((size_t)3 * M, 0);   // body[M] | xy[M][2]
  std::memcpy(W.data(), body, (size_t)n * 4);
  std::memcpy(W.data() + M, xy, (size_t)n * 8);
  const bool from_gc = b->model->md.floating;
  bool off_root = false;
  for (int i = 0; i < n; i++) off_root = off_root || !(body[i] == 0 && from_gc);
  CK(cudaSetDevice(b->device));
  CK(b->scan_tab.ensure(W.size() * 4, b->stream));   // sized for RSB_MAX_SCAN_POINTS: the layout never moves
  CK(cudaMemcpyAsync(b->scan_tab.get(), W.data(), W.size() * 4, cudaMemcpyHostToDevice, b->stream));
  CK(cudaStreamSynchronize(b->stream));   // the pageable source goes out of scope here
  const int* T = b->scan_tab.get();
  b->scan = ScanTable{n, align, from_gc ? 1 : 0, T, (const float*)(T + M)};
  b->scan_off_root = off_root;
  return RSB_OK;
}
int rsb_batch_get_height_scan(rsb_batch* b, int env_begin, int env_count, float* height, float* xy_out, int where) {
  int rc = check_range(b, env_begin, env_count, where); if (rc) return rc;
  if (b->scan.n == 0) return fail(RSB_ERR_INVALID, "no height-scan points: call rsb_batch_set_height_scan() first");
  if (b->ter.type != 1 && b->ter.type != 2) return fail(RSB_ERR_INVALID, "height scan: no terrain (set a ground or a height map first)");
  if (env_count == 0 || !(height || xy_out)) return RSB_OK;
  CK(cudaSetDevice(b->device));
  // poses off a floating root come from the kinematics pass; after integrate2() its buffers hold the state before the step
  if (b->scan_off_root) { rc = b->kin_prestep ? rsb_batch_update_kinematics(b) : ensure_kinematics(b); if (rc) return rc; }
  const size_t rows = (size_t)env_count * b->scan.n;
  float *dh = height, *dxy = xy_out;
  if (where == RSB_HOST) {
    float* s = staging(b, (height ? rows : 0) + (xy_out ? 2 * rows : 0)); if (!s) return RSB_ERR_CUDA;
    if (height) { dh = s; s += rows; }
    if (xy_out) dxy = s;
  }
  const int threads = 256;
  const unsigned blocks = (unsigned)((rows + threads - 1) / threads);
  rsb_height_scan_kernel<<<blocks, threads, 0, b->stream>>>(b->scan, b->ter, b->gc.get(), b->gc_stride, b->dbg_R.get(), b->dbg_p.get(), b->nb, env_begin, env_count, dh, dxy);
  CK(cudaGetLastError());
  b->launches++;
  if (where != RSB_HOST) return RSB_OK;
  if (height) { rc = copy_out(b, height, dh, rows * 4, RSB_HOST); if (rc) return rc; }
  return xy_out ? copy_out(b, xy_out, dxy, rows * 2 * 4, RSB_HOST) : RSB_OK;
}
// ---- ray casts: a body-mounted depth camera or lidar, one launch of rsb_ray_cast_kernel ----------------------------------------------
int rsb_batch_set_rays(rsb_batch* b, const int32_t* body, const float* origin, const float* dir, int n, float max_distance, int targets) {
  if (!b) return fail(RSB_ERR_INVALID, "null batch");
  if (n < 0 || n > RSB_MAX_RAYS) return fail(RSB_ERR_INVALID, "at most " + std::to_string(RSB_MAX_RAYS) + " rays per batch (got " + std::to_string(n) + ")");
  if (n > 0 && (!body || !origin || !dir)) return fail(RSB_ERR_INVALID, "null ray body, origin or direction list");
  if (!std::isfinite(max_distance) || !(max_distance > 0.f)) return fail(RSB_ERR_INVALID, "ray max_distance must be finite and > 0");
  if (targets != RSB_RAYS_TERRAIN && targets != RSB_RAYS_TERRAIN_AND_ROBOT) return fail(RSB_ERR_INVALID, "ray targets must be RSB_RAYS_TERRAIN or RSB_RAYS_TERRAIN_AND_ROBOT");
  const Model& md = b->model->md;
  const int M = RSB_MAX_RAYS, ncoll = md.ncoll();
  if (ncoll > RAY_MAX_SHAPES) return fail(RSB_ERR_UNSUPPORTED, "ray casts: more than " + std::to_string(RAY_MAX_SHAPES) + " collision bodies");
  std::vector<float> W((size_t)7 * M + (size_t)RAY_SHAPE_WORDS * ncoll, 0.f);   // body[M] | origin[M][3] | dir[M][3] | shapes
  int32_t* Wb = reinterpret_cast<int32_t*>(W.data());
  for (int i = 0; i < n; i++) {
    const std::string at = "ray " + std::to_string(i) + ": ";
    if (body[i] < 0 || body[i] >= b->nb) return fail(RSB_ERR_INVALID, at + "body index out of range (the model has " + std::to_string(b->nb) + ")");
    double d2 = 0;
    for (int k = 0; k < 3; k++) {
      if (!std::isfinite(origin[3 * i + k]) || !std::isfinite(dir[3 * i + k])) return fail(RSB_ERR_INVALID, at + "origin or direction is not finite");
      d2 += (double)dir[3 * i + k] * dir[3 * i + k];
    }
    const double nrm = std::sqrt(d2);
    if (!(nrm >= 1e-6)) return fail(RSB_ERR_INVALID, at + "direction is shorter than 1e-6");
    Wb[i] = body[i];
    for (int k = 0; k < 3; k++) { W[M + 3 * i + k] = origin[3 * i + k]; W[4 * M + 3 * i + k] = (float)(dir[3 * i + k] / nrm); }
  }
  if (n == 0) { b->rays.n = 0; return RSB_OK; }
  float* S = W.data() + (size_t)7 * M;
  for (int c = 0; c < ncoll; c++, S += RAY_SHAPE_WORDS) {
    const double* sz = &md.csize[3 * c];
    int32_t ib[2] = {md.cbody[c], md.ctype[c]};
    std::memcpy(S, ib, 8);
    for (int k = 0; k < 3; k++) { S[2 + k] = (float)sz[k]; S[5 + k] = (float)md.cpos[3 * c + k]; }
    for (int k = 0; k < 9; k++) S[8 + k] = (float)md.crot[9 * c + k];
    double bound = sz[0];   // sphere
    if (md.ctype[c] == CT_BOX) bound = std::sqrt(sz[0] * sz[0] + sz[1] * sz[1] + sz[2] * sz[2]);
    else if (md.ctype[c] != CT_SPHERE) bound = sz[0] + sz[1];
    S[17] = (float)(bound * 1.0001 + 1e-6);   // widened so that float32 rounding never culls a ray that touches the shape
  }
  const bool from_gc = md.floating && targets == RSB_RAYS_TERRAIN;
  bool kin = targets == RSB_RAYS_TERRAIN_AND_ROBOT;
  for (int i = 0; i < n; i++) kin = kin || !(body[i] == 0 && from_gc);
  CK(cudaSetDevice(b->device));
  CK(b->ray_tab.ensure((size_t)(7 * M + RAY_SHAPE_WORDS * RAY_MAX_SHAPES) * 4, b->stream));   // sized for the largest list: the layout never moves
  CK(cudaMemcpyAsync(b->ray_tab.get(), W.data(), W.size() * 4, cudaMemcpyHostToDevice, b->stream));
  CK(cudaStreamSynchronize(b->stream));   // the pageable source goes out of scope here
  const float* T = b->ray_tab.get();
  b->rays = RayTable{n, targets, from_gc ? 1 : 0, ncoll, max_distance, reinterpret_cast<const int*>(T), T + M, T + 4 * M, T + 7 * M};
  b->ray_kin = kin;
  return RSB_OK;
}
int rsb_batch_get_ray_casts(rsb_batch* b, int env_begin, int env_count, float* distance, int32_t* hit, int where) {
  int rc = check_range(b, env_begin, env_count, where); if (rc) return rc;
  if (b->rays.n == 0) return fail(RSB_ERR_INVALID, "no rays: call rsb_batch_set_rays() first");
  if (env_count == 0 || !(distance || hit)) return RSB_OK;
  CK(cudaSetDevice(b->device));
  // poses from the kinematics pass; after integrate2() its buffers hold the state before the step
  if (b->ray_kin) { rc = b->kin_prestep ? rsb_batch_update_kinematics(b) : ensure_kinematics(b); if (rc) return rc; }
  const size_t rows = (size_t)env_count * b->rays.n;
  float* dd = distance;
  int* dh = hit;
  if (where == RSB_HOST) {
    float* s = staging(b, (distance ? rows : 0) + (hit ? rows : 0)); if (!s) return RSB_ERR_CUDA;
    if (distance) { dd = s; s += rows; }
    if (hit) dh = reinterpret_cast<int*>(s);
  }
  const dim3 grid((unsigned)env_count, (unsigned)((b->rays.n + 255) / 256));
  rsb_ray_cast_kernel<<<grid, 256, 0, b->stream>>>(b->rays, b->ter, b->gc.get(), b->gc_stride, b->dbg_R.get(), b->dbg_p.get(), b->nb, env_begin, dd, dh);
  CK(cudaGetLastError());
  b->launches++;
  if (where != RSB_HOST) return RSB_OK;
  if (distance) { rc = copy_out(b, distance, dd, rows * 4, RSB_HOST); if (rc) return rc; }
  return hit ? copy_out(b, hit, dh, rows * 4, RSB_HOST) : RSB_OK;
}
int rsb_batch_get_contacts(rsb_batch* b, rsb_contact* out, int32_t* counts, int env_begin, int env_count, int where) {
  int rc = check_range(b, env_begin, env_count, where); if (rc) return rc;
  rc = out ? copy_out(b, out, b->contacts.get() + (size_t)env_begin * KMAX, (size_t)env_count * KMAX * sizeof(rsb_contact), where) : RSB_OK; if (rc) return rc;
  return counts ? copy_out(b, counts, b->ncontacts.get() + env_begin, (size_t)env_count * 4, where) : RSB_OK;
}
int rsb_batch_get_contact_points(rsb_batch* b, int32_t* pt, int env_begin, int env_count, int where) {
  int rc = check_range(b, env_begin, env_count, where); if (rc) return rc;
  if (!pt) return fail(RSB_ERR_INVALID, "null output buffer");
  return copy_out(b, pt, b->contact_pt.get() + (size_t)env_begin * KMAX, (size_t)env_count * KMAX * 4, where);
}
int rsb_batch_get_solver_iterations(rsb_batch* b, int32_t* it, int env_begin, int env_count, int where) {
  int rc = check_range(b, env_begin, env_count, where); if (rc) return rc;
  if (!it) return fail(RSB_ERR_INVALID, "null output buffer");
  return copy_out(b, it, b->iters.get() + env_begin, (size_t)env_count * 4, where);
}
int rsb_batch_get_solver_status(rsb_batch* b, int32_t* status, int env_begin, int env_count, int where) {
  int rc = check_range(b, env_begin, env_count, where); if (rc) return rc;
  if (!status) return fail(RSB_ERR_INVALID, "null output buffer");
  return copy_out(b, status, b->solver_status.get() + env_begin, (size_t)env_count * 4, where);
}
int rsb_batch_get_solver_residual(rsb_batch* b, float* resid, int env_begin, int env_count, int where) {
  int rc = check_range(b, env_begin, env_count, where); if (rc) return rc;
  if (!resid) return fail(RSB_ERR_INVALID, "null output buffer");
  return copy_out(b, resid, b->resid.get() + env_begin, (size_t)env_count * 4, where);
}
int rsb_batch_get_diverged(rsb_batch* b, int32_t* flags, int env_begin, int env_count, int where) {
  int rc = check_range(b, env_begin, env_count, where); if (rc) return rc;
  if (!flags) return fail(RSB_ERR_INVALID, "null output buffer");
  return copy_out(b, flags, b->diverged.get() + env_begin, (size_t)env_count * 4, where);
}
int rsb_batch_device_ptrs(rsb_batch* b, rsb_device_view* v) {
  if (!b || !v) return fail(RSB_ERR_INVALID, "null argument");
  v->num_envs = b->N; v->nq = b->nq; v->nv = b->nv; v->gc_stride = b->gc_stride; v->gv_stride = b->gv_stride;
  v->gc = b->gc.get(); v->gv = b->gv.get(); v->tau_ff = b->tau.get(); v->ptarget = b->pt.get(); v->vtarget = b->vt.get();
  v->ncontacts = b->ncontacts.get(); v->contacts = b->contacts.get();
  return RSB_OK;
}
int64_t rsb_batch_launch_count(const rsb_batch* b) { return b ? b->launches : 0; }

int rsb_batch_ob_dim(const rsb_batch* b) {
  if (!b) return 0;
  return b->model->md.floating ? (b->nq + b->nv - 3) : (b->nq + b->nv);
}
static int observe_impl(rsb_batch* b, float* obs, int env_begin, int env_count, int where) {
  const int od = rsb_batch_ob_dim(b);
  float* dst = obs;
  if (where == RSB_HOST && !(dst = staging(b, (size_t)env_count * od))) return RSB_ERR_CUDA;
  int threads = 128, blocks = (env_count * 32 + threads - 1) / threads;
  rsb_observe_kernel<<<blocks, threads, 0, b->stream>>>(b->gc.get() + (size_t)env_begin * b->gc_stride, b->gv.get() + (size_t)env_begin * b->gv_stride,
                                                         b->gc_stride, b->gv_stride, b->nq, b->nv, b->model->md.floating, env_count, dst, od);
  CK(cudaGetLastError());
  b->launches++;
  return where == RSB_HOST ? copy_out(b, obs, dst, (size_t)env_count * od * 4, RSB_HOST) : RSB_OK;
}
int rsb_batch_observe(rsb_batch* b, float* obs, int env_begin, int env_count, int where) {
  int rc = check_range(b, env_begin, env_count, where); if (rc) return rc;
  if (!obs) return fail(RSB_ERR_INVALID, "null obs");
  if (env_count == 0) return RSB_OK;
  CK(cudaSetDevice(b->device));
  return observe_impl(b, obs, env_begin, env_count, where);
}

// VectorizedEnvironment::step() for the whole batch in ONE call: PD targets in, `substeps` fused
// World::integrate() calls, observation rows out.  Host buffers should be pinned (cudaHostAlloc /
// torch pin_memory) so that the copies overlap; the call returns after the observations have landed.
int rsb_batch_control_step(rsb_batch* b, const float* ptarget, const float* vtarget, int where_in, int substeps, float* obs, int where_out) {
  if (!b || substeps < 1) return fail(RSB_ERR_INVALID, "bad arguments to rsb_batch_control_step");
  if (bad_where(where_in) || bad_where(where_out)) return fail(RSB_ERR_INVALID, "`where_in` and `where_out` must be RSB_HOST or RSB_DEVICE");
  CK(cudaSetDevice(b->device));
  // Host buffers in pinned (page-locked, mapped) memory are read and written IN PLACE by the step kernel over PCIe:
  // no staging copy, no separate H2D / D2H operations on the stream.  Pageable buffers take the staged path.
  // Targets given here end a persistent rsb_batch_bind_pd_target() binding; pinned ones are read in place by this launch only.
  const bool pd_mode = pd_active(b);
  LaunchIO io;
  int rc = RSB_OK;
  if (ptarget) {
    b->pt_bound = nullptr;
    io.pt = (where_in == RSB_HOST && pd_mode) ? mapped_alias(ptarget) : nullptr;
    if (!io.pt) { rc = copy_rows_in(b, b->pt.get(), b->gc_stride, ptarget, b->nq, 0, b->N, where_in); if (rc) return rc; }
  }
  if (vtarget) {
    b->vt_bound = nullptr;
    io.vt = (where_in == RSB_HOST && pd_mode) ? mapped_alias(vtarget) : nullptr;
    if (!io.vt) { rc = copy_rows_in(b, b->vt.get(), b->gv_stride, vtarget, b->nv, 0, b->N, where_in); if (rc) return rc; }
  }
  const bool in_place = io.pt || io.vt;   // the caller may reuse its pinned target buffer when the call returns
  if (!obs || !b->model->md.floating) {
    rc = do_launch(b, substeps, 0, false, io); if (rc) return rc;
    if (obs) rc = observe_impl(b, obs, 0, b->N, where_out);
    if (in_place) CK(cudaStreamSynchronize(b->stream));
    return rc;
  }
  // observation rows are written by the step kernel itself (no separate observe launch)
  const int od = rsb_batch_ob_dim(b);
  io.obs = where_out == RSB_HOST ? const_cast<float*>(mapped_alias(obs)) : nullptr;
  if (io.obs) {   // observation rows go straight to the caller's pinned buffer as each environment finishes
    rc = do_launch(b, substeps, 0, false, io); if (rc) return rc;
    CK(cudaStreamSynchronize(b->stream));
    return RSB_OK;
  }
  if (where_out == RSB_HOST) {
    if (!(io.obs = staging(b, (size_t)b->N * od))) return RSB_ERR_CUDA;
    rc = do_launch(b, substeps, 0, false, io); if (rc) return rc;
    return copy_out(b, obs, io.obs, (size_t)b->N * od * 4, RSB_HOST);
  }
  io.obs = obs; io.peers = true;
  rc = do_launch(b, substeps, 0, false, io); if (rc) return rc;
  if (in_place) CK(cudaStreamSynchronize(b->stream));
  return RSB_OK;
}

// ---- RaisimGym ANYmal task (SURVEY 8f N1): VectorizedEnvironment::{reset, step, observe} for the whole batch ----
int rsb_batch_gym_configure(rsb_batch* b, const float* gc_init, const float* gv_init, const float* action_mean, const float* action_std,
                            const int32_t* foot_bodies, int n_foot, float torque_coeff, float forward_vel_coeff, float terminal_reward) {
  if (!b || !gc_init || !gv_init || !action_mean || !action_std || (n_foot > 0 && !foot_bodies)) return fail(RSB_ERR_INVALID, "null argument");
  if (!b->model->md.floating) return fail(RSB_ERR_UNSUPPORTED, "the gym task needs a floating-base robot");
  CK(cudaSetDevice(b->device));
  const int nq = b->nq, nv = b->nv, nj = nq - 7;
  std::vector<float> h((size_t)nq + nv + 2 * nj);
  std::memcpy(h.data(), gc_init, nq * 4); std::memcpy(h.data() + nq, gv_init, nv * 4);
  std::memcpy(h.data() + nq + nv, action_mean, nj * 4); std::memcpy(h.data() + nq + nv + nj, action_std, nj * 4);
  CK(b->gym_const.ensure(h.size() * 4, b->stream));
  CK(b->gym_action.ensure((size_t)b->N * nj * 4, b->stream));
  CK(b->gym_obs.ensure((size_t)b->N * rsb_batch_ob_dim(b) * 4, b->stream));
  CK(b->gym_reward.ensure((size_t)b->N * 4, b->stream));
  CK(b->gym_done.ensure((size_t)b->N, b->stream));
  CK(cudaMemcpyAsync(b->gym_const.get(), h.data(), h.size() * 4, cudaMemcpyHostToDevice, b->stream));
  CK(cudaStreamSynchronize(b->stream));
  const float* c = b->gym_const.get();
  b->gym.gc_init = c; b->gym.gv_init = c + nq; b->gym.action_mean = c + nq + nv; b->gym.action_std = c + nq + nv + nj;
  b->gym.foot_mask = 0;
  for (int i = 0; i < n_foot; i++) {
    if (foot_bodies[i] < 0 || foot_bodies[i] >= b->nb) return fail(RSB_ERR_INVALID, "foot body index out of range");
    b->gym.foot_mask |= 1u << foot_bodies[i];
  }
  b->gym.torque_coeff = torque_coeff; b->gym.forward_vel_coeff = forward_vel_coeff; b->gym.terminal_reward = terminal_reward;
  b->gym_ready = true;
  return RSB_OK;
}

// ENVIRONMENT::reset() for every environment: state and PD target back to the initial configuration
int rsb_batch_gym_reset(rsb_batch* b) {
  if (!b || !b->gym_ready) return fail(RSB_ERR_INVALID, "call rsb_batch_gym_configure() first");
  CK(cudaSetDevice(b->device));
  int threads = 128, blocks = (b->N * 32 + threads - 1) / threads;
  rsb_gym_reset_kernel<<<blocks, threads, 0, b->stream>>>(b->gc.get(), b->gv.get(), b->pt.get(), b->vt.get(), b->gym, b->gc_stride, b->gv_stride, b->nq, b->nv, b->N,
                                                          b->an_dofs.empty() ? nullptr : b->an_hist.get(), (int)an_hist_words(b),
                                                          b->delay_active ? b->delay_state.get() : nullptr);
  CK(cudaGetLastError());
  b->kin_dirty = true;
  b->launches++;
  return RSB_OK;
}

// VectorizedEnvironment::step(action, reward, done) + observe(ob): action rows [N][nq-7] in; `substeps` fused
// World::integrate() calls; reward [N], done [N] (uint8) and observation rows [N][ob_dim] out.
int rsb_batch_gym_step(rsb_batch* b, const float* action, int where_in, int substeps, float* obs, float* reward, unsigned char* done, int where_out) {
  if (!b || !b->gym_ready) return fail(RSB_ERR_INVALID, "call rsb_batch_gym_configure() first");
  if (!action || substeps < 1) return fail(RSB_ERR_INVALID, "bad arguments to rsb_batch_gym_step");
  if (bad_where(where_in) || bad_where(where_out)) return fail(RSB_ERR_INVALID, "`where_in` and `where_out` must be RSB_HOST or RSB_DEVICE");
  CK(cudaSetDevice(b->device));
  const int nj = b->nq - 7, od = rsb_batch_ob_dim(b);
  b->pt_bound = nullptr;              // the task writes its own PD-target rows
  // pinned host buffers are read / written in place by the task kernels (see rsb_batch_control_step)
  const float* act = action;
  if (where_in == RSB_HOST) {
    act = mapped_alias(action);
    if (!act) {
      CK(cudaMemcpyAsync(b->gym_action.get(), action, (size_t)b->N * nj * 4, cudaMemcpyHostToDevice, b->stream));
      act = b->gym_action.get();
    }
  }
  const bool host_out = where_out == RSB_HOST;
  float* a_obs = (host_out && obs) ? const_cast<float*>(mapped_alias(obs)) : nullptr;
  float* a_rew = (host_out && reward) ? const_cast<float*>(mapped_alias(reward)) : nullptr;
  unsigned char* a_done = (host_out && done) ? reinterpret_cast<unsigned char*>(const_cast<float*>(mapped_alias(done))) : nullptr;
  float* d_obs = a_obs ? a_obs : (host_out || !obs) ? b->gym_obs.get() : obs;
  float* d_rew = a_rew ? a_rew : (host_out || !reward) ? b->gym_reward.get() : reward;
  unsigned char* d_done = a_done ? a_done : (host_out || !done) ? b->gym_done.get() : done;
  // ONE launch: action rows -> PD targets, `substeps` x World::integrate(), reward, isTerminalState(), reset() of the terminated
  // environments and the observation rows of the resulting state (the task used to be an action kernel and a post kernel around the step)
  if (!pd_active(b)) return fail(RSB_ERR_INVALID, "the gym task drives the robot through PD targets: call rsb_batch_set_pd_gains(), rsb_batch_set_actuator_params() or rsb_batch_set_actuator_network() first");
  LaunchIO io;
  io.obs = d_obs; io.gym_action = act; io.gym_reward = d_rew; io.gym_done = d_done;
  int rc = do_launch(b, substeps, 0, false, io); if (rc) return rc;
  if (where_out == RSB_HOST) {
    if (obs && !a_obs) CK(cudaMemcpyAsync(obs, d_obs, (size_t)b->N * od * 4, cudaMemcpyDeviceToHost, b->stream));
    if (reward && !a_rew) CK(cudaMemcpyAsync(reward, d_rew, (size_t)b->N * 4, cudaMemcpyDeviceToHost, b->stream));
    if (done && !a_done) CK(cudaMemcpyAsync(done, d_done, (size_t)b->N, cudaMemcpyDeviceToHost, b->stream));
    CK(cudaStreamSynchronize(b->stream));
  } else if (where_in == RSB_HOST && act != b->gym_action.get()) {
    CK(cudaStreamSynchronize(b->stream));   // the action rows were read in place from pinned host memory: the caller may reuse them on return
  }
  return RSB_OK;
}

// ---- fused observation all-gather over NVLink peer memory (SURVEY 8e; one process per GPU or one process for all) ----
// Buffers that other processes map: plain cudaMalloc memory + a CUDA IPC handle (64 bytes) to ship over any host channel.
int rsb_peer_buffer_create(int device, size_t bytes, void** dev_ptr, unsigned char* handle64) {
  if (!dev_ptr || bytes == 0) return fail(RSB_ERR_INVALID, "bad arguments to rsb_peer_buffer_create");
  CK(cudaSetDevice(device));
  void* p = nullptr;
  CK(cudaMalloc(&p, bytes));
  cudaError_t e = cudaMemset(p, 0, bytes);
  if (e == cudaSuccess && handle64) {
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle is 64 bytes");
    cudaIpcMemHandle_t h;
    e = cudaIpcGetMemHandle(&h, p);
    if (e == cudaSuccess) std::memcpy(handle64, &h, 64);
  }
  if (e != cudaSuccess) { cudaFree(p); return fail(RSB_ERR_CUDA, std::string("rsb_peer_buffer_create: ") + cudaGetErrorString(e)); }
  *dev_ptr = p;
  return RSB_OK;
}
int rsb_peer_buffer_open(int device, const unsigned char* handle64, void** dev_ptr) {
  if (!dev_ptr || !handle64) return fail(RSB_ERR_INVALID, "null argument");
  CK(cudaSetDevice(device));
  cudaIpcMemHandle_t h;
  std::memcpy(&h, handle64, 64);
  CK(cudaIpcOpenMemHandle(dev_ptr, h, cudaIpcMemLazyEnablePeerAccess));
  return RSB_OK;
}
int rsb_peer_buffer_close(void* dev_ptr) { if (dev_ptr) CK(cudaIpcCloseMemHandle(dev_ptr)); return RSB_OK; }
int rsb_peer_buffer_destroy(void* dev_ptr) { if (dev_ptr) CK(cudaFree(dev_ptr)); return RSB_OK; }

// obs_all[2 * world]: for every rank r, its two gathered-rows buffers (parity 0, 1), each [world * num_envs][ob_dim] float32, as
// device pointers valid in THIS process (own allocations, IPC mappings, or peer-enabled pointers of other devices of this process);
// flags[world]: rank r's arrival counters, unsigned[world], zero-initialised.  From now on every control step that returns
// observation rows on the device also stores them into the buffer (step parity) of every rank and bumps flags[r][rank] once
// per finished CTA.  world = 0 switches the fused gather off.  Every rank must run the same num_envs.
int rsb_batch_set_observation_peers(rsb_batch* b, int world, int rank, void* const* obs_all, void* const* flags) {
  if (!b) return fail(RSB_ERR_INVALID, "null batch");
  if (world == 0) { b->peer_world = 0; return RSB_OK; }
  if (world < 1 || world > MAX_PEERS || rank < 0 || rank >= world || !obs_all || !flags) return fail(RSB_ERR_INVALID, "bad arguments to rsb_batch_set_observation_peers");
  if (!b->model->md.floating) return fail(RSB_ERR_UNSUPPORTED, "fused observation rows need a floating-base robot");
  for (int p = 0; p < world; p++) if (!obs_all[2 * p] || !obs_all[2 * p + 1] || !flags[p]) return fail(RSB_ERR_INVALID, "null peer buffer");
  CK(cudaSetDevice(b->device));
  CK(cudaStreamSynchronize(b->stream));
  b->peer_world = 0;              // a failure below leaves the batch without peers
  CK(b->peer_done.ensure(sizeof(unsigned), b->stream));
  CK(cudaMemsetAsync(b->peer_done.get(), 0, sizeof(unsigned), b->stream));
  for (int p = 0; p < world; p++) { b->peer_obs[p][0] = (float*)obs_all[2 * p]; b->peer_obs[p][1] = (float*)obs_all[2 * p + 1]; b->peer_flag[p] = (unsigned*)flags[p]; }
  b->peer_world = world; b->peer_rank = rank; b->peer_epoch = 0;
  return RSB_OK;
}
// *buffer_parity (optional) = which of this rank's two buffers holds the rows of the LAST control step of every rank.  The arrival
// wait itself is part of that control step's launch (its last CTA stays until every rank's rows have landed), so in stream order
// after the step the rows are complete and nothing is enqueued here.
int rsb_batch_wait_observation_peers(rsb_batch* b, int* buffer_parity) {
  if (!b || b->peer_world <= 0 || b->peer_epoch == 0) return fail(RSB_ERR_INVALID, "no fused observation gather in flight");
  if (buffer_parity) *buffer_parity = (int)((b->peer_epoch - 1) & 1);
  return RSB_OK;
}

// ---- hooks for comm.cu -----------------------------------------------------------------------------
int rsb_internal_batch_info(rsb_batch* b, int* device, void** stream, int* num_envs) {
  if (!b) return fail(RSB_ERR_INVALID, "null batch");
  if (device) *device = b->device;
  if (stream) *stream = (void*)b->stream;
  if (num_envs) *num_envs = b->N;
  return RSB_OK;
}
// profiling hook (tools/balance_probe.py): device buffer [num_envs][4][8] of SM-clock stamps, or null to switch off
int rsb_internal_set_profile(rsb_batch* b, unsigned* dev) { if (!b) return -1; b->prof = dev; return 0; }
// profiling hook (tools/stage_probe.py): device buffer [num_envs][4][4] of SM-clock stamps inside stage A, or null to switch off
int rsb_internal_set_profile_stage_a(rsb_batch* b, unsigned* dev) { if (!b) return -1; b->prof_a = dev; return 0; }
// launch shape of the step kernel (tools/stage_probe.py, tests): warps per CTA and CTAs; environment e runs in round
// e / (wpc * grid) on CTA (e % (wpc * grid)) / wpc.  RSB_FORCE_WPC is dropped without a message when the CTA does not fit in shared
// memory, so a caller that forces a configuration reads back what it got here.
int rsb_internal_launch_config(const rsb_batch* b, int* wpc, int* grid) {
  if (!b || !wpc || !grid) return fail(RSB_ERR_INVALID, "null argument");
  *wpc = b->cfg.wpc; *grid = b->cfg.grid;
  return RSB_OK;
}
// compiled instance of the step kernel that the batch launches (dispatch_spec): spec 0 generic, 1 quadruped, 2 humanoid; slots =
// candidate points per lane (tests).  A hook of its own, so that callers of rsb_internal_launch_config keep their signature
int rsb_internal_launch_instance(const rsb_batch* b, int* spec, int* slots) {
  if (!b || !spec || !slots) return fail(RSB_ERR_INVALID, "null argument");
  *spec = b->cfg.spec; *slots = b->cfg.slots;
  return RSB_OK;
}
// the stage-B cull height of a height-map terrain (TerrainDesc::hmax) the next launch uses (tests: it must stay the exact maximum over all maps)
int rsb_internal_terrain_hmax(const rsb_batch* b, float* hmax) {
  if (!b || !hmax) return fail(RSB_ERR_INVALID, "null argument");
  if (b->ter.type != 2) return fail(RSB_ERR_INVALID, "no height map");
  *hmax = b->ter.hmax;
  return RSB_OK;
}
void rsb_internal_set_error(const char* msg) { g_err = msg ? msg : ""; }

}  // extern "C"
