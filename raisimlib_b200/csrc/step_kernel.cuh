// Fused World::integrate() for a batch of environments -- hand-written sm_90a CUDA.
//
// One warp == one environment (BASELINE.json north_star).  A CTA of WPC warps shares the model
// constant block, staged global -> shared ONCE per CTA by a TMA bulk copy (cp.async.bulk +
// mbarrier; SASS: UBLKCP).  Every per-environment intermediate (body poses, M / its Cholesky
// factor, contact Jacobians, Delassus matrix) lives in that warp's shared-memory workspace; HBM is
// touched only for the coalesced state rows in, state rows + contact records out.
//
// Stages (SURVEY.md section 8a rows a2..a10, same math as oracle/rbd_oracle.hpp):
//   A  lane = body   : FK + RNEA forward walk down each body's own ancestor chain (registers),
//                      per-body force / composite-inertia terms, subtree sums by warp shuffles
//                      -> h, M (CRBA in a world-aligned frame centred on the base)
//   B  lane = point  : candidate point vs Ground / HeightMap, ballot-compacted contact list
//   C  lane = entry / column : b, Mhat = M + dt Kd + dt^2 Kp, branch-sparse Mhat = L^T L (Featherstone RBDA
//                      6.5) in compact-by-depth storage, z = L^-T b, Y = L^-T J^T (only the contact's own
//                      ancestor chain is touched), G = Y^T Y (sum up to the LCA depth)
//   D  lane = row    : per-contact Gauss-Seidel; slip by a 32-way section search (all lanes probe)
//   E  lane = dof    : v+ = v + L^-1 (dt z + Y lam), q+ = q (+) dt v+
//
// Compact-by-depth storage: the ancestors of a dof have distinct depths 0..d, so row i of the lower
// triangle of M (non-zero only at ancestors) is stored as Lc[i][t], t = depth of the ancestor.  For
// k in subtree(i), "the ancestor of k at depth(i)" IS i, which turns every tree-sparse update into
// plain strided loops over the contiguous DFS range of descendants.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/rsb.h"
#include "contact_solver.cuh"

namespace rsb {

constexpr int KMAX = RSB_KMAX;
constexpr int CMAX = 3 * KMAX;      // contact rows
constexpr int LMAX = RSB_LMAX;      // joint-limit rows (first LMAX violated joints)
constexpr int RMAX = CMAX + LMAX;   // constraint rows: one lane each (<= 32)
constexpr int CP = RMAX + 1;        // Y row stride (odd)
constexpr int GP = RMAX + 1;        // G row stride (odd: conflict-free row access by lane)
static_assert(RMAX <= 32, "one constraint row per lane");
constexpr int NSEC = 32;
constexpr int NROUNDS = 2;         // 32-section rounds of the slip search: bracket 2*pi/32^(r+1); two regula-falsi steps finish it (contact_solver.cuh)
constexpr int SEC_STRIDE = 36;      // (NSEC+1) padded
constexpr int CT_WORDS = 16;        // per-contact shared record
constexpr int EXT_WORDS = 12;       // external wrench row: body (int bits), force(3), torque(3), point in the body frame(3), 2 pad
constexpr int BI_WORDS = 12;        // per-environment inertial row of one body: mass, com(3), inertia xx xy xz yy yz zz, 2 pad (three float4)
constexpr int MAX_PT_SLOTS = 2;     // candidate points per lane (npts <= 64)
constexpr int HIST_WORDS = 6 * 32;  // Anderson history of the Gauss-Seidel sweep map (stage D)
constexpr int MAX_PEERS = 8;        // GPUs of one NVSwitch domain that receive this GPU's observation rows (fused all-gather)
constexpr unsigned FULL = 0xffffffffu;

enum BodyField {
  BF_PARENT = 0, BF_JTYPE = 1, BF_QIDX = 2, BF_VIDX = 3, BF_DEPTH = 4, BF_SUBTREE = 5,
  BF_JPOS = 6, BF_JROT = 9, BF_AXIS = 18, BF_MASS = 21, BF_COM = 22, BF_INERTIA = 25, BF_LO = 31, BF_HI = 32, BF_COUNT = 33
};
enum PoseField { PF_R = 0, PF_P = 9, PF_A = 12, PF_COUNT = 15 };
enum CtField { CF_POS = 0, CF_N = 3, CF_T1 = 6, CF_T2 = 9, CF_DEPTH = 12, CF_PT = 13, CF_BODY = 14, CF_PAIR = 15 };

// Model dimensions that fix every table offset.  A kernel can be compiled for a given Dims
// (offsets become immediates) or read them from the blob header at run time (generic path).
struct Dims { int nb, nq, nv, floating, maxdepth, maxdd; };

__host__ __device__ constexpr int round_up_c(int x, int m) { return (x + m - 1) / m * m; }
__host__ __device__ constexpr int max_c(int a, int b) { return a > b ? a : b; }

// header of the model constant blob (first 32 words)
struct BlobHeader {
  int nb, nq, nv, npts, floating, maxdepth, nbp, nptp, nvp, nqp;
  int off_body, off_anc, off_pts, off_gain, off_dofq, off_sec;
  // dof tree (floating base = chain of 6 dofs) for the branch-sparse factorisation
  int nbase, maxdd, dlp, nent;
  int off_ddepth, off_dsub, off_danc, off_dbody, off_bdof, off_lvl, off_lvldofs, off_entstart, off_ent, off_lcad;
  int off_coll, ncoll; // collision-body table (box features): [ncoll][COLL_WORDS] = half extents, body-frame position, rotation
  int words, flags;    // flags bit0: every joint origin has identity rotation (rpy = 0 in the URDF); bits 8..15: largest
                       // non-root subtree size - 1 (loop bound of stage A's subtree accumulation)
  int npairs, off_pair; // enabled self-collision pairs (rsb_batch_set_self_collision; 0 = off) and their table: [npairs][PAIR_WORDS]
};
static_assert(sizeof(BlobHeader) == 144, "header is 36 words");
constexpr int HEADER_WORDS = 36;      // a 16-byte multiple
constexpr int PT_ROWS = 15;           // candidate table rows: body, pos(3), radius, friction override, type, pos2(3), collision body, cull point(3), cull radius
constexpr int COLL_WORDS = 16;
constexpr int MAX_SELF_PAIRS = RSB_MAX_SELF_PAIRS;   // one lane of stage B each
// Self-collision pair row (one contact per pair, candidate index npts + j).  Geometry in the frames of two bodies A and B: kind 0 = the
// segment a0..a1 swept by rA against b0..b1 swept by rB (a sphere is a segment of length 0), kind 1 = the sphere a0, rA against the box of
// centre b0, half extents b1 and rotation bR in the frame of B.  The normal points from B to A, negated when flip = 1 (the caller listed
// the box first).  The impulse acts on body1, its negative on body2.  Cull radii: bounding spheres about the middle of a0..a1 and of
// b0..b1 (kind 0) or about b0 (kind 1).
enum PairField { PR_KIND = 0, PR_FLIP = 1, PR_BODY1 = 2, PR_BODY2 = 3, PR_BA = 4, PR_BB = 5, PR_A0 = 6, PR_A1 = 9, PR_B0 = 12, PR_B1 = 15,
                 PR_BR = 18, PR_RA = 27, PR_RB = 28, PR_MU = 29, PR_CULL_A = 30, PR_CULL_B = 31, PAIR_WORDS = 32 };

// Every offset except off_ent / words depends on Dims only: the two variable-size tables
// (candidate points, factorisation entry list) sit at the end.
__host__ __device__ constexpr BlobHeader make_blob_header(Dims d, int npts, int nent, int ncoll = 0, int npairs = 0) {
  BlobHeader H{};
  H.nb = d.nb; H.nq = d.nq; H.nv = d.nv; H.npts = npts; H.floating = d.floating; H.maxdepth = d.maxdepth;
  H.nbp = d.nb | 1;                       // odd stride: field-major reads by body index stay conflict-free
  H.nptp = max_c(1, npts);
  H.nvp = round_up_c(max_c(d.nv, 1), 4);
  H.nqp = round_up_c(max_c(d.nq, 1), 4);
  H.nbase = d.floating ? 6 : 0; H.maxdd = d.maxdd; H.dlp = (d.maxdd + 1) | 1; H.nent = nent;
  const int DL = d.maxdd + 1;
  int off = HEADER_WORDS;
  H.off_body = off; off += 33 * H.nbp;
  H.off_anc = off; off += max_c(1, d.maxdepth) * H.nbp;
  H.off_gain = off; off += 3 * H.nvp;                 // kp, kd, actuator effort limit per dof
  H.off_dofq = off; off += H.nvp;
  H.off_sec = off; off += 2 * NROUNDS * SEC_STRIDE;
  H.off_ddepth = off; off += H.nvp;
  H.off_dsub = off; off += H.nvp;
  H.off_danc = off; off += DL * H.nvp;
  H.off_dbody = off; off += H.nvp;
  H.off_bdof = off; off += H.nbp;
  H.off_lvl = off; off += DL + 1;
  H.off_lvldofs = off; off += H.nvp;
  H.off_entstart = off; off += DL + 1;
  H.off_lcad = off; off += (d.nb * H.nbp + 3) / 4;
  H.off_pts = off; off += PT_ROWS * H.nptp;           // body, pos(3), radius, friction override (< 0: default material), type, pos2(3), collision body, cull point(3) + radius
  H.ncoll = ncoll; H.off_coll = off; off += COLL_WORDS * ncoll;
  H.off_ent = off; off += max_c(1, nent);
  H.npairs = npairs; H.off_pair = off; off += PAIR_WORDS * npairs;   // at the end: without pairs the blob is what it was
  H.words = round_up_c(off, 4);
  return H;
}

// second column block of the self contacts (stage C): Y of the pair's second body, [ancestor depth][contact row], at the end of the
// workspace; allocated only when pairs are enabled (make_ws_layout)
__host__ __device__ constexpr int self_y_words(int maxdd) { return round_up_c((maxdd + 1) * (3 * RSB_KMAX + RSB_LMAX + 1), 4); }

// stage B's per-warp hit list (stage_b_narrow_phase): HL_CAP rows of HL_WORDS words
constexpr int HL_WORDS = 9;            // depth (<= 0: dropped), normal, position, pair, candidate index; odd stride: conflict-free by lane
constexpr int HL_CAP = 64;             // two candidate slots per lane at most

// per-warp workspace layout (word offsets)
struct WsLayout {
  int o_gc, o_gv, o_tau, o_pt, o_vt, o_L, o_invd, o_rhs, o_z, o_ct, o_Y, o_lam, o_u, o_lim, o_hist, o_sat;   // persistent
  int o_h, o_b, o_pose;                                                                  // union A
  int o_G;                                                                               // union B
  int words;
};

__host__ __device__ constexpr WsLayout make_ws_layout(Dims d, int npairs = 0) {
  WsLayout L{};
  const int nvp = round_up_c(max_c(d.nv, 1), 4), nqp = round_up_c(max_c(d.nq, 1), 4), nbp = d.nb | 1, dlp = (d.maxdd + 1) | 1;
  int o = 0;
  L.o_gc = o; o += nqp;
  L.o_gv = o; o += nvp;
  L.o_tau = o; o += nvp;
  L.o_pt = o; o += nqp;
  L.o_vt = o; o += nvp;
  L.o_L = o; o += round_up_c(max_c(1, d.nv) * dlp, 4);            // compact rows: [dof][ancestor depth]
  L.o_invd = o; o += nvp;
  L.o_rhs = o; o += nvp;
  L.o_z = o; o += nvp;
  L.o_ct = o; o += KMAX * CT_WORDS;
  L.o_Y = o; o += round_up_c((d.maxdd + 1) * CP, 4);              // [ancestor depth][contact row]
  L.o_lam = o; o += 32;
  L.o_u = o; o += CB_WORDS * KMAX;                                // per contact: G_ii (6), friction, its inverse (6): contact_solver.cuh
  L.o_lim = o; o += 4 * LMAX;                                     // joint-limit rows: dof, sign, violation
  L.o_sat = o; o += nvp;                                          // dof driven at its actuator effort limit in this sub-step (stage C -> E)
  L.o_hist = o; o += HIST_WORDS;                                  // Anderson acceleration: u0, x, g, f, dG, dF (one value per constraint row each)
  if (o - L.o_Y < HL_CAP * HL_WORDS) o = L.o_Y + HL_CAP * HL_WORDS;   // stage B keeps its hit list in [o_Y, here): dead until stage C
  if (npairs > 0 && o - L.o_Y < (HL_CAP + npairs) * HL_WORDS) o = L.o_Y + (HL_CAP + npairs) * HL_WORDS;   // ... and one row per self-collision pair
  // union: {h, b, poses} (stages A-C) overlaid by G (stages C-D)
  int ua = 0;
  L.o_h = o + ua; ua += nvp;
  L.o_b = o + ua; ua += nvp;
  L.o_pose = o + ua; ua += round_up_c(15 * nbp, 4);
  L.o_G = o;
  const int ub = round_up_c(RMAX * GP, 4);
  o += max_c(ua, ub);
  if (npairs > 0) o += self_y_words(d.maxdd);                     // the self contacts' second column block: the last self_y_words of the workspace
  L.words = round_up_c(o, 32);
  return L;
}

struct TerrainDesc {
  int type;            // 0 none, 1 Ground, 2 HeightMap
  float ground_z;
  int xs, ys;
  float x0, y0, dx, dy, xmax, ymax;   // grid origin, pitch, index bounds (xs-1, ys-1 as float)
  const float* h;
  const int* env_map;  // terrain atlas: height-map index of every environment (null: one shared map)
  int map_words;       // xs * ys
  float hmax;          // largest height of the map(s): a candidate whose lowest point is above it cannot touch (stage B cull)
  float inv_dx, inv_dy; // reciprocal pitch (sphere groups: cell of a point without an IEEE division)
};

// RaisimGym ANYmal locomotion task (SURVEY.md 8f N1; [RECALL] raisimGymTorch envs/rsg_anymal/Environment.hpp): constants of
// ENVIRONMENT::step() / isTerminalState() / reset(), all device pointers
struct GymConfig {
  const float* gc_init;      // [nq]
  const float* gv_init;      // [nv]
  const float* action_mean;  // [nq - 7]
  const float* action_std;   // [nq - 7]
  uint32_t foot_mask;        // bit b set: contacts on body b do not terminate the episode
  float torque_coeff, forward_vel_coeff, terminal_reward;
};

// learned actuator network (rsb_batch_set_actuator_network: an MLP, or rsb_batch_set_actuator_lstm: an LSTM), read by stage C;
// params == null: no network, or a launch that applies no PD laws (force mode)
constexpr int AN_MAX_DOFS = 64;          // >= nv of every model (32 bodies)
struct ActNetDesc {
  // MLP: per hidden layer: weights transposed [n_in][W] (lanes read consecutive words), bias [W]; output weights [W], bias.
  // LSTM: per layer: weights [n_in + W][4][W] (input then recurrent columns, gates i f g o), summed bias [4][W]; output weights [W], bias
  const float* params;
  // MLP: [num_envs][n][2][H - 1]: errors then velocities of the last H - 1 sub-steps, most recent first.
  // LSTM: [num_envs][n][L][2][W]: h then c of every layer
  float* hist;
  unsigned long long mask;   // bit i: dof i is listed
  int lstm;                  // 0: the MLP, 1: the LSTM (H unused)
  int n, H, L, W;
  int words;                 // hist words of one environment
  uint8_t dof[AN_MAX_DOFS];
};

// StepArgs::phase_mask bits of the launches that stop early (the host's getters and integrate1())
constexpr int PHASE_NO_UPDATE = 1;    // stop after stage B (integrate1: no state update)
constexpr int PHASE_KINEMATICS = 4;   // stop after stage A (stage A + the getters' buffers; the contact records of the last integrate() stay)

struct StepArgs {
  int num_envs, substeps;
  int gc_stride, gv_stride, pt_stride, vt_stride;   // vt_stride likewise for vtarget; pt_stride: row stride of ptarget (own padded buffer or a bound caller buffer)
  float *gc, *gv;
  const float *tau, *ptarget, *vtarget;
  int use_pd;
  float* pt_store;     // when the targets are read in place from a caller buffer (zero-copy, possibly pinned host memory):
  float* vt_store;     // keep a copy in the batch's own rows, so that setPdTarget semantics (targets persist) hold
  rsb_params prm;
  TerrainDesc ter;
  WsLayout ws;
  int blob_words;
  const uint32_t* blob;
  // outputs
  int* ncontacts;
  rsb_contact* contacts;
  int* contact_pt;     // [N][KMAX]
  int* iters;          // [N]
  int* diverged;       // [N] 1 when the stored state holds a non-finite value (caller resets those environments)
  float* resid;        // [N] largest impulse update of the last Gauss-Seidel sweep (< threshold: the solve converged)
  int* solver_status;  // [N] RSB_SOLVER_* of the last sub-step's solve
  float* tau_applied;  // [N][gv_stride] generalized force actually applied in the last sub-step (getGeneralizedForce)
  // contact forces per body over the whole launch (rsb_batch_set_contact_bodies); cf_force null = none listed or the launch does not
  // advance the state.  The list sits in the kernel parameters: lane s reads its body with one constant-bank load at its own index
  float* cf_force;     // [N][cf_n][3] mean world force on body cf_body[s]: the row itself is the accumulator over the sub-steps
  int* cf_steps;       // [N][cf_n] sub-steps in which the body had a contact in the list
  int cf_n;
  uint8_t cf_body[RSB_MAX_CONTACT_BODIES];
  // IMU readings over the whole launch (rsb_batch_set_imus); imu_lin null = no sensors set or the launch does not advance the state.
  // Sensor k hangs on body imu_body[k] at imu_pos[k] with orientation imu_rot[k] (row-major), both in the body frame
  float* imu_lin;      // [N][imu_n][3] mean specific force in the sensor frame: the row itself is the accumulator over the sub-steps
  float* imu_ang;      // [N][imu_n][3] mean angular rate in the sensor frame, likewise
  int imu_n;
  uint8_t imu_body[RSB_MAX_IMUS];
  float imu_pos[RSB_MAX_IMUS][3];
  float imu_rot[RSB_MAX_IMUS][9];
  float *dbg_M, *dbg_h, *dbg_R, *dbg_p;   // optional (integrate1 / getters)
  float* obs;          // optional [N][ob_dim]: RaisimGym observation row of the final state, written by this kernel
  int ob_dim;
  const float* ext;    // optional [num_envs][EXT_WORDS] external wrench rows (body, F world, T world, point in body frame); null = none
  const float* body_inertia;   // optional [num_envs][nb][BI_WORDS] inertial rows (rsb_batch_set_body_inertia) read by stage A in place
                               // of the blob's BF_MASS / BF_COM / BF_INERTIA; null = the model's values for every environment
  const float* contact_friction;   // optional [num_envs][ncoll] terrain friction rows (rsb_batch_set_contact_friction) read by stage C;
                                   // an entry >= 0 replaces the batch-level value of the collision body's terrain contacts; null = none
  const float* actuator;   // optional [num_envs][3][nv] kp | kd | effort limit rows (rsb_batch_set_actuator_params) read by stages C and E;
                           // an entry >= 0 replaces the blob's value of that dof; null = none
  unsigned* prof;      // optional [num_envs][4 sub-steps][8] SM-clock stamps at the stage boundaries (tools/balance_probe.py)
  unsigned* prof_a;    // optional [num_envs][4 sub-steps][4] SM-clock stamps inside stage A: after the FK walk, the per-body terms, the
                       // subtree sums, the M columns (tools/stage_probe.py)
  // fused observation all-gather (SURVEY 8e): every rank's kernel stores its observation rows straight into every peer's
  // [world * num_envs][ob_dim] buffer over NVLink (peer memory mapped into this process), then signals one counter per peer
  float* peer_obs[MAX_PEERS];      // peer p's gathered-rows buffer of this step (null = not in use)
  unsigned* peer_flag[MAX_PEERS];  // peer p's arrival counters [world]: += 1 per finished CTA of this rank
  int peer_world, peer_rank;
  unsigned peer_expected;          // arrival count every rank's counter reaches when its rows of THIS step have landed (steps so far x CTAs)
  unsigned* peer_done;             // CTAs of this launch that finished: the last one waits for the peers (set whenever peer_world > 0)
  // RaisimGym task fused into the step (rsb_batch_gym_step): the launch turns the action rows into PD targets before the first
  // sub-step and, after the last one, computes reward and termination, resets the terminated environments and writes the
  // observation rows of the (possibly reset) state -- VectorizedEnvironment::step() + observe() in ONE launch
  const float* gym_action;         // [num_envs][nq - 7] action rows (device memory or mapped pinned host memory); null = no task
  GymConfig gym;
  float* gym_reward;               // [num_envs]
  unsigned char* gym_done;         // [num_envs]
  int phase_mask;      // 0 (a full step) or PHASE_NO_UPDATE, optionally with PHASE_KINEMATICS
  int substep_barrier; // non-zero: re-align the CTA's warps of one round at every sub-step
  int pair_stage_a;    // 1: quadruped instance, CTAs that keep the sub-step barrier: one warp runs stage A of two environments
  ActNetDesc an;       // learned actuator network (stages C and E, the gym epilogue); an.params null = none
  // actuation delay (rsb_batch_set_actuation_delay), read by the DL instances only; null = none, or a launch that does not advance the
  // state.  delay_state [num_envs][2]: the delay d and the advancing sub-steps t since the history was emptied (actuation_delay);
  // delay_ring [num_envs][DELAY_SLOTS][3][nv - nbase]: the command ring
  int* delay_state;
  float* delay_ring;
};

// ------------------------------------------------------------------ small device math ----------
struct f3 { float x, y, z; };
__device__ __forceinline__ f3 mk(float x, float y, float z) { f3 r; r.x = x; r.y = y; r.z = z; return r; }
__device__ __forceinline__ f3 operator+(f3 a, f3 b) { return mk(a.x + b.x, a.y + b.y, a.z + b.z); }
__device__ __forceinline__ f3 operator-(f3 a, f3 b) { return mk(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ f3 operator*(float s, f3 a) { return mk(s * a.x, s * a.y, s * a.z); }
__device__ __forceinline__ float dot(f3 a, f3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ f3 cross(f3 a, f3 b) { return mk(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }
__device__ __forceinline__ f3 mulR(const float* R, f3 v) {
  return mk(R[0] * v.x + R[1] * v.y + R[2] * v.z, R[3] * v.x + R[4] * v.y + R[5] * v.z, R[6] * v.x + R[7] * v.y + R[8] * v.z);
}
__device__ __forceinline__ f3 mulRt(const float* R, f3 v) {
  return mk(R[0] * v.x + R[3] * v.y + R[6] * v.z, R[1] * v.x + R[4] * v.y + R[7] * v.z, R[2] * v.x + R[5] * v.y + R[8] * v.z);
}
__device__ __forceinline__ void matmul3(const float* A, const float* B, float* C) {
#pragma unroll
  for (int i = 0; i < 3; i++)
#pragma unroll
    for (int j = 0; j < 3; j++) C[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
}
__device__ __forceinline__ f3 shfl3(f3 v, int src) {
  return mk(__shfl_sync(FULL, v.x, src), __shfl_sync(FULL, v.y, src), __shfl_sync(FULL, v.z, src));
}

// ------------------------------------------------------------------ TMA bulk copy + mbarrier ---
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n" : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  // bounded spin: a TMA that never lands must trap, not hang the GPU
  for (uint32_t spin = 0; !mbar_try_wait(bar, parity); spin++)
    if (spin > (1u << 26)) __trap();
}
__device__ __forceinline__ void cp_async4(float* dst_smem, const float* src_gmem) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(dst_smem)), "l"(src_gmem) : "memory");
}
__device__ __forceinline__ void tma_bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// Observation row of a floating-base robot, written by rsb_observe_kernel and fused into rsb_step_kernel (one warp per row; q, v: the
// state rows): [z, R^T e_z, q_j, R^T v, R^T w, qdot_j].  Explicit round-to-nearest intrinsics keep the rotation part independent of
// what the compiler contracts around it.
// c = column `col` (0..2) of the base rotation matrix of the unit quaternion (qw, qx, qy, qz).
__device__ __forceinline__ void obs_rot_column(float qw, float qx, float qy, float qz, int col, float& c0, float& c1, float& c2) {
  const float xx = __fmul_rn(qx, qx), yy = __fmul_rn(qy, qy), zz = __fmul_rn(qz, qz);
  const float xy = __fmul_rn(qx, qy), xz = __fmul_rn(qx, qz), yz = __fmul_rn(qy, qz);
  const float wx = __fmul_rn(qw, qx), wy = __fmul_rn(qw, qy), wz = __fmul_rn(qw, qz);
  const float r00 = __fsub_rn(1.f, __fmul_rn(2.f, __fadd_rn(yy, zz))), r01 = __fmul_rn(2.f, __fsub_rn(xy, wz)), r02 = __fmul_rn(2.f, __fadd_rn(xz, wy));
  const float r10 = __fmul_rn(2.f, __fadd_rn(xy, wz)), r11 = __fsub_rn(1.f, __fmul_rn(2.f, __fadd_rn(xx, zz))), r12 = __fmul_rn(2.f, __fsub_rn(yz, wx));
  const float r20 = __fmul_rn(2.f, __fsub_rn(xz, wy)), r21 = __fmul_rn(2.f, __fadd_rn(yz, wx)), r22 = __fsub_rn(1.f, __fmul_rn(2.f, __fadd_rn(xx, yy)));
  c0 = col == 0 ? r00 : col == 1 ? r01 : r02;
  c1 = col == 0 ? r10 : col == 1 ? r11 : r12;
  c2 = col == 0 ? r20 : col == 1 ? r21 : r22;
}
__device__ __forceinline__ float obs_dot3(float c0, float c1, float c2, float x, float y, float z) {
  return __fmaf_rn(c2, z, __fmaf_rn(c1, y, __fmul_rn(c0, x)));
}
__device__ __forceinline__ float* write_obs_row(float* obs, const int& ob_dim, int env, const float* q, const float* v, int nq, int lane) {
  float qw = q[3], qx = q[4], qy = q[5], qz = q[6];
  const float inv = 1.0f / sqrtf(qw * qw + qx * qx + qy * qy + qz * qz);
  qw *= inv; qx *= inv; qy *= inv; qz *= inv;
  float* o = obs + (size_t)env * ob_dim;   // after the quaternion loads: the other order costs the 72-register instances spill reloads
  const int nj = nq - 7;
  if (lane == 0) o[0] = q[2];
  if (lane < 3) {
    float c0, c1, c2;
    obs_rot_column(qw, qx, qy, qz, lane, c0, c1, c2);
    o[1 + lane] = c2;
    o[4 + nj + lane] = obs_dot3(c0, c1, c2, v[0], v[1], v[2]);
    o[7 + nj + lane] = obs_dot3(c0, c1, c2, v[3], v[4], v[5]);
  }
#pragma unroll 1
  for (int i = lane; i < nj; i += 32) { o[4 + i] = q[7 + i]; o[10 + nj + i] = v[6 + i]; }
  return o;
}

// ------------------------------------------------------------------ terrain --------------------
__device__ __forceinline__ bool terrain_query(const TerrainDesc& t, int hm_offset, f3 P, float& dist, f3& n, int& pair) {
  if (t.type == 1) { dist = P.z - t.ground_z; n = mk(0.f, 0.f, 1.f); pair = 0; return true; }
  if (t.type != 2) return false;
  float gx = (P.x - t.x0) / t.dx, gy = (P.y - t.y0) / t.dy;
  if (!(gx >= 0.f) || !(gy >= 0.f) || !(gx < t.xmax) || !(gy < t.ymax)) return false;
  int ix = (int)gx, iy = (int)gy;
  float fx = gx - (float)ix, fy = gy - (float)iy;
  const float* H = t.h + hm_offset + iy * t.xs + ix;
  float h00 = __ldg(H), h10 = __ldg(H + 1), h01 = __ldg(H + t.xs), h11 = __ldg(H + t.xs + 1);
  float sx, sy; int tri;
  if (fx >= fy) { sx = h10 - h00; sy = h11 - h10; tri = 0; }
  else { sx = h11 - h01; sy = h01 - h00; tri = 1; }
  float zt = h00 + sx * fx + sy * fy;
  float nx = -sx / t.dx, ny = -sy / t.dy;
  float inv = 1.0f / sqrtf(nx * nx + ny * ny + 1.0f);
  n = mk(nx * inv, ny * inv, inv);
  dist = (P.z - zt) * inv;
  pair = 2 * (iy * (t.xs - 1) + ix) + tri;
  return true;
}

#include "narrow_phase.cuh"

// getters of integrate1(): full symmetric M rebuilt from the compact rows, h, body poses (cold path)
__device__ __noinline__ void write_debug(const StepArgs& args, int env, int lane, int nv, int nb, int nvp, int DLP, const float* s_L,
                                         const float* s_h, const int* ddepth, const int* danc, bool bvalid, const float* s_pose, int nbp) {
  float* gM = args.dbg_M + (size_t)env * nv * nv;
  for (int i = lane; i < nv * nv; i += 32) {
    int r = i / nv, c = i % nv;
    if (r < c) { int t = r; r = c; c = t; }
    int dc = ddepth[c];
    gM[i] = (dc <= ddepth[r] && danc[dc * nvp + r] == c) ? s_L[r * DLP + dc] : 0.f;
  }
  float* gh = args.dbg_h + (size_t)env * nv;
  for (int i = lane; i < nv; i += 32) gh[i] = s_h[i];
  if (bvalid) {
    float* gR = args.dbg_R + ((size_t)env * nb + lane) * 9;
    float* gp = args.dbg_p + ((size_t)env * nb + lane) * 3;
    for (int k = 0; k < 9; k++) gR[k] = s_pose[(PF_R + k) * nbp + lane];   // poses were published to shared memory by stage A
    for (int k = 0; k < 3; k++) gp[k] = s_pose[(PF_P + k) * nbp + lane];
  }
}


// 1/sqrt(x) and sqrt(x) for x > 0: MUFU.RSQ + one Newton step (relative error < 2e-7, the level of a float32 rounding);
// the IEEE sqrtf / division pair of the generic path costs ~27 instructions per pivot.
__device__ __forceinline__ float rsqrt_nr(float x) {
  float r;
  asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r * (1.5f - 0.5f * x * r * r);
}

// IMU sensor `lane` (rsb_batch_set_imus, lane < imu_n) at the end of stage E of sub-step `sub`, before the state update: s_gc, s_gv hold
// the sub-step's start state (q_s, v_s) and s_rhs the velocity change dv of stage E.  The lane walks its body's chain from the root with
// stage A's classical-acceleration recursion plus the generalized acceleration qdd = dv / dt, and carries the angular velocity of
// v_s + dv (the sum stage E stores) beside it.  It does not use stage A's poses: from stage C on the Delassus matrix G overlays them
// whenever there is a constraint row.  The accumulator is the environment's own output row, which only this lane touches: stored at the
// first sub-step, read back and added to at the later ones, scaled by 1 / substeps at the last.
__device__ __forceinline__ void imu_substep(const StepArgs& args, int env, int sub, int lane, const float* bodyf, const int* bodyi,
                                            const int* anc, int nbp, int floating, bool jrot_identity, const float* s_gc,
                                            const float* s_gv, const float* s_rhs) {
  float* lo = args.imu_lin + ((size_t)env * args.imu_n + lane) * 3;
  float* ao = args.imu_ang + ((size_t)env * args.imu_n + lane) * 3;
  f3 acc_f = mk(0.f, 0.f, 0.f), acc_w = mk(0.f, 0.f, 0.f);
  if (sub > 0) { acc_f = mk(lo[0], lo[1], lo[2]); acc_w = mk(ao[0], ao[1], ao[2]); }   // issued before the walk, which hides the L2 round trip
  const float idt = 1.0f / args.prm.dt;
  float R[9];
  f3 w, w1, wd, vd;      // angular velocity at v_s and at v_s + dv, angular and classical linear acceleration of the body origin
  if (floating) {
    float qw = s_gc[3], qx = s_gc[4], qy = s_gc[5], qz = s_gc[6];
    const float inv = 1.0f / sqrtf(qw * qw + qx * qx + qy * qy + qz * qz);
    qw *= inv; qx *= inv; qy *= inv; qz *= inv;
    R[0] = 1.f - 2.f * (qy * qy + qz * qz); R[1] = 2.f * (qx * qy - qw * qz); R[2] = 2.f * (qx * qz + qw * qy);
    R[3] = 2.f * (qx * qy + qw * qz); R[4] = 1.f - 2.f * (qx * qx + qz * qz); R[5] = 2.f * (qy * qz - qw * qx);
    R[6] = 2.f * (qx * qz - qw * qy); R[7] = 2.f * (qy * qz + qw * qx); R[8] = 1.f - 2.f * (qx * qx + qy * qy);
    w = mk(s_gv[3], s_gv[4], s_gv[5]);
    w1 = mk(s_gv[3] + s_rhs[3], s_gv[4] + s_rhs[4], s_gv[5] + s_rhs[5]);
    wd = idt * mk(s_rhs[3], s_rhs[4], s_rhs[5]);
    vd = idt * mk(s_rhs[0], s_rhs[1], s_rhs[2]);
  } else {
#pragma unroll
    for (int k = 0; k < 9; k++) R[k] = bodyf[(BF_JROT + k) * nbp];
    w = w1 = wd = vd = mk(0.f, 0.f, 0.f);
  }
  vd = vd - mk(args.prm.gravity[0], args.prm.gravity[1], args.prm.gravity[2]);
  const int b = args.imu_body[lane];
  const int depth = bodyi[BF_DEPTH * nbp + b];
#pragma unroll 1
  for (int d = 1; d <= depth; d++) {
    const int j = anc[(d - 1) * nbp + b];
    const f3 jp = mk(bodyf[(BF_JPOS + 0) * nbp + j], bodyf[(BF_JPOS + 1) * nbp + j], bodyf[(BF_JPOS + 2) * nbp + j]);
    const f3 al = mk(bodyf[(BF_AXIS + 0) * nbp + j], bodyf[(BF_AXIS + 1) * nbp + j], bodyf[(BF_AXIS + 2) * nbp + j]);
    float Rj[9];
    if (jrot_identity) {
#pragma unroll
      for (int k = 0; k < 9; k++) Rj[k] = R[k];
    } else {
      float Jr[9];
#pragma unroll
      for (int k = 0; k < 9; k++) Jr[k] = bodyf[(BF_JROT + k) * nbp + j];
      matmul3(R, Jr, Rj);
    }
    const f3 aj = mulR(Rj, al);
    const int vi = bodyi[BF_VIDX * nbp + j];
    const float q = s_gc[bodyi[BF_QIDX * nbp + j]], qd = s_gv[vi], dq = s_rhs[vi];
    const bool rev = bodyi[BF_JTYPE * nbp + j] == 1;
    f3 r = mulR(R, jp);
    if (!rev) r = r + q * aj;
    vd = vd + cross(wd, r) + cross(w, cross(w, r));
    const f3 qa = qd * aj, qdda = (dq * idt) * aj;
    if (rev) {
      float sq, cq;
      sincosf(q, &sq, &cq);
      const float t = 1.f - cq;
      const float Rq[9] = {t * al.x * al.x + cq, t * al.x * al.y - sq * al.z, t * al.x * al.z + sq * al.y,
                           t * al.x * al.y + sq * al.z, t * al.y * al.y + cq, t * al.y * al.z - sq * al.x,
                           t * al.x * al.z - sq * al.y, t * al.y * al.z + sq * al.x, t * al.z * al.z + cq};
      matmul3(Rj, Rq, R);
      wd = wd + cross(w, qa) + qdda;
      w = w + qa;
      w1 = w1 + (qd + dq) * aj;
    } else {
#pragma unroll
      for (int k = 0; k < 9; k++) R[k] = Rj[k];
      vd = vd + 2.f * cross(w, qa) + qdda;
    }
  }
  // the sensor point: a = a_origin + wd x r + w x (w x r), r = R pos; both readings turned into the sensor frame, (R rot)^T = rot^T R^T
  const f3 rs = mulR(R, mk(args.imu_pos[lane][0], args.imu_pos[lane][1], args.imu_pos[lane][2]));
  const f3 fb = mulRt(R, vd + cross(wd, rs) + cross(w, cross(w, rs))), wb = mulRt(R, w1);
  const float* Ro = args.imu_rot[lane];
  f3 f = acc_f + mulRt(Ro, fb), g = acc_w + mulRt(Ro, wb);
  if (sub == args.substeps - 1) { const float s = 1.0f / (float)args.substeps; f = s * f; g = s * g; }
  lo[0] = f.x; lo[1] = f.y; lo[2] = f.z;
  ao[0] = g.x; ao[1] = g.y; ao[2] = g.z;
}

// ---- compile-time topology: floating base + four serial chains of three joints (every 12-joint quadruped) -------------
// dof 0..5 = base, dof 6 + 3 leg + j = joint j of that leg (j = 0 hip abduction, 1 hip flexion, 2 knee); body b >= 1 carries
// dof 5 + b.  The compact row of dof (leg, j) holds its 6 base couplings at t = 0..5 and its chain entries at t = 6..6+j.
// Lane (leg = lane >> 3, t = lane & 7) keeps column t of its leg's three rows in registers: the leg blocks factorise with
// four shuffles per level and no table look-ups (the generic path walks entry lists, subtree ranges and level tables).
constexpr int QDLP = 9;   // compact row stride of the quadruped (maxdd + 1 = 9)
struct QuadLeg { float k, h, a, i8, i7, i6, k7, k6, h6; };   // column t of the knee / hip-flexion / hip-abduction rows; inverse pivots; couplings

__device__ __forceinline__ QuadLeg quad_factor_legs(float* s_L, float* s_invd, int lane) {
  const int leg = lane >> 3, t = lane & 7, l0 = lane & 24;
  const int rA = 6 + 3 * leg, rH = rA + 1, rK = rA + 2;
  QuadLeg q;
  q.k = s_L[rK * QDLP + t];
  q.h = s_L[rH * QDLP + t];
  q.a = t < 7 ? s_L[rA * QDLP + t] : 0.f;
  const float k8 = s_L[rK * QDLP + 8];
  q.i8 = rsqrt_nr(k8);
  q.k *= q.i8;                                          // level 8: the knee row has no descendants
  q.k7 = __shfl_sync(FULL, q.k, l0 + 7);
  q.h -= q.k7 * q.k;                                    // level 7: hip flexion, descendant = knee
  const float h7 = __shfl_sync(FULL, q.h, l0 + 7);
  q.i7 = rsqrt_nr(h7);
  q.h = (t == 7) ? h7 * q.i7 : q.h * q.i7;
  q.k6 = __shfl_sync(FULL, q.k, l0 + 6); q.h6 = __shfl_sync(FULL, q.h, l0 + 6);
  q.a -= q.k6 * q.k + q.h6 * q.h;                       // level 6: hip abduction, descendants = flexion, knee
  const float a6 = __shfl_sync(FULL, q.a, l0 + 6);
  q.i6 = rsqrt_nr(a6);
  q.a = (t == 6) ? a6 * q.i6 : q.a * q.i6;
  __syncwarp();   // every lane of the leg has read the knee pivot k8 above; lane t == 0 overwrites it below (racecheck: read / write without a barrier)
  s_L[rK * QDLP + t] = q.k; s_L[rH * QDLP + t] = q.h;
  if (t < 7) s_L[rA * QDLP + t] = q.a;
  if (t == 0) { s_L[rK * QDLP + 8] = k8 * q.i8; s_invd[rK] = q.i8; s_invd[rH] = q.i7; s_invd[rA] = q.i6; }
  return q;
}


// ------------------------------------------------------------------ stage B: narrow phase ------
// lane = contact candidate (SLOTS x 32 of them): Ground / HeightMap queries, ballot-compacted contact list in candidate order, the
// RSB_KMAX deepest kept.  Returns the number of contacts written to s_ct.
// Stage B writes every penetrating candidate into a per-warp hit list in shared memory (rows of HL_WORDS words, candidate order), keeps
// the KMAX deepest and emits the contact records.  Nothing per candidate survives in registers across the candidate slots, so the
// stage needs no register arrays (which ptxas had placed in local memory).  It is inlined into the kernel (an out-of-line stage B is
// one of the dead ends of DESIGN §6); the segment / box shape routines it calls stay out of line.

// ---- self-collision pairs (generic instance only): the narrow phase of one pair, the oracle's SelfPair routine in float32
// (oracle/self_collision.hpp self_pair_geometry: same closest-point rule for parallel and degenerate segments, same face rule inside a box)
__device__ __forceinline__ void self_closest_segments(f3 p1, f3 d1, f3 p2, f3 d2, float& s, float& t) {
  const f3 r = p1 - p2;
  const float a = dot(d1, d1), e = dot(d2, d2), f = dot(d2, r);
  if (a == 0.f && e == 0.f) { s = t = 0.f; return; }
  if (a == 0.f) { s = 0.f; t = fminf(fmaxf(f / e, 0.f), 1.f); return; }
  const float c = dot(d1, r);
  if (e == 0.f) { t = 0.f; s = fminf(fmaxf(-c / a, 0.f), 1.f); return; }
  const float b = dot(d1, d2), den = a * e - b * b;
  s = den > 1e-6f * a * e ? fminf(fmaxf((b * f - c * e) / den, 0.f), 1.f) : 0.f;
  t = (b * s + f) / e;
  if (t < 0.f) { t = 0.f; s = fminf(fmaxf(-c / a, 0.f), 1.f); }
  else if (t > 1.f) { t = 1.f; s = fminf(fmaxf((b - c) / a, 0.f), 1.f); }
}
// pair row pr (PairField), body poses of stage A: false when the shapes do not overlap; else depth, normal (second body -> first), position
__device__ __noinline__ bool self_pair_contact(const float* pr, const float* s_pose, int nbp, float& depth, f3& n, f3& pos) {
  const int* pri = reinterpret_cast<const int*>(pr);
  const int bA = pri[PR_BA], bB = pri[PR_BB];
  float RA[9], RB[9];
#pragma unroll
  for (int q = 0; q < 9; q++) { RA[q] = s_pose[(PF_R + q) * nbp + bA]; RB[q] = s_pose[(PF_R + q) * nbp + bB]; }
  const f3 pA = mk(s_pose[(PF_P + 0) * nbp + bA], s_pose[(PF_P + 1) * nbp + bA], s_pose[(PF_P + 2) * nbp + bA]);
  const f3 pB = mk(s_pose[(PF_P + 0) * nbp + bB], s_pose[(PF_P + 1) * nbp + bB], s_pose[(PF_P + 2) * nbp + bB]);
  const float ra = pr[PR_RA], rb = pr[PR_RB];
  f3 ng, SA, SB;
  if (pri[PR_KIND] == 0) {
    const f3 A0 = pA + mulR(RA, mk(pr[PR_A0], pr[PR_A0 + 1], pr[PR_A0 + 2])), A1 = pA + mulR(RA, mk(pr[PR_A1], pr[PR_A1 + 1], pr[PR_A1 + 2]));
    const f3 B0 = pB + mulR(RB, mk(pr[PR_B0], pr[PR_B0 + 1], pr[PR_B0 + 2])), B1 = pB + mulR(RB, mk(pr[PR_B1], pr[PR_B1 + 1], pr[PR_B1 + 2]));
    float s, t;
    self_closest_segments(A0, A1 - A0, B0, B1 - B0, s, t);
    const f3 QA = A0 + s * (A1 - A0), QB = B0 + t * (B1 - B0), v = QA - QB;
    const float dist = sqrtf(dot(v, v));
    depth = ra + rb - dist;
    if (!(depth > 0.f)) return false;
    ng = dist > 1e-9f ? (1.0f / dist) * v : mk(0.f, 0.f, 1.f);      // coincident centres / axes: +z, a fixed rule
    SA = QA - ra * ng; SB = QB + rb * ng;
  } else {
    const f3 C = pA + mulR(RA, mk(pr[PR_A0], pr[PR_A0 + 1], pr[PR_A0 + 2])), cb = pB + mulR(RB, mk(pr[PR_B0], pr[PR_B0 + 1], pr[PR_B0 + 2]));
    float R[9];
    matmul3(RB, pr + PR_BR, R);
    const f3 q = mulRt(R, C - cb), h = mk(pr[PR_B1], pr[PR_B1 + 1], pr[PR_B1 + 2]);
    const f3 cl = mk(fminf(fmaxf(q.x, -h.x), h.x), fminf(fmaxf(q.y, -h.y), h.y), fminf(fmaxf(q.z, -h.z), h.z));
    f3 nl, bp;
    if (q.x != cl.x || q.y != cl.y || q.z != cl.z) {                  // centre outside the box: the clamped point is the closest one
      const f3 d = q - cl;
      const float dist = sqrtf(dot(d, d));
      depth = ra - dist;
      if (!(depth > 0.f)) return false;
      nl = (1.0f / dist) * d; bp = cl;
    } else {                                                           // inside: out through the nearest face, ties to the lowest axis
      const float px = h.x - fabsf(q.x), py = h.y - fabsf(q.y), pz = h.z - fabsf(q.z);
      bp = q;
      if (px <= py && px <= pz) { depth = ra + px; nl = mk(q.x >= 0.f ? 1.f : -1.f, 0.f, 0.f); bp.x = nl.x * h.x; }
      else if (py <= pz) { depth = ra + py; nl = mk(0.f, q.y >= 0.f ? 1.f : -1.f, 0.f); bp.y = nl.y * h.y; }
      else { depth = ra + pz; nl = mk(0.f, 0.f, q.z >= 0.f ? 1.f : -1.f); bp.z = nl.z * h.z; }
    }
    ng = mulR(R, nl);
    SA = C - ra * ng; SB = cb + mulR(R, bp);
  }
  n = pri[PR_FLIP] ? -1.f * ng : ng;
  pos = 0.5f * (SA + SB);
  return true;
}

// ter: the kernel parameter itself (constant bank); ter_s: its shared-memory copy, for the out-of-line shape routines
// SELF: the generic instance, which also runs the self-collision pairs of the blob (lane = pair, after the terrain candidates)
template <int SLOTS, bool SELF = false>
__device__ __forceinline__ int stage_b_narrow_phase(const TerrainDesc& ter, const TerrainDesc& ter_s, const uint32_t* blob_s, const float* s_pose, float* s_ct, float* s_list,
                                              int env, int lane, int nbp, unsigned* prof) {
  const BlobHeader& H = *reinterpret_cast<const BlobHeader*>(blob_s);
  const float* ptsf = reinterpret_cast<const float*>(blob_s + H.off_pts);
  const int* ptsi = reinterpret_cast<const int*>(blob_s + H.off_pts);
  const int hm_offset = ter.env_map ? __ldg(ter.env_map + env) * ter.map_words : 0;   // terrain atlas
  const bool on_hm = ter.type == 2;
  // nothing whose lowest point is above the highest point of the terrain (the plane itself for a Ground) can touch it
  const float zcull = on_hm ? ter.hmax : ter.ground_z;
  const unsigned lt = (1u << lane) - 1u;
  int cnt = 0;
#pragma unroll 1
  for (int s = 0; s < SLOTS; s++) {
    const int k = lane + 32 * s;
    // ---- cull on the height alone: every candidate carries a bounding sphere (rows 11-14: centre in the body frame, radius; a body
    // welded to the world has radius -3e38 and never passes); third row of the body rotation, one dot product.  An upright robot
    // keeps its feet.
    bool alive = false;
    int pb = 0;
    if (k < H.npts && ter.type != 0) {
      pb = ptsi[0 * H.nptp + k];
      const float zc = s_pose[(PF_P + 2) * nbp + pb] + s_pose[(PF_R + 6) * nbp + pb] * ptsf[11 * H.nptp + k] + s_pose[(PF_R + 7) * nbp + pb] * ptsf[12 * H.nptp + k] +
                       s_pose[(PF_R + 8) * nbp + pb] * ptsf[13 * H.nptp + k];
      alive = zc - ptsf[14 * H.nptp + k] <= zcull;
    }
    if (!__any_sync(FULL, alive)) continue;
    bool hit = false, sph = false; float depth = 0.f; f3 n = mk(0, 0, 1), pos = mk(0, 0, 0); int pair = 0;
    if (alive) {
      const int ptype = ptsi[6 * H.nptp + k]; const float rad = ptsf[4 * H.nptp + k];
      const f3 pl = mk(ptsf[1 * H.nptp + k], ptsf[2 * H.nptp + k], ptsf[3 * H.nptp + k]);
      float Rb[9];
#pragma unroll
      for (int q = 0; q < 9; q++) Rb[q] = s_pose[(PF_R + q) * nbp + pb];
      const f3 pb_pos = mk(s_pose[(PF_P + 0) * nbp + pb], s_pose[(PF_P + 1) * nbp + pb], s_pose[(PF_P + 2) * nbp + pb]);
      f3 P = pb_pos + mulR(Rb, pl);
      float prad = rad;
      bool as_point = ptype == 0 && !(on_hm && rad > 0.f), live = true;
      if (ptype == 3) {
        // cylinder cap: the lowest point of its rim circle (centre P, radius rad, axis a), the point of the circle furthest along -z
        f3 a = P - (pb_pos + mulR(Rb, mk(ptsf[7 * H.nptp + k], ptsf[8 * H.nptp + k], ptsf[9 * H.nptp + k])));
        a = (1.0f / sqrtf(dot(a, a))) * a;
        const f3 dd = mk(a.z * a.x, a.z * a.y, a.z * a.z - 1.f);
        const float dn = sqrtf(dot(dd, dd));
        if (dn > 1e-6f) { P = P + (rad / dn) * dd; prad = 0.f; as_point = true; }
        else live = false;                                  // cap parallel to the ground: the fixed rim samples carry it
      }
      if (on_hm && as_point && P.z - prad > ter.hmax) live = false;
      if (!live) {
      } else if (as_point) {
        // Ground plane, or a zero-radius point on a HeightMap (box corner, cylinder rim point): the triangle directly beneath
        float dist; f3 nn; int pr;
        if (terrain_query(ter, hm_offset, P, dist, nn, pr)) {
          const float d = prad - dist;
          if (d > 0.f) { hit = true; depth = d; pair = pr; n = nn; pos = P - prad * nn; }
        }
      } else if (on_hm) {
        // HeightMap: the shape against every triangle under its bounding box (narrow_phase.cuh)
        if (ptype == 0) {
          sph = true; pos = P; depth = rad;     // parked: eight lanes take it below
        } else {
          HmBest hb; hb.hit = false;
          if (ptype == 1) {
            const f3 P2 = pb_pos + mulR(Rb, mk(ptsf[7 * H.nptp + k], ptsf[8 * H.nptp + k], ptsf[9 * H.nptp + k]));
            if (fminf(P.z, P2.z) - rad <= ter.hmax) hb = segment_vs_heightmap(ter_s, hm_offset, P, P2, rad);
          } else {
            const float* cb = reinterpret_cast<const float*>(blob_s + H.off_coll) + COLL_WORDS * ptsi[10 * H.nptp + k];
            const f3 hsz = mk(cb[0], cb[1], cb[2]);
            float Rw[9];
            matmul3(Rb, cb + 6, Rw);
            const f3 cw = pb_pos + mulR(Rb, mk(cb[3], cb[4], cb[5]));
            const float ez = fabsf(Rw[6]) * hsz.x + fabsf(Rw[7]) * hsz.y + fabsf(Rw[8]) * hsz.z;
            if (cw.z - ez <= ter.hmax) hb = box_vs_heightmap(ter_s, hm_offset, cw, Rw, hsz);
          }
          if (hb.hit) { hit = true; depth = hb.depth; pair = hb.pair; n = hb.n; pos = hb.pos; }
        }
      }
    }
    // ---- this slot's direct hits go to the list at once (nothing of them stays in registers across the sphere groups).  The three
    // appends of this function stay written out: one shared helper raised the spill stores of the one-slot 14- and 28-warp instances
    // from 252-308 to 358-414 bytes (-Xptxas -v)
    {
      const unsigned hmask = __ballot_sync(FULL, hit);
      if (hit) {
        float* e = s_list + HL_WORDS * (cnt + __popc(hmask & lt));
        e[0] = depth; e[1] = n.x; e[2] = n.y; e[3] = n.z; e[4] = pos.x; e[5] = pos.y; e[6] = pos.z; e[7] = __int_as_float(pair); e[8] = __int_as_float(k);
      }
      cnt += __popc(hmask);
    }
    // ---- sphere candidates on a HeightMap: four at a time, eight lanes (= the eight triangles of the 2 x 2 cell block under it) each;
    // the lane whose triangle wins appends the contact itself (position = centre - r n)
    const unsigned sm = __ballot_sync(FULL, sph);
    if (sm != 0u) {
      const int nsph = __popc(sm);
#pragma unroll 1
      for (int base = 0; base < nsph; base += 4) {
        const int rk = base + (lane >> 3);
        const bool gvalid = rk < nsph;
        const int olane = gvalid ? __fns(sm, 0, rk + 1) : 0;
        const f3 C = shfl3(pos, olane); const float r = __shfl_sync(FULL, depth, olane);
        const SphereTri st = sphere_vs_heightmap_group(ter, hm_offset, C, r, gvalid, lane);
        const bool win = gvalid && st.winner == lane;
        const unsigned wmask = __ballot_sync(FULL, win);
        if (win) {
          float* e = s_list + HL_WORDS * (cnt + __popc(wmask & lt));
          e[0] = st.depth; e[1] = st.n.x; e[2] = st.n.y; e[3] = st.n.z; e[4] = C.x - r * st.n.x; e[5] = C.y - r * st.n.y; e[6] = C.z - r * st.n.z;
          e[7] = __int_as_float(st.pair); e[8] = __int_as_float(olane + 32 * s);
        }
        cnt += __popc(wmask);
      }
    }
  }
  if constexpr (SELF) {
    // self-collision pairs (with or without terrain): lane = pair j, candidate index npts + j, pair index -1 - second body.  Cull on the
    // bounding spheres of the two shapes; a warp without survivors skips the narrow phase.
    if (H.npairs > 0) {
      const float* pr = reinterpret_cast<const float*>(blob_s + H.off_pair) + PAIR_WORDS * min(lane, H.npairs - 1);
      const int* pri = reinterpret_cast<const int*>(pr);
      bool alive = false;
      if (lane < H.npairs) {
        const int bA = pri[PR_BA], bB = pri[PR_BB];
        float RA[9], RB[9];
#pragma unroll
        for (int q = 0; q < 9; q++) { RA[q] = s_pose[(PF_R + q) * nbp + bA]; RB[q] = s_pose[(PF_R + q) * nbp + bB]; }
        const f3 cA = mk(s_pose[(PF_P + 0) * nbp + bA], s_pose[(PF_P + 1) * nbp + bA], s_pose[(PF_P + 2) * nbp + bA]) +
                      mulR(RA, 0.5f * (mk(pr[PR_A0], pr[PR_A0 + 1], pr[PR_A0 + 2]) + mk(pr[PR_A1], pr[PR_A1 + 1], pr[PR_A1 + 2])));
        const f3 lB = pri[PR_KIND] == 0 ? 0.5f * (mk(pr[PR_B0], pr[PR_B0 + 1], pr[PR_B0 + 2]) + mk(pr[PR_B1], pr[PR_B1 + 1], pr[PR_B1 + 2]))
                                        : mk(pr[PR_B0], pr[PR_B0 + 1], pr[PR_B0 + 2]);
        const f3 cB = mk(s_pose[(PF_P + 0) * nbp + bB], s_pose[(PF_P + 1) * nbp + bB], s_pose[(PF_P + 2) * nbp + bB]) + mulR(RB, lB);
        const f3 dc = cA - cB;
        const float rr = pr[PR_CULL_A] + pr[PR_CULL_B];
        alive = dot(dc, dc) <= rr * rr;
      }
      if (__any_sync(FULL, alive)) {
        float depth = 0.f; f3 n = mk(0.f, 0.f, 1.f), pos = mk(0.f, 0.f, 0.f);
        const bool hit = alive && self_pair_contact(pr, s_pose, nbp, depth, n, pos);
        const unsigned hmask = __ballot_sync(FULL, hit);
        if (hit) {
          float* e = s_list + HL_WORDS * (cnt + __popc(hmask & lt));
          e[0] = depth; e[1] = n.x; e[2] = n.y; e[3] = n.z; e[4] = pos.x; e[5] = pos.y; e[6] = pos.z;
          e[7] = __int_as_float(-1 - pri[PR_BODY2]); e[8] = __int_as_float(H.npts + lane);
        }
        cnt += __popc(hmask);
      }
    }
  }
  __syncwarp();
  if (prof && lane == 0) { prof[6] = (unsigned)clock64(); prof[7] = (unsigned)cnt; }
  int total = cnt;
#pragma unroll 1
  while (total > KMAX) {   // drop the shallowest (ties: highest candidate index) until KMAX remain
    float dmin = 3.0e38f; int cmin = -1, imin = 0;     // depth, candidate index, list row of the entry to drop
#pragma unroll 1
    for (int e = lane; e < cnt; e += 32) {
      const float d = s_list[HL_WORDS * e]; const int c = __float_as_int(s_list[HL_WORDS * e + 8]);
      if (d > 0.f && (d < dmin || (d == dmin && c > cmin))) { dmin = d; cmin = c; imin = e; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float d2 = __shfl_xor_sync(FULL, dmin, o); const int c2 = __shfl_xor_sync(FULL, cmin, o), i2 = __shfl_xor_sync(FULL, imin, o);
      if (d2 < dmin || (d2 == dmin && c2 > cmin)) { dmin = d2; cmin = c2; imin = i2; }
    }
    __syncwarp();                                       // the scan above read the row that lane 0 now clears
    if (lane == 0) s_list[HL_WORDS * imin] = 0.f;
    __syncwarp();
    total--;
  }
  // contact records in candidate order (the list holds each slot's direct hits before its sphere hits): rank = live entries with a smaller index
#pragma unroll 1
  for (int e0 = 0; e0 < cnt; e0 += 32) {
    const int e = e0 + lane;
    const float* le = s_list + HL_WORDS * min(e, cnt - 1);
    const float depth = le[0];
    const bool live = e < cnt && depth > 0.f;
    const int cand = __float_as_int(le[8]);
    int rank = 0;
#pragma unroll 1
    for (int j = 0; j < cnt; j++) rank += (s_list[HL_WORDS * j] > 0.f && __float_as_int(s_list[HL_WORDS * j + 8]) < cand) ? 1 : 0;
    if (live) {
      float* ct = s_ct + rank * CT_WORDS;
      const f3 n = mk(le[1], le[2], le[3]);
      const f3 ex = (fabsf(n.x) < 0.9f) ? mk(1.f, 0.f, 0.f) : mk(0.f, 1.f, 0.f);
      const f3 t = ex - dot(ex, n) * n;
      const float inv = rsqrt_nr(dot(t, t));
      const f3 t1 = inv * t, t2 = cross(n, t1);
      ct[CF_POS] = le[4]; ct[CF_POS + 1] = le[5]; ct[CF_POS + 2] = le[6];
      ct[CF_N] = n.x; ct[CF_N + 1] = n.y; ct[CF_N + 2] = n.z;
      ct[CF_T1] = t1.x; ct[CF_T1 + 1] = t1.y; ct[CF_T1 + 2] = t1.z;
      ct[CF_T2] = t2.x; ct[CF_T2 + 1] = t2.y; ct[CF_T2 + 2] = t2.z;
      ct[CF_DEPTH] = depth;
      if constexpr (SELF) {   // a self contact's body is the first body of its pair
        const int body = cand < H.npts ? ptsi[cand] : reinterpret_cast<const int*>(blob_s + H.off_pair)[PAIR_WORDS * (cand - H.npts) + PR_BODY1];
        ct[CF_PT] = __int_as_float(cand); ct[CF_BODY] = __int_as_float(body); ct[CF_PAIR] = le[7];
      } else {
        ct[CF_PT] = __int_as_float(cand); ct[CF_BODY] = __int_as_float(ptsi[cand]); ct[CF_PAIR] = le[7];
      }
    }
  }
  return total;
}

// Stage C, static humanoid and generic instances: the compact-by-depth column Y = L^-T J^T of constraint row c along the chain of dof i0
// (depth m; -1 = a body welded to the world: a zero column), into column c of Y, and yz = Y . z.  fill: J is the direction axd at the
// point pos (base columns included), and jv += J v; otherwise the caller has put J into Y and jv.  The generic instance also computes
// the second half of a self contact's column with it (the chain of the pair's second body).
template <int UNR>
__device__ __forceinline__ void chain_column(float* Y, int c, bool fill, f3 pos, f3 axd, f3 O, int i0, int m, int floating, int nbase, int nvp,
                                             int DLP, int nbp, const int* danc, const int* dbody, const int* bodyi, const float* s_pose,
                                             const float* s_gv, const float* s_L, const float* s_invd, const float* s_z, float& jv, float& yz) {
  if (fill) {
    if (floating) {
      const f3 rc = cross(pos - O, axd);
      Y[0 * CP + c] = axd.x; Y[1 * CP + c] = axd.y; Y[2 * CP + c] = axd.z;
      Y[3 * CP + c] = rc.x; Y[4 * CP + c] = rc.y; Y[5 * CP + c] = rc.z;
      jv = axd.x * s_gv[0] + axd.y * s_gv[1] + axd.z * s_gv[2] + rc.x * s_gv[3] + rc.y * s_gv[4] + rc.z * s_gv[5];
    }
#pragma unroll (UNR > 1 ? 2 : 1)
    for (int t = nbase; t <= m; t++) {
      const int a_t = danc[t * nvp + i0], j = dbody[a_t];
      const f3 aj = mk(s_pose[(PF_A + 0) * nbp + j], s_pose[(PF_A + 1) * nbp + j], s_pose[(PF_A + 2) * nbp + j]);
      f3 col = aj;
      if (bodyi[BF_JTYPE * nbp + j] == 1) {
        const f3 pj = mk(s_pose[(PF_P + 0) * nbp + j], s_pose[(PF_P + 1) * nbp + j], s_pose[(PF_P + 2) * nbp + j]);
        col = cross(aj, pos - pj);
      }
      const float val = dot(col, axd);
      Y[t * CP + c] = val;
      jv += val * s_gv[a_t];
    }
  }
  yz = 0.f;
#pragma unroll 1
  for (int sI = m; sI >= 0; sI--) {
    const int a_s = danc[sI * nvp + i0];
    const float y = Y[sI * CP + c] * s_invd[a_s];
    Y[sI * CP + c] = y;
    yz += y * s_z[a_s];
#pragma unroll (UNR)
    for (int t = 0; t < sI; t++) Y[t * CP + c] -= s_L[a_s * DLP + t] * y;
  }
}

// Stage C, static humanoid and generic instances: subtracts the bias of constraint row c from its velocity u_c: ERP on a joint-limit
// violation (lm) or on a contact's depth (ct, normal rows, d == 2), plus restitution on a normal approach speed jv beyond
// rest_threshold.  The quadruped instance keeps the same lines inline (see there).
__device__ __forceinline__ void apply_row_bias(float& u_c, const rsb_params& prm, bool is_lim, int d, const float* lm, const float* ct, float jv) {
  if (is_lim) u_c -= prm.erp * lm[2] / prm.dt;
  else if (d == 2) {
    float target = prm.erp * ct[CF_DEPTH] / prm.dt;
    if (prm.restitution > 0.f && jv < -prm.rest_threshold) target += -prm.restitution * jv;
    u_c -= target;
  }
}

// Stage C: the actuator network of every listed dof of environment env at the start of the sub-step; net[i] = its output for listed dof i.
// Lane j is hidden unit j.  The listed dofs go through in groups of AN_G, each lane carrying one accumulator per dof of the group, so
// that every weight load (read-only path, transposed: the lanes read consecutive words) serves AN_G dofs.  A layer's inputs sit in s_x
// as [input][AN_G]: one 16-byte broadcast load gives one input of the whole group.  This sub-step's (e, v) go in front of the
// environment's history, which is shifted in place.  s_x: RSB_ACTNET_MAX_WIDTH * AN_G words of scratch (16-byte aligned), dead outside
// this call.
constexpr int AN_G = 4;
static_assert(RSB_ACTNET_MAX_WIDTH * AN_G <= HIST_WORDS, "the network's scratch is the Anderson history");
__device__ __forceinline__ void actuator_network(const ActNetDesc& an, int env, int lane, const float* s_gc, const float* s_gv, const float* s_pt,
                                                 const int* dofq, float* s_x, float* net) {
  const int H = an.H, W = an.W, F = 2 * H, hw = H - 1, n = an.n;
  float* const hist = an.hist + (size_t)env * n * 2 * hw;
#pragma unroll 1
  for (int g0 = 0; g0 < n; g0 += AN_G) {
    // features of the group: lane = (dof d of the group, feature k), AN_G * 2H <= 32; 0 past the end of the list
    float x = 0.f;
    int hi = -1;
    if (lane < AN_G * F) {
      const int d = lane / F, k = lane - d * F, s = g0 + d;
      if (s < n) {
        const int c = k >= H ? 1 : 0, t = k - c * H;   // c: 0 error, 1 velocity; t: sub-steps back
        const int i = an.dof[s];
        if (t > 0) x = hist[(s * 2 + c) * hw + t - 1];
        else if (c) x = s_gv[i];
        else { const int q = dofq[i]; x = s_pt[q] - s_gc[q]; }
        if (t < hw) hi = (s * 2 + c) * hw + t;
      }
      s_x[k * AN_G + d] = x;
    }
    __syncwarp();
    if (hi >= 0) hist[hi] = x;   // every lane has read the old history above
    const float* p = an.params;
    float h0 = 0.f, h1 = 0.f, h2 = 0.f, h3 = 0.f;
#pragma unroll 1
    for (int l = 0, nin = F; l < an.L; l++, nin = W) {
      float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
      if (lane < W) { a0 = a1 = a2 = a3 = __ldg(p + nin * W + lane); }
#pragma unroll 4
      for (int k = 0; k < nin; k++) {
        const float w = lane < W ? __ldg(p + k * W + lane) : 0.f;
        const float4 xk = *reinterpret_cast<const float4*>(s_x + k * AN_G);
        a0 = fmaf(w, xk.x, a0); a1 = fmaf(w, xk.y, a1); a2 = fmaf(w, xk.z, a2); a3 = fmaf(w, xk.w, a3);
      }
      p += nin * W + W;
      h0 = a0 / (1.f + fabsf(a0)); h1 = a1 / (1.f + fabsf(a1)); h2 = a2 / (1.f + fabsf(a2)); h3 = a3 / (1.f + fabsf(a3));
      __syncwarp();   // every lane has read this layer's inputs
      if (lane < W) *reinterpret_cast<float4*>(s_x + lane * AN_G) = make_float4(h0, h1, h2, h3);
      __syncwarp();
    }
    // output layer: a butterfly sum over the hidden units (lanes >= W hold 0)
    const float wo = lane < W ? __ldg(p + lane) : 0.f;
    float o0 = wo * h0, o1 = wo * h1, o2 = wo * h2, o3 = wo * h3;
#pragma unroll
    for (int m = 16; m > 0; m >>= 1) {
      o0 += __shfl_xor_sync(FULL, o0, m); o1 += __shfl_xor_sync(FULL, o1, m);
      o2 += __shfl_xor_sync(FULL, o2, m); o3 += __shfl_xor_sync(FULL, o3, m);
    }
    const float o = lane == 0 ? o0 : lane == 1 ? o1 : lane == 2 ? o2 : o3;
    if (lane < AN_G && g0 + lane < n) net[an.dof[g0 + lane]] = __ldg(p + W) + o;
    __syncwarp();   // s_x is refilled by the next group
  }
}

// Stage C: the LSTM actuator network of every listed dof of environment env, one cell step per sub-step from x = (e, v) at its start;
// net[i] = its output for listed dof i, and the environment's (h, c) rows advance in place.  The mapping is the MLP's: lane j is hidden
// unit j and holds its four gate pre-activations for the AN_G dofs of a group, every weight load serving the whole group.  A layer's
// pre-activations are accumulated in two passes over s_x ([input][AN_G], 16-byte broadcast loads): the layer input first, then this
// layer's h of the last sub-step, so that the scratch never holds more than RSB_ACTNET_MAX_WIDTH inputs.  Every lane reads and writes
// only its own unit's (h, c) words.  The evaluation order is fixed (bias, input columns, recurrent columns, one fmaf each), so the
// result does not depend on the launch shape.
__device__ __forceinline__ float an_sigmoid(float a) { return 1.f / (1.f + expf(-a)); }
__device__ __forceinline__ void actuator_lstm(const ActNetDesc& an, int env, int lane, const float* s_gc, const float* s_gv, const float* s_pt,
                                              const int* dofq, float* s_x, float* net) {
  const int L = an.L, W = an.W, n = an.n, W4 = 4 * W;
  const bool on = lane < W;
  float* const st = an.hist + (size_t)env * an.words;
#pragma unroll 1
  for (int g0 = 0; g0 < n; g0 += AN_G) {
    // layer 0's input: lane = (dof d of the group, feature k); 0 past the end of the list
    if (lane < 2 * AN_G) {
      const int d = lane >> 1, k = lane & 1, s = g0 + d;
      float x = 0.f;
      if (s < n) {
        const int i = an.dof[s];
        if (k) x = s_gv[i];
        else { const int q = dofq[i]; x = s_pt[q] - s_gc[q]; }
      }
      s_x[k * AN_G + d] = x;
    }
    __syncwarp();
    const float* p = an.params;
    float h[AN_G] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 1
    for (int l = 0, nin = 2; l < L; l++, nin = W) {
      float a[4][AN_G];
#pragma unroll
      for (int g = 0; g < 4; g++) {
        const float bg = on ? __ldg(p + (nin + W) * W4 + g * W + lane) : 0.f;
#pragma unroll
        for (int d = 0; d < AN_G; d++) a[g][d] = bg;
      }
      // pass 1: the layer input
#pragma unroll 2
      for (int k = 0; k < nin; k++) {
        const float4 xk = *reinterpret_cast<const float4*>(s_x + k * AN_G);
#pragma unroll
        for (int g = 0; g < 4; g++) {
          const float w = on ? __ldg(p + (k * 4 + g) * W + lane) : 0.f;
          a[g][0] = fmaf(w, xk.x, a[g][0]); a[g][1] = fmaf(w, xk.y, a[g][1]); a[g][2] = fmaf(w, xk.z, a[g][2]); a[g][3] = fmaf(w, xk.w, a[g][3]);
        }
      }
      __syncwarp();   // every lane has read the layer input
      // this layer's state of the last sub-step: h staged for pass 2, c kept in the lane
      float c[AN_G];
#pragma unroll
      for (int d = 0; d < AN_G; d++) {
        h[d] = 0.f; c[d] = 0.f;
        if (on && g0 + d < n) {
          const float* r = st + ((size_t)((g0 + d) * L + l) * 2) * W + lane;
          h[d] = r[0]; c[d] = r[W];
        }
      }
      if (on) *reinterpret_cast<float4*>(s_x + lane * AN_G) = make_float4(h[0], h[1], h[2], h[3]);
      __syncwarp();
      // pass 2: the recurrent input
      const float* pr = p + nin * W4;
#pragma unroll 2
      for (int k = 0; k < W; k++) {
        const float4 xk = *reinterpret_cast<const float4*>(s_x + k * AN_G);
#pragma unroll
        for (int g = 0; g < 4; g++) {
          const float w = on ? __ldg(pr + (k * 4 + g) * W + lane) : 0.f;
          a[g][0] = fmaf(w, xk.x, a[g][0]); a[g][1] = fmaf(w, xk.y, a[g][1]); a[g][2] = fmaf(w, xk.z, a[g][2]); a[g][3] = fmaf(w, xk.w, a[g][3]);
        }
      }
      // the cell (torch gate order i, f, g, o); lanes >= W end with h = c = 0
#pragma unroll
      for (int d = 0; d < AN_G; d++) {
        const float ig = an_sigmoid(a[0][d]) * tanhf(a[2][d]);
        c[d] = fmaf(an_sigmoid(a[1][d]), c[d], ig);
        h[d] = an_sigmoid(a[3][d]) * tanhf(c[d]);
        if (on && g0 + d < n) {
          float* r = st + ((size_t)((g0 + d) * L + l) * 2) * W + lane;
          r[0] = h[d];
          r[W] = c[d];
        }
      }
      p += (nin + W) * W4 + W4;
      __syncwarp();   // every lane has read the recurrent input
      if (on) *reinterpret_cast<float4*>(s_x + lane * AN_G) = make_float4(h[0], h[1], h[2], h[3]);   // the next layer's input
      __syncwarp();
    }
    // read-out: a butterfly sum over the hidden units (lanes >= W hold 0)
    const float wo = on ? __ldg(p + lane) : 0.f;
    float o0 = wo * h[0], o1 = wo * h[1], o2 = wo * h[2], o3 = wo * h[3];
#pragma unroll
    for (int m = 16; m > 0; m >>= 1) {
      o0 += __shfl_xor_sync(FULL, o0, m); o1 += __shfl_xor_sync(FULL, o1, m);
      o2 += __shfl_xor_sync(FULL, o2, m); o3 += __shfl_xor_sync(FULL, o3, m);
    }
    const float o = lane == 0 ? o0 : lane == 1 ? o1 : lane == 2 ? o2 : o3;
    if (lane < AN_G && g0 + lane < n) net[an.dof[g0 + lane]] = __ldg(p + W) + o;
    __syncwarp();   // s_x is refilled by the next group
  }
}

// Stage C: the actuation delay of environment env at one advancing sub-step.  The command of a joint dof j (nbase + j) is the triple
// (ptarget[q], vtarget, tau_ff); it goes into ring slot t % DELAY_SLOTS, and the one of sub-step max(t - d, 0) replaces it in s_pt,
// s_vt and s_tau, where the PD law, the actuator network and stage E read it.  At sub-step 0 of a launch the command is what the
// prologue fetched; later sub-steps of the launch repeat it, from the slot the sub-step before wrote, since s_* then hold applied values.
// A slot is overwritten DELAY_SLOTS sub-steps after it was written, later than any delay reads it.  t is kept in [0, 2 DELAY_SLOTS):
// from DELAY_SLOTS on, t - d >= 0 and only t % DELAY_SLOTS matters.  Each lane touches its own ring words only, but its s_* words are
// read by other lanes: the first __syncwarp orders the pt_store / vt_store copies of sub-step 0 (lane i reads word i) before this
// lane's writes, the second orders every lane's read of t and of s_* before the counter and the PD law move on.
constexpr int DELAY_SLOTS = RSB_MAX_ACTUATION_DELAY + 1;
__device__ __forceinline__ void actuation_delay(int* state, float* rings, int env, int sub, int nbase, int nv, const int* dofq, float* s_pt,
                                                float* s_vt, float* s_tau, int lane) {
  __syncwarp();
  const int nj = nv - nbase, row = 3 * nj;
  int* const st = state + 2 * env;
  float* const ring = rings + (size_t)env * DELAY_SLOTS * row;
  const int2 dt = *reinterpret_cast<const int2*>(st);
  const int d = dt.x, t = dt.y;
  float* const cur = ring + (t % DELAY_SLOTS) * row;
  const float* const prev = ring + ((t + DELAY_SLOTS - 1) % DELAY_SLOTS) * row;
  const float* const app = ring + (max(t - d, 0) % DELAY_SLOTS) * row;
#pragma unroll 1
  for (int j = lane; j < nj; j += 32) {
    const int i = nbase + j, q = dofq[i];
    float p, v, f;
    if (sub == 0) { p = s_pt[q]; v = s_vt[i]; f = s_tau[i]; }
    else { p = prev[j]; v = prev[nj + j]; f = prev[2 * nj + j]; }
    cur[j] = p; cur[nj + j] = v; cur[2 * nj + j] = f;
    s_pt[q] = app[j]; s_vt[i] = app[nj + j]; s_tau[i] = app[2 * nj + j];
  }
  __syncwarp();
  if (lane == 0) st[1] = t + 1 < 2 * DELAY_SLOTS ? t + 1 : t + 1 - DELAY_SLOTS;
}

// Stages C and E: kp, kd and effort limit of dof i in environment env.  The blob's value (gain: kp | kd | effort, nvp each) unless the
// environment has a row (StepArgs::actuator) whose entry is >= 0; the gains are 0 outside PD mode (use_pd), the effort limit holds in
// both control modes
__device__ __forceinline__ void dof_actuator(const StepArgs& args, const float* gain, int nvp, int env, int nv, int i, float& kpi, float& kdi, float& emi) {
  kpi = args.use_pd ? gain[i] : 0.f; kdi = args.use_pd ? gain[nvp + i] : 0.f; emi = gain[2 * nvp + i];
  if (args.actuator) {
    const float* r = args.actuator + (size_t)env * 3 * nv + i;
    if (args.use_pd) {
      const float rp = r[0], rd = r[nv];
      if (rp >= 0.f) kpi = rp;
      if (rd >= 0.f) kdi = rd;
    }
    const float re = r[2 * nv];
    if (re >= 0.f) emi = re;
  }
}

// Stage E, static humanoid and generic instances: adds Y[di] . lam of the contacts whose column block Y (rows 3k..3k+2) lies on a chain
// through dof i (depth di) to sacc; SECOND: the self contacts' second halves (the chain of the pair's second body), subtracted
template <int UNR, bool SECOND>
__device__ __forceinline__ void chain_gather(float& sacc, const float* Y, const float* s_lam, const float* s_ct, int K, int i, int di, const int* bdof,
                                             const int* ddepth, const int* danc, int nvp) {
#pragma unroll (UNR)
  for (int k = 0; k < K; k++) {
    int i0;
    if (SECOND) {
      const int pr = __float_as_int(s_ct[k * CT_WORDS + CF_PAIR]);
      i0 = pr < 0 ? bdof[-1 - pr] : -1;
    } else {
      i0 = bdof[__float_as_int(s_ct[k * CT_WORDS + CF_BODY])];
    }
    if (i0 >= 0 && ddepth[i0] >= di && danc[di * nvp + i0] == i) {
      const float y = Y[di * CP + 3 * k] * s_lam[3 * k] + Y[di * CP + 3 * k + 1] * s_lam[3 * k + 1] + Y[di * CP + 3 * k + 2] * s_lam[3 * k + 2];
      if (SECOND) sacc -= y;
      else sacc += y;
    }
  }
}

// ------------------------------------------------------------------ the kernel -----------------
// The compiled instances (SPEC, the value rsb_internal_launch_instance reports).  The generic instance reads the model dimensions from
// the blob header and is the only one that runs self-collision pairs; the others have the dimensions of SPEC_DIMS compiled in, so every
// table and workspace offset is an immediate.  pick_config (batch.cu) takes a static instance for a model of exactly its dimensions:
// every 12-joint quadruped (ANYmal, A1, Go1, ...) whose parent table is base + 4 chains of 3, and the Atlas-like humanoid.
enum Spec { SPEC_GENERIC = 0, SPEC_QUAD = 1, SPEC_HUMANOID = 2, SPEC_COUNT = 3 };
constexpr Dims SPEC_DIMS[SPEC_COUNT] = {{0, 0, 0, 0, 0, 0}, {13, 19, 18, 1, 3, 8}, {31, 37, 36, 1, 10, 15}};
__host__ __device__ constexpr bool operator==(const Dims& a, const Dims& b) {
  return a.nb == b.nb && a.nq == b.nq && a.nv == b.nv && a.floating == b.floating && a.maxdepth == b.maxdepth && a.maxdd == b.maxdd;
}

// AN: the instance with the actuator network (launched only while one is set and PD laws apply); DL: the one with actuation delays
// (launched only while they are set, by the launches that advance the state).  Without them the step is what it was: inlined into
// every instance, either one changed the register allocation of many of them (ptxas, CUDA 12.9; DESIGN.md §2)
template <int WPC, int SLOTS, int SPEC, bool AN, bool DL>
__global__ void __launch_bounds__(WPC * 32, (WPC == 14 ? 2 : 1)) rsb_step_kernel(const __grid_constant__ StepArgs args) {
  extern __shared__ __align__(128) uint32_t smem[];
  __shared__ __align__(8) uint64_t tma_bar;
  const int lane = threadIdx.x & 31;     // (re-read wherever needed at 72 registers; S2R SR_LANEID instead, with or without a range assumption, measured 12 % slower)
  // the shuffle marks the warp index as warp-uniform for the compiler: the workspace base then lives in a uniform register
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  constexpr bool SELF = SPEC == SPEC_GENERIC;   // dimensions from the blob header; self-collision pairs
  constexpr bool ST = !SELF;                    // dimensions compiled in
  constexpr bool QUAD = SPEC == SPEC_QUAD;      // the 4 x 3-chain topology compiled in as well
  // deep trees on few resident warps (the humanoid instance: 14 warps per SM, latency-bound) get their dependent shared-memory loops of
  // stage C unrolled for memory-level parallelism; everything else keeps them rolled (instruction cache)
  constexpr int UNR = SPEC == SPEC_HUMANOID ? 4 : 1;
  constexpr Dims SD = SPEC_DIMS[SPEC];
  // lanes >= nb hold exact zeros in stage A's root sum: with at most 16 bodies its xor-16 butterfly step adds 0 and is skipped
  constexpr int ROOT_XOR = (ST && SD.nb <= 16) ? 8 : 16;
  constexpr WsLayout LS = make_ws_layout(SD);
  constexpr BlobHeader HS = make_blob_header(SD, 0, 0);
#define WSO(f) (ST ? LS.f : args.ws.f)
  // shared memory: [WPC workspaces][model constant blob]
  uint32_t* const blob_s = smem + WPC * WSO(words);

  // ---- stage the model constant block once per CTA with one TMA bulk copy ----------------------
  // the out-of-line stages read the terrain descriptor and the solver parameters from shared memory: a reference to the kernel
  // parameters is a generic pointer there, and every field read through it a global-latency load (ncu: long scoreboard)
  __shared__ TerrainDesc s_ter;
  __shared__ rsb_params s_prm;
  if (threadIdx.x == 0) {
    mbar_init(&tma_bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    s_ter = args.ter; s_prm = args.prm;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_expect_tx(&tma_bar, (uint32_t)args.blob_words * 4u);
    tma_bulk_g2s(blob_s, args.blob, (uint32_t)args.blob_words * 4u, &tma_bar);
  }
  mbar_wait(&tma_bar, 0);

  const BlobHeader& H = *reinterpret_cast<const BlobHeader*>(blob_s);
#define HO(f) (ST ? HS.f : H.f)
  const int nb = HO(nb), nq = HO(nq), nv = HO(nv), floating = HO(floating), maxdepth = HO(maxdepth);
  const int nbp = HO(nbp), nvp = HO(nvp);

  const float* bodyf = reinterpret_cast<const float*>(blob_s + HO(off_body));
  const int* bodyi = reinterpret_cast<const int*>(blob_s + HO(off_body));
  const int* anc = reinterpret_cast<const int*>(blob_s + HO(off_anc));
  const float* ptsf = reinterpret_cast<const float*>(blob_s + HO(off_pts));
  // kp | kd | actuator effort limit per dof (URDF <limit effort>, 3e38 = none), each nvp long (dof_actuator)
  const float* gain = reinterpret_cast<const float*>(blob_s + HO(off_gain));
  const int* dofq = reinterpret_cast<const int*>(blob_s + HO(off_dofq));
  const float* sec_c = reinterpret_cast<const float*>(blob_s + HO(off_sec));
  const int nbase = HO(nbase), maxdd = HO(maxdd), DLP = HO(dlp);
  const int* ddepth = reinterpret_cast<const int*>(blob_s + HO(off_ddepth));
  const int* dsub = reinterpret_cast<const int*>(blob_s + HO(off_dsub));
  const int* danc = reinterpret_cast<const int*>(blob_s + HO(off_danc));
  const int* dbody = reinterpret_cast<const int*>(blob_s + HO(off_dbody));
  const int* bdof = reinterpret_cast<const int*>(blob_s + HO(off_bdof));
  const int* lvl = reinterpret_cast<const int*>(blob_s + HO(off_lvl));
  const int* lvldofs = reinterpret_cast<const int*>(blob_s + HO(off_lvldofs));
  const int* entstart = reinterpret_cast<const int*>(blob_s + HO(off_entstart));
  const int* ent = reinterpret_cast<const int*>(blob_s + H.off_ent);
  const int8_t* lcad = reinterpret_cast<const int8_t*>(blob_s + HO(off_lcad));

  float* const ws = reinterpret_cast<float*>(smem) + warp * WSO(words);
  float* s_gc = ws + WSO(o_gc); float* s_gv = ws + WSO(o_gv); float* s_tau = ws + WSO(o_tau); float* s_pt = ws + WSO(o_pt); float* s_vt = ws + WSO(o_vt);
  float* s_L = ws + WSO(o_L); float* s_invd = ws + WSO(o_invd); float* s_rhs = ws + WSO(o_rhs); float* s_z = ws + WSO(o_z); float* s_ct = ws + WSO(o_ct);
  float* s_Y = ws + WSO(o_Y); float* s_lam = ws + WSO(o_lam); float* s_u = ws + WSO(o_u); float* s_lim = ws + WSO(o_lim); float* s_hist = ws + WSO(o_hist); float* s_sat = ws + WSO(o_sat);
  float* s_h = ws + WSO(o_h); float* s_b = ws + WSO(o_b); float* s_pose = ws + WSO(o_pose); float* s_G = ws + WSO(o_G);
#undef WSO
#undef HO
  // Long-lived per-thread values are kept to a minimum: at 72 registers (28 warps x 32 lanes per SM) everything cached
  // here is spilled, and 28 warps' spill slots do not fit the L1 next to the terrain gathers -- every reload was an L2
  // round trip on the critical path.  Kernel parameters are read in place (constant bank), model constants from the
  // shared-memory blob at the point of use.

  // body constants of this lane (lane == body)
  const int b = lane;
  const bool bvalid = b < nb;
  const int bb = bvalid ? b : 0;
#define MYB(f) (bodyi[(f) * nbp + bb])
  // (row, col) of the base 6x6 lower triangle owned by lanes 0..20, packed row | col << 3: one table per CTA
  __shared__ uint8_t s_tri[32];
  __shared__ int s_work[2];   // this CTA's environments in the last launch: sum over rounds of (warps x the round's largest solver work), total work
  if (threadIdx.x < 32) {
    int pr = 0;
    for (int r = 0, e = 0; r < 6; r++) for (int c = 0; c <= r; c++, e++) if (e == (int)threadIdx.x) pr = r | (c << 3);
    s_tri[threadIdx.x] = (uint8_t)pr;
    if (threadIdx.x < 2) s_work[threadIdx.x] = 0;
  }
  __syncthreads();

  const int warps_total = gridDim.x * WPC;
  // The sub-step barrier makes every warp of a round wait for the round's slowest solve at each sub-step.  It pays (instruction-cache
  // locality; the slowest warp finishes alone at single-warp speed) while the largest solver work of a round is at most twice the
  // mean: on an H100, 4096 quadrupeds standing on rough ground (ratio 1.6) and humanoids standing on box feet (1.3) run 28 % and
  // 12 % faster with it, fallen quadrupeds under random torques (ratio 3.1) 20 % slower.  Each CTA decides for itself from the work
  // (sweeps x contacts of the last sub-step) that the environments of its rounds and of the same rounds of the next NEIGH - 1 CTAs
  // did in the last launch: one CTA's two rounds alone scatter too widely (on the H100, per-CTA ratios of the first workload reach
  // 2.0, those of the third go down to 1.8).  Every thread reads the same integer sums, so all warps of the CTA agree (kept in shared
  // memory: a register live across the loop costs spills at 72 registers); another CTA may already have stored new work for some of
  // those environments, which changes the decision of this CTA, never a result.
  if (args.substep_barrier) {
    constexpr int NEIGH = 8;
    const int neigh = min(NEIGH, (int)gridDim.x);
#pragma unroll 1
    for (int q = warp; (q / neigh) * warps_total < args.num_envs; q += WPC) {   // round q / neigh of CTA blockIdx + q % neigh: lane = warp
      const int first = (q / neigh) * warps_total + (((int)blockIdx.x + q % neigh) % (int)gridDim.x) * WPC, e = first + lane;
      const int w = (lane < WPC && e < args.num_envs) ? args.iters[e] * args.ncontacts[e] : 0;
      const int wmax = __reduce_max_sync(FULL, w), wsum = __reduce_add_sync(FULL, w);
      if (lane == 0 && first < args.num_envs) { atomicAdd(&s_work[0], min(WPC, args.num_envs - first) * wmax); atomicAdd(&s_work[1], wsum); }
    }
    __syncthreads();
  }
#pragma unroll 1
  for (int env = blockIdx.x * WPC + warp; env < args.num_envs; env += warps_total) {
    // ---- load this environment's rows (coalesced: one row per warp) -----------------------------
    {
      const float* g_gc = args.gc + (size_t)env * args.gc_stride;
      const float* g_gv = args.gv + (size_t)env * args.gv_stride;
#pragma unroll 1
      for (int i = lane; i < nq; i += 32) s_gc[i] = g_gc[i];
#pragma unroll 1
      for (int i = lane; i < nv; i += 32) s_gv[i] = g_gv[i];
#pragma unroll 1
      for (int i = lane; i < nv; i += 32) s_tau[i] = args.tau ? args.tau[(size_t)env * args.gv_stride + i] : 0.f;
      if (args.use_pd || DL) {
        // PD targets are first needed in stage C: fetch them asynchronously (cp.async, global -> shared) so that a
        // caller buffer in pinned host memory (zero-copy control step) is read over PCIe behind stages A and B.  With an actuation
        // delay they are fetched in force mode too: the command history records them in both control modes
        // gym task: the joint part of the position target is action * actionStd + actionMean (ENVIRONMENT::step(), first half); the base
        // part comes from the batch's own rows like every other target
        const int nfetch = args.gym_action ? 7 : nq;
#pragma unroll 1
        for (int i = lane; i < nfetch; i += 32) cp_async4(&s_pt[i], &args.ptarget[(size_t)env * args.pt_stride + i]);
#pragma unroll 1
        for (int i = lane; i < nv; i += 32) cp_async4(&s_vt[i], &args.vtarget[(size_t)env * args.vt_stride + i]);
        asm volatile("cp.async.commit_group;" ::: "memory");
        if (args.gym_action) {
          const int nj = nq - 7;
#pragma unroll 1
          for (int i = lane; i < nj; i += 32) s_pt[7 + i] = args.gym_action[(size_t)env * nj + i] * args.gym.action_std[i] + args.gym.action_mean[i];
        }
      }
    }
    __syncwarp();
    // Paired stage A (quadruped instance): stage A uses 13 of 32 lanes and the sub-step barrier releases the warps of a round into it
    // together, so warps w and w ^ 4 (the same scheduler when warps map to schedulers by w % 4) share one instruction stream there:
    // the leader w runs its own environment on lanes 0-15 and the partner's on lanes 16-31, reading and writing the partner's
    // workspace, while the partner waits on their named barrier (2-13), then runs stages B-E itself.  Only where the CTA keeps the
    // sub-step barrier: its bar.sync orders the partner's previous sub-step (and row load) before the leader's reads.  pair_a: 1 leader
    // with a partner, -1 partner, 0 alone (other instances; a leader whose partner has no environment in this round).
    int pair_a = 0;
    if constexpr (QUAD) {
      if (args.pair_stage_a && args.substep_barrier && s_work[0] <= 2 * s_work[1])
        pair_a = (warp & 4) ? -1 : (warp + 4 < min(WPC, args.num_envs - (env - warp)) ? 1 : 0);
    }
    int K = 0, iters = 0;
    float resid = 0.f; int gs_status = RSB_SOLVER_CONVERGED;

#pragma unroll 1
    for (int sub = 0; sub < args.substeps; sub++) {
      // Re-align the round's warps (instruction-cache locality: warps drifting through a 75 KB kernel miss the instruction
      // cache far more often than warps in the same stage, and the slowest warp of a sub-step finishes its solve alone).
      // The barrier counts the warps of this CTA that own an environment in this round (env - warp = the CTA's first one).  Counts
      // of two rounds never meet on barrier 1: a warp arrives at it only at the sub-steps of its current round, and the last barrier
      // of round r (its last sub-step) completes only once every warp of round r has arrived, so no round-r warp is still to arrive
      // when the first warp of round r + 1 does.  A warp without an environment in round r + 1 (environments are dense, so those are
      // the highest warps of the CTA) leaves the loop and never arrives again.
      if (args.substep_barrier && s_work[0] <= 2 * s_work[1])
        asm volatile("bar.sync 1, %0;" ::"r"(min(WPC, args.num_envs - (env - warp)) * 32));
      if (args.prof && lane == 0) args.prof[((size_t)env * 4 + (sub & 3)) * 8 + 0] = (unsigned)clock64();
      // =========================== stage A: FK + RNEA + CRBA =====================================
      f3 O;                                  // base origin: centre of the world-aligned CRBA frame (stages A and C)
      if (pair_a >= 0) {
        // the environment this lane computes (pair_a: lanes 16-31 of a leader take the partner's) and its workspace, a_*; with 16 lanes
        // per environment the quadruped's body is lane & 15, the upper lanes of a warp that runs alone hold no body
        const bool up = QUAD && lane >= 16 && pair_a > 0;
        const int envA = up ? env + 4 : env;
        float* const wsA = up ? ws + 4 * LS.words : ws;
        const float* const a_gc = wsA + (s_gc - ws); const float* const a_gv = wsA + (s_gv - ws);
        float* const a_L = wsA + (s_L - ws); float* const a_h = wsA + (s_h - ws); float* const a_pose = wsA + (s_pose - ws);
        const int b = QUAD ? (lane & 15) : lane;
        const bool bvalid = b < nb && (!QUAD || lane < 16 || pair_a > 0);
        const int bb = bvalid ? b : 0;
        unsigned* const prof_a = (QUAD && args.prof_a && bvalid && b == 0) ? args.prof_a + ((size_t)envA * 4 + (sub & 3)) * 4 : nullptr;   // quadruped only
        float R[9]; f3 p, w, v, wd, vd, ax;
        if (floating) {
          float qw = a_gc[3], qx = a_gc[4], qy = a_gc[5], qz = a_gc[6];
          float inv = 1.0f / sqrtf(qw * qw + qx * qx + qy * qy + qz * qz);
          qw *= inv; qx *= inv; qy *= inv; qz *= inv;
          R[0] = 1.f - 2.f * (qy * qy + qz * qz); R[1] = 2.f * (qx * qy - qw * qz); R[2] = 2.f * (qx * qz + qw * qy);
          R[3] = 2.f * (qx * qy + qw * qz); R[4] = 1.f - 2.f * (qx * qx + qz * qz); R[5] = 2.f * (qy * qz - qw * qx);
          R[6] = 2.f * (qx * qz - qw * qy); R[7] = 2.f * (qy * qz + qw * qx); R[8] = 1.f - 2.f * (qx * qx + qy * qy);
          p = mk(a_gc[0], a_gc[1], a_gc[2]);
          v = mk(a_gv[0], a_gv[1], a_gv[2]); w = mk(a_gv[3], a_gv[4], a_gv[5]);
        } else {
#pragma unroll
          for (int k = 0; k < 9; k++) R[k] = bodyf[(BF_JROT + k) * nbp];
          p = mk(bodyf[(BF_JPOS + 0) * nbp], bodyf[(BF_JPOS + 1) * nbp], bodyf[(BF_JPOS + 2) * nbp]);
          v = mk(0.f, 0.f, 0.f); w = mk(0.f, 0.f, 0.f);
        }
        O = p;
        const bool jrot_identity = (H.flags & 1) != 0;
        wd = mk(0.f, 0.f, 0.f); vd = mk(-args.prm.gravity[0], -args.prm.gravity[1], -args.prm.gravity[2]); ax = mk(0.f, 0.f, 0.f);
#pragma unroll 1
        for (int d = 1; d <= maxdepth; d++) {
          int j = (bvalid && d <= MYB(BF_DEPTH)) ? anc[(d - 1) * nbp + b] : -1;
          if (j >= 0) {
            f3 jp = mk(bodyf[(BF_JPOS + 0) * nbp + j], bodyf[(BF_JPOS + 1) * nbp + j], bodyf[(BF_JPOS + 2) * nbp + j]);
            float Rj[9];
            f3 al = mk(bodyf[(BF_AXIS + 0) * nbp + j], bodyf[(BF_AXIS + 1) * nbp + j], bodyf[(BF_AXIS + 2) * nbp + j]);
            f3 r = mulR(R, jp);
            if (jrot_identity) {
#pragma unroll
              for (int k = 0; k < 9; k++) Rj[k] = R[k];
            } else {
              float Jr[9];      // scoped here: declared outside the branch it was a maybe-uninitialised value carried (through the stack) round the loop
#pragma unroll
              for (int k = 0; k < 9; k++) Jr[k] = bodyf[(BF_JROT + k) * nbp + j];
              matmul3(R, Jr, Rj);
            }
            f3 aj = mulR(Rj, al);
            float q = a_gc[bodyi[BF_QIDX * nbp + j]], qd = a_gv[bodyi[BF_VIDX * nbp + j]];
            const bool rev = bodyi[BF_JTYPE * nbp + j] == 1;
            if (!rev) r = r + q * aj;
            f3 wxr = cross(w, r);
            f3 vn = v + wxr;
            f3 vdn = vd + cross(wd, r) + cross(w, wxr);
            f3 qa = qd * aj;
            if (rev) {
              float sq, cq;
              sincosf(q, &sq, &cq);
              float t = 1.f - cq;
              float Rq[9] = {t * al.x * al.x + cq, t * al.x * al.y - sq * al.z, t * al.x * al.z + sq * al.y,
                             t * al.x * al.y + sq * al.z, t * al.y * al.y + cq, t * al.y * al.z - sq * al.x,
                             t * al.x * al.z - sq * al.y, t * al.y * al.z + sq * al.x, t * al.z * al.z + cq};
              matmul3(Rj, Rq, R);
              wd = wd + cross(w, qa);
              w = w + qa;
            } else {
#pragma unroll
              for (int k = 0; k < 9; k++) R[k] = Rj[k];
              vn = vn + qa;
              vdn = vdn + 2.f * cross(w, qa);
            }
            p = p + r; v = vn; vd = vdn; ax = aj;
          }
        }
        // publish poses for stages B and C
        if (bvalid) {
#pragma unroll
          for (int k = 0; k < 9; k++) a_pose[(PF_R + k) * nbp + b] = R[k];
          a_pose[(PF_P + 0) * nbp + b] = p.x; a_pose[(PF_P + 1) * nbp + b] = p.y; a_pose[(PF_P + 2) * nbp + b] = p.z;
          a_pose[(PF_A + 0) * nbp + b] = ax.x; a_pose[(PF_A + 1) * nbp + b] = ax.y; a_pose[(PF_A + 2) * nbp + b] = ax.z;
        }
        if (prof_a) prof_a[0] = (unsigned)clock64();
        // per-body force and inertia terms about O
        float X[16];   // F(3) N_O(3) m h(3) I_O(6)
        {
          // inertial parameters: the model's (blob) or this environment's own row (envA: a leader's upper lanes read the partner's),
          // the same floats into the same expressions either way
          float m; f3 cl; float I0, I1, I2, I3, I4, I5;
          if (args.body_inertia) {
            const float4* row = reinterpret_cast<const float4*>(args.body_inertia + ((size_t)envA * nb + bb) * BI_WORDS);
            const float4 r0 = __ldg(row), r1 = __ldg(row + 1), r2 = __ldg(row + 2);
            m = r0.x; cl = mk(r0.y, r0.z, r0.w);
            I0 = r1.x; I1 = r1.y; I2 = r1.z; I3 = r1.w; I4 = r2.x; I5 = r2.y;
          } else {
            m = bodyf[BF_MASS * nbp + bb];
            cl = mk(bodyf[(BF_COM + 0) * nbp + bb], bodyf[(BF_COM + 1) * nbp + bb], bodyf[(BF_COM + 2) * nbp + bb]);
            I0 = bodyf[(BF_INERTIA + 0) * nbp + bb]; I1 = bodyf[(BF_INERTIA + 1) * nbp + bb]; I2 = bodyf[(BF_INERTIA + 2) * nbp + bb];
            I3 = bodyf[(BF_INERTIA + 3) * nbp + bb]; I4 = bodyf[(BF_INERTIA + 4) * nbp + bb]; I5 = bodyf[(BF_INERTIA + 5) * nbp + bb];
          }
          if (!bvalid) { m = 0.f; I0 = I1 = I2 = I3 = I4 = I5 = 0.f; }
          f3 c = mulR(R, cl);
          f3 cO = (p - O) + c;
          f3 ac = vd + cross(wd, c) + cross(w, cross(w, c));
          f3 f = m * ac;
          // Iw = R I R^T
          float RI[9];
#pragma unroll
          for (int r = 0; r < 3; r++) {
            RI[3 * r + 0] = R[3 * r] * I0 + R[3 * r + 1] * I1 + R[3 * r + 2] * I2;
            RI[3 * r + 1] = R[3 * r] * I1 + R[3 * r + 1] * I3 + R[3 * r + 2] * I4;
            RI[3 * r + 2] = R[3 * r] * I2 + R[3 * r + 1] * I4 + R[3 * r + 2] * I5;
          }
          float W0 = RI[0] * R[0] + RI[1] * R[1] + RI[2] * R[2], W1 = RI[0] * R[3] + RI[1] * R[4] + RI[2] * R[5], W2 = RI[0] * R[6] + RI[1] * R[7] + RI[2] * R[8];
          float W3 = RI[3] * R[3] + RI[4] * R[4] + RI[5] * R[5], W4 = RI[3] * R[6] + RI[4] * R[7] + RI[5] * R[8], W5 = RI[6] * R[6] + RI[7] * R[7] + RI[8] * R[8];
          f3 Iw = mk(W0 * w.x + W1 * w.y + W2 * w.z, W1 * w.x + W3 * w.y + W4 * w.z, W2 * w.x + W4 * w.y + W5 * w.z);
          f3 Iwd = mk(W0 * wd.x + W1 * wd.y + W2 * wd.z, W1 * wd.x + W3 * wd.y + W4 * wd.z, W2 * wd.x + W4 * wd.y + W5 * wd.z);
          f3 n = Iwd + cross(w, Iw) + cross(cO, f);
          float cc = dot(cO, cO);
          X[0] = f.x; X[1] = f.y; X[2] = f.z; X[3] = n.x; X[4] = n.y; X[5] = n.z;
          X[6] = m; X[7] = m * cO.x; X[8] = m * cO.y; X[9] = m * cO.z;
          X[10] = W0 + m * (cc - cO.x * cO.x); X[11] = W1 - m * cO.x * cO.y; X[12] = W2 - m * cO.x * cO.z;
          X[13] = W3 + m * (cc - cO.y * cO.y); X[14] = W4 - m * cO.y * cO.z; X[15] = W5 + m * (cc - cO.z * cO.z);
        }
        if (args.ext) {   // ArticulatedSystem::setExternalForce / setExternalTorque: h -= J^T wrench, through the RNEA force terms
          const float* e = args.ext + (size_t)envA * EXT_WORDS;
          if (bvalid && __float_as_int(e[0]) == b) {
            const f3 Fe = mk(e[1], e[2], e[3]), Te = mk(e[4], e[5], e[6]);
            const f3 re = (p - O) + mulR(R, mk(e[7], e[8], e[9]));
            const f3 Me = cross(re, Fe) + Te;
            X[0] -= Fe.x; X[1] -= Fe.y; X[2] -= Fe.z; X[3] -= Me.x; X[4] -= Me.y; X[5] -= Me.z;
          }
        }
        if (prof_a) prof_a[1] = (unsigned)clock64();
        // subtree sums: bodies are in DFS pre-order, so subtree(b) = lanes [b, b + size)
        float A[16];
#pragma unroll
        for (int k = 0; k < 16; k++) A[k] = X[k];
        const int my_sub = MYB(BF_SUBTREE);
        const int max_inner = (H.flags >> 8) & 0xff;   // largest non-root subtree size - 1
#pragma unroll 1
        for (int s = 1; s <= max_inner; s++) {
          bool take = (b > 0) && (s < my_sub);
#pragma unroll
          for (int k = 0; k < 16; k++) {
            float x = __shfl_down_sync(FULL, X[k], s);
            if (take) A[k] += x;
          }
        }
        {   // root: everything
          float T[16];
#pragma unroll
          for (int k = 0; k < 16; k++) {
            float t = X[k];
#pragma unroll
            for (int o = ROOT_XOR; o > 0; o >>= 1) t += __shfl_xor_sync(FULL, t, o);
            T[k] = t;
          }
          if (b == 0) {
#pragma unroll
            for (int k = 0; k < 16; k++) A[k] = T[k];
          }
        }
        if (prof_a) prof_a[2] = (unsigned)clock64();
        // bias force h and CRBA columns (row i of M stored compactly: column index = ancestor depth)
        f3 rO = p - O;
        const bool rev = MYB(BF_JTYPE) == 1;
        f3 Sw = rev ? ax : mk(0.f, 0.f, 0.f);
        f3 Sv = rev ? cross(rO, ax) : ax;
        f3 Fc = mk(A[0], A[1], A[2]), Nc = mk(A[3], A[4], A[5]);
        f3 hh = mk(A[7], A[8], A[9]);
        f3 ff = A[6] * Sv + cross(Sw, hh);
        f3 nn = mk(A[10] * Sw.x + A[11] * Sw.y + A[12] * Sw.z, A[11] * Sw.x + A[13] * Sw.y + A[14] * Sw.z, A[12] * Sw.x + A[14] * Sw.y + A[15] * Sw.z) + cross(hh, Sv);
        const int my_vidx = MYB(BF_VIDX);
        const int my_dd = nbase + MYB(BF_DEPTH) - 1;          // depth of this body's dof in the dof tree
        if (bvalid && b > 0) {
          float* row = a_L + my_vidx * DLP;
          a_h[my_vidx] = dot(Sw, Nc) + dot(Sv, Fc);      // S^T [N_O; F]  (moment about O)
          row[my_dd] = dot(Sw, nn) + dot(Sv, ff);
          if (floating) { row[0] = ff.x; row[1] = ff.y; row[2] = ff.z; row[3] = nn.x; row[4] = nn.y; row[5] = nn.z; }
        }
        if (bvalid && b == 0 && floating) {
          a_h[0] = Fc.x; a_h[1] = Fc.y; a_h[2] = Fc.z; a_h[3] = Nc.x; a_h[4] = Nc.y; a_h[5] = Nc.z;
          // lower triangle of [ m 1, -[h]x ; [h]x, I_O ]
          a_L[0 * DLP + 0] = A[6]; a_L[1 * DLP + 0] = 0.f; a_L[1 * DLP + 1] = A[6];
          a_L[2 * DLP + 0] = 0.f; a_L[2 * DLP + 1] = 0.f; a_L[2 * DLP + 2] = A[6];
          a_L[3 * DLP + 0] = 0.f; a_L[3 * DLP + 1] = -hh.z; a_L[3 * DLP + 2] = hh.y;
          a_L[4 * DLP + 0] = hh.z; a_L[4 * DLP + 1] = 0.f; a_L[4 * DLP + 2] = -hh.x;
          a_L[5 * DLP + 0] = -hh.y; a_L[5 * DLP + 1] = hh.x; a_L[5 * DLP + 2] = 0.f;
          a_L[3 * DLP + 3] = A[10]; a_L[4 * DLP + 3] = A[11]; a_L[5 * DLP + 3] = A[12];
          a_L[4 * DLP + 4] = A[13]; a_L[5 * DLP + 4] = A[14]; a_L[5 * DLP + 5] = A[15];
        }
        {   // M[vi][vj] for proper ancestors j (excluding the root): column = depth of j's dof
          int j = (bvalid && b > 0) ? MYB(BF_PARENT) : 0;
          int tj = my_dd - 1;
#pragma unroll 1
          for (int d = 2; d <= maxdepth; d++) {
            int src = (j > 0 ? j : 0) + (QUAD ? (lane & 16) : 0);      // the lane of body j in this lane's environment
            f3 Swj = shfl3(Sw, src), Svj = shfl3(Sv, src);
            if (j > 0) {
              a_L[my_vidx * DLP + tj] = dot(Swj, nn) + dot(Svj, ff);
              j = bodyi[BF_PARENT * nbp + j];
              tj--;
            }
          }
        }
        __syncwarp();
        if (prof_a) prof_a[3] = (unsigned)clock64();
      }
      if constexpr (QUAD) {
        if (pair_a != 0) asm volatile("bar.sync %0, 64;" ::"r"(2 + (warp & 3) + 4 * (warp >> 3)) : "memory");   // the pair's stage A is done
        O = mk(s_gc[0], s_gc[1], s_gc[2]);   // this warp's own base (= p of the base lane in stage A)
      }
      if (args.prof && lane == 0) args.prof[((size_t)env * 4 + (sub & 3)) * 8 + 1] = (unsigned)clock64();
      if (args.dbg_M)   // getters (integrate1): cold path, kept out of line to spare the instruction cache
        write_debug(args, env, lane, nv, nb, nvp, DLP, s_L, s_h, ddepth, danc, bvalid, s_pose, nbp);
      if (args.phase_mask & PHASE_KINEMATICS) { asm volatile("cp.async.wait_all;" ::: "memory"); __syncwarp(); break; }   // kinematics for the getters only

      // =========================== stage B: narrow phase ========================================
      K = stage_b_narrow_phase<SLOTS, SELF>(args.ter, s_ter, blob_s, s_pose, s_ct, s_Y, env, lane, nbp, args.prof ? args.prof + ((size_t)env * 4 + (sub & 3)) * 8 : nullptr);
      const int C = 3 * K;
      if (args.prof && lane == 0) args.prof[((size_t)env * 4 + (sub & 3)) * 8 + 2] = (unsigned)clock64();
      if (args.phase_mask & PHASE_NO_UPDATE) { asm volatile("cp.async.wait_all;" ::: "memory"); __syncwarp(); break; }   // integrate1(): kinematics, collision, M, h only

      // =========================== stage C: b, Mhat = L^T L, z, Y, G ==============================
      // a9 joint limits: the first LMAX joints found beyond their URDF limit become unilateral rows sign * qdot >= target
      int Lm = 0;
      if (args.prm.joint_limits) {
        float q = 0.f, lo = -3.0e38f, hi = 3.0e38f;
        if (bvalid && b > 0) { q = s_gc[bodyi[BF_QIDX * nbp + b]]; lo = bodyf[BF_LO * nbp + b]; hi = bodyf[BF_HI * nbp + b]; }
        const bool act = q < lo || q > hi;
        const unsigned lm_mask = __ballot_sync(FULL, act);
        const int slot = __popc(lm_mask & ((1u << lane) - 1u));
        if (act && slot < LMAX) {
          s_lim[4 * slot + 0] = __int_as_float(MYB(BF_VIDX));
          s_lim[4 * slot + 1] = q < lo ? 1.f : -1.f;
          s_lim[4 * slot + 2] = q < lo ? lo - q : q - hi;
        }
        Lm = min(__popc(lm_mask), LMAX);
        __syncwarp();
      }
      const int C3 = C, CR = C3 + Lm;   // contact rows, all constraint rows
      if (sub == 0 && (args.use_pd || DL)) {     // the asynchronous target fetch of the prologue lands here
        asm volatile("cp.async.wait_all;" ::: "memory");
        __syncwarp();
        if (args.pt_store) {
#pragma unroll 1
          for (int i = lane; i < nq; i += 32) args.pt_store[(size_t)env * args.gc_stride + i] = s_pt[i];
        }
        if (args.vt_store) {
#pragma unroll 1
          for (int i = lane; i < nv; i += 32) args.vt_store[(size_t)env * args.gv_stride + i] = s_vt[i];
        }
      }
      // actuation delay: the commanded rows were stored above; from here on s_pt, s_vt and s_tau hold the applied command
      if constexpr (DL) actuation_delay(args.delay_state, args.delay_ring, env, sub, nbase, nv, dofq, s_pt, s_vt, s_tau, lane);
      // actuator network: a listed dof has no PD law and the feed-forward torque tau_ff + net, its network torque kept in s_vt (its
      // velocity target, which it does not use; reloaded by every launch) for stage E.  Scratch: the Anderson history of stage D
      if constexpr (AN) {
        if (args.an.lstm) actuator_lstm(args.an, env, lane, s_gc, s_gv, s_pt, dofq, s_hist, s_vt);
        else actuator_network(args.an, env, lane, s_gc, s_gv, s_pt, dofq, s_hist, s_vt);
        __syncwarp();
      }
#pragma unroll 1
      for (int i = lane; i < nv; i += 32) {
        const bool an = AN && ((args.an.mask >> i) & 1ull);
        const float tff = an ? s_tau[i] + s_vt[i] : s_tau[i];
        float bi = tff - s_h[i];
        // actuator effort limit (oracle step()): when feed-forward + PD law at the current state exceed it, the joint is driven by the
        // constant limit torque over this step and gets no implicit PD terms
        float te = tff;
        float kpi, kdi, emi;
        dof_actuator(args, gain, nvp, env, nv, i, kpi, kdi, emi);
        if (an) { kpi = 0.f; kdi = 0.f; }
        const bool pd = kpi != 0.f || kdi != 0.f;
        const int qi = pd ? dofq[i] : 0;
        if (pd) te += kpi * (s_pt[qi] - s_gc[qi]) + kdi * (s_vt[i] - s_gv[i]);
        // ... judged on the torque the implicit law would really apply (the explicit value over 1 + (dt kd + dt^2 kp) / M_dd)
        const float soft = args.prm.dt * kdi + args.prm.dt * args.prm.dt * kpi;
        const bool sat = fabsf(te) > emi * (1.f + soft / s_L[i * DLP + ddepth[i]]);
        s_sat[i] = sat ? 1.f : 0.f;          // remembered for stage E (generalized force applied)
        if (sat) bi += copysignf(emi, te) - tff;
        else if (pd) {
          bi += kpi * (s_pt[qi] - s_gc[qi] - args.prm.dt * s_gv[i]) + kdi * (s_vt[i] - s_gv[i]);
          s_L[i * DLP + ddepth[i]] += args.prm.dt * kdi + args.prm.dt * args.prm.dt * kpi;
        }
        s_b[i] = bi;
      }
      __syncwarp();
      if constexpr (QUAD) {
        // ---- Mhat = L^T L with the topology compiled in: leg blocks in registers (quad_factor_legs), base block by 21 lanes
        static_assert(!QUAD || make_blob_header(SD, 0, 0).dlp == QDLP, "compact row stride");
        const QuadLeg ql = quad_factor_legs(s_L, s_invd, lane);
        __syncwarp();
        const int er = s_tri[lane] & 7, ec = s_tri[lane] >> 3;
        float val = 0.f;
        if (lane < 21) {
          val = s_L[er * QDLP + ec];
#pragma unroll
          for (int k = 6; k < 18; k++) val -= s_L[k * QDLP + er] * s_L[k * QDLP + ec];
        }
#pragma unroll
        for (int i = 5; i >= 0; i--) {
          const int ti = i * (i + 1) / 2;
          const float dd = __shfl_sync(FULL, val, ti + i);
          const float inv = rsqrt_nr(dd);
          if (er == i) val = (ec == i) ? dd * inv : val * inv;
          const float lir = __shfl_sync(FULL, val, ti + min(er, i));
          const float lic = __shfl_sync(FULL, val, ti + min(ec, i));
          if (lane < 21 && er < i) val -= lir * lic;
          if (lane == 0) s_invd[i] = inv;
        }
        if (lane < 21) s_L[er * QDLP + ec] = val;
        // ---- z = L^-T b: the three chain dofs of a leg in registers, then the base against every leg
        const int leg = lane >> 3, t = lane & 7, rA = 6 + 3 * leg;
        const float zK = s_b[rA + 2] * ql.i8;
        const float zH = (s_b[rA + 1] - ql.k7 * zK) * ql.i7;
        const float zA = (s_b[rA] - ql.h6 * zH - ql.k6 * zK) * ql.i6;
        if (t == 0) { s_z[rA] = zA; s_z[rA + 1] = zH; s_z[rA + 2] = zK; }
        float part = t < 6 ? ql.k * zK + ql.h * zH + ql.a * zA : 0.f;     // this leg's share of sum_k L[k][t] z_k
        part += __shfl_xor_sync(FULL, part, 8);
        part += __shfl_xor_sync(FULL, part, 16);
        __syncwarp();          // the base block and invd[0..5] written above are read below
        float acc = lane < 6 ? s_b[lane] - part : 0.f;
#pragma unroll
        for (int i = 5; i >= 0; i--) {
          const float zi = __shfl_sync(FULL, acc, i) * s_invd[i];
          if (lane < i) acc -= s_L[i * QDLP + lane] * zi;
          if (lane == i) s_z[i] = zi;
        }
        __syncwarp();
      } else {
        // ---- branch-sparse factorisation Mhat = L^T L, "pull" form, one dof-tree level at a time (deepest first):
        //      L[i][t] = (M[i][t] - sum_{k in subtree(i), k != i} L[k][depth i] L[k][t]) / L[i][i]
  #pragma unroll 1
        for (int lev = maxdd; lev >= nbase; lev--) {
          const int e0 = entstart[lev], ne = entstart[lev + 1] - e0;
  #pragma unroll 1
          for (int e = lane; e < ne; e += 32) {
            const int pk = ent[e0 + e], i = pk & 255, t = pk >> 8;
            float acc = s_L[i * DLP + t];
            const int kend = i + dsub[i];
  #pragma unroll (UNR)
            for (int k = i + 1; k < kend; k++) acc -= s_L[k * DLP + lev] * s_L[k * DLP + t];
            s_L[i * DLP + t] = acc;
          }
          __syncwarp();
          const int d0 = lvl[lev], nd = lvl[lev + 1] - d0;
          if (lane < nd) {
            const int i = lvldofs[d0 + lane];
            float d = sqrtf(s_L[i * DLP + lev]);
            s_L[i * DLP + lev] = d;
            s_invd[i] = 1.0f / d;
          }
          __syncwarp();
  #pragma unroll 1
          for (int e = lane; e < ne; e += 32) {
            const int pk = ent[e0 + e], i = pk & 255, t = pk >> 8;
            if (t < lev) s_L[i * DLP + t] *= s_invd[i];
          }
          __syncwarp();
        }
        if (floating) {   // base 6x6 block: every other dof is a descendant of every base dof
          const int er = s_tri[lane] & 7, ec = s_tri[lane] >> 3;
          float val = 0.f;
          if (lane < 21) {
            val = s_L[er * DLP + ec];
  #pragma unroll 4
            for (int k = 6; k < nv; k++) val -= s_L[k * DLP + er] * s_L[k * DLP + ec];
          }
  #pragma unroll 1
          for (int i = 5; i >= 0; i--) {
            const int ti = i * (i + 1) / 2;
            float d = sqrtf(__shfl_sync(FULL, val, ti + i));
            float inv = 1.0f / d;
            if (er == i) val = (ec == i) ? d : val * inv;
            float lir = __shfl_sync(FULL, val, ti + min(er, i));
            float lic = __shfl_sync(FULL, val, ti + min(ec, i));
            if (lane < 21 && er < i) val -= lir * lic;
            if (lane == 0) s_invd[i] = inv;
          }
          if (lane < 21) s_L[er * DLP + ec] = val;
          __syncwarp();
        }
        // ---- z = L^-T b  (leaves to root)
  #pragma unroll 1
        for (int lev = maxdd; lev >= nbase; lev--) {
          const int d0 = lvl[lev], nd = lvl[lev + 1] - d0;
          if (lane < nd) {
            const int i = lvldofs[d0 + lane];
            float acc = s_b[i];
            const int kend = i + dsub[i];
  #pragma unroll (UNR)
            for (int k = i + 1; k < kend; k++) acc -= s_L[k * DLP + lev] * s_z[k];
            s_z[i] = acc * s_invd[i];
          }
          __syncwarp();
        }
        if (floating) {
          float acc = 0.f;
          if (lane < 6) {
            acc = s_b[lane];
  #pragma unroll 4
            for (int k = 6; k < nv; k++) acc -= s_L[k * DLP + lane] * s_z[k];
          }
  #pragma unroll 1
          for (int i = 5; i >= 0; i--) {
            float zi = __shfl_sync(FULL, acc, i) * s_invd[i];
            if (lane < i) acc -= s_L[i * DLP + lane] * zi;
            if (lane == i) s_z[i] = zi;
          }
          __syncwarp();
        }
      }
      // ---- Y = L^-T J^T, one constraint row per lane, only along the row's own ancestor chain
      float u_c = 0.f;
      int row_lm = 5;          // QUAD: (leg << 4) | depth of this lane's row (chain = base dofs 0..5, then 3 leg + t for t = 6..depth)
      if constexpr (QUAD) {
        if (lane < CR) {
          const int c = lane;
          const bool is_lim = c >= C3;
          const float* ct = s_ct + (is_lim ? 0 : c / 3) * CT_WORDS;
          const float* lm = s_lim + 4 * (is_lim ? c - C3 : 0);
          const int d = c % 3;
          const int fo = (d == 0) ? CF_T1 : (d == 1 ? CF_T2 : CF_N);
          const f3 axd = mk(ct[fo], ct[fo + 1], ct[fo + 2]);
          const f3 pos = mk(ct[CF_POS], ct[CF_POS + 1], ct[CF_POS + 2]);
          const int i0 = is_lim ? __float_as_int(lm[0]) : 5 + __float_as_int(ct[CF_BODY]);   // body b >= 1 carries dof 5 + b; the base "dof" is 5
          const int leg = i0 >= 6 ? (i0 - 6) / 3 : 0;
          const int m = i0 >= 6 ? i0 - 3 * leg : 5;                                           // depth of that dof in the dof tree
          row_lm = (leg << 4) | m;
          float y[9];
          float jv;
          if (is_lim) {   // J = sign * e_dof
#pragma unroll
            for (int t = 0; t < 9; t++) y[t] = (t == m) ? lm[1] : 0.f;
            jv = lm[1] * s_gv[i0];
          } else {
            const f3 rc = cross(pos - O, axd);
            y[0] = axd.x; y[1] = axd.y; y[2] = axd.z; y[3] = rc.x; y[4] = rc.y; y[5] = rc.z;
            jv = axd.x * s_gv[0] + axd.y * s_gv[1] + axd.z * s_gv[2] + rc.x * s_gv[3] + rc.y * s_gv[4] + rc.z * s_gv[5];
#pragma unroll
            for (int t = 6; t < 9; t++) {
              y[t] = 0.f;
              if (t <= m) {
                const int j = 3 * leg + t - 5;         // body of chain dof 3 leg + t
                const f3 aj = mk(s_pose[(PF_A + 0) * nbp + j], s_pose[(PF_A + 1) * nbp + j], s_pose[(PF_A + 2) * nbp + j]);
                f3 col = aj;
                if (bodyi[BF_JTYPE * nbp + j] == 1) {
                  const f3 pj = mk(s_pose[(PF_P + 0) * nbp + j], s_pose[(PF_P + 1) * nbp + j], s_pose[(PF_P + 2) * nbp + j]);
                  col = cross(aj, pos - pj);
                }
                y[t] = dot(col, axd);
                jv += y[t] * s_gv[3 * leg + t];
              }
            }
          }
          float yz = 0.f;
#pragma unroll
          for (int sI = 8; sI >= 0; sI--) {
            if (sI <= m) {
              const int a_s = sI < 6 ? sI : 3 * leg + sI;
              const float ys = y[sI] * s_invd[a_s];
              y[sI] = ys;
              yz += ys * s_z[a_s];
#pragma unroll
              for (int t = 0; t < sI; t++) y[t] -= s_L[a_s * QDLP + t] * ys;
            }
          }
#pragma unroll
          for (int t = 0; t < 9; t++) if (t <= m) s_Y[t * CP + c] = y[t];
          u_c = jv + args.prm.dt * yz;
          // apply_row_bias, written out: calling it here changes this instance's code (the headline's) without saving anything
          if (is_lim) u_c -= args.prm.erp * lm[2] / args.prm.dt;
          else if (d == 2) {
            float target = args.prm.erp * ct[CF_DEPTH] / args.prm.dt;
            if (args.prm.restitution > 0.f && jv < -args.prm.rest_threshold) target += -args.prm.restitution * jv;
            u_c -= target;
          }
        }
      } else {
        if (lane < CR) {
          const int c = lane;
          const bool is_lim = c >= C3;
          const float* ct = s_ct + (is_lim ? 0 : c / 3) * CT_WORDS;
          const float* lm = s_lim + 4 * (is_lim ? c - C3 : 0);
          const int d = c % 3;
          const int fo = (d == 0) ? CF_T1 : (d == 1 ? CF_T2 : CF_N);
          const f3 axd = mk(ct[fo], ct[fo + 1], ct[fo + 2]);
          const f3 pos = mk(ct[CF_POS], ct[CF_POS + 1], ct[CF_POS + 2]);
          const int i0 = is_lim ? __float_as_int(lm[0]) : bdof[__float_as_int(ct[CF_BODY])];
          const int m = i0 >= 0 ? ddepth[i0] : -1;
          float jv = 0.f, yz;
          if (is_lim) {   // J = sign * e_dof
  #pragma unroll 1
            for (int t = 0; t < m; t++) s_Y[t * CP + c] = 0.f;
            s_Y[m * CP + c] = lm[1];
            jv = lm[1] * s_gv[i0];
          }
          chain_column<UNR>(s_Y, c, !is_lim, pos, axd, O, i0, m, floating, nbase, nvp, DLP, nbp, danc, dbody, bodyi, s_pose, s_gv, s_L, s_invd, s_z, jv, yz);
          u_c = jv + args.prm.dt * yz;
          if constexpr (SELF) {
            // self contact: the column is Y_first - Y_second; the second half (the second body's chain column at the same point, base
            // columns included) goes to its own block s_Y2, and u_c, the relative velocity jv, are differences of the two halves.  A body
            // welded to the world (fixed base only) has no dof: m = -1 and no base columns, a zero column.
            const int pair = __float_as_int(ct[CF_PAIR]);
            if (!is_lim && pair < 0) {
              float* s_Y2 = ws + args.ws.words - self_y_words(maxdd);
              const int i2 = bdof[-1 - pair];
              float jv2 = 0.f, yz2;
              chain_column<1>(s_Y2, c, true, pos, axd, O, i2, i2 >= 0 ? ddepth[i2] : -1, floating, nbase, nvp, DLP, nbp, danc, dbody, bodyi, s_pose, s_gv,
                              s_L, s_invd, s_z, jv2, yz2);
              u_c -= jv2 + args.prm.dt * yz2;
              jv -= jv2;
            }
          }
          apply_row_bias(u_c, args.prm, is_lim, d, lm, ct, jv);
        }
      }
      iters = 0; resid = 0.f; gs_status = RSB_SOLVER_CONVERGED;
      if (CR > 0) {
        __syncwarp();      // h / b / poses are dead from here: G overlays them
        // G = Y^T Y; rows a, b share ancestors exactly up to the depth of their bodies' LCA
        if constexpr (QUAD) {
          const int ng = 32 / CR;
          const int a = lane % CR, g = lane / CR;
          const int pa = __shfl_sync(FULL, row_lm, a);
          const int nit = (CR / 2 + ng) / ng;              // ceil((CR / 2 + 1) / ng): every lane runs the same trip count (warp-wide shuffle inside)
#pragma unroll 1
          for (int itr = 0; itr < nit; itr++) {
            const int dd = g + itr * ng;
            const bool active = g < ng && dd <= CR / 2;
            int bcol = a + dd; if (bcol >= CR) bcol -= CR;
            if (!active) bcol = 0;
            const int pb = __shfl_sync(FULL, row_lm, bcol);
            // same leg: the chains agree down to the shallower of the two; different legs (or a base row): the six base dofs only
            const int tmax = ((pa ^ pb) >> 4) == 0 ? min(pa & 15, pb & 15) : 5;
            if (active) {
              float sacc = 0.f;
#pragma unroll
              for (int t = 0; t < 9; t++) if (t <= tmax) sacc += s_Y[t * CP + a] * s_Y[t * CP + bcol];
              s_G[a * GP + bcol] = sacc; s_G[bcol * GP + a] = sacc;
            }
          }
        } else {
          {
            const int ng = 32 / CR;                   // CR <= 28 -> ng >= 1
            const int a = lane % CR, g = lane / CR;
            if (g < ng) {
              const int ba = a < C3 ? __float_as_int(s_ct[(a / 3) * CT_WORDS + CF_BODY]) : dbody[__float_as_int(s_lim[4 * (a - C3)])];
  #pragma unroll 1
              for (int dd = g; dd <= CR / 2; dd += ng) {
                int bcol = a + dd; if (bcol >= CR) bcol -= CR;
                const int bbody = bcol < C3 ? __float_as_int(s_ct[(bcol / 3) * CT_WORDS + CF_BODY]) : dbody[__float_as_int(s_lim[4 * (bcol - C3)])];
                const int tmax = lcad[ba * nbp + bbody];
                float sacc = 0.f;
  #pragma unroll (UNR)
                for (int t = 0; t <= tmax; t++) sacc += s_Y[t * CP + a] * s_Y[t * CP + bcol];
                if constexpr (SELF) {
                  // self contacts: G_ab = (Y1_a - Y2_a) . (Y1_b - Y2_b), each product along the two chains' common part (lcad)
                  if (H.npairs > 0) {
                    const float* s_Y2 = ws + args.ws.words - self_y_words(maxdd);
                    const int pa = a < C3 ? __float_as_int(s_ct[(a / 3) * CT_WORDS + CF_PAIR]) : 0;
                    const int pb = bcol < C3 ? __float_as_int(s_ct[(bcol / 3) * CT_WORDS + CF_PAIR]) : 0;
                    if (pa < 0) {
                      const int t2 = lcad[(-1 - pa) * nbp + bbody];
                      for (int t = 0; t <= t2; t++) sacc -= s_Y2[t * CP + a] * s_Y[t * CP + bcol];
                    }
                    if (pb < 0) {
                      const int t2 = lcad[ba * nbp + (-1 - pb)];
                      for (int t = 0; t <= t2; t++) sacc -= s_Y[t * CP + a] * s_Y2[t * CP + bcol];
                    }
                    if (pa < 0 && pb < 0) {
                      const int t2 = lcad[(-1 - pa) * nbp + (-1 - pb)];
                      for (int t = 0; t <= t2; t++) sacc += s_Y2[t * CP + a] * s_Y2[t * CP + bcol];
                    }
                  }
                }
                s_G[a * GP + bcol] = sacc; s_G[bcol * GP + a] = sacc;
              }
            }
          }
        }
        __syncwarp();
        // per-contact constants: symmetric 3x3 block, friction and the block's inverse (lane i < K computes, all read)
        if (lane < K) {
          const int i3 = 3 * lane;
          float a = s_G[i3 * GP + i3], bq = s_G[i3 * GP + i3 + 1], cc = s_G[i3 * GP + i3 + 2];
          float d = s_G[(i3 + 1) * GP + i3 + 1], e = s_G[(i3 + 1) * GP + i3 + 2], f = s_G[(i3 + 2) * GP + i3 + 2];
          float c00 = d * f - e * e, c01 = cc * e - bq * f, c02 = bq * e - cc * d;
          float c11 = a * f - cc * cc, c12 = bq * cc - a * e, c22 = a * d - bq * bq;
          float id = 1.0f / (a * c00 + bq * c01 + cc * c02);
          float* o = s_u + CB_WORDS * lane;
          float pm;
          const int cand = __float_as_int(s_ct[lane * CT_WORDS + CF_PT]);
          if constexpr (SELF) {   // a self contact (candidate npts + j) takes the friction of its pair
            pm = cand < H.npts ? ptsf[5 * H.nptp + cand] : reinterpret_cast<const float*>(blob_s + H.off_pair)[PAIR_WORDS * (cand - H.npts) + PR_MU];
          } else {
            pm = ptsf[5 * H.nptp + cand];
          }
          if (args.contact_friction && (!SELF || cand < H.npts)) {   // this environment's row for the candidate's collision body, if >= 0
            const float pe = args.contact_friction[(size_t)env * H.ncoll + reinterpret_cast<const int*>(ptsf)[10 * H.nptp + cand]];
            if (pe >= 0.f) pm = pe;
          }
          o[0] = a; o[1] = bq; o[2] = cc; o[3] = d; o[4] = e; o[5] = f;
          o[6] = pm >= 0.f ? pm : args.prm.mu;     // per-collision-body friction (World::setMaterialPairProp analogue)
          o[8] = c00 * id; o[9] = c01 * id; o[10] = c02 * id; o[11] = c11 * id; o[12] = c12 * id; o[13] = c22 * id;
        }
        __syncwarp();
        if (args.prof && lane == 0) args.prof[((size_t)env * 4 + (sub & 3)) * 8 + 3] = (unsigned)clock64();
        // =========================== stage D: per-contact Gauss-Seidel ===========================
        const GsResult gs = gs_solve(s_prm, s_G, GP, s_u, s_hist, sec_c, SEC_STRIDE, lane, K, Lm, u_c);
        iters = gs.iters; resid = gs.resid; gs_status = gs.status;
        if (lane < CR) s_lam[lane] = gs.lam;
        __syncwarp();
      }
      __syncwarp();
      if (args.prof && lane == 0) args.prof[((size_t)env * 4 + (sub & 3)) * 8 + 4] = (unsigned)clock64();
      // =========================== stage E: v+ = v + L^-1 (dt z + Y lam), integration ============
      if constexpr (QUAD) {
        // w_i = dt z_i + sum over the rows whose chain holds dof i of Y[depth i][row] lam_row, lane = dof
        const int i = min(lane, 17);
        const int legi = i >= 6 ? (i - 6) / 3 : 0, di = i >= 6 ? i - 3 * legi : i;
        float sacc = args.prm.dt * s_z[i];
#pragma unroll 1
        for (int k = 0; k < K; k++) {
          const int pr = __shfl_sync(FULL, row_lm, 3 * k);
          if (i < 6 || ((pr >> 4) == legi && (pr & 15) >= di))
            sacc += s_Y[di * CP + 3 * k] * s_lam[3 * k] + s_Y[di * CP + 3 * k + 1] * s_lam[3 * k + 1] + s_Y[di * CP + 3 * k + 2] * s_lam[3 * k + 2];
        }
#pragma unroll 1
        for (int l = 0; l < Lm; l++) {
          const int pr = __shfl_sync(FULL, row_lm, C3 + l);
          if (i < 6 || ((pr >> 4) == legi && (pr & 15) >= di)) sacc += s_Y[di * CP + C3 + l] * s_lam[C3 + l];
        }
        // x = L^-1 w, root to leaves: the base chain by shuffles, then the three joints of every leg by shuffles from the parent lanes
        float acc = lane < 6 ? sacc : 0.f;
#pragma unroll
        for (int t = 0; t < 6; t++) {
          const float xt = __shfl_sync(FULL, acc, t) * s_invd[t];
          if (lane > t && lane < 6) acc -= s_L[lane * QDLP + t] * xt;
          if (lane == t) acc = xt;
        }
        // acc (lanes 0..5) = x of the base dofs
        float legacc = sacc;
#pragma unroll
        for (int t = 0; t < 6; t++) legacc -= s_L[i * QDLP + t] * __shfl_sync(FULL, acc, t);
        const int j = i >= 6 ? di - 6 : 0;
        const float inv = s_invd[i];
        const float x0 = legacc * inv;                                            // joint 0 of a leg
        const float xa1 = __shfl_up_sync(FULL, x0, 1);
        const float x1 = (legacc - s_L[i * QDLP + 6] * xa1) * inv;               // joint 1: parent = joint 0
        const float xa2 = __shfl_up_sync(FULL, x0, 2), xh2 = __shfl_up_sync(FULL, x1, 1);
        const float x2 = (legacc - s_L[i * QDLP + 6] * xa2 - s_L[i * QDLP + 7] * xh2) * inv;   // joint 2: ancestors = joints 0, 1
        if (lane < 18) s_rhs[lane] = lane < 6 ? acc : (j == 0 ? x0 : (j == 1 ? x1 : x2));
        __syncwarp();
      } else {
  #pragma unroll 1
        for (int i = lane; i < nv; i += 32) {   // w = dt z + Y lam, gathered per dof over the contacts whose chain holds it
          float sacc = args.prm.dt * s_z[i];
          const int di = ddepth[i];
          chain_gather<UNR, false>(sacc, s_Y, s_lam, s_ct, K, i, di, bdof, ddepth, danc, nvp);
          if constexpr (SELF) {
            // self contacts: the second body's half of the column with -lambda
            if (H.npairs > 0) chain_gather<1, true>(sacc, ws + args.ws.words - self_y_words(maxdd), s_lam, s_ct, K, i, di, bdof, ddepth, danc, nvp);
          }
  #pragma unroll 1
          for (int l = 0; l < Lm; l++) {
            const int i0 = __float_as_int(s_lim[4 * l]);
            if (ddepth[i0] >= di && danc[di * nvp + i0] == i) sacc += s_Y[di * CP + C3 + l] * s_lam[C3 + l];
          }
          s_rhs[i] = sacc;
        }
        __syncwarp();
        if (floating) {   // x = L^-1 w, root to leaves: base chain by shuffles, then one tree level at a time
          float acc = lane < 6 ? s_rhs[lane] : 0.f;
  #pragma unroll 1
          for (int t = 0; t < 6; t++) {
            float xt = __shfl_sync(FULL, acc, t) * s_invd[t];
            if (lane > t && lane < 6) acc -= s_L[lane * DLP + t] * xt;
            if (lane == t) s_rhs[t] = xt;
          }
          __syncwarp();
        }
  #pragma unroll 1
        for (int lev = nbase; lev <= maxdd; lev++) {
          const int d0 = lvl[lev], nd = lvl[lev + 1] - d0;
          if (lane < nd) {
            const int i = lvldofs[d0 + lane];
            float acc = s_rhs[i];
            // base dofs are ancestors of every other dof and are their own index: no ancestor lookup
  #pragma unroll
            for (int t = 0; t < 6; t++) if (t < nbase) acc -= s_L[i * DLP + t] * s_rhs[t];
  #pragma unroll (UNR)
            for (int t = nbase; t < lev; t++) acc -= s_L[i * DLP + t] * s_rhs[danc[t * nvp + i]];
            s_rhs[i] = acc * s_invd[i];
          }
          __syncwarp();
        }
      }
      if (args.imu_lin) {   // IMU readings (rsb_batch_set_imus): a launch-uniform branch
        if (lane < args.imu_n) imu_substep(args, env, sub, lane, bodyf, bodyi, anc, nbp, floating, (H.flags & 1) != 0, s_gc, s_gv, s_rhs);
        __syncwarp();       // every sensor lane has read v_s before the update below overwrites it
      }
#pragma unroll 1
      for (int i = lane; i < nv; i += 32) {
        const float v0 = s_gv[i], vp = v0 + s_rhs[i];
        s_gv[i] = vp;
        // generalized force applied over this step (implicit PD evaluated at q + dt v+, v+; the effort limit where it was hit): getGeneralizedForce()
        const bool an = AN && ((args.an.mask >> i) & 1ull);   // network dof: the explicit torque of stage C
        float ta = an ? s_tau[i] + s_vt[i] : s_tau[i];
        float kpi, kdi, emi;
        dof_actuator(args, gain, nvp, env, nv, i, kpi, kdi, emi);
        if (an) { kpi = 0.f; kdi = 0.f; }
        const bool pd = kpi != 0.f || kdi != 0.f;
        const int qi = pd ? dofq[i] : 0;
        float te = ta;
        if (pd) te += kpi * (s_pt[qi] - s_gc[qi]) + kdi * (s_vt[i] - v0);
        if (s_sat[i] != 0.f) ta = copysignf(emi, te);
        else if (pd) ta += kpi * (s_pt[qi] - s_gc[qi] - args.prm.dt * vp) + kdi * (s_vt[i] - vp);
        s_b[i] = ta;
      }
      __syncwarp();
      if (floating) {
        if (lane < 3) s_gc[lane] += args.prm.dt * s_gv[lane];
        f3 wn = mk(s_gv[3], s_gv[4], s_gv[5]);
        float wnorm = sqrtf(dot(wn, wn)), ang = wnorm * args.prm.dt;
        float qw, qx, qy, qz;
        if (ang > 1e-10f) { float sh, ch; sincosf(0.5f * ang, &sh, &ch); float s = sh / wnorm; qw = ch; qx = s * wn.x; qy = s * wn.y; qz = s * wn.z; }
        else { qw = 1.f; qx = 0.5f * args.prm.dt * wn.x; qy = 0.5f * args.prm.dt * wn.y; qz = 0.5f * args.prm.dt * wn.z; }
        float pw = s_gc[3], px = s_gc[4], py = s_gc[5], pz = s_gc[6];
        float nw = qw * pw - qx * px - qy * py - qz * pz;
        float nx = qw * px + qx * pw + qy * pz - qz * py;
        float ny = qw * py - qx * pz + qy * pw + qz * px;
        float nz = qw * pz + qx * py - qy * px + qz * pw;
        float inv = 1.0f / sqrtf(nw * nw + nx * nx + ny * ny + nz * nz);
        __syncwarp();
        if (lane == 0) { s_gc[3] = nw * inv; s_gc[4] = nx * inv; s_gc[5] = ny * inv; s_gc[6] = nz * inv; }
      }
#pragma unroll 1
      for (int i = lane; i < nv; i += 32) {
        int qi = dofq[i];
        if (qi >= (floating ? 7 : 0)) s_gc[qi] += args.prm.dt * s_gv[i];
      }
      __syncwarp();
      if (args.cf_force && lane < args.cf_n) {
        // contact forces per body: lane s adds this sub-step's world impulses on body cf_body[s], formed as the contact records form
        // them, in list order (+ on a contact's own body, - on the second body of a self contact).  The accumulator is the
        // environment's own output row, which only this lane touches: stored at the first sub-step, read back and added to at the
        // later ones, turned into the mean force at the last.  Nothing is carried in a register across the sub-step loop.
        const int body = args.cf_body[lane];
        float* fo = args.cf_force + ((size_t)env * args.cf_n + lane) * 3;
        int* so = args.cf_steps + (size_t)env * args.cf_n + lane;
        float ax = 0.f, ay = 0.f, az = 0.f;
        int hit = 0;
        if (sub > 0) { ax = fo[0]; ay = fo[1]; az = fo[2]; hit = *so; }   // issued before the walk over the contacts, which hides the L2 round trip
        float fx = 0.f, fy = 0.f, fz = 0.f;
        bool any = false;
#pragma unroll 2
        for (int k = 0; k < K; k++) {
          const float* ct = s_ct + k * CT_WORDS;
          const int pr = __float_as_int(ct[CF_PAIR]);
          const bool first = __float_as_int(ct[CF_BODY]) == body, second = pr < 0 && -1 - pr == body;
          const float lx = s_lam[3 * k], ly = s_lam[3 * k + 1], lz = s_lam[3 * k + 2];
          const float ix = ct[CF_T1] * lx + ct[CF_T2] * ly + ct[CF_N] * lz;
          const float iy = ct[CF_T1 + 1] * lx + ct[CF_T2 + 1] * ly + ct[CF_N + 1] * lz;
          const float iz = ct[CF_T1 + 2] * lx + ct[CF_T2 + 2] * ly + ct[CF_N + 2] * lz;
          fx += first ? ix : (second ? -ix : 0.f); fy += first ? iy : (second ? -iy : 0.f); fz += first ? iz : (second ? -iz : 0.f);
          any |= first || second;
        }
        fx = ax + fx; fy = ay + fy; fz = az + fz; hit += any ? 1 : 0;
        if (sub == args.substeps - 1) { const float s = 1.0f / ((float)args.substeps * args.prm.dt); fx *= s; fy *= s; fz *= s; }
        fo[0] = fx; fo[1] = fy; fo[2] = fz; *so = hit;
      }
      if (args.prof && lane == 0) args.prof[((size_t)env * 4 + (sub & 3)) * 8 + 5] = (unsigned)clock64();
    }   // substeps

    if (args.gym_action) {
      // ENVIRONMENT::step() second half + isTerminalState() + reset(), same arithmetic as the stand-alone task kernel it replaces:
      // reward = torque_coeff |tau|^2 + forward_vel_coeff min(4, body-frame x velocity); any contact on a non-foot body ends the episode
      float qw = s_gc[3], qx = s_gc[4], qy = s_gc[5], qz = s_gc[6];
      const float inv = 1.0f / sqrtf(qw * qw + qx * qx + qy * qy + qz * qz);
      qw *= inv; qx *= inv; qy *= inv; qz *= inv;
      const float r00 = 1.f - 2.f * (qy * qy + qz * qz), r10 = 2.f * (qx * qy + qw * qz), r20 = 2.f * (qx * qz - qw * qy);
      const float vbx = r00 * s_gv[0] + r10 * s_gv[1] + r20 * s_gv[2];
      float t2 = 0.f;
#pragma unroll 1
      for (int i = lane; i < nv; i += 32) t2 += s_b[i] * s_b[i];          // s_b: generalized force applied in the last sub-step (stage E)
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) t2 += __shfl_xor_sync(FULL, t2, o);
      bool bad = false;
      if (lane < K) bad = ((args.gym.foot_mask >> __float_as_int(s_ct[lane * CT_WORDS + CF_BODY])) & 1u) == 0u;
      const bool term = __any_sync(FULL, bad);
      float r = args.gym.torque_coeff * t2 + args.gym.forward_vel_coeff * fminf(4.0f, vbx);
      __syncwarp();
      if (term) {
        r += args.gym.terminal_reward;
#pragma unroll 1
        for (int i = lane; i < nq; i += 32) { const float g0 = args.gym.gc_init[i]; s_gc[i] = g0; if (args.pt_store) args.pt_store[(size_t)env * args.gc_stride + i] = g0; }
#pragma unroll 1
        for (int i = lane; i < nv; i += 32) s_gv[i] = args.gym.gv_init[i];
        if constexpr (AN) {
          const int hw = args.an.words;
#pragma unroll 1
          for (int i = lane; i < hw; i += 32) args.an.hist[(size_t)env * hw + i] = 0.f;
        }
        if (DL && lane == 0) args.delay_state[2 * env + 1] = 0;   // the command history is emptied, the delay kept
      }
      if (lane == 0) { args.gym_reward[env] = r; args.gym_done[env] = term ? 1 : 0; }
      __syncwarp();
    }
    // ---- store state rows and contact records -----------------------------------------------------
    if (!(args.phase_mask & PHASE_NO_UPDATE)) {
      float* g_gc = args.gc + (size_t)env * args.gc_stride;
      float* g_gv = args.gv + (size_t)env * args.gv_stride;
#pragma unroll 1
      for (int i = lane; i < nq; i += 32) g_gc[i] = s_gc[i];
#pragma unroll 1
      for (int i = lane; i < nv; i += 32) { g_gv[i] = s_gv[i]; args.tau_applied[(size_t)env * args.gv_stride + i] = s_b[i]; }
    }
    if (args.obs && floating) {   // VectorizedEnvironment::observe() fused into the step
      const float* o = write_obs_row(args.obs, args.ob_dim, env, s_gc, s_gv, nq, lane);
      if (args.peer_world > 0) {   // fused all-gather: the finished row goes to every GPU of the job (this one included) over NVLink
        __syncwarp();
        const size_t row = ((size_t)args.peer_rank * args.num_envs + env) * args.ob_dim;
#pragma unroll 1
        for (int i = lane; i < args.ob_dim; i += 32) {
          const float v = o[i];                                          // re-read of this warp's own row (L2 hit), once for all peers
#pragma unroll 1
          for (int pr = 0; pr < args.peer_world; pr++) args.peer_obs[pr][row + i] = v;
        }
      }
    }
    if (args.phase_mask & PHASE_KINEMATICS) { __syncwarp(); continue; }   // kinematics only: contact records, iteration counts and flags of the last integrate() stay
    {   // failure detection: a non-finite coordinate or velocity marks the environment as diverged
      bool bad = false;
#pragma unroll 1
      for (int i = lane; i < nq; i += 32) bad |= !isfinite(s_gc[i]);
#pragma unroll 1
      for (int i = lane; i < nv; i += 32) bad |= !isfinite(s_gv[i]);
      const bool any_bad = __any_sync(FULL, bad);
      if (lane == 0) args.diverged[env] = any_bad ? 1 : 0;
    }
    if (lane == 0) { args.ncontacts[env] = K; args.iters[env] = iters; args.resid[env] = resid; args.solver_status[env] = gs_status; }
    if (lane < KMAX) {
      rsb_contact rc;
      int pt = -1;
      if (lane < K) {
        const float* ct = s_ct + lane * CT_WORDS;
        float lx = 0.f, ly = 0.f, lz = 0.f;
        if (!(args.phase_mask & PHASE_NO_UPDATE)) { lx = s_lam[3 * lane]; ly = s_lam[3 * lane + 1]; lz = s_lam[3 * lane + 2]; }
        rc.local_body = __float_as_int(ct[CF_BODY]); rc.pair_index = __float_as_int(ct[CF_PAIR]);
        pt = __float_as_int(ct[CF_PT]);
#pragma unroll
        for (int k = 0; k < 3; k++) {
          rc.position[k] = ct[CF_POS + k]; rc.normal[k] = ct[CF_N + k];
          rc.impulse[k] = ct[CF_T1 + k] * lx + ct[CF_T2 + k] * ly + ct[CF_N + k] * lz;
        }
        rc.depth = ct[CF_DEPTH];
      } else {
        rc.local_body = -1; rc.pair_index = -1; rc.depth = 0.f;
#pragma unroll
        for (int k = 0; k < 3; k++) { rc.position[k] = 0.f; rc.normal[k] = 0.f; rc.impulse[k] = 0.f; }
      }
      args.contacts[(size_t)env * KMAX + lane] = rc;
      args.contact_pt[(size_t)env * KMAX + lane] = pt;
    }
    __syncwarp();
  }
  if (args.peer_world > 0 && args.obs) {
    // every row this CTA stored must be visible on the peers before they see the arrival count: the CTA barrier orders the warps'
    // stores before the signalling threads, whose release at system scope is cumulative over them (one fence per signalling
    // thread instead of one per thread of the CTA)
    __syncthreads();
    if ((int)threadIdx.x < args.peer_world)
      asm volatile("red.release.sys.global.add.u32 [%0], %1;" ::"l"(args.peer_flag[threadIdx.x] + args.peer_rank), "r"(1u) : "memory");
    // the arrival wait folded into the launch: the last CTA to finish stays until every rank's rows of this step have landed in
    // THIS GPU's buffer, so the launch completes exactly when the gathered rows do (no separate wait kernel, no launch gap).
    // Bounded: a dead peer traps instead of hanging the GPU.
    __shared__ int s_last;
    if (threadIdx.x == 0) {
      const unsigned d = atomicAdd(args.peer_done, 1u);
      s_last = d == gridDim.x - 1 ? 1 : 0;
      if (s_last) *args.peer_done = 0u;           // every CTA has counted itself: ready for the next launch
    }
    __syncthreads();
    if (s_last && (int)threadIdx.x < args.peer_world) {
      const unsigned* f = args.peer_flag[args.peer_rank] + threadIdx.x;
      const long long t0 = clock64();
      for (;;) {
        unsigned v;
        asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(f) : "memory");
        if ((int)(v - args.peer_expected) >= 0) break;
        if (clock64() - t0 > 20000000000ll) __trap();
      }
    }
  }
}

}  // namespace rsb
