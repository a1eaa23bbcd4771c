// Observation row of the RaisimGym ANYmal locomotion task (SURVEY.md 8f N1, [RECALL]
// raisimGymTorch envs/rsg_anymal/Environment.hpp updateObservation()):
//   [ z | R^T e_z (3) | joint q | R^T v_base (3) | R^T w_base (3) | joint rates ]
// One warp per environment, coalesced row reads and writes; fixed-base models get [q | qdot].
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/rsb.h"

namespace rsb {

// write_obs_row: step_kernel.cuh (shared with the fused observation write)
__global__ void rsb_observe_kernel(const float* __restrict__ gc, const float* __restrict__ gv, int gc_stride, int gv_stride, int nq, int nv,
                                   int floating, int num_envs, float* __restrict__ obs, int ob_dim) {
  const int lane = threadIdx.x & 31;
  const int env = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (env >= num_envs) return;
  const float* q = gc + (size_t)env * gc_stride;
  const float* v = gv + (size_t)env * gv_stride;
  if (!floating) {
    float* o = obs + (size_t)env * ob_dim;
    for (int i = lane; i < nq; i += 32) o[i] = q[i];
    for (int i = lane; i < nv; i += 32) o[nq + i] = v[i];
    return;
  }
  write_obs_row(obs, ob_dim, env, q, v, nq, lane);
}

// external wrench rows for rsb_step_kernel (StepArgs::ext): [body | F(3) | T(3) | point in body frame(3) | pad(2)]
__global__ void rsb_ext_pack_kernel(float* rows, int body, const float* __restrict__ force, const float* __restrict__ torque, float px, float py, float pz,
                                    int count) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= count) return;
  float* r = rows + (size_t)e * EXT_WORDS;
  r[0] = __int_as_float(body);
  for (int k = 0; k < 3; k++) { r[1 + k] = force ? force[(size_t)e * 3 + k] : 0.f; r[4 + k] = torque ? torque[(size_t)e * 3 + k] : 0.f; }
  r[7] = px; r[8] = py; r[9] = pz; r[10] = 0.f; r[11] = 0.f;
}

// per-environment inertial rows (rsb_batch_set_body_inertia, StepArgs::body_inertia): `rows` tight rows of the caller [mass | com(3) |
// inertia xx xy xz yy yz zz] checked and repacked to BI_WORDS.  A refused row lowers *bad to row * 4 + reason (1 not finite, 2 negative
// mass, 3 inertia not positive semidefinite); *bad is left alone when every row is accepted.  PSD within a tolerance relative to the
// trace t: every principal minor of order k >= -eps t^k (double precision)
enum BodyInertiaFault { BI_NOT_FINITE = 1, BI_NEGATIVE_MASS = 2, BI_NOT_PSD = 3 };
__global__ void rsb_body_inertia_pack_kernel(float* __restrict__ out, const float* __restrict__ src, int rows, double eps, int* bad) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  float v[10];
  bool finite = true;
  for (int k = 0; k < 10; k++) { v[k] = src[(size_t)r * 10 + k]; finite = finite && isfinite(v[k]); }
  float* o = out + (size_t)r * BI_WORDS;
  for (int k = 0; k < 10; k++) o[k] = v[k];
  o[10] = 0.f; o[11] = 0.f;
  const double xx = v[4], xy = v[5], xz = v[6], yy = v[7], yz = v[8], zz = v[9], t = xx + yy + zz;
  const double m2 = eps * t * t;
  const bool psd = xx >= -eps * t && yy >= -eps * t && zz >= -eps * t && xx * yy - xy * xy >= -m2 && xx * zz - xz * xz >= -m2 && yy * zz - yz * yz >= -m2 &&
                   xx * (yy * zz - yz * yz) - xy * (xy * zz - yz * xz) + xz * (xy * yz - yy * xz) >= -m2 * t;
  const int fault = !finite ? BI_NOT_FINITE : !(v[0] >= 0.f) ? BI_NEGATIVE_MASS : !psd ? BI_NOT_PSD : 0;
  if (fault) atomicMin(bad, r * 4 + fault);
}

// per-environment terrain friction rows (rsb_batch_set_contact_friction, StepArgs::contact_friction): `n` values of the caller copied as
// they are.  A value that is NaN or +-inf lowers *bad to its index; *bad is left alone when every value is accepted
__global__ void rsb_contact_friction_check_kernel(float* __restrict__ out, const float* __restrict__ src, int n, int* bad) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float v = src[i];
  out[i] = v;
  if (!isfinite(v)) atomicMin(bad, i);
}

// per-environment actuator rows (rsb_batch_set_actuator_params, StepArgs::actuator): the caller's [envs][nv][3] (kp, kd, effort limit)
// repacked planar to [envs][3][nv], so that the lanes of a warp read one field of consecutive dofs.  The first `nbase` dofs (a floating
// base: not actuated) are stored as -1; an effort limit >= 0 is clamped to the blob's "none" value 3e38 (+inf: no limit).  NaN
// anywhere, +-inf in kp or kd and -inf in the effort limit lower *bad to (env * nv + dof) * 3 + field; *bad is left alone when every
// value is accepted
__global__ void rsb_actuator_params_check_kernel(float* __restrict__ out, const float* __restrict__ src, int envs, int nv, int nbase, int* bad) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= envs * nv) return;
  const int e = r / nv, i = r - e * nv;
  float* o = out + (size_t)e * 3 * nv + i;
  for (int f = 0; f < 3; f++) {
    float v = src[(size_t)r * 3 + f];
    const bool ok = f < 2 ? isfinite(v) : !isnan(v) && v != -INFINITY;
    if (!ok) atomicMin(bad, r * 3 + f);
    if (f == 2 && v >= 0.f) v = fminf(v, 3.0e38f);
    o[(size_t)f * nv] = i < nbase ? -1.f : v;
  }
}

// ---- frame kinematics (rsb_batch_set_frames / get_frame_states / get_frame_jacobians) ----------------------------------------------
// Frames rigidly attached to bodies and, per dof, what its Jacobian column needs; device arrays uploaded by rsb_batch_set_frames.
// A dof turns or slides along the axis a of its body k (a = R_k axis: the joint frame's rotation about its own axis leaves the axis
// where it is); the six dofs of a floating base are three slides and three turns about the world axes through the base origin, so
// one column rule serves both: revolute (a x (x - p_k), a), prismatic (a, 0).
enum FrameFlag { FRAME_AT_ORIGIN = 1, FRAME_IDENTITY = 2 };   // pos == 0 / rot == I exactly: the body pose is copied, bit for bit
enum DofKind { DOF_WORLD_AXIS = 4 };                          // added to JT_REVOLUTE / JT_PRISMATIC: dof_axis is in the world frame
struct FrameTable {
  int nf, nb, nv;
  const int* body;          // [nf] body index
  const int* flags;         // [nf] FrameFlag bits
  const float* pos;         // [nf][3] origin in the body frame
  const float* rot;         // [nf][9] row-major orientation in the body frame
  const int* dof_body;      // [nv] body whose joint carries the dof (the base for the base dofs)
  const int* dof_kind;      // [nv] JT_REVOLUTE / JT_PRISMATIC (+ DOF_WORLD_AXIS)
  const float* dof_axis;    // [nv][3] unit axis in the frame of dof_body (world frame with DOF_WORLD_AXIS)
  const unsigned* anc;      // [nb] bit k: body k is the body itself or one of its ancestors
};

// One warp per (environment, frame), lanes over the dof columns: the Jacobian rows are written coalesced, and the frame velocity is
// the warp sum of the same columns times gv, so lin_vel / ang_vel and J gv come from one routine.  Poses are the kinematics pass's
// (R [N][nb][9], P [N][nb][3]); outputs are tight rows of the environments [env_begin, env_begin + count) in (environment, frame)
// order; a null output is skipped.
__global__ void __launch_bounds__(128) rsb_frame_kernel(FrameTable ft, const float* __restrict__ R, const float* __restrict__ P,
                                                        const float* __restrict__ gv, int gv_stride, int env_begin, int count,
                                                        float* pos_out, float* rot_out, float* lin_out, float* ang_out, float* jac_out) {
  const int lane = threadIdx.x & 31;
  const long w = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;   // output row: (environment - env_begin) * nf + frame
  if (w >= (long)count * ft.nf) return;
  const int f = (int)(w % ft.nf);
  const long e = env_begin + w / ft.nf;
  const int b = ft.body[f], flags = ft.flags[f];
  const float* Rb = R + (e * ft.nb + b) * 9;
  const float* pb = P + (e * ft.nb + b) * 3;
  const float* fp = ft.pos + 3 * f;
  float x[3];
  #pragma unroll
  for (int k = 0; k < 3; k++) x[k] = (flags & FRAME_AT_ORIGIN) ? pb[k] : pb[k] + (Rb[3 * k] * fp[0] + Rb[3 * k + 1] * fp[1] + Rb[3 * k + 2] * fp[2]);
  if (pos_out && lane < 3) pos_out[w * 3 + lane] = lane == 0 ? x[0] : lane == 1 ? x[1] : x[2];
  if (rot_out && lane < 9) {
    const int i = lane / 3, j = lane % 3;
    const float* fr = ft.rot + 9 * f;
    rot_out[w * 9 + lane] = (flags & FRAME_IDENTITY) ? Rb[lane] : Rb[3 * i] * fr[j] + Rb[3 * i + 1] * fr[3 + j] + Rb[3 * i + 2] * fr[6 + j];
  }
  const unsigned anc = ft.anc[b];
  const float* v = gv + e * gv_stride;
  float lin[3] = {0.f, 0.f, 0.f}, ang[3] = {0.f, 0.f, 0.f};
  for (int c = lane; c < ft.nv; c += 32) {
    float jt[3] = {0.f, 0.f, 0.f}, jr[3] = {0.f, 0.f, 0.f};
    const int k = ft.dof_body[c];
    if ((anc >> k) & 1u) {
      const int kind = ft.dof_kind[c];
      const float* ax = ft.dof_axis + 3 * c;
      const float* Rk = R + (e * ft.nb + k) * 9;
      float a[3];
      #pragma unroll
      for (int q = 0; q < 3; q++) a[q] = (kind & DOF_WORLD_AXIS) ? ax[q] : Rk[3 * q] * ax[0] + Rk[3 * q + 1] * ax[1] + Rk[3 * q + 2] * ax[2];
      if ((kind & 3) == JT_REVOLUTE) {
        const float* pk = P + (e * ft.nb + k) * 3;
        const float d0 = x[0] - pk[0], d1 = x[1] - pk[1], d2 = x[2] - pk[2];
        jt[0] = a[1] * d2 - a[2] * d1; jt[1] = a[2] * d0 - a[0] * d2; jt[2] = a[0] * d1 - a[1] * d0;
        jr[0] = a[0]; jr[1] = a[1]; jr[2] = a[2];
      } else {
        jt[0] = a[0]; jt[1] = a[1]; jt[2] = a[2];
      }
    }
    const float vc = v[c];
    #pragma unroll
    for (int q = 0; q < 3; q++) { lin[q] += jt[q] * vc; ang[q] += jr[q] * vc; }
    if (jac_out) {
      float* J = jac_out + w * 6 * ft.nv + c;
      #pragma unroll
      for (int q = 0; q < 3; q++) { J[q * ft.nv] = jt[q]; J[(3 + q) * ft.nv] = jr[q]; }
    }
  }
  if (!lin_out && !ang_out) return;
  #pragma unroll
  for (int s = 16; s > 0; s >>= 1)
    #pragma unroll
    for (int q = 0; q < 3; q++) { lin[q] += __shfl_xor_sync(0xffffffffu, lin[q], s); ang[q] += __shfl_xor_sync(0xffffffffu, ang[q], s); }
  if (lane < 3) {
    if (lin_out) lin_out[w * 3 + lane] = lane == 0 ? lin[0] : lane == 1 ? lin[1] : lin[2];
    if (ang_out) ang_out[w * 3 + lane] = lane == 0 ? ang[0] : lane == 1 ? ang[1] : ang[2];
  }
}

}  // namespace rsb

// ---- RaisimGym ANYmal locomotion task on the device (SURVEY.md 8f N1; [RECALL] raisimGymTorch
//      envs/rsg_anymal/Environment.hpp + VectorizedEnvironment.hpp::perAgentStep) -----------------------
namespace rsb {

// GymConfig: step_kernel.cuh.  ENVIRONMENT::step() -- action -> PD targets, the sub-steps, reward, isTerminalState(), reset() of the
// terminated environments, observe() -- is ONE launch of rsb_step_kernel (StepArgs::gym_action); only reset() of the whole batch is a kernel here.

// ENVIRONMENT::reset() for every environment
__global__ void rsb_gym_reset_kernel(float* gc, float* gv, float* ptarget, float* vtarget, GymConfig cfg, int gc_stride, int gv_stride, int nq, int nv, int num_envs) {
  const int lane = threadIdx.x & 31;
  const int env = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (env >= num_envs) return;
  for (int i = lane; i < nq; i += 32) { gc[(size_t)env * gc_stride + i] = cfg.gc_init[i]; ptarget[(size_t)env * gc_stride + i] = cfg.gc_init[i]; }
  for (int i = lane; i < nv; i += 32) { gv[(size_t)env * gv_stride + i] = cfg.gv_init[i]; vtarget[(size_t)env * gv_stride + i] = 0.f; }
}

}  // namespace rsb
