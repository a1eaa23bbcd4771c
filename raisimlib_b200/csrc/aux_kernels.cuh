// Observation row of the RaisimGym ANYmal locomotion task (SURVEY.md 8f N1, [RECALL]
// raisimGymTorch envs/rsg_anymal/Environment.hpp updateObservation()):
//   [ z | R^T e_z (3) | joint q | R^T v_base (3) | R^T w_base (3) | joint rates ]
// One warp per environment, coalesced row reads and writes; fixed-base models get [q | qdot].
#pragma once
#include <cuda_runtime.h>
#include <climits>
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

// per-environment terrain friction rows (rsb_batch_set_contact_friction, StepArgs::contact_friction) and actuator history rows
// (rsb_batch_set_actuator_history, ActNetDesc::hist): `n` values of the caller copied as they are.  A value that is NaN or +-inf lowers
// *bad to its index; *bad is left alone when every value is accepted
__global__ void rsb_finite_rows_check_kernel(float* __restrict__ out, const float* __restrict__ src, int n, int* bad) {
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

// int32 entries of a range of environments: atlas map indices (rsb_batch_set_heightmap_index, TerrainDesc::env_map) and actuation
// delays (rsb_batch_set_actuation_delay): `n` entries of the caller copied as they are (out may be src: the check runs in place on a
// host source's staged copy).  An entry outside [lo, hi] lowers *bad to its position; *bad is left alone when every entry is accepted
__global__ void rsb_int_rows_check_kernel(int* out, const int* src, int n, int lo, int hi, int* bad) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int v = src[i];
  out[i] = v;
  if (v < lo || v > hi) atomicMin(bad, i);
}

// actuation delays of `n` environments (rsb_batch_set_actuation_delay) committed to their [n][2] (delay, sub-steps since the history
// was emptied) rows, StepArgs::delay_state: an entry d >= 0 sets the delay and empties the history, -1 leaves the row; delays == null
// sets 0 and empties every row
__global__ void rsb_actuation_delay_commit_kernel(int* state, const int* delays, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int d = delays ? delays[i] : 0;
  if (d >= 0) { state[2 * i] = d; state[2 * i + 1] = 0; }
}

// ordered-integer image of a float: signed integer order is the float order (-0 just below +0), so atomicMax on it takes the largest
// value whatever the order in which the threads arrive
__device__ __forceinline__ int float_order_key(float v) {
  const int i = __float_as_int(v);
  return i >= 0 ? i : i ^ 0x7fffffff;
}

// height maps replacing maps of the atlas (rsb_batch_update_heightmaps): `count` maps of `words` heights each, copied as they are (out
// may be src, as above); blockIdx.y strides over the maps, so any count runs on a grid of at most 65535 rows.  A value that is not finite
// lowers *bad to its position in the caller's array; the largest value of map m goes to map_max[m] as float_order_key (the caller starts
// it at INT_MIN).  One atomic per warp and map
__global__ void __launch_bounds__(256) rsb_heightmap_check_kernel(float* out, const float* src, int words, int count, int* bad, int* map_max) {
  for (int m = blockIdx.y; m < count; m += gridDim.y) {
    const size_t base = (size_t)m * words;
    int key = INT_MIN;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < words; i += gridDim.x * blockDim.x) {
      const float v = src[base + i];
      out[base + i] = v;
      if (isfinite(v)) key = max(key, float_order_key(v));
      else atomicMin(bad, (int)(base + i));
    }
    key = __reduce_max_sync(0xffffffffu, key);
    if ((threadIdx.x & 31) == 0 && key != INT_MIN) atomicMax(map_max + m, key);
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

// ---- terrain height scans (rsb_batch_set_height_scan / get_height_scan) ----------------------------------------------------------
// World z of the collision surface under (x, y), clamped to the nearest border point outside a height map as HeightMap::getHeight
// does.  Inside the map the float arithmetic is terrain_query's (step_kernel.cuh): the division by the pitch, fx >= fy picking the
// triangle, zt = h00 + sx fx + sy fy; so the scan reports the heights the narrow phase collides with.  A coordinate that is not finite
// gives NaN (clamping it would report a corner of the map for a diverged environment).
__device__ __forceinline__ float scan_surface_height(const TerrainDesc& t, int hm_offset, float x, float y) {
  if (!isfinite(x) || !isfinite(y)) return __int_as_float(0x7fffffff);
  if (t.type == 1) return t.ground_z;
  const float gx = fminf(fmaxf((x - t.x0) / t.dx, 0.f), t.xmax), gy = fminf(fmaxf((y - t.y0) / t.dy, 0.f), t.ymax);
  const int ix = min((int)gx, t.xs - 2), iy = min((int)gy, t.ys - 2);
  const float fx = gx - (float)ix, fy = gy - (float)iy;
  const float* H = t.h + hm_offset + iy * t.xs + ix;
  const float h00 = __ldg(H), h10 = __ldg(H + 1), h01 = __ldg(H + t.xs), h11 = __ldg(H + t.xs + 1);
  float sx, sy;
  if (fx >= fy) { sx = h10 - h00; sy = h11 - h10; }
  else { sx = h11 - h01; sy = h01 - h00; }
  return h00 + sx * fx + sy * fy;
}

// The points of rsb_batch_set_height_scan: body [RSB_MAX_SCAN_POINTS] | offsets xy [RSB_MAX_SCAN_POINTS][2], one device allocation.
struct ScanTable {
  int n, align;             // points, RSB_SCAN_YAW / RSB_SCAN_WORLD
  int root_from_gc;         // a floating base: points on body 0 take its pose from gc
  const int* body;
  const float* xy;
};

// One thread per (environment, point), in flat output order: height is written coalesced.  R [N][nb][9], P [N][nb][3]: the kinematics
// pass's poses (read only for points off a floating root); outputs are tight rows of the environments [env_begin, env_begin + count);
// a null output is skipped.
__global__ void __launch_bounds__(256) rsb_height_scan_kernel(ScanTable st, TerrainDesc ter, const float* __restrict__ gc, int gc_stride,
                                                              const float* __restrict__ R, const float* __restrict__ P, int nb, int env_begin,
                                                              int count, float* __restrict__ height_out, float* __restrict__ xy_out) {
  const long w = (long)blockIdx.x * blockDim.x + threadIdx.x;   // output row: (environment - env_begin) * n + point
  if (w >= (long)count * st.n) return;
  const int i = (int)(w % st.n);
  const long e = env_begin + w / st.n;
  const int b = __ldg(st.body + i);
  const float ox = __ldg(st.xy + 2 * i), oy = __ldg(st.xy + 2 * i + 1);
  float px, py, c0, c1;                           // anchor position and (R00, R10) of its rotation
  if (b == 0 && st.root_from_gc) {
    const float* q = gc + e * gc_stride;
    px = q[0]; py = q[1];
    float qw = q[3], qx = q[4], qy = q[5], qz = q[6];
    const float inv = 1.0f / sqrtf(qw * qw + qx * qx + qy * qy + qz * qz);   // as write_obs_row normalises it
    qw *= inv; qx *= inv; qy *= inv; qz *= inv;
    float c2;
    obs_rot_column(qw, qx, qy, qz, 0, c0, c1, c2);
  } else {
    const float* Rb = R + (e * nb + b) * 9;
    const float* pb = P + (e * nb + b) * 3;
    px = pb[0]; py = pb[1]; c0 = Rb[0]; c1 = Rb[3];
  }
  float sx = px + ox, sy = py + oy;
  if (st.align == RSB_SCAN_YAW) {
    const float nrm = sqrtf(c0 * c0 + c1 * c1);
    float c = 1.f, s = 0.f;
    if (!(nrm < 1e-6f)) { c = c0 / nrm; s = c1 / nrm; }   // a NaN heading stays NaN
    sx = px + (c * ox - s * oy);
    sy = py + (s * ox + c * oy);
  }
  if (xy_out) { xy_out[2 * w] = sx; xy_out[2 * w + 1] = sy; }
  if (height_out) {
    const int hm_offset = ter.env_map ? __ldg(ter.env_map + e) * ter.map_words : 0;   // terrain atlas
    height_out[w] = scan_surface_height(ter, hm_offset, sx, sy);
  }
}

}  // namespace rsb

// ---- RaisimGym ANYmal locomotion task on the device (SURVEY.md 8f N1; [RECALL] raisimGymTorch
//      envs/rsg_anymal/Environment.hpp + VectorizedEnvironment.hpp::perAgentStep) -----------------------
namespace rsb {

// GymConfig: step_kernel.cuh.  ENVIRONMENT::step() -- action -> PD targets, the sub-steps, reward, isTerminalState(), reset() of the
// terminated environments, observe() -- is ONE launch of rsb_step_kernel (StepArgs::gym_action); only reset() of the whole batch is a kernel here.

// ENVIRONMENT::reset() for every environment
// an_hist: the actuator network's history rows of an_words words per environment, zeroed (null: no network); delay_state: the
// actuation delay rows (StepArgs::delay_state), whose command histories are emptied and delays kept (null: no delay)
__global__ void rsb_gym_reset_kernel(float* gc, float* gv, float* ptarget, float* vtarget, GymConfig cfg, int gc_stride, int gv_stride, int nq, int nv, int num_envs,
                                     float* an_hist, int an_words, int* delay_state) {
  const int lane = threadIdx.x & 31;
  const int env = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (env >= num_envs) return;
  for (int i = lane; i < nq; i += 32) { gc[(size_t)env * gc_stride + i] = cfg.gc_init[i]; ptarget[(size_t)env * gc_stride + i] = cfg.gc_init[i]; }
  for (int i = lane; i < nv; i += 32) { gv[(size_t)env * gv_stride + i] = cfg.gv_init[i]; vtarget[(size_t)env * gv_stride + i] = 0.f; }
  if (an_hist) for (int i = lane; i < an_words; i += 32) an_hist[(size_t)env * an_words + i] = 0.f;
  if (delay_state && lane == 0) delay_state[2 * env + 1] = 0;
}

}  // namespace rsb
