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
