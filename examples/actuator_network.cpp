// A learned actuator network in an upstream-shaped ENVIRONMENT: the constructor gives the batch one seeded network (history 3, two
// softsign layers of 32) on the 12 joints of an ANYmal-like robot in place of their PD law, and reset() zeroes the environment's
// history.  One sub-step per control step, so that the torque the step applied is a function of the state and history seen before it.
// Checks: one step launch per control step, and getGeneralizedForce of every joint equals a float64 restatement of the network at the
// state, targets and history read before the step (environments reset by the previous step are skipped).
#include <cmath>
#include <cstdio>
#include <memory>
#include <random>
#include <vector>

#include "raisim/VectorizedEnvironment.hpp"

namespace raisim {

constexpr int H = 3, L = 2, W = 32;
static const double kStance[19] = {0, 0, 0.57, 1, 0, 0, 0, 0.03, 0.4, -0.8, -0.03, 0.4, -0.8, 0.03, -0.4, 0.8, -0.03, -0.4, 0.8};

// torch.nn.Linear order: W1[W][2H], b1[W], W2[W][W], b2[W], Wout[1][W], bout[1]; output weights give torques of tens of N m
std::vector<float> networkParams() {
  std::mt19937 rng(11);
  std::uniform_real_distribution<float> u(-1.f, 1.f);
  std::vector<float> p;
  int nin = 2 * H;
  for (int l = 0; l < L; l++) {
    for (int k = 0; k < W * nin; k++) p.push_back(u(rng) * 1.5f / std::sqrt(float(nin)));
    for (int k = 0; k < W; k++) p.push_back(0.3f * u(rng));
    nin = W;
  }
  for (int k = 0; k < W; k++) p.push_back(u(rng) * 40.f / std::sqrt(float(W)));
  p.push_back(0.f);
  return p;
}

// float64 restatement: x = [e_t, e_{t-1}, e_{t-2}, v_t, v_{t-1}, v_{t-2}]
double networkTorque(const std::vector<float>& p, const double* x) {
  std::vector<double> in(x, x + 2 * H), out;
  size_t o = 0;
  for (int l = 0; l < L; l++) {
    const int nin = int(in.size());
    out.assign(W, 0.0);
    for (int j = 0; j < W; j++) {
      double a = p[o + size_t(W) * nin + j];
      for (int k = 0; k < nin; k++) a += double(p[o + size_t(j) * nin + k]) * in[k];
      out[j] = a / (1.0 + std::fabs(a));
    }
    o += size_t(W) * nin + W;
    in = out;
  }
  double y = p[o + W];
  for (int j = 0; j < W; j++) y += double(p[o + j]) * in[j];
  return y;
}

struct NetCfg { std::string urdf = "raisimlib_b200/rsc/anymal_c_like.urdf"; double simulation_dt = 0.0025, control_dt = 0.0025; int episode = 40; };

class NetEnv : public RaisimGymEnv {
 public:
  NetEnv(const std::string& resourceDir, const NetCfg& cfg, bool) : RaisimGymEnv(resourceDir), episode_(cfg.episode) {
    world_ = std::make_unique<raisim::World>();
    world_->setTimeStep(cfg.simulation_dt);
    robot_ = world_->addArticulatedSystem(cfg.urdf);
    world_->addGround();
    simulation_dt_ = cfg.simulation_dt; control_dt_ = cfg.control_dt;
    gcDim_ = int(robot_->getGeneralizedCoordinateDim()); gvDim_ = int(robot_->getDOF()); nJoints_ = gvDim_ - 6;
    gc_.setZero(gcDim_); gc_init_.setZero(gcDim_); gv_.setZero(gvDim_); gv_init_.setZero(gvDim_); pTarget_.setZero(gcDim_); vTarget_.setZero(gvDim_);
    for (int i = 0; i < gcDim_; i++) gc_init_[i] = kStance[i];
    robot_->setControlMode(raisim::ControlMode::PD_PLUS_FEEDFORWARD_TORQUE);
    std::vector<size_t> dofs;
    for (int i = 6; i < gvDim_; i++) dofs.push_back(size_t(i));
    robot_->setActuatorNetwork(dofs, H, L, W, networkParams());   // the same network in every environment: set once for the batch
    obDim_ = 3 + 2 * nJoints_;
    actionDim_ = nJoints_;
  }
  void init() final { reset(); }
  void reset() final {
    gc_ = gc_init_; gv_ = gv_init_;
    gc_[0] = 2.0 * robot_->env();
    robot_->setState(gc_, gv_); robot_->setPdTarget(gc_, gv_);
    robot_->resetActuatorHistory();          // setState keeps the history: a new episode starts from zeros
    steps_ = 0;
  }
  float step(const RowRef& action) final {
    pTarget_ = gc_init_;
    for (int i = 0; i < nJoints_; i++) pTarget_[7 + i] = gc_init_[7 + i] + 0.2 * action[i];
    robot_->setPdTarget(pTarget_, vTarget_);
    const int loopCount = int(control_dt_ / simulation_dt_ + 1e-10);
    for (int i = 0; i < loopCount; i++) world_->integrate();
    robot_->getState(gc_, gv_);
    steps_++;
    return float(gv_[0]);
  }
  void observe(RowRef ob) final {
    for (int i = 0; i < 3; i++) ob[i] = float(gc_[i]);
    for (int i = 0; i < nJoints_; i++) { ob[3 + i] = float(gc_[7 + i]); ob[3 + nJoints_ + i] = float(gv_[6 + i]); }
  }
  bool isTerminalState(float& terminalReward) final { terminalReward = 0.f; return steps_ >= episode_ || gc_[2] < 0.25; }

 private:
  raisim::ArticulatedSystem* robot_ = nullptr;
  int gcDim_ = 0, gvDim_ = 0, nJoints_ = 0;
  VecDyn gc_, gc_init_, gv_, gv_init_, pTarget_, vTarget_;
  int steps_ = 0, episode_ = 0;
};

}  // namespace raisim

int main(int argc, char** argv) {
  using namespace raisim;
  NetCfg cfg;
  if (argc > 1) cfg.urdf = argv[1];
  const int N = argc > 2 ? std::atoi(argv[2]) : 64, steps = 120;
  VectorizedEnvironment<NetEnv> vec("", cfg, N);
  vec.init();
  const int A = vec.getActionDim(), O = vec.getObDim(), nq = 19, nv = 18, nj = 12, hw = 2 * (H - 1);
  std::vector<float> action(size_t(N) * A), ob(size_t(N) * O), reward(N);
  std::vector<char> done(N, 0);
  std::mt19937 rng(3);
  std::normal_distribution<float> nd(0.f, 1.f);
  rsb_batch* b = vec.world().batch();
  rsb_model_tables t;
  rsbCheck(rsb_model_get_tables(vec.world().model(), &t), "tables");
  std::vector<double> limit(nv, 1e30);
  for (int k = 1; k < t.nb; k++) limit[t.vidx[k]] = t.jeffort[k];
  const std::vector<float> params = networkParams();
  std::vector<float> gc(size_t(N) * nq), gv(size_t(N) * nv), hist(size_t(N) * nj * hw), tau(size_t(N) * nv);
  double worst = 0.0, largest = 0.0;
  long compared = 0, resets = 0;
  const long l0 = vec.launches();
  for (int s = 0; s < steps; s++) {
    for (float& a : action) a = nd(rng);
    // what the step will start from: state and history on the device (environments reset by the last step still have theirs in the mirror)
    rsbCheck(rsb_batch_get_state(b, gc.data(), gv.data(), 0, N, RSB_HOST), "getState");
    rsbCheck(rsb_batch_get_actuator_history(b, hist.data(), 0, N, RSB_HOST), "getActuatorHistory");
    const std::vector<char> skip = done;
    vec.step(action.data(), reward.data(), reinterpret_cast<bool*>(done.data()));
    vec.observe(ob.data());
    rsbCheck(rsb_batch_get_generalized_force(b, tau.data(), 0, N, RSB_HOST), "getGeneralizedForce");
    for (int e = 0; e < N; e++) {
      if (skip[e] || s == 0) continue;
      for (int j = 0; j < nj; j++) {
        const int d = 6 + j, q = 7 + j;
        const float pt = float(kStance[q] + 0.2 * double(action[size_t(e) * A + j]));
        const float* h = &hist[(size_t(e) * nj + j) * hw];
        const double x[2 * H] = {double(pt - gc[size_t(e) * nq + q]), h[0], h[1], double(gv[size_t(e) * nv + d]), h[2], h[3]};
        double ref = networkTorque(params, x);
        ref = std::max(-limit[d], std::min(limit[d], ref));
        const double err = std::fabs(tau[size_t(e) * nv + d] - ref) / (1.0 + std::fabs(ref));
        if (!(err <= worst)) worst = err;
        largest = std::max(largest, std::fabs(ref));
        compared++;
      }
    }
    for (int e = 0; e < N; e++) resets += done[e];
  }
  const long stepLaunches = vec.launches() - l0;
  std::printf("%d environments x %d control steps: %ld step launches (launches per control step %.2f), %ld resets\n", N, steps, stepLaunches,
              double(stepLaunches) / steps, resets);
  std::printf("getGeneralizedForce against the float64 network: %ld joint torques compared, largest |tau| %.1f N m, largest |dtau| / (1 + |tau|) %.3g\n",
              compared, largest, worst);
  const bool ok = stepLaunches == steps && compared > 0 && worst <= 1e-4 && largest > 5.0 && resets > 0;
  std::printf(ok ? "ok\n" : "FAILED\n");
  return ok ? 0 : 1;
}
