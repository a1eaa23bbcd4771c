// An LSTM actuator network in an upstream-shaped ENVIRONMENT, shaped like the ANYmal actuator model of legged_gym and Isaac Lab: the
// constructor gives the batch one seeded 2-layer LSTM of hidden size 8 on the 12 joints in place of their PD law, and reset() zeroes
// the environment's (h, c) state.  A control step is 4 integrate() calls, which run as ONE launch; the cell advances once per sub-step.
// Checks: one step launch per control step, and a few environments of a batch of 256 equal, bit for bit, stand-alone Worlds with the
// same network that run one integrate() (one launch of one sub-step) at a time.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <memory>
#include <random>
#include <vector>

#include "raisim/VectorizedEnvironment.hpp"

namespace raisim {

constexpr int L = 2, Hd = 8, kEpisode = 25;
static const double kStance[19] = {0, 0, 0.57, 1, 0, 0, 0, 0.03, 0.4, -0.8, -0.03, 0.4, -0.8, 0.03, -0.4, 0.8, -0.03, -0.4, 0.8};

// torch order: per layer weight_ih [4 Hd][n_in], weight_hh [4 Hd][Hd], bias_ih [4 Hd], bias_hh [4 Hd]; read-out weight [1][Hd], bias [1].
// The read-out gives torques of tens of N m
std::vector<float> lstmParams() {
  std::mt19937 rng(17);
  std::uniform_real_distribution<float> u(-1.f, 1.f);
  std::vector<float> p;
  for (int l = 0; l < L; l++) {
    const int nin = l == 0 ? 2 : Hd;
    for (int k = 0; k < 4 * Hd * nin; k++) p.push_back(u(rng) * (l == 0 ? 4.f : 1.f) / std::sqrt(float(nin)));
    for (int k = 0; k < 4 * Hd * Hd; k++) p.push_back(u(rng) / std::sqrt(float(Hd)));
    for (int k = 0; k < 8 * Hd; k++) p.push_back(0.2f * u(rng));
  }
  for (int k = 0; k < Hd; k++) p.push_back(u(rng) * 30.f);
  p.push_back(0.f);
  return p;
}
std::vector<size_t> jointDofs() {
  std::vector<size_t> d;
  for (size_t i = 6; i < 18; i++) d.push_back(i);
  return d;
}
void target(const float* action, VecDyn& pt) {
  pt.setZero(19);
  for (int i = 0; i < 19; i++) pt[i] = kStance[i];
  for (int i = 0; i < 12; i++) pt[7 + i] += 0.3 * action[i];
}
void initialState(int env, VecDyn& gc, VecDyn& gv) {
  gc.setZero(19); gv.setZero(18);
  for (int i = 0; i < 19; i++) gc[i] = kStance[i];
  gc[0] = 2.0 * env;
}

struct LstmCfg { std::string urdf = "raisimlib_b200/rsc/anymal_c_like.urdf"; double simulation_dt = 0.0025, control_dt = 0.01; };

class LstmEnv : public RaisimGymEnv {
 public:
  LstmEnv(const std::string& resourceDir, const LstmCfg& cfg, bool) : RaisimGymEnv(resourceDir) {
    world_ = std::make_unique<raisim::World>();
    world_->setTimeStep(cfg.simulation_dt);
    robot_ = world_->addArticulatedSystem(cfg.urdf);
    world_->addGround();
    simulation_dt_ = cfg.simulation_dt; control_dt_ = cfg.control_dt;
    robot_->setControlMode(raisim::ControlMode::PD_PLUS_FEEDFORWARD_TORQUE);
    robot_->setActuatorLstm(jointDofs(), L, Hd, lstmParams());   // the same network in every environment: set once for the batch
    vTarget_.setZero(18);
    obDim_ = 3 + 24;
    actionDim_ = 12;
  }
  void init() final { reset(); }
  void reset() final {
    initialState(robot_->env(), gc_, gv_);
    robot_->setState(gc_, gv_); robot_->setPdTarget(gc_, vTarget_);
    robot_->resetActuatorHistory();          // setState keeps the (h, c) state: a new episode starts from zeros
    steps_ = 0;
  }
  float step(const RowRef& action) final {
    target(action.p, pTarget_);
    robot_->setPdTarget(pTarget_, vTarget_);
    const int loopCount = int(control_dt_ / simulation_dt_ + 1e-10);
    for (int i = 0; i < loopCount; i++) world_->integrate();
    robot_->getState(gc_, gv_);
    steps_++;
    return float(gv_[0]);
  }
  void observe(RowRef ob) final {
    for (int i = 0; i < 3; i++) ob[i] = float(gc_[i]);
    for (int i = 0; i < 12; i++) { ob[3 + i] = float(gc_[7 + i]); ob[15 + i] = float(gv_[6 + i]); }
  }
  bool isTerminalState(float& terminalReward) final { terminalReward = 0.f; return steps_ >= kEpisode || gc_[2] < 0.25; }

 private:
  raisim::ArticulatedSystem* robot_ = nullptr;
  VecDyn gc_, gv_, pTarget_, vTarget_;
  int steps_ = 0;
};

// environment env in a World of its own with the same network: one integrate() per sub-step
struct StandAlone {
  int env;
  std::unique_ptr<World> world;
  ArticulatedSystem* robot = nullptr;
  StandAlone(int e, const std::string& urdf, double dt) : env(e), world(new World) {
    world->setTimeStep(dt);
    robot = world->addArticulatedSystem(urdf);
    world->addGround();
    robot->setControlMode(ControlMode::PD_PLUS_FEEDFORWARD_TORQUE);
    robot->setActuatorLstm(jointDofs(), L, Hd, lstmParams());
    reset();
  }
  void reset() {
    VecDyn gc, gv;
    initialState(env, gc, gv);
    robot->setState(gc, gv);
    robot->resetActuatorHistory();
  }
  void controlStep(const float* action, int subSteps) {
    VecDyn pt, vt;
    target(action, pt);
    vt.setZero(18);
    robot->setPdTarget(pt, vt);
    for (int s = 0; s < subSteps; s++) world->integrate();
  }
};

}  // namespace raisim

int main(int argc, char** argv) {
  using namespace raisim;
  LstmCfg cfg;
  if (argc > 1) cfg.urdf = argv[1];
  const int N = argc > 2 ? std::atoi(argv[2]) : 256, steps = 60, subSteps = int(cfg.control_dt / cfg.simulation_dt + 1e-10);
  VectorizedEnvironment<LstmEnv> vec("", cfg, N);
  vec.init();
  std::vector<std::unique_ptr<StandAlone>> ref;
  for (int e : {0, 1, N / 2, N - 1}) ref.emplace_back(new StandAlone(e, cfg.urdf, cfg.simulation_dt));
  const int A = vec.getActionDim(), O = vec.getObDim();
  std::vector<float> action(size_t(N) * A), ob(size_t(N) * O), reward(N), gc(size_t(N) * 19), gv(size_t(N) * 18), tau(size_t(N) * 18);
  std::vector<char> done(N, 0);
  std::mt19937 rng(7);
  std::normal_distribution<float> nd(0.f, 1.f);
  rsb_batch* b = vec.world().batch();
  long compared = 0, differing = 0, resets = 0;
  double largest = 0.0;
  const long l0 = vec.launches();
  for (int s = 0; s < steps; s++) {
    for (float& a : action) a = nd(rng);
    vec.step(action.data(), reward.data(), reinterpret_cast<bool*>(done.data()));
    vec.observe(ob.data());
    rsbCheck(rsb_batch_get_generalized_force(b, tau.data(), 0, N, RSB_HOST), "getGeneralizedForce");
    for (int e = 0; e < N; e++)
      for (int j = 6; j < 18; j++) largest = std::max(largest, double(std::fabs(tau[size_t(e) * 18 + j])));
    // the device holds the state the step ended in, or the reset state of an environment that terminated (step() pushes resets)
    rsbCheck(rsb_batch_get_state(b, gc.data(), gv.data(), 0, N, RSB_HOST), "getState");
    for (auto& r : ref) {
      r->controlStep(&action[size_t(r->env) * A], subSteps);
      if (done[r->env]) r->reset();
      VecDyn rq, rv;
      r->robot->getState(rq, rv);
      for (int i = 0; i < 19; i++) differing += float(rq[i]) != gc[size_t(r->env) * 19 + i];
      for (int i = 0; i < 18; i++) differing += float(rv[i]) != gv[size_t(r->env) * 18 + i];
      compared += 37;
    }
    for (int e = 0; e < N; e++) resets += done[e];
  }
  const long stepLaunches = vec.launches() - l0;
  std::printf("%d environments x %d control steps of %d sub-steps, 12 joints on a %d-layer LSTM of hidden size %d: %ld step launches "
              "(launches per control step %.2f), %ld resets, largest joint torque %.1f N m\n",
              N, steps, subSteps, L, Hd, stepLaunches, double(stepLaunches) / steps, resets, largest);
  std::printf("against stand-alone Worlds, environments 0, 1, %d, %d: %ld state words compared, %ld differ\n", N / 2, N - 1, compared, differing);
  const bool ok = stepLaunches == steps && compared > 0 && differing == 0 && resets > 0 && largest > 5.0;
  std::printf(ok ? "ok\n" : "FAILED\n");
  return ok ? 0 : 1;
}
