// Actuation latency in an upstream-shaped ENVIRONMENT: reset() draws a seeded delay of 0-8 physics sub-steps (0-20 ms at 2.5 ms) for
// the episode and sets it with ArticulatedSystem::setActuationDelay; step() sets PD targets as usual, and the batch applies each one
// that many sub-steps late, also in the middle of a 4-sub-step control step.
// Checks: one step launch per control step, and a few environments equal, bit for bit, a stand-alone World without a delay that runs
// one integrate() per sub-step and sets the shifted target itself: at sub-step t of an episode, the target of sub-step max(t - d, 0).
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <memory>
#include <random>
#include <vector>

#include "raisim/VectorizedEnvironment.hpp"

namespace raisim {

static const double kStance[19] = {0, 0, 0.57, 1, 0, 0, 0, 0.03, 0.4, -0.8, -0.03, 0.4, -0.8, 0.03, -0.4, 0.8, -0.03, -0.4, 0.8};
constexpr int kEpisode = 25, kMaxDelay = 8;

// the delay of episode `episode` of environment env: seeded, so that a restatement can draw the same one
int drawDelay(int env, int episode) {
  std::mt19937 rng(1000u * unsigned(env) + unsigned(episode));
  return std::uniform_int_distribution<int>(0, kMaxDelay)(rng);
}
void gains(VecDyn& kp, VecDyn& kd) {
  kp.setZero(18); kd.setZero(18);
  for (int i = 6; i < 18; i++) { kp[i] = 80.0; kd[i] = 1.5; }
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

struct DelayCfg { std::string urdf = "raisimlib_b200/rsc/anymal_c_like.urdf"; double simulation_dt = 0.0025, control_dt = 0.01; };

class DelayEnv : public RaisimGymEnv {
 public:
  DelayEnv(const std::string& resourceDir, const DelayCfg& cfg, bool) : RaisimGymEnv(resourceDir) {
    world_ = std::make_unique<raisim::World>();
    world_->setTimeStep(cfg.simulation_dt);
    robot_ = world_->addArticulatedSystem(cfg.urdf);
    world_->addGround();
    simulation_dt_ = cfg.simulation_dt; control_dt_ = cfg.control_dt;
    VecDyn kp, kd;
    gains(kp, kd);
    robot_->setControlMode(raisim::ControlMode::PD_PLUS_FEEDFORWARD_TORQUE);
    robot_->setPdGains(kp, kd);
    vTarget_.setZero(18);
    obDim_ = 3 + 24;
    actionDim_ = 12;
  }
  void init() final { reset(); }
  void reset() final {
    initialState(robot_->env(), gc_, gv_);
    robot_->setState(gc_, gv_); robot_->setPdTarget(gc_, vTarget_);
    robot_->setActuationDelay(size_t(drawDelay(robot_->env(), episode_++)));   // empties the command history: a new episode
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
  bool isTerminalState(float& terminalReward) final { terminalReward = 0.f; return steps_ >= kEpisode; }

 private:
  raisim::ArticulatedSystem* robot_ = nullptr;
  VecDyn gc_, gv_, pTarget_, vTarget_;
  int steps_ = 0, episode_ = 0;
};

// environment env restated in a World of its own without a delay: one integrate() per sub-step, the shifted target set before each
struct Restatement {
  int env, episode = 0, delay = 0, t = 0;
  std::unique_ptr<World> world;
  ArticulatedSystem* robot = nullptr;
  std::vector<VecDyn> commands;   // the target of every control step of the episode
  Restatement(int e, const std::string& urdf, double dt) : env(e), world(new World) {
    world->setTimeStep(dt);
    robot = world->addArticulatedSystem(urdf);
    world->addGround();
    VecDyn kp, kd;
    gains(kp, kd);
    robot->setControlMode(ControlMode::PD_PLUS_FEEDFORWARD_TORQUE);
    robot->setPdGains(kp, kd);
    reset();
  }
  void reset() {
    VecDyn gc, gv;
    initialState(env, gc, gv);
    robot->setState(gc, gv);
    delay = drawDelay(env, episode++);
    t = 0;
    commands.clear();
  }
  void controlStep(const float* action, int subSteps) {
    commands.emplace_back();
    target(action, commands.back());
    VecDyn vt;
    vt.setZero(18);
    for (int s = 0; s < subSteps; s++, t++) {
      robot->setPdTarget(commands[size_t(std::max(t - delay, 0) / subSteps)], vt);
      world->integrate();
    }
  }
};

}  // namespace raisim

int main(int argc, char** argv) {
  using namespace raisim;
  DelayCfg cfg;
  if (argc > 1) cfg.urdf = argv[1];
  const int N = argc > 2 ? std::atoi(argv[2]) : 64, steps = 60, subSteps = int(cfg.control_dt / cfg.simulation_dt + 1e-10);
  VectorizedEnvironment<DelayEnv> vec("", cfg, N);
  vec.init();
  std::vector<std::unique_ptr<Restatement>> ref;
  for (int e : {0, 1, N / 2, N - 1}) ref.emplace_back(new Restatement(e, cfg.urdf, cfg.simulation_dt));
  const int A = vec.getActionDim(), O = vec.getObDim();
  std::vector<float> action(size_t(N) * A), ob(size_t(N) * O), reward(N), gc(size_t(N) * 19), gv(size_t(N) * 18);
  std::vector<char> done(N, 0);
  std::mt19937 rng(5);
  std::normal_distribution<float> nd(0.f, 1.f);
  rsb_batch* b = vec.world().batch();
  long compared = 0, differing = 0, resets = 0, delayed = 0;
  const long l0 = vec.launches();
  for (int s = 0; s < steps; s++) {
    for (float& a : action) a = nd(rng);
    vec.step(action.data(), reward.data(), reinterpret_cast<bool*>(done.data()));
    vec.observe(ob.data());
    // the device holds the state the step ended in, or the reset state of an environment that terminated (step() pushes resets)
    rsbCheck(rsb_batch_get_state(b, gc.data(), gv.data(), 0, N, RSB_HOST), "getState");
    for (auto& r : ref) {
      r->controlStep(&action[size_t(r->env) * A], subSteps);
      delayed += r->delay > 0;
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
  std::printf("%d environments x %d control steps of %d sub-steps, delays 0-%d sub-steps drawn at every reset: %ld step launches (launches per control step %.2f), %ld resets\n",
              N, steps, subSteps, kMaxDelay, stepLaunches, double(stepLaunches) / steps, resets);
  std::printf("against a stand-alone World fed the shifted targets, environments 0, 1, %d, %d: %ld state words compared, %ld differ\n", N / 2, N - 1,
              compared, differing);
  const bool ok = stepLaunches == steps && compared > 0 && differing == 0 && resets > 0 && delayed > 0;
  std::printf(ok ? "ok\n" : "FAILED\n");
  return ok ? 0 : 1;
}
