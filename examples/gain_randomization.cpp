// Actuator randomisation in an upstream-shaped ENVIRONMENT: every reset() draws a seeded P gain, D gain and motor strength (a scale of
// the URDF effort limits) and sets them with ArticulatedSystem::setPdGains and setActuationLimits -- the usual Kp / Kd / torque-limit
// randomisation of legged-locomotion training.  In a VectorizedEnvironment each environment's calls set its own actuator row.  Checks:
// N environments take 1.00 launches per control step, getActuationUpperLimits() returns the environment's own limits, and every
// environment equals, bit for bit, the same class in a stand-alone World (a batch of one) that draws the same gains and limits.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <memory>
#include <random>
#include <vector>

#include "raisim/VectorizedEnvironment.hpp"

namespace raisim {

struct GainCfg { std::string urdf = "raisimlib_b200/rsc/anymal_c_like.urdf"; double simulation_dt = 0.0025, control_dt = 0.01; unsigned seed = 7; int episode = 20; };

class GainEnv : public RaisimGymEnv {
 public:
  static int& created() { static int n = 0; return n; }       // environments built so far: the index that seeds the draws
  static int& limitErrors() { static int n = 0; return n; }   // getActuationUpperLimits() that did not return the limits just set
  GainEnv(const std::string& resourceDir, const GainCfg& cfg, bool) : RaisimGymEnv(resourceDir), rng_(cfg.seed + unsigned(created()++)), episode_(cfg.episode) {
    world_ = std::make_unique<raisim::World>();
    world_->setTimeStep(cfg.simulation_dt);
    robot_ = world_->addArticulatedSystem(cfg.urdf);
    world_->addGround();
    simulation_dt_ = cfg.simulation_dt; control_dt_ = cfg.control_dt;
    gcDim_ = int(robot_->getGeneralizedCoordinateDim()); gvDim_ = int(robot_->getDOF()); nJoints_ = gvDim_ - 6;
    gc_.setZero(gcDim_); gc_init_.setZero(gcDim_); gv_.setZero(gvDim_); gv_init_.setZero(gvDim_); pTarget_.setZero(gcDim_); vTarget_.setZero(gvDim_);
    const double stance[19] = {0, 0, 0.57, 1, 0, 0, 0, 0.03, 0.4, -0.8, -0.03, 0.4, -0.8, 0.03, -0.4, 0.8, -0.03, -0.4, 0.8};
    for (int i = 0; i < gcDim_; i++) gc_init_[i] = stance[i];
    urdfEffort_ = robot_->getActuationUpperLimits();
    robot_->setControlMode(raisim::ControlMode::PD_PLUS_FEEDFORWARD_TORQUE);
    obDim_ = 6 + nJoints_;          // base position, kp, kd, motor strength, joint angles
    actionDim_ = nJoints_;
  }
  void init() final { reset(); }
  void reset() final {
    kp_ = std::uniform_real_distribution<double>(100.0, 400.0)(rng_);
    kd_ = std::uniform_real_distribution<double>(1.0, 8.0)(rng_);
    strength_ = std::uniform_real_distribution<double>(0.1, 1.0)(rng_);   // weak motors saturate under the stiffer gains
    VecDyn kp(gvDim_), kd(gvDim_), upper(gvDim_), lower(gvDim_);
    for (int i = 6; i < gvDim_; i++) { kp[i] = kp_; kd[i] = kd_; }
    for (int i = 0; i < gvDim_; i++) { upper[i] = strength_ * urdfEffort_[i]; lower[i] = -upper[i]; }
    robot_->setPdGains(kp, kd);
    robot_->setActuationLimits(upper, lower);
    const VecDyn got = robot_->getActuationUpperLimits();
    for (int i = 6; i < gvDim_; i++) if (got[i] != upper[i]) limitErrors()++;
    robot_->setState(gc_init_, gv_init_); robot_->setPdTarget(gc_init_, gv_init_); gc_ = gc_init_; gv_ = gv_init_;
    steps_ = 0;
  }
  float step(const RowRef& action) final {
    for (int i = 0; i < gcDim_; i++) pTarget_[i] = gc_init_[i];
    for (int i = 0; i < nJoints_; i++) pTarget_[7 + i] += 0.4 * action[i];
    robot_->setPdTarget(pTarget_, vTarget_);
    const int loopCount = int(control_dt_ / simulation_dt_ + 1e-10);
    for (int i = 0; i < loopCount; i++) world_->integrate();
    robot_->getState(gc_, gv_);
    steps_++;
    return float(gc_[2]);
  }
  void observe(RowRef ob) final {
    for (int i = 0; i < 3; i++) ob[i] = float(gc_[i]);
    ob[3] = float(kp_); ob[4] = float(kd_); ob[5] = float(strength_);
    for (int i = 0; i < nJoints_; i++) ob[6 + i] = float(gc_[7 + i]);
  }
  bool isTerminalState(float& terminalReward) final { terminalReward = 0.f; return steps_ >= episode_; }   // new actuators every episode

 private:
  raisim::ArticulatedSystem* robot_ = nullptr;
  int gcDim_ = 0, gvDim_ = 0, nJoints_ = 0;
  VecDyn gc_, gc_init_, gv_, gv_init_, pTarget_, vTarget_, urdfEffort_;
  std::mt19937 rng_;
  double kp_ = 0, kd_ = 0, strength_ = 0;
  int steps_ = 0, episode_ = 0;
};

}  // namespace raisim

int main(int argc, char** argv) {
  raisim::GainCfg cfg;
  if (argc > 1) cfg.urdf = argv[1];
  const int N = argc > 2 ? std::atoi(argv[2]) : 32, steps = 50;
  raisim::VectorizedEnvironment<raisim::GainEnv> vec("", cfg, N);
  vec.init();
  raisim::GainEnv::created() = 0;                           // stand-alone Worlds, one per environment: the same gains and limits
  std::vector<std::unique_ptr<raisim::GainEnv>> solo;
  for (int i = 0; i < N; i++) { solo.emplace_back(new raisim::GainEnv("", cfg, false)); solo.back()->init(); }
  const int A = vec.getActionDim(), O = vec.getObDim();
  std::vector<float> action(size_t(N) * A), ob(size_t(N) * O), reward(N), ob1(O);
  std::vector<char> done(N);
  std::mt19937 rng(13);
  std::normal_distribution<float> nd(0.f, 1.f);
  const long l0 = vec.launches();
  int differ = 0;
  for (int s = 0; s < steps; s++) {
    for (float& a : action) a = nd(rng);
    vec.step(action.data(), reward.data(), reinterpret_cast<bool*>(done.data()));
    vec.observe(ob.data());
    for (int i = 0; i < N; i++) {   // upstream perAgentStep() on environment i's own World
      const float r1 = solo[size_t(i)]->step(raisim::RowRef{action.data() + size_t(i) * A, A});
      float terminal = 0.f;
      if (solo[size_t(i)]->isTerminalState(terminal)) solo[size_t(i)]->reset();
      solo[size_t(i)]->observe(raisim::RowRef{ob1.data(), O});
      if (std::memcmp(&ob[size_t(i) * O], ob1.data(), size_t(O) * sizeof(float)) != 0 || std::memcmp(&reward[size_t(i)], &r1, sizeof(float)) != 0) differ++;
    }
  }
  const long launches = vec.launches() - l0;
  std::printf("%d environments x %d control steps of 4 integrate() calls, new gains and effort limits every %d: %ld batched launches (%.2f per control step)\n",
              N, steps, cfg.episode, launches, double(launches) / steps);
  std::printf("every environment vs a stand-alone World drawing the same gains and limits: %d of %d observation rows and rewards differ\n", differ, N * steps);
  std::printf("getActuationUpperLimits() after setActuationLimits(): %d dofs differ from the limits set\n", raisim::GainEnv::limitErrors());
  const bool ok = launches == steps && differ == 0 && raisim::GainEnv::limitErrors() == 0;
  std::printf(ok ? "ok\n" : "FAILED\n");
  return ok ? 0 : 1;
}
