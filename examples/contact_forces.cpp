// Foot contact flags and foot forces of a whole control step in an upstream-shaped ENVIRONMENT (ArticulatedSystem::setContactBodies /
// getBodyContactSteps / getBodyContactForce: extensions, see include/raisim/World.hpp).  Under upstream the environment would loop
// over getContacts() after each world_->integrate(); here the integrate() calls of a control step run as ONE launch, which gathers the
// same thing.  Checks: N environments in VectorizedEnvironment take 1.00 launches per control step although every environment reads
// its foot forces; environment 0 of the batch equals, bit for bit, the same class alone in a VectorizedEnvironment of one; every foot
// in the contact list of the last sub-step is flagged (the flags may show more: touches of earlier sub-steps); and a World of its own
// (each integrate() a launch of its own: the getters then cover that call) agrees with getContacts().
#include <cmath>
#include <cstdio>
#include <cstring>
#include <random>
#include <vector>

#include "raisim/VectorizedEnvironment.hpp"

namespace raisim {

struct FootCfg { std::string urdf = "raisimlib_b200/rsc/anymal_c_like.urdf"; double simulation_dt = 0.0025, control_dt = 0.01; };

class FootEnv : public RaisimGymEnv {
 public:
  FootEnv(const std::string& resourceDir, const FootCfg& cfg, bool) : RaisimGymEnv(resourceDir) {
    world_ = std::make_unique<raisim::World>();
    world_->setTimeStep(cfg.simulation_dt);
    robot_ = world_->addArticulatedSystem(cfg.urdf);
    world_->addGround();
    simulation_dt_ = cfg.simulation_dt; control_dt_ = cfg.control_dt;
    gcDim_ = int(robot_->getGeneralizedCoordinateDim()); gvDim_ = int(robot_->getDOF()); nJoints_ = gvDim_ - 6;
    gc_.setZero(gcDim_); gc_init_.setZero(gcDim_); gv_.setZero(gvDim_); gv_init_.setZero(gvDim_); pTarget_.setZero(gcDim_); vTarget_.setZero(gvDim_);
    const double stance[19] = {0, 0, 0.57, 1, 0, 0, 0, 0.03, 0.4, -0.8, -0.03, 0.4, -0.8, 0.03, -0.4, 0.8, -0.03, -0.4, 0.8};
    for (int i = 0; i < gcDim_; i++) gc_init_[i] = stance[i];
    VecDyn kp(gvDim_), kd(gvDim_);
    for (int i = 6; i < gvDim_; i++) { kp[i] = 80.0; kd[i] = 1.5; }
    robot_->setControlMode(raisim::ControlMode::PD_PLUS_FEEDFORWARD_TORQUE);
    robot_->setPdGains(kp, kd);
    for (const char* n : {"LF_FOOT", "RF_FOOT", "LH_FOOT", "RH_FOOT"}) feet_.push_back(robot_->getBodyIdx(n));
    robot_->setContactBodies(feet_);
    obDim_ = 1 + nJoints_ + 2 * 4;          // height, joint angles, per foot: touched during the control step, mean vertical force / 500 N
    actionDim_ = nJoints_;
  }
  void init() final { reset(); }
  void reset() final { robot_->setState(gc_init_, gv_init_); robot_->setPdTarget(gc_init_, gv_init_); gc_ = gc_init_; gv_ = gv_init_; }
  float step(const RowRef& action) final {
    for (int i = 0; i < gcDim_; i++) pTarget_[i] = gc_init_[i];
    for (int i = 0; i < nJoints_; i++) pTarget_[7 + i] += 0.4 * action[i];
    robot_->setPdTarget(pTarget_, vTarget_);
    const int loopCount = int(control_dt_ / simulation_dt_ + 1e-10);
    for (int i = 0; i < loopCount; i++) world_->integrate();
    robot_->getState(gc_, gv_);
    float airborne = 0.f;
    for (size_t f = 0; f < 4; f++) {
      steps_[f] = robot_->getBodyContactSteps(feet_[f]);
      Vec<3> force; robot_->getBodyContactForce(feet_[f], force);
      forceZ_[f] = float(force[2]);
      airborne += steps_[f] == 0 ? 1.f : 0.f;
    }
    lastListFeet_ = 0;                      // what the contact list of the last integrate() alone shows
    for (auto& c : robot_->getContacts()) for (size_t f = 0; f < 4; f++) if (c.getlocalBodyIndex() == feet_[f]) lastListFeet_ |= 1 << f;
    return float(0.3 * gv_[0] - 0.1 * airborne);
  }
  void observe(RowRef ob) final {
    ob[0] = float(gc_[2]);
    for (int i = 0; i < nJoints_; i++) ob[1 + i] = float(gc_[7 + i]);
    for (int f = 0; f < 4; f++) { ob[1 + nJoints_ + f] = steps_[f] > 0 ? 1.f : 0.f; ob[5 + nJoints_ + f] = forceZ_[f] / 500.f; }
  }
  bool isTerminalState(float& terminalReward) final { terminalReward = -5.f; if (gc_[2] < 0.25) return true; terminalReward = 0.f; return false; }
  const int* steps() const { return steps_; }
  int lastListFeet() const { return lastListFeet_; }

 private:
  raisim::ArticulatedSystem* robot_ = nullptr;
  int gcDim_ = 0, gvDim_ = 0, nJoints_ = 0;
  VecDyn gc_, gc_init_, gv_, gv_init_, pTarget_, vTarget_;
  std::vector<size_t> feet_;
  int steps_[4] = {0, 0, 0, 0}, lastListFeet_ = 0;
  float forceZ_[4] = {0, 0, 0, 0};
};

}  // namespace raisim

int main(int argc, char** argv) {
  raisim::FootCfg cfg;
  if (argc > 1) cfg.urdf = argv[1];
  const int N = argc > 2 ? std::atoi(argv[2]) : 256, steps = 60;
  raisim::VectorizedEnvironment<raisim::FootEnv> vec("", cfg, N), one("", cfg, 1);
  vec.init(); one.init();
  const int A = vec.getActionDim(), O = vec.getObDim();
  std::vector<float> action(size_t(N) * A), ob(size_t(N) * O), reward(N), ob1(O), reward1(1);
  std::vector<char> done(N), done1(1);
  std::mt19937 rng(11);
  std::normal_distribution<float> nd(0.f, 1.f);
  const long l0 = vec.launches();
  long touchedOnly = 0, touched = 0, partial = 0, lastBits = 0;
  bool same = true, flagsCoverList = true;
  for (int k = 0; k < steps; k++) {
    for (float& a : action) a = nd(rng);
    vec.step(action.data(), reward.data(), reinterpret_cast<bool*>(done.data()));
    vec.observe(ob.data());
    one.step(action.data(), reward1.data(), reinterpret_cast<bool*>(done1.data()));
    one.observe(ob1.data());
    same = same && std::memcmp(ob.data(), ob1.data(), size_t(O) * sizeof(float)) == 0 && std::memcmp(&reward[0], &reward1[0], sizeof(float)) == 0;
    for (int i = 0; i < N; i++) {
      const raisim::FootEnv& e = vec.environment(i);
      for (int f = 0; f < 4; f++) {
        const bool last = (e.lastListFeet() >> f) & 1, any = e.steps()[f] > 0;
        flagsCoverList = flagsCoverList && (!last || any);
        touched += any; touchedOnly += any && !last; partial += any && e.steps()[f] < 4; lastBits += last;
      }
    }
  }
  const long launches = vec.launches() - l0;
  std::printf("%d environments x %d control steps of 4 integrate() calls: %ld batched launches (%.2f per control step)\n", N, steps, launches, double(launches) / steps);
  std::printf("foot touches seen over the control step %ld, by the last contact list %ld; seen only by the fused launch %ld; in contact for part of the step %ld\n",
              touched, lastBits, touchedOnly, partial);
  std::printf("environment 0 of the batch vs the same class in a batch of one: observations and rewards %s\n", same ? "bit-identical" : "DIFFER");
  // a World of its own: every integrate() is a launch, the getters cover that call and agree with its contact list
  raisim::FootEnv solo("", cfg, false);
  solo.init();
  bool soloOk = true;
  std::vector<float> a0(A);
  for (int k = 0; k < steps; k++) {
    for (float& a : a0) a = nd(rng);
    solo.step(raisim::RowRef{a0.data(), A});
    for (int f = 0; f < 4; f++) soloOk = soloOk && ((solo.steps()[f] > 0) == bool((solo.lastListFeet() >> f) & 1)) && solo.steps()[f] <= 1;
  }
  std::printf("stand-alone World: flags of the last integrate() %s its contact list\n", soloOk ? "equal" : "DIFFER from");
  const bool ok = launches == steps && same && flagsCoverList && touched > 0 && soloOk;
  std::printf(ok ? "ok\n" : "FAILED\n");
  return ok ? 0 : 1;
}
