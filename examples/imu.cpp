// An upstream-shaped ANYmal ENVIRONMENT whose policy observes the base IMU instead of the base linear velocity, as a policy meant for
// hardware must (ArticulatedSystem::setImus / getImuLinearAcceleration / getImuAngularVelocity: extensions, see
// include/raisim/World.hpp).  The readings are the means over the control step's integrate() calls, which run as ONE launch.  Checks:
// N environments in VectorizedEnvironment take 1.00 launches per control step although every environment reads its IMU; environment 0
// of the batch equals, bit for bit, the same class alone in a VectorizedEnvironment of one; and a World of its own standing still reads
// the specific force +|g| about the base's z axis and no rotation.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <random>
#include <vector>

#include "raisim/VectorizedEnvironment.hpp"

namespace raisim {

struct ImuCfg { std::string urdf = "raisimlib_b200/rsc/anymal_c_like.urdf"; double simulation_dt = 0.0025, control_dt = 0.01; };

class ImuEnv : public RaisimGymEnv {
 public:
  ImuEnv(const std::string& resourceDir, const ImuCfg& cfg, bool) : RaisimGymEnv(resourceDir) {
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
    robot_->setImus({robot_->getFrameIdxByName("base")});
    obDim_ = 3 + nJoints_ + 3 + 3 + nJoints_;   // projected gravity, joint angles, IMU specific force / 10, IMU angular rate, joint rates
    actionDim_ = nJoints_;
  }
  void init() final { reset(); }
  void reset() final { robot_->setState(gc_init_, gv_init_); robot_->setPdTarget(gc_init_, gv_init_); gc_ = gc_init_; gv_ = gv_init_; }
  float step(const RowRef& action) final {
    for (int i = 0; i < gcDim_; i++) pTarget_[i] = gc_init_[i];
    for (int i = 0; i < nJoints_; i++) pTarget_[7 + i] += scale_ * action[i];
    robot_->setPdTarget(pTarget_, vTarget_);
    const int loopCount = int(control_dt_ / simulation_dt_ + 1e-10);
    for (int i = 0; i < loopCount; i++) world_->integrate();
    robot_->getState(gc_, gv_);
    robot_->getImuLinearAcceleration(0, acc_);
    robot_->getImuAngularVelocity(0, rate_);
    return float(-0.01 * (rate_[0] * rate_[0] + rate_[1] * rate_[1] + rate_[2] * rate_[2]));
  }
  void observe(RowRef ob) final {
    const double w = gc_[3], x = gc_[4], y = gc_[5], z = gc_[6];
    const double g[3] = {2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)};   // R^T e_z: the third row of R
    for (int k = 0; k < 3; k++) ob[k] = float(g[k]);
    for (int i = 0; i < nJoints_; i++) ob[3 + i] = float(gc_[7 + i]);
    for (int k = 0; k < 3; k++) { ob[3 + nJoints_ + k] = float(acc_[k] / 10.0); ob[6 + nJoints_ + k] = float(rate_[k]); }
    for (int i = 0; i < nJoints_; i++) ob[9 + nJoints_ + i] = float(gv_[6 + i]);
  }
  bool isTerminalState(float& terminalReward) final { terminalReward = -5.f; if (gc_[2] < 0.25) return true; terminalReward = 0.f; return false; }
  void setActionScale(double s) { scale_ = s; }
  const Vec<3>& acc() const { return acc_; }
  const Vec<3>& rate() const { return rate_; }

 private:
  raisim::ArticulatedSystem* robot_ = nullptr;
  int gcDim_ = 0, gvDim_ = 0, nJoints_ = 0;
  double scale_ = 0.4;
  VecDyn gc_, gc_init_, gv_, gv_init_, pTarget_, vTarget_;
  Vec<3> acc_, rate_;
};

}  // namespace raisim

int main(int argc, char** argv) {
  raisim::ImuCfg cfg;
  if (argc > 1) cfg.urdf = argv[1];
  const int N = argc > 2 ? std::atoi(argv[2]) : 256, steps = 60;
  raisim::VectorizedEnvironment<raisim::ImuEnv> vec("", cfg, N), one("", cfg, 1);
  vec.init(); one.init();
  const int A = vec.getActionDim(), O = vec.getObDim();
  std::vector<float> action(size_t(N) * A), ob(size_t(N) * O), reward(N), ob1(O), reward1(1);
  std::vector<char> done(N), done1(1);
  std::mt19937 rng(13);
  std::normal_distribution<float> nd(0.f, 1.f);
  const long l0 = vec.launches();
  bool same = true;
  double accMean = 0.0;
  for (int k = 0; k < steps; k++) {
    for (float& a : action) a = nd(rng);
    vec.step(action.data(), reward.data(), reinterpret_cast<bool*>(done.data()));
    vec.observe(ob.data());
    one.step(action.data(), reward1.data(), reinterpret_cast<bool*>(done1.data()));
    one.observe(ob1.data());
    same = same && std::memcmp(ob.data(), ob1.data(), size_t(O) * sizeof(float)) == 0 && std::memcmp(&reward[0], &reward1[0], sizeof(float)) == 0;
    for (int i = 0; i < N; i++) {
      const auto& a = vec.environment(i).acc();
      accMean += std::sqrt(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]) / (double(N) * steps);
    }
  }
  const long launches = vec.launches() - l0;
  std::printf("%d environments x %d control steps of 4 integrate() calls: %ld batched launches (%.2f per control step)\n", N, steps, launches, double(launches) / steps);
  std::printf("mean |specific force| at the base under random actions %.2f m/s^2\n", accMean);
  std::printf("environment 0 of the batch vs the same class in a batch of one: observations and rewards %s\n", same ? "bit-identical" : "DIFFER");
  // a World of its own holding its stance: every integrate() is a launch of its own, the getters cover that call
  raisim::ImuEnv solo("", cfg, false);
  solo.init();
  solo.setActionScale(0.0);
  std::vector<float> a0(A, 0.f);
  for (int k = 0; k < 200; k++) solo.step(raisim::RowRef{a0.data(), A});
  const auto &f = solo.acc(), &w = solo.rate();
  const bool still = std::fabs(std::sqrt(f[0] * f[0] + f[1] * f[1] + f[2] * f[2]) - 9.81) < 0.05 && f[2] > 9.6 && std::sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]) < 0.01;
  std::printf("stand-alone World standing still: specific force (%.4f, %.4f, %.4f) m/s^2, rate (%.5f, %.5f, %.5f) rad/s: %s\n", f[0], f[1], f[2],
              w[0], w[1], w[2], still ? "+|g|, about the base z axis" : "UNEXPECTED");
  const bool ok = launches == steps && same && still;
  std::printf(ok ? "ok\n" : "FAILED\n");
  return ok ? 0 : 1;
}
