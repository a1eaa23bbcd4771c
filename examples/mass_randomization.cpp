// Payload randomisation in an upstream-shaped ENVIRONMENT: every environment adds a seeded random payload (mass and centre-of-mass
// offset) to its robot's base in its constructor, composed with the body's own inertial parameters by the parallel-axis theorem, and
// calls updateMassInfo() -- upstream's getMass()[i] / getBodyCOM_B()[i] / getInertia()[i] idiom.  Checks: N environments in
// VectorizedEnvironment take 1.00 launches per control step; environment k equals, bit for bit, the same class in a stand-alone World
// with the same payload; the host-side getTotalMass() reads each environment's own payload; and heavier robots sink deeper.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <random>
#include <vector>

#include "raisim/VectorizedEnvironment.hpp"

namespace raisim {

struct PayloadCfg { std::string urdf = "raisimlib_b200/rsc/anymal_c_like.urdf"; double simulation_dt = 0.0025, control_dt = 0.01; unsigned seed = 17; };

// a point payload of mass pm at p (body frame) added to a body of mass m with centre of mass c and inertia I about it
inline void addPayload(double& m, Vec<3>& c, Mat<3, 3>& I, double pm, const Vec<3>& p) {
  const double mt = m + pm;
  Vec<3> cn;
  for (size_t k = 0; k < 3; k++) cn[k] = (m * c[k] + pm * p[k]) / mt;
  auto shift = [&](double mass, const Vec<3>& x) {   // mass (|d|^2 1 - d d^T), d = x - cn
    double d[3] = {x[0] - cn[0], x[1] - cn[1], x[2] - cn[2]}, dd = d[0] * d[0] + d[1] * d[1] + d[2] * d[2];
    for (size_t r = 0; r < 3; r++) for (size_t s = 0; s < 3; s++) I(r, s) += mass * ((r == s ? dd : 0.0) - d[r] * d[s]);
  };
  shift(m, c); shift(pm, p);
  m = mt; c = cn;
}

class PayloadEnv : public RaisimGymEnv {
 public:
  static int& created() { static int n = 0; return n; }       // environments built so far: the index that seeds the payload
  PayloadEnv(const std::string& resourceDir, const PayloadCfg& cfg, bool) : RaisimGymEnv(resourceDir) {
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
    for (int i = 6; i < gvDim_; i++) { kp[i] = 200.0; kd[i] = 4.0; }
    robot_->setControlMode(raisim::ControlMode::PD_PLUS_FEEDFORWARD_TORQUE);
    robot_->setPdGains(kp, kd);
    // the payload: 0-10 kg, its centre up to 5 cm off the base's centre of mass sideways and 5-10 cm above it
    std::mt19937 rng(cfg.seed + unsigned(created()++));
    std::uniform_real_distribution<double> u(0.0, 1.0);
    payload_ = 10.0 * u(rng);
    Vec<3> p = robot_->getBodyCOM_B()[0];
    p[0] += 0.1 * u(rng) - 0.05; p[1] += 0.1 * u(rng) - 0.05; p[2] += 0.05 + 0.05 * u(rng);
    addPayload(robot_->getMass()[0], robot_->getBodyCOM_B()[0], robot_->getInertia()[0], payload_, p);
    robot_->updateMassInfo();
    obDim_ = 2 + nJoints_;          // base height, total mass / 100 kg, joint angles
    actionDim_ = nJoints_;
  }
  void init() final { reset(); }
  void reset() final { robot_->setState(gc_init_, gv_init_); robot_->setPdTarget(gc_init_, gv_init_); gc_ = gc_init_; gv_ = gv_init_; }
  float step(const RowRef& action) final {
    for (int i = 0; i < gcDim_; i++) pTarget_[i] = gc_init_[i];
    for (int i = 0; i < nJoints_; i++) pTarget_[7 + i] += 0.1 * action[i];
    robot_->setPdTarget(pTarget_, vTarget_);
    const int loopCount = int(control_dt_ / simulation_dt_ + 1e-10);
    for (int i = 0; i < loopCount; i++) world_->integrate();
    robot_->getState(gc_, gv_);
    return float(0.3 * gv_[0]);
  }
  void observe(RowRef ob) final {
    ob[0] = float(gc_[2]); ob[1] = float(robot_->getTotalMass() / 100.0);
    for (int i = 0; i < nJoints_; i++) ob[2 + i] = float(gc_[7 + i]);
  }
  bool isTerminalState(float& terminalReward) final { terminalReward = 0.f; return false; }
  double payload() const { return payload_; }

 private:
  raisim::ArticulatedSystem* robot_ = nullptr;
  int gcDim_ = 0, gvDim_ = 0, nJoints_ = 0;
  VecDyn gc_, gc_init_, gv_, gv_init_, pTarget_, vTarget_;
  double payload_ = 0;
};

}  // namespace raisim

int main(int argc, char** argv) {
  raisim::PayloadCfg cfg;
  if (argc > 1) cfg.urdf = argv[1];
  const int N = argc > 2 ? std::atoi(argv[2]) : 256, steps = 100, k = N / 3;
  raisim::VectorizedEnvironment<raisim::PayloadEnv> vec("", cfg, N);
  vec.init();
  raisim::PayloadEnv::created() = k;                        // the stand-alone World of environment k: the same payload
  raisim::PayloadEnv solo("", cfg, false);
  solo.init();
  const int A = vec.getActionDim(), O = vec.getObDim();
  std::vector<float> action(size_t(N) * A), ob(size_t(N) * O), reward(N), ob1(O);
  std::vector<char> done(N);
  std::mt19937 rng(11);
  std::normal_distribution<float> nd(0.f, 1.f);
  const long l0 = vec.launches();
  bool same = true;
  for (int s = 0; s < steps; s++) {
    for (float& a : action) a = nd(rng);
    vec.step(action.data(), reward.data(), reinterpret_cast<bool*>(done.data()));
    vec.observe(ob.data());
    const float r1 = solo.step(raisim::RowRef{action.data() + size_t(k) * A, A});
    solo.observe(raisim::RowRef{ob1.data(), O});
    same = same && std::memcmp(&ob[size_t(k) * O], ob1.data(), size_t(O) * sizeof(float)) == 0 && std::memcmp(&reward[k], &r1, sizeof(float)) == 0;
  }
  const long launches = vec.launches() - l0;
  // total mass: the robot's plus each environment's payload; the heaviest quarter stands lower than the lightest quarter
  double massErr = 0, lightZ = 0, heavyZ = 0; int nl = 0, nh = 0;
  const double robot = double(ob[1]) * 100.0 - vec.environment(0).payload();
  for (int i = 0; i < N; i++) {
    const double p = vec.environment(i).payload();
    massErr = std::fmax(massErr, std::fabs(double(ob[size_t(i) * O + 1]) * 100.0 - (robot + p)));
    if (p < 2.5) { lightZ += ob[size_t(i) * O]; nl++; }
    if (p > 7.5) { heavyZ += ob[size_t(i) * O]; nh++; }
  }
  lightZ /= std::max(nl, 1); heavyZ /= std::max(nh, 1);
  std::printf("%d environments x %d control steps of 4 integrate() calls: %ld batched launches (%.2f per control step)\n", N, steps, launches, double(launches) / steps);
  std::printf("environment %d of the batch vs a stand-alone World with the same %.3f kg payload: observations and rewards %s\n", k,
              vec.environment(k).payload(), same ? "bit-identical" : "DIFFER");
  std::printf("getTotalMass() = robot + payload within %.1e kg; mean base height with payload < 2.5 kg %.4f m, > 7.5 kg %.4f m\n", massErr, lightZ, heavyZ);
  const bool ok = launches == steps && same && massErr < 1e-4 && heavyZ < lightZ && nl > 0 && nh > 0;
  std::printf(ok ? "ok\n" : "FAILED\n");
  return ok ? 0 : 1;
}
