// Height scans in an upstream-shaped ENVIRONMENT on rough terrain: the constructor hangs legged_gym's 11 x 17 grid (187 points, 1.6 m x
// 1.0 m) on the base, yaw-aligned, and observe() appends the terrain height under every point, relative to the base height -- what an
// upstream observe() builds with one HeightMap::getHeight call per point.  In a VectorizedEnvironment the first environment's
// getHeightScan() scans every environment in one launch.  Checks: N environments take one step launch and one scan launch per
// control step, and every height equals HeightMap::getHeight at the returned sample location.
#include <cmath>
#include <cstdio>
#include <memory>
#include <random>
#include <vector>

#include "raisim/VectorizedEnvironment.hpp"

namespace raisim {

struct ScanCfg { std::string urdf = "raisimlib_b200/rsc/anymal_c_like.urdf"; double simulation_dt = 0.0025, control_dt = 0.01; int episode = 25; };

class ScanEnv : public RaisimGymEnv {
 public:
  static double& worstError() { static double e = 0; return e; }   // largest |scan - HeightMap::getHeight| seen by any observe()
  ScanEnv(const std::string& resourceDir, const ScanCfg& cfg, bool) : RaisimGymEnv(resourceDir), episode_(cfg.episode) {
    world_ = std::make_unique<raisim::World>();
    world_->setTimeStep(cfg.simulation_dt);
    robot_ = world_->addArticulatedSystem(cfg.urdf);
    TerrainProperties tp;
    tp.xSize = tp.ySize = 16.0; tp.xSamples = tp.ySamples = 161; tp.frequency = 0.6; tp.zScale = 0.25; tp.fractalOctaves = 3; tp.seed = 7;
    terrain_ = world_->addHeightMap(0.0, 0.0, tp);
    std::vector<size_t> bodies;
    std::vector<Vec<2>> offsets;
    for (int i = 0; i < 11; i++)
      for (int j = 0; j < 17; j++) { bodies.push_back(0); offsets.push_back({-0.8 + 0.16 * i, -0.5 + 0.0625 * j}); }
    robot_->setHeightScan(bodies, offsets);                   // the same list in every environment: set once for the batch
    simulation_dt_ = cfg.simulation_dt; control_dt_ = cfg.control_dt;
    gcDim_ = int(robot_->getGeneralizedCoordinateDim()); gvDim_ = int(robot_->getDOF()); nJoints_ = gvDim_ - 6;
    gc_.setZero(gcDim_); gc_init_.setZero(gcDim_); gv_.setZero(gvDim_); gv_init_.setZero(gvDim_); pTarget_.setZero(gcDim_); vTarget_.setZero(gvDim_);
    const double stance[19] = {0, 0, 0.0, 1, 0, 0, 0, 0.03, 0.4, -0.8, -0.03, 0.4, -0.8, 0.03, -0.4, 0.8, -0.03, -0.4, 0.8};
    for (int i = 0; i < gcDim_; i++) gc_init_[i] = stance[i];
    VecDyn kp(gvDim_), kd(gvDim_);
    for (int i = 6; i < gvDim_; i++) { kp[i] = 200.0; kd[i] = 4.0; }
    robot_->setControlMode(raisim::ControlMode::PD_PLUS_FEEDFORWARD_TORQUE);
    robot_->setPdGains(kp, kd);
    obDim_ = 3 + nJoints_ + int(bodies.size());
    actionDim_ = nJoints_;
  }
  void init() final { reset(); }
  void reset() final {   // drop the robot at a spot and heading that depend on the environment, just above the terrain there
    const int e = robot_->env();
    const double x = -5.0 + 0.37 * (e % 27), y = -4.0 + 0.29 * (e % 23), psi = 0.41 * e;
    gc_ = gc_init_;
    gc_[0] = x; gc_[1] = y; gc_[2] = terrain_->getHeight(x, y) + 0.62;
    gc_[3] = std::cos(0.5 * psi); gc_[6] = std::sin(0.5 * psi);
    gv_ = gv_init_;
    robot_->setState(gc_, gv_); robot_->setPdTarget(gc_, gv_);
    pTarget_ = gc_;
    steps_ = 0;
  }
  float step(const RowRef& action) final {
    for (int i = 0; i < nJoints_; i++) pTarget_[7 + i] = gc_init_[7 + i] + 0.2 * action[i];
    robot_->setPdTarget(pTarget_, vTarget_);
    const int loopCount = int(control_dt_ / simulation_dt_ + 1e-10);
    for (int i = 0; i < loopCount; i++) world_->integrate();
    robot_->getState(gc_, gv_);
    steps_++;
    return float(gv_[0]);
  }
  void observe(RowRef ob) final {
    robot_->getHeightScan(scan_, &samples_);
    for (int i = 0; i < 3; i++) ob[i] = float(gc_[i]);
    for (int i = 0; i < nJoints_; i++) ob[3 + i] = float(gc_[7 + i]);
    for (size_t k = 0; k < scan_.size(); k++) {
      ob[3 + nJoints_ + int(k)] = float(gc_[2] - scan_[k]);
      const double err = std::fabs(scan_[k] - terrain_->getHeight(samples_[k][0], samples_[k][1]));
      if (!(err <= worstError())) worstError() = err;       // NaN counts as the worst
    }
  }
  bool isTerminalState(float& terminalReward) final { terminalReward = 0.f; return steps_ >= episode_; }

 private:
  raisim::ArticulatedSystem* robot_ = nullptr;
  raisim::HeightMap* terrain_ = nullptr;
  int gcDim_ = 0, gvDim_ = 0, nJoints_ = 0;
  VecDyn gc_, gc_init_, gv_, gv_init_, pTarget_, vTarget_, scan_;
  std::vector<Vec<2>> samples_;
  int steps_ = 0, episode_ = 0;
};

}  // namespace raisim

int main(int argc, char** argv) {
  raisim::ScanCfg cfg;
  if (argc > 1) cfg.urdf = argv[1];
  const int N = argc > 2 ? std::atoi(argv[2]) : 64, steps = 60;
  raisim::VectorizedEnvironment<raisim::ScanEnv> vec("", cfg, N);
  vec.init();
  const int A = vec.getActionDim(), O = vec.getObDim();
  std::vector<float> action(size_t(N) * A), ob(size_t(N) * O), reward(N);
  std::vector<char> done(N);
  std::mt19937 rng(3);
  std::normal_distribution<float> nd(0.f, 1.f);
  rsb_batch* b = vec.world().batch();
  const long l0 = vec.launches();
  const int64_t k0 = rsb_batch_launch_count(b);
  for (int s = 0; s < steps; s++) {
    for (float& a : action) a = nd(rng);
    vec.step(action.data(), reward.data(), reinterpret_cast<bool*>(done.data()));
    vec.observe(ob.data());
  }
  const long stepLaunches = vec.launches() - l0;
  const int64_t all = rsb_batch_launch_count(b) - k0;
  // a 1e-4 m bound: the float32 grid coordinate times the local slope, far below the map's features
  const double worst = raisim::ScanEnv::worstError();
  std::printf("%d environments x %d control steps, 187 base points each: %ld step launches and %ld scan launches (%.2f and %.2f per control step)\n",
              N, steps, stepLaunches, long(all - stepLaunches), double(stepLaunches) / steps, double(all - stepLaunches) / steps);
  std::printf("largest |scan - HeightMap::getHeight at the returned sample| over all environments and steps: %.3g m\n", worst);
  const bool ok = stepLaunches == steps && all == 2 * steps && worst <= 1e-4;
  std::printf(ok ? "ok\n" : "FAILED\n");
  return ok ? 0 : 1;
}
