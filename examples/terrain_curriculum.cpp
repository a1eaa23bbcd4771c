// A terrain curriculum in an upstream-shaped ENVIRONMENT: L terrain levels (TerrainProperties with zScale growing by level and a seed
// per level), environment i starting at level i % L, and a deterministic rule in reset() that moves an environment one level up when its
// base travelled further in the episode than in the one before, else one level down -- the legged_gym pattern, written the raisimGym way:
// each environment builds its own terrain with World::addHeightMap.  observe() appends legged_gym's 11 x 17 base grid of terrain heights.
// In a VectorizedEnvironment every environment collides with, and scans, its own map: the maps go to the device as one terrain atlas,
// and moving environments among levels already there is one index call, no map upload.  Checks: every scan height equals the
// environment's own HeightMap::getHeight at the returned sample, one step launch per control step, and no map upload after init().
#include <cmath>
#include <cstdio>
#include <memory>
#include <random>
#include <vector>

#include "raisim/VectorizedEnvironment.hpp"

namespace raisim {

struct CurriculumCfg { std::string urdf = "raisimlib_b200/rsc/anymal_c_like.urdf"; double simulation_dt = 0.0025, control_dt = 0.01; int episode = 8, levels = 5; };

class CurriculumEnv : public RaisimGymEnv {
 public:
  static double& worstError() { static double e = 0; return e; }   // largest |scan - own HeightMap::getHeight| seen by any observe()
  static long& moves() { static long m = 0; return m; }             // level changes made by reset()
  CurriculumEnv(const std::string& resourceDir, const CurriculumCfg& cfg, bool) : RaisimGymEnv(resourceDir), episode_(cfg.episode), levels_(cfg.levels) {
    world_ = std::make_unique<raisim::World>();
    world_->setTimeStep(cfg.simulation_dt);
    robot_ = world_->addArticulatedSystem(cfg.urdf);
    level_ = robot_->env() % levels_;
    terrain_ = world_->addHeightMap(0.0, 0.0, terrainOf(level_));
    std::vector<size_t> bodies;
    std::vector<Vec<2>> offsets;
    for (int i = 0; i < 11; i++)
      for (int j = 0; j < 17; j++) { bodies.push_back(0); offsets.push_back({-0.8 + 0.16 * i, -0.5 + 0.0625 * j}); }
    robot_->setHeightScan(bodies, offsets);
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
  static TerrainProperties terrainOf(int level) {
    TerrainProperties tp;
    tp.xSize = tp.ySize = 16.0; tp.xSamples = tp.ySamples = 161; tp.frequency = 0.6; tp.fractalOctaves = 3;
    tp.zScale = 0.05 + 0.08 * level; tp.seed = 11 + 7 * level;
    return tp;
  }
  void init() final { reset(); }
  void reset() final {
    if (steps_ > 0) {   // the curriculum: up a level after a longer walk than the episode before, else down
      const double travelled = std::hypot(gc_[0] - x0_, gc_[1] - y0_);
      const int next = std::max(0, std::min(levels_ - 1, level_ + (travelled > lastTravelled_ ? 1 : -1)));
      lastTravelled_ = travelled;
      if (next != level_) { level_ = next; terrain_ = world_->addHeightMap(0.0, 0.0, terrainOf(level_)); moves()++; }
    }
    const int e = robot_->env();
    x0_ = -5.0 + 0.37 * (e % 27); y0_ = -4.0 + 0.29 * (e % 23);
    const double psi = 0.41 * e;
    gc_ = gc_init_;
    gc_[0] = x0_; gc_[1] = y0_; gc_[2] = terrain_->getHeight(x0_, y0_) + 0.62;
    gc_[3] = std::cos(0.5 * psi); gc_[6] = std::sin(0.5 * psi);
    gv_ = gv_init_;
    robot_->setState(gc_, gv_); robot_->setPdTarget(gc_, gv_);
    pTarget_ = gc_;
    steps_ = 0;
  }
  float step(const RowRef& action) final {
    for (int i = 0; i < nJoints_; i++) pTarget_[7 + i] = gc_init_[7 + i] + 0.3 * action[i];
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
  int level() const { return level_; }

 private:
  raisim::ArticulatedSystem* robot_ = nullptr;
  raisim::HeightMap* terrain_ = nullptr;
  int gcDim_ = 0, gvDim_ = 0, nJoints_ = 0;
  VecDyn gc_, gc_init_, gv_, gv_init_, pTarget_, vTarget_, scan_;
  std::vector<Vec<2>> samples_;
  int steps_ = 0, episode_ = 0, levels_ = 0, level_ = 0;
  double x0_ = 0, y0_ = 0, lastTravelled_ = 0;
};

}  // namespace raisim

int main(int argc, char** argv) {
  raisim::CurriculumCfg cfg;
  if (argc > 1) cfg.urdf = argv[1];
  const int N = argc > 2 ? std::atoi(argv[2]) : 64, steps = 60;
  raisim::VectorizedEnvironment<raisim::CurriculumEnv> vec("", cfg, N);
  vec.init();
  const raisim::LockStep& ls = *vec.world().lockStep();
  const long maps0 = ls.mapUploads, index0 = ls.indexUploads, l0 = vec.launches();
  const int A = vec.getActionDim(), O = vec.getObDim();
  std::vector<float> action(size_t(N) * A), ob(size_t(N) * O), reward(N);
  std::vector<char> done(N);
  std::mt19937 rng(5);
  std::normal_distribution<float> nd(0.f, 1.f);
  for (int s = 0; s < steps; s++) {
    for (float& a : action) a = nd(rng);
    vec.step(action.data(), reward.data(), reinterpret_cast<bool*>(done.data()));
    vec.observe(ob.data());
  }
  const long stepLaunches = vec.launches() - l0, mapUploads = ls.mapUploads - maps0, indexMoves = ls.indexUploads - index0;
  std::vector<int> perLevel(size_t(cfg.levels), 0);
  for (int i = 0; i < N; i++) perLevel[size_t(vec.environment(i).level())]++;
  const double worst = raisim::CurriculumEnv::worstError();
  std::printf("%d environments x %d control steps on %d terrain levels: %ld level changes, %ld index calls and %ld map uploads after init(), %ld step launches (%.2f per control step)\n",
              N, steps, cfg.levels, raisim::CurriculumEnv::moves(), indexMoves, mapUploads, stepLaunches, double(stepLaunches) / steps);
  std::printf("environments per level at the end:");
  for (int c : perLevel) std::printf(" %d", c);
  std::printf("\nlargest |scan - own HeightMap::getHeight at the returned sample| over all environments and steps: %.3g m\n", worst);
  const bool ok = worst <= 1e-4 && stepLaunches == steps && mapUploads == 0 && indexMoves > 0 && raisim::CurriculumEnv::moves() > 0;
  std::printf(ok ? "ok\n" : "FAILED\n");
  return ok ? 0 : 1;
}
