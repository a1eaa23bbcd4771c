// A depth camera in an upstream-shaped ENVIRONMENT on rough terrain: the constructor hangs a 32 x 24 pinhole camera (87 degrees wide)
// on the front of the base, pitched 30 degrees down, that sees the terrain and the robot's own legs, and observe() appends its z-depth
// image (the distance along the optical axis, misses at the maximum range).  In a VectorizedEnvironment the first environment's
// getRayCasts() casts every environment's rays in one launch.  Checks: N environments take one step launch, one kinematics pass and
// one ray launch per control step, and every pixel that hit the terrain has its hit point on HeightMap::getHeight within 1e-4 m.
#include <cmath>
#include <cstdio>
#include <memory>
#include <random>
#include <vector>

#include "raisim/VectorizedEnvironment.hpp"

namespace raisim {

struct CamCfg { std::string urdf = "raisimlib_b200/rsc/anymal_c_like.urdf"; double simulation_dt = 0.0025, control_dt = 0.01; int episode = 25; };

constexpr int W = 32, H = 24;
constexpr double HFOV = 87.0 * M_PI / 180.0, PITCH = 30.0 * M_PI / 180.0, RANGE = 10.0;
const double CAM_POS[3] = {0.35, 0.0, 0.05};   // on the front of the base, in the base frame

class DepthEnv : public RaisimGymEnv {
 public:
  static double& worstError() { static double e = 0; return e; }   // largest |hit z - HeightMap::getHeight| over every terrain pixel
  static long& terrainPixels() { static long c = 0; return c; }
  static long& robotPixels() { static long c = 0; return c; }
  DepthEnv(const std::string& resourceDir, const CamCfg& cfg, bool) : RaisimGymEnv(resourceDir), episode_(cfg.episode) {
    world_ = std::make_unique<raisim::World>();
    world_->setTimeStep(cfg.simulation_dt);
    robot_ = world_->addArticulatedSystem(cfg.urdf);
    TerrainProperties tp;
    tp.xSize = tp.ySize = 16.0; tp.xSamples = tp.ySamples = 161; tp.frequency = 0.6; tp.zScale = 0.25; tp.fractalOctaves = 3; tp.seed = 7;
    terrain_ = world_->addHeightMap(0.0, 0.0, tp);
    // pinhole rays through the pixel centres, row-major from the top-left pixel: camera frame x forward, -y right, -z down; then
    // pitched down about the base's y axis.  zAxis_ keeps each ray's component along the optical axis for the z-depth.
    const double f = 0.5 * W / std::tan(0.5 * HFOV);
    std::vector<size_t> bodies;
    std::vector<Vec<3>> origins, dirs;
    for (int r = 0; r < H; r++)
      for (int c = 0; c < W; c++) {
        const double u = c + 0.5 - 0.5 * W, v = r + 0.5 - 0.5 * H, nrm = std::sqrt(f * f + u * u + v * v);
        const double x = f / nrm, y = -u / nrm, z = -v / nrm;
        zAxis_.push_back(x);
        bodies.push_back(0);
        origins.push_back({CAM_POS[0], CAM_POS[1], CAM_POS[2]});
        dirs.push_back({std::cos(PITCH) * x + std::sin(PITCH) * z, y, -std::sin(PITCH) * x + std::cos(PITCH) * z});
      }
    camDirs_ = dirs;
    robot_->setRays(bodies, origins, dirs, RANGE, true);   // the same list in every environment: set once for the batch
    simulation_dt_ = cfg.simulation_dt; control_dt_ = cfg.control_dt;
    gcDim_ = int(robot_->getGeneralizedCoordinateDim()); gvDim_ = int(robot_->getDOF()); nJoints_ = gvDim_ - 6;
    gc_.setZero(gcDim_); gc_init_.setZero(gcDim_); gv_.setZero(gvDim_); gv_init_.setZero(gvDim_); pTarget_.setZero(gcDim_); vTarget_.setZero(gvDim_);
    const double stance[19] = {0, 0, 0.0, 1, 0, 0, 0, 0.03, 0.4, -0.8, -0.03, 0.4, -0.8, 0.03, -0.4, 0.8, -0.03, -0.4, 0.8};
    for (int i = 0; i < gcDim_; i++) gc_init_[i] = stance[i];
    VecDyn kp(gvDim_), kd(gvDim_);
    for (int i = 6; i < gvDim_; i++) { kp[i] = 200.0; kd[i] = 4.0; }
    robot_->setControlMode(raisim::ControlMode::PD_PLUS_FEEDFORWARD_TORQUE);
    robot_->setPdGains(kp, kd);
    obDim_ = 3 + nJoints_ + W * H;
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
    robot_->getRayCasts(dist_, &hits_);
    for (int i = 0; i < 3; i++) ob[i] = float(gc_[i]);
    for (int i = 0; i < nJoints_; i++) ob[3 + i] = float(gc_[7 + i]);
    // the base pose the rays hang on, from the state: p = gc[0:3], R from the normalised quaternion gc[3:7]
    double qw = gc_[3], qx = gc_[4], qy = gc_[5], qz = gc_[6];
    const double qn = std::sqrt(qw * qw + qx * qx + qy * qy + qz * qz);
    qw /= qn; qx /= qn; qy /= qn; qz /= qn;
    const double R[9] = {1 - 2 * (qy * qy + qz * qz), 2 * (qx * qy - qw * qz), 2 * (qx * qz + qw * qy),
                         2 * (qx * qy + qw * qz), 1 - 2 * (qx * qx + qz * qz), 2 * (qy * qz - qw * qx),
                         2 * (qx * qz - qw * qy), 2 * (qy * qz + qw * qx), 1 - 2 * (qx * qx + qy * qy)};
    for (size_t k = 0; k < dist_.size(); k++) {
      const double t = dist_[k];
      ob[3 + nJoints_ + int(k)] = float(std::isfinite(t) ? t * zAxis_[k] : RANGE);   // z-depth; a miss reads the maximum range
      if (hits_[k] >= 0) robotPixels()++;
      if (hits_[k] != RSB_RAY_TERRAIN) continue;
      terrainPixels()++;
      double hit[3];
      for (int i = 0; i < 3; i++) {
        const double o = gc_[i] + R[3 * i] * CAM_POS[0] + R[3 * i + 1] * CAM_POS[1] + R[3 * i + 2] * CAM_POS[2];
        const double d = R[3 * i] * camDirs_[k][0] + R[3 * i + 1] * camDirs_[k][1] + R[3 * i + 2] * camDirs_[k][2];
        hit[i] = o + t * d;
      }
      const double err = std::fabs(hit[2] - terrain_->getHeight(hit[0], hit[1]));
      if (!(err <= worstError())) worstError() = err;       // NaN counts as the worst
    }
  }
  bool isTerminalState(float& terminalReward) final { terminalReward = 0.f; return steps_ >= episode_; }

 private:
  raisim::ArticulatedSystem* robot_ = nullptr;
  raisim::HeightMap* terrain_ = nullptr;
  int gcDim_ = 0, gvDim_ = 0, nJoints_ = 0;
  VecDyn gc_, gc_init_, gv_, gv_init_, pTarget_, vTarget_, dist_;
  std::vector<int> hits_;
  std::vector<double> zAxis_;
  std::vector<Vec<3>> camDirs_;
  int steps_ = 0, episode_ = 0;
};

}  // namespace raisim

int main(int argc, char** argv) {
  raisim::CamCfg cfg;
  if (argc > 1) cfg.urdf = argv[1];
  const int N = argc > 2 ? std::atoi(argv[2]) : 64, steps = 60;
  raisim::VectorizedEnvironment<raisim::DepthEnv> vec("", cfg, N);
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
  // a 1e-4 m bound: float32 poses and arithmetic move a hit point by a few micrometres, far below the map's features
  const double worst = raisim::DepthEnv::worstError();
  std::printf("%d environments x %d control steps, %d x %d pixels each: %ld step launches and %ld other launches (%.2f and %.2f per control step)\n",
              N, steps, raisim::W, raisim::H, stepLaunches, long(all - stepLaunches), double(stepLaunches) / steps, double(all - stepLaunches) / steps);
  std::printf("pixels on the terrain %ld, on the robot %ld; largest |hit z - HeightMap::getHeight at the hit| %.3g m\n",
              raisim::DepthEnv::terrainPixels(), raisim::DepthEnv::robotPixels(), worst);
  const bool ok = stepLaunches == steps && all == 3 * steps && worst <= 1e-4 && raisim::DepthEnv::terrainPixels() > 0;
  std::printf(ok ? "ok\n" : "FAILED\n");
  return ok ? 0 : 1;
}
