// Scripted use of the raisim:: facade against the recording stub of the C ABI (rsb_recording_stub.cpp, no GPU): prints the log of
// rsb_batch_* calls the facade issues, with "#" lines marking the script's phases and hashing the values the getters return.
// usage: facade_trace standalone | vecenv | sync
//   standalone  a stand-alone World with a joint order, through every state, actuation, material, inertia, terrain and getter accessor
//   vecenv      a VectorizedEnvironment of 3 environments with their own gains, friction, inertia, delays, history resets and two maps
//   sync        getters that read the device (M, h, positions, the solver loop counter) inside step() after integrate(), and after a
//               setState in reset()
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "raisim/VectorizedEnvironment.hpp"

std::string& rsb_stub_log();

namespace {
using raisim::MatDyn;
using raisim::Vec;
using raisim::VecDyn;

void mark(const std::string& s) { rsb_stub_log() += "# " + s + "\n"; }
uint64_t fnv(const double* p, size_t n) {
  uint64_t h = 1469598103934665603ull;
  for (size_t i = 0; i < n; i++) { uint64_t u; std::memcpy(&u, &p[i], 8); for (int b = 0; b < 8; b++) h = (h ^ ((u >> (8 * b)) & 0xff)) * 1099511628211ull; }
  return h;
}
void value(const char* what, const double* p, size_t n) {
  char b[96];
  std::snprintf(b, sizeof b, "= %s %016llx\n", what, (unsigned long long)fnv(p, n));
  rsb_stub_log() += b;
}
void value(const char* what, const VecDyn& v) { value(what, v.ptr(), v.size()); }
void value(const char* what, const MatDyn& m) { value(what, m.v.data(), m.v.size()); }
template <size_t k> void value(const char* what, const Vec<k>& v) { value(what, v.ptr(), k); }
void value(const char* what, double x) { value(what, &x, 1); }

const std::vector<std::string> kOrder = {"j3", "j1", "j2"};   // the batch's order is j1, j2, j3

VecDyn vec(size_t n, double a, double b) { VecDyn v(n); for (size_t i = 0; i < n; i++) v[i] = a + b * double(i); return v; }
VecDyn stance(double x) { VecDyn q = vec(10, 0.0, 0.1); q[0] = x; q[2] = 0.5; q[3] = 1; q[4] = q[5] = q[6] = 0; return q; }
std::vector<float> netParams(int H, int L, int W) {
  const size_t count = size_t(2 * H) * W + W + size_t(L - 1) * (size_t(W) * W + W) + W + 1;
  std::vector<float> p(count);
  for (size_t i = 0; i < count; i++) p[i] = 0.01f * float(int(i % 11) - 5);
  return p;
}

// every getter a view offers, each value hashed into the log
void readAll(raisim::World& w, raisim::ArticulatedSystem* r, bool deviceGetters) {
  VecDyn q, v;
  r->getState(q, v); value("gc", q); value("gv", v);
  value("tau", r->getGeneralizedForce());
  for (auto& c : r->getContacts()) { value("contact", c.getPosition()); value("impulse", c.getImpulse()); }
  Vec<3> f; r->getBodyContactForce(1, f); value("contact force", f);
  value("contact steps", double(r->getBodyContactSteps(2)));
  VecDyn h; std::vector<Vec<2>> xy;
  r->getHeightScan(h, &xy); value("scan", h); for (auto& p : xy) value("scan xy", p);
  r->getHeightScan(h); value("scan", h);
  Vec<3> p; r->getBodyPosition(2, p); value("body position", p);
  r->getFramePosition(3, p); value("frame position", p);
  MatDyn J; r->getDenseJacobian(2, p, J); value("jacobian", J);
  value("com", r->getCOM());
  if (deviceGetters) {   // the getters the lock-step mirror did not bring up to date before this change
    value("M", r->getMassMatrix());
    value("h", r->getNonlinearities());
    r->getPosition(1, {0.1, 0.0, 0.0}, p); value("position", p);
    value("loop counter", double(w.getContactSolver().getLoopCounter()));
    value("kinetic energy", r->getKineticEnergy());
  }
  value("world time", w.getWorldTime());
}

void standalone() {
  raisim::World w;
  w.setTimeStep(0.002);
  w.setGravity({0.0, 0.0, -9.7});
  mark("addArticulatedSystem");
  raisim::ArticulatedSystem* r = w.addArticulatedSystem("stub.urdf", "", kOrder);
  w.addGround(0.0, "default");
  mark("materials");
  w.setDefaultMaterial(0.7, 0.1, 0.02);
  r->getCollisionBody("l1/0").setMaterial("rubber");
  w.setMaterialPairProp("rubber", "default", 0.9);
  r->getCollisionBody("l3/0").setMaterial("steel");
  w.integrate();
  r->setCollisionBodyFriction(2, 0.4);
  w.setMaterialPairProp("steel", "default", 0.3);
  mark("state");
  r->setState(stance(0.2), vec(9, 0.01, 0.02));
  r->setGeneralizedCoordinate(stance(0.3));
  r->setGeneralizedVelocity(vec(9, -0.01, 0.03));
  r->setBasePos({0.1, 0.2, 0.45});
  r->setBaseOrientation(Vec<4>{0.9, 0.1, 0.0, 0.1});
  r->setGeneralizedForce(vec(9, 0.5, -0.1));
  mark("actuation");
  r->setControlMode(raisim::ControlMode::PD_PLUS_FEEDFORWARD_TORQUE);
  r->setPdGains(vec(9, 10.0, 1.0), vec(9, 0.5, 0.1));
  r->setPGains(vec(9, 20.0, 1.0));
  r->setDGains(vec(9, 0.2, 0.1));
  r->setPdTarget(stance(0.0), vec(9, 0.0, 0.0));
  r->setPTarget(stance(0.1));
  r->setDTarget(vec(9, 0.1, 0.0));
  r->setActuationLimits(vec(9, 5.0, 1.0), vec(9, -5.0, -1.0));
  mark("inertia");
  r->getMass()[1] = 1.25;
  r->getBodyCOM_B()[2][0] = 0.05;
  r->getInertia()[3](0, 0) = 0.02;
  r->updateMassInfo();
  mark("extensions");
  r->setContactBodies({1, 2});
  r->setHeightScan({0, 0, 2}, {{0.1, 0.2}, {-0.3, 0.1}, {0.0, 0.0}});
  r->setActuatorNetwork({7, 8}, 2, 1, 4, netParams(2, 1, 4));
  r->setActuationDelay(2);
  r->resetActuatorHistory();
  r->setExternalForce(1, {1.0, 2.0, 3.0});
  r->setSelfCollisionPairs({{"l1/0", "l3/0"}});
  mark("height map");
  std::vector<double> hm(5 * 4);
  for (size_t i = 0; i < hm.size(); i++) hm[i] = 0.01 * double(i % 6);
  w.addHeightMap(5, 4, 4.0, 3.0, 0.0, 0.0, hm);
  raisim::TerrainProperties tp; tp.xSamples = 5; tp.ySamples = 4; tp.xSize = 4.0; tp.ySize = 3.0;
  w.addHeightMap(0.0, 0.0, tp);
  mark("getters");
  readAll(w, r, true);
  for (int s = 0; s < 3; s++) {
    mark("control step");
    r->setPdTarget(stance(0.05 * s), vec(9, 0.0, 0.0));
    for (int i = 0; i < 4; i++) w.integrate();
    VecDyn q, v;
    r->getState(q, v);
    mark("end control step");
    value("gc", q);
  }
  mark("getters");
  readAll(w, r, true);
  mark("view of a shared batch");
  raisim::BatchedWorld bw("stub.urdf", 3);
  raisim::World view(&bw, 1);
  raisim::ArticulatedSystem* vr = view.getRobot();
  vr->setJointOrder(kOrder);
  vr->setState(stance(1.0), vec(9, 0.2, 0.0));
  vr->setPdTarget(stance(1.0), vec(9, 0.0, 0.0));
  vr->setGeneralizedForce(vec(9, 0.1, 0.1));
  view.integrate();
  VecDyn q, v;
  vr->getState(q, v); value("gc", q); value("gv", v);
  value("M", vr->getMassMatrix());
  mark("end");
}

struct Cfg { bool sync = false; };

class TraceEnv : public raisim::RaisimGymEnv {
 public:
  TraceEnv(const std::string& dir, const Cfg& cfg, bool) : RaisimGymEnv(dir), sync_(cfg.sync) {
    world_ = std::make_unique<raisim::World>();
    world_->setTimeStep(0.0025);
    robot_ = world_->addArticulatedSystem("stub.urdf", "", kOrder);
    e_ = robot_->env();
    if (sync_) { world_->addGround(); obDim_ = 1; actionDim_ = 3; return; }
    std::vector<double> h(6 * 5);
    for (size_t i = 0; i < h.size(); i++) h[i] = 0.02 * double((i + size_t(e_ % 2) * 3) % 7);   // two maps: even and odd environments
    terrain_ = world_->addHeightMap(6, 5, 5.0, 4.0, 0.5, 0.0, h);
    robot_->setContactBodies({1, 3});
    robot_->setHeightScan({0, 0}, {{0.2, 0.0}, {0.0, 0.2}});
    robot_->setActuatorNetwork({6, 8}, 3, 1, 3, netParams(3, 1, 3));
    robot_->setControlMode(raisim::ControlMode::PD_PLUS_FEEDFORWARD_TORQUE);
    robot_->getCollisionBody("l2/0").setMaterial("rubber");
    world_->setMaterialPairProp("rubber", "default", 0.5 + 0.1 * e_);
    world_->setDefaultMaterial(0.6 + 0.05 * e_, 0.0, 0.01);
    obDim_ = 4; actionDim_ = 3;
  }
  void init() final { reset(); }
  void reset() final {
    mark("reset " + std::to_string(e_));
    robot_->setState(stance(0.3 * e_), vec(9, 0.01 * e_, 0.0));
    if (sync_) { value("M", robot_->getMassMatrix()); return; }
    robot_->setPdTarget(stance(0.3 * e_), vec(9, 0.0, 0.0));
    robot_->setPdGains(vec(9, 30.0 + e_, 0.0), vec(9, 0.3 + 0.1 * e_, 0.0));
    robot_->setActuationLimits(vec(9, 10.0 + e_, 0.0), vec(9, -10.0 - e_, 0.0));
    robot_->getMass()[2] = 0.5 + 0.1 * e_;
    robot_->updateMassInfo();
    robot_->setCollisionBodyFriction(0, 0.2 + 0.1 * e_);
    robot_->setActuationDelay(size_t(e_ % 3));
    if (e_ != 1) robot_->resetActuatorHistory();
    steps_ = 0;
  }
  float step(const raisim::RowRef& a) final {
    mark("step " + std::to_string(e_));
    VecDyn pt = stance(0.3 * e_);
    for (int i = 0; i < 3; i++) pt[7 + i] += 0.1 * a[i];
    robot_->setPdTarget(pt, vec(9, 0.0, 0.0));
    robot_->setGeneralizedForce(vec(9, 0.1 * e_, 0.01));
    for (int i = 0; i < 4; i++) world_->integrate();
    if (sync_) {
      value("M", robot_->getMassMatrix());
      value("h", robot_->getNonlinearities());
      Vec<3> p; robot_->getPosition(1, {0.1, 0.0, 0.0}, p); value("position", p);
      value("loop counter", double(world_->getContactSolver().getLoopCounter()));
    }
    VecDyn q, v;
    robot_->getState(q, v); value("gc", q); value("gv", v);
    if (sync_) return 0.f;
    value("tau", robot_->getGeneralizedForce());
    for (auto& c : robot_->getContacts()) value("contact", c.getPosition());
    Vec<3> f; robot_->getBodyContactForce(3, f); value("contact force", f);
    value("contact steps", double(robot_->getBodyContactSteps(1)));
    steps_++;
    return float(q[0]);
  }
  void observe(raisim::RowRef ob) final {
    if (sync_) { ob[0] = 0.f; return; }
    VecDyn h; std::vector<Vec<2>> xy;
    robot_->getHeightScan(h, &xy); value("scan", h);
    Vec<3> p; robot_->getBodyPosition(2, p); value("body position", p);
    value("com", robot_->getCOM());
    for (int i = 0; i < 2; i++) ob[i] = float(h[i]);
    ob[2] = float(terrain_->getHeight(xy[0][0], xy[0][1]));
    ob[3] = float(steps_);
  }
  bool isTerminalState(float& r) final { r = -1.f; return !sync_ && steps_ >= 2; }

 private:
  raisim::ArticulatedSystem* robot_ = nullptr;
  raisim::HeightMap* terrain_ = nullptr;
  bool sync_;
  int e_ = 0, steps_ = 0;
};

void vecenv(bool sync) {
  const int n = sync ? 2 : 3;
  Cfg cfg; cfg.sync = sync;
  mark("construct");
  raisim::VectorizedEnvironment<TraceEnv> vec("", cfg, n);
  mark("init");
  vec.init();
  std::vector<float> action(size_t(n) * vec.getActionDim()), ob(size_t(n) * vec.getObDim()), reward(n);
  bool done[3] = {false, false, false};
  for (int s = 0; s < 3; s++) {
    for (size_t i = 0; i < action.size(); i++) action[i] = 0.1f * float(int((i + size_t(s)) % 5) - 2);
    mark("vec step " + std::to_string(s));
    vec.step(action.data(), reward.data(), done);
    mark("vec observe " + std::to_string(s));
    vec.observe(ob.data());
    value("ob", std::vector<double>(ob.begin(), ob.end()).data(), ob.size());
  }
  mark("vec reset");
  vec.reset();
  char b[64]; std::snprintf(b, sizeof b, "launches %ld\n", vec.launches());
  rsb_stub_log() += b;
  mark("end");
}
}  // namespace

int main(int argc, char** argv) {
  const std::string what = argc > 1 ? argv[1] : "";
  try {
    if (what == "standalone") standalone();
    else if (what == "vecenv") vecenv(false);
    else if (what == "sync") vecenv(true);
    else { std::fprintf(stderr, "usage: facade_trace standalone | vecenv | sync\n"); return 2; }
  } catch (const std::exception& e) {
    std::fputs(rsb_stub_log().c_str(), stdout);
    std::fprintf(stderr, "facade_trace: %s\n", e.what());
    return 1;
  }
  std::fputs(rsb_stub_log().c_str(), stdout);
  return 0;
}
