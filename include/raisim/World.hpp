// raisim::World / raisim::ArticulatedSystem / raisim::Contact -- header-only facade over the C-ABI
// (include/rsb.h).  Keeps the reference's API surface for the hot path so RaisimGym-style
// ENVIRONMENT code compiles against it (SURVEY.md 8b lists the upstream signatures, [RECALL]:
// include/raisim/World.hpp, object/ArticulatedSystem/ArticulatedSystem.hpp, contact/Contact.hpp;
// none of them is in the reference snapshot).
//
// Design inversion: the batch lives UNDER World.  A raisim::BatchedWorld owns N environments of
// SoA state on one GPU; raisim::World and raisim::ArticulatedSystem are thin per-environment VIEWS
// {batch, env index}.  A World constructed standalone owns a batch of one (config 1 semantics).
// VectorizedEnvironment.hpp issues ONE batched launch per control step instead of N OpenMP iterations.
//
// Errors: the reference aborts through RSFATAL; here every failing C-ABI call throws
// std::runtime_error with rsb_last_error() (define RAISIM_B200_ABORT_ON_ERROR to abort instead).
// Units and conventions are the reference's: gc = [xyz | qw qx qy qz | joints], gv = [v | w | joint rates].
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <optional>
#include <stdexcept>
#include <string>
#include <vector>

#include "../rsb.h"
#include "math.hpp"

namespace raisim {

using CollisionGroup = unsigned long;

inline void rsbCheck(int rc, const char* what) {
  if (rc >= 0) return;
#ifdef RAISIM_B200_ABORT_ON_ERROR
  std::fprintf(stderr, "[RSFATAL] %s: %s\n", what, rsb_last_error());
  std::abort();
#else
  throw std::runtime_error(std::string(what) + ": " + rsb_last_error());
#endif
}

namespace ControlMode {
enum Type : int { FORCE_AND_TORQUE = RSB_FORCE_AND_TORQUE, PD_PLUS_FEEDFORWARD_TORQUE = RSB_PD_PLUS_FEEDFORWARD_TORQUE };
}

// contact::Contact read-back (ArticulatedSystem::getContacts())
class Contact {
 public:
  explicit Contact(const rsb_contact& c) : c_(c) {}
  size_t getlocalBodyIndex() const { return size_t(c_.local_body); }
  size_t getPairObjectIndex() const { return 0; }            // the terrain is object 0 of the world
  // self-collision (ArticulatedSystem::setSelfCollisionPairs): a contact between two bodies of the robot.  The impulse and the normal act
  // on getlocalBodyIndex() (normal from the other body towards it); the other body receives the negative impulse.
  bool isSelfCollision() const { return c_.pair_index < 0; }
  int getPairLocalBodyIndex() const { return c_.pair_index < 0 ? -1 - c_.pair_index : -1; }   // the other body of a self contact, -1 on terrain
  int getPairContactIndexInPairObject() const { return c_.pair_index; }
  Vec<3> getPosition() const { return {c_.position[0], c_.position[1], c_.position[2]}; }
  Vec<3> getNormal() const { return {c_.normal[0], c_.normal[1], c_.normal[2]}; }
  Vec<3> getImpulse() const { return {c_.impulse[0], c_.impulse[1], c_.impulse[2]}; }   // world frame, on the robot
  double getDepth() const { return c_.depth; }
  // Rows t1, t2, n of the contact frame (DESIGN.md section 2: t1 = normalise(e_x - (e_x . n) n), e_y when |n_x| >= 0.9; t2 = n x t1), so
  // that frame^T * (impulse in the contact frame) = world-frame impulse, the product user code forms with upstream's frame.
  Mat<3, 3> getContactFrame() const {
    const double n[3] = {c_.normal[0], c_.normal[1], c_.normal[2]};
    const int a = std::fabs(n[0]) < 0.9 ? 0 : 1;
    double t1[3] = {-n[a] * n[0], -n[a] * n[1], -n[a] * n[2]};
    t1[a] += 1.0;
    const double inv = 1.0 / std::sqrt(t1[0] * t1[0] + t1[1] * t1[1] + t1[2] * t1[2]);
    for (double& x : t1) x *= inv;
    const double t2[3] = {n[1] * t1[2] - n[2] * t1[1], n[2] * t1[0] - n[0] * t1[2], n[0] * t1[1] - n[1] * t1[0]};
    Mat<3, 3> F;
    for (int j = 0; j < 3; j++) { F(0, j) = t1[j]; F(1, j) = t2[j]; F(2, j) = n[j]; }
    return F;
  }
  Vec<3> getImpulseInContactFrame() const {       // (tangential 1, tangential 2, normal): what the solver iterates on
    const Mat<3, 3> F = getContactFrame();
    Vec<3> l;
    for (int i = 0; i < 3; i++) l[i] = F(i, 0) * c_.impulse[0] + F(i, 1) * c_.impulse[1] + F(i, 2) * c_.impulse[2];
    return l;
  }
  bool isObjectA() const { return true; }
  bool skip() const { return false; }
 private:
  rsb_contact c_;
};

// Host mirror of one batch's per-environment rows: every World / ArticulatedSystem view writes its environment's row here and reads it
// after the mirror has made it current.  Two upload policies:
//  * immediate (a stand-alone World, a view built with World(BatchedWorld*, env)): a write goes up before the setter returns, World::
//    integrate() launches at once, and a read fetches the reader's row alone -- per call, the C-ABI call of a per-environment accessor;
//  * deferred (VectorizedEnvironment<ENVIRONMENT>: N unmodified per-environment programs in lock step on one batch): World::integrate()
//    only counts.  The first access that needs the result (getState, getContacts, setPdTarget after an integrate ...) suspends that
//    environment until every environment has reached the same point; then the rows written go up in one copy per array, ONE launch
//    integrates the counted sub-steps of every environment (the usual RaisimGym loop `for (i < control_dt / simulation_dt)
//    world_->integrate();` becomes a single fused launch), and reads refill every environment's rows, one copy per array and control step.
struct LockStep {
  // rows [n][w] of one array and the environments [lo, hi) written since the last upload
  template <class T> struct Rows {
    std::vector<T> v;
    size_t w = 0;
    int lo = 0, hi = 0;
    void init(int n, size_t width, T fill) { w = width; v.assign(size_t(n) * w, fill); }
    T* row(int e) { return v.data() + size_t(e) * w; }
    bool dirty() const { return hi > lo; }
    void mark(int e) { lo = dirty() ? std::min(lo, e) : e; hi = std::max(hi, e + 1); }
    void clean() { lo = hi = 0; }
  };
  rsb_batch* batch = nullptr;
  const rsb_model* model = nullptr;
  int n = 0, nq = 0, nv = 0, nb = 0, ncoll = 0;
  bool deferred = false;
  // rows the views write; pt and vt (setPdTarget), gc and gv (setState) go up in one call each
  Rows<float> gc, gv, pt, vt, tau;
  Rows<float> bodyInertia;                  // [nb][10] inertial rows (ArticulatedSystem::updateMassInfo); empty until the first one
  Rows<float> friction;                     // [ncoll] terrain friction (World materials; -1: the batch's value); empty until the first one
  Rows<float> actuator;                     // [nv][3] kp, kd, effort limit (setPdGains / setActuationLimits; -1: the batch's); empty until the first one
  Rows<int32_t> delay;                      // [1] ArticulatedSystem::setActuationDelay since the last upload (-1: unchanged); empty until the first one
  Rows<char> actHistReset;                  // [1] ArticulatedSystem::resetActuatorHistory() since the last upload
  size_t actHistWords = 0;                  // words of one environment's actuator-network history or LSTM state (0: no network, or history 1)
  // rows the device fills: deferred, every environment's, valid until the next launch (the height scan: until the next state write or
  // terrain upload); immediate, the reader's row of the last read
  Rows<float> tauApplied, cfForce, scan, scanXy;   // [nv], [S][3] and [S] of the contact bodies (setContactBodies), [P] and [P][2] of the scan
  Rows<float> imuLin, imuAng;               // [I][3] each: the IMUs' readings (setImus)
  Rows<float> rayDist;                      // [R] the ray casts' distances (setRays), valid as the height scan is
  Rows<int32_t> rayHit;                     // [R] what each ray hit
  Rows<int32_t> ncontacts, cfSteps;
  Rows<rsb_contact> contacts;               // [RSB_KMAX]
  int cfBodies = 0, scanPoints = 0, imus = 0, rays = 0;
  bool stateValid = false, tauAppliedValid = false, contactsValid = false, cfValid = false, scanValid = false, imuValid = false, rayValid = false;
  // terrain of every environment of a deferred mirror (World::addHeightMap / addGround), uploaded by pushTerrain().  Environments holding
  // the same heights share one MapEntry; `atlas` is what the device holds, in atlas order (atlasSingle: one map set without an index)
  struct MapEntry {
    int xs = 0, ys = 0;
    double xSize = 0, ySize = 0, cx = 0, cy = 0;
    std::vector<float> h;
    uint64_t hash = 0;
    bool sameGeometry(const MapEntry& o) const { return xs == o.xs && ys == o.ys && xSize == o.xSize && ySize == o.ySize && cx == o.cx && cy == o.cy; }
    bool sameMap(const MapEntry& o) const { return hash == o.hash && sameGeometry(o) && h == o.h; }
  };
  std::vector<std::shared_ptr<const MapEntry>> envMap, atlas;   // [n] map of every environment (null: none), maps on the device
  std::vector<char> envGround;              // [n] the environment added a ground
  std::vector<int32_t> atlasIndex;          // [n] map of every environment on the device (empty with atlasSingle)
  bool atlasSingle = false, terrainDirty = false;
  long mapUploads = 0, indexUploads = 0;    // terrain calls issued: maps uploaded (rsb_batch_set_heightmap / _heightmaps), index moves
  std::vector<int> pending;                 // World::integrate() calls not executed yet, per environment
  long launches = 0;
  std::function<void(int)> suspend;         // installed by the scheduler: park the calling environment until the batch was flushed

  void init(rsb_batch* b, const rsb_model* m, int n_) {
    batch = b; model = m; n = n_;
    rsbCheck(rsb_model_dims(m, &nq, &nv, &nb, &ncoll, nullptr), "dims");
    gc.init(n, nq, 0.f); gv.init(n, nv, 0.f); pt.init(n, nq, 0.f); vt.init(n, nv, 0.f); tau.init(n, nv, 0.f);
    tauApplied.init(n, nv, 0.f); contacts.init(n, RSB_KMAX, rsb_contact{}); ncontacts.init(n, 1, 0);
    pending.assign(n, 0);
    envMap.assign(n, nullptr); envGround.assign(n, 0);
  }
  // an environment is about to read or write the world: whatever it integrated before must have happened
  void sync(int env) {
    if (pending[env] == 0) return;
    if (!suspend) throw std::runtime_error("World: state access with integrate() calls pending outside VectorizedEnvironment::step()");
    suspend(env);
  }

  // ---- writes: environment env's row of an array, marked for the next upload; commit() after filling it ----
  template <class T> T* write(int env, Rows<T>& a) { sync(env); a.mark(env); return a.row(env); }
  template <class T> T* write(int env, Rows<T>& a, size_t width, T fill) {   // an array kept empty until its first write
    if (a.v.empty()) a.init(n, width, fill);
    return write(env, a);
  }
  // gc or gv: a deferred upload spans every row between the lowest and the highest environment written, so the mirror must hold the
  // other environments' rows first; a written state also makes the height scan stale
  float* stateRow(int env, Rows<float>& a) {
    sync(env);
    if (deferred) needState(env);
    scanValid = rayValid = false;
    return write(env, a);
  }
  float* inertiaRow(int env) {               // every environment starts from the model's rows
    if (bodyInertia.v.empty()) {
      rsb_model_tables t; rsbCheck(rsb_model_get_tables(model, &t), "getTables");
      bodyInertia.init(n, size_t(nb) * 10, 0.f);
      for (int e = 0; e < n; e++)
        for (int b = 0; b < nb; b++) {
          float* r = bodyInertia.row(e) + size_t(b) * 10;
          r[0] = float(t.mass[b]);
          for (int k = 0; k < 3; k++) r[1 + k] = float(t.com[3 * b + k]);
          for (int k = 0; k < 6; k++) r[4 + k] = float(t.inertia[6 * b + k]);
        }
    }
    return write(env, bodyInertia);
  }
  float* actuatorRow(int env) { return write(env, actuator, size_t(nv) * 3, -1.f); }
  void setFriction(int env, size_t collisionBody, double mu) {
    if (collisionBody >= size_t(ncoll)) throw std::runtime_error("setCollisionBodyFriction: collision body index out of range");
    write(env, friction, size_t(ncoll), -1.f)[collisionBody] = float(mu);
    commit();
  }
  // environment env's actuator-network history goes to zero, its actuation delay is set (and its command history emptied)
  void resetActuatorHistory(int env) { *write(env, actHistReset, 1, char(0)) = 1; commit(); }
  void setActuationDelay(int env, int subSteps) { *write(env, delay, 1, int32_t(-1)) = subSteps; commit(); }
  // the rows written go up now, unless uploads wait for the next launch or device read
  void commit() { if (!deferred) pushWrites(); }

  // ---- uploads ----
  template <class T, class F> void push(Rows<T>& a, F call) {
    if (!a.dirty()) return;
    call(a.row(a.lo), a.lo, a.hi - a.lo);
    a.clean();
  }
  // two arrays one call sets: both over the union of their ranges, one nobody wrote as nullptr
  template <class F> void push(Rows<float>& a, Rows<float>& b, F call) {
    if (!a.dirty() && !b.dirty()) return;
    const int lo = !a.dirty() ? b.lo : !b.dirty() ? a.lo : std::min(a.lo, b.lo), hi = std::max(a.hi, b.hi);
    call(a.dirty() ? a.row(lo) : nullptr, b.dirty() ? b.row(lo) : nullptr, lo, hi - lo);
    a.clean(); b.clean();
  }
  // every row written since the last upload, one call per array over the environments written
  void pushWrites() {
    push(gc, gv, [&](float* q, float* v, int lo, int k) { rsbCheck(rsb_batch_set_state(batch, q, v, lo, k, RSB_HOST), "setState"); });
    push(pt, vt, [&](float* p, float* v, int lo, int k) { rsbCheck(rsb_batch_set_pd_target(batch, p, v, lo, k, RSB_HOST), "setPdTarget"); });
    push(tau, [&](float* r, int lo, int k) { rsbCheck(rsb_batch_set_generalized_force(batch, r, lo, k, RSB_HOST), "setGeneralizedForce"); });
    push(bodyInertia, [&](float* r, int lo, int k) { rsbCheck(rsb_batch_set_body_inertia(batch, r, lo, k, RSB_HOST), "updateMassInfo"); });
    push(friction, [&](float* r, int lo, int k) { rsbCheck(rsb_batch_set_contact_friction(batch, r, lo, k, RSB_HOST), "setMaterialPairProp"); });
    push(actuator, [&](float* r, int lo, int k) { rsbCheck(rsb_batch_set_actuator_params(batch, r, lo, k, RSB_HOST), "setPdGains"); });
    pushTerrain();
    // the marked environments' history rows zeroed: one call when every environment of the range was marked, else one get and one set
    push(actHistReset, [&](char* m, int lo, int k) {
      if (actHistWords > 0 && std::all_of(m, m + k, [](char c) { return c != 0; })) {
        rsbCheck(rsb_batch_set_actuator_history(batch, nullptr, lo, k, RSB_HOST), "resetActuatorHistory");
      } else if (actHistWords > 0) {
        std::vector<float> h(size_t(k) * actHistWords);
        rsbCheck(rsb_batch_get_actuator_history(batch, h.data(), lo, k, RSB_HOST), "resetActuatorHistory");
        for (int e = 0; e < k; e++)
          if (m[e]) std::fill(h.begin() + size_t(e) * actHistWords, h.begin() + size_t(e + 1) * actHistWords, 0.f);
        rsbCheck(rsb_batch_set_actuator_history(batch, h.data(), lo, k, RSB_HOST), "resetActuatorHistory");
      }
      std::fill(m, m + k, 0);
    });
    push(delay, [&](int32_t* d, int lo, int k) {
      rsbCheck(rsb_batch_set_actuation_delay(batch, d, lo, k, RSB_HOST), "setActuationDelay");
      std::fill(d, d + k, -1);
    });
  }
  // upload, then one launch of k sub-steps for every environment
  void launch(int k) {
    pushWrites();
    rsbCheck(rsb_batch_integrate(batch, k), "integrate");
    launches++;
    for (int& p : pending) p = 0;
    stateValid = tauAppliedValid = contactsValid = cfValid = scanValid = imuValid = rayValid = false;
  }
  // every environment is parked (or finished) with the same number of integrate() calls pending
  void flush() {
    int k = 0;
    for (int e = 0; e < n; e++) k = pending[e] > k ? pending[e] : k;
    if (k == 0) return;
    for (int e = 0; e < n; e++)
      if (pending[e] != k) throw std::runtime_error("VectorizedEnvironment: environments disagree on the number of World::integrate() calls between two state accesses");
    launch(k);
  }

  // ---- reads ----
  // The gate of every read the device computes from the current state and parameters (M, h, poses, the height scan, the solver's loop
  // counter): whatever env integrated has happened and every row written since is up
  void current(int env) { sync(env); pushWrites(); }
  // rows of the last launch's results, and the state: fetch(lo, count, all) refills rows [lo, lo + count), all of what the mirror keeps
  // (all) or what the reader asked for.  The mirror holds every write to them, so they need no upload
  template <class F> void refill(int env, bool& valid, F fetch) {
    sync(env);
    if (valid) return;
    if (deferred) { fetch(0, n, true); valid = true; }
    else fetch(env, 1, false);
  }
  void needState(int env) {
    refill(env, stateValid, [&](int lo, int k, bool) { rsbCheck(rsb_batch_get_state(batch, gc.row(lo), gv.row(lo), lo, k, RSB_HOST), "getState"); });
  }
  void needTauApplied(int env) {
    refill(env, tauAppliedValid, [&](int lo, int k, bool) { rsbCheck(rsb_batch_get_generalized_force(batch, tauApplied.row(lo), lo, k, RSB_HOST), "getGeneralizedForce"); });
  }
  void needContacts(int env) {
    refill(env, contactsValid, [&](int lo, int k, bool) { rsbCheck(rsb_batch_get_contacts(batch, contacts.row(lo), ncontacts.row(lo), lo, k, RSB_HOST), "getContacts"); });
  }
  void needContactForces(int env, bool force, bool steps) {
    if (cfForce.w != size_t(cfBodies) * 3) { cfForce.init(n, size_t(cfBodies) * 3, 0.f); cfSteps.init(n, size_t(cfBodies), 0); cfValid = false; }
    refill(env, cfValid, [&](int lo, int k, bool all) {
      rsbCheck(rsb_batch_get_body_contact_forces(batch, lo, k, all || force ? cfForce.row(lo) : nullptr, all || steps ? cfSteps.row(lo) : nullptr, RSB_HOST),
               "getBodyContactForce");
    });
  }
  void needImuReadings(int env, bool lin, bool ang) {
    if (imuLin.w != size_t(imus) * 3) { imuLin.init(n, size_t(imus) * 3, 0.f); imuAng.init(n, size_t(imus) * 3, 0.f); imuValid = false; }
    refill(env, imuValid, [&](int lo, int k, bool all) {
      rsbCheck(rsb_batch_get_imu_readings(batch, lo, k, all || lin ? imuLin.row(lo) : nullptr, all || ang ? imuAng.row(lo) : nullptr, RSB_HOST),
               "getImuReadings");
    });
  }
  // deferred: one call scans every environment, after the rows written since the last launch went up (a reset() that moved a robot is seen)
  void needHeightScan(int env, bool samples) {
    current(env);
    if (scan.w != size_t(scanPoints)) { scan.init(n, size_t(scanPoints), 0.f); scanXy.init(n, size_t(scanPoints) * 2, 0.f); scanValid = false; }
    refill(env, scanValid, [&](int lo, int k, bool all) {
      rsbCheck(rsb_batch_get_height_scan(batch, lo, k, scan.row(lo), all || samples ? scanXy.row(lo) : nullptr, RSB_HOST), "getHeightScan");
    });
  }
  // the ray casts, by the height scan's rule: deferred, one call casts every environment after the rows written since the last launch
  // went up
  void needRayCasts(int env, bool hits) {
    current(env);
    if (rayDist.w != size_t(rays)) { rayDist.init(n, size_t(rays), 0.f); rayHit.init(n, size_t(rays), 0); rayValid = false; }
    refill(env, rayValid, [&](int lo, int k, bool all) {
      rsbCheck(rsb_batch_get_ray_casts(batch, lo, k, rayDist.row(lo), all || hits ? rayHit.row(lo) : nullptr, RSB_HOST), "getRayCasts");
    });
  }

  // ---- terrain of a deferred mirror ----
  // environment env's height map (World::addHeightMap), uploaded with the next launch or read: environments holding the same heights
  // share one entry, found by a hash and confirmed by comparison
  void setHeightMap(int env, int xs, int ys, double xSize, double ySize, double cx, double cy, std::vector<float> h) {
    sync(env);
    auto e = std::make_shared<MapEntry>();
    e->xs = xs; e->ys = ys; e->xSize = xSize; e->ySize = ySize; e->cx = cx; e->cy = cy; e->h = std::move(h);
    uint64_t x = 1469598103934665603ull;   // FNV-1a over the float32 words
    for (float v : e->h) { uint32_t u; std::memcpy(&u, &v, 4); x = (x ^ u) * 1099511628211ull; }
    e->hash = x;
    std::shared_ptr<const MapEntry> found;
    for (const auto& m : atlas) if (!found && m->sameMap(*e)) found = m;
    for (const auto& m : envMap) if (!found && m && m->sameMap(*e)) found = m;
    envMap[size_t(env)] = found ? found : e;
    envGround[size_t(env)] = 0;
    terrainDirty = true;
  }
  // environment env added a ground, which World::addGround sets on the batch at once (dropping any map there)
  void setGround(int env) {
    envMap[size_t(env)] = nullptr; envGround[size_t(env)] = 1;
    atlas.clear(); atlasIndex.clear(); atlasSingle = false;
    terrainDirty = true;
  }
  // the environments' maps onto the device, with the cheapest call that does it: nothing when the device already has them; one index
  // move when every map in use is in the atlas (a curriculum moving environments among its levels); else one upload of the maps in use,
  // a single map when every environment holds the same heights.  An environment that added no terrain of its own shares the map of the
  // lowest-numbered environment that did (with one common map, the map every environment collided with before maps were per environment).
  // A rebuilt atlas keeps maps of the previous one that no environment holds right now (a curriculum level nobody is on), up to twice
  // as many maps as are in use, so that moving back to them needs no upload
  void pushTerrain() {
    if (!terrainDirty) return;
    int firstMap = -1, firstGround = -1, firstNone = -1;
    for (int e = 0; e < n; e++) {
      int& first = envMap[size_t(e)] ? firstMap : envGround[size_t(e)] ? firstGround : firstNone;
      if (first < 0) first = e;
    }
    if (firstMap < 0) { terrainDirty = false; return; }
    if (firstGround >= 0)
      throw std::runtime_error("VectorizedEnvironment: environment " + std::to_string(firstGround) + " added a ground and environment " + std::to_string(firstMap) +
                               " a height map; every environment must use the same kind of terrain");
    std::vector<std::shared_ptr<const MapEntry>> use(envMap);
    for (auto& m : use) if (!m) m = envMap[size_t(firstMap)];
    const MapEntry& g = *use[size_t(firstMap)];
    for (int e = 0; e < n; e++)
      if (!use[size_t(e)]->sameGeometry(g))
        throw std::runtime_error("VectorizedEnvironment: the height maps of environments " + std::to_string(firstMap) + " and " + std::to_string(e) +
                                 " differ in samples, size or centre; the maps of one batch must share them");
    std::vector<int32_t> idx(size_t(n), -1);
    bool inAtlas = true;
    for (int e = 0; e < n && inAtlas; e++) {
      for (size_t m = 0; m < atlas.size(); m++) if (atlas[m] == use[size_t(e)]) { idx[size_t(e)] = int32_t(m); break; }
      inAtlas = idx[size_t(e)] >= 0;
    }
    if (inAtlas && !atlasSingle) {
      int lo = 0, hi = n;
      while (lo < n && idx[size_t(lo)] == atlasIndex[size_t(lo)]) lo++;
      while (hi > lo && idx[size_t(hi - 1)] == atlasIndex[size_t(hi - 1)]) hi--;
      if (hi > lo) {
        rsbCheck(rsb_batch_set_heightmap_index(batch, idx.data() + lo, lo, hi - lo, RSB_HOST), "addHeightMap");
        atlasIndex = idx;
        indexUploads++;
      }
    } else if (!inAtlas) {
      std::vector<std::shared_ptr<const MapEntry>> maps;   // the maps in use, in order of first appearance
      for (int e = 0; e < n; e++) {
        size_t m = 0;
        while (m < maps.size() && maps[m] != use[size_t(e)]) m++;
        if (m == maps.size()) maps.push_back(use[size_t(e)]);
        idx[size_t(e)] = int32_t(m);
      }
      const size_t inUse = maps.size();
      for (const auto& old : atlas)
        if (maps.size() < 2 * inUse && old->sameGeometry(g) && std::find(maps.begin(), maps.end(), old) == maps.end()) maps.push_back(old);
      atlas.clear(); atlasIndex.clear();
      if (maps.size() == 1) {
        rsbCheck(rsb_batch_set_heightmap(batch, g.xs, g.ys, float(g.xSize), float(g.ySize), float(g.cx), float(g.cy), g.h.data()), "addHeightMap");
        atlasSingle = true;
      } else {
        std::vector<float> all;
        all.reserve(maps.size() * g.h.size());
        for (const auto& m : maps) all.insert(all.end(), m->h.begin(), m->h.end());
        rsbCheck(rsb_batch_set_heightmaps(batch, int(maps.size()), g.xs, g.ys, float(g.xSize), float(g.ySize), float(g.cx), float(g.cy), all.data(), idx.data()), "addHeightMap");
        atlasSingle = false; atlasIndex = idx;
      }
      atlas = std::move(maps);
      mapUploads++;
    }
    terrainDirty = false;
    scanValid = rayValid = false;
  }
};

// One GPU batch of N identical worlds (new; the reference has no equivalent -- its batching is the
// OpenMP loop of VectorizedEnvironment).
class BatchedWorld {
 public:
  BatchedWorld(const std::string& urdfPathOrXml, int numEnvs, int device = 0) {
    rsbCheck(rsb_model_create_from_urdf(urdfPathOrXml.c_str(), &model_), "addArticulatedSystem");
    rsbCheck(rsb_batch_create(model_, numEnvs, device, &batch_), "BatchedWorld");
    rsbCheck(rsb_model_dims(model_, &nq_, &nv_, &nb_, nullptr, nullptr), "dims");
    n_ = numEnvs;
    ls_.init(batch_, model_, n_);
  }
  ~BatchedWorld() { if (batch_) rsb_batch_destroy(batch_); if (model_) rsb_model_destroy(model_); }
  BatchedWorld(const BatchedWorld&) = delete;
  BatchedWorld& operator=(const BatchedWorld&) = delete;
  rsb_batch* batch() const { return batch_; }
  rsb_model* model() const { return model_; }
  int numEnvs() const { return n_; }
  int nq() const { return nq_; }
  int nv() const { return nv_; }
  int nb() const { return nb_; }
  rsb_params params() const { rsb_params p; rsbCheck(rsb_batch_get_params(batch_, &p), "getParams"); return p; }
  void setParams(const rsb_params& p) { rsbCheck(rsb_batch_set_params(batch_, &p), "setParams"); }
  void integrate(int substeps = 1) { rsbCheck(rsb_batch_integrate(batch_, substeps), "integrate"); worldTime_ += substeps * params().dt; }
  void integrate1() { rsbCheck(rsb_batch_integrate1(batch_), "integrate1"); }
  void integrate2() { rsbCheck(rsb_batch_integrate2(batch_), "integrate2"); worldTime_ += params().dt; }
  double worldTime() const { return worldTime_; }
  void advanceTime(double t) { worldTime_ += t; }
  // the host mirror every view reads and writes through; lock-step mode (VectorizedEnvironment<ENVIRONMENT>) defers its uploads
  LockStep* lockStep() { return &ls_; }
  void enableLockStep() { ls_.deferred = true; }
  // World::integrate() of environment env: deferred, one more sub-step for the next launch (the world time follows environment 0);
  // immediate, one launch now.  Returns whether it launched
  bool integrateEnv(int env) {
    if (ls_.deferred) {
      ls_.pending[env]++;
      if (env == 0) advanceTime(params().dt);
      return false;
    }
    ls_.launch(1);
    advanceTime(params().dt);
    return true;
  }
  // ---- what a stand-alone World sets for its batch and a VectorizedEnvironment per environment ----
  // PD gains in the batch's gv order: a stand-alone World's are its batch's; in a VectorizedEnvironment each environment's are its own,
  // kept in its actuator row and uploaded before the next launch (no launch of their own), as upstream's per-World gains are
  void setPdGains(int env, const std::vector<float>& kp, const std::vector<float>& kd) {
    if (!ls_.deferred) { rsbCheck(rsb_batch_set_pd_gains(batch_, kp.data(), kd.data()), "setPdGains"); return; }
    float* r = ls_.actuatorRow(env);
    for (int i = 0; i < nv_; i++) { r[3 * i] = kp[size_t(i)]; r[3 * i + 1] = kd[size_t(i)]; }
  }
  // friction of one collision body against the terrain (mu < 0: the default material): a stand-alone World sets it for its batch; in a
  // VectorizedEnvironment it is environment env's own, kept in its friction row and uploaded with the next launch
  // (include/rsb.h rsb_batch_set_contact_friction)
  void setCollisionFriction(int env, size_t collisionBody, double mu) {
    if (ls_.deferred) ls_.setFriction(env, collisionBody, mu);
    else rsbCheck(rsb_batch_set_collision_friction(batch_, int(collisionBody), float(mu)), "setCollisionBodyFriction");
  }
  // World's materials of environment env: pairMu holds each collision body with a material and the friction of its pair with the
  // terrain's material (none: no such pair), defaultMu the environment's setDefaultMaterial friction (< 0: not set).  A stand-alone World
  // sets the friction of those bodies for its batch (-1 without a pair); in a VectorizedEnvironment they fill environment env's whole
  // friction row, the default where a body has no pair
  void setMaterialFriction(int env, const std::map<size_t, std::optional<double>>& pairMu, double defaultMu) {
    if (!ls_.deferred) {
      for (const auto& kv : pairMu) setCollisionFriction(env, kv.first, kv.second ? *kv.second : -1.0);
      return;
    }
    if (ls_.friction.v.empty() && pairMu.empty() && defaultMu < 0) return;   // every entry -1: no rows needed
    for (int c = 0; c < ls_.ncoll; c++) {
      auto m = pairMu.find(size_t(c));
      setCollisionFriction(env, size_t(c), m != pairMu.end() && m->second ? *m->second : defaultMu);
    }
  }
  // setDefaultMaterial: restitution is the batch's.  The friction is rsb_params.mu for a stand-alone World, which self-collision pairs
  // use too; in a VectorizedEnvironment it is environment env's own, through its friction row, and self pairs keep the batch's mu
  void setDefaultMaterial(int env, double friction, double restitution, double resThreshold, const std::map<size_t, std::optional<double>>& pairMu) {
    rsb_params p = params(); p.restitution = float(restitution); p.rest_threshold = float(resThreshold);
    if (!ls_.deferred) p.mu = float(friction);
    setParams(p);
    if (ls_.deferred) setMaterialFriction(env, pairMu, friction);
  }
  // terrain: a stand-alone World, or a view, sets it for the whole batch at once; in a VectorizedEnvironment each environment's map is
  // its own, uploaded with the next launch or read (LockStep::pushTerrain), and a ground is set at once
  void setHeightMap(int env, int xs, int ys, double xSize, double ySize, double cx, double cy, const std::vector<float>& h) {
    if (ls_.deferred) ls_.setHeightMap(env, xs, ys, xSize, ySize, cx, cy, h);
    else rsbCheck(rsb_batch_set_heightmap(batch_, xs, ys, float(xSize), float(ySize), float(cx), float(cy), h.data()), "addHeightMap");
  }
  void setGround(int env, double z) {
    if (ls_.deferred) ls_.setGround(env);
    rsbCheck(rsb_batch_set_ground(batch_, float(z)), "addGround");
  }
  // bodies whose contact force every integrate() gathers (ArticulatedSystem::setContactBodies): one list for all environments
  void setContactBodies(const std::vector<size_t>& bodies) {
    if (bodies == contactBodies_) return;      // every environment of a VectorizedEnvironment sets the same list in its constructor
    std::vector<int32_t> b(bodies.begin(), bodies.end());
    rsbCheck(rsb_batch_set_contact_bodies(batch_, b.data(), int(b.size())), "setContactBodies");
    contactBodies_ = bodies;
    ls_.cfBodies = int(bodies.size()); ls_.cfValid = false;
  }
  size_t contactBodySlot(size_t bodyIdx) const {
    for (size_t s = 0; s < contactBodies_.size(); s++) if (contactBodies_[s] == bodyIdx) return s;
    throw std::runtime_error("getBodyContactForce: body " + std::to_string(bodyIdx) + " is not among the bodies given to setContactBodies()");
  }
  size_t numContactBodies() const { return contactBodies_.size(); }
  // IMUs at model frames (ArticulatedSystem::setImus): one list for all environments
  void setImus(const std::vector<size_t>& frames) {
    if (frames == imuFrames_) return;          // every environment of a VectorizedEnvironment sets the same list in its constructor
    std::vector<int32_t> body(frames.size());
    std::vector<float> pos(3 * frames.size()), rot(9 * frames.size());
    for (size_t k = 0; k < frames.size(); k++) {
      double p[3], r[9];
      rsbCheck(rsb_model_frame(model_, int(frames[k]), &body[k], p, r), "setImus");
      for (int c = 0; c < 3; c++) pos[3 * k + c] = float(p[c]);
      for (int c = 0; c < 9; c++) rot[9 * k + c] = float(r[c]);
    }
    rsbCheck(rsb_batch_set_imus(batch_, body.data(), pos.data(), rot.data(), int(frames.size())), "setImus");
    imuFrames_ = frames;
    ls_.imus = int(frames.size()); ls_.imuValid = false;
  }
  size_t numImus() const { return imuFrames_.size(); }
  // terrain height-scan points (ArticulatedSystem::setHeightScan): one list for all environments
  void setHeightScan(const std::vector<int32_t>& bodies, const std::vector<float>& xy, bool yawAligned) {
    if (bodies == scanBodies_ && xy == scanXy_ && yawAligned == scanYaw_) return;   // every environment sets the same list in its constructor
    if (xy.size() != 2 * bodies.size()) throw std::runtime_error("setHeightScan: one offset per body");
    rsbCheck(rsb_batch_set_height_scan(batch_, bodies.data(), xy.data(), int(bodies.size()), yawAligned ? RSB_SCAN_YAW : RSB_SCAN_WORLD), "setHeightScan");
    scanBodies_ = bodies; scanXy_ = xy; scanYaw_ = yawAligned;
    ls_.scanPoints = int(bodies.size()); ls_.scanValid = false;
  }
  size_t numHeightScanPoints() const { return scanBodies_.size(); }
  // rays (ArticulatedSystem::setRays): one list for all environments
  void setRays(const std::vector<int32_t>& bodies, const std::vector<float>& origins, const std::vector<float>& dirs, float maxDistance, bool seeRobot) {
    if (bodies == rayBodies_ && origins == rayOrigins_ && dirs == rayDirs_ && maxDistance == rayMax_ && seeRobot == raySeeRobot_) return;   // every environment sets the same list in its constructor
    if (origins.size() != 3 * bodies.size() || dirs.size() != 3 * bodies.size()) throw std::runtime_error("setRays: one origin and one direction per body");
    rsbCheck(rsb_batch_set_rays(batch_, bodies.data(), origins.data(), dirs.data(), int(bodies.size()), maxDistance,
                                seeRobot ? RSB_RAYS_TERRAIN_AND_ROBOT : RSB_RAYS_TERRAIN), "setRays");
    rayBodies_ = bodies; rayOrigins_ = origins; rayDirs_ = dirs; rayMax_ = maxDistance; raySeeRobot_ = seeRobot;
    ls_.rays = int(bodies.size()); ls_.rayValid = false;
  }
  size_t numRays() const { return rayBodies_.size(); }
  // the learned actuator network (ArticulatedSystem::setActuatorNetwork): one for the batch.  Setting it zeroes every history, so a
  // repeat of the network already set (every environment of a VectorizedEnvironment sets it in its constructor) is not passed on
  void setActuatorNetwork(const std::vector<int32_t>& dofs, int history, int layers, int width, const std::vector<float>& params) {
    if (!anLstm_ && dofs == anDofs_ && history == anH_ && layers == anL_ && width == anW_ && params == anParams_) return;
    if (!dofs.empty()) {
      const size_t count = size_t(2 * history) * width + width + size_t(layers - 1) * (size_t(width) * width + width) + width + 1;
      if (history < 1 || layers < 1 || width < 1 || params.size() != count)
        throw std::runtime_error("setActuatorNetwork: " + std::to_string(params.size()) + " parameters for history " + std::to_string(history) +
                                 ", " + std::to_string(layers) + " layers of width " + std::to_string(width));
    }
    rsbCheck(rsb_batch_set_actuator_network(batch_, dofs.data(), int(dofs.size()), history, layers, width, params.data()), "setActuatorNetwork");
    anLstm_ = false; anDofs_ = dofs; anH_ = history; anL_ = layers; anW_ = width; anParams_ = params;
    ls_.actHistWords = dofs.empty() ? 0 : dofs.size() * 2 * size_t(history - 1); ls_.actHistReset = {};
  }
  // the LSTM actuator network (ArticulatedSystem::setActuatorLstm), in place of any network set before; a repeat of the one already
  // set is not passed on, as for setActuatorNetwork
  void setActuatorLstm(const std::vector<int32_t>& dofs, int layers, int hidden, const std::vector<float>& params) {
    if (anLstm_ && dofs == anDofs_ && layers == anL_ && hidden == anW_ && params == anParams_) return;
    if (!dofs.empty()) {
      size_t count = size_t(hidden) + 1;
      for (int l = 0; l < layers; l++) count += size_t(4 * hidden) * ((l == 0 ? 2 : hidden) + hidden + 2);
      if (layers < 1 || hidden < 1 || params.size() != count)
        throw std::runtime_error("setActuatorLstm: " + std::to_string(params.size()) + " parameters for " + std::to_string(layers) +
                                 " layers of hidden size " + std::to_string(hidden));
    }
    rsbCheck(rsb_batch_set_actuator_lstm(batch_, dofs.data(), int(dofs.size()), layers, hidden, params.data()), "setActuatorLstm");
    anLstm_ = true; anDofs_ = dofs; anH_ = 0; anL_ = layers; anW_ = hidden; anParams_ = params;
    ls_.actHistWords = dofs.size() * size_t(layers) * 2 * size_t(hidden); ls_.actHistReset = {};
  }
  // zero environment env's actuator history, and set its actuation delay in sub-steps (ArticulatedSystem::setActuationDelay)
  void resetActuatorHistory(int env) { ls_.resetActuatorHistory(env); }
  void setActuationDelay(int env, int subSteps) { ls_.setActuationDelay(env, subSteps); }
  // getContactSolver().getLoopCounter() of environment env
  int solverIterations(int env) {
    ls_.current(env);
    int32_t it = 0;
    rsbCheck(rsb_batch_get_solver_iterations(batch_, &it, env, 1, RSB_HOST), "getLoopCounter");
    return it;
  }
  const std::string& urdf() const { return urdf_; }
  void rememberUrdf(const std::string& u) { urdf_ = u; }
 private:
  LockStep ls_;
  std::vector<size_t> contactBodies_;
  std::vector<size_t> imuFrames_;
  std::vector<int32_t> scanBodies_;
  std::vector<float> scanXy_;
  std::vector<int32_t> rayBodies_;
  std::vector<float> rayOrigins_, rayDirs_;
  float rayMax_ = 0.f;
  bool raySeeRobot_ = false;
  std::vector<int32_t> anDofs_;
  bool anLstm_ = false;                  // anDofs_ .. anParams_ describe the LSTM (setActuatorLstm), else the MLP
  int anH_ = 0, anL_ = 0, anW_ = 0;
  std::vector<float> anParams_;
  bool scanYaw_ = true;
  std::string urdf_;
  rsb_model* model_ = nullptr;
  rsb_batch* batch_ = nullptr;
  int n_ = 0, nq_ = 0, nv_ = 0, nb_ = 0;
  double worldTime_ = 0;
};

// raisim::Ground / raisim::HeightMap ([RECALL] object/terrain/Ground.hpp, HeightMap.hpp): host-side descriptions of the terrain the
// batch collides with -- what user code queries when it places a robot (getHeight) or builds height scans
class Ground {
 public:
  double getHeight(double /*x*/ = 0, double /*y*/ = 0) const { return z_; }
  void setHeight(double z) { z_ = z; }
 private:
  double z_ = 0;
};
class HeightMap {
 public:
  void set(size_t xs, size_t ys, double xSize, double ySize, double cx, double cy, std::vector<double> h) {
    xs_ = xs; ys_ = ys; xSize_ = xSize; ySize_ = ySize; cx_ = cx; cy_ = cy; h_ = std::move(h);
  }
  size_t getXSamples() const { return xs_; }
  size_t getYSamples() const { return ys_; }
  double getXSize() const { return xSize_; }
  double getYSize() const { return ySize_; }
  double getCenterX() const { return cx_; }
  double getCenterY() const { return cy_; }
  const std::vector<double>& getHeightVector() const { return h_; }
  // height of the collision surface at (x, y): the triangle of the cell beneath the point, two triangles per cell split along the
  // P00-P11 diagonal exactly as the narrow phase does (DESIGN.md section 2); outside the map: the nearest border point
  double getHeight(double x, double y) const {
    if (xs_ < 2 || ys_ < 2) return 0.0;
    const double dx = xSize_ / double(xs_ - 1), dy = ySize_ / double(ys_ - 1);
    double gx = (x - (cx_ - 0.5 * xSize_)) / dx, gy = (y - (cy_ - 0.5 * ySize_)) / dy;
    gx = std::fmin(std::fmax(gx, 0.0), double(xs_ - 1)); gy = std::fmin(std::fmax(gy, 0.0), double(ys_ - 1));
    size_t ix = size_t(gx), iy = size_t(gy);
    if (ix > xs_ - 2) ix = xs_ - 2;
    if (iy > ys_ - 2) iy = ys_ - 2;
    const double fx = gx - double(ix), fy = gy - double(iy);
    const double h00 = h_[iy * xs_ + ix], h10 = h_[iy * xs_ + ix + 1], h01 = h_[(iy + 1) * xs_ + ix], h11 = h_[(iy + 1) * xs_ + ix + 1];
    return fx >= fy ? h00 + (h10 - h00) * fx + (h11 - h10) * fy : h00 + (h11 - h01) * fx + (h01 - h00) * fy;
  }
 private:
  size_t xs_ = 0, ys_ = 0;
  double xSize_ = 0, ySize_ = 0, cx_ = 0, cy_ = 0;
  std::vector<double> h_;
};

// ArticulatedSystem::getSparseJacobian(): the non-zero columns of a 3 x dof Jacobian (the ancestors' dofs only)
class SparseJacobian {
 public:
  size_t size = 0;             // number of non-zero columns
  std::vector<size_t> idx;     // their generalized-velocity indices, ascending
  MatDyn v;                    // 3 x size
  void resize(size_t cols) { size = cols; idx.assign(cols, 0); v.resize(3, cols); }
};

// ArticulatedSystem::setIntegrationScheme ([RECALL] ArticulatedSystem.hpp)
enum class IntegrationScheme : int { TRAPEZOID = 0, SEMI_IMPLICIT, EULER, RUNGE_KUTTA_4 };

// raisim::TerrainProperties ([RECALL] include/raisim/object/terrain/HeightMap.hpp)
struct TerrainProperties {
  double frequency = 0.1, xSize = 10.0, ySize = 10.0, zScale = 2.0, fractalLacunarity = 2.0, fractalGain = 0.5, stepSize = 0.0, heightOffset = 0.0;
  size_t xSamples = 100, ySamples = 100, fractalOctaves = 5;
  std::uint32_t seed = 1;
};

// raisim::ArticulatedSystem -- a view of one environment's robot
class ArticulatedSystem {
 public:
  ArticulatedSystem(BatchedWorld* w, int env) : w_(w), m_(*w->lockStep()), env_(env) { setJointOrder({}); }
  // upstream addArticulatedSystem(urdf, resDir, jointOrder): the order of the joints in gc / gv as the caller wants it.  The batch keeps
  // its depth-first order; this view permutes on the way in and out (base coordinates first, as always).
  void setJointOrder(const std::vector<std::string>& jointOrder) {
    qmap_.resize(size_t(w_->nq())); vmap_.resize(size_t(w_->nv()));
    for (size_t i = 0; i < qmap_.size(); i++) qmap_[i] = int(i);
    for (size_t i = 0; i < vmap_.size(); i++) vmap_[i] = int(i);
    if (jointOrder.empty()) return;
    rsb_model_tables t; rsbCheck(rsb_model_get_tables(w_->model(), &t), "getTables");
    const int nj = t.nb - 1, q0 = t.floating ? 7 : 0, v0 = t.floating ? 6 : 0;
    if (int(jointOrder.size()) != nj) throw std::runtime_error("addArticulatedSystem: jointOrder must name every movable joint exactly once");
    std::vector<bool> seen(size_t(t.nb), false);
    for (int k = 0; k < nj; k++) {
      int body = -1;
      for (int b = 1; b < t.nb; b++) if (jointOrder[k] == rsb_model_joint_name(w_->model(), b)) body = b;
      if (body < 0 || seen[body]) throw std::runtime_error("addArticulatedSystem: jointOrder names an unknown joint or one joint twice: '" + jointOrder[k] + "'");
      seen[body] = true;
      qmap_[q0 + k] = t.qidx[body]; vmap_[v0 + k] = t.vidx[body];
    }
  }
  size_t getGeneralizedCoordinateDim() const { return size_t(w_->nq()); }
  size_t getDOF() const { return size_t(w_->nv()); }
  void setName(const std::string& n) { name_ = n; }
  const std::string& getName() const { return name_; }

  // State, targets and forces go through this environment's rows of the batch's host mirror (LockStep), permuted between the caller's
  // joint order and the batch's by fromBatch / toBatch
  void getState(VecDyn& gc, VecDyn& gv) const {
    m_.needState(env_);
    gc = fromBatch(m_.gc.row(env_), qmap_); gv = fromBatch(m_.gv.row(env_), vmap_);
  }
  VecDyn getGeneralizedCoordinate() const { VecDyn q, v; getState(q, v); return q; }
  VecDyn getGeneralizedVelocity() const { VecDyn q, v; getState(q, v); return v; }
  template <class VQ, class VV> void setState(const VQ& gc, const VV& gv) {
    toBatch(gc, qmap_, m_.stateRow(env_, m_.gc)); toBatch(gv, vmap_, m_.stateRow(env_, m_.gv)); m_.commit();
  }
  template <class VQ> void setGeneralizedCoordinate(const VQ& gc) { toBatch(gc, qmap_, m_.stateRow(env_, m_.gc)); m_.commit(); }
  template <class VV> void setGeneralizedVelocity(const VV& gv) { toBatch(gv, vmap_, m_.stateRow(env_, m_.gv)); m_.commit(); }
  template <class VV> void setGeneralizedForce(const VV& tau) { toBatch(tau, vmap_, m_.write(env_, m_.tau)); m_.commit(); }
  // A stand-alone World sets the gains of its batch; in a VectorizedEnvironment they are this environment's own (BatchedWorld::setPdGains)
  template <class VV> void setPdGains(const VV& p, const VV& d) {
    std::vector<float> kp(size_t(w_->nv())), kd(size_t(w_->nv()));
    toBatch(p, vmap_, kp.data()); toBatch(d, vmap_, kd.data());
    w_->setPdGains(env_, kp, kd);
  }
  template <class VQ, class VV> void setPdTarget(const VQ& posTarget, const VV& velTarget) {
    toBatch(posTarget, qmap_, m_.write(env_, m_.pt)); toBatch(velTarget, vmap_, m_.write(env_, m_.vt)); m_.commit();
  }
  void setControlMode(ControlMode::Type m) { rsbCheck(rsb_batch_set_control_mode(w_->batch(), int(m)), "setControlMode"); }

  // lazy getters: always describe the current state (the C-ABI refreshes M, h and the poses when the state changed)
  MatDyn getMassMatrix() const {
    const int nv = w_->nv();
    std::vector<float> m(size_t(nv) * nv);
    m_.current(env_);
    rsbCheck(rsb_batch_get_mass_matrix(w_->batch(), env_, 1, m.data(), RSB_HOST), "getMassMatrix");
    MatDyn M; M.resize(nv, nv);
    for (int i = 0; i < nv; i++) for (int j = 0; j < nv; j++) M(i, j) = m[vi(size_t(i)) * size_t(nv) + vi(size_t(j))];   // the caller's dof order (jointOrder)
    return M;
  }
  // M^-1 from the lazy M getter (dense Cholesky on the host: a convenience getter, not the hot path -- the kernel
  // never forms M^-1, it keeps the branch-sparse factor on chip)
  MatDyn getInverseMassMatrix() const {
    MatDyn M = getMassMatrix();
    const int n = int(M.rows());
    std::vector<double> L(size_t(n) * n, 0.0);
    for (int j = 0; j < n; j++) {
      double s = M(j, j);
      for (int k = 0; k < j; k++) s -= L[j * n + k] * L[j * n + k];
      const double d = std::sqrt(s);
      L[j * n + j] = d;
      for (int i = j + 1; i < n; i++) {
        double t = M(i, j);
        for (int k = 0; k < j; k++) t -= L[i * n + k] * L[j * n + k];
        L[i * n + j] = t / d;
      }
    }
    MatDyn Minv; Minv.resize(n, n);
    std::vector<double> x(n);
    for (int c = 0; c < n; c++) {
      for (int i = 0; i < n; i++) { double s = (i == c) ? 1.0 : 0.0; for (int k = 0; k < i; k++) s -= L[i * n + k] * x[k]; x[i] = s / L[i * n + i]; }
      for (int i = n - 1; i >= 0; i--) { double s = x[i]; for (int k = i + 1; k < n; k++) s -= L[k * n + i] * x[k]; x[i] = s / L[i * n + i]; }
      for (int i = 0; i < n; i++) Minv(i, c) = x[i];
    }
    return Minv;
  }
  VecDyn getGeneralizedForce() const { m_.needTauApplied(env_); return fromBatch(m_.tauApplied.row(env_), vmap_); }
  // upstream: setExternalForce(localIdx, force) acts at the body COM, setExternalForce(localIdx, pos_in_body, force) at a
  // point fixed in the body, setExternalTorque(localIdx, torque); world frame, valid for the next integrate() only.
  // One wrench (force + torque on the same body) per environment.
  void setExternalForce(size_t localIdx, const Vec<3>& force) {
    rsb_model_tables t; rsbCheck(rsb_model_get_tables(w_->model(), &t), "getTables");
    Vec<3> c{comOf(t, int(localIdx), 0), comOf(t, int(localIdx), 1), comOf(t, int(localIdx), 2)};
    setExternalForce(localIdx, c, force);
  }
  void setExternalForce(size_t localIdx, const Vec<3>& posInBody, const Vec<3>& force) {
    if (extBody_ >= 0 && extBody_ != int(localIdx)) throw std::runtime_error("setExternalForce: one external wrench per environment (force and torque must act on the same body)");
    extBody_ = int(localIdx); extHasForce_ = true;
    for (int k = 0; k < 3; k++) { extF_[k] = float(force[k]); extP_[k] = float(posInBody[k]); }
    pushWrench();
  }
  void setExternalTorque(size_t localIdx, const Vec<3>& torque) {
    if (extBody_ >= 0 && extBody_ != int(localIdx)) throw std::runtime_error("setExternalTorque: one external wrench per environment (force and torque must act on the same body)");
    extBody_ = int(localIdx);
    for (int k = 0; k < 3; k++) extT_[k] = float(torque[k]);
    pushWrench();
  }
  void clearExternalWrench() { extBody_ = -1; extHasForce_ = false; for (int k = 0; k < 3; k++) extF_[k] = extT_[k] = extP_[k] = 0.f; }   // called by World::integrate()
  // upstream: robot->getCollisionBody("LF_FOOT/0").setMaterial("rubber"); world.setMaterialPairProp("rubber", "default", mu, ...)
  class CollisionBodyRef {
   public:
    CollisionBodyRef(ArticulatedSystem* a, size_t idx) : a_(a), idx_(idx) {}
    void setMaterial(const std::string& name) { a_->collisionMaterial_[idx_] = name; a_->materialsDirty_ = true; }
    const std::string& getMaterial() const { static const std::string d = "default"; auto it = a_->collisionMaterial_.find(idx_); return it == a_->collisionMaterial_.end() ? d : it->second; }
    size_t index() const { return idx_; }
   private:
    ArticulatedSystem* a_; size_t idx_;
  };
  CollisionBodyRef getCollisionBody(const std::string& name) {
    int i = rsb_model_collision_index(w_->model(), name.c_str());
    rsbCheck(i, "getCollisionBody");
    return CollisionBodyRef(this, size_t(i));
  }
  const std::map<size_t, std::string>& collisionMaterials() const { return collisionMaterial_; }
  bool materialsDirty() const { return materialsDirty_; }
  void materialsApplied() { materialsDirty_ = false; }
  // friction of one collision body against the terrain (upstream: getCollisionBody(name).setMaterial + setMaterialPairProp); mu < 0:
  // the default material.  A stand-alone World sets it for its batch; in a VectorizedEnvironment it is this environment's own
  // (BatchedWorld::setCollisionFriction)
  void setCollisionBodyFriction(size_t collisionBodyIdx, double mu) { w_->setCollisionFriction(env_, collisionBodyIdx, mu); }
  // Self-collision.  Upstream checks the bodies of an articulated system against each other and user code switches single pairs off
  // with ignoreCollisionBetween; here self-collision is OFF until explicit pairs of collision bodies are enabled ("LINK/k" names as in
  // getCollisionBody; at most RSB_MAX_SELF_PAIRS; sphere / capsule pairs and sphere-box), optionally each with its own friction.  The
  // pairs hold for every environment of the batch.  An empty list switches self-collision off again.
  void setSelfCollisionPairs(const std::vector<std::pair<std::string, std::string>>& pairs, const std::vector<double>& mu = {}) {
    if (!mu.empty() && mu.size() != pairs.size()) throw std::runtime_error("setSelfCollisionPairs: one friction value per pair");
    std::vector<int32_t> idx;
    for (const auto& p : pairs) {
      for (const std::string* n : {&p.first, &p.second}) {
        const int i = rsb_model_collision_index(w_->model(), n->c_str());
        rsbCheck(i, "setSelfCollisionPairs");
        idx.push_back(i);
      }
    }
    applySelfPairs(idx, std::vector<float>(mu.begin(), mu.end()));
  }
  // removes the enabled self-collision pairs between the two bodies (local body indices), in either order
  void ignoreCollisionBetween(size_t bodyIdx1, size_t bodyIdx2) {
    rsb_model_tables t{};
    rsbCheck(rsb_model_get_tables(w_->model(), &t), "ignoreCollisionBetween");
    std::vector<int32_t> idx; std::vector<float> mu;
    for (size_t j = 0; j < selfMu_.size(); j++) {
      const int b1 = t.cbody[selfPairs_[2 * j]], b2 = t.cbody[selfPairs_[2 * j + 1]];
      if ((b1 == int(bodyIdx1) && b2 == int(bodyIdx2)) || (b1 == int(bodyIdx2) && b2 == int(bodyIdx1))) continue;
      idx.push_back(selfPairs_[2 * j]); idx.push_back(selfPairs_[2 * j + 1]); mu.push_back(selfMu_[j]);
    }
    applySelfPairs(idx, mu);
  }
  size_t getNumberOfSelfCollisionPairs() const { return selfMu_.size(); }
  VecDyn getNonlinearities() const {
    std::vector<float> h(w_->nv());
    m_.current(env_);
    rsbCheck(rsb_batch_get_nonlinearities(w_->batch(), env_, 1, h.data(), RSB_HOST), "getNonlinearities");
    return fromBatch(h.data(), vmap_);
  }
  size_t getBodyIdx(const std::string& name) const {
    int i = rsb_model_body_index(w_->model(), name.c_str());
    rsbCheck(i, "getBodyIdx");
    return size_t(i);
  }
  size_t getFrameIdxByName(const std::string& name) const {
    int i = rsb_model_frame_index(w_->model(), name.c_str());
    rsbCheck(i, "getFrameIdxByName");
    return size_t(i);
  }
  void getPosition(size_t bodyIdx, const Vec<3>& pointInBody, Vec<3>& out) const {
    const Poses P = poses();
    const float* R = &P.R[bodyIdx * 9]; const float* p = &P.p[bodyIdx * 3];
    for (int r = 0; r < 3; r++) out[r] = p[r] + R[3 * r] * pointInBody[0] + R[3 * r + 1] * pointInBody[1] + R[3 * r + 2] * pointInBody[2];
  }
  // ---- kinematic getters (host algebra on body poses the kernel computes for the current state) ----
  // upstream: getBodyPosition/Orientation, getFramePosition/Orientation/Velocity/AngularVelocity,
  // getVelocity/getAngularVelocity(bodyIdx), getDenseJacobian(bodyIdx, point_W, J), getDenseRotationalJacobian,
  // getDenseFrameJacobian / getDenseFrameRotationalJacobian ([RECALL] ArticulatedSystem.hpp; SURVEY.md 8b)
  void getBodyPosition(size_t bodyIdx, Vec<3>& out) const { Poses P = poses(); for (int r = 0; r < 3; r++) out[r] = P.p[bodyIdx * 3 + r]; }
  void getBodyOrientation(size_t bodyIdx, Mat<3, 3>& out) const {
    Poses P = poses();
    for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) out(r, c) = P.R[bodyIdx * 9 + 3 * r + c];
  }
  void getBasePosition(Vec<3>& out) const { getBodyPosition(0, out); }
  void getBaseOrientation(Mat<3, 3>& out) const { getBodyOrientation(0, out); }
  void getFramePosition(size_t frameIdx, Vec<3>& out) const { Poses P = poses(); FrameW f = frameWorld(P, frameIdx); out = f.pos; }
  void getFrameOrientation(size_t frameIdx, Mat<3, 3>& out) const { Poses P = poses(); FrameW f = frameWorld(P, frameIdx); out = f.rot; }
  void getDenseJacobian(size_t bodyIdx, const Vec<3>& point_W, MatDyn& J) const { Poses P = poses(); jacobian(P, bodyIdx, point_W, &J, nullptr); }
  void getDenseRotationalJacobian(size_t bodyIdx, MatDyn& J) const { Poses P = poses(); jacobian(P, bodyIdx, Vec<3>{0, 0, 0}, nullptr, &J); }
  void getDenseFrameJacobian(size_t frameIdx, MatDyn& J) const { Poses P = poses(); FrameW f = frameWorld(P, frameIdx); jacobian(P, size_t(f.body), f.pos, &J, nullptr); }
  void getDenseFrameRotationalJacobian(size_t frameIdx, MatDyn& J) const { Poses P = poses(); FrameW f = frameWorld(P, frameIdx); jacobian(P, size_t(f.body), f.pos, nullptr, &J); }
  void getVelocity(size_t bodyIdx, const Vec<3>& point_W, Vec<3>& out) const {
    Poses P = poses(); MatDyn J; jacobian(P, bodyIdx, point_W, &J, nullptr); mulGv(J, out);
  }
  void getVelocity(size_t bodyIdx, Vec<3>& out) const { Vec<3> o; getBodyPosition(bodyIdx, o); getVelocity(bodyIdx, o, out); }
  void getAngularVelocity(size_t bodyIdx, Vec<3>& out) const { Poses P = poses(); MatDyn J; jacobian(P, bodyIdx, Vec<3>{0, 0, 0}, nullptr, &J); mulGv(J, out); }
  void getFrameVelocity(size_t frameIdx, Vec<3>& out) const { MatDyn J; getDenseFrameJacobian(frameIdx, J); mulGv(J, out); }
  void getFrameAngularVelocity(size_t frameIdx, Vec<3>& out) const { MatDyn J; getDenseFrameRotationalJacobian(frameIdx, J); mulGv(J, out); }

  // ---- model queries and whole-body quantities (host algebra on the model tables, the poses and M of the current state;
  //      upstream names, [RECALL] ArticulatedSystem.hpp) --------------------------------------------------------------
  std::vector<std::string> getBodyNames() const {
    std::vector<std::string> r;
    for (int b = 0; b < w_->nb(); b++) r.emplace_back(rsb_model_body_name(w_->model(), b));
    return r;
  }
  // movable joints in the order of the generalized coordinates the caller sees (jointOrder if one was given)
  std::vector<std::string> getMovableJointNames() const {
    const rsb_model_tables t = tables();
    const int q0 = t.floating ? 7 : 0;
    std::vector<std::string> r(size_t(t.nq - q0));
    for (int k = 0; k < t.nq - q0; k++)
      for (int b = 1; b < t.nb; b++) if (t.qidx[b] == int(qi(size_t(q0 + k)))) r[size_t(k)] = rsb_model_joint_name(w_->model(), b);
    return r;
  }
  // [lower, upper] per generalized velocity index (URDF <limit lower upper>; the base dofs and unlimited joints: -/+ 1e30 as parsed)
  std::vector<Vec<2>> getJointLimits() const {
    const rsb_model_tables t = tables();
    std::vector<Vec<2>> r(size_t(t.nv));
    for (int i = 0; i < t.nv; i++) { r[size_t(i)][0] = -1e30; r[size_t(i)][1] = 1e30; }
    for (int i = 0; i < t.nv; i++)
      for (int b = 1; b < t.nb; b++) if (t.vidx[b] == int(vi(size_t(i)))) { r[size_t(i)][0] = t.jlimit[2 * b]; r[size_t(i)][1] = t.jlimit[2 * b + 1]; }
    return r;
  }
  // actuator effort limits per generalized velocity index (URDF <limit effort>, or this environment's setActuationLimits; none: 1e30
  // or +inf); the step kernel saturates the commanded torque there
  VecDyn getActuationUpperLimits() const {
    const rsb_model_tables t = tables();
    VecDyn r(size_t(t.nv));
    for (int i = 0; i < t.nv; i++) {
      r[size_t(i)] = 1e30;
      for (int b = 1; b < t.nb; b++) if (t.vidx[b] == int(vi(size_t(i)))) r[size_t(i)] = effort_.empty() ? t.jeffort[b] : effort_[size_t(i)];
    }
    return r;
  }
  VecDyn getActuationLowerLimits() const { VecDyn r = getActuationUpperLimits(); for (size_t i = 0; i < r.size(); i++) r[i] = -r[i]; return r; }
  // the whole-body getters below read this environment's inertial parameters: the model's until updateMassInfo(), then the last ones
  // it pushed
  double getMass(size_t localIdx) const { return massOf(tables(), int(localIdx)); }
  double getTotalMass() const { const rsb_model_tables t = tables(); double m = 0; for (int b = 0; b < t.nb; b++) m += massOf(t, b); return m; }
  std::vector<Vec<3>> getBodyCOM_B() const {
    const rsb_model_tables t = tables();
    std::vector<Vec<3>> r(size_t(t.nb));
    for (int b = 0; b < t.nb; b++) for (int k = 0; k < 3; k++) r[size_t(b)][size_t(k)] = comOf(t, b, k);
    return r;
  }
  // Upstream's idiom for changing a robot's inertial parameters: edit getMass()[i], getBodyCOM_B()[i] (body frame) and getInertia()[i]
  // (about the centre of mass, body frame; symmetric), then updateMassInfo().  The vectors are this environment's editable copy,
  // filled from the model on first use.  updateMassInfo() makes them the parameters this environment integrates: a stand-alone World
  // uploads them at once; in a VectorizedEnvironment they go up before the next launch (no launch of their own).  The batch refuses a copy that is not finite, has a negative mass or an inertia that is not positive semidefinite
  // (include/rsb.h) when it arrives: at once stand-alone, at the upload in a VectorizedEnvironment.
  std::vector<double>& getMass() { initMassInfo(); return mass_; }
  std::vector<Vec<3>>& getBodyCOM_B() { initMassInfo(); return com_; }
  std::vector<Mat<3, 3>>& getInertia() { initMassInfo(); return inertia_; }
  void updateMassInfo() {
    initMassInfo();
    float* row = m_.inertiaRow(env_);
    for (size_t b = 0; b < mass_.size(); b++) {
      float* r = &row[b * 10];
      const Mat<3, 3>& I = inertia_[b];
      r[0] = float(mass_[b]);
      for (size_t k = 0; k < 3; k++) r[1 + k] = float(com_[b][k]);
      r[4] = float(I(0, 0)); r[5] = float(I(0, 1)); r[6] = float(I(0, 2)); r[7] = float(I(1, 1)); r[8] = float(I(1, 2)); r[9] = float(I(2, 2));
    }
    m_.commit();
    appliedMass_ = mass_; appliedCom_ = com_;
  }
  std::vector<Vec<3>> getBodyCOM_W() const {
    const rsb_model_tables t = tables(); const Poses P = poses();
    std::vector<Vec<3>> r(size_t(t.nb));
    for (int b = 0; b < t.nb; b++) r[size_t(b)] = comWorld(t, P, b);
    return r;
  }
  Vec<3> getCOM() const {      // centre of mass of the whole robot, world frame
    const rsb_model_tables t = tables(); const Poses P = poses();
    Vec<3> c; double m = 0;
    for (int b = 0; b < t.nb; b++) { const Vec<3> cb = comWorld(t, P, b); for (int k = 0; k < 3; k++) c[size_t(k)] += massOf(t, b) * cb[size_t(k)]; m += massOf(t, b); }
    for (int k = 0; k < 3; k++) c[size_t(k)] /= m;
    return c;
  }
  VecDyn getGeneralizedMomentum() const {      // M gv (M from the kernel's CRBA)
    const MatDyn M = getMassMatrix(); const VecDyn gv = getGeneralizedVelocity();
    VecDyn r(size_t(M.rows()));
    for (size_t i = 0; i < M.rows(); i++) { double s = 0; for (size_t j = 0; j < M.cols(); j++) s += M(i, j) * gv[j]; r[i] = s; }
    return r;
  }
  double getKineticEnergy() const {
    const MatDyn M = getMassMatrix(); const VecDyn gv = getGeneralizedVelocity();
    double e = 0;
    for (size_t i = 0; i < M.rows(); i++) for (size_t j = 0; j < M.cols(); j++) e += 0.5 * gv[i] * M(i, j) * gv[j];
    return e;
  }
  double getPotentialEnergy(const Vec<3>& gravity) const {
    const rsb_model_tables t = tables(); const Poses P = poses();
    double e = 0;
    for (int b = 0; b < t.nb; b++) { const Vec<3> c = comWorld(t, P, b); e -= massOf(t, b) * (gravity[0] * c[0] + gravity[1] * c[1] + gravity[2] * c[2]); }
    return e;
  }
  double getEnergy(const Vec<3>& gravity) const { return getKineticEnergy() + getPotentialEnergy(gravity); }
  Vec<3> getLinearMomentum() const {           // sum of m_b v_com,b through the body Jacobians
    const rsb_model_tables t = tables(); const Poses P = poses(); const VecDyn gv = getGeneralizedVelocity();
    Vec<3> p;
    for (int b = 0; b < t.nb; b++) {
      MatDyn J; jacobian(P, size_t(b), comWorld(t, P, b), &J, nullptr);
      for (int r = 0; r < 3; r++) { double s = 0; for (size_t c = 0; c < J.cols(); c++) s += J(size_t(r), c) * gv[c]; p[size_t(r)] += massOf(t, b) * s; }
    }
    return p;
  }
  void getSparseJacobian(size_t bodyIdx, const Vec<3>& point_W, SparseJacobian& J) const {
    const rsb_model_tables t = tables(); const Poses P = poses();
    MatDyn D; jacobian(P, bodyIdx, point_W, &D, nullptr);
    std::vector<size_t> cols;        // dofs of the chain root .. body, in the caller's order
    for (int i = int(bodyIdx); i >= 0; i = t.parent[i]) {
      const int nd = t.jtype[i] == 3 ? 6 : (t.jtype[i] == 1 || t.jtype[i] == 2 ? 1 : 0);
      for (int k = 0; k < nd; k++) cols.push_back(vinv(size_t(t.vidx[i] + k)));
    }
    std::sort(cols.begin(), cols.end());
    J.resize(cols.size());
    for (size_t k = 0; k < cols.size(); k++) { J.idx[k] = cols[k]; for (size_t r = 0; r < 3; r++) J.v(r, k) = D(r, cols[k]); }
  }
  // base pose setters (floating base): the other coordinates stay as they are
  void setBasePos(const Vec<3>& pos) {
    VecDyn gc = getGeneralizedCoordinate();
    if (gc.size() < 7 || !tables().floating) throw std::runtime_error("setBasePos: the robot has a fixed base");
    for (size_t k = 0; k < 3; k++) gc[k] = pos[k];
    setGeneralizedCoordinate(gc);
  }
  void setBaseOrientation(const Vec<4>& quat) {
    VecDyn gc = getGeneralizedCoordinate();
    if (gc.size() < 7 || !tables().floating) throw std::runtime_error("setBaseOrientation: the robot has a fixed base");
    const double n = std::sqrt(quat[0] * quat[0] + quat[1] * quat[1] + quat[2] * quat[2] + quat[3] * quat[3]);
    for (size_t k = 0; k < 4; k++) gc[3 + k] = quat[k] / n;
    setGeneralizedCoordinate(gc);
  }
  void setBaseOrientation(const Mat<3, 3>& rot) { Vec<4> q; rotMatToQuat(rot, q); setBaseOrientation(q); }
  // upstream's separate target / gain setters: the other half keeps its last value
  template <class VQ> void setPTarget(const VQ& posTarget) {
    lastP_.resize(size_t(w_->nq())); for (size_t i = 0; i < lastP_.size(); i++) lastP_[i] = posTarget[i];
    if (lastD_.size() != size_t(w_->nv())) lastD_.resize(size_t(w_->nv()));
    setPdTarget(lastP_, lastD_);
  }
  template <class VV> void setDTarget(const VV& velTarget) {
    lastD_.resize(size_t(w_->nv())); for (size_t i = 0; i < lastD_.size(); i++) lastD_[i] = velTarget[i];
    if (lastP_.size() != size_t(w_->nq())) lastP_ = getGeneralizedCoordinate();     // no position target given yet: hold the current pose
    setPdTarget(lastP_, lastD_);
  }
  template <class VV> void setPGains(const VV& p) {
    kpLast_.resize(size_t(w_->nv())); for (size_t i = 0; i < kpLast_.size(); i++) kpLast_[i] = p[i];
    if (kdLast_.size() != kpLast_.size()) kdLast_.resize(kpLast_.size());
    setPdGains(kpLast_, kdLast_);
  }
  template <class VV> void setDGains(const VV& d) {
    kdLast_.resize(size_t(w_->nv())); for (size_t i = 0; i < kdLast_.size(); i++) kdLast_[i] = d[i];
    if (kpLast_.size() != kdLast_.size()) kpLast_.resize(kdLast_.size());
    setPdGains(kpLast_, kdLast_);
  }
  // This environment's actuator effort limits, per generalized velocity index: the commanded torque (feed-forward + PD) saturates at
  // +-upper.  The step saturates symmetrically, so lower must be -upper with upper >= 0 (+inf: no limit); anything else fails loudly.
  // The base dofs of a floating robot are not actuated and their entries are ignored.  They go to this environment's actuator row: up
  // at once from a stand-alone World, before the next launch in a VectorizedEnvironment.
  template <class VV> void setActuationLimits(const VV& upper, const VV& lower) {
    const int nv = w_->nv();
    for (int i = 0; i < nv; i++)
      if (!(upper[i] >= 0.0) || !(lower[i] == -upper[i]))
        throw std::runtime_error("setActuationLimits: dof " + std::to_string(i) + ": only symmetric limits (lower = -upper, upper >= 0) are implemented by the batched step");
    float* r = m_.actuatorRow(env_);      // gains -1 until this environment sets its own: the batch's
    for (int i = 0; i < nv; i++) r[3 * vi(i) + 2] = float(upper[i]);
    m_.commit();
    effort_.assign(size_t(nv), 0.0);
    for (int i = 0; i < nv; i++) effort_[size_t(i)] = upper[i];
  }
  // The batch integrates semi-implicitly (DESIGN.md section 2: v+ from the implicit PD / contact solve, then q+ = q (+) dt v+);
  // asking for another scheme fails loudly instead of silently integrating differently from what the caller expects.
  void setIntegrationScheme(IntegrationScheme scheme) {
    if (scheme != IntegrationScheme::SEMI_IMPLICIT) throw std::runtime_error("setIntegrationScheme: only IntegrationScheme::SEMI_IMPLICIT is implemented by the batched step");
  }

  std::vector<Contact>& getContacts() {
    m_.needContacts(env_);
    contacts_.clear();
    for (int i = 0; i < *m_.ncontacts.row(env_); i++) contacts_.emplace_back(m_.contacts.row(env_)[i]);
    return contacts_;
  }
  // ---- Extensions upstream does not have.  Under upstream an ENVIRONMENT calls World::integrate() once per simulation step and sees
  // every step's getContacts() in between; here the integrate() calls of a control step run as one fused launch and getContacts()
  // shows the last of them only, so the launch gathers for the caller what that loop would have gathered.
  // setContactBodies: the bodies (getBodyIdx order, at most RSB_MAX_CONTACT_BODIES) to gather for.  The list belongs to the batch: every
  // environment shares it, and each environment of a VectorizedEnvironment may set the same list in its constructor.
  void setContactBodies(const std::vector<size_t>& bodies) { w_->setContactBodies(bodies); }
  // mean contact force on the body [N, world frame] over the integrate() calls since the last state access (the fused launch); over
  // the one step of a stand-alone integrate()
  void getBodyContactForce(size_t bodyIdx, Vec<3>& out) {
    const size_t s = w_->contactBodySlot(bodyIdx);
    m_.needContactForces(env_, true, false);
    for (int k = 0; k < 3; k++) out[k] = m_.cfForce.row(env_)[s * 3 + k];
  }
  // the number of those integrate() calls in which the body had a contact (> 0: it touched something during the control step)
  int getBodyContactSteps(size_t bodyIdx) {
    const size_t s = w_->contactBodySlot(bodyIdx);
    m_.needContactForces(env_, false, true);
    return m_.cfSteps.row(env_)[s];
  }
  // setImus: IMUs at the model frames frameIndices (getFrameIdxByName order, at most RSB_MAX_IMUS), the sensor's axes those of the frame.
  // The list belongs to the batch: every environment shares it, and each environment of a VectorizedEnvironment may set the same list in
  // its constructor.
  void setImus(const std::vector<size_t>& frameIndices) { w_->setImus(frameIndices); }
  // IMU i's mean specific force [m/s^2, sensor frame] over the integrate() calls since the last state access (the fused launch; the one
  // step of a stand-alone integrate()): what an accelerometer measures, +|g| upwards at rest and 0 in free fall
  void getImuLinearAcceleration(size_t i, Vec<3>& out) {
    if (i >= w_->numImus()) throw std::runtime_error("getImuLinearAcceleration: IMU " + std::to_string(i) + " was not given to setImus()");
    m_.needImuReadings(env_, true, false);
    for (int k = 0; k < 3; k++) out[k] = m_.imuLin.row(env_)[i * 3 + k];
  }
  // IMU i's mean angular rate [rad/s, sensor frame] over the same integrate() calls
  void getImuAngularVelocity(size_t i, Vec<3>& out) {
    if (i >= w_->numImus()) throw std::runtime_error("getImuAngularVelocity: IMU " + std::to_string(i) + " was not given to setImus()");
    m_.needImuReadings(env_, false, true);
    for (int k = 0; k < 3; k++) out[k] = m_.imuAng.row(env_)[i * 3 + k];
  }
  // setHeightScan: terrain height samples at horizontal offsets (x, y) from bodies (getBodyIdx order, at most RSB_MAX_SCAN_POINTS),
  // turned with each body's heading (yawAligned) or along the world axes: what an upstream observe() builds with one
  // HeightMap::getHeight call per point.  The list belongs to the batch: every environment shares it, and each environment of a
  // VectorizedEnvironment may set the same list in its constructor.
  void setHeightScan(const std::vector<size_t>& bodies, const std::vector<Vec<2>>& offsets, bool yawAligned = true) {
    if (offsets.size() != bodies.size()) throw std::runtime_error("setHeightScan: one offset per body");
    std::vector<int32_t> b(bodies.begin(), bodies.end());
    std::vector<float> xy(2 * offsets.size());
    for (size_t i = 0; i < offsets.size(); i++) { xy[2 * i] = float(offsets[i][0]); xy[2 * i + 1] = float(offsets[i][1]); }
    w_->setHeightScan(b, xy, yawAligned);
  }
  // setRays: rays from bodies (getBodyIdx order, at most RSB_MAX_RAYS), each with an origin and a direction in the body frame (any
  // length, normalised when set): a depth camera or a lidar on the robot.  getRayCasts reports the first hit within maxDistance against
  // the terrain and, with seeRobot, the robot's own collision bodies (a shape that contains a ray's origin is ignored, so a camera inside
  // the base box sees out of it).  The list belongs to the batch: every environment shares it, and each environment of a
  // VectorizedEnvironment may set the same list in its constructor.
  void setRays(const std::vector<size_t>& bodies, const std::vector<Vec<3>>& origins, const std::vector<Vec<3>>& directions, double maxDistance,
               bool seeRobot = false) {
    if (origins.size() != bodies.size() || directions.size() != bodies.size()) throw std::runtime_error("setRays: one origin and one direction per body");
    std::vector<int32_t> b(bodies.begin(), bodies.end());
    std::vector<float> o(3 * bodies.size()), d(3 * bodies.size());
    for (size_t i = 0; i < bodies.size(); i++)
      for (int k = 0; k < 3; k++) { o[3 * i + k] = float(origins[i][k]); d[3 * i + k] = float(directions[i][k]); }
    w_->setRays(b, o, d, float(maxDistance), seeRobot);
  }
  // setActuatorNetwork: the learned actuator network of rsb_batch_set_actuator_network (include/rsb.h) for the dofs listed (generalized
  // velocity indices of joints), with params in torch.nn.Linear order.  The network belongs to the batch: every environment shares it,
  // and each environment of a VectorizedEnvironment may set the same one in its constructor.  Setting it zeroes every history.
  void setActuatorNetwork(const std::vector<size_t>& dofs, int history, int layers, int width, const std::vector<float>& params) {
    w_->setActuatorNetwork(std::vector<int32_t>(dofs.begin(), dofs.end()), history, layers, width, params);
  }
  // setActuatorLstm: the LSTM actuator network of rsb_batch_set_actuator_lstm (include/rsb.h) for the dofs listed, with params in
  // torch.nn.LSTM order (weight_ih_l0, weight_hh_l0, bias_ih_l0, bias_hh_l0, ..., then the read-out weight and bias).  It replaces any
  // network set before and belongs to the batch as setActuatorNetwork's does.  Setting it zeroes every (h, c) state.
  void setActuatorLstm(const std::vector<size_t>& dofs, int layers, int hidden, const std::vector<float>& params) {
    w_->setActuatorLstm(std::vector<int32_t>(dofs.begin(), dofs.end()), layers, hidden, params);
  }
  // zero this environment's actuator-network history, or the LSTM's (h, c) state (setState keeps either): call it in reset()
  void resetActuatorHistory() { w_->resetActuatorHistory(env_); }
  // setActuationDelay: from now on every joint command (PD targets, feed-forward torque) of this robot takes effect subSteps physics
  // sub-steps after it was set (rsb_batch_set_actuation_delay, include/rsb.h); setting it empties the command history, so the first
  // command then holds for subSteps + 1 sub-steps.  Call it in reset() to draw a delay per episode.  In a VectorizedEnvironment the
  // delays of all environments go up with the next launch in one call.
  void setActuationDelay(size_t subSteps) {
    if (subSteps > RSB_MAX_ACTUATION_DELAY)
      throw std::runtime_error("setActuationDelay: " + std::to_string(subSteps) + " sub-steps, at most " + std::to_string(RSB_MAX_ACTUATION_DELAY));
    w_->setActuationDelay(env_, int(subSteps));
  }
  // the world z of the collision surface under every point at the current state, in setHeightScan order, and (samples, optional) the
  // world (x, y) each was taken at.  In a VectorizedEnvironment one call scans every environment for the control step; a stand-alone
  // World scans this environment
  void getHeightScan(VecDyn& heights, std::vector<Vec<2>>* samples = nullptr) {
    const size_t P = w_->numHeightScanPoints();
    if (P == 0) throw std::runtime_error("getHeightScan: call setHeightScan() first");
    m_.needHeightScan(env_, samples != nullptr);
    const float *h = m_.scan.row(env_), *xy = m_.scanXy.row(env_);
    heights.resize(P);
    for (size_t i = 0; i < P; i++) heights[i] = h[i];
    if (samples) {
      samples->resize(P);
      for (size_t i = 0; i < P; i++) { (*samples)[i][0] = xy[2 * i]; (*samples)[i][1] = xy[2 * i + 1]; }
    }
  }
  // the first hit along every ray at the current state, in setRays order: distances (+inf: nothing within maxDistance, NaN: a diverged
  // state) and (hits, optional) what each hit: RSB_RAY_TERRAIN, the collision-body index, or RSB_RAY_MISS.  In a VectorizedEnvironment
  // one call casts every environment's rays for the control step; a stand-alone World casts this environment's
  void getRayCasts(VecDyn& distances, std::vector<int>* hits = nullptr) {
    const size_t R = w_->numRays();
    if (R == 0) throw std::runtime_error("getRayCasts: call setRays() first");
    m_.needRayCasts(env_, hits != nullptr);
    const float* d = m_.rayDist.row(env_);
    distances.resize(R);
    for (size_t i = 0; i < R; i++) distances[i] = d[i];
    if (hits) {
      const int32_t* h = m_.rayHit.row(env_);
      hits->assign(h, h + R);
    }
  }
  int env() const { return env_; }
 private:
  void pushWrench() {
    rsbCheck(rsb_batch_set_external_wrench(w_->batch(), extBody_, extF_, extT_, extP_, env_, 1, RSB_HOST), "setExternalForce");
  }
  void applySelfPairs(const std::vector<int32_t>& idx, const std::vector<float>& mu) {
    const int n = int(idx.size() / 2);
    rsbCheck(rsb_batch_set_self_collision(w_->batch(), idx.data(), n, mu.empty() ? nullptr : mu.data()), "setSelfCollisionPairs");
    selfPairs_ = idx;
    selfMu_ = mu.empty() ? std::vector<float>(n, -1.f) : mu;
  }
  std::map<size_t, std::string> collisionMaterial_;   // collision body -> material name (absent = "default")
  bool materialsDirty_ = false;
  std::vector<int32_t> selfPairs_;                    // enabled self-collision pairs: [n][2] collision bodies
  std::vector<float> selfMu_;                         // their friction (< 0: default material)
  int extBody_ = -1; bool extHasForce_ = false;
  float extF_[3] = {0, 0, 0}, extT_[3] = {0, 0, 0}, extP_[3] = {0, 0, 0};
  struct Poses { std::vector<float> R, p; };
  struct FrameW { int body; Vec<3> pos; Mat<3, 3> rot; };
  Poses poses() const {
    Poses P; P.R.resize(size_t(w_->nb()) * 9); P.p.resize(size_t(w_->nb()) * 3);
    m_.current(env_);
    // the C-ABI getter is lazy: it runs a kinematics-only pass when the state changed (upstream's updateKinematics()); the contact
    // records and impulses of the last integrate() stay valid across kinematic getters, as upstream's getContacts() does
    rsbCheck(rsb_batch_get_body_poses(w_->batch(), env_, 1, P.R.data(), P.p.data(), RSB_HOST), "getBodyPoses");
    return P;
  }
  FrameW frameWorld(const Poses& P, size_t frameIdx) const {
    FrameW f; double pos[3], rot[9];
    rsbCheck(rsb_model_frame(w_->model(), int(frameIdx), &f.body, pos, rot), "getFrame");
    const float* R = &P.R[size_t(f.body) * 9];
    for (int r = 0; r < 3; r++) {
      f.pos[r] = P.p[size_t(f.body) * 3 + r] + R[3 * r] * pos[0] + R[3 * r + 1] * pos[1] + R[3 * r + 2] * pos[2];
      for (int c = 0; c < 3; c++) f.rot(r, c) = R[3 * r] * rot[c] + R[3 * r + 1] * rot[3 + c] + R[3 * r + 2] * rot[6 + c];
    }
    return f;
  }
  // geometric Jacobians of a world point attached to `body`: v_point = Jp gv, omega_body = Jr gv
  void jacobian(const Poses& P, size_t body, const Vec<3>& pt, MatDyn* Jp, MatDyn* Jr) const {
    rsb_model_tables t; rsbCheck(rsb_model_get_tables(w_->model(), &t), "getTables");
    if (Jp) Jp->resize(3, size_t(t.nv));
    if (Jr) Jr->resize(3, size_t(t.nv));
    for (int i = int(body); i >= 0; i = t.parent[i]) {
      const float* R = &P.R[size_t(i) * 9]; const float* o = &P.p[size_t(i) * 3];
      const double r[3] = {pt[0] - o[0], pt[1] - o[1], pt[2] - o[2]};
      if (t.jtype[i] == 3) {          // floating base: [v_world | omega_world]
        if (Jp) {
          for (int k = 0; k < 3; k++) (*Jp)(k, k) = 1.0;
          (*Jp)(0, 4) = r[2]; (*Jp)(0, 5) = -r[1]; (*Jp)(1, 3) = -r[2]; (*Jp)(1, 5) = r[0]; (*Jp)(2, 3) = r[1]; (*Jp)(2, 4) = -r[0];   // -[r]x
        }
        if (Jr) for (int k = 0; k < 3; k++) (*Jr)(k, 3 + k) = 1.0;
      } else if (t.jtype[i] == 1 || t.jtype[i] == 2) {
        const double* ab = &t.axis[size_t(i) * 3];
        double a[3];
        for (int k = 0; k < 3; k++) a[k] = R[3 * k] * ab[0] + R[3 * k + 1] * ab[1] + R[3 * k + 2] * ab[2];
        const size_t c = vinv(size_t(t.vidx[i]));      // column in the caller's dof order (jointOrder)
        if (t.jtype[i] == 1) {
          if (Jp) { (*Jp)(0, c) = a[1] * r[2] - a[2] * r[1]; (*Jp)(1, c) = a[2] * r[0] - a[0] * r[2]; (*Jp)(2, c) = a[0] * r[1] - a[1] * r[0]; }
          if (Jr) for (int k = 0; k < 3; k++) (*Jr)(k, c) = a[k];
        } else if (Jp) for (int k = 0; k < 3; k++) (*Jp)(k, c) = a[k];
      }
    }
  }
  void mulGv(const MatDyn& J, Vec<3>& out) const {
    VecDyn gv = getGeneralizedVelocity();
    for (int r = 0; r < 3; r++) { double s = 0; for (size_t c = 0; c < J.cols(); c++) s += J(r, c) * gv[c]; out[r] = s; }
  }
  size_t qi(size_t i) const { return size_t(qmap_[i]); }     // caller's coordinate index -> the batch's
  size_t vi(size_t i) const { return size_t(vmap_[i]); }
  // a row in the batch's order from the caller's values (map: qmap_ or vmap_), and back
  template <class V> static void toBatch(const V& x, const std::vector<int>& map, float* row) {
    for (size_t i = 0; i < map.size(); i++) row[map[i]] = float(x[i]);
  }
  static VecDyn fromBatch(const float* row, const std::vector<int>& map) {
    VecDyn x(map.size());
    for (size_t i = 0; i < map.size(); i++) x[i] = row[map[i]];
    return x;
  }
  size_t vinv(size_t batchIdx) const {                                            // the batch's velocity index -> the caller's
    for (size_t i = 0; i < vmap_.size(); i++) if (size_t(vmap_[i]) == batchIdx) return i;
    return batchIdx;
  }
  rsb_model_tables tables() const { rsb_model_tables t; rsbCheck(rsb_model_get_tables(w_->model(), &t), "getTables"); return t; }
  Vec<3> comWorld(const rsb_model_tables& t, const Poses& P, int b) const {
    const float* R = &P.R[size_t(b) * 9]; const float* o = &P.p[size_t(b) * 3];
    const double c[3] = {comOf(t, b, 0), comOf(t, b, 1), comOf(t, b, 2)};
    Vec<3> r;
    for (int k = 0; k < 3; k++) r[size_t(k)] = o[k] + R[3 * k] * c[0] + R[3 * k + 1] * c[1] + R[3 * k + 2] * c[2];
    return r;
  }
  // this environment's inertial parameters: the model's until updateMassInfo() pushed its own
  double massOf(const rsb_model_tables& t, int b) const { return appliedMass_.empty() ? t.mass[b] : appliedMass_[size_t(b)]; }
  double comOf(const rsb_model_tables& t, int b, int k) const { return appliedCom_.empty() ? t.com[3 * b + k] : appliedCom_[size_t(b)][size_t(k)]; }
  void initMassInfo() {
    if (!mass_.empty()) return;
    const rsb_model_tables t = tables();
    mass_.resize(size_t(t.nb)); com_.resize(size_t(t.nb)); inertia_.resize(size_t(t.nb));
    for (int b = 0; b < t.nb; b++) {
      mass_[size_t(b)] = t.mass[b];
      for (int k = 0; k < 3; k++) com_[size_t(b)][size_t(k)] = t.com[3 * b + k];
      const double* I = &t.inertia[6 * b];
      const double full[9] = {I[0], I[1], I[2], I[1], I[3], I[4], I[2], I[4], I[5]};
      for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) inertia_[size_t(b)](size_t(r), size_t(c)) = full[3 * r + c];
    }
  }
  std::vector<double> mass_, appliedMass_;            // editable copy (getMass()) and the values last pushed by updateMassInfo()
  std::vector<Vec<3>> com_, appliedCom_;
  std::vector<Mat<3, 3>> inertia_;
  VecDyn lastP_, lastD_, kpLast_, kdLast_;
  std::vector<double> effort_;                        // the last setActuationLimits() upper limits in the caller's order (empty: the URDF's)
  std::vector<int> qmap_, vmap_;
  BatchedWorld* w_;
  LockStep& m_;
  int env_;
  std::string name_;
  std::vector<Contact> contacts_;
};

// raisim::World -- standalone it owns a batch of one environment; as a view it forwards to a shared batch
// While a VectorizedEnvironment<ENVIRONMENT> constructs its environments, every `raisim::World` they create becomes a view of
// ONE shared batch instead of a batch of one: environment i's World is view i; the first addArticulatedSystem() creates the
// batch (num_envs environments of that URDF, lock-step mode), the others attach to it.
struct BatchContext {
  int numEnvs = 0, device = 0, envIndex = 0;
  std::unique_ptr<BatchedWorld> batch;
  static BatchContext*& current() { static thread_local BatchContext* c = nullptr; return c; }
};

class World {
 public:
  World() { if (BatchContext* c = BatchContext::current()) { ctx_ = c; env_ = c->envIndex; } }
  World(BatchedWorld* shared, int env) : w_(shared), env_(env) { robot_.reset(new ArticulatedSystem(w_, env_)); }
  static void setActivationKey(const std::string&) {}          // licence check of the reference: not a capability

  ArticulatedSystem* addArticulatedSystem(const std::string& urdfPathOrXml, const std::string& = "", const std::vector<std::string>& jointOrder = {},
                                          CollisionGroup = 1, CollisionGroup = CollisionGroup(-1)) {
    if (w_) throw std::runtime_error("addArticulatedSystem: this World is a view of a BatchedWorld (one robot per environment)");
    if (ctx_) {   // environment of a VectorizedEnvironment: attach to (or create) the shared batch
      if (!ctx_->batch) {
        ctx_->batch.reset(new BatchedWorld(urdfPathOrXml, ctx_->numEnvs, ctx_->device));
        ctx_->batch->rememberUrdf(urdfPathOrXml);
        ctx_->batch->enableLockStep();
      } else if (ctx_->batch->urdf() != urdfPathOrXml) throw std::runtime_error("VectorizedEnvironment: every environment must load the same robot description");
      w_ = ctx_->batch.get();
    } else {
      owned_.reset(new BatchedWorld(urdfPathOrXml, 1));
      w_ = owned_.get(); env_ = 0;
    }
    rsb_params p = w_->params();
    p.dt = float(dt_); p.gravity[0] = float(g_[0]); p.gravity[1] = float(g_[1]); p.gravity[2] = float(g_[2]);
    w_->setParams(p);
    if (haveGround_) setGround();
    robot_.reset(new ArticulatedSystem(w_, env_));
    robot_->setJointOrder(jointOrder);
    return robot_.get();
  }
  Ground* addGround(double zHeight = 0.0, const std::string& material = "default", CollisionGroup = CollisionGroup(-1)) {
    haveGround_ = true; groundZ_ = zHeight; terrainMaterial_ = material; ground_.setHeight(zHeight);
    if (robot_) applyMaterials(true);
    if (w_) setGround();
    return &ground_;
  }
  HeightMap* addHeightMap(size_t xSamples, size_t ySamples, double xSize, double ySize, double centerX, double centerY,
                          const std::vector<double>& height, const std::string& = "default", CollisionGroup = 1, CollisionGroup = CollisionGroup(-1)) {
    need();
    return useHeightMap(int(xSamples), int(ySamples), xSize, ySize, centerX, centerY, std::vector<float>(height.begin(), height.end()));
  }
  HeightMap* addHeightMap(double centerX, double centerY, const TerrainProperties& tp, const std::string& = "default", CollisionGroup = 1,
                          CollisionGroup = CollisionGroup(-1)) {
    need();
    rsb_terrain_properties p{int(tp.xSamples), int(tp.ySamples), tp.xSize, tp.ySize, tp.frequency, tp.zScale, int(tp.fractalOctaves), tp.fractalLacunarity,
                             tp.fractalGain, tp.stepSize, tp.heightOffset, tp.seed};
    std::vector<float> h(tp.xSamples * tp.ySamples);
    rsbCheck(rsb_terrain_generate(&p, h.data()), "TerrainGenerator");
    return useHeightMap(int(tp.xSamples), int(tp.ySamples), tp.xSize, tp.ySize, centerX, centerY, std::move(h));
  }
  // height-map files (upstream overloads of the same name; [RECALL] formats, see include/rsb.h)
  HeightMap* addHeightMap(const std::string& raisimHeightMapFileName, double centerX, double centerY, const std::string& = "default",
                          CollisionGroup = 1, CollisionGroup = CollisionGroup(-1)) {
    need();
    int xs = 0, ys = 0; double sx = 0, sy = 0;
    rsbCheck(rsb_heightmap_read_text(raisimHeightMapFileName.c_str(), &xs, &ys, &sx, &sy, nullptr, 0), "addHeightMap");
    std::vector<float> h(size_t(xs) * ys);
    rsbCheck(rsb_heightmap_read_text(raisimHeightMapFileName.c_str(), &xs, &ys, &sx, &sy, h.data(), int(h.size())), "addHeightMap");
    return useHeightMap(xs, ys, sx, sy, centerX, centerY, std::move(h));
  }
  HeightMap* addHeightMap(const std::string& pngFileName, double centerX, double centerY, double xSize, double ySize, double heightScale,
                          double heightOffset, const std::string& = "default", CollisionGroup = 1, CollisionGroup = CollisionGroup(-1)) {
    need();
    int xs = 0, ys = 0;
    rsbCheck(rsb_heightmap_read_png(pngFileName.c_str(), heightScale, heightOffset, &xs, &ys, nullptr, 0), "addHeightMap");
    std::vector<float> h(size_t(xs) * ys);
    rsbCheck(rsb_heightmap_read_png(pngFileName.c_str(), heightScale, heightOffset, &xs, &ys, h.data(), int(h.size())), "addHeightMap");
    return useHeightMap(xs, ys, xSize, ySize, centerX, centerY, std::move(h));
  }
  void setTimeStep(double dt) { dt_ = dt; if (w_) { rsb_params p = w_->params(); p.dt = float(dt); w_->setParams(p); } }
  double getTimeStep() const { return dt_; }
  void setGravity(const Vec<3>& g) { g_ = g; if (w_) { rsb_params p = w_->params(); for (int k = 0; k < 3; k++) p.gravity[k] = float(g[k]); w_->setParams(p); } }
  void setERP(double erp, double = 0) { need(); rsb_params p = w_->params(); p.erp = float(erp); w_->setParams(p); }
  void setContactSolverParam(double alpha_init, double alpha_min, double alpha_decay, int maxIter, double threshold) {
    need(); rsb_params p = w_->params();
    p.alpha_init = float(alpha_init); p.alpha_min = float(alpha_min); p.alpha_decay = float(alpha_decay); p.max_iter = maxIter; p.threshold = float(threshold);
    w_->setParams(p);
  }
  // In a VectorizedEnvironment the friction is this environment's own: every collision body without a material pair of its own takes it
  // (through the environment's friction row); restitution, and the default friction of self-collision pairs, stay batch-wide
  void setDefaultMaterial(double friction, double restitution, double resThreshold) {
    need(); defaultFriction_ = friction;
    w_->setDefaultMaterial(env_, friction, restitution, resThreshold, materialFriction());
  }
  // named material pairs: friction of (collision-body material, terrain material); restitution is global (setDefaultMaterial)
  void setMaterialPairProp(const std::string& m1, const std::string& m2, double friction, double /*restitution*/ = 0, double /*resThreshold*/ = 0) {
    pairFriction_[m1 < m2 ? std::make_pair(m1, m2) : std::make_pair(m2, m1)] = friction;
    if (robot_) applyMaterials(true);
  }
  struct ContactSolverView {            // World::getContactSolver().getLoopCounter()
    const World* w;
    int getLoopCounter() const { return w->w_->solverIterations(w->env_); }
  };
  ContactSolverView getContactSolver() const { need(); return ContactSolverView{this}; }
  ArticulatedSystem* getObject(const std::string& name) { return (robot_ && robot_->getName() == name) ? robot_.get() : nullptr; }
  // object-object collisions are not part of this path (one robot against the terrain): nothing to ignore.  Self-collision pairs of the
  // robot are removed with ArticulatedSystem::ignoreCollisionBetween(bodyIdx1, bodyIdx2).
  void ignoreCollisionBetween(size_t, size_t, size_t, size_t) {}
  // one World::integrate() of THIS environment's batch.  Views of a shared batch must not call this
  // per environment -- the vectorized wrapper steps the whole batch once (see VectorizedEnvironment.hpp).
  void integrate() {
    need(); applyMaterials(false);
    if (w_->integrateEnv(env_)) robot_->clearExternalWrench();
  }
  void integrate1() { need(); applyMaterials(false); w_->integrate1(); }
  void integrate2() { need(); w_->integrate2(); if (robot_) robot_->clearExternalWrench(); }
  double getWorldTime() const { return w_ ? w_->worldTime() : 0.0; }
  ArticulatedSystem* getRobot() { return robot_.get(); }
  BatchedWorld* batched() { return w_; }
 private:
  void need() const { if (!w_) throw std::runtime_error("World: call addArticulatedSystem() first (the batch is created with the robot)"); }
  // the terrain of this environment (BatchedWorld::setHeightMap).  hm_ holds the float32 heights the batch collides with, so
  // HeightMap::getHeight answers for them
  HeightMap* useHeightMap(int xs, int ys, double xSize, double ySize, double cx, double cy, std::vector<float> h) {
    w_->setHeightMap(env_, xs, ys, xSize, ySize, cx, cy, h);
    hm_.set(size_t(xs), size_t(ys), xSize, ySize, cx, cy, std::vector<double>(h.begin(), h.end()));
    return &hm_;
  }
  void setGround() { w_->setGround(env_, groundZ_); }
  // the robot's collision bodies with a material -> the friction of their pair with the terrain's material (none: no such pair)
  std::map<size_t, std::optional<double>> materialFriction() const {
    std::map<size_t, std::optional<double>> mu;
    for (const auto& kv : robot_->collisionMaterials()) {
      const std::string& a = kv.second; const std::string& b = terrainMaterial_;
      auto it = pairFriction_.find(a < b ? std::make_pair(a, b) : std::make_pair(b, a));
      mu[kv.first] = it == pairFriction_.end() ? std::nullopt : std::optional<double>(it->second);
    }
    return mu;
  }
  void applyMaterials(bool force) {
    if (!robot_ || (!force && !robot_->materialsDirty())) return;
    w_->setMaterialFriction(env_, materialFriction(), defaultFriction_);
    robot_->materialsApplied();
  }
  std::map<std::pair<std::string, std::string>, double> pairFriction_;
  std::string terrainMaterial_ = "default";
  double defaultFriction_ = -1;        // VectorizedEnvironment: this environment's setDefaultMaterial friction (< 0: not set, the batch's)
  std::unique_ptr<BatchedWorld> owned_;
  BatchedWorld* w_ = nullptr;
  BatchContext* ctx_ = nullptr;
  int env_ = 0;
  std::unique_ptr<ArticulatedSystem> robot_;
  Ground ground_; HeightMap hm_;
  bool haveGround_ = false;
  double groundZ_ = 0, dt_ = 0.005;
  Vec<3> g_{0, 0, -9.81};
};

}  // namespace raisim
