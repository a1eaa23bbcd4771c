// ORACLE -- test infrastructure, NOT product code.
// Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
// compile, link or call anything under oracle/.  The product path (raisimlib_b200/csrc) never does.
//
// PARITY UNPINNED: the reference snapshot (/root/reference) contains no source, binary, test or
// golden vector for this path (.SUBMODULES.json:2 "bytes": 0; upstream's engine is the closed
// libraisim.so).  This file restates the PUBLISHED algorithms the reference is documented to use
// (SURVEY.md section 8c):
//   * Featherstone, "Rigid Body Dynamics Algorithms" (2008): RNEA (Table 5.1), CRBA (Table 6.2),
//     floating-base conventions (ch. 9)
//   * Hwangbo, Lee, Hutter, "Per-Contact Iteration Method for Solving Contact Dynamics",
//     IEEE RA-L 3(2) 2018, sections III-IV: per-contact Gauss-Seidel; opening / stick / slip with a
//     1-D search along the (friction-cone surface) x (zero normal velocity plane) curve
// and is validated by analytic known-answer tests (tests/test_oracle_*.py).
// What it stands in for: raisim::World::integrate() = integrate1() + integrate2()  (SURVEY 3.2, a1-a10).
//
// Conventions (SURVEY section 7, all [RECALL]):
//   gc = [x y z | qw qx qy qz | joints],  gv = [v_base(world) | w_base(world) | joint rates]
//   gravity (0,0,-9.81); semi-implicit Euler (v first, then q with v+); PD implicit in M
//   contact normal points from terrain into the robot; contacts ordered by candidate-point index
#pragma once
#include <cmath>
#include <cstring>
#include <vector>
#include <algorithm>

namespace orc {

constexpr int JT_FIXED = 0, JT_REVOLUTE = 1, JT_PRISMATIC = 2, JT_FLOATING = 3;
constexpr int KMAX = 8;            // contacts kept per environment (deepest KMAX of the candidates) == RSB_KMAX
constexpr int LMAX = 4;            // joint-limit constraints kept per environment (first LMAX violated joints) == RSB_LMAX
constexpr int RMAX = 3 * KMAX + LMAX;   // constraint rows
constexpr int NSEC = 32;           // sections per refinement round of the slip search
constexpr int NROUNDS = 2;         // 32-section rounds: bracket 2*pi/32^(r+1) = 6e-3 rad after both (or after the local fan alone)
constexpr int ACCEL_MAX_RESETS = 2; // Anderson acceleration is switched off for the rest of a solve after this many history drops
constexpr int NREF = 2;            // then NREF regula-falsi steps (Illinois variant): direction exact to float32 rounding (< 1e-6 rad)

template <typename T> struct V3 { T x, y, z; };
template <typename T> inline V3<T> operator+(V3<T> a, V3<T> b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
template <typename T> inline V3<T> operator-(V3<T> a, V3<T> b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
template <typename T> inline V3<T> operator*(T s, V3<T> a) { return {s * a.x, s * a.y, s * a.z}; }
template <typename T> inline T dot(V3<T> a, V3<T> b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
template <typename T> inline V3<T> cross(V3<T> a, V3<T> b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }

template <typename T> struct M3 {
  T m[9];  // row-major
  V3<T> operator*(V3<T> v) const { return {m[0] * v.x + m[1] * v.y + m[2] * v.z, m[3] * v.x + m[4] * v.y + m[5] * v.z, m[6] * v.x + m[7] * v.y + m[8] * v.z}; }
  M3 operator*(const M3& o) const {
    M3 r;
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) r.m[3 * i + j] = m[3 * i] * o.m[j] + m[3 * i + 1] * o.m[3 + j] + m[3 * i + 2] * o.m[6 + j];
    return r;
  }
  V3<T> tmul(V3<T> v) const { return {m[0] * v.x + m[3] * v.y + m[6] * v.z, m[1] * v.x + m[4] * v.y + m[7] * v.z, m[2] * v.x + m[5] * v.y + m[8] * v.z}; }
};

// Rodrigues rotation about unit axis a by angle q
template <typename T> inline M3<T> axis_angle(V3<T> a, T q) {
  T c = std::cos(q), s = std::sin(q), t = T(1) - c;
  return {{t * a.x * a.x + c, t * a.x * a.y - s * a.z, t * a.x * a.z + s * a.y,
           t * a.x * a.y + s * a.z, t * a.y * a.y + c, t * a.y * a.z - s * a.x,
           t * a.x * a.z - s * a.y, t * a.y * a.z + s * a.x, t * a.z * a.z + c}};
}

template <typename T> inline M3<T> quat_to_rot(T w, T x, T y, T z) {
  return {{T(1) - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
           2 * (x * y + w * z), T(1) - 2 * (x * x + z * z), 2 * (y * z - w * x),
           2 * (x * z - w * y), 2 * (y * z + w * x), T(1) - 2 * (x * x + y * y)}};
}

struct ModelDesc {   // plain-C description handed over the oracle's C API (all arrays double / int)
  int nb, nq, nv, floating;
  const int *parent, *jtype, *qidx, *vidx;
  const double *jpos, *jrot, *axis, *mass, *com, *inertia;
  const double* jlimit;   // [nb][2] lower/upper (|.| >= 1e29 = none); may be null
  const double* jeffort;  // [nb] actuator effort limit of the joint (>= 1e29 = none); may be null
  int npts;
  const int *pt_body;
  const double *pt_pos, *pt_rad;
  // typed candidates (model.hpp FeatType): 0 point / sphere, 1 segment pt_pos .. pt_pos2 swept by pt_rad, 2 box of collision body pt_coll
  const int *pt_type, *pt_coll;      // may be null: every candidate is a point
  const double* pt_pos2;
  int ncoll;
  const double *coll_size, *coll_pos, *coll_rot;   // [ncoll][3], [ncoll][3], [ncoll][9]: half extents and body-frame pose of the collision bodies
};

struct Params {
  double dt = 0.0025;
  double gravity[3] = {0, 0, -9.81};
  double erp = 0.0;             // World::setERP
  double alpha_init = 1.0, alpha_min = 1.0, alpha_decay = 1.0;   // World::setContactSolverParam
  int max_iter = 150;
  double threshold = 1e-7;
  double mu = 0.8;              // World::setDefaultMaterial friction
  double restitution = 0.0, rest_threshold = 0.01;
  int joint_limits = 1;         // enforce the URDF <limit lower upper> of revolute/prismatic joints (unilateral rows in the solver)
  int stall_window = 8;         // stagnation check of the Gauss-Seidel loop (0 = off), see include/rsb.h
  double stall_ratio = 0.5;
  double stall_reg = 0.02;      // first stall: go on with G + stall_reg * mean(diag G) * I (a compliant contact set); second stall: exit.  0 = exit at once
  int slip_bisect = 0;          // 1: after the first 32-probe round, refine the bracket by plain bisection (what a CPU
                                // implementation of the published method does); 0: 32-section rounds, probe-for-probe the
                                // kernel's search.  Both end in the same bracket width; results agree to ~1e-7.
  int accel_m = 2;              // Anderson acceleration of the Gauss-Seidel sweep map (DESIGN.md section 5; rsb_params.accel_m): history of
  int accel_start = 6;          // accel_m (<= 3; the kernel implements 0 and 2) differences, first extrapolation after sweep accel_start
  int slip_local = 1;           // from the 2nd Gauss-Seidel iteration on, a contact that slipped searches a 2*pi/32 fan centred on
                                // its previous slip direction first (31 sections) and falls back to the full circle if no
                                // sign change is inside; saves one 32-probe round per slip update
  int warm_start = 0;           // EXPERIMENT, oracle only (the kernel starts from zero like the published method): start
                                // Gauss-Seidel from the previous step's impulses matched by candidate point.  Measured on the
                                // Atlas-like model standing on box feet: 29 -> 17 iterations, not enough to justify it yet.
};

struct Terrain {
  int type = 0;                 // 0 none, 1 ground plane (World::addGround), 2 height map (World::addHeightMap)
  double ground_z = 0.0;
  int xs = 0, ys = 0;
  double x_size = 0, y_size = 0, cx = 0, cy = 0;
  std::vector<double> h;        // h[iy * xs + ix]; `count` maps back to back for a terrain atlas
  int count = 1;                // terrain atlas: number of same-sized height maps
  std::vector<int> env_map;     // terrain atlas: map index of every environment (empty = everyone on map 0)
};

template <typename T> struct SlipDir { bool valid = false; T cs = 1, sn = 0; };   // last slip direction of a contact (per step)

template <typename T> struct Contact {
  int pt;          // candidate-point index (defines the order)
  int body;        // local body index on the robot  (raisim::Contact::getlocalBodyIndex)
  int pair;        // terrain feature: 0 for the plane, 2*cell+tri for the height map
  V3<T> pos;       // world position of the contact point on the robot surface
  V3<T> n, t1, t2; // contact frame, n = normal into the robot
  T depth;
  V3<T> lam;       // impulse in the contact frame (t1, t2, n)
  SlipDir<T> sdir; // last slip direction inside this step's Gauss-Seidel loop
};

template <typename T> struct Limit { int dof; T sign, viol, lam; };   // joint-limit row: sign * qdot >= 0

template <typename T> struct Workspace {
  int nb, nv;
  // external wrench of this step (ArticulatedSystem::setExternalForce / setExternalTorque): body < 0 = none
  int ext_body = -1; V3<T> ext_f{0, 0, 0}, ext_t{0, 0, 0}, ext_pos{0, 0, 0};
  int hm_offset = 0;              // terrain atlas: offset of this environment's height map inside Sim::hmap
  long long counts[4] = {0, 0, 0, 0};   // per-contact rule outcomes: opening, stick, slip, slip found by the local fan (statistics only)
  std::vector<M3<T>> R;
  std::vector<V3<T>> p, a, w, v, wd, vd, F, N;
  std::vector<T> Ic;             // 10 per body: m, h(3), I_O(6: xx xy xz yy yz zz)
  std::vector<T> S;              // 6 per body: [ang(3); lin_at_O(3)]
  std::vector<T> M, Mh, L, h, b, z, Jt, Y, G, u, u0, rhs, tau_applied, b_sat;
  std::vector<char> sat;          // dof driven at its effort limit in this step
  std::vector<Contact<T>> contacts, all;
  std::vector<Limit<T>> limits;
  int iters = 0;
  T resid = 0;                    // largest impulse update of the last Gauss-Seidel sweep (< threshold: converged)
  int status = 0;                 // 0 converged, 1 converged on the compliant contact set (stall_reg), 2 stalled, 3 max_iter == RSB_SOLVER_*
  // warm-start cache: candidate-point id and WORLD-frame impulse of the previous step's contacts
  int prev_pt[KMAX]; V3<T> prev_imp[KMAX];
  Workspace() { for (int k = 0; k < KMAX; k++) { prev_pt[k] = -1; prev_imp[k] = {0, 0, 0}; } }
};

template <typename T> class Sim {
 public:
  int nb, nq, nv, floating, npts;
  std::vector<int> parent, jtype, qidx, vidx, pt_body, pt_type, pt_coll;
  std::vector<V3<T>> jpos, axis, com, pt_pos, pt_pos2, coll_size, coll_pos;
  std::vector<M3<T>> coll_rot;
  std::vector<M3<T>> jrot;
  std::vector<T> mass, inertia, pt_rad, jlo, jhi, jeff, pt_mu;   // pt_mu < 0: default material friction; jeff: effort limit per body
  Params prm;
  Terrain ter;
  std::vector<T> hmap;
  T sec_c[NROUNDS][NSEC + 1], sec_s[NROUNDS][NSEC + 1];

  explicit Sim(const ModelDesc& d) {
    nb = d.nb; nq = d.nq; nv = d.nv; floating = d.floating; npts = d.npts;
    parent.assign(d.parent, d.parent + nb); jtype.assign(d.jtype, d.jtype + nb);
    qidx.assign(d.qidx, d.qidx + nb); vidx.assign(d.vidx, d.vidx + nb);
    jpos.resize(nb); axis.resize(nb); com.resize(nb); jrot.resize(nb); mass.resize(nb); inertia.resize(6 * nb);
    for (int i = 0; i < nb; i++) {
      jpos[i] = {T(d.jpos[3 * i]), T(d.jpos[3 * i + 1]), T(d.jpos[3 * i + 2])};
      axis[i] = {T(d.axis[3 * i]), T(d.axis[3 * i + 1]), T(d.axis[3 * i + 2])};
      com[i] = {T(d.com[3 * i]), T(d.com[3 * i + 1]), T(d.com[3 * i + 2])};
      for (int k = 0; k < 9; k++) jrot[i].m[k] = T(d.jrot[9 * i + k]);
      mass[i] = T(d.mass[i]);
      for (int k = 0; k < 6; k++) inertia[6 * i + k] = T(d.inertia[6 * i + k]);
    }
    jlo.assign(nb, T(-1e30)); jhi.assign(nb, T(1e30));
    if (d.jlimit) for (int i = 0; i < nb; i++) { jlo[i] = T(d.jlimit[2 * i]); jhi[i] = T(d.jlimit[2 * i + 1]); }
    jeff.assign(nb, T(1e30));
    if (d.jeffort) for (int i = 0; i < nb; i++) jeff[i] = T(std::min(d.jeffort[i], 1e30));
    pt_body.assign(d.pt_body, d.pt_body + npts); pt_pos.resize(npts); pt_rad.resize(npts); pt_mu.assign(npts, T(-1));
    for (int i = 0; i < npts; i++) {
      pt_pos[i] = {T(d.pt_pos[3 * i]), T(d.pt_pos[3 * i + 1]), T(d.pt_pos[3 * i + 2])};
      pt_rad[i] = T(d.pt_rad[i]);
    }
    pt_type.assign(npts, 0); pt_coll.assign(npts, 0); pt_pos2 = pt_pos;
    if (d.pt_type) {
      pt_type.assign(d.pt_type, d.pt_type + npts); pt_coll.assign(d.pt_coll, d.pt_coll + npts);
      for (int i = 0; i < npts; i++) pt_pos2[i] = {T(d.pt_pos2[3 * i]), T(d.pt_pos2[3 * i + 1]), T(d.pt_pos2[3 * i + 2])};
      coll_size.resize(d.ncoll); coll_pos.resize(d.ncoll); coll_rot.resize(d.ncoll);
      for (int c = 0; c < d.ncoll; c++) {
        coll_size[c] = {T(d.coll_size[3 * c]), T(d.coll_size[3 * c + 1]), T(d.coll_size[3 * c + 2])};
        coll_pos[c] = {T(d.coll_pos[3 * c]), T(d.coll_pos[3 * c + 1]), T(d.coll_pos[3 * c + 2])};
        for (int k = 0; k < 9; k++) coll_rot[c].m[k] = T(d.coll_rot[9 * c + k]);
      }
    }
    // direction tables of the slip search: round r covers a bracket of width 2*pi/32^r in 32 sections
    for (int r = 0; r < NROUNDS; r++) {
      double width = 2.0 * M_PI / std::pow(double(NSEC), r);
      for (int k = 0; k <= NSEC; k++) {
        sec_c[r][k] = T(std::cos(width * k / NSEC));
        sec_s[r][k] = T(std::sin(width * k / NSEC));
      }
    }
  }
  virtual ~Sim() = default;

  void set_terrain(const Terrain& t) {
    ter = t;
    hmap.resize(t.h.size());
    for (size_t i = 0; i < t.h.size(); i++) hmap[i] = T(t.h[i]);
  }

  void init_ws(Workspace<T>& ws) const {
    ws.nb = nb; ws.nv = nv;
    ws.R.resize(nb); ws.p.resize(nb); ws.a.resize(nb); ws.w.resize(nb); ws.v.resize(nb); ws.wd.resize(nb); ws.vd.resize(nb);
    ws.F.resize(nb); ws.N.resize(nb); ws.Ic.resize(10 * nb); ws.S.resize(6 * nb);
    ws.M.resize(nv * nv); ws.Mh.resize(nv * nv); ws.L.resize(nv * nv); ws.h.resize(nv); ws.tau_applied.resize(nv); ws.b.resize(nv); ws.z.resize(nv); ws.rhs.resize(nv); ws.b_sat.assign(nv, T(0)); ws.sat.assign(nv, 0);
    ws.Jt.resize(nv * RMAX); ws.Y.resize(nv * RMAX); ws.G.resize(RMAX * RMAX); ws.u.resize(RMAX); ws.u0.resize(RMAX);
  }

  // ---- a2: forward kinematics (ArticulatedSystem::updateKinematics) -----------------------------
  void fk(const T* gc, Workspace<T>& ws) const {
    for (int i = 0; i < nb; i++) {
      if (parent[i] < 0) {
        if (floating) {
          T qw = gc[3], qx = gc[4], qy = gc[5], qz = gc[6];
          T inv = T(1) / std::sqrt(qw * qw + qx * qx + qy * qy + qz * qz);
          ws.R[i] = quat_to_rot(qw * inv, qx * inv, qy * inv, qz * inv);
          ws.p[i] = {gc[0], gc[1], gc[2]};
        } else {
          ws.R[i] = jrot[i]; ws.p[i] = jpos[i];
        }
        ws.a[i] = {0, 0, 0};
        continue;
      }
      int pr = parent[i];
      M3<T> Rj = ws.R[pr] * jrot[i];
      ws.a[i] = Rj * axis[i];
      ws.p[i] = ws.p[pr] + ws.R[pr] * jpos[i];
      T q = gc[qidx[i]];
      if (jtype[i] == JT_REVOLUTE) ws.R[i] = Rj * axis_angle(axis[i], q);
      else { ws.R[i] = Rj; ws.p[i] = ws.p[i] + q * ws.a[i]; }
    }
  }

  // ---- a4: RNEA with zero joint acceleration, gravity included (getNonlinearities) ---------------
  // classical (non-spatial) Newton-Euler in world coordinates, Featherstone Table 5.1 restated
  void rnea_bias(const T* gv, Workspace<T>& ws) const {
    V3<T> g = {T(prm.gravity[0]), T(prm.gravity[1]), T(prm.gravity[2])};
    for (int i = 0; i < nb; i++) {
      int pr = parent[i];
      if (pr < 0) {
        if (floating) { ws.v[i] = {gv[0], gv[1], gv[2]}; ws.w[i] = {gv[3], gv[4], gv[5]}; }
        else { ws.v[i] = {0, 0, 0}; ws.w[i] = {0, 0, 0}; }
        ws.wd[i] = {0, 0, 0};
        ws.vd[i] = T(-1) * g;            // fictitious upward acceleration carries gravity to every body
        continue;
      }
      V3<T> r = ws.p[i] - ws.p[pr];
      T qd = gv[vidx[i]];
      V3<T> wp = ws.w[pr];
      if (jtype[i] == JT_REVOLUTE) {
        ws.w[i] = wp + qd * ws.a[i];
        ws.v[i] = ws.v[pr] + cross(wp, r);
        ws.wd[i] = ws.wd[pr] + cross(wp, qd * ws.a[i]);
        ws.vd[i] = ws.vd[pr] + cross(ws.wd[pr], r) + cross(wp, cross(wp, r));
      } else {
        ws.w[i] = wp;
        ws.v[i] = ws.v[pr] + cross(wp, r) + qd * ws.a[i];
        ws.wd[i] = ws.wd[pr];
        ws.vd[i] = ws.vd[pr] + cross(ws.wd[pr], r) + cross(wp, cross(wp, r)) + T(2) * cross(wp, qd * ws.a[i]);
      }
    }
    for (int i = 0; i < nb; i++) {
      V3<T> c = ws.R[i] * com[i];                      // COM offset from the body origin, world axes
      V3<T> ac = ws.vd[i] + cross(ws.wd[i], c) + cross(ws.w[i], cross(ws.w[i], c));
      V3<T> f = mass[i] * ac;
      // world inertia about the COM:  R I R^T
      V3<T> Iw = world_inertia_mul(i, ws, ws.w[i]);
      V3<T> Iwd = world_inertia_mul(i, ws, ws.wd[i]);
      V3<T> n = Iwd + cross(ws.w[i], Iw);
      ws.F[i] = f;
      ws.N[i] = n + cross(c, f);                       // moment about the body origin
    }
    for (int i = nb - 1; i >= 0; i--) {
      int pr = parent[i];
      if (pr >= 0) {
        if (jtype[i] == JT_REVOLUTE) ws.h[vidx[i]] = dot(ws.a[i], ws.N[i]);
        else ws.h[vidx[i]] = dot(ws.a[i], ws.F[i]);
        ws.F[pr] = ws.F[pr] + ws.F[i];
        ws.N[pr] = ws.N[pr] + ws.N[i] + cross(ws.p[i] - ws.p[pr], ws.F[i]);
      } else if (floating) {
        ws.h[0] = ws.F[i].x; ws.h[1] = ws.F[i].y; ws.h[2] = ws.F[i].z;
        ws.h[3] = ws.N[i].x; ws.h[4] = ws.N[i].y; ws.h[5] = ws.N[i].z;
      }
    }
  }

  V3<T> world_inertia_mul(int i, const Workspace<T>& ws, V3<T> x) const {
    V3<T> xl = ws.R[i].tmul(x);
    const T* I = &inertia[6 * i];
    V3<T> yl = {I[0] * xl.x + I[1] * xl.y + I[2] * xl.z, I[1] * xl.x + I[3] * xl.y + I[4] * xl.z, I[2] * xl.x + I[4] * xl.y + I[5] * xl.z};
    return ws.R[i] * yl;
  }

  // ---- a3: CRBA (getMassMatrix), Featherstone Table 6.2 in a world-aligned frame at O = p[0] ----
  // spatial inertia about O stored as (m, h = m c, I_O); spatial motion = [ang; lin at O]
  void crba(Workspace<T>& ws) const {
    V3<T> O = ws.p[0];
    for (int i = 0; i < nb; i++) {
      V3<T> c = (ws.p[i] - O) + ws.R[i] * com[i];
      T m = mass[i];
      T* X = &ws.Ic[10 * i];
      // R I R^T
      const T* I = &inertia[6 * i];
      const T* R = ws.R[i].m;
      T Il[9] = {I[0], I[1], I[2], I[1], I[3], I[4], I[2], I[4], I[5]};
      T RI[9];
      for (int r = 0; r < 3; r++) for (int k = 0; k < 3; k++) RI[3 * r + k] = R[3 * r] * Il[k] + R[3 * r + 1] * Il[3 + k] + R[3 * r + 2] * Il[6 + k];
      T Iw[9];
      for (int r = 0; r < 3; r++) for (int k = 0; k < 3; k++) Iw[3 * r + k] = RI[3 * r] * R[3 * k] + RI[3 * r + 1] * R[3 * k + 1] + RI[3 * r + 2] * R[3 * k + 2];
      T cc = dot(c, c);
      X[0] = m; X[1] = m * c.x; X[2] = m * c.y; X[3] = m * c.z;
      X[4] = Iw[0] + m * (cc - c.x * c.x); X[5] = Iw[1] - m * c.x * c.y; X[6] = Iw[2] - m * c.x * c.z;
      X[7] = Iw[4] + m * (cc - c.y * c.y); X[8] = Iw[5] - m * c.y * c.z; X[9] = Iw[8] + m * (cc - c.z * c.z);
      T* S = &ws.S[6 * i];
      if (parent[i] >= 0) {
        V3<T> r = ws.p[i] - O;
        if (jtype[i] == JT_REVOLUTE) { V3<T> l = cross(r, ws.a[i]); S[0] = ws.a[i].x; S[1] = ws.a[i].y; S[2] = ws.a[i].z; S[3] = l.x; S[4] = l.y; S[5] = l.z; }
        else { S[0] = S[1] = S[2] = 0; S[3] = ws.a[i].x; S[4] = ws.a[i].y; S[5] = ws.a[i].z; }
      }
    }
    for (int i = nb - 1; i > 0; i--) for (int k = 0; k < 10; k++) ws.Ic[10 * parent[i] + k] += ws.Ic[10 * i + k];
    std::fill(ws.M.begin(), ws.M.end(), T(0));
    for (int i = nb - 1; i > 0; i--) {
      // spatial force F = Ic_i * S_i  -> (n_O, f)
      const T* X = &ws.Ic[10 * i]; const T* S = &ws.S[6 * i];
      V3<T> wv = {S[0], S[1], S[2]}, vO = {S[3], S[4], S[5]}, hh = {X[1], X[2], X[3]};
      V3<T> f = X[0] * vO + cross(wv, hh);
      V3<T> Iw = {X[4] * wv.x + X[5] * wv.y + X[6] * wv.z, X[5] * wv.x + X[7] * wv.y + X[8] * wv.z, X[6] * wv.x + X[8] * wv.y + X[9] * wv.z};
      V3<T> n = Iw + cross(hh, vO);
      int vi = vidx[i];
      ws.M[vi * nv + vi] = S[0] * n.x + S[1] * n.y + S[2] * n.z + S[3] * f.x + S[4] * f.y + S[5] * f.z;
      for (int j = parent[i]; j > 0; j = parent[j]) {
        const T* Sj = &ws.S[6 * j];
        T val = Sj[0] * n.x + Sj[1] * n.y + Sj[2] * n.z + Sj[3] * f.x + Sj[4] * f.y + Sj[5] * f.z;
        ws.M[vi * nv + vidx[j]] = val; ws.M[vidx[j] * nv + vi] = val;
      }
      if (floating) {   // base columns: generalized velocity order is [lin; ang] at O
        T col[6] = {f.x, f.y, f.z, n.x, n.y, n.z};
        for (int k = 0; k < 6; k++) { ws.M[vi * nv + k] = col[k]; ws.M[k * nv + vi] = col[k]; }
      }
    }
    if (floating) {
      const T* X = &ws.Ic[0];
      T m = X[0]; V3<T> hh = {X[1], X[2], X[3]};
      // [ m 1 , -[h]x ; [h]x , I_O ]  in (lin, ang) order
      T hx[9] = {0, -hh.z, hh.y, hh.z, 0, -hh.x, -hh.y, hh.x, 0};
      T IO[9] = {X[4], X[5], X[6], X[5], X[7], X[8], X[6], X[8], X[9]};
      for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) {
        ws.M[r * nv + c] = (r == c) ? m : T(0);
        ws.M[r * nv + 3 + c] = -hx[3 * r + c];
        ws.M[(3 + r) * nv + c] = hx[3 * r + c];
        ws.M[(3 + r) * nv + 3 + c] = IO[3 * r + c];
      }
    }
  }

  // ---- a6: narrow phase (Ground / HeightMap vs collision bodies expanded to candidate points) ----
  bool terrain_query(V3<T> P, T& dist, V3<T>& n, int& pair, int hm_offset = 0) const {
    if (ter.type == 1) { dist = P.z - T(ter.ground_z); n = {0, 0, 1}; pair = 0; return true; }
    if (ter.type != 2) return false;
    T dx = T(ter.x_size) / T(ter.xs - 1), dy = T(ter.y_size) / T(ter.ys - 1);
    T x0 = T(ter.cx) - T(0.5) * T(ter.x_size), y0 = T(ter.cy) - T(0.5) * T(ter.y_size);
    T gx = (P.x - x0) / dx, gy = (P.y - y0) / dy;
    if (!(gx >= T(0)) || !(gy >= T(0)) || !(gx < T(ter.xs - 1)) || !(gy < T(ter.ys - 1))) return false;
    int ix = int(gx), iy = int(gy);
    T fx = gx - T(ix), fy = gy - T(iy);
    const T* H = hmap.data() + hm_offset;
    T h00 = H[iy * ter.xs + ix], h10 = H[iy * ter.xs + ix + 1], h01 = H[(iy + 1) * ter.xs + ix], h11 = H[(iy + 1) * ter.xs + ix + 1];
    T sx, sy; int tri;
    if (fx >= fy) { sx = (h10 - h00); sy = (h11 - h10); tri = 0; }
    else { sx = (h11 - h01); sy = (h01 - h00); tri = 1; }
    T zt = h00 + sx * fx + sy * fy;
    T nx = -sx / dx, ny = -sy / dy;
    T inv = T(1) / std::sqrt(nx * nx + ny * ny + T(1));
    n = {nx * inv, ny * inv, inv};
    dist = (P.z - zt) * inv;
    pair = 2 * (iy * (ter.xs - 1) + ix) + tri;
    return true;
  }

  // ---- height-map geometry (SURVEY 8a row a6: shape against every triangle under the shape's AABB) -------------------
  // Cell (ix, iy) holds two triangles split along the diagonal P00-P11: tri 0 = (P00, P10, P11), tri 1 = (P00, P11, P01).
  struct HmGrid { T x0, y0, dx, dy; int xs, ys; const T* H; };
  HmGrid grid(int hm_offset) const {
    return {T(ter.cx) - T(0.5) * T(ter.x_size), T(ter.cy) - T(0.5) * T(ter.y_size), T(ter.x_size) / T(ter.xs - 1), T(ter.y_size) / T(ter.ys - 1), ter.xs, ter.ys,
            hmap.data() + hm_offset};
  }
  static V3<T> vertex(const HmGrid& g, int ix, int iy) { return {g.x0 + T(ix) * g.dx, g.y0 + T(iy) * g.dy, g.H[iy * g.xs + ix]}; }
  // closest point of triangle (a, b, c) to p (Ericson, Real-Time Collision Detection 5.1.5: Voronoi regions of the triangle)
  static V3<T> closest_on_triangle(V3<T> p, V3<T> a, V3<T> b, V3<T> c) {
    const V3<T> ab = b - a, ac = c - a, ap = p - a;
    const T d1 = dot(ab, ap), d2 = dot(ac, ap);
    if (d1 <= T(0) && d2 <= T(0)) return a;
    const V3<T> bp = p - b;
    const T d3 = dot(ab, bp), d4 = dot(ac, bp);
    if (d3 >= T(0) && d4 <= d3) return b;
    const T vc = d1 * d4 - d3 * d2;
    if (vc <= T(0) && d1 >= T(0) && d3 <= T(0)) return a + (d1 / (d1 - d3)) * ab;
    const V3<T> cp = p - c;
    const T d5 = dot(ab, cp), d6 = dot(ac, cp);
    if (d6 >= T(0) && d5 <= d6) return c;
    const T vb = d5 * d2 - d1 * d6;
    if (vb <= T(0) && d2 >= T(0) && d6 <= T(0)) return a + (d2 / (d2 - d6)) * ac;
    const T va = d3 * d6 - d5 * d4;
    if (va <= T(0) && (d4 - d3) >= T(0) && (d5 - d6) >= T(0)) return b + ((d4 - d3) / ((d4 - d3) + (d5 - d6))) * (c - b);
    const T den = T(1) / (va + vb + vc);
    return a + (vb * den) * ab + (vc * den) * ac;
  }
  // closest points of segments p1 + s d1 and p2 + t d2, s, t in [0, 1] (Ericson 5.1.9)
  static void closest_segments(V3<T> p1, V3<T> d1, V3<T> p2, V3<T> d2, T& s, T& t) {
    const V3<T> r = p1 - p2;
    const T a = dot(d1, d1), e = dot(d2, d2), f = dot(d2, r), eps = T(1e-12);
    if (a <= eps && e <= eps) { s = t = T(0); return; }
    if (a <= eps) { s = T(0); t = std::min(std::max(f / e, T(0)), T(1)); return; }
    const T c = dot(d1, r);
    if (e <= eps) { t = T(0); s = std::min(std::max(-c / a, T(0)), T(1)); return; }
    const T b = dot(d1, d2), den = a * e - b * b;
    s = den > eps * a * e ? std::min(std::max((b * f - c * e) / den, T(0)), T(1)) : T(0);
    t = (b * s + f) / e;
    if (t < T(0)) { t = T(0); s = std::min(std::max(-c / a, T(0)), T(1)); }
    else if (t > T(1)) { t = T(1); s = std::min(std::max((b - c) / a, T(0)), T(1)); }
  }
  // One candidate of a feature loop: keeps the deepest contact; a later triangle must be deeper by more than TIE to replace an
  // earlier one (two triangles that share the touched edge give the same depth to rounding: the lower pair index wins everywhere).
  struct Best { bool hit = false; T depth = 0; V3<T> n{0, 0, 1}, pos{0, 0, 0}; int pair = 0; };
  static void offer(Best& b, T depth, V3<T> n, V3<T> pos, int pair) {
    if (!(depth > T(0))) return;
    if (!b.hit || depth > b.depth + T(1e-6)) { b.hit = true; b.depth = depth; b.n = n; b.pos = pos; b.pair = pair; }
  }
  static V3<T> tri_normal(V3<T> a, V3<T> b, V3<T> c) {
    V3<T> n = cross(b - a, c - a);
    T inv = T(1) / std::sqrt(dot(n, n));
    if (n.z < T(0)) inv = -inv;
    return inv * n;
  }
  // cells [ix0, ix1] x [iy0, iy1] under the axis-aligned box [lo, hi] (all of them, clamped to the map); false: the shape's centre
  // (cxp, cyp) is off the map, no contact
  static bool cell_range(const HmGrid& g, T lox, T hix, T loy, T hiy, T cxp, T cyp, int& ix0, int& ix1, int& iy0, int& iy1) {
    const T gx = (cxp - g.x0) / g.dx, gy = (cyp - g.y0) / g.dy;
    if (!(gx >= T(0)) || !(gy >= T(0)) || !(gx < T(g.xs - 1)) || !(gy < T(g.ys - 1))) return false;
    ix0 = std::max(int(std::floor((lox - g.x0) / g.dx)), 0); ix1 = std::min(int(std::floor((hix - g.x0) / g.dx)), g.xs - 2);
    iy0 = std::max(int(std::floor((loy - g.y0) / g.dy)), 0); iy1 = std::min(int(std::floor((hiy - g.y0) / g.dy)), g.ys - 2);
    return true;
  }
  // sphere (centre C, radius r > 0) against the triangles under its footprint [C +- r]: the terrain point closest to the centre decides.
  // Centre above the surface (the usual case): depth = r - distance, pushed out along the line to that point (face, edge or vertex);
  // centre under the surface (deep penetration; inside / outside from the triangle directly beneath the centre): depth = r + distance,
  // along that triangle's normal.  The cells are visited in 2 x 2 blocks, eight triangles per block (slot k: cell (k >> 1) & 1, k >> 2
  // of the block, triangle k & 1; the kernel gives each slot a lane): when the footprint fits in the 2 x 2 block nearest to the centre
  // (always for radii up to half the pitch) that block alone, else the blocks from the footprint's first cell on, in steps of two
  // cells, iy-major.  Each slot keeps its closest triangle (a later block's only when strictly closer); of the slots within 1e-6 m of
  // the smallest distance (they share the touched edge or vertex) the lowest pair index wins.
  void sphere_vs_heightmap(const HmGrid& g, V3<T> C, T r, Best& best) const {
    const T gx = (C.x - g.x0) / g.dx, gy = (C.y - g.y0) / g.dy;
    if (!(gx >= T(0)) || !(gy >= T(0)) || !(gx < T(g.xs - 1)) || !(gy < T(g.ys - 1))) return;
    const int ccx = int(gx), ccy = int(gy);
    int bx = std::min(std::max(int(std::floor(gx - T(0.5))), 0), std::max(g.xs - 3, 0)), by = std::min(std::max(int(std::floor(gy - T(0.5))), 0), std::max(g.ys - 3, 0));
    const int fx0 = std::max(int(std::floor(gx - r / g.dx)), 0), fx1 = std::min(int(std::floor(gx + r / g.dx)), g.xs - 2);
    const int fy0 = std::max(int(std::floor(gy - r / g.dy)), 0), fy1 = std::min(int(std::floor(gy + r / g.dy)), g.ys - 2);
    int nbx = 1, nby = 1;
    if (fx0 < bx || fx1 > bx + 1 || fy0 < by || fy1 > by + 1) { bx = fx0; by = fy0; nbx = (fx1 - fx0 + 2) >> 1; nby = (fy1 - fy0 + 2) >> 1; }
    T dist[8]; V3<T> vv[8], nn[8]; int pr[8]; bool ok[8];
    for (int k = 0; k < 8; k++) ok[k] = false;
    bool inside = false; T dmin = T(3.0e38);
    for (int p = 0; p < nbx * nby; p++)
      for (int k = 0; k < 8; k++) {
        const int ix = bx + 2 * (p % nbx) + ((k >> 1) & 1), iy = by + 2 * (p / nbx) + (k >> 2), tri = k & 1;
        if (ix > g.xs - 2 || iy > g.ys - 2) continue;
        const V3<T> a = vertex(g, ix, iy), b = tri == 0 ? vertex(g, ix + 1, iy) : vertex(g, ix + 1, iy + 1), c = tri == 0 ? vertex(g, ix + 1, iy + 1) : vertex(g, ix, iy + 1);
        const V3<T> nt = tri_normal(a, b, c);
        const T side = dot(C - a, nt);
        if (ix == ccx && iy == ccy) {                            // the triangle directly beneath the centre tells inside from outside
          const T fx = gx - T(ccx), fy = gy - T(ccy);
          if ((fx >= fy) == (tri == 0)) inside = side < T(0);
        }
        if (side - r > T(0)) continue;                           // the whole sphere is above this triangle's plane
        const V3<T> Q = closest_on_triangle(C, a, b, c);
        const V3<T> v = C - Q;
        const T d = std::sqrt(dot(v, v));
        if (ok[k] && !(d < dist[k])) continue;                   // the slot keeps its closest triangle
        vv[k] = v; nn[k] = nt; dist[k] = d;
        pr[k] = 2 * (iy * (g.xs - 1) + ix) + tri;
        ok[k] = true;
        dmin = std::min(dmin, d);
      }
    int win = -1;
    for (int k = 0; k < 8; k++) if (ok[k] && dist[k] <= dmin + T(1e-6) && (win < 0 || pr[k] < pr[win])) win = k;
    if (win < 0) return;
    const T d = dist[win];
    const V3<T> n = (!inside && d > T(1e-9)) ? (T(1) / d) * vv[win] : nn[win];
    offer(best, inside ? r + d : r - d, n, C - r * n, pr[win]);
  }
  // interior of segment A-B swept by radius r against the terrain edges under its AABB (the end spheres are candidates of their own)
  void segment_vs_heightmap(const HmGrid& g, V3<T> A, V3<T> B, T r, Best& best) const {
    int ix0, ix1, iy0, iy1;
    const V3<T> M = T(0.5) * (A + B);
    if (!cell_range(g, std::min(A.x, B.x) - r, std::max(A.x, B.x) + r, std::min(A.y, B.y) - r, std::max(A.y, B.y) + r, M.x, M.y, ix0, ix1, iy0, iy1)) return;
    const V3<T> d1 = B - A;
    for (int iy = iy0; iy <= iy1; iy++) for (int ix = ix0; ix <= ix1; ix++) {
      const V3<T> p00 = vertex(g, ix, iy), p10 = vertex(g, ix + 1, iy), p01 = vertex(g, ix, iy + 1), p11 = vertex(g, ix + 1, iy + 1);
      const V3<T> n0 = tri_normal(p00, p10, p11), n1 = tri_normal(p00, p11, p01);
      // the five edges of the cell: bottom, right (tri 0), diagonal (both), top, left (tri 1); o0 / o1 = the third vertex of the
      // cell's triangle(s) on that edge
      const V3<T> e0[5] = {p00, p10, p00, p01, p00}, e1[5] = {p10, p11, p11, p11, p01};
      const V3<T> o0[5] = {p11, p00, p10, p00, p11}, o1[5] = {p11, p00, p01, p00, p11};
      for (int k = 0; k < 5; k++) {
        T sgm, tt;
        closest_segments(A, d1, e0[k], e1[k] - e0[k], sgm, tt);
        if (!(sgm > T(1e-3)) || !(sgm < T(1) - T(1e-3))) continue;      // an end of the segment: the end sphere's business
        const V3<T> Ps = A + sgm * d1, Pe = e0[k] + tt * (e1[k] - e0[k]);
        const V3<T> v = Ps - Pe;
        const T dist = std::sqrt(dot(v, v));
        const int tri = k < 3 ? 0 : 1;
        const V3<T> nt = tri == 0 ? n0 : n1;
        // a true edge contact: the segment point lies beyond the edge as seen from the triangle(s) of this cell on it (v . m < 0, m = the
        // in-plane direction from the edge into the triangle).  Over a face (or a flat / concave edge) the segment interior is never the
        // first thing to touch -- the end spheres are -- so a flat height map gives exactly the contacts of a ground plane.
        const V3<T> ed = e1[k] - e0[k];
        const T ee = dot(ed, ed);
        bool convex = true;
        for (int q = 0; q < 2; q++) {
          const V3<T> w = (q == 0 ? o0[k] : o1[k]) - e0[k];
          const V3<T> m = w - (dot(w, ed) / ee) * ed;
          if (!(dot(v, m) < T(-1e-6) * dist * std::sqrt(dot(m, m)))) convex = false;
        }
        if (!convex) continue;
        if (!(dot(v, nt) > T(0)) || !(dist < r) || !(dist > T(1e-9))) continue;   // from above only: a segment under the surface is the end spheres' business
        const V3<T> n = (T(1) / dist) * v;
        offer(best, r - dist, n, Ps - r * n, 2 * (iy * (g.xs - 1) + ix) + tri);
      }
    }
  }
  // terrain vertices inside the box (centre c, rotation R, half extents h): the vertex deepest inside, pushed out through its nearest face
  void box_vs_heightmap(const HmGrid& g, V3<T> c, const M3<T>& R, V3<T> h, Best& best) const {
    const T ex = std::fabs(R.m[0]) * h.x + std::fabs(R.m[1]) * h.y + std::fabs(R.m[2]) * h.z, ey = std::fabs(R.m[3]) * h.x + std::fabs(R.m[4]) * h.y + std::fabs(R.m[5]) * h.z;
    int ix0, ix1, iy0, iy1;
    if (!cell_range(g, c.x - ex, c.x + ex, c.y - ey, c.y + ey, c.x, c.y, ix0, ix1, iy0, iy1)) return;
    for (int iy = iy0; iy <= iy1 + 1; iy++) for (int ix = ix0; ix <= ix1 + 1; ix++) {
      const V3<T> V = vertex(g, ix, iy);
      // only a vertex that stands proud of its four neighbours (a peak, a ridge point) can reach a face before the box's own corners
      // reach the terrain: on a flat or evenly sloping map this candidate adds nothing to the corners (flat height map == ground plane)
      const T hn = T(0.25) * (g.H[iy * g.xs + std::max(ix - 1, 0)] + g.H[iy * g.xs + std::min(ix + 1, g.xs - 1)] + g.H[std::max(iy - 1, 0) * g.xs + ix] + g.H[std::min(iy + 1, g.ys - 1) * g.xs + ix]);
      if (!(V.z - hn > T(1e-6))) continue;
      const V3<T> q = R.tmul(V - c);
      const T px = h.x - std::fabs(q.x), py = h.y - std::fabs(q.y), pz = h.z - std::fabs(q.z);
      if (!(px > T(0)) || !(py > T(0)) || !(pz > T(0))) continue;
      // nearest face; its outward normal is the way the terrain vertex leaves the box, the contact normal (terrain -> robot) is its opposite
      V3<T> nf; T pen;
      if (px <= py && px <= pz) { pen = px; nf = {q.x >= T(0) ? T(1) : T(-1), 0, 0}; }
      else if (py <= pz) { pen = py; nf = {0, q.y >= T(0) ? T(1) : T(-1), 0}; }
      else { pen = pz; nf = {0, 0, q.z >= T(0) ? T(1) : T(-1)}; }
      const V3<T> n = T(-1) * (R * nf);
      const int cix = std::min(ix, g.xs - 2), ciy = std::min(iy, g.ys - 2);
      offer(best, pen, n, V, 2 * (ciy * (g.xs - 1) + cix));
    }
  }

  // every terrain hit into ws.all in candidate order, ranked into ws.contacts.  Virtual, like jacobians(): the two stages of step()
  // that the self-collision restatement (self_collision.hpp) replaces
  virtual void collide(Workspace<T>& ws) const {
    std::vector<Contact<T>>& all = ws.all;
    all.clear();
    const bool hm = ter.type == 2;
    const HmGrid g = hm ? grid(ws.hm_offset) : HmGrid{};
    for (int k = 0; k < npts; k++) {
      int b = pt_body[k];
      if (b == 0 && !floating) continue;               // a body welded to the world cannot collide
      Best best;
      V3<T> P = ws.p[b] + ws.R[b] * pt_pos[k];
      T rad = pt_rad[k];
      bool as_point = pt_type[k] == 0 && !(hm && rad > T(0));
      if (pt_type[k] == 3) {
        // cylinder cap: the lowest point of its rim circle (centre P, radius rad, axis a) -- the point of the circle furthest along -z
        V3<T> a = P - (ws.p[b] + ws.R[b] * pt_pos2[k]);
        a = (T(1) / std::sqrt(dot(a, a))) * a;
        V3<T> dd = {a.z * a.x, a.z * a.y, a.z * a.z - T(1)};        // -(e_z - (e_z . a) a)
        const T dn = std::sqrt(dot(dd, dd));
        if (!(dn > T(1e-6))) continue;                              // cap parallel to the ground: the fixed rim samples carry it
        P = P + (rad / dn) * dd; rad = T(0); as_point = true;
      }
      if (as_point) {
        // plane, or a zero-radius point on a height map (box corner, cylinder rim point): the triangle directly beneath
        T dist; V3<T> n; int pair;
        if (!terrain_query(P, dist, n, pair, ws.hm_offset)) continue;
        offer(best, rad - dist, n, P - rad * n, pair);
      } else if (!hm) continue;                        // segment interiors and box faces add nothing on a plane: ends and corners are deeper
      else if (pt_type[k] == 0) sphere_vs_heightmap(g, P, rad, best);
      else if (pt_type[k] == 1) segment_vs_heightmap(g, P, ws.p[b] + ws.R[b] * pt_pos2[k], rad, best);
      else {
        const int ci = pt_coll[k];
        box_vs_heightmap(g, ws.p[b] + ws.R[b] * coll_pos[ci], ws.R[b] * coll_rot[ci], coll_size[ci], best);
      }
      if (!best.hit) continue;
      Contact<T> c;
      c.pt = k; c.body = b; c.pair = best.pair; c.n = best.n; c.depth = best.depth; c.pos = best.pos;
      tangent_frame(c);
      c.lam = {0, 0, 0};
      c.sdir = SlipDir<T>();
      all.push_back(c);
    }
    rank_contacts(ws);
  }

  // tangent basis: t1 = normalised projection of e_x (or e_y when n is nearly along x)
  static void tangent_frame(Contact<T>& c) {
    V3<T> e = (std::fabs(c.n.x) < T(0.9)) ? V3<T>{1, 0, 0} : V3<T>{0, 1, 0};
    V3<T> t = e - dot(e, c.n) * c.n;
    T inv = T(1) / std::sqrt(dot(t, t));
    c.t1 = inv * t; c.t2 = cross(c.n, c.t1);
  }

  // ws.contacts = the KMAX deepest of ws.all (ties: lower candidate index wins), emitted in candidate order
  static void rank_contacts(Workspace<T>& ws) {
    const std::vector<Contact<T>>& all = ws.all;
    ws.contacts.clear();
    if ((int)all.size() > KMAX) {
      std::vector<int> idx(all.size());
      for (size_t i = 0; i < idx.size(); i++) idx[i] = int(i);
      std::stable_sort(idx.begin(), idx.end(), [&](int a, int b) { return all[a].depth > all[b].depth; });
      idx.resize(KMAX);
      std::sort(idx.begin(), idx.end());
      for (int i : idx) ws.contacts.push_back(all[i]);
    } else ws.contacts = all;
  }

  // ---- dense Cholesky  A = L L^T (lower), a5 getInverseMassMatrix ---------------------------------
  static void cholesky(const T* A, T* L, int n) {
    for (int j = 0; j < n; j++) {
      T s = A[j * n + j];
      for (int k = 0; k < j; k++) s -= L[j * n + k] * L[j * n + k];
      T d = std::sqrt(s); L[j * n + j] = d;
      T inv = T(1) / d;
      for (int i = j + 1; i < n; i++) {
        T t = A[i * n + j];
        for (int k = 0; k < j; k++) t -= L[i * n + k] * L[j * n + k];
        L[i * n + j] = t * inv;
      }
      for (int i = 0; i < j; i++) L[i * n + j] = T(0);
    }
  }
  static void fwd_solve(const T* L, T* x, int n, int stride = 1) {   // x <- L^-1 x
    for (int i = 0; i < n; i++) {
      T s = x[i * stride];
      for (int k = 0; k < i; k++) s -= L[i * n + k] * x[k * stride];
      x[i * stride] = s / L[i * n + i];
    }
  }
  static void bwd_solve(const T* L, T* x, int n) {   // x <- L^-T x
    for (int i = n - 1; i >= 0; i--) {
      T s = x[i];
      for (int k = i + 1; k < n; k++) s -= L[k * n + i] * x[k];
      x[i] = s / L[i * n + i];
    }
  }

  // ---- a7: contact Jacobian rows in the contact frame; Jt is nv x 3K (row r of Jt = dof r) -------
  virtual void jacobians(Workspace<T>& ws) const {
    int K = int(ws.contacts.size()), C = 3 * K + int(ws.limits.size());
    std::fill(ws.Jt.begin(), ws.Jt.begin() + nv * C, T(0));
    for (size_t l = 0; l < ws.limits.size(); l++) ws.Jt[ws.limits[l].dof * C + 3 * K + int(l)] = ws.limits[l].sign;
    for (int ci = 0; ci < K; ci++) {
      const Contact<T>& c = ws.contacts[ci];
      V3<T> ax[3] = {c.t1, c.t2, c.n};
      if (floating) {
        V3<T> r = c.pos - ws.p[0];
        for (int d = 0; d < 3; d++) {
          V3<T> rc = cross(r, ax[d]);        // (e_k x r) . ax = e_k . (r x ax)
          ws.Jt[0 * C + 3 * ci + d] = ax[d].x; ws.Jt[1 * C + 3 * ci + d] = ax[d].y; ws.Jt[2 * C + 3 * ci + d] = ax[d].z;
          ws.Jt[3 * C + 3 * ci + d] = rc.x; ws.Jt[4 * C + 3 * ci + d] = rc.y; ws.Jt[5 * C + 3 * ci + d] = rc.z;
        }
      }
      for (int j = c.body; parent[j] >= 0; j = parent[j]) {
        V3<T> col = (jtype[j] == JT_REVOLUTE) ? cross(ws.a[j], c.pos - ws.p[j]) : ws.a[j];
        for (int d = 0; d < 3; d++) ws.Jt[vidx[j] * C + 3 * ci + d] = dot(col, ax[d]);
      }
    }
  }

  // ---- a8: per-contact solve (Hwangbo et al. 2018, section IV) ------------------------------------
  // G: 3x3 (rows/cols t1,t2,n) block G_ii; c: contact velocity without this contact's own impulse
  // (already shifted by the ERP / restitution target).  Returns the new impulse.
  void solve_one(const T* G, V3<T> c, T mu, V3<T>& lam, SlipDir<T>* sd = nullptr, long long* counts = nullptr) const {
    SlipDir<T> prev; if (sd) { prev = *sd; sd->valid = false; }
    if (c.z > T(0)) { lam = {0, 0, 0}; if (counts) counts[0]++; return; }                 // opening
    // stick candidate: lam = -G^-1 c
    T a = G[0], b = G[1], cc = G[2], d = G[4], e = G[5], f = G[8];
    T c00 = d * f - e * e, c01 = cc * e - b * f, c02 = b * e - cc * d;
    T c11 = a * f - cc * cc, c12 = b * cc - a * e, c22 = a * d - b * b;
    T det = a * c00 + b * c01 + cc * c02;
    T id = T(1) / det;
    V3<T> ls = {-(c00 * c.x + c01 * c.y + c02 * c.z) * id, -(c01 * c.x + c11 * c.y + c12 * c.z) * id, -(c02 * c.x + c12 * c.y + c22 * c.z) * id};
    if (ls.z >= T(0) && ls.x * ls.x + ls.y * ls.y <= mu * mu * ls.z * ls.z) { lam = ls; if (counts) counts[1]++; return; }   // stick
    if (counts) counts[2]++;
    // slip: lam(theta) = lz(theta) * (mu cos, mu sin, 1),  lz = -c_z / (G_zz + mu (G_zx cos + G_zy sin))
    // minimise f = c.lam + 1/2 lam^T G lam on that curve: find the - to + sign change of
    //   g(theta) = (v_t . u_perp) D - mu (G_zt . u_perp)(v_t . u),    v_t = tangential part of c + G lam
    // by NSEC-section search (a bisection generalised to 32 simultaneous probes), NROUNDS rounds.
    auto eval = [&](T cs, T sn, T& gval, T& fval, V3<T>& l) -> bool {
      T D = f + mu * (cc * cs + e * sn);
      if (!(D > T(1e-12))) return false;
      T lz = -c.z / D;
      l = {mu * lz * cs, mu * lz * sn, lz};
      T vx = c.x + a * l.x + b * l.y + cc * l.z;
      T vy = c.y + b * l.x + d * l.y + e * l.z;
      gval = (-vx * sn + vy * cs) * D - mu * (-cc * sn + e * cs) * (vx * cs + vy * sn);
      fval = c.x * l.x + c.y * l.y + c.z * l.z + T(0.5) * (l.x * vx + l.y * vy - l.z * c.z) - T(0.5) * (c.x * l.x + c.y * l.y);
      return true;
    };
    // note: fval above equals c.lam + 1/2 lam^T G lam with (G lam)_z = -c_z on the curve:
    //   1/2 lam.(G lam) = 1/2 (lx (vx - cx) + ly (vy - cy) + lz (-cz))
    T base_c = T(1), base_s = T(0);       // bracket start direction (contact-frame +x for round 0)
    V3<T> best = {0, 0, 0};
    bool have = false;
    T glo = 0, ghi = 0; T lo_c = 1, lo_s = 0, hi_c = 1, hi_s = 0;
    int r_start = 0;
    if (prev.valid && prm.slip_local && !prm.slip_bisect) {
      // local fan first: 32 probes = 31 sections of the round-1 table, centred on the previous slip direction
      const T hc = T(std::cos(M_PI / NSEC)), hs = T(std::sin(M_PI / NSEC));
      const T b_c = prev.cs * hc + prev.sn * hs, b_s = prev.sn * hc - prev.cs * hs;
      T gk[NSEC], fk[NSEC]; bool ok[NSEC]; V3<T> lk[NSEC]; T dc[NSEC], ds[NSEC];
      for (int k = 0; k < NSEC; k++) {
        dc[k] = b_c * sec_c[1][k] - b_s * sec_s[1][k];
        ds[k] = b_s * sec_c[1][k] + b_c * sec_s[1][k];
        ok[k] = eval(dc[k], ds[k], gk[k], fk[k], lk[k]);
      }
      int pick = -1; T fbest = 0;
      for (int k = 0; k + 1 < NSEC; k++)
        if (ok[k] && ok[k + 1] && gk[k] < T(0) && gk[k + 1] >= T(0) && (pick < 0 || fk[k] < fbest)) { pick = k; fbest = fk[k]; }
      if (pick >= 0) {
        lo_c = dc[pick]; lo_s = ds[pick]; hi_c = dc[pick + 1]; hi_s = ds[pick + 1]; glo = gk[pick]; ghi = gk[pick + 1];
        base_c = lo_c; base_s = lo_s; have = true; best = lk[pick];
        r_start = NROUNDS;
        if (counts) counts[3]++;
      }
    }
    for (int r = r_start; r < (prm.slip_bisect ? 1 : NROUNDS); r++) {
      T gk[NSEC + 1], fk[NSEC + 1]; bool ok[NSEC + 1]; V3<T> lk[NSEC + 1];
      T dc[NSEC + 1], ds[NSEC + 1];
      for (int k = 0; k < NSEC; k++) {
        dc[k] = base_c * sec_c[r][k] - base_s * sec_s[r][k];
        ds[k] = base_s * sec_c[r][k] + base_c * sec_s[r][k];
        ok[k] = eval(dc[k], ds[k], gk[k], fk[k], lk[k]);
      }
      // the closing direction is never re-evaluated: probe 0 again in round 0 (full circle), the
      // previous round's upper end afterwards
      if (r == 0) { dc[NSEC] = dc[0]; ds[NSEC] = ds[0]; ok[NSEC] = ok[0]; gk[NSEC] = gk[0]; fk[NSEC] = fk[0]; lk[NSEC] = lk[0]; }
      else { dc[NSEC] = hi_c; ds[NSEC] = hi_s; ok[NSEC] = true; gk[NSEC] = ghi; fk[NSEC] = T(0); lk[NSEC] = best; }
      int pick = -1; T fbest = 0;
      for (int k = 0; k < NSEC; k++) {
        if (!ok[k] || !ok[k + 1]) continue;
        if (gk[k] < T(0) && gk[k + 1] >= T(0)) {
          if (pick < 0 || fk[k] < fbest) { pick = k; fbest = fk[k]; }
        }
      }
      if (pick < 0) {
        if (!have) {   // no bracket on the whole circle: take the probe with the least energy
          int kb = -1;
          for (int k = 0; k < NSEC; k++) if (ok[k] && (kb < 0 || fk[k] < fk[kb])) kb = k;
          if (kb >= 0) { lam = lk[kb]; } else { lam = {0, 0, std::max(T(0), -c.z / f)}; }
          return;
        }
        break;         // keep the bracket of the previous round
      }
      T cs0 = dc[pick], sn0 = ds[pick], cs1 = dc[pick + 1], sn1 = ds[pick + 1];
      lo_c = cs0; lo_s = sn0; hi_c = cs1; hi_s = sn1; glo = gk[pick]; ghi = gk[pick + 1];
      base_c = cs0; base_s = sn0; have = true; best = lk[pick];
    }
    if (!prm.slip_bisect && have) {
      // regula falsi inside the final bracket, Illinois variant (an end kept twice has its value halved): every step is ONE
      // probe, the direction is the normalised chord point.  2 steps from a 6e-3 rad bracket: exact to float32 rounding.
      T wlo = glo, whi = ghi; int side = 0;
      T cs = lo_c, sn = lo_s; V3<T> l = best;
      for (int st = 0; st < NREF; st++) {
        T tt = wlo / (wlo - whi);
        T c2 = lo_c + tt * (hi_c - lo_c), s2 = lo_s + tt * (hi_s - lo_s);
        T inv = T(1) / std::sqrt(c2 * c2 + s2 * s2);
        c2 *= inv; s2 *= inv;
        T g2, f2; V3<T> l2;
        if (!eval(c2, s2, g2, f2, l2)) break;
        cs = c2; sn = s2; l = l2;
        if (g2 < T(0)) { lo_c = c2; lo_s = s2; wlo = g2; if (side == -1) whi *= T(0.5); side = -1; }
        else { hi_c = c2; hi_s = s2; whi = g2; if (side == 1) wlo *= T(0.5); side = 1; }
      }
      lam = l;
      if (sd) { sd->valid = true; sd->cs = cs; sd->sn = sn; }
      return;
    }
    if (prm.slip_bisect) {   // CPU-tuned variant: 10 halvings of the round-0 bracket (2*pi/32768), then the secant step below
      for (int it = 0; it < 10; it++) {
        T mc = lo_c + hi_c, ms = lo_s + hi_s;
        T inv = T(1) / std::sqrt(mc * mc + ms * ms);
        mc *= inv; ms *= inv;
        T gm, fm; V3<T> lm;
        if (!eval(mc, ms, gm, fm, lm)) break;
        if (gm < T(0)) { lo_c = mc; lo_s = ms; glo = gm; best = lm; } else { hi_c = mc; hi_s = ms; ghi = gm; }
      }
    }
    // secant step inside the final bracket, direction re-normalised
    T tt = (ghi - glo) != T(0) ? (-glo / (ghi - glo)) : T(0.5);
    T cs = lo_c + tt * (hi_c - lo_c), sn = lo_s + tt * (hi_s - lo_s);
    T inv = T(1) / std::sqrt(cs * cs + sn * sn);
    cs *= inv; sn *= inv;
    T gv_, fv_; V3<T> l;
    if (eval(cs, sn, gv_, fv_, l)) lam = l; else { lam = best; cs = lo_c; sn = lo_s; }
    if (sd) { sd->valid = true; sd->cs = cs; sd->sn = sn; }
  }

  // ---- a1: one World::integrate() for one environment -------------------------------------------
  // ctrl arrays may be null (treated as zero).  gc/gv updated in place.
  void step(T* gc, T* gv, const T* tau_ff, const T* ptarget, const T* vtarget, const T* kp, const T* kd, Workspace<T>& ws) const {
    T dt = T(prm.dt);
    fk(gc, ws);
    rnea_bias(gv, ws);
    crba(ws);
    collide(ws);
    // a5: generalized force with implicit PD (ArticulatedSystem::setPdGains / setPdTarget):
    //   b = tau_ff + Kp (q* - q - dt v) + Kd (v* - v) - h ;   Mhat = M + dt Kd + dt^2 Kp
    for (int i = 0; i < nv; i++) ws.b[i] = (tau_ff ? tau_ff[i] : T(0)) - ws.h[i];
    if (ws.ext_body >= 0) {   // b += J_p^T F + J_r^T T for a world-frame wrench at a point fixed in the body
      const int eb = ws.ext_body;
      const V3<T> P = ws.p[eb] + ws.R[eb] * ws.ext_pos;
      if (floating) {
        const V3<T> m = cross(P - ws.p[0], ws.ext_f) + ws.ext_t;
        ws.b[0] += ws.ext_f.x; ws.b[1] += ws.ext_f.y; ws.b[2] += ws.ext_f.z; ws.b[3] += m.x; ws.b[4] += m.y; ws.b[5] += m.z;
      }
      for (int j = eb; parent[j] >= 0; j = parent[j]) {
        if (jtype[j] == JT_REVOLUTE) ws.b[vidx[j]] += dot(cross(ws.a[j], P - ws.p[j]), ws.ext_f) + dot(ws.a[j], ws.ext_t);
        else if (jtype[j] == JT_PRISMATIC) ws.b[vidx[j]] += dot(ws.a[j], ws.ext_f);
      }
    }
    ws.Mh = ws.M;
    std::vector<T>& Mh = ws.Mh;
    for (int i = 1; i < nb; i++) {
      int vi = vidx[i], qi = qidx[i];
      T kpi = kp ? kp[vi] : T(0), kdi = kd ? kd[vi] : T(0);
      // actuator effort limit (URDF <limit effort>; upstream setActuationLimits): when the commanded torque -- feed-forward plus the PD
      // law at the current state -- exceeds it, the joint is driven by the constant limit torque over this step (no implicit PD terms)
      const T tff = tau_ff ? tau_ff[vi] : T(0);
      T te = tff;
      if (kpi != T(0) || kdi != T(0)) te += kpi * ((ptarget ? ptarget[qi] : T(0)) - gc[qi]) + kdi * ((vtarget ? vtarget[vi] : T(0)) - gv[vi]);
      // ... judged on the torque the implicit law would really apply: for a stiff loop (dt^2 kp >> inertia) that is the explicit value
      // divided by 1 + (dt kd + dt^2 kp) / M_dd, so a stiff controller sitting near its target is not mistaken for a saturated one
      ws.sat[vi] = std::fabs(te) > jeff[i] * (T(1) + (dt * kdi + dt * dt * kpi) / ws.M[vi * nv + vi]);
      if (ws.sat[vi]) { ws.b_sat[vi] = te > T(0) ? jeff[i] : -jeff[i]; ws.b[vi] += ws.b_sat[vi] - tff; continue; }
      if (kpi != T(0) || kdi != T(0)) {
        T qt = ptarget ? ptarget[qi] : T(0), vt = vtarget ? vtarget[vi] : T(0);
        ws.b[vi] += kpi * (qt - gc[qi] - dt * gv[vi]) + kdi * (vt - gv[vi]);
        Mh[vi * nv + vi] += dt * kdi + dt * dt * kpi;
      }
    }
    cholesky(Mh.data(), ws.L.data(), nv);
    for (int i = 0; i < nv; i++) ws.z[i] = ws.b[i];
    fwd_solve(ws.L.data(), ws.z.data(), nv);
    int K = int(ws.contacts.size());
    // a9 (joint limits): the first LMAX joints found beyond their limit become unilateral rows  sign * qdot >= erp * viol / dt
    ws.limits.clear();
    if (prm.joint_limits)
      for (int i = 1; i < nb && (int)ws.limits.size() < LMAX; i++) {
        T q = gc[qidx[i]];
        if (q < jlo[i]) ws.limits.push_back({vidx[i], T(1), jlo[i] - q, T(0)});
        else if (q > jhi[i]) ws.limits.push_back({vidx[i], T(-1), q - jhi[i], T(0)});
      }
    const int Lm = int(ws.limits.size()), C3 = 3 * K, C = C3 + Lm;
    for (int i = 0; i < nv; i++) ws.rhs[i] = dt * ws.z[i];
    ws.iters = 0; ws.resid = T(0); ws.status = 0;
    if (C > 0) {
      jacobians(ws);
      // Y = L^-1 J^T (nv x C);  G = Y^T Y;  u0 = J v + dt Y^T z - target
      for (int i = 0; i < nv * C; i++) ws.Y[i] = ws.Jt[i];
      for (int c = 0; c < C; c++) fwd_solve(ws.L.data(), ws.Y.data() + c, nv, C);
      for (int a = 0; a < C; a++) for (int b2 = 0; b2 < C; b2++) {
        T s = 0;
        for (int r = 0; r < nv; r++) s += ws.Y[r * C + a] * ws.Y[r * C + b2];
        ws.G[a * C + b2] = s;
      }
      for (int a = 0; a < C; a++) {
        T s = 0, s0 = 0;
        for (int r = 0; r < nv; r++) { s0 += ws.Jt[r * C + a] * gv[r]; s += ws.Y[r * C + a] * ws.z[r]; }
        ws.u[a] = s0 + dt * s;
        if (a >= C3) ws.u[a] -= T(prm.erp) * ws.limits[a - C3].viol / dt;
        else if (a % 3 == 2) {
          const Contact<T>& ct = ws.contacts[a / 3];
          T target = T(prm.erp) * ct.depth / dt;
          if (prm.restitution > 0 && s0 < -T(prm.rest_threshold)) target += -T(prm.restitution) * s0;
          ws.u[a] -= target;
        }
      }
      for (int a = 0; a < C; a++) ws.u0[a] = ws.u[a];
      if (prm.warm_start) {
        for (int i = 0; i < K; i++) {
          Contact<T>& ct = ws.contacts[i];
          for (int j = 0; j < KMAX; j++) if (ws.prev_pt[j] == ct.pt) {
            const V3<T>& w = ws.prev_imp[j];
            ct.lam = {dot(ct.t1, w), dot(ct.t2, w), dot(ct.n, w)};
          }
        }
        for (int a = 0; a < C; a++) {
          T s = 0;
          for (int i = 0; i < K; i++) {
            const V3<T>& l = ws.contacts[i].lam;
            s += ws.G[a * C + 3 * i] * l.x + ws.G[a * C + 3 * i + 1] * l.y + ws.G[a * C + 3 * i + 2] * l.z;
          }
          ws.u[a] += s;
        }
      }
      // a8: Gauss-Seidel over contacts (BisectionContactSolver::solve)
      T alpha = T(prm.alpha_init), mu = T(prm.mu);
      T err_ckpt = T(3.0e38);
      int next_ckpt = prm.stall_window;
      // Anderson acceleration state: sweep outputs g_k and residuals f_k = g_k - x_k of the last accel_m + 1 sweeps
      const int AM = std::min(std::max(prm.accel_m, 0), 3);
      std::vector<T> hx, hg, hf;          // current x, and history rows [slot][C]
      int hcount = 0, resets = 0;
      bool regularised = false;
      ws.status = 3;
      if (AM > 0) { hx.assign(C, T(0)); hg.assign((size_t)(AM + 1) * C, T(0)); hf.assign((size_t)(AM + 1) * C, T(0)); }
      for (int it = 0; it < prm.max_iter; it++) {
        T err = 0;
        if (AM > 0) {
          for (int i = 0; i < K; i++) { hx[3 * i] = ws.contacts[i].lam.x; hx[3 * i + 1] = ws.contacts[i].lam.y; hx[3 * i + 2] = ws.contacts[i].lam.z; }
          for (int l = 0; l < Lm; l++) hx[C3 + l] = ws.limits[l].lam;
        }
        for (int i = 0; i < K; i++) {
          Contact<T>& ct = ws.contacts[i];
          T Gii[9];
          for (int r = 0; r < 3; r++) for (int c2 = 0; c2 < 3; c2++) Gii[3 * r + c2] = ws.G[(3 * i + r) * C + 3 * i + c2];
          V3<T> l0 = ct.lam;
          V3<T> c0 = {ws.u[3 * i] - (Gii[0] * l0.x + Gii[1] * l0.y + Gii[2] * l0.z),
                      ws.u[3 * i + 1] - (Gii[3] * l0.x + Gii[4] * l0.y + Gii[5] * l0.z),
                      ws.u[3 * i + 2] - (Gii[6] * l0.x + Gii[7] * l0.y + Gii[8] * l0.z)};
          V3<T> ln;
          solve_one(Gii, c0, pt_mu[ct.pt] >= T(0) ? pt_mu[ct.pt] : mu, ln, &ct.sdir, ws.counts);
          V3<T> dl = alpha * (ln - l0);
          ct.lam = l0 + dl;
          for (int a = 0; a < C; a++) ws.u[a] += ws.G[a * C + 3 * i] * dl.x + ws.G[a * C + 3 * i + 1] * dl.y + ws.G[a * C + 3 * i + 2] * dl.z;
          err = std::max(err, std::max(std::fabs(dl.x), std::max(std::fabs(dl.y), std::fabs(dl.z))));
        }
        for (int l = 0; l < Lm; l++) {   // joint limits: lam >= 0, sign * qdot+ >= target, complementary
          const int r = C3 + l;
          Limit<T>& lm = ws.limits[l];
          T Grr = ws.G[r * C + r];
          T c0 = ws.u[r] - Grr * lm.lam;
          T ln = std::max(T(0), -c0 / Grr);
          T dl = alpha * (ln - lm.lam);
          lm.lam += dl;
          for (int a = 0; a < C; a++) ws.u[a] += ws.G[a * C + r] * dl;
          err = std::max(err, std::fabs(dl));
        }
        ws.iters = it + 1; ws.resid = err;
        alpha = std::max(T(prm.alpha_min), alpha * T(prm.alpha_decay));
        if (err < T(prm.threshold)) { ws.status = regularised ? 1 : 0; break; }
        // the stagnation check comes before the extrapolation, and the last sweep is not extrapolated: whatever ends the loop, the impulses
        // returned are the output of a projected sweep (inside their friction cones, normal parts >= 0)
        if (it + 1 == next_ckpt) {
          if (it + 1 >= 2 * prm.stall_window && err > T(prm.stall_ratio) * err_ckpt) {
            if (regularised || !(prm.stall_reg > 0)) { ws.status = 2; break; }
            // The per-contact rule is cycling on this contact set (typically a joint stop fighting a sticking contact of the same leg).
            // Go on with a slightly compliant set: G + eps I, eps = stall_reg * mean(diag G)  (constraint-force mixing, only here).
            T tr = 0;
            for (int a = 0; a < C; a++) tr += ws.G[a * C + a];
            const T eps = T(prm.stall_reg) * tr / T(C);
            for (int a = 0; a < C; a++) ws.G[a * C + a] += eps;
            for (int i = 0; i < K; i++) { const V3<T>& l = ws.contacts[i].lam; ws.u[3 * i] += eps * l.x; ws.u[3 * i + 1] += eps * l.y; ws.u[3 * i + 2] += eps * l.z; }
            for (int l = 0; l < Lm; l++) ws.u[C3 + l] += eps * ws.limits[l].lam;
            regularised = true; hcount = 0; resets = 0;
            err_ckpt = T(3.0e38); next_ckpt = it + 1 + prm.stall_window;
            continue;
          }
          err_ckpt = err; next_ckpt += prm.stall_window;
        }
        if (AM > 0 && it + 1 >= prm.accel_start - AM && resets < ACCEL_MAX_RESETS && it + 1 < prm.max_iter) {   // the history starts AM sweeps before the first extrapolation: nothing is kept (or paid for) on quickly converging problems
          // push (g, f) of this sweep; slots are a shift register, newest last
          if (hcount == AM + 1) {
            for (int sl = 0; sl < AM; sl++) for (int a = 0; a < C; a++) { hg[(size_t)sl * C + a] = hg[(size_t)(sl + 1) * C + a]; hf[(size_t)sl * C + a] = hf[(size_t)(sl + 1) * C + a]; }
            hcount = AM;
          }
          T* g = &hg[(size_t)hcount * C]; T* f = &hf[(size_t)hcount * C];
          for (int i = 0; i < K; i++) { g[3 * i] = ws.contacts[i].lam.x; g[3 * i + 1] = ws.contacts[i].lam.y; g[3 * i + 2] = ws.contacts[i].lam.z; }
          for (int l = 0; l < Lm; l++) g[C3 + l] = ws.limits[l].lam;
          T fn = 0, fp = 0;
          for (int a = 0; a < C; a++) { f[a] = g[a] - hx[a]; fn += f[a] * f[a]; }
          if (hcount > 0) for (int a = 0; a < C; a++) fp += hf[(size_t)(hcount - 1) * C + a] * hf[(size_t)(hcount - 1) * C + a];
          hcount++;
          if (hcount > 1 && fn > T(4) * fp) {          // residual doubled: drop the history, continue from the plain sweep output
            for (int a = 0; a < C; a++) { hg[a] = g[a]; hf[a] = f[a]; }
            hcount = 1; resets++;      // after ACCEL_MAX_RESETS such failures the plain sweeps finish the solve (rank-deficient
                                       // contact sets have a continuum of fixed points along which an extrapolation can run away)
          } else if (hcount > 1 && it + 1 >= prm.accel_start) {
            const int md = hcount - 1;                 // differences available
            T A[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, rhs[3] = {0, 0, 0}, gam[3] = {0, 0, 0};
            for (int p2 = 0; p2 < md; p2++) {
              for (int q2 = 0; q2 < md; q2++) {
                T sacc = 0;
                for (int a = 0; a < C; a++) sacc += (hf[(size_t)(p2 + 1) * C + a] - hf[(size_t)p2 * C + a]) * (hf[(size_t)(q2 + 1) * C + a] - hf[(size_t)q2 * C + a]);
                A[3 * p2 + q2] = sacc;
              }
              T sacc = 0;
              for (int a = 0; a < C; a++) sacc += (hf[(size_t)(p2 + 1) * C + a] - hf[(size_t)p2 * C + a]) * f[a];
              rhs[p2] = sacc;
            }
            T tr = 0; for (int p2 = 0; p2 < md; p2++) tr += A[3 * p2 + p2];
            for (int p2 = 0; p2 < md; p2++) A[3 * p2 + p2] += T(1e-10) * tr + T(1e-30);
            // Gaussian elimination without pivoting (SPD + ridge)
            bool ok = true;
            for (int p2 = 0; p2 < md && ok; p2++) {
              T piv = A[3 * p2 + p2];
              if (!(piv > T(0))) { ok = false; break; }
              for (int r2 = p2 + 1; r2 < md; r2++) {
                T m2 = A[3 * r2 + p2] / piv;
                for (int c2 = p2; c2 < md; c2++) A[3 * r2 + c2] -= m2 * A[3 * p2 + c2];
                rhs[r2] -= m2 * rhs[p2];
              }
            }
            if (ok) {
              for (int p2 = md - 1; p2 >= 0; p2--) {
                T sacc = rhs[p2];
                for (int c2 = p2 + 1; c2 < md; c2++) sacc -= A[3 * p2 + c2] * gam[c2];
                gam[p2] = sacc / A[3 * p2 + p2];
              }
              // x_next = g - sum_j gamma_j (g_{j+1} - g_j); then rebuild the contact velocities u = u0 + G x_next
              std::vector<T> xn(g, g + C);
              for (int p2 = 0; p2 < md; p2++) for (int a = 0; a < C; a++) xn[a] -= gam[p2] * (hg[(size_t)(p2 + 1) * C + a] - hg[(size_t)p2 * C + a]);
              for (int i = 0; i < K; i++) ws.contacts[i].lam = {xn[3 * i], xn[3 * i + 1], xn[3 * i + 2]};
              for (int l = 0; l < Lm; l++) ws.limits[l].lam = xn[C3 + l];
              for (int a = 0; a < C; a++) {
                T sacc = ws.u0[a];
                for (int b2 = 0; b2 < C; b2++) sacc += ws.G[a * C + b2] * xn[b2];
                ws.u[a] = sacc;
              }
            }
          }
        }
      }
      for (int r = 0; r < nv; r++) {
        T s = 0;
        for (int i = 0; i < K; i++) {
          const V3<T>& l = ws.contacts[i].lam;
          s += ws.Y[r * C + 3 * i] * l.x + ws.Y[r * C + 3 * i + 1] * l.y + ws.Y[r * C + 3 * i + 2] * l.z;
        }
        for (int l = 0; l < Lm; l++) s += ws.Y[r * C + C3 + l] * ws.limits[l].lam;
        ws.rhs[r] += s;
      }
    }
    for (int k = 0; k < KMAX; k++) {   // contact cache for the next step's warm start
      if (k < K) {
        const Contact<T>& ct = ws.contacts[k];
        ws.prev_pt[k] = ct.pt;
        ws.prev_imp[k] = ct.lam.x * ct.t1 + ct.lam.y * ct.t2 + ct.lam.z * ct.n;
      } else ws.prev_pt[k] = -1;
    }
    // a9: v+ = v + L^-T (dt z + Y lam);  q+ = q (+) dt v+
    bwd_solve(ws.L.data(), ws.rhs.data(), nv);
    for (int i = 0; i < nv; i++) gv[i] += ws.rhs[i];
    // generalized force applied over this step (implicit PD at q + dt v+, v+): ArticulatedSystem::getGeneralizedForce()
    for (int i = 0; i < nv; i++) ws.tau_applied[i] = tau_ff ? tau_ff[i] : T(0);
    for (int i = 1; i < nb; i++) {
      int vi = vidx[i], qi = qidx[i];
      T kpi = kp ? kp[vi] : T(0), kdi = kd ? kd[vi] : T(0);
      if (ws.sat[vi]) { ws.tau_applied[vi] = ws.tau_applied[vi] + (ws.b_sat[vi] - ws.tau_applied[vi]); continue; }
      if (kpi != T(0) || kdi != T(0)) {
        T qt = ptarget ? ptarget[qi] : T(0), vt = vtarget ? vtarget[vi] : T(0);
        ws.tau_applied[vi] += kpi * (qt - gc[qi] - dt * gv[vi]) + kdi * (vt - gv[vi]);
      }
    }
    if (floating) {
      for (int k = 0; k < 3; k++) gc[k] += dt * gv[k];
      V3<T> w = {gv[3], gv[4], gv[5]};
      T wn = std::sqrt(dot(w, w)), ang = wn * dt;
      T qw, qx, qy, qz;
      if (ang > T(1e-10)) { T s = std::sin(T(0.5) * ang) / wn; qw = std::cos(T(0.5) * ang); qx = s * w.x; qy = s * w.y; qz = s * w.z; }
      else { qw = 1; qx = T(0.5) * dt * w.x; qy = T(0.5) * dt * w.y; qz = T(0.5) * dt * w.z; }
      T pw = gc[3], px = gc[4], py = gc[5], pz = gc[6];
      T nw = qw * pw - qx * px - qy * py - qz * pz;     // dq (x) q : world-frame angular velocity
      T nx = qw * px + qx * pw + qy * pz - qz * py;
      T ny = qw * py - qx * pz + qy * pw + qz * px;
      T nz = qw * pz + qx * py - qy * px + qz * pw;
      T inv = T(1) / std::sqrt(nw * nw + nx * nx + ny * ny + nz * nz);
      gc[3] = nw * inv; gc[4] = nx * inv; gc[5] = ny * inv; gc[6] = nz * inv;
    }
    for (int i = 1; i < nb; i++) gc[qidx[i]] += dt * gv[vidx[i]];
  }
};

}  // namespace orc
