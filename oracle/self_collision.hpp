// ORACLE -- test infrastructure, NOT product code (see rbd_oracle.hpp).
// Self-collision between explicit pairs of a robot's collision bodies (rsb_batch_set_self_collision), restated on top of the oracle's
// Sim: SelfSim<T> adds the pair narrow phase, the ranking of terrain and self hits together, the self-contact Jacobian
// J = J_first(p) - J_second(p) and the per-pair friction.  Its step() is the text of Sim::step() with those two stages swapped in
// (collide_self, jacobians_self); without pairs it computes exactly what Sim::step() computes.
//
// A self contact (DESIGN.md section 2): candidate index npts + j for pair j, body = the pair's first body, pair = -1 - the pair's
// second body (terrain pair indices are >= 0), normal from the second body to the first.
#pragma once
#include "rbd_oracle.hpp"

namespace orc {

// One enabled self-collision pair.  Geometry in the frames of two bodies A and B: kind 0 = segment a0..a1 swept by ra against segment
// b0..b1 swept by rb (a sphere is a segment of length 0); kind 1 = sphere (centre a0, radius ra) against the box of centre b0, half
// extents b1 and rotation bR in the frame of B.  The normal points from B to A; flip = 1 when the caller listed the pair the other way
// round (first = B), which negates it.  The contact's first / second bodies are body1 / body2.
template <typename T> struct SelfPair {
  int kind = 0, flip = 0, body1 = 0, body2 = 0, bA = 0, bB = 0;
  V3<T> a0{0, 0, 0}, a1{0, 0, 0}, b0{0, 0, 0}, b1{0, 0, 0};
  M3<T> bR;
  T ra = 0, rb = 0, mu = -1;   // mu < 0: default material
};

template <typename T> class SelfSim : public Sim<T> {
 public:
  using Sim<T>::nb; using Sim<T>::nq; using Sim<T>::nv; using Sim<T>::floating; using Sim<T>::npts; using Sim<T>::prm;
  using Sim<T>::parent; using Sim<T>::jtype; using Sim<T>::qidx; using Sim<T>::vidx; using Sim<T>::jlo; using Sim<T>::jhi; using Sim<T>::jeff;
  using Sim<T>::pt_mu; using Sim<T>::fk; using Sim<T>::rnea_bias; using Sim<T>::crba; using Sim<T>::cholesky; using Sim<T>::fwd_solve;
  using Sim<T>::bwd_solve; using Sim<T>::solve_one;

  std::vector<SelfPair<T>> self_pairs;   // enabled pairs: candidate npts + j

  explicit SelfSim(const ModelDesc& d) : Sim<T>(d) {}

  // the pairs, and their friction as the friction of candidates npts + j (step() reads pt_mu[candidate])
  void set_pairs(const std::vector<SelfPair<T>>& p) {
    self_pairs = p;
    pt_mu.resize(npts + p.size());
    for (size_t j = 0; j < p.size(); j++) pt_mu[npts + j] = p[j].mu;
  }

  // closest points of segments p1 + s d1 and p2 + t d2 for the self-collision pairs (Ericson 5.1.9).  Deterministic rule for the
  // degenerate cases: a segment of length 0 (a sphere) takes s = 0 / t = 0; nearly parallel segments (sin^2 of the angle < 1e-6)
  // take s = 0, the start of the first segment, and its projection on the second (clamped, then s re-projected).
  static void closest_segments_self(V3<T> p1, V3<T> d1, V3<T> p2, V3<T> d2, T& s, T& t) {
    const V3<T> r = p1 - p2;
    const T a = dot(d1, d1), e = dot(d2, d2), f = dot(d2, r);
    if (a == T(0) && e == T(0)) { s = t = T(0); return; }
    if (a == T(0)) { s = T(0); t = std::min(std::max(f / e, T(0)), T(1)); return; }
    const T c = dot(d1, r);
    if (e == T(0)) { t = T(0); s = std::min(std::max(-c / a, T(0)), T(1)); return; }
    const T b = dot(d1, d2), den = a * e - b * b;
    s = den > T(1e-6) * a * e ? std::min(std::max((b * f - c * e) / den, T(0)), T(1)) : T(0);
    t = (b * s + f) / e;
    if (t < T(0)) { t = T(0); s = std::min(std::max(-c / a, T(0)), T(1)); }
    else if (t > T(1)) { t = T(1); s = std::min(std::max((b - c) / a, T(0)), T(1)); }
  }
  // Narrow phase of one self-collision pair with the two bodies at (RA, pA), (RB, pB): the deepest point, one contact.  Normal from
  // the second body to the first, position = midpoint of the two surface points, depth = rA + rB - distance (sphere-box: the sphere
  // radius minus the distance from the centre to the box, or plus the distance to the nearest face when the centre is inside; ties
  // of that face go to the lowest axis).  Returns false when the shapes do not overlap.
  static bool self_pair_geometry(const SelfPair<T>& sp, const M3<T>& RA, V3<T> pA, const M3<T>& RB, V3<T> pB, T& depth, V3<T>& n, V3<T>& pos) {
    V3<T> ng, SA, SB;
    if (sp.kind == 0) {
      const V3<T> A0 = pA + RA * sp.a0, A1 = pA + RA * sp.a1, B0 = pB + RB * sp.b0, B1 = pB + RB * sp.b1;
      T s, t;
      closest_segments_self(A0, A1 - A0, B0, B1 - B0, s, t);
      const V3<T> QA = A0 + s * (A1 - A0), QB = B0 + t * (B1 - B0), v = QA - QB;
      const T dist = std::sqrt(dot(v, v));
      depth = sp.ra + sp.rb - dist;
      if (!(depth > T(0))) return false;
      ng = dist > T(1e-9) ? (T(1) / dist) * v : V3<T>{0, 0, 1};       // coincident centres / axes: +z, a fixed rule
      SA = QA - sp.ra * ng; SB = QB + sp.rb * ng;
    } else {
      const V3<T> C = pA + RA * sp.a0, cb = pB + RB * sp.b0;
      const M3<T> R = RB * sp.bR;
      const V3<T> q = R.tmul(C - cb), h = sp.b1;
      const V3<T> cl = {std::min(std::max(q.x, -h.x), h.x), std::min(std::max(q.y, -h.y), h.y), std::min(std::max(q.z, -h.z), h.z)};
      V3<T> nl, bp;
      if (q.x != cl.x || q.y != cl.y || q.z != cl.z) {                // centre outside the box: the clamped point is the closest one
        const V3<T> d = q - cl;
        const T dist = std::sqrt(dot(d, d));
        depth = sp.ra - dist;
        if (!(depth > T(0))) return false;
        nl = (T(1) / dist) * d; bp = cl;
      } else {                                                         // inside: out through the nearest face, ties to the lowest axis
        const T px = h.x - std::fabs(q.x), py = h.y - std::fabs(q.y), pz = h.z - std::fabs(q.z);
        bp = q;
        if (px <= py && px <= pz) { depth = sp.ra + px; nl = {q.x >= T(0) ? T(1) : T(-1), 0, 0}; bp.x = nl.x * h.x; }
        else if (py <= pz) { depth = sp.ra + py; nl = {0, q.y >= T(0) ? T(1) : T(-1), 0}; bp.y = nl.y * h.y; }
        else { depth = sp.ra + pz; nl = {0, 0, q.z >= T(0) ? T(1) : T(-1)}; bp.z = nl.z * h.z; }
      }
      ng = R * nl;
      SA = C - sp.ra * ng; SB = cb + R * bp;
    }
    n = sp.flip ? T(-1) * ng : ng;
    pos = T(0.5) * (SA + SB);
    return true;
  }

  // terrain candidates (Sim::collide), then the pairs, ranked together: the KMAX deepest (ties: lower candidate index) in candidate order
  void collide_self(Workspace<T>& ws) const {
    Sim<T>::collide(ws);                                 // ws.all: every terrain hit, in candidate order
    std::vector<Contact<T>>& all = ws.all;
    for (int j = 0; j < (int)self_pairs.size(); j++) {
      const SelfPair<T>& sp = self_pairs[j];
      Contact<T> c;
      if (!self_pair_geometry(sp, ws.R[sp.bA], ws.p[sp.bA], ws.R[sp.bB], ws.p[sp.bB], c.depth, c.n, c.pos)) continue;
      c.pt = npts + j; c.body = sp.body1; c.pair = -1 - sp.body2;
      V3<T> e = (std::fabs(c.n.x) < T(0.9)) ? V3<T>{1, 0, 0} : V3<T>{0, 1, 0};
      V3<T> t = e - dot(e, c.n) * c.n;
      T inv = T(1) / std::sqrt(dot(t, t));
      c.t1 = inv * t; c.t2 = cross(c.n, c.t1);
      c.lam = {0, 0, 0};
      c.sdir = SlipDir<T>();
      all.push_back(c);
    }
    if (self_pairs.empty()) return;                      // Sim::collide's list as it is
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

  // Sim::jacobians, then the self contacts' columns rewritten as J_first(p) - J_second(p): the floating-base columns of the two halves
  // are equal and cancel, so do the columns of the common ancestors (the same point, the same joint)
  void jacobians_self(Workspace<T>& ws) const {
    Sim<T>::jacobians(ws);
    const int K = int(ws.contacts.size()), C = 3 * K + int(ws.limits.size());
    for (int ci = 0; ci < K; ci++) {
      const Contact<T>& c = ws.contacts[ci];
      if (c.pair >= 0) continue;
      const V3<T> ax[3] = {c.t1, c.t2, c.n};
      for (int r = 0; r < nv; r++) for (int d = 0; d < 3; d++) ws.Jt[r * C + 3 * ci + d] = T(0);
      for (int j = c.body; parent[j] >= 0; j = parent[j]) {
        V3<T> col = (jtype[j] == JT_REVOLUTE) ? cross(ws.a[j], c.pos - ws.p[j]) : ws.a[j];
        for (int d = 0; d < 3; d++) ws.Jt[vidx[j] * C + 3 * ci + d] += dot(col, ax[d]);
      }
      for (int j = -1 - c.pair; parent[j] >= 0; j = parent[j]) {
        V3<T> col = (jtype[j] == JT_REVOLUTE) ? cross(ws.a[j], c.pos - ws.p[j]) : ws.a[j];
        for (int d = 0; d < 3; d++) ws.Jt[vidx[j] * C + 3 * ci + d] -= dot(col, ax[d]);
      }
    }
  }

  // contact list and contact Jacobian of the state gc (no step, no joint-limit rows): the tests compare the self-contact rows with
  // finite differences and evaluate the contact velocities of a result
  void contacts_and_jacobian(const T* gc, Workspace<T>& ws) const {
    fk(gc, ws);
    collide_self(ws);
    ws.limits.clear();
    if (!ws.contacts.empty()) jacobians_self(ws);
  }

  // ---- a1: one World::integrate() for one environment -------------------------------------------
  // ctrl arrays may be null (treated as zero).  gc/gv updated in place.
  void step(T* gc, T* gv, const T* tau_ff, const T* ptarget, const T* vtarget, const T* kp, const T* kd, Workspace<T>& ws) const {
    T dt = T(prm.dt);
    fk(gc, ws);
    rnea_bias(gv, ws);
    crba(ws);
    collide_self(ws);          // terrain candidates, then the self-collision pairs, one ranking
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
      jacobians_self(ws);      // self contacts: J_first - J_second
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
