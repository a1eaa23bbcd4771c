// ORACLE -- test infrastructure, NOT product code (see rbd_oracle.hpp).
// Self-collision between explicit pairs of a robot's collision bodies (rsb_batch_set_self_collision), restated on top of the oracle's
// Sim: SelfSim<T> runs Sim's step() and overrides two of its stages, collide() (the pair narrow phase, terrain and self hits ranked
// together) and jacobians() (the self-contact Jacobian J = J_first(p) - J_second(p)), and gives the pairs their friction.  Without
// pairs it computes exactly what Sim computes.
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
  using Sim<T>::nv; using Sim<T>::npts; using Sim<T>::parent; using Sim<T>::jtype; using Sim<T>::vidx; using Sim<T>::pt_mu;

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
  void collide(Workspace<T>& ws) const override {
    Sim<T>::collide(ws);                                 // ws.all: every terrain hit, in candidate order
    if (self_pairs.empty()) return;                      // Sim::collide's list as it is
    for (int j = 0; j < (int)self_pairs.size(); j++) {
      const SelfPair<T>& sp = self_pairs[j];
      Contact<T> c;
      if (!self_pair_geometry(sp, ws.R[sp.bA], ws.p[sp.bA], ws.R[sp.bB], ws.p[sp.bB], c.depth, c.n, c.pos)) continue;
      c.pt = npts + j; c.body = sp.body1; c.pair = -1 - sp.body2;
      Sim<T>::tangent_frame(c);
      c.lam = {0, 0, 0};
      c.sdir = SlipDir<T>();
      ws.all.push_back(c);
    }
    Sim<T>::rank_contacts(ws);
  }

  // Sim::jacobians, then the self contacts' columns rewritten as J_first(p) - J_second(p): the floating-base columns of the two halves
  // are equal and cancel, so do the columns of the common ancestors (the same point, the same joint)
  void jacobians(Workspace<T>& ws) const override {
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
    this->fk(gc, ws);
    collide(ws);
    ws.limits.clear();
    if (!ws.contacts.empty()) jacobians(ws);
  }
};

}  // namespace orc
