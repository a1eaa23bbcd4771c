// ORACLE C API of the self-collision restatement -- test infrastructure, NOT product code (see rbd_oracle.hpp).
// Builds liboracle_self.so: the oracle's C API (oracle_capi.cpp, included as it is) over SelfSim<T> (self_collision.hpp) in place of
// Sim<T> -- every orc_* entry point of liboracle.so, with the same arguments, on the restatement that also collides the enabled
// self-collision pairs -- plus the entry points that set the pairs and expose their narrow phase and Jacobian to the tests.
#include "counting_scalar.hpp"
#include "rbd_oracle.hpp"
#include "self_collision.hpp"

#define Sim SelfSim
#include "oracle_capi.cpp"
#undef Sim

template <typename T>
static void set_pairs(SelfSim<T>& sim, int n, const int* idesc, const double* geo) {
  std::vector<SelfPair<T>> pairs(n);
  for (int j = 0; j < n; j++) {
    SelfPair<T>& sp = pairs[j];
    const int* d = idesc + 6 * j; const double* g = geo + 24 * j;
    sp.kind = d[0]; sp.flip = d[1]; sp.body1 = d[2]; sp.body2 = d[3]; sp.bA = d[4]; sp.bB = d[5];
    auto v = [&](int o) { return V3<T>{T(g[o]), T(g[o + 1]), T(g[o + 2])}; };
    sp.a0 = v(0); sp.a1 = v(3); sp.b0 = v(6); sp.b1 = v(9);
    for (int k = 0; k < 9; k++) sp.bR.m[k] = T(g[12 + k]);
    sp.ra = T(g[21]); sp.rb = T(g[22]); sp.mu = T(g[23]);
  }
  sim.set_pairs(pairs);
}

template <typename T>
static int pair_geometry(const SelfSim<T>& sim, int j, const double* RA, const double* pA, const double* RB, const double* pB, double* out) {
  M3<T> Ra, Rb;
  for (int k = 0; k < 9; k++) { Ra.m[k] = T(RA[k]); Rb.m[k] = T(RB[k]); }
  T depth = T(0); V3<T> n{T(0), T(0), T(0)}, pos{T(0), T(0), T(0)};
  const bool hit = sim.self_pair_geometry(sim.self_pairs[j], Ra, V3<T>{T(pA[0]), T(pA[1]), T(pA[2])}, Rb, V3<T>{T(pB[0]), T(pB[1]), T(pB[2])}, depth, n, pos);
  const double o[7] = {double(depth), double(n.x), double(n.y), double(n.z), double(pos.x), double(pos.y), double(pos.z)};
  for (int k = 0; k < 7; k++) out[k] = o[k];
  return hit ? 1 : 0;
}

template <typename T>
static void contact_jacobians(const SelfSim<T>& sim, int n, const double* gc, int* ncontacts, int* c_pt, double* Jt) {
  Workspace<T> ws;
  sim.init_ws(ws);
  std::vector<T> q(sim.nq);
  for (int e = 0; e < n; e++) {
    for (int i = 0; i < sim.nq; i++) q[i] = T(gc[(size_t)e * sim.nq + i]);
    ws.hm_offset = 0;
    sim.contacts_and_jacobian(q.data(), ws);
    const int K = int(ws.contacts.size()), C = 3 * K;
    ncontacts[e] = K;
    for (int k = 0; k < KMAX; k++) c_pt[(size_t)e * KMAX + k] = k < K ? ws.contacts[k].pt : -1;
    for (int r = 0; r < sim.nv; r++)
      for (int a = 0; a < 3 * KMAX; a++) Jt[((size_t)e * sim.nv + r) * 3 * KMAX + a] = a < C ? double(ws.Jt[r * C + a]) : 0.0;
  }
}

extern "C" {

// self-collision pairs (self_collision.hpp SelfPair): idesc [n][6] = kind, flip, body1, body2, bA, bB; geo [n][24] = a0, a1, b0, b1,
// bR (9), ra, rb, mu.  n = 0 clears them.
void orc_set_self_pairs(void* hv, int n, const int* idesc, const double* geo) {
  Handle* h = static_cast<Handle*>(hv);
  if (h->d) set_pairs(*h->d, n, idesc, geo); else if (h->f) set_pairs(*h->f, n, idesc, geo); else set_pairs(*h->c, n, idesc, geo);
}

// narrow phase of pair j alone, bodies A and B of the pair at the given poses (row-major R): out = depth, normal (3), position (3)
int orc_self_pair_geometry(void* hv, int j, const double* RA, const double* pA, const double* RB, const double* pB, double* out) {
  Handle* h = static_cast<Handle*>(hv);
  return h->d ? pair_geometry(*h->d, j, RA, pA, RB, pB, out) : pair_geometry(*h->f, j, RA, pA, RB, pB, out);
}

// contact lists of the states gc [n][nq] (one map: no terrain atlas) and their contact Jacobians, transposed: Jt [n][nv][3 KMAX],
// column 3 k + (t1, t2, n) of contact k
void orc_self_contact_jacobians(void* hv, int n, const double* gc, int* ncontacts, int* c_pt, double* Jt) {
  Handle* h = static_cast<Handle*>(hv);
  if (h->d) contact_jacobians(*h->d, n, gc, ncontacts, c_pt, Jt); else contact_jacobians(*h->f, n, gc, ncontacts, c_pt, Jt);
}

}  // extern "C"
