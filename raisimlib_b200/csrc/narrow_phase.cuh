// Stage B helpers: collision bodies against a HeightMap (SURVEY 8a row a6: raisimODE dCollide* / dHeightfield -- a shape against
// every triangle under the shape's axis-aligned bounding box, two triangles per cell).  Same geometry, same tie rule and the same
// candidate order as oracle/rbd_oracle.hpp (sphere_vs_heightmap, segment_vs_heightmap, box_vs_heightmap), written for one lane per
// contact candidate.  Included by step_kernel.cuh inside namespace rsb, after the f3 helpers and TerrainDesc.
//
// Cell (ix, iy) holds two triangles split along the diagonal P00-P11: tri 0 = (P00, P10, P11), tri 1 = (P00, P11, P01);
// pair index = 2 * cell + tri.  Every cell under the shape's horizontal reach is visited, whatever its size against the pitch
// (a sphere: its footprint [C +- r]; a capsule side or a box face: its axis-aligned bounding box); a shape whose centre is off the
// map has no contact.
#pragma once

struct HmBest { bool hit; float depth; f3 n, pos; int pair; };

// approximate reciprocal / reciprocal square root (MUFU, ~1e-7 relative): distances and normals here feed a 1e-6 m tie rule and a
// float32 pose, an IEEE division (15 instructions with its slow path) buys nothing
__device__ __forceinline__ float np_rcp(float x) { float r; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
__device__ __forceinline__ float np_rsqrt(float x) { float r; asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }

// keeps the deepest contact; a later triangle must be deeper by more than 1e-6 m to replace an earlier one (two triangles sharing the
// touched edge give the same depth to rounding: the lower pair index wins, in the oracle and here alike)
__device__ __forceinline__ void hm_offer(HmBest& b, float depth, f3 n, f3 pos, int pair) {
  if (!(depth > 0.f)) return;
  if (!b.hit || depth > b.depth + 1e-6f) { b.hit = true; b.depth = depth; b.n = n; b.pos = pos; b.pair = pair; }
}
__device__ __forceinline__ f3 hm_vertex(const TerrainDesc& t, const float* H, int ix, int iy) {
  return mk(t.x0 + (float)ix * t.dx, t.y0 + (float)iy * t.dy, __ldg(H + iy * t.xs + ix));
}
__device__ __forceinline__ f3 hm_tri_normal(f3 a, f3 b, f3 c) {
  f3 n = cross(b - a, c - a);
  float inv = np_rsqrt(dot(n, n));
  if (n.z < 0.f) inv = -inv;
  return inv * n;
}
__device__ __forceinline__ bool hm_cell_range(const TerrainDesc& t, float lox, float hix, float loy, float hiy, float cxp, float cyp, int& ix0, int& ix1, int& iy0, int& iy1) {
  const float gx = (cxp - t.x0) / t.dx, gy = (cyp - t.y0) / t.dy;
  if (!(gx >= 0.f) || !(gy >= 0.f) || !(gx < t.xmax) || !(gy < t.ymax)) return false;
  ix0 = max((int)floorf((lox - t.x0) / t.dx), 0); ix1 = min((int)floorf((hix - t.x0) / t.dx), t.xs - 2);
  iy0 = max((int)floorf((loy - t.y0) / t.dy), 0); iy1 = min((int)floorf((hiy - t.y0) / t.dy), t.ys - 2);
  return true;
}
// closest point of triangle (a, b, c) to p: Voronoi regions of the triangle (Ericson, Real-Time Collision Detection 5.1.5)
__device__ __forceinline__ f3 closest_on_triangle(f3 p, f3 a, f3 b, f3 c) {
  const f3 ab = b - a, ac = c - a, ap = p - a;
  const float d1 = dot(ab, ap), d2 = dot(ac, ap);
  if (d1 <= 0.f && d2 <= 0.f) return a;
  const f3 bp = p - b;
  const float d3 = dot(ab, bp), d4 = dot(ac, bp);
  if (d3 >= 0.f && d4 <= d3) return b;
  const float vc = d1 * d4 - d3 * d2;
  if (vc <= 0.f && d1 >= 0.f && d3 <= 0.f) return a + (d1 * np_rcp(d1 - d3)) * ab;
  const f3 cp = p - c;
  const float d5 = dot(ab, cp), d6 = dot(ac, cp);
  if (d6 >= 0.f && d5 <= d6) return c;
  const float vb = d5 * d2 - d1 * d6;
  if (vb <= 0.f && d2 >= 0.f && d6 <= 0.f) return a + (d2 * np_rcp(d2 - d6)) * ac;
  const float va = d3 * d6 - d5 * d4;
  if (va <= 0.f && (d4 - d3) >= 0.f && (d5 - d6) >= 0.f) return b + ((d4 - d3) * np_rcp((d4 - d3) + (d5 - d6))) * (c - b);
  const float den = np_rcp(va + vb + vc);
  return a + (vb * den) * ab + (vc * den) * ac;
}
// closest points of segments p1 + s d1 and p2 + t d2, s, t in [0, 1] (Ericson 5.1.9)
__device__ __forceinline__ void closest_segments(f3 p1, f3 d1, f3 p2, f3 d2, float& s, float& t) {
  const f3 r = p1 - p2;
  const float a = dot(d1, d1), e = dot(d2, d2), f = dot(d2, r), eps = 1e-12f;
  if (a <= eps && e <= eps) { s = t = 0.f; return; }
  if (a <= eps) { s = 0.f; t = fminf(fmaxf(f / e, 0.f), 1.f); return; }
  const float c = dot(d1, r);
  if (e <= eps) { t = 0.f; s = fminf(fmaxf(-c / a, 0.f), 1.f); return; }
  const float b = dot(d1, d2), den = a * e - b * b;
  s = den > eps * a * e ? fminf(fmaxf((b * f - c * e) / den, 0.f), 1.f) : 0.f;
  t = (b * s + f) / e;
  if (t < 0.f) { t = 0.f; s = fminf(fmaxf(-c / a, 0.f), 1.f); }
  else if (t > 1.f) { t = 1.f; s = fminf(fmaxf((b - c) / a, 0.f), 1.f); }
}

// Sphere (centre C, radius r > 0) against the triangles under its footprint [C +- r] (oracle sphere_vs_heightmap), in 2 x 2 cell
// blocks of eight triangles.  EIGHT LANES share one sphere, one triangle of each block each (sub = lane & 7: cell (sub >> 1) & 1,
// sub >> 2 of the block, triangle sub & 1).  When the footprint fits in the 2 x 2 block nearest to the centre (always for radii up to
// half the pitch) that block is the only pass; else the group steps over the blocks from the footprint's first cell on, two cells at
// a time, iy-major, and each lane keeps its closest triangle (a later block's only when strictly closer).  The pass count is the
// warp's largest, so the shuffles below see every lane.  The group then reduces to the closest terrain point with xor shuffles inside
// its aligned 8-lane segment; of several lanes within 1e-6 m of the smallest distance (they share the touched edge or vertex) the
// lowest pair index wins.
// Every lane returns the contact ITS triangle would give (depth, normal, pair) and the lane of its group whose triangle won
// (winner, the same in all eight lanes; -1 = no contact): the lane that owns the sphere fetches the winner's answer with shuffles.
// `valid` = this group holds a sphere at all.
struct SphereTri { int winner; float depth; f3 n; int pair; };
__device__ __forceinline__ SphereTri sphere_vs_heightmap_group(const TerrainDesc& t, int hm_offset, f3 C, float r, bool valid, int lane) {
  const float gx = (C.x - t.x0) * t.inv_dx, gy = (C.y - t.y0) * t.inv_dy;
  const bool in_map = valid && gx >= 0.f && gy >= 0.f && gx < t.xmax && gy < t.ymax;
  const int ccx = (int)gx, ccy = (int)gy;
  int bx = min(max((int)floorf(gx - 0.5f), 0), max(t.xs - 3, 0)), by = min(max((int)floorf(gy - 0.5f), 0), max(t.ys - 3, 0));
  const int fx0 = max((int)floorf(gx - r * t.inv_dx), 0), fx1 = min((int)floorf(gx + r * t.inv_dx), t.xs - 2);
  const int fy0 = max((int)floorf(gy - r * t.inv_dy), 0), fy1 = min((int)floorf(gy + r * t.inv_dy), t.ys - 2);
  int nbx = 1, npass = in_map ? 1 : 0;
  if (in_map && (fx0 < bx || fx1 > bx + 1 || fy0 < by || fy1 > by + 1)) { bx = fx0; by = fy0; nbx = (fx1 - fx0 + 2) >> 1; npass = nbx * ((fy1 - fy0 + 2) >> 1); }
  const int sub = lane & 7, tri = sub & 1;
  float dist = 3.0e38f; f3 v = mk(0.f, 0.f, 0.f), nt = mk(0.f, 0.f, 1.f); int pair = 0x7fffffff; bool beneath_inside = false;
  const int passes = __reduce_max_sync(0xffffffffu, npass);
  int qx = 0, qy = 0;                                           // this pass's block: (bx + 2 qx, by + 2 qy), iy-major
#pragma unroll 1
  for (int p = 0; p < passes; p++) {
    const int ix = bx + 2 * qx + ((sub >> 1) & 1), iy = by + 2 * qy + (sub >> 2);
    if (++qx == nbx) { qx = 0; qy++; }
    if (p < npass && ix <= t.xs - 2 && iy <= t.ys - 2) {
      const float* H = t.h + hm_offset + iy * t.xs + ix;
      const float h00 = __ldg(H), h11 = __ldg(H + t.xs + 1), h3 = __ldg(tri == 0 ? H + 1 : H + t.xs);
      const float X0 = t.x0 + (float)ix * t.dx, X1 = t.x0 + (float)(ix + 1) * t.dx, Y0 = t.y0 + (float)iy * t.dy, Y1 = t.y0 + (float)(iy + 1) * t.dy;
      const f3 a = mk(X0, Y0, h00), p11 = mk(X1, Y1, h11), p3 = tri == 0 ? mk(X1, Y0, h3) : mk(X0, Y1, h3);
      const f3 b = tri == 0 ? p3 : p11, c = tri == 0 ? p11 : p3;      // tri 0 = (P00, P10, P11), tri 1 = (P00, P11, P01)
      const f3 ntp = hm_tri_normal(a, b, c);
      const float side = dot(C - a, ntp);
      if (ix == ccx && iy == ccy) {                             // the triangle directly beneath the centre tells inside from outside
        const float fx = gx - (float)ccx, fy = gy - (float)ccy;
        if ((fx >= fy) == (tri == 0)) beneath_inside = side < 0.f;
      }
      if (!(side - r > 0.f)) {                                  // else: the whole sphere is above this triangle's plane
        const f3 Q = closest_on_triangle(C, a, b, c);
        const f3 vp = C - Q;
        const float d2 = dot(vp, vp);
        const float dp = d2 * np_rsqrt(fmaxf(d2, 1e-30f));
        if (dp < dist) { dist = dp; v = vp; nt = ntp; pair = 2 * (iy * (t.xs - 1) + ix) + tri; }   // the lane keeps its closest triangle
      }
    }
  }
  const unsigned seg = 0xffu << (lane & 24);
  const bool inside = (__ballot_sync(0xffffffffu, beneath_inside) & seg) != 0u;
  float dmin = dist;
  dmin = fminf(dmin, __shfl_xor_sync(0xffffffffu, dmin, 1)); dmin = fminf(dmin, __shfl_xor_sync(0xffffffffu, dmin, 2)); dmin = fminf(dmin, __shfl_xor_sync(0xffffffffu, dmin, 4));
  const int key = (dist < 3.0e38f && dist <= dmin + 1e-6f) ? pair : 0x7fffffff;
  int kmin = key;
  kmin = min(kmin, __shfl_xor_sync(0xffffffffu, kmin, 1)); kmin = min(kmin, __shfl_xor_sync(0xffffffffu, kmin, 2)); kmin = min(kmin, __shfl_xor_sync(0xffffffffu, kmin, 4));
  SphereTri st;
  st.depth = inside ? r + dist : r - dist;
  st.n = (!inside && dist > 1e-9f) ? np_rcp(dist) * v : nt;
  st.pair = pair;
  const unsigned wm = __ballot_sync(0xffffffffu, key == kmin && kmin != 0x7fffffff && st.depth > 0.f) & seg;
  st.winner = wm ? __ffs(wm) - 1 : -1;
  return st;
}

// interior of segment A-B swept by radius r against the terrain edges under its AABB (the end spheres are candidates of their own)
__device__ __noinline__ HmBest segment_vs_heightmap(const TerrainDesc& t, int hm_offset, f3 A, f3 B, float r) {
  HmBest best; best.hit = false; best.depth = 0.f; best.n = mk(0.f, 0.f, 1.f); best.pos = A; best.pair = 0;
  int ix0, ix1, iy0, iy1;
  const f3 M = 0.5f * (A + B);
  if (!hm_cell_range(t, fminf(A.x, B.x) - r, fmaxf(A.x, B.x) + r, fminf(A.y, B.y) - r, fmaxf(A.y, B.y) + r, M.x, M.y, ix0, ix1, iy0, iy1)) return best;
  const float* H = t.h + hm_offset;
  const f3 d1 = B - A;
#pragma unroll 1
  for (int iy = iy0; iy <= iy1; iy++)
#pragma unroll 1
    for (int ix = ix0; ix <= ix1; ix++) {
      const f3 p00 = hm_vertex(t, H, ix, iy), p10 = hm_vertex(t, H, ix + 1, iy), p01 = hm_vertex(t, H, ix, iy + 1), p11 = hm_vertex(t, H, ix + 1, iy + 1);
      const f3 n0 = hm_tri_normal(p00, p10, p11), n1 = hm_tri_normal(p00, p11, p01);
#pragma unroll 1
      for (int k = 0; k < 5; k++) {   // the five edges of the cell: bottom, right (tri 0), diagonal (both), top, left (tri 1)
        const f3 e0 = k == 1 ? p10 : (k == 3 ? p01 : p00);
        const f3 e1 = k == 0 ? p10 : (k == 4 ? p01 : p11);
        float sgm, tt;
        closest_segments(A, d1, e0, e1 - e0, sgm, tt);
        if (!(sgm > 1e-3f) || !(sgm < 1.f - 1e-3f)) continue;   // an end of the segment: the end sphere's business
        const f3 Ps = A + sgm * d1, Pe = e0 + tt * (e1 - e0);
        const f3 v = Ps - Pe;
        const float dist = sqrtf(dot(v, v));
        const int tri = k < 3 ? 0 : 1;
        const f3 nt = tri == 0 ? n0 : n1;
        // a true edge contact: the segment point lies beyond the edge as seen from the triangle(s) of this cell on it (v . m < 0, m = the
        // in-plane direction from the edge into the triangle); over a face or a flat / concave edge the end spheres touch first, so a
        // flat height map gives exactly the contacts of a ground plane (oracle segment_vs_heightmap)
        const f3 ed = e1 - e0;
        const float ee = dot(ed, ed);
        const f3 oa = (k == 0 || k == 4) ? p11 : (k == 2 ? p10 : p00), ob = k == 2 ? p01 : oa;   // third vertex of the cell's triangle(s) on the edge
        const f3 wa = oa - e0, wb = ob - e0;
        const f3 ma = wa - (dot(wa, ed) / ee) * ed, mb = wb - (dot(wb, ed) / ee) * ed;
        if (!(dot(v, ma) < -1e-6f * dist * sqrtf(dot(ma, ma))) || !(dot(v, mb) < -1e-6f * dist * sqrtf(dot(mb, mb)))) continue;
        if (!(dot(v, nt) > 0.f) || !(dist < r) || !(dist > 1e-9f)) continue;   // from above only: a segment under the surface is the end spheres' business
        const f3 n = (1.0f / dist) * v;
        hm_offer(best, r - dist, n, Ps - r * n, 2 * (iy * (t.xs - 1) + ix) + tri);
      }
    }
  return best;
}

// terrain vertices inside the box (centre c, rotation Rb row-major, half extents h): the vertex deepest inside, pushed out through its nearest face
__device__ __noinline__ HmBest box_vs_heightmap(const TerrainDesc& t, int hm_offset, f3 c, const float* Rb, f3 h) {
  HmBest best; best.hit = false; best.depth = 0.f; best.n = mk(0.f, 0.f, 1.f); best.pos = c; best.pair = 0;
  const float ex = fabsf(Rb[0]) * h.x + fabsf(Rb[1]) * h.y + fabsf(Rb[2]) * h.z, ey = fabsf(Rb[3]) * h.x + fabsf(Rb[4]) * h.y + fabsf(Rb[5]) * h.z;
  int ix0, ix1, iy0, iy1;
  if (!hm_cell_range(t, c.x - ex, c.x + ex, c.y - ey, c.y + ey, c.x, c.y, ix0, ix1, iy0, iy1)) return best;
  const float* H = t.h + hm_offset;
#pragma unroll 1
  for (int iy = iy0; iy <= iy1 + 1; iy++)
#pragma unroll 1
    for (int ix = ix0; ix <= ix1 + 1; ix++) {
      const f3 V = hm_vertex(t, H, ix, iy);
      // only a vertex that stands proud of its four neighbours (a peak, a ridge point) can reach a face before the box's own corners do
      const float hn = 0.25f * (__ldg(H + iy * t.xs + max(ix - 1, 0)) + __ldg(H + iy * t.xs + min(ix + 1, t.xs - 1)) + __ldg(H + max(iy - 1, 0) * t.xs + ix) + __ldg(H + min(iy + 1, t.ys - 1) * t.xs + ix));
      if (!(V.z - hn > 1e-6f)) continue;
      const f3 q = mulRt(Rb, V - c);
      const float px = h.x - fabsf(q.x), py = h.y - fabsf(q.y), pz = h.z - fabsf(q.z);
      if (!(px > 0.f) || !(py > 0.f) || !(pz > 0.f)) continue;
      f3 nf; float pen;
      if (px <= py && px <= pz) { pen = px; nf = mk(q.x >= 0.f ? 1.f : -1.f, 0.f, 0.f); }
      else if (py <= pz) { pen = py; nf = mk(0.f, q.y >= 0.f ? 1.f : -1.f, 0.f); }
      else { pen = pz; nf = mk(0.f, 0.f, q.z >= 0.f ? 1.f : -1.f); }
      const f3 n = -1.0f * mulR(Rb, nf);       // contact normal (terrain -> robot) = opposite of the face's outward normal
      const int cix = min(ix, t.xs - 2), ciy = min(iy, t.ys - 2);
      hm_offer(best, pen, n, V, 2 * (ciy * (t.xs - 1) + cix));
    }
  return best;
}
