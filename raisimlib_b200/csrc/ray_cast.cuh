// Ray casts against the terrain and the robot's own collision bodies (rsb_batch_set_rays / rsb_batch_get_ray_casts): a body-mounted
// depth camera or lidar for every environment, in one launch that reads the state and writes only its outputs.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/rsb.h"

namespace rsb {

constexpr int RAY_MAX_SHAPES = 64;   // collision bodies of a model: at most one per contact candidate
constexpr int RAY_SHAPE_WORDS = 20;  // per collision body (RayTable::shape)

// The rays of rsb_batch_set_rays and the model's collision bodies, in one device allocation:
//   body [RSB_MAX_RAYS] | origin [RSB_MAX_RAYS][3] | unit direction [RSB_MAX_RAYS][3] | shapes [ncoll][RAY_SHAPE_WORDS]
// shape words: 0 body (int bits), 1 CollType (int bits), 2-4 size (sphere r; box half extents; capsule / cylinder r and half length
// along the local z axis), 5-7 position and 8-16 rotation (row-major) in the body frame, 17 radius of a sphere about the position that
// holds the whole shape.
struct RayTable {
  int n, targets;          // rays, RSB_RAYS_TERRAIN / RSB_RAYS_TERRAIN_AND_ROBOT
  int root_from_gc;        // RSB_RAYS_TERRAIN on a floating base: rays on body 0 take its pose from gc
  int ncoll;
  float max_distance;
  const int* body;
  const float* origin;
  const float* dir;
  const float* shape;
};

// A collision body in the world frame, as a CTA keeps it in shared memory: centre, rotation (columns = the shape's local axes), size
// and the radius of a sphere about the centre that holds the whole shape.
struct RayShape {
  float c[3], R[9], s[3], bound;
  int type;
};

// ---- one ray against one convex shape in its local frame: the entry t > 0 (0 when there is none).  The origin is outside the shape
// (the caller has skipped shapes that contain it).  Quadratics use the distance of closest approach (the discriminant r^2 - |q|^2 of the
// perpendicular q), which keeps its precision when the shape is small and far away.

// sphere of radius r about the origin: entry along the unit ray o + t d
__device__ __forceinline__ float ray_sphere(float ox, float oy, float oz, float dx, float dy, float dz, float r) {
  const float tc = -(ox * dx + oy * dy + oz * dz);
  const float qx = ox + tc * dx, qy = oy + tc * dy, qz = oz + tc * dz;
  const float disc = r * r - (qx * qx + qy * qy + qz * qz);
  if (disc < 0.f) return 0.f;
  const float t = tc - sqrtf(disc);
  return t > 0.f ? t : 0.f;
}

// the side of the infinite cylinder of radius r about the local z axis, where |z| <= hl: the entry through it
__device__ __forceinline__ float ray_cyl_side(float ox, float oy, float oz, float dx, float dy, float dz, float r, float hl) {
  const float a = dx * dx + dy * dy;
  if (!(a > 0.f)) return 0.f;
  const float tc = -(ox * dx + oy * dy) / a;
  const float qx = ox + tc * dx, qy = oy + tc * dy;
  const float disc = r * r - (qx * qx + qy * qy);
  if (disc < 0.f) return 0.f;
  const float t = tc - sqrtf(disc / a);
  if (!(t > 0.f) || fabsf(oz + t * dz) > hl) return 0.f;
  return t;
}

__device__ __forceinline__ float min_hit(float a, float b) { return a > 0.f && (b == 0.f || a < b) ? a : b; }

// entry t of the unit ray (world o, d) into shape S, 0 when it does not enter it or starts inside or on it
__device__ float ray_shape(const RayShape& S, float ox, float oy, float oz, float dx, float dy, float dz) {
  const float wx = ox - S.c[0], wy = oy - S.c[1], wz = oz - S.c[2];
  // bounding sphere: the ray must pass within S.bound of the centre, ahead of the origin
  {
    const float tc = -(wx * dx + wy * dy + wz * dz);
    const float qx = wx + tc * dx, qy = wy + tc * dy, qz = wz + tc * dz;
    const float w2 = wx * wx + wy * wy + wz * wz, b2 = S.bound * S.bound;
    if (qx * qx + qy * qy + qz * qz > b2 || (tc < 0.f && w2 > b2)) return 0.f;
  }
  // the local frame: o_l = R^T (o - c), d_l = R^T d
  const float lx = S.R[0] * wx + S.R[3] * wy + S.R[6] * wz, ly = S.R[1] * wx + S.R[4] * wy + S.R[7] * wz, lz = S.R[2] * wx + S.R[5] * wy + S.R[8] * wz;
  const float ex = S.R[0] * dx + S.R[3] * dy + S.R[6] * dz, ey = S.R[1] * dx + S.R[4] * dy + S.R[7] * dz, ez = S.R[2] * dx + S.R[5] * dy + S.R[8] * dz;
  const float r = S.s[0];
  if (S.type == 0) {   // CT_SPHERE
    if (lx * lx + ly * ly + lz * lz <= r * r) return 0.f;
    return ray_sphere(lx, ly, lz, ex, ey, ez, r);
  }
  if (S.type == 1) {   // CT_BOX (a mesh's bounding box too): slabs
    const float h[3] = {S.s[0], S.s[1], S.s[2]}, o[3] = {lx, ly, lz}, d[3] = {ex, ey, ez};
    if (fabsf(lx) <= h[0] && fabsf(ly) <= h[1] && fabsf(lz) <= h[2]) return 0.f;
    float tn = 0.f, tf = 3.0e38f;
#pragma unroll
    for (int k = 0; k < 3; k++) {
      if (d[k] == 0.f) {
        if (fabsf(o[k]) > h[k]) return 0.f;
        continue;
      }
      const float inv = 1.f / d[k];
      float t0 = (-h[k] - o[k]) * inv, t1 = (h[k] - o[k]) * inv;
      if (t0 > t1) { const float s = t0; t0 = t1; t1 = s; }
      tn = fmaxf(tn, t0); tf = fminf(tf, t1);
    }
    return tn <= tf && tn > 0.f ? tn : 0.f;
  }
  const float hl = S.s[1];
  if (S.type == 2) {   // CT_CAPSULE: the side and the two end spheres
    const float zc = fminf(fmaxf(lz, -hl), hl);
    if (lx * lx + ly * ly + (lz - zc) * (lz - zc) <= r * r) return 0.f;
    float t = ray_cyl_side(lx, ly, lz, ex, ey, ez, r, hl);
    t = min_hit(ray_sphere(lx, ly, lz - hl, ex, ey, ez, r), t);
    return min_hit(ray_sphere(lx, ly, lz + hl, ex, ey, ez, r), t);
  }
  // CT_CYLINDER: the side and the two cap discs
  if (lx * lx + ly * ly <= r * r && fabsf(lz) <= hl) return 0.f;
  float t = ray_cyl_side(lx, ly, lz, ex, ey, ez, r, hl);
  if (ez != 0.f) {
    const float zp = lz > hl ? hl : lz < -hl ? -hl : 0.f;   // the cap facing the origin (none when it lies between the caps)
    if (zp != 0.f && (zp - lz) * ez > 0.f) {
      const float tp = (zp - lz) / ez, px = lx + tp * ex, py = ly + tp * ey;
      if (px * px + py * py <= r * r) t = min_hit(tp, t);
    }
  }
  return t;
}

// ---- the height map: the first crossing from the upper side of the surface to its lower side along o + t d, t in (t_lo, t_hi].
// Grid coordinates g = (p - x0) / pitch; the ray's xy projection is walked cell by cell (Amanatides-Woo).  In a cell the ray's height
// above the surface f(t) = z(t) - h(t) is linear on each side of the P00-P11 diagonal: it is evaluated at the entry, at the crossing
// of the diagonal and at the exit, and the first change of sign from + to - is solved as a linear root.  The value at the exit is
// carried into the next cell as its entry value, never recomputed there, so a ray that crosses the surface exactly on a cell boundary,
// a vertex or a diagonal cannot slip through between two evaluations.  Returns the hit t, or 0.
__device__ float ray_heightmap(const TerrainDesc& T, const float* __restrict__ H, float ox, float oy, float oz, float dx, float dy, float dz,
                               float t_hi) {
  const float gox = (ox - T.x0) / T.dx, goy = (oy - T.y0) / T.dy;
  const float gdx = dx / T.dx, gdy = dy / T.dy;
  float t_lo = 0.f;
  // clip: the map's rectangle and z <= hmax (above every sample the ray is above the surface)
  if (gdx != 0.f) {
    float a = -gox / gdx, b = (T.xmax - gox) / gdx;
    if (a > b) { const float s = a; a = b; b = s; }
    t_lo = fmaxf(t_lo, a); t_hi = fminf(t_hi, b);
  } else if (!(gox >= 0.f && gox <= T.xmax)) return 0.f;
  if (gdy != 0.f) {
    float a = -goy / gdy, b = (T.ymax - goy) / gdy;
    if (a > b) { const float s = a; a = b; b = s; }
    t_lo = fmaxf(t_lo, a); t_hi = fminf(t_hi, b);
  } else if (!(goy >= 0.f && goy <= T.ymax)) return 0.f;
  const float zmax = T.hmax + 1e-4f * (1.f + fabsf(T.hmax));   // a little above the highest sample: the ray is above the surface there
  if (dz >= 0.f) {
    if (oz > zmax) return 0.f;
    if (dz > 0.f) t_hi = fminf(t_hi, (zmax - oz) / dz);
  } else {
    t_lo = fmaxf(t_lo, (zmax - oz) / dz);
  }
  if (!(t_lo <= t_hi)) return 0.f;
  // the first cell: the one under the point at t_lo (on a boundary either neighbour will do: the walk then leaves it at once)
  int ix = min(max((int)floorf(gox + t_lo * gdx), 0), T.xs - 2), iy = min(max((int)floorf(goy + t_lo * gdy), 0), T.ys - 2);
  const int sx = gdx > 0.f ? 1 : -1, sy = gdy > 0.f ? 1 : -1;
  const float idx = gdx != 0.f ? 1.f / gdx : 0.f, idy = gdy != 0.f ? 1.f / gdy : 0.f;
  const float* P = H + iy * T.xs + ix;
  float h00 = __ldg(P), h10 = __ldg(P + 1), h01 = __ldg(P + T.xs), h11 = __ldg(P + T.xs + 1);
  // the ray's height above the surface of cell (ix, iy) at t, on the triangle picked by tri (0: fx >= fy)
  auto above = [&](float t, int tri) {
    const float fx = gox + t * gdx - (float)ix, fy = goy + t * gdy - (float)iy;
    const float h = tri == 0 ? h00 + (h10 - h00) * fx + (h11 - h10) * fy : h00 + (h11 - h01) * fx + (h01 - h00) * fy;
    return oz + t * dz - h;
  };
  float ta = t_lo;
  const float g0 = (gox + ta * gdx - (float)ix) - (goy + ta * gdy - (float)iy);
  float fa = above(ta, g0 >= 0.f ? 0 : 1);
  // at the origin itself, lying on the surface is not being above it; at the edge of the map it is
  bool up = ta > 0.f ? fa >= 0.f : fa > 0.f;
  const float gg = gdx - gdy;   // d(fx - fy)/dt
  for (;;) {
    // exit of this cell: the next boundary in x or y, or the end of the range
    const float tx = gdx != 0.f ? ((float)(ix + (sx > 0)) - gox) * idx : 3.0e38f;
    const float ty = gdy != 0.f ? ((float)(iy + (sy > 0)) - goy) * idy : 3.0e38f;
    const float tb = fminf(fminf(tx, ty), t_hi);
    // the diagonal fx = fy inside (ta, tb)
    const float da = (gox + ta * gdx - (float)ix) - (goy + ta * gdy - (float)iy);
    float tm = tb;
    if (gg != 0.f) {
      const float t = ta - da / gg;
      if (t > ta && t < tb) tm = t;
    }
    int tri = (da + 0.5f * (tm - ta) * gg) >= 0.f ? 0 : 1;   // the triangle of (ta, tm)
    float fm = above(tm, tri);
    if (up && fm < 0.f) return ta + (tm - ta) * (fa / (fa - fm));
    up = fm >= 0.f;
    if (tm < tb) {
      const float fb = above(tb, 1 - tri);
      if (up && fb < 0.f) return tm + (tb - tm) * (fm / (fm - fb));
      up = fb >= 0.f;
      fm = fb;
    }
    if (tb >= t_hi) return 0.f;
    // step into the next cell, reusing the edge it shares with this one
    ta = tb; fa = fm;
    if (tx <= ty) {
      ix += sx;
      if (ix < 0 || ix > T.xs - 2) return 0.f;
      if (sx > 0) { h00 = h10; h01 = h11; P += 1; h10 = __ldg(P + 1); h11 = __ldg(P + T.xs + 1); }
      else { h10 = h00; h11 = h01; P -= 1; h00 = __ldg(P); h01 = __ldg(P + T.xs); }
    } else {
      iy += sy;
      if (iy < 0 || iy > T.ys - 2) return 0.f;
      if (sy > 0) { h00 = h01; h10 = h11; P += T.xs; h01 = __ldg(P + T.xs); h11 = __ldg(P + T.xs + 1); }
      else { h01 = h00; h11 = h10; P -= T.xs; h00 = __ldg(P); h10 = __ldg(P + 1); }
    }
  }
}

// One thread per (environment, ray), the ray index fastest: a warp is 32 consecutive rays of one environment (neighbouring pixels of a
// camera), so their traversals stay together and their stores coalesce.  grid.x = environments (there may be more than 65535),
// grid.y = blocks of 256 rays.  With RSB_RAYS_TERRAIN_AND_ROBOT the CTA first puts its environment's collision bodies in the world
// frame into shared memory.  R [N][nb][9], P [N][nb][3]: the kinematics pass's poses.  Outputs are tight rows of the environments
// [env_begin, env_begin + gridDim.x); a null output is skipped.
__global__ void __launch_bounds__(256) rsb_ray_cast_kernel(RayTable rt, TerrainDesc ter, const float* __restrict__ gc, int gc_stride,
                                                           const float* __restrict__ R, const float* __restrict__ P, int nb, int env_begin,
                                                           float* __restrict__ dist_out, int* __restrict__ hit_out) {
  __shared__ RayShape sh[RAY_MAX_SHAPES];
  const long e = env_begin + (long)blockIdx.x;
  const bool robot = rt.targets == RSB_RAYS_TERRAIN_AND_ROBOT;
  if (robot) {
    for (int c = threadIdx.x; c < rt.ncoll; c += blockDim.x) {
      const float* w = rt.shape + c * RAY_SHAPE_WORDS;
      const int b = __float_as_int(w[0]);
      const float* Rb = R + (e * nb + b) * 9;
      const float* pb = P + (e * nb + b) * 3;
      RayShape& S = sh[c];
      S.type = __float_as_int(w[1]);
      S.s[0] = w[2]; S.s[1] = w[3]; S.s[2] = w[4];
#pragma unroll
      for (int i = 0; i < 3; i++) {
        S.c[i] = pb[i] + Rb[3 * i] * w[5] + Rb[3 * i + 1] * w[6] + Rb[3 * i + 2] * w[7];
#pragma unroll
        for (int j = 0; j < 3; j++) S.R[3 * i + j] = Rb[3 * i] * w[8 + j] + Rb[3 * i + 1] * w[11 + j] + Rb[3 * i + 2] * w[14 + j];
      }
      S.bound = w[17];
    }
    __syncthreads();
  }
  const int i = blockIdx.y * blockDim.x + threadIdx.x;
  if (i >= rt.n) return;
  const long w = (e - env_begin) * rt.n + i;   // output row
  const int b = __ldg(rt.body + i);
  float R00, R01, R02, R10, R11, R12, R20, R21, R22, px, py, pz;
  if (b == 0 && rt.root_from_gc) {
    const float* q = gc + e * gc_stride;
    px = q[0]; py = q[1]; pz = q[2];
    float qw = q[3], qx = q[4], qy = q[5], qz = q[6];
    const float inv = 1.0f / sqrtf(qw * qw + qx * qx + qy * qy + qz * qz);   // as write_obs_row normalises it
    qw *= inv; qx *= inv; qy *= inv; qz *= inv;
    obs_rot_column(qw, qx, qy, qz, 0, R00, R10, R20);
    obs_rot_column(qw, qx, qy, qz, 1, R01, R11, R21);
    obs_rot_column(qw, qx, qy, qz, 2, R02, R12, R22);
  } else {
    const float* Rb = R + (e * nb + b) * 9;
    const float* pb = P + (e * nb + b) * 3;
    R00 = Rb[0]; R01 = Rb[1]; R02 = Rb[2]; R10 = Rb[3]; R11 = Rb[4]; R12 = Rb[5]; R20 = Rb[6]; R21 = Rb[7]; R22 = Rb[8];
    px = pb[0]; py = pb[1]; pz = pb[2];
  }
  const float lx = __ldg(rt.origin + 3 * i), ly = __ldg(rt.origin + 3 * i + 1), lz = __ldg(rt.origin + 3 * i + 2);
  const float ux = __ldg(rt.dir + 3 * i), uy = __ldg(rt.dir + 3 * i + 1), uz = __ldg(rt.dir + 3 * i + 2);
  const float ox = px + R00 * lx + R01 * ly + R02 * lz, oy = py + R10 * lx + R11 * ly + R12 * lz, oz = pz + R20 * lx + R21 * ly + R22 * lz;
  const float dx = R00 * ux + R01 * uy + R02 * uz, dy = R10 * ux + R11 * uy + R12 * uz, dz = R20 * ux + R21 * uy + R22 * uz;
  float best = rt.max_distance;
  int id = RSB_RAY_MISS;
  if (!(isfinite(ox) && isfinite(oy) && isfinite(oz) && isfinite(dx) && isfinite(dy) && isfinite(dz))) {
    best = __int_as_float(0x7fffffff);
  } else {
    if (robot)   // the robot first: its hit shortens the terrain walk
      for (int c = 0; c < rt.ncoll; c++) {
        const float t = ray_shape(sh[c], ox, oy, oz, dx, dy, dz);
        if (t > 0.f && t <= best && (id == RSB_RAY_MISS || t < best)) { best = t; id = c; }
      }
    if (ter.type == 1) {
      if (dz < 0.f && oz > ter.ground_z) {
        const float t = (ter.ground_z - oz) / dz;
        if (t > 0.f && t <= best && (id == RSB_RAY_MISS || t < best)) { best = t; id = RSB_RAY_TERRAIN; }
      }
    } else if (ter.type == 2) {
      const int hm_offset = ter.env_map ? __ldg(ter.env_map + e) * ter.map_words : 0;   // terrain atlas
      const float t = ray_heightmap(ter, ter.h + hm_offset, ox, oy, oz, dx, dy, dz, best);
      if (t > 0.f && t <= best && (id == RSB_RAY_MISS || t < best)) { best = t; id = RSB_RAY_TERRAIN; }
    }
    if (id == RSB_RAY_MISS) best = __int_as_float(0x7f800000);   // +inf
  }
  if (dist_out) dist_out[w] = best;
  if (hit_out) hit_out[w] = id;
}

}  // namespace rsb
