// The LockStep terrain mirror of the raisim:: facade on one batch (needs a GPU): which terrain call each push issues, and which map each
// environment then collides with, read back through a world-aligned height scan and compared with HeightMap::getHeight of that map.
// usage: terrain_mirror_check <urdf>; prints one line per check and exits 0 when all hold
#include <cmath>
#include <cstdio>
#include <string>
#include <vector>

#include "raisim/World.hpp"

using raisim::BatchedWorld;
using raisim::LockStep;

static const int XS = 65, YS = 49;
static const double SX = 12.8, SY = 9.6, CX = 0.1, CY = -0.2;
static bool ok = true;

static void expect(bool c, const std::string& what) { std::printf("%s %s\n", c ? "ok  " : "FAIL", what.c_str()); ok = ok && c; }

static std::vector<float> level(int k) {   // a tilted plane per level: every map differs everywhere
  std::vector<float> h(size_t(XS) * YS);
  for (int y = 0; y < YS; y++) for (int x = 0; x < XS; x++) h[size_t(y) * XS + x] = float(0.1 * k + 0.01 * (k + 1) * x - 0.005 * y);
  return h;
}
static void put(LockStep& ls, int env, int k) { ls.setHeightMap(env, XS, YS, SX, SY, CX, CY, level(k)); }

// every environment's scan against the level it should collide with
static bool collides(LockStep& ls, const std::vector<int>& want) {
  ls.scanValid = false;
  ls.needHeightScan(0, true);
  for (int e = 0; e < ls.n; e++) {
    const std::vector<float> h = level(want[size_t(e)]);
    raisim::HeightMap hm;
    hm.set(XS, YS, SX, SY, CX, CY, std::vector<double>(h.begin(), h.end()));
    for (int p = 0; p < ls.scanPoints; p++) {
      const size_t i = size_t(e) * ls.scanPoints + p;
      if (!(std::fabs(ls.scan.v[i] - hm.getHeight(ls.scanXy.v[2 * i], ls.scanXy.v[2 * i + 1])) <= 1e-4)) return false;
    }
  }
  return true;
}

int main(int argc, char** argv) {
  if (argc < 2) { std::fprintf(stderr, "usage: terrain_mirror_check <urdf>\n"); return 2; }
  const int n = 4;
  BatchedWorld bw(argv[1], n);
  bw.enableLockStep();
  LockStep& ls = *bw.lockStep();
  bw.setHeightScan({0, 0, 0}, {0.3f, 0.2f, -1.1f, 0.7f, 2.5f, -1.9f}, false);
  for (int e = 0; e < n; e++) ls.stateRow(e, ls.gc)[0] = float(0.5 * e);   // base x: the environments sample different places

  // environments without terrain of their own share the lowest-numbered environment's map: one common map is one plain upload
  put(ls, 1, 0); put(ls, 3, 0);
  ls.pushWrites();
  expect(ls.mapUploads == 1 && ls.atlasSingle && collides(ls, {0, 0, 0, 0}), "one common map added by some environments: one single-map upload, shared by all");
  // distinct maps: an atlas; environment 2 (no map) takes environment 0's
  put(ls, 0, 1); put(ls, 3, 2);
  ls.pushWrites();
  expect(ls.mapUploads == 2 && !ls.atlasSingle && collides(ls, {1, 0, 1, 2}), "distinct maps: one atlas upload, a map-less environment shares environment 0's");
  // a curriculum: levels 0..2 in use, then everyone on level 0 (index only), then a new level 3 appears while 1 and 2 are unused:
  // the rebuilt atlas keeps them, so moving back to level 1 uploads no map
  put(ls, 0, 0); put(ls, 1, 1); put(ls, 2, 2); put(ls, 3, 0);
  ls.pushWrites();
  const long m0 = ls.mapUploads;
  for (int e = 0; e < n; e++) put(ls, e, 0);
  ls.pushWrites();
  expect(ls.mapUploads == m0 && collides(ls, {0, 0, 0, 0}), "every environment back on level 0: index move only");
  put(ls, 0, 3);
  ls.pushWrites();
  expect(ls.mapUploads == m0 + 1 && ls.atlas.size() == 4 && collides(ls, {3, 0, 0, 0}), "a new level: one upload that keeps the unused levels 1 and 2");
  const long i0 = ls.indexUploads;
  put(ls, 1, 1); put(ls, 2, 2);
  ls.pushWrites();
  expect(ls.mapUploads == m0 + 1 && ls.indexUploads == i0 + 1 && collides(ls, {3, 1, 2, 0}), "back to the kept levels: one index move, no upload");
  // a ground in one environment and a map in another cannot share a batch
  ls.setGround(2);
  bool threw = false;
  try { ls.pushWrites(); } catch (const std::runtime_error& e) { threw = std::string(e.what()).find("same kind of terrain") != std::string::npos; }
  expect(threw, "ground in one environment, height maps in others: refused");
  std::printf(ok ? "ok\n" : "FAILED\n");
  return ok ? 0 : 1;
}
