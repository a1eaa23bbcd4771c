// Self-collision through the raisim:: facade: an ANYmal-like robot floating in zero gravity with its front legs turned inwards until
// the knees and the thighs cross.  With the knee and thigh pairs enabled getContacts() reports both as self contacts; after
// ignoreCollisionBetween(LF_SHANK, RF_SHANK) only the thighs touch.  Runs on the GPU (batch of one).
#include <cstdio>
#include <string>
#include "raisim/World.hpp"

static int countSelf(raisim::ArticulatedSystem* robot, size_t b1, size_t b2) {
  int n = 0;
  for (auto& c : robot->getContacts()) {
    if (!c.isSelfCollision()) continue;
    const size_t other = size_t(c.getPairLocalBodyIndex());
    std::printf("  self contact: body %zu against body %zu, depth %.4f, normal impulse %.4f\n", c.getlocalBodyIndex(), other, c.getDepth(),
                c.getImpulseInContactFrame()[2]);
    if ((c.getlocalBodyIndex() == b1 && other == b2) || (c.getlocalBodyIndex() == b2 && other == b1)) n++;
  }
  return n;
}

int main(int argc, char** argv) {
  std::string urdf = argc > 1 ? argv[1] : "raisimlib_b200/rsc/anymal_c_like.urdf";
  raisim::World world;
  world.setTimeStep(0.0025);
  world.setGravity({0, 0, 0});
  auto* robot = world.addArticulatedSystem(urdf);
  raisim::VecDyn gc(robot->getGeneralizedCoordinateDim()), gv(robot->getDOF());
  const double pose[19] = {0, 0, 1.0, 1, 0, 0, 0, -1.0, 0.4, -0.8, 1.0, 0.4, -0.8, 0.03, -0.4, 0.8, -0.03, -0.4, 0.8};
  for (size_t i = 0; i < 19; i++) gc[i] = pose[i];
  robot->setSelfCollisionPairs({{"LF_SHANK/0", "RF_SHANK/0"}, {"LF_THIGH/0", "RF_THIGH/0"}});
  const size_t lfs = robot->getBodyIdx("LF_SHANK"), rfs = robot->getBodyIdx("RF_SHANK"), lft = robot->getBodyIdx("LF_THIGH"), rft = robot->getBodyIdx("RF_THIGH");
  robot->setState(gc, gv);
  world.integrate();
  const int knees = countSelf(robot, lfs, rfs), thighs = countSelf(robot, lft, rft);
  std::printf("pairs %zu: knee contacts %d, thigh contacts %d\n", robot->getNumberOfSelfCollisionPairs(), knees, thighs);
  robot->ignoreCollisionBetween(rfs, lfs);
  robot->setState(gc, gv);
  world.integrate();
  const int knees2 = countSelf(robot, lfs, rfs), thighs2 = countSelf(robot, lft, rft);
  std::printf("after ignoreCollisionBetween: pairs %zu: knee contacts %d, thigh contacts %d\n", robot->getNumberOfSelfCollisionPairs(), knees2, thighs2);
  return (knees == 1 && thighs == 1 && knees2 == 0 && thighs2 == 1 && robot->getNumberOfSelfCollisionPairs() == 1) ? 0 : 1;
}
