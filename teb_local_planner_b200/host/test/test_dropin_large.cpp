/*
 * test_dropin_large.cpp — the drop-in classes on a scene the way a local costmap without a costmap converter produces
 * it: 3000 PointObstacles on a 5 cm grid (walls of cells on both sides of the corridor).
 *   TebOptimalPlanner::plan(start, goal) from a cold start; prints LARGE_OK and the band as "KEY v0 v1 ..." lines that
 *   tests/test_host_dropin_large.py compares with tebgpu_optimize_batch on the same inputs.
 *   HomotopyClassPlanner::plan on the same container: false (its H-signature stops at 1024 obstacles).
 */
#include <cstdio>

#include "teb_local_planner/homotopy_class_planner.h"
#include "teb_local_planner/optimal_planner.h"

using namespace teb_local_planner;

/* cell k: column k % 160 (x = -4 .. 3.95), row k / 160 alternating above and below the band, |y| = 1.0 .. 1.9 */
static void costmap_points(ObstContainer& obst, int count) {
  for (int k = 0; k < count; ++k) {
    const int col = k % 160, row = k / 160;
    const double y = (row % 2 ? -1.0 : 1.0) * (1.0 + 0.05 * (row / 2));
    obst.push_back(ObstaclePtr(new PointObstacle(-4.0 + 0.05 * col, y)));
  }
}

int main() {
  TebConfig cfg;
  ObstContainer obst;
  costmap_points(obst, 3000);
  ViaPointContainer via;
  TebOptimalPlanner planner(cfg, &obst, TebVisualizationPtr(), &via);
  const bool ok = planner.plan(PoseSE2(-4, 0, 0), PoseSE2(4, 0, 0));
  std::printf("LARGE_OK %d\nLARGE_STATUS %d\n", ok ? 1 : 0, planner.lastStatus());
  std::printf("LARGE_N %d\n", planner.teb().sizePoses());
  for (int i = 0; i < planner.teb().sizePoses(); ++i)
    std::printf("LARGE_POSE %d %.17g %.17g %.17g %.17g\n", i, planner.teb().Pose(i).x(), planner.teb().Pose(i).y(),
                planner.teb().Pose(i).theta(), i < planner.teb().sizeTimeDiffs() ? planner.teb().TimeDiff(i) : 0.0);
  HomotopyClassPlanner hcp(cfg, &obst, TebVisualizationPtr(), &via);
  const bool hok = hcp.plan(PoseSE2(-4, 0, 0), PoseSE2(4, 0, 0), NULL);
  std::printf("LARGE_HCP_OK %d\n", hok ? 1 : 0);
  std::printf("RESULT DONE\n");
  return 0;
}
