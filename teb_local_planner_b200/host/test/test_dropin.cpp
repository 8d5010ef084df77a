/*
 * test_dropin.cpp — exercises the drop-in C++ classes the way the reference's own callers do.
 *   (no argument)  CPU-only checks: the three gtests of the reference (test/teb_basics.cpp:5-68) restated against this
 *                  TimedElasticBand, cold-start initialisation, config defaults.
 *   gpu            the test_optim_node scene (src/test_optim_node.cpp:106-117, :168) through TebOptimalPlanner::plan()
 *                  and three seeded candidates through HomotopyClassPlanner::plan(); prints the results as
 *                  "KEY v0 v1 ..." lines that tests/test_host_dropin.py compares with the CPU oracle.
 */
#include <cmath>
#include <cstdio>
#include <cuda_runtime_api.h>
#include <cstring>
#include <string>

#include "teb_local_planner/homotopy_class_planner.h"
#include "teb_local_planner/optimal_planner.h"

using namespace teb_local_planner;

static int g_fail = 0;
#define CHECK(cond)                                                          \
  do {                                                                       \
    if (!(cond)) { std::printf("CHECK FAILED %s:%d %s\n", __FILE__, __LINE__, #cond); ++g_fail; } \
  } while (0)

static void check_dts(const TimedElasticBand& teb, double dt, double hyst) {
  for (int i = 0; i < teb.sizeTimeDiffs(); ++i) {
    CHECK(teb.TimeDiff(i) <= dt + hyst + 1e-3);
    CHECK(dt - hyst - 1e-3 <= teb.TimeDiff(i));
  }
}

/* TEST(TEBBasic, autoResizeLargeValueAtEnd) test/teb_basics.cpp:5 */
static void autoResizeLargeValueAtEnd() {
  double dt = 0.1, dt_hysteresis = dt / 3.;
  TimedElasticBand teb;
  teb.addPose(PoseSE2(0., 0., 0.));
  for (int i = 1; i < 10; ++i) teb.addPoseAndTimeDiff(PoseSE2(i * 1., 0., 0.), dt);
  teb.addPoseAndTimeDiff(PoseSE2(10., 0., 0.), dt + 2 * dt_hysteresis);
  teb.autoResize(dt, dt_hysteresis, 3, 100, false);
  check_dts(teb, dt, dt_hysteresis);
}
/* TEST(TEBBasic, autoResizeSmallValueAtEnd) test/teb_basics.cpp:27 */
static void autoResizeSmallValueAtEnd() {
  double dt = 0.1, dt_hysteresis = dt / 3.;
  TimedElasticBand teb;
  teb.addPose(PoseSE2(0., 0., 0.));
  for (int i = 1; i < 10; ++i) teb.addPoseAndTimeDiff(PoseSE2(i * 1., 0., 0.), dt);
  teb.addPoseAndTimeDiff(PoseSE2(10., 0., 0.), dt - 2 * dt_hysteresis);
  teb.autoResize(dt, dt_hysteresis, 3, 100, false);
  check_dts(teb, dt, dt_hysteresis);
}
/* TEST(TEBBasic, autoResize) test/teb_basics.cpp:49 */
static void autoResizeMiddle() {
  double dt = 0.1, dt_hysteresis = dt / 3.;
  TimedElasticBand teb;
  teb.addPose(PoseSE2(0., 0., 0.));
  for (int i = 1; i < 10; ++i) teb.addPoseAndTimeDiff(PoseSE2(i * 1., 0., 0.), dt);
  teb.TimeDiff(5) = dt + 2 * dt_hysteresis;
  teb.addPoseAndTimeDiff(PoseSE2(10., 0., 0.), dt - 2 * dt_hysteresis);
  teb.autoResize(dt, dt_hysteresis, 3, 100, false);
  check_dts(teb, dt, dt_hysteresis);
}

static void cpu_checks() {
  autoResizeLargeValueAtEnd();
  autoResizeSmallValueAtEnd();
  autoResizeMiddle();
  /* cold start of plan(start, goal): start, one forced mid sample, goal (timed_elastic_band.cpp:325-387) */
  TimedElasticBand teb;
  CHECK(teb.initTrajectoryToGoal(PoseSE2(-4, 0, 0), PoseSE2(4, 0, 0), 0, 0.4, 3, false));
  CHECK(teb.sizePoses() == 3 && teb.sizeTimeDiffs() == 2);
  CHECK(std::fabs(teb.Pose(1).x()) < 1e-15 && std::fabs(teb.TimeDiff(0) - 10.0) < 1e-12);
  CHECK(!teb.initTrajectoryToGoal(PoseSE2(-4, 0, 0), PoseSE2(4, 0, 0)));  /* already initialised */
  /* warm start pruning (timed_elastic_band.cpp:555-597) */
  TimedElasticBand w;
  w.addPose(0, 0, 0);
  for (int i = 1; i <= 12; ++i) w.addPoseAndTimeDiff(0.1 * i, 0, 0, 0.25);
  PoseSE2 ns(0.21, 0, 0), ng(1.3, 0, 0);
  w.updateAndPruneTEB(ns, ng, 3);
  CHECK(w.sizePoses() == 11 && std::fabs(w.Pose(0).x() - 0.21) < 1e-15 && std::fabs(w.BackPose().x() - 1.3) < 1e-15);
  CHECK(std::fabs(w.Pose(1).x() - 0.3) < 1e-12);
  /* config defaults == C-ABI defaults */
  TebConfig cfg;
  TebParams a = cfg.toParams(), b;
  tebgpu_default_params(&b);
  CHECK(std::memcmp(&a, &b, sizeof(TebParams)) == 0);
  PointObstacle po(1, 2);
  CHECK(!po.isDynamic());
  po.setCentroidVelocity(Eigen::Vector2d(0.1, 0));
  CHECK(po.isDynamic() && po.toRow().dynamic == 1);
  TwoCirclesRobotFootprint fp(0.3, 0.2, 0.2, 0.25);
  CircularObstacle co(2, 0, 0.5);
  CHECK(std::fabs(fp.calculateDistance(PoseSE2(0, 0, 0), &co) - (2 - 0.3 - 0.5 - 0.2)) < 1e-12);
  /* Line / Pill / Polygon obstacles and Line / Polygon footprints: host-side queries (obstacles.h:597-1045,
   * robot_footprint_model.h:439-775) */
  LineObstacle lo(1, -1, 1, 1);
  CHECK(lo.getMinimumDistance(Eigen::Vector2d(0, 0)) == 1.0 && lo.getCentroid().x() == 1.0 && lo.getCentroid().y() == 0.0);
  CHECK(lo.toRow().type == TEB_OBST_LINE);
  PillObstacle pill(1, -1, 1, 1, 0.2);
  CHECK(std::fabs(pill.getMinimumDistance(Eigen::Vector2d(0, 0)) - 0.8) < 1e-15 && pill.toRow().type == TEB_OBST_PILL);
  PolygonObstacle sq;
  sq.pushBackVertex(1, -1); sq.pushBackVertex(3, -1); sq.pushBackVertex(3, 1); sq.pushBackVertex(1, 1); sq.pushBackVertex(1, -1);
  sq.finalizePolygon();
  CHECK(sq.noVertices() == 4 && std::fabs(sq.getCentroid().x() - 2.0) < 1e-15 && std::fabs(sq.getCentroid().y()) < 1e-15);
  CHECK(sq.getMinimumDistance(Eigen::Vector2d(0, 0)) == 1.0 && sq.checkCollision(Eigen::Vector2d(2, 0), 0.0));
  sq.setCentroidVelocity(Eigen::Vector2d(1, 0));
  CHECK(sq.getMinimumSpatioTemporalDistance(Eigen::Vector2d(0, 0), 2.0) == 3.0);
  LineRobotFootprint lf(Eigen::Vector2d(-0.5, 0), Eigen::Vector2d(0.5, 0));
  CHECK(std::fabs(lf.calculateDistance(PoseSE2(0, 0, M_PI / 2), &lo) - 1.0) < 1e-15);
  LineObstacle cross(-1, 0.1, 1, 0.1);
  CHECK(lf.calculateDistance(PoseSE2(0, 0, M_PI / 2), &cross) == 0.0);
  Point2dContainer unit = {Eigen::Vector2d(-0.5, -0.5), Eigen::Vector2d(0.5, -0.5), Eigen::Vector2d(0.5, 0.5), Eigen::Vector2d(-0.5, 0.5)};
  PolygonRobotFootprint pf(unit);
  PointObstacle far(2, 0);
  CHECK(std::fabs(pf.calculateDistance(PoseSE2(0, 0, M_PI / 4), &far) - (2 - std::sqrt(0.5))) < 1e-15);
  CHECK(std::fabs(pf.getInscribedRadius() - 0.5) < 1e-15);
  std::vector<double> pool;
  TebObstacle row = sq.toRow();
  sq.appendVertices(pool, row);
  CHECK(row.type == TEB_OBST_POLYGON && row.vertex_begin == 0 && row.vertex_count == 4 && pool.size() == 8 && row.dynamic == 1);
  TebParams fpp;
  tebgpu_default_params(&fpp);
  pf.fillParams(fpp);
  CHECK(fpp.footprint_type == TEB_FOOTPRINT_POLYGON && fpp.footprint_vertex_count == 4 && fpp.footprint_vertices[2] == 0.5);
}

/* costmap stand-in: a wall x in [lo, hi] is lethal */
struct WallModel : public base_local_planner::CostmapModel {
  double lo, hi;
  int queries = 0;
  WallModel(double l, double h) : lo(l), hi(h) {}
  double footprintCost(double x, double, double, const std::vector<geometry_msgs::Point>&, double, double) override {
    ++queries;
    return (x >= lo && x <= hi) ? -1.0 : 1.0;
  }
};

static void postprocessing_checks() {
  /* getFullTrajectory / isTrajectoryFeasible (optimal_planner.cpp:1197-1306) on a hand-made band */
  TebConfig cfg;
  TebOptimalPlanner pl(cfg);
  for (int i = 0; i < 5; ++i) {
    if (i == 0) pl.teb().addPose(0, 0, 0);
    else pl.teb().addPoseAndTimeDiff(0.5 * i, 0, 0, 1.0 + 0.5 * (i - 1)); /* dt = 1, 1.5, 2, 2.5 */
  }
  std::vector<TrajectoryPointMsg> traj;
  pl.getFullTrajectory(traj);
  CHECK(traj.size() == 5 && traj[0].time_from_start == 0 && std::fabs(traj[4].time_from_start - 7.0) < 1e-15);
  CHECK(std::fabs(traj[1].velocity.linear.x - 0.5 * (0.5 / 1.0 + 0.5 / 1.5)) < 1e-15 && traj[4].velocity.linear.x == 0);
  std::vector<geometry_msgs::Point> fp;
  WallModel open_space(10, 11), wall(1.1, 1.2), far_wall(1.9, 2.1);
  CHECK(pl.isTrajectoryFeasible(&open_space, fp, 0.6, 0.8, -1));
  CHECK(open_space.queries == 5);                       /* poses 0.5 m apart, inscribed radius 0.6: no extra samples */
  /* the wall lies between the poses at x = 1.0 and 1.5: only the two interpolated samples (inscribed radius 0.2:
   * x = 1.167, 1.333) can see it */
  CHECK(pl.isTrajectoryFeasible(&wall, fp, 0.6, 0.8, -1));
  CHECK(!pl.isTrajectoryFeasible(&wall, fp, 0.2, 0.8, -1));
  CHECK(!pl.isTrajectoryFeasible(&far_wall, fp, 0.6, 0.8, -1));
  CHECK(pl.isTrajectoryFeasible(&far_wall, fp, 0.6, 0.8, 2));            /* look-ahead index stops before the wall */
  CHECK(pl.isTrajectoryFeasible(&far_wall, fp, 0.6, 0.8, -1, 1.2));     /* look-ahead distance: poses up to x = 1.0 */
}

static void print_band(const char* key, const TimedElasticBand& teb) {
  std::printf("%s_N %d\n", key, teb.sizePoses());
  for (int i = 0; i < teb.sizePoses(); ++i)
    std::printf("%s_POSE %d %.17g %.17g %.17g %.17g\n", key, i, teb.Pose(i).x(), teb.Pose(i).y(), teb.Pose(i).theta(),
                i < teb.sizeTimeDiffs() ? teb.TimeDiff(i) : 0.0);
}

static std::vector<geometry_msgs::PoseStamped> sine_plan(double amp, int m) {
  std::vector<geometry_msgs::PoseStamped> plan(m);
  for (int i = 0; i < m; ++i) {
    double s = (double)i / (m - 1);
    plan[i].pose.position.x = -4 + 8 * s;
    plan[i].pose.position.y = amp * std::sin(M_PI * s);
    plan[i].pose.orientation = tf::createQuaternionFromYaw(0);
  }
  return plan;
}

static int gpu_checks() {
  /* ---- test_optim_node scene: TebOptimalPlanner::plan(start, goal) twice (cold start, then warm start) */
  TebConfig cfg;
  ObstContainer obst;
  obst.push_back(ObstaclePtr(new PointObstacle(-3, 1)));
  obst.push_back(ObstaclePtr(new PointObstacle(6, 2)));
  obst.push_back(ObstaclePtr(new PointObstacle(0, 0.1)));
  obst[0]->setCentroidVelocity(Eigen::Vector2d(0.1, -0.3));
  obst[1]->setCentroidVelocity(Eigen::Vector2d(-0.3, -0.2));
  ViaPointContainer via;
  TebOptimalPlanner planner(cfg, &obst, TebVisualizationPtr(), &via);
  bool ok = planner.plan(PoseSE2(-4, 0, 0), PoseSE2(4, 0, 0));
  std::printf("SINGLE_OK %d\nSINGLE_STATUS %d\n", ok ? 1 : 0, planner.lastStatus());
  print_band("SINGLE", planner.teb());
  double vx, vy, om;
  CHECK(planner.getVelocityCommand(vx, vy, om, 1));
  std::printf("SINGLE_CMD %.17g %.17g %.17g\n", vx, vy, om);
  planner.computeCurrentCost(1.0, 1.0, false);
  std::printf("SINGLE_COST %.17g\n", planner.getCurrentCost());
  geometry_msgs::Twist v0;
  v0.linear.x = vx;
  v0.angular.z = om;
  ok = planner.plan(PoseSE2(-3.9, 0.01, 0.02), PoseSE2(4, 0, 0), &v0);
  std::printf("WARM_OK %d\n", ok ? 1 : 0);
  print_band("WARM", planner.teb());
  {
    /* optimizeTEB's argument edges (optimal_planner.cpp:182-231): no outer iteration returns true and leaves
     * isOptimized() false; no inner iteration makes optimizeGraph fail (:393), so it returns false */
    const int n_before = planner.teb().sizePoses();
    const bool r0 = planner.optimizeTEB(5, 0, true);
    const bool opt0 = planner.isOptimized();
    CHECK(r0 && !opt0 && planner.teb().sizePoses() == n_before);
    const bool r1 = planner.optimizeTEB(0, 3, true);
    CHECK(!r1 && !planner.isOptimized());
    std::printf("EDGES %d %d %d\n", r0 ? 1 : 0, opt0 ? 1 : 0, r1 ? 1 : 0);
  }

  /* ---- HomotopyClassPlanner: three seeded candidates, one batched optimisation, selection */
  TebConfig hcfg;
  hcfg.obstacles.include_dynamic_obstacles = false;
  hcfg.hcp.max_number_classes = 3; /* the three seeded classes fill the container: no graph search in this scene */
  ObstContainer hob;
  hob.push_back(ObstaclePtr(new PointObstacle(0, 0.1)));
  hob.push_back(ObstaclePtr(new PointObstacle(-1.5, -0.4)));
  hob.push_back(ObstaclePtr(new CircularObstacle(2, 0.6, 0.2)));
  HomotopyClassPlanner hcp(hcfg, &hob);
  auto p0 = sine_plan(0.0, 21), p1 = sine_plan(1.2, 21), p2 = sine_plan(-1.0, 21);
  hcp.addAndInitNewTeb(p1, NULL);
  hcp.addAndInitNewTeb(p2, NULL);
  /* a second band of the class of p1 (same side of every obstacle) is not kept (addEquivalenceClassIfNew) */
  auto dup = sine_plan(0.9, 21);
  std::printf("HCP_DUP_REJECTED %d\n", hcp.addAndInitNewTeb(dup, NULL) ? 0 : 1);
  ok = hcp.plan(p0, NULL);  /* the initial-plan candidate is created by exploreEquivalenceClassesAndInitTebs */
  std::printf("HCP_OK %d\nHCP_NUM %d\nHCP_BEST %d\n", ok ? 1 : 0, (int)hcp.getTrajectoryContainer().size(), hcp.bestTebIdx());
  {
    int c = 0;
    for (const auto& eq : hcp.getEquivalenceClassRef()) { /* signatures of the bands as they were when classified */
      const HSignature* h = dynamic_cast<const HSignature*>(eq.first.get());
      if (h) std::printf("HCP_H %d %.17g %.17g\n", c, h->value().real(), h->value().imag());
      ++c;
    }
  }
  int k = 0;
  for (auto& t : hcp.getTrajectoryContainer()) {
    std::printf("HCP_COST %d %.17g\n", k, t->getCurrentCost());
    char key[32];
    std::snprintf(key, sizeof(key), "HCP%d", k);
    print_band(key, t->teb());
    ++k;
  }
  CHECK(hcp.bestTeb() != nullptr);
  CHECK(hcp.getVelocityCommand(vx, vy, om, 1));
  { /* ---- polygon footprint among line / pill / polygon obstacles (one static, one moving) */
    TebConfig scfg;
    ObstContainer so;
    so.push_back(ObstaclePtr(new LineObstacle(-1.0, 0.6, 0.5, 1.4)));
    so.push_back(ObstaclePtr(new PillObstacle(1.0, -1.2, 2.0, -0.5, 0.15)));
    PolygonObstacle* po = new PolygonObstacle();
    po->pushBackVertex(-0.3, -0.6); po->pushBackVertex(0.4, -0.7); po->pushBackVertex(0.2, -0.1);
    po->finalizePolygon();
    so.push_back(ObstaclePtr(po));
    so[1]->setCentroidVelocity(Eigen::Vector2d(-0.1, 0.1));
    ViaPointContainer svia;
    TebOptimalPlanner sp(scfg, &so, TebVisualizationPtr(), &svia);
    Point2dContainer body = {Eigen::Vector2d(-0.25, -0.2), Eigen::Vector2d(0.35, -0.2), Eigen::Vector2d(0.35, 0.2), Eigen::Vector2d(-0.25, 0.2)};
    sp.updateRobotModel(RobotFootprintModelPtr(new PolygonRobotFootprint(body)));
    bool sok = sp.plan(PoseSE2(-4, 0, 0), PoseSE2(4, 0, 0));
    std::printf("SHAPES_OK %d\nSHAPES_STATUS %d\n", sok ? 1 : 0, sp.lastStatus());
    print_band("SHAPES", sp.teb());
  }
  { /* ---- the whole cycle with nothing seeded: explore (key-point graph) -> one batched optimisation -> select */
    TebConfig acfg;
    acfg.hcp.simple_exploration = true;
    acfg.obstacles.include_dynamic_obstacles = false;
    acfg.hcp.max_number_classes = 4;
    ObstContainer aob;
    aob.push_back(ObstaclePtr(new PointObstacle(-1.5, 0.3)));
    aob.push_back(ObstaclePtr(new CircularObstacle(0.5, -0.4, 0.3)));
    aob.push_back(ObstaclePtr(new PointObstacle(2.0, 0.5)));
    HomotopyClassPlanner ahcp(acfg, &aob);
    bool aok = ahcp.plan(PoseSE2(-4, 0, 0.1), PoseSE2(4, 0.2, -0.2), NULL);
    std::printf("AUTO_OK %d\nAUTO_NUM %d\nAUTO_BEST %d\n", aok ? 1 : 0, (int)ahcp.getTrajectoryContainer().size(), ahcp.bestTebIdx());
    int q = 0;
    for (auto& t : ahcp.getTrajectoryContainer()) {
      std::printf("AUTO_COST %d %.17g\n", q, t->getCurrentCost());
      char key[32];
      std::snprintf(key, sizeof(key), "AUTO%d", q++);
      print_band(key, t->teb());
    }
  }
  { /* ---- optimizeAllTEBs sharded over two device contexts (device 1 when the box has one, else twice device 0): the
     * candidates, their costs and the winner must be those of the single-context run */
    int devices = 0;
    cudaGetDeviceCount(&devices);
    auto run = [&](bool sharded, std::vector<double>& costs, int& best) {
      TebConfig mcfg;
      mcfg.obstacles.include_dynamic_obstacles = false;
      mcfg.hcp.max_number_classes = 3;
      HomotopyClassPlanner m(mcfg, &hob);
      if (sharded) {
        std::vector<TebGpuContextPtr> ctxs;
        ctxs.push_back(TebGpuContextPtr(new TebGpuContext(8, 512, 64, 8, 0)));
        ctxs.push_back(TebGpuContextPtr(new TebGpuContext(8, 512, 64, 8, devices > 1 ? 1 : 0)));
        m.setGpuContexts(ctxs);
      }
      m.addAndInitNewTeb(p1, NULL);
      m.addAndInitNewTeb(p2, NULL);
      const bool mok = m.plan(p0, NULL);
      CHECK(mok);
      for (auto& t : m.getTrajectoryContainer()) costs.push_back(t->getCurrentCost());
      best = m.bestTebIdx();
    };
    std::vector<double> c_single, c_sharded;
    int b_single = -2, b_sharded = -3;
    run(false, c_single, b_single);
    run(true, c_sharded, b_sharded);
    CHECK(c_single.size() == c_sharded.size() && b_single == b_sharded);
    bool same = c_single.size() == c_sharded.size();
    for (size_t q = 0; same && q < c_single.size(); ++q) same = c_single[q] == c_sharded[q];
    CHECK(same);
    std::printf("SHARDED_OK %d devices %d candidates %d\n", same ? 1 : 0, devices, (int)c_sharded.size());
  }
  /* second cycle: hysteresis path of selectBestTeb + warm start of all candidates */
  ok = hcp.plan(PoseSE2(-3.95, 0, 0), PoseSE2(4, 0, 0), NULL);
  std::printf("HCP2_OK %d\nHCP2_BEST %d\nHCP2_NUM %d\n", ok ? 1 : 0, hcp.bestTebIdx(), (int)hcp.getTrajectoryContainer().size());
  return 0;
}

/* exploreEquivalenceClassesAndInitTebs alone (no optimisation): the candidate bands the graph search proposes */
static void explore_checks() {
  for (int variant = 0; variant < 4; ++variant) {
    TebConfig cfg;
    cfg.hcp.simple_exploration = (variant & 1) != 0;            /* 0: ProbRoadmapGraph, 1: lrKeyPointGraph */
    cfg.obstacles.include_dynamic_obstacles = (variant & 2) != 0; /* 2-D signature / x-y-t signature */
    cfg.hcp.max_number_classes = 6;
    ObstContainer obst;
    obst.push_back(ObstaclePtr(new PointObstacle(-1.5, 0.3)));
    obst.push_back(ObstaclePtr(new CircularObstacle(0.5, -0.4, 0.3)));
    obst.push_back(ObstaclePtr(new PointObstacle(2.0, 0.5)));
    obst.push_back(ObstaclePtr(new LineObstacle(-3.0, -1.5, -2.5, -0.8)));
    if (variant & 2) obst[2]->setCentroidVelocity(Eigen::Vector2d(-0.1, 0.05));
    HomotopyClassPlanner hcp(cfg, &obst);
    for (int cycle = 0; cycle < 2; ++cycle) { /* the second cycle starts from the kept bands and a continued random stream */
      hcp.exploreEquivalenceClassesAndInitTebs(PoseSE2(-4, 0, 0.1), PoseSE2(4, 0.2, -0.2), cfg.obstacles.min_obstacle_dist, NULL);
      std::printf("EXPLORE%d_%d_NUM %d\n", variant, cycle, (int)hcp.getTrajectoryContainer().size());
      int k = 0;
      for (auto& t : hcp.getTrajectoryContainer()) {
        char key[40];
        std::snprintf(key, sizeof(key), "EXPLORE%d_%d_%d", variant, cycle, k++);
        print_band(key, t->teb());
      }
      if (cycle == 0) hcp.clearPlanner(); /* fresh container, random stream continues (member of the graph object) */
    }
  }
}

int main(int argc, char** argv) {
  cpu_checks();
  postprocessing_checks();
  if (argc > 1 && std::string(argv[1]) == "gpu") gpu_checks();
  if (argc > 1 && std::string(argv[1]) == "explore") explore_checks();
  std::printf("RESULT %s (%d failed checks)\n", g_fail ? "FAIL" : "PASS", g_fail);
  return g_fail ? 1 : 0;
}
