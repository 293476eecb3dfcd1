// Drives FlatPoseGraph::mark_for_init / solve_with_multiple_init through the C ABI (plain g++, no OpenCV).
// Build: g++ -std=c++17 -I include tests/cpp/multistart_smoke.cpp -L omni-swarm_b200/csrc -lomniswarm_b200 -o multistart_smoke
// Without a GPU it only checks that osb_solver_create reports OSB_ERR_NO_DEVICE.
#include <cmath>
#include <cstring>
#include "omniswarm_b200_adapters.hpp"

int main() {
  osb_solver* solver = nullptr;
  const osb_status st = osb_solver_create(&solver, 64, 256);
  if (st == OSB_ERR_NO_DEVICE) { std::printf("no device\n"); return 0; }
  osb::check(st, "osb_solver_create");
  // two drones, 8 frames each: odometry chains and one UWB range per frame; drone 0 starts at its ground truth (first
  // frame constant), drone 1 starts at the origin and is re-initialised at random
  const int F = 8;
  double gt[2][F][4], est[2][F][4];
  for (int k = 0; k < F; ++k) {
    const double a = 0.5 * k;
    const double p0[4] = {2.0 * std::cos(a), 2.0 * std::sin(a), 0.1 * k, a};
    const double p1[4] = {3.0 + 1.5 * std::sin(a), 1.0 - 1.5 * std::cos(a), 0.5, -0.2 * k};
    std::memcpy(gt[0][k], p0, sizeof(p0)); std::memcpy(gt[1][k], p1, sizeof(p1));
    std::memcpy(est[0][k], p0, sizeof(p0));
    for (int j = 0; j < 4; ++j) est[1][k][j] = j == 3 ? p1[3] : 0.0;     // odometry yaw, as random_init_pose keeps it
  }
  double S[16] = {0};
  for (int i = 0; i < 4; ++i) S[i * 5] = 10.0;
  osb::FlatPoseGraph g;
  for (int d = 0; d < 2; ++d)
    for (int k = 0; k + 1 < F; ++k) {                       // RelativePoseFactor4d: pose k+1 in the frame of pose k
      const double* A = gt[d][k]; const double* B = gt[d][k + 1];
      const double c = std::cos(A[3]), s = std::sin(A[3]), dx = B[0] - A[0], dy = B[1] - A[1];
      const double meas[4] = {c * dx + s * dy, -s * dx + c * dy, B[2] - A[2], B[3] - A[3]};
      g.add_relative_pose(est[d][k], est[d][k + 1], meas, S, false);
    }
  for (int k = 0; k < F; ++k) {
    const double dx = gt[0][k][0] - gt[1][k][0], dy = gt[0][k][1] - gt[1][k][1], dz = gt[0][k][2] - gt[1][k][2];
    g.add_distance(est[0][k], est[1][k], std::sqrt(dx * dx + dy * dy + dz * dz), 10.0, true);
  }
  g.set_constant(est[0][0]);
  for (int k = 0; k < F; ++k) g.mark_for_init(est[1][k]);

  osb_multistart_options ms{};
  ms.n_trials = 8; ms.normalise = 1; ms.window_size = F; ms.seed = 11; ms.rand_xy = 5.0; ms.rand_z = 1.0;
  ms.acpt_cost = -1.0;                                      // nothing can be accepted: the pose blocks stay as they are
  double before[2][F][4];
  std::memcpy(before, est, sizeof(est));
  if (g.solve_with_multiple_init(solver, ms)) { std::printf("accepted below a negative acpt_cost\n"); return 2; }
  if (std::memcmp(before, est, sizeof(est)) != 0) { std::printf("poses changed although no trial was accepted\n"); return 3; }
  ms.acpt_cost = 1e30;                                      // the best finite trial is accepted and written back
  if (!g.solve_with_multiple_init(solver, ms)) { std::printf("no trial accepted\n"); return 4; }
  if (est[0][0][0] != gt[0][0][0] || est[0][0][3] != gt[0][0][3]) { std::printf("constant pose moved\n"); return 5; }
  bool moved = false;
  for (int k = 0; k < F; ++k)
    for (int j = 0; j < 4; ++j) {
      if (!std::isfinite(est[1][k][j])) { std::printf("non-finite pose\n"); return 6; }
      moved = moved || est[1][k][j] != before[1][k][j];
    }
  if (!moved) { std::printf("the accepted trial did not move drone 1\n"); return 7; }
  osb_solver_destroy(solver);
  std::printf("multistart ok: equv_cost %.3g, drone 1 frame 0 at (%.3f, %.3f, %.3f)\n", g.cost_now, est[1][0][0],
              est[1][0][1], est[1][0][2]);
  return 0;
}
