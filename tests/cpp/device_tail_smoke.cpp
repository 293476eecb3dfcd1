// Drives ResidentPoseGraph::solve_with_device_factors through the C ABI (plain g++ + the CUDA runtime for the device rows).
// Build: g++ -std=c++17 -I include -I <cuda>/include tests/cpp/device_tail_smoke.cpp -L omni-swarm_b200/csrc
//        -lomniswarm_b200 -L <cuda>/lib64 -lcudart -o device_tail_smoke
// Without a GPU it only checks that osb_solver_create reports OSB_ERR_NO_DEVICE.
#include <cuda_runtime.h>
#include <cmath>
#include <cstring>
#include "omniswarm_b200_adapters.hpp"

int main() {
  osb_solver *solver = nullptr, *flat = nullptr;
  const osb_status st = osb_solver_create(&solver, 64, 256);
  if (st == OSB_ERR_NO_DEVICE) { std::printf("no device\n"); return 0; }
  osb::check(st, "osb_solver_create");
  osb::check(osb_solver_create(&flat, 64, 256), "osb_solver_create");
  // two drones, 8 frames each: odometry chains and one UWB range per frame in the resident window, started 0.2 m off
  const int F = 8;
  double gt[2][F][4], est[2][F][4];
  for (int k = 0; k < F; ++k) {
    const double a = 0.5 * k;
    const double p0[4] = {2.0 * std::cos(a), 2.0 * std::sin(a), 0.1 * k, a};
    const double p1[4] = {3.0 + 1.5 * std::sin(a), 1.0 - 1.5 * std::cos(a), 0.5, -0.2 * k};
    std::memcpy(gt[0][k], p0, sizeof(p0)); std::memcpy(gt[1][k], p1, sizeof(p1));
    for (int j = 0; j < 4; ++j) { est[0][k][j] = p0[j] + (k ? 0.2 : 0.0); est[1][k][j] = p1[j] + 0.2; }
  }
  double S[16] = {0};
  for (int i = 0; i < 16; i += 5) S[i] = 10.0;
  auto rel = [](const double* A, const double* B, double* m) {
    const double c = std::cos(A[3]), s = std::sin(A[3]), dx = B[0] - A[0], dy = B[1] - A[1];
    m[0] = c * dx + s * dy; m[1] = -s * dx + c * dy; m[2] = B[2] - A[2]; m[3] = B[3] - A[3];
  };
  osb::ResidentPoseGraph g(solver);
  for (int d = 0; d < 2; ++d)
    for (int k = 0; k < F; ++k) g.node(est[d][k]);        // node ids: drone-major append order
  for (int d = 0; d < 2; ++d)
    for (int k = 0; k + 1 < F; ++k) { double m[4]; rel(gt[d][k], gt[d][k + 1], m); g.add_relative_pose(est[d][k], est[d][k + 1], m, S, false); }
  for (int k = 0; k < F; ++k) {
    const double dx = gt[0][k][0] - gt[1][k][0], dy = gt[0][k][1] - gt[1][k][1], dz = gt[0][k][2] - gt[1][k][2];
    g.add_distance(est[0][k], est[1][k], std::sqrt(dx * dx + dy * dy + dz * dz), 10.0, true);
  }
  g.set_constant(est[0][0]);
  // the tail: four inter-drone loops, as osb_anchor_compact_factors_dev leaves them in device memory
  const int K = 4;
  int32_t type[K], ia[K], ib[K];
  uint8_t huber[K];
  double payload[K][OSB_PAYLOAD_LEN] = {};
  for (int q = 0; q < K; ++q) {
    const int ka = 2 * q, kb = 2 * q + 1;
    type[q] = OSB_FACTOR_RELPOSE; ia[q] = ka; ib[q] = F + kb; huber[q] = 1;
    rel(gt[0][ka], gt[1][kb], payload[q]);
    for (int i = 0; i < 16; ++i) payload[q][4 + i] = S[i];
  }
  int32_t *d_type, *d_ia, *d_ib, *d_count;
  double* d_payload;
  uint8_t* d_huber;
  if (cudaMalloc(&d_type, sizeof(type)) || cudaMalloc(&d_ia, sizeof(ia)) || cudaMalloc(&d_ib, sizeof(ib)) ||
      cudaMalloc(&d_count, sizeof(int32_t)) || cudaMalloc(&d_payload, sizeof(payload)) || cudaMalloc(&d_huber, sizeof(huber))) {
    std::printf("cudaMalloc failed\n"); return 2;
  }
  const int32_t count = K;
  cudaMemcpy(d_type, type, sizeof(type), cudaMemcpyHostToDevice); cudaMemcpy(d_ia, ia, sizeof(ia), cudaMemcpyHostToDevice);
  cudaMemcpy(d_ib, ib, sizeof(ib), cudaMemcpyHostToDevice); cudaMemcpy(d_count, &count, sizeof(count), cudaMemcpyHostToDevice);
  cudaMemcpy(d_payload, payload, sizeof(payload), cudaMemcpyHostToDevice);
  cudaMemcpy(d_huber, huber, sizeof(huber), cudaMemcpyHostToDevice);
  cudaStream_t stream;
  cudaStreamCreate(&stream);
  osb_solve_options o;
  osb_solve_default_options(&o);
  o.function_tolerance = 1e-14; o.pcg_tolerance = 1e-8; o.max_pcg_iterations = 2000;
  double start[2][F][4];
  std::memcpy(start, est, sizeof(est));
  const osb_solve_summary s = g.solve_with_device_factors(16, d_type, d_ia, d_ib, d_payload, d_huber, d_count, stream, &o);
  // the same list (window, then tail) solved one-shot from the same start
  std::vector<int32_t> ft, fa, fb;
  std::vector<uint8_t> fh, fixed(2 * F, 0);
  std::vector<double> pl;
  fixed[0] = 1;
  auto push = [&](int t, int a, int b, const double* p, int h) {
    ft.push_back(t); fa.push_back(a); fb.push_back(b); fh.push_back((uint8_t)h); pl.insert(pl.end(), p, p + OSB_PAYLOAD_LEN);
  };
  for (int d = 0; d < 2; ++d)
    for (int k = 0; k + 1 < F; ++k) {
      double p[OSB_PAYLOAD_LEN] = {0};
      rel(gt[d][k], gt[d][k + 1], p);
      for (int i = 0; i < 16; ++i) p[4 + i] = S[i];
      push(OSB_FACTOR_RELPOSE, d * F + k, d * F + k + 1, p, 0);
    }
  for (int k = 0; k < F; ++k) {
    const double dx = gt[0][k][0] - gt[1][k][0], dy = gt[0][k][1] - gt[1][k][1], dz = gt[0][k][2] - gt[1][k][2];
    const double p[OSB_PAYLOAD_LEN] = {std::sqrt(dx * dx + dy * dy + dz * dz), 10.0};
    push(OSB_FACTOR_DISTANCE, k, F + k, p, 1);
  }
  for (int q = 0; q < K; ++q) push(type[q], ia[q], ib[q], payload[q], huber[q]);
  osb_solve_summary s1{};
  osb::check(osb_solver_solve(flat, 2 * F, &start[0][0][0], fixed.data(), (int)ft.size(), ft.data(), fa.data(), fb.data(),
                              pl.data(), fh.data(), &o, &s1), "osb_solver_solve");
  double diff = 0.0, err = 0.0;
  for (int d = 0; d < 2; ++d)
    for (int k = 0; k < F; ++k)
      for (int j = 0; j < 4; ++j) {
        diff = std::fmax(diff, std::fabs(est[d][k][j] - start[d][k][j]));
        if (j < 3) err = std::fmax(err, std::fabs(est[d][k][j] - gt[d][k][j]));
      }
  if (s.n_residuals != s1.n_residuals) { std::printf("n_residuals %d != %d\n", s.n_residuals, s1.n_residuals); return 3; }
  if (!(diff < 1e-6)) { std::printf("device tail and one-shot solves differ by %g\n", diff); return 4; }
  if (!(err < 1e-4)) { std::printf("solution %g from the ground truth\n", err); return 5; }
  cudaFree(d_type); cudaFree(d_ia); cudaFree(d_ib); cudaFree(d_count); cudaFree(d_payload); cudaFree(d_huber);
  cudaStreamDestroy(stream);
  osb_solver_destroy(flat);
  osb_solver_destroy(solver);
  std::printf("device tail ok: %d residuals, %d iterations, max |device - one-shot| %.3g\n", s.n_residuals, s.iterations, diff);
  return 0;
}
