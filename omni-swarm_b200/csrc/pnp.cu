// pnp.cu -- relative pose of a loop candidate on the device: deterministic PnP-RANSAC + the reference's acceptance checks.
//
// Replaces LoopDetector::compute_relative_pose (swarm_loop/src/loop_detector.cpp:355-413: cv::solvePnPRansac on
// matched_3d_now / matched_2d_norm_old with K = I, 100 or 1000 iterations, reprojection error 3; then PnPRestoCamPose,
// DeltaPose, RPerror :338-351 and pnp_result_verify :317-336) and check_loop_odometry_consistency (:294-315) -- the last
// CPU stage before a LoopEdge exists (SURVEY.md section 8f-1, second half).
//
// OpenCV's RANSAC is randomised; its RESULT is the Levenberg-Marquardt minimiser of the squared reprojection error over
// the inliers of the best model.  The library defines a deterministic RANSAC with the same error / threshold rule / result
// (oracle/pnp_ref.py, pinned there against cv2.solvePnPRansac: same inliers, pose to 1e-10 on separated data):
//   hypothesis h draws 4 correspondences from the counter-based hash of the homography filter (geom.cu), its model is a
//   fixed-schedule LM fit of those 4 points started from the caller's odometry prior; first best hypothesis wins; the
//   pose is refined by LM over the winner's inliers.
// One CTA per candidate: thread = hypothesis (fit + scoring over all points, fp64), packed-key block reduction for the
// winner, then the block refines cooperatively (28 sums per LM iteration by warp shuffles) and thread 0 applies the checks.
#include "common.cuh"
#include "kernels.cuh"
#include "pose_algebra.cuh"

namespace osb {

// PNP_THREADS and PNP_MAXN: kernels.cuh
constexpr int PNP_HYP_ITERS = 8;        // oracle/pnp_ref.py HYP_ITERS
constexpr int PNP_REFINE_ITERS = 12;    // REFINE_ITERS

__host__ __device__ __forceinline__ uint32_t pnp_lowbias32(uint32_t x) {
  x ^= x >> 16; x *= 0x7FEB352Du; x ^= x >> 15; x *= 0x846CA68Bu; x ^= x >> 16;
  return x;
}
__device__ bool pnp_draw4(uint32_t seed, int h, int n, int (&idx)[4]) {          // geometry_ref.draw4
  for (int slot = 0; slot < 4; ++slot) {
    bool ok = false;
    for (int t = 0; t < 16 && !ok; ++t) {
      const int v = (int)(pnp_lowbias32(seed ^ pnp_lowbias32((uint32_t)((h * 4 + slot) * 16 + t) + 0x9E3779B9u)) % (uint32_t)n);
      bool dup = false;
      for (int j = 0; j < slot; ++j) dup |= (idx[j] == v);
      if (!dup) { idx[slot] = v; ok = true; }
    }
    if (!ok) return false;
  }
  return true;
}

// residual and Jacobian rows of one correspondence: unknowns (d_theta, d_t), left perturbation (pnp_ref._normal_eq)
__device__ __forceinline__ void pnp_point(const PoseD& P, const float3 X, const float2 m, double& r0, double& r1, double (&J0)[6],
                                          double (&J1)[6]) {
  const double x[3] = {(double)X.x, (double)X.y, (double)X.z};
  double y[3];
  q_rot(P.q, x, y);
  const double p0 = y[0] + P.t[0], p1 = y[1] + P.t[1], p2 = y[2] + P.t[2];
  const double iz = 1.0 / p2;
  r0 = p0 * iz - (double)m.x; r1 = p1 * iz - (double)m.y;
  const double a[3] = {iz, 0.0, -p0 * iz * iz}, b[3] = {0.0, iz, -p1 * iz * iz};
  J0[0] = y[1] * a[2] - y[2] * a[1]; J0[1] = y[2] * a[0] - y[0] * a[2]; J0[2] = y[0] * a[1] - y[1] * a[0];
  J0[3] = a[0]; J0[4] = a[1]; J0[5] = a[2];
  J1[0] = y[1] * b[2] - y[2] * b[1]; J1[1] = y[2] * b[0] - y[0] * b[2]; J1[2] = y[0] * b[1] - y[1] * b[0];
  J1[3] = b[0]; J1[4] = b[1]; J1[5] = b[2];
}
__device__ __forceinline__ double pnp_err(const PoseD& P, const float3 X, const float2 m) {
  const double x[3] = {(double)X.x, (double)X.y, (double)X.z};
  double y[3];
  q_rot(P.q, x, y);
  const double iz = 1.0 / (y[2] + P.t[2]);
  const double du = (y[0] + P.t[0]) * iz - (double)m.x, dv = (y[1] + P.t[1]) * iz - (double)m.y;
  return du * du + dv * dv;
}
// (A + lam diag(A) + 1e-12 I) d = -g by unpivoted Cholesky; A symmetric 6x6 (full storage); false if not SPD / not finite
__device__ bool pnp_solve6(const double (&A)[36], const double (&g)[6], double lam, double (&d)[6]) {
  double L[6][6];
  for (int j = 0; j < 6; ++j) {
    double s = A[j * 6 + j] + lam * A[j * 6 + j] + 1e-12;
    for (int k = 0; k < j; ++k) s -= L[j][k] * L[j][k];
    if (!(s > 0.0)) return false;
    L[j][j] = sqrt(s);
    for (int i = j + 1; i < 6; ++i) {
      double c = A[i * 6 + j];
      for (int k = 0; k < j; ++k) c -= L[i][k] * L[j][k];
      L[i][j] = c / L[j][j];
    }
  }
  double y[6];
  for (int i = 0; i < 6; ++i) {
    double c = -g[i];
    for (int k = 0; k < i; ++k) c -= L[i][k] * y[k];
    y[i] = c / L[i][i];
  }
  for (int i = 5; i >= 0; --i) {
    double c = y[i];
    for (int k = i + 1; k < 6; ++k) c -= L[k][i] * d[k];
    d[i] = c / L[i][i];
  }
  bool fin = true;
  for (int i = 0; i < 6; ++i) fin &= isfinite(d[i]);
  return fin;
}
__device__ __forceinline__ PoseD pnp_apply(const PoseD& P, const double (&d)[6]) {
  PoseD o;
  double dq[4], rt[3];
  quat_from_rotvec(d, dq);
  q_rot(dq, P.t, rt);
  o.t[0] = rt[0] + d[3]; o.t[1] = rt[1] + d[4]; o.t[2] = rt[2] + d[5];
  q_mul(dq, P.q, o.q);
  const double n = sqrt(o.q[0] * o.q[0] + o.q[1] * o.q[1] + o.q[2] * o.q[2] + o.q[3] * o.q[3]);
  o.q[0] /= n; o.q[1] /= n; o.q[2] /= n; o.q[3] /= n;
  return o;
}

// fixed-schedule LM on 4 correspondences, one thread (pnp_ref.lm_pose)
__device__ PoseD pnp_fit4(PoseD P, const float3* X, const float2* uv, const int (&idx)[4]) {
  double A[36], g[6], cost;
  auto normal = [&](const PoseD& Q) {
    for (int i = 0; i < 36; ++i) A[i] = 0.0;
    for (int i = 0; i < 6; ++i) g[i] = 0.0;
    cost = 0.0;
    for (int k = 0; k < 4; ++k) {
      double r0, r1, J0[6], J1[6];
      pnp_point(Q, X[idx[k]], uv[idx[k]], r0, r1, J0, J1);
      cost += r0 * r0 + r1 * r1;
      for (int i = 0; i < 6; ++i) {
        for (int j = 0; j < 6; ++j) A[i * 6 + j] += J0[i] * J0[j] + J1[i] * J1[j];
        g[i] += J0[i] * r0 + J1[i] * r1;
      }
    }
  };
  normal(P);
  double lam = 1e-3;
  for (int it = 0; it < PNP_HYP_ITERS; ++it) {
    double d[6];
    bool ok = pnp_solve6(A, g, lam, d);
    PoseD cand;
    if (ok) {
      cand = pnp_apply(P, d);
      double c = 0.0;
      for (int k = 0; k < 4; ++k) c += pnp_err(cand, X[idx[k]], uv[idx[k]]);
      ok = isfinite(c) && c < cost;
    }
    if (ok) { P = cand; normal(P); lam = fmax(lam * 0.1, 1e-9); }
    else lam = fmin(lam * 10.0, 1e6);
  }
  return P;
}

__device__ __forceinline__ double block_sum(double v, double* scratch /*[8]*/) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) scratch[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
  for (int w = 0; w < PNP_THREADS / 32; ++w) s += scratch[w];
  return s;
}

__global__ void __launch_bounds__(PNP_THREADS)
pnp_ransac_kernel(const float* __restrict__ pts3d, const float* __restrict__ pts2d, const int32_t* __restrict__ n_pts, int max_n,
                  const osb_pnp_params* __restrict__ params, uint8_t* __restrict__ mask_out, osb_pnp_result* __restrict__ results) {
  __shared__ float3 sX[PNP_MAXN];
  __shared__ float2 sU[PNP_MAXN];
  __shared__ uint8_t sM[PNP_MAXN];
  __shared__ unsigned long long s_best;
  __shared__ double s_pose[7];
  __shared__ double s_red[8];
  __shared__ double s_sys[43];          // A (36), g (6), cost
  __shared__ double s_cand[8];          // candidate pose + accept flag
  const int c = blockIdx.x, tid = threadIdx.x;
  const osb_pnp_params& prm = params[c];
  const int n = min(n_pts[c], max_n);
  osb_pnp_result* res = results + c;
  uint8_t* mk = mask_out + (size_t)c * max_n;
  for (int i = tid; i < max_n; i += PNP_THREADS) mk[i] = 0;
  for (int i = tid; i < n; i += PNP_THREADS) {
    sX[i] = make_float3(pts3d[((size_t)c * max_n + i) * 3], pts3d[((size_t)c * max_n + i) * 3 + 1], pts3d[((size_t)c * max_n + i) * 3 + 2]);
    sU[i] = make_float2(pts2d[((size_t)c * max_n + i) * 2], pts2d[((size_t)c * max_n + i) * 2 + 1]);
  }
  if (tid == 0) s_best = 0ull;
  __syncthreads();
  const PoseD prior = load_pose(prm.prior);
  const double t2 = (double)prm.reproj_thresh * (double)prm.reproj_thresh;
  auto write_fail = [&](int n_inl, int winner) {
    if (tid == 0) {
      res->pnp_success = 0; res->n_inliers = n_inl; res->winner = winner; res->verified = 0; res->odometry_consistent = 1;
      res->rperr = 0.0; res->md = 0.0;
      for (int i = 0; i < 7; ++i) res->pose_cam[i] = prm.prior[i];
      for (int i = 0; i < 4; ++i) res->dp_old_to_new[i] = 0.0;
    }
  };
  if (n < 4) { write_fail(0, -1); return; }
  // ---- hypotheses: fit + score, key = (inliers + 1) << 32 | ~h  (most inliers, then smallest h) ----
  unsigned long long my_key = 0ull;
  PoseD my_pose = prior;
  for (int h = tid; h < prm.iterations; h += PNP_THREADS) {
    int idx[4];
    if (!pnp_draw4(prm.seed, h, n, idx)) continue;
    const PoseD P = pnp_fit4(prior, sX, sU, idx);
    int cnt = 0;
    for (int i = 0; i < n; ++i) cnt += pnp_err(P, sX[i], sU[i]) <= t2;      // NaN compares false
    const unsigned long long key = ((unsigned long long)(cnt + 1) << 32) | (unsigned long long)(0xFFFFFFFFu - (uint32_t)h);
    if (key > my_key) { my_key = key; my_pose = P; }
  }
  if (my_key) atomicMax(&s_best, my_key);
  __syncthreads();
  const unsigned long long best = s_best;
  const int best_cnt = (int)(best >> 32) - 1;
  const int winner = best ? (int)(0xFFFFFFFFu - (uint32_t)(best & 0xFFFFFFFFull)) : -1;
  if (best_cnt < 4) { write_fail(max(best_cnt, 0), winner); return; }
  if (my_key == best) {                                      // exactly one thread owns the winning hypothesis
    for (int i = 0; i < 3; ++i) s_pose[i] = my_pose.t[i];
    for (int i = 0; i < 4; ++i) s_pose[3 + i] = my_pose.q[i];
  }
  __syncthreads();
  PoseD P = load_pose(s_pose);
  for (int i = tid; i < n; i += PNP_THREADS) {
    const uint8_t in = pnp_err(P, sX[i], sU[i]) <= t2;
    sM[i] = in; mk[i] = in;
  }
  __syncthreads();
  // ---- refinement: LM over the winner's inliers, the block accumulates the normal equations ----
  auto normal_block = [&](const PoseD& Q) {
    double acc[28];                                         // 21 upper-triangle entries of A, 6 of g, cost
    for (int i = 0; i < 28; ++i) acc[i] = 0.0;
    for (int k = tid; k < n; k += PNP_THREADS) {
      if (!sM[k]) continue;
      double r0, r1, J0[6], J1[6];
      pnp_point(Q, sX[k], sU[k], r0, r1, J0, J1);
      int e = 0;
      for (int i = 0; i < 6; ++i)
        for (int j = i; j < 6; ++j) acc[e++] += J0[i] * J0[j] + J1[i] * J1[j];
      for (int i = 0; i < 6; ++i) acc[21 + i] += J0[i] * r0 + J1[i] * r1;
      acc[27] += r0 * r0 + r1 * r1;
    }
    for (int i = 0; i < 28; ++i) {
      const double s = block_sum(acc[i], s_red);
      if (tid == 0) {
        if (i < 21) {
          int e = 0, a = 0, b = 0;
          for (a = 0; a < 6; ++a) { bool f = false; for (b = a; b < 6; ++b) { if (e == i) { f = true; break; } ++e; } if (f) break; }
          s_sys[a * 6 + b] = s; s_sys[b * 6 + a] = s;
        } else {
          s_sys[36 + (i - 21)] = s;
        }
      }
    }
    __syncthreads();
  };
  normal_block(P);
  double lam = 1e-3;
  for (int it = 0; it < PNP_REFINE_ITERS; ++it) {
    if (tid == 0) {
      double A[36], g[6], d[6];
      for (int i = 0; i < 36; ++i) A[i] = s_sys[i];
      for (int i = 0; i < 6; ++i) g[i] = s_sys[36 + i];
      const bool ok = pnp_solve6(A, g, lam, d);
      if (ok) {
        const PoseD cand = pnp_apply(P, d);
        for (int i = 0; i < 3; ++i) s_cand[i] = cand.t[i];
        for (int i = 0; i < 4; ++i) s_cand[3 + i] = cand.q[i];
      }
      s_cand[7] = ok ? 1.0 : 0.0;
    }
    __syncthreads();
    bool ok = s_cand[7] != 0.0;
    PoseD cand = P;
    if (ok) {
      cand = load_pose(s_cand);
      double cpart = 0.0;
      for (int k = tid; k < n; k += PNP_THREADS)
        if (sM[k]) cpart += pnp_err(cand, sX[k], sU[k]);
      const double cnew = block_sum(cpart, s_red);
      ok = isfinite(cnew) && cnew < s_sys[42];
    }
    __syncthreads();
    if (ok) { P = cand; normal_block(P); lam = fmax(lam * 0.1, 1e-9); }
    else lam = fmin(lam * 10.0, 1e6);
  }
  if (tid != 0) return;
  // ---- what compute_relative_pose does with the pose (:396-407) and the odometry check (:294-315) ----
  res->pnp_success = 1; res->n_inliers = best_cnt; res->winner = winner;
  for (int i = 0; i < 3; ++i) res->pose_cam[i] = P.t[i];
  for (int i = 0; i < 4; ++i) res->pose_cam[3 + i] = P.q[i];
  const PoseD p_cam_old_in_new = pose_inv(P);                               // PnPRestoCamPose
  const PoseD p_drone_old_in_new = pose_mul(p_cam_old_in_new, pose_inv(load_pose(prm.extrinsic)));
  const PoseD now = load_pose(prm.drone_pose_now), old = load_pose(prm.drone_pose_old);
  PoseD dp;
  double yaw;
  if (prm.is_4dof) {                                                        // DeltaPose(a, b, true): factors.hpp:139-149
    double ea[3], eb[3];
    quat2eulers(p_drone_old_in_new.q, ea); quat2eulers(now.q, eb);
    const double cs = cos(ea[2]), sn = sin(ea[2]);
    const double dx = now.t[0] - p_drone_old_in_new.t[0], dy = now.t[1] - p_drone_old_in_new.t[1];
    dp.t[0] = cs * dx + sn * dy; dp.t[1] = -sn * dx + cs * dy; dp.t[2] = now.t[2] - p_drone_old_in_new.t[2];
    double a = eb[2] - ea[2];
    a = a - 2.0 * M_PI * floor((a + M_PI) / (2.0 * M_PI));
    const double rv[3] = {0.0, 0.0, a};
    quat_from_rotvec(rv, dp.q);
  } else {
    dp = pose_mul(pose_inv(p_drone_old_in_new), now);
  }
  { double e[3]; quat2eulers(dp.q, e); yaw = e[2]; }
  res->dp_old_to_new[0] = dp.t[0]; res->dp_old_to_new[1] = dp.t[1]; res->dp_old_to_new[2] = dp.t[2]; res->dp_old_to_new[3] = yaw;
  double rperr;
  {                                                                         // RPerror (:338-351)
    const PoseD dp6 = pose_mul(pose_inv(p_drone_old_in_new), now);
    const PoseD predict = pose_mul(old, dp6);
    double qo[4] = {predict.q[0], predict.q[1], predict.q[2], predict.q[3]}, qn[4] = {now.q[0], now.q[1], now.q[2], now.q[3]};
    const double no = sqrt(qo[0] * qo[0] + qo[1] * qo[1] + qo[2] * qo[2] + qo[3] * qo[3]);
    const double nn = sqrt(qn[0] * qn[0] + qn[1] * qn[1] + qn[2] * qn[2] + qn[3] * qn[3]);
    for (int i = 0; i < 4; ++i) { qo[i] /= no; qn[i] /= nn; }
    double eo[3], en[3];
    quat2eulers(qo, eo); quat2eulers(qn, en);
    const double rv[3] = {0.0, 0.0, en[2] - eo[2]};
    double qz[4], qo2[4];
    quat_from_rotvec(rv, qz);
    q_mul(qz, qo, qo2);
    quat2eulers(qo2, eo);
    rperr = sqrt((eo[0] - en[0]) * (eo[0] - en[0]) + (eo[1] - en[1]) * (eo[1] - en[1]) + (eo[2] - en[2]) * (eo[2] - en[2]));
  }
  res->rperr = rperr;
  // rounded step by step, as oracle/pnp_ref.loop_distance: a contracted sum would make the distance check depend on which
  // fma order the compiler picks, not on the returned dp alone
  const double dist = sqrt(__dadd_rn(__dadd_rn(__dmul_rn(dp.t[0], dp.t[0]), __dmul_rn(dp.t[1], dp.t[1])), __dmul_rn(dp.t[2], dp.t[2])));
  res->verified = (rperr <= prm.rperr_thres && best_cnt >= prm.min_loop_num && fabs(yaw) < prm.accept_loop_yaw_rad &&
                   dist < prm.max_loop_dis) ? 1 : 0;                        // pnp_result_verify (:317-336)
  res->odometry_consistent = 1; res->md = 0.0;
  if (prm.same_drone) {                                                     // check_loop_odometry_consistency (:294-315)
    const PoseD d = pose_mul(pose_inv(dp), load_pose(prm.odom_rel));
    double v[6];
    pose_log(d, v);
    const double md = smd6(v, prm.odom_edge_cov);
    res->md = md;
    res->odometry_consistent = (md > prm.odometry_consistency_threshold) ? 0 : 1;
  }
}

}  // namespace osb

using namespace osb;

extern "C" osb_status osb_pnp_ransac_dev(const float* pts3d_dev, const float* pts2d_dev, const int32_t* n_dev, int n_cand,
                                         int max_n, const osb_pnp_params* params_dev, uint8_t* mask_dev,
                                         osb_pnp_result* results_dev, void* stream) {
  OSB_REQUIRE(pts3d_dev && pts2d_dev && n_dev && params_dev && mask_dev && results_dev, "null argument");
  OSB_REQUIRE(n_cand > 0 && max_n > 0 && max_n <= PNP_MAXN, "max_n must be in 1..1024");
  osb_status s = require_device();
  if (s != OSB_OK) return s;
  OSB_LAUNCH(pnp_ransac_kernel, n_cand, PNP_THREADS, 0, (cudaStream_t)stream, pts3d_dev, pts2d_dev, n_dev, max_n, params_dev,
             mask_dev, results_dev);
  OSB_CHECK_LAUNCH();
  return OSB_OK;
}

extern "C" osb_status osb_pnp_ransac(const float* pts3d, const float* pts2d, const int32_t* n, int n_cand, int max_n,
                                     const osb_pnp_params* params, uint8_t* mask, osb_pnp_result* results) {
  OSB_REQUIRE(pts3d && pts2d && n && params && mask && results, "null argument");
  OSB_REQUIRE(n_cand > 0 && max_n > 0 && max_n <= PNP_MAXN, "max_n must be in 1..1024");
  OSB_TRY(require_device());
  const size_t np = (size_t)n_cand * max_n;
  Resources res;
  float *d3 = nullptr, *d2 = nullptr;
  int32_t* dn = nullptr;
  osb_pnp_params* dp = nullptr;
  osb_pnp_result* dr = nullptr;
  uint8_t* dm = nullptr;
  OSB_TRY(res.upload(&d3, pts3d, np * 3));
  OSB_TRY(res.upload(&d2, pts2d, np * 2));
  OSB_TRY(res.upload(&dn, n, n_cand));
  OSB_TRY(res.upload(&dp, params, n_cand));
  OSB_TRY(res.alloc(&dr, n_cand));
  OSB_TRY(res.alloc(&dm, np));
  OSB_TRY(osb_pnp_ransac_dev(d3, d2, dn, n_cand, max_n, dp, dm, dr, nullptr));
  OSB_CUDA(cudaMemcpy(mask, dm, np, cudaMemcpyDeviceToHost));
  OSB_CUDA(cudaMemcpy(results, dr, n_cand * sizeof(osb_pnp_result), cudaMemcpyDeviceToHost));
  return OSB_OK;
}
