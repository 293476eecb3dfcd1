// lift.cu -- keypoints -> 3-D landmarks + landmarks_flag on the device (SURVEY.md section 8f-3).
//
// Replaces the per-keypoint loops of LoopCam::generate_stereo_image_descriptor (swarm_loop/src/loop_cam.cpp:393-432:
// liftProjective, triangulatePoint :73-106, err <= TRIANGLE_THRES and in-front test) and of
// generate_gray_depth_image_descriptor (:276-302: depth look-up, DEPTH_NEAR_THRES < dep < DEPTH_FAR_THRES, lift through
// pose_cam).  With them the keyframe record carries the reference's own landmarks_3d / landmarks_flag -- the flag the loop
// matcher's geometric filter tests (loop_detector.cpp:574) and the 3-D points the PnP stage consumes.
// The flattened virtual cameras are distortion-free pinholes: liftProjective(x, y) = ((x - cx)/fx, (y - cy)/fy, 1).
// triangulatePoint's 4x4 SVD becomes the smallest eigenvector of D^T D by cyclic Jacobi rotations (fp64, one thread per
// keypoint); the 3-D point is a ratio of its components, so it equals Eigen's JacobiSVD result to rounding.
#include "common.cuh"
#include "kernels.cuh"
#include "pose_algebra.cuh"

namespace osb {

// smallest eigenvector of the symmetric 4x4 S (cyclic Jacobi, 10 sweeps)
__device__ void smallest_eigvec4(double (&S)[4][4], double (&v)[4]) {
  double V[4][4] = {{1, 0, 0, 0}, {0, 1, 0, 0}, {0, 0, 1, 0}, {0, 0, 0, 1}};
  for (int sweep = 0; sweep < 10; ++sweep) {
    for (int p = 0; p < 3; ++p)
      for (int q = p + 1; q < 4; ++q) {
        const double apq = S[p][q];
        if (fabs(apq) < 1e-300) continue;
        const double theta = (S[q][q] - S[p][p]) / (2.0 * apq);
        const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < 4; ++k) {                    // S <- J^T S J
          const double skp = S[k][p], skq = S[k][q];
          S[k][p] = c * skp - s * skq; S[k][q] = s * skp + c * skq;
        }
        for (int k = 0; k < 4; ++k) {
          const double spk = S[p][k], sqk = S[q][k];
          S[p][k] = c * spk - s * sqk; S[q][k] = s * spk + c * sqk;
        }
        for (int k = 0; k < 4; ++k) {
          const double vkp = V[k][p], vkq = V[k][q];
          V[k][p] = c * vkp - s * vkq; V[k][q] = s * vkp + c * vkq;
        }
      }
  }
  int m = 0;
  for (int i = 1; i < 4; ++i) if (S[i][i] < S[m][m]) m = i;
  for (int k = 0; k < 4; ++k) v[k] = V[k][m];
}

__device__ __forceinline__ void rot_rows(const double* q, double (&R)[3][3]) {    // R[i][j] = (R e_j)_i
  const double e[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
  for (int j = 0; j < 3; ++j) {
    double c[3];
    q_rot(q, e[j], c);
    R[0][j] = c[0]; R[1][j] = c[1]; R[2][j] = c[2];
  }
}

struct LiftCam { double fx, fy, cx, cy; };

// one thread per up keypoint of one direction.  DOWN (LOWER_CAM_AS_MAIN): the 3-D point goes to the down keypoint's slot,
// as ides_down.landmarks_3d[idx_down] (loop_cam.cpp:443-444); the in-front test stays on the up camera (:418-425).  The
// slots of unflagged down keypoints are left as they are (each slot has at most one writer, the thread of its up partner,
// so there is nothing to clear them without a race): read pts3d only where flag_down is set.
template <bool DOWN>
__global__ void stereo_lift_kernel(const float* __restrict__ kp_up, const float* __restrict__ kp_down,
                                   const int32_t* __restrict__ match, const int32_t* __restrict__ n_up,
                                   const int32_t* __restrict__ n_down, int max_n, LiftCam cam,
                                   const double* __restrict__ pose_up, const double* __restrict__ pose_down,
                                   double triangle_thres, int min_pts, float* __restrict__ pts3d, uint8_t* __restrict__ flag_up,
                                   uint8_t* __restrict__ flag_down) {
  const int d = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= max_n) return;
  const size_t o = (size_t)d * max_n + i;
  if (!DOWN) { pts3d[o * 3] = 0.f; pts3d[o * 3 + 1] = 0.f; pts3d[o * 3 + 2] = 0.f; }
  flag_up[o] = 0;
  // (flag_down is cleared by the caller: several up keypoints never share a down keypoint -- the match is one-to-one)
  const int nu = n_up[d];
  if (i >= nu || nu <= min_pts) return;                  // the stereo stage is skipped for sparse images (:385-391)
  const int j = match[o];
  if (j < 0 || j >= n_down[d]) return;
  const double a0 = ((double)kp_up[o * 2] - cam.cx) / cam.fx, a1 = ((double)kp_up[o * 2 + 1] - cam.cy) / cam.fy;
  const size_t oj = (size_t)d * max_n + j;
  const double b0 = ((double)kp_down[oj * 2] - cam.cx) / cam.fx, b1 = ((double)kp_down[oj * 2 + 1] - cam.cy) / cam.fy;
  const double* pu = pose_up + d * 7;
  const double* pd = pose_down + d * 7;
  double R0[3][3], R1[3][3];
  rot_rows(pu + 3, R0); rot_rows(pd + 3, R1);
  // Pose = [R^T | -R^T t]
  double P0[3][4], P1[3][4];
  for (int r = 0; r < 3; ++r) {
    P0[r][0] = R0[0][r]; P0[r][1] = R0[1][r]; P0[r][2] = R0[2][r];
    P0[r][3] = -(R0[0][r] * pu[0] + R0[1][r] * pu[1] + R0[2][r] * pu[2]);
    P1[r][0] = R1[0][r]; P1[r][1] = R1[1][r]; P1[r][2] = R1[2][r];
    P1[r][3] = -(R1[0][r] * pd[0] + R1[1][r] * pd[1] + R1[2][r] * pd[2]);
  }
  double D[4][4];
  for (int k = 0; k < 4; ++k) {
    D[0][k] = a0 * P0[2][k] - P0[0][k];
    D[1][k] = a1 * P0[2][k] - P0[1][k];
    D[2][k] = b0 * P1[2][k] - P1[0][k];
    D[3][k] = b1 * P1[2][k] - P1[1][k];
  }
  double S[4][4], v[4];
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 4; ++c) {
      double s = 0.0;
      for (int k = 0; k < 4; ++k) s += D[k][r] * D[k][c];
      S[r][c] = s;
    }
  smallest_eigvec4(S, v);
  const double p[3] = {v[0] / v[3], v[1] / v[3], v[2] / v[3]};
  double e2 = 0.0;
  for (int r = 0; r < 4; ++r) {
    const double e = D[r][0] * p[0] + D[r][1] * p[1] + D[r][2] * p[2] + D[r][3];
    e2 += e * e;
  }
  const double err = sqrt(e2) / 4.0;
  // in front of the up camera: (R0^T (p - t0)).z
  const double zc = R0[0][2] * (p[0] - pu[0]) + R0[1][2] * (p[1] - pu[1]) + R0[2][2] * (p[2] - pu[2]);
  if (err > triangle_thres || zc < 0.0 || !(isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]))) return;
  const size_t op = DOWN ? oj : o;
  pts3d[op * 3] = (float)p[0]; pts3d[op * 3 + 1] = (float)p[1]; pts3d[op * 3 + 2] = (float)p[2];
  flag_up[o] = 1;
  flag_down[oj] = 1;
}

__global__ void depth_lift_kernel(const float* __restrict__ kp, const int32_t* __restrict__ n_kp, int max_n,
                                  const uint16_t* __restrict__ depth_mm, int H, int W, LiftCam cam,
                                  const double* __restrict__ pose_cam, double near_thres, double far_thres, int min_pts,
                                  float* __restrict__ pts3d, uint8_t* __restrict__ flag) {
  const int d = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= max_n) return;
  const size_t o = (size_t)d * max_n + i;
  pts3d[o * 3] = 0.f; pts3d[o * 3 + 1] = 0.f; pts3d[o * 3 + 2] = 0.f;
  flag[o] = 0;
  const int n = n_kp[d];
  if (i >= n || n <= min_pts) return;
  const double x = kp[o * 2], y = kp[o * 2 + 1];
  if (x < 0 || x > W || y < 0 || y > H) return;            // :282 (the reference hard-codes 640 x 480)
  const int xi = (int)rint(x), yi = (int)rint(y);          // cv::Mat::at(Point2f -> Point) rounds
  if (xi >= W || yi >= H) return;
  const double dep = depth_mm[((size_t)d * H + yi) * W + xi] / 1000.0;
  if (!(dep > near_thres && dep < far_thres)) return;
  const double ray[3] = {(x - cam.cx) / cam.fx * dep, (y - cam.cy) / cam.fy * dep, dep};
  double r[3];
  q_rot(pose_cam + d * 7 + 3, ray, r);
  pts3d[o * 3] = (float)(r[0] + pose_cam[d * 7]); pts3d[o * 3 + 1] = (float)(r[1] + pose_cam[d * 7 + 1]);
  pts3d[o * 3 + 2] = (float)(r[2] + pose_cam[d * 7 + 2]);
  flag[o] = 1;
}

osb_status stereo_lift_device(const float* kp_up, const float* kp_down, const int32_t* match, const int32_t* n_up,
                              const int32_t* n_down, int n_dirs, int max_n, const double* K, const double* pose_up,
                              const double* pose_down, double triangle_thres, int min_pts, float* pts3d, uint8_t* flag_up,
                              uint8_t* flag_down, cudaStream_t st, bool down_main) {
  OSB_CUDA(cudaMemsetAsync(flag_down, 0, (size_t)n_dirs * max_n, st));
  const LiftCam cam{K[0], K[1], K[2], K[3]};
  if (down_main)
    OSB_LAUNCH(stereo_lift_kernel<true>, dim3(cdiv(max_n, 64), n_dirs), 64, 0, st, kp_up, kp_down, match, n_up, n_down, max_n,
               cam, pose_up, pose_down, triangle_thres, min_pts, pts3d, flag_up, flag_down);
  else
    OSB_LAUNCH(stereo_lift_kernel<false>, dim3(cdiv(max_n, 64), n_dirs), 64, 0, st, kp_up, kp_down, match, n_up, n_down, max_n,
               cam, pose_up, pose_down, triangle_thres, min_pts, pts3d, flag_up, flag_down);
  OSB_CHECK_LAUNCH();
  return OSB_OK;
}

osb_status depth_lift_device(const float* kp, const int32_t* n_kp, int n_dirs, int max_n, const uint16_t* depth_mm, int H,
                             int W, const double* K, const double* pose_cam, double near_thres, double far_thres,
                             int min_pts, float* pts3d, uint8_t* flag, cudaStream_t st) {
  const LiftCam cam{K[0], K[1], K[2], K[3]};
  OSB_LAUNCH(depth_lift_kernel, dim3(cdiv(max_n, 64), n_dirs), 64, 0, st, kp, n_kp, max_n, depth_mm, H, W, cam, pose_cam,
             near_thres, far_thres, min_pts, pts3d, flag);
  OSB_CHECK_LAUNCH();
  return OSB_OK;
}

}  // namespace osb

using namespace osb;

extern "C" osb_status osb_stereo_lift_dev(const float* kp_up_dev, const float* kp_down_dev, const int32_t* stereo_match_dev,
                                          const int32_t* n_up_dev, const int32_t* n_down_dev, int n_dirs, int max_n,
                                          const double* intrinsics /*host [4]*/, const double* pose_up_dev,
                                          const double* pose_down_dev, double triangle_thres, int accept_min_3d_pts,
                                          float* pts3d_dev, uint8_t* flag_up_dev, uint8_t* flag_down_dev, void* stream) {
  OSB_REQUIRE(kp_up_dev && kp_down_dev && stereo_match_dev && n_up_dev && n_down_dev && intrinsics && pose_up_dev &&
              pose_down_dev && pts3d_dev && flag_up_dev && flag_down_dev, "null argument");
  OSB_REQUIRE(n_dirs > 0 && max_n > 0, "bad sizes");
  osb_status s = require_device();
  if (s != OSB_OK) return s;
  return stereo_lift_device(kp_up_dev, kp_down_dev, stereo_match_dev, n_up_dev, n_down_dev, n_dirs, max_n, intrinsics,
                            pose_up_dev, pose_down_dev, triangle_thres, accept_min_3d_pts, pts3d_dev, flag_up_dev,
                            flag_down_dev, (cudaStream_t)stream);
}

extern "C" osb_status osb_depth_lift_dev(const float* kp_dev, const int32_t* n_dev, int n_dirs, int max_n,
                                         const uint16_t* depth_mm_dev, int height, int width, const double* intrinsics,
                                         const double* pose_cam_dev, double near_thres, double far_thres,
                                         int accept_min_3d_pts, float* pts3d_dev, uint8_t* flag_dev, void* stream) {
  OSB_REQUIRE(kp_dev && n_dev && depth_mm_dev && intrinsics && pose_cam_dev && pts3d_dev && flag_dev, "null argument");
  OSB_REQUIRE(n_dirs > 0 && max_n > 0 && height > 0 && width > 0, "bad sizes");
  osb_status s = require_device();
  if (s != OSB_OK) return s;
  return depth_lift_device(kp_dev, n_dev, n_dirs, max_n, depth_mm_dev, height, width, intrinsics, pose_cam_dev, near_thres,
                           far_thres, accept_min_3d_pts, pts3d_dev, flag_dev, (cudaStream_t)stream);
}

// host-buffer convenience forms (tests, small callers)
extern "C" osb_status osb_stereo_lift(const float* kp_up, const float* kp_down, const int32_t* stereo_match, const int32_t* n_up,
                                      const int32_t* n_down, int n_dirs, int max_n, const double* intrinsics,
                                      const double* pose_up, const double* pose_down, double triangle_thres,
                                      int accept_min_3d_pts, float* pts3d, uint8_t* flag_up, uint8_t* flag_down) {
  OSB_REQUIRE(kp_up && kp_down && stereo_match && n_up && n_down && intrinsics && pose_up && pose_down && pts3d && flag_up &&
              flag_down, "null argument");
  OSB_TRY(require_device());
  const size_t np = (size_t)n_dirs * max_n;
  Resources res;
  float *d_u = nullptr, *d_d = nullptr, *d_p = nullptr;
  int32_t *d_m = nullptr, *d_nu = nullptr, *d_nd = nullptr;
  double *d_pu = nullptr, *d_pd = nullptr;
  uint8_t *d_fu = nullptr, *d_fd = nullptr;
  OSB_TRY(res.upload(&d_u, kp_up, np * 2));
  OSB_TRY(res.upload(&d_d, kp_down, np * 2));
  OSB_TRY(res.alloc(&d_p, np * 3));
  OSB_TRY(res.upload(&d_m, stereo_match, np));
  OSB_TRY(res.upload(&d_nu, n_up, n_dirs));
  OSB_TRY(res.upload(&d_nd, n_down, n_dirs));
  OSB_TRY(res.upload(&d_pu, pose_up, n_dirs * 7));
  OSB_TRY(res.upload(&d_pd, pose_down, n_dirs * 7));
  OSB_TRY(res.alloc(&d_fu, np));
  OSB_TRY(res.alloc(&d_fd, np));
  OSB_TRY(osb_stereo_lift_dev(d_u, d_d, d_m, d_nu, d_nd, n_dirs, max_n, intrinsics, d_pu, d_pd, triangle_thres,
                              accept_min_3d_pts, d_p, d_fu, d_fd, nullptr));
  OSB_CUDA(cudaMemcpy(pts3d, d_p, np * 3 * sizeof(float), cudaMemcpyDeviceToHost));
  OSB_CUDA(cudaMemcpy(flag_up, d_fu, np, cudaMemcpyDeviceToHost));
  OSB_CUDA(cudaMemcpy(flag_down, d_fd, np, cudaMemcpyDeviceToHost));
  return OSB_OK;
}

extern "C" osb_status osb_depth_lift(const float* kp, const int32_t* n, int n_dirs, int max_n, const uint16_t* depth_mm,
                                     int height, int width, const double* intrinsics, const double* pose_cam, double near_thres,
                                     double far_thres, int accept_min_3d_pts, float* pts3d, uint8_t* flag) {
  OSB_REQUIRE(kp && n && depth_mm && intrinsics && pose_cam && pts3d && flag, "null argument");
  OSB_TRY(require_device());
  const size_t np = (size_t)n_dirs * max_n, nd = (size_t)n_dirs * height * width;
  Resources res;
  float *d_k = nullptr, *d_p = nullptr;
  int32_t* d_n = nullptr;
  uint16_t* d_dep = nullptr;
  double* d_pc = nullptr;
  uint8_t* d_f = nullptr;
  OSB_TRY(res.upload(&d_k, kp, np * 2));
  OSB_TRY(res.alloc(&d_p, np * 3));
  OSB_TRY(res.upload(&d_n, n, n_dirs));
  OSB_TRY(res.upload(&d_dep, depth_mm, nd));
  OSB_TRY(res.upload(&d_pc, pose_cam, n_dirs * 7));
  OSB_TRY(res.alloc(&d_f, np));
  OSB_TRY(osb_depth_lift_dev(d_k, d_n, n_dirs, max_n, d_dep, height, width, intrinsics, d_pc, near_thres, far_thres,
                             accept_min_3d_pts, d_p, d_f, nullptr));
  OSB_CUDA(cudaMemcpy(pts3d, d_p, np * 3 * sizeof(float), cudaMemcpyDeviceToHost));
  OSB_CUDA(cudaMemcpy(flag, d_f, np, cudaMemcpyDeviceToHost));
  return OSB_OK;
}
