// geom.cu -- geometric filter of the loop matcher: homography-RANSAC inlier mask.
//
// Replaces cv::findHomography(old_2d, new_2d, CV_RANSAC, 3, mask) in LoopDetector::compute_correspond_features
// (swarm_loop/src/loop_detector.cpp:589-598) for the direction pairs of one keyframe.  OpenCV's RANSAC samples from cv::RNG
// and is not reproducible; the library defines a deterministic RANSAC with the same model (4-point homography), error
// (|new - H old|^2) and threshold (err <= thresh^2, the winner is the first hypothesis with the most inliers), stated in
// oracle/geometry_ref.py and pinned there against cv2.  This file is bit-exact against that statement: every floating-point
// operation is an explicitly rounded IEEE double operation (no fused multiply-add).  The 4-point model is built in
// closed form (projective basis), so a hypothesis costs ~150 register-resident flops.
#include <mutex>
#include <algorithm>
#include "common.cuh"
#include "kernels.cuh"

namespace osb {

constexpr int HG_HYP = 512;            // hypotheses per pair
constexpr int HG_THREADS = 256;
constexpr int HG_MAXN = 256;           // matches per pair (<= OSB_MAX_KPTS)

__host__ __device__ __forceinline__ uint32_t lowbias32(uint32_t x) {
  x ^= x >> 16; x *= 0x7FEB352Du; x ^= x >> 15; x *= 0x846CA68Bu; x ^= x >> 16;
  return x;
}

// 4 distinct match indices for hypothesis h (oracle: draw4)
__device__ bool hg_draw4(uint32_t seed, int h, int n, int (&idx)[4]) {
  for (int slot = 0; slot < 4; ++slot) {
    bool ok = false;
    for (int t = 0; t < 16 && !ok; ++t) {
      const int v = (int)(lowbias32(seed ^ lowbias32((uint32_t)((h * 4 + slot) * 16 + t) + 0x9E3779B9u)) % (uint32_t)n);
      bool dup = false;
      for (int j = 0; j < slot; ++j) dup |= (idx[j] == v);
      if (!dup) { idx[slot] = v; ok = true; }
    }
    if (!ok) return false;
  }
  return true;
}

// Projective-basis construction of the 4-point homography (closed form, branch-free, registers only):
//   frame(p1..p4) = [p1 p2 p3] diag(v),  v = adj([p1 p2 p3]) p4   (p_i homogeneous; any scale of v serves)
//   H = frame(dst) adj(frame(src))       (unnormalised: the inlier test is homogeneous in H)
// A sample is degenerate when one of the four triangles of a quadruple has twice-area <= 1 px^2.
struct HgFrame { double m[9]; bool ok; };

__device__ __forceinline__ HgFrame hg_frame(float2 q1, float2 q2, float2 q3, float2 q4) {
  const double x1 = q1.x, y1 = q1.y, x2 = q2.x, y2 = q2.y, x3 = q3.x, y3 = q3.y, x4 = q4.x, y4 = q4.y;
  const double a00 = __dsub_rn(y2, y3), a01 = __dsub_rn(x3, x2), a02 = __dsub_rn(__dmul_rn(x2, y3), __dmul_rn(x3, y2));
  const double a10 = __dsub_rn(y3, y1), a11 = __dsub_rn(x1, x3), a12 = __dsub_rn(__dmul_rn(x3, y1), __dmul_rn(x1, y3));
  const double a20 = __dsub_rn(y1, y2), a21 = __dsub_rn(x2, x1), a22 = __dsub_rn(__dmul_rn(x1, y2), __dmul_rn(x2, y1));
  const double det = __dadd_rn(__dadd_rn(a02, a12), a22);
  const double v0 = __dadd_rn(__dadd_rn(__dmul_rn(a00, x4), __dmul_rn(a01, y4)), a02);
  const double v1 = __dadd_rn(__dadd_rn(__dmul_rn(a10, x4), __dmul_rn(a11, y4)), a12);
  const double v2 = __dadd_rn(__dadd_rn(__dmul_rn(a20, x4), __dmul_rn(a21, y4)), a22);
  HgFrame f;
  f.ok = fabs(det) > 1.0 && fabs(v0) > 1.0 && fabs(v1) > 1.0 && fabs(v2) > 1.0;
  f.m[0] = __dmul_rn(x1, v0); f.m[1] = __dmul_rn(x2, v1); f.m[2] = __dmul_rn(x3, v2);
  f.m[3] = __dmul_rn(y1, v0); f.m[4] = __dmul_rn(y2, v1); f.m[5] = __dmul_rn(y3, v2);
  f.m[6] = v0; f.m[7] = v1; f.m[8] = v2;
  return f;
}

__device__ bool hg_solve(const float2* __restrict__ src, const float2* __restrict__ dst, const int (&idx)[4], double (&h)[9]) {
  const HgFrame A = hg_frame(src[idx[0]], src[idx[1]], src[idx[2]], src[idx[3]]);
  const HgFrame B = hg_frame(dst[idx[0]], dst[idx[1]], dst[idx[2]], dst[idx[3]]);
  if (!(A.ok && B.ok)) return false;
  const double* a = A.m;
  double c[9];                                         // adj(A), row-major
  c[0] = __dsub_rn(__dmul_rn(a[4], a[8]), __dmul_rn(a[5], a[7]));
  c[1] = __dsub_rn(__dmul_rn(a[2], a[7]), __dmul_rn(a[1], a[8]));
  c[2] = __dsub_rn(__dmul_rn(a[1], a[5]), __dmul_rn(a[2], a[4]));
  c[3] = __dsub_rn(__dmul_rn(a[5], a[6]), __dmul_rn(a[3], a[8]));
  c[4] = __dsub_rn(__dmul_rn(a[0], a[8]), __dmul_rn(a[2], a[6]));
  c[5] = __dsub_rn(__dmul_rn(a[2], a[3]), __dmul_rn(a[0], a[5]));
  c[6] = __dsub_rn(__dmul_rn(a[3], a[7]), __dmul_rn(a[4], a[6]));
  c[7] = __dsub_rn(__dmul_rn(a[1], a[6]), __dmul_rn(a[0], a[7]));
  c[8] = __dsub_rn(__dmul_rn(a[0], a[4]), __dmul_rn(a[1], a[3]));
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j)
      h[i * 3 + j] = __dadd_rn(__dadd_rn(__dmul_rn(B.m[i * 3], c[j]), __dmul_rn(B.m[i * 3 + 1], c[3 + j])),
                               __dmul_rn(B.m[i * 3 + 2], c[6 + j]));
  return true;
}

// |new - H old|^2 <= thresh^2 written without the division: with (px, py, w) = H (x, y, 1),
//   (u w - px)^2 + (v w - py)^2 <= thresh^2 w^2        (w = 0 makes the right side 0: such a point is never an inlier
// unless it maps exactly, as in the divided form)
__device__ __forceinline__ bool hg_inlier(const double (&h)[9], float2 s, float2 d, double t2) {
  const double x = s.x, y = s.y;
  const double w = __dadd_rn(__dadd_rn(__dmul_rn(h[6], x), __dmul_rn(h[7], y)), h[8]);
  const double px = __dadd_rn(__dadd_rn(__dmul_rn(h[0], x), __dmul_rn(h[1], y)), h[2]);
  const double py = __dadd_rn(__dadd_rn(__dmul_rn(h[3], x), __dmul_rn(h[4], y)), h[5]);
  const double ex = __dsub_rn(__dmul_rn((double)d.x, w), px), ey = __dsub_rn(__dmul_rn((double)d.y, w), py);
  return __dadd_rn(__dmul_rn(ex, ex), __dmul_rn(ey, ey)) <= __dmul_rn(t2, __dmul_rn(w, w));
}

// HG_SPLIT CTAs per pair (fp64 scoring is bound by one SM's fp64 pipe: 512 x 200 inlier tests).  src / dst:
// [n_pairs][max_n] float2 (old_2d / new_2d of the flagged matches, in match order).
// Phase A: the CTA's 64 hypotheses are solved by its first 64 threads (model -> shared memory).  Phase B: a warp scores
// one hypothesis at a time, its lanes splitting the matches; the count goes into the pair's global atomicMax key
// (inliers, -hypothesis).  Phase C: the last CTA of the pair to finish (ticket) rebuilds the winner and writes the mask.
constexpr int HG_SPLIT = 8;
constexpr int HG_PER_CTA = HG_HYP / HG_SPLIT;
__global__ void __launch_bounds__(HG_THREADS)
homography_ransac_kernel(const float2* __restrict__ src, const float2* __restrict__ dst, const int32_t* __restrict__ n_pts,
                         int max_n, float thresh, uint32_t seed, uint8_t* __restrict__ mask, int32_t* __restrict__ n_inl,
                         int32_t* __restrict__ winner, unsigned int* __restrict__ g_key, unsigned int* __restrict__ g_ticket) {
  __shared__ float2 s_src[HG_MAXN], s_dst[HG_MAXN];
  __shared__ double s_h[HG_PER_CTA][9];
  __shared__ unsigned char s_ok[HG_PER_CTA];
  __shared__ int s_last;
  const int pair = blockIdx.x, part = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int n = min(n_pts[pair], min(max_n, HG_MAXN));
  uint8_t* mk = mask + (size_t)pair * max_n;
  if (n < 4) {                                         // the reference rejects the pair (loop_detector.cpp:598-600)
    if (part == 0) {
      for (int i = tid; i < max_n; i += HG_THREADS) mk[i] = 0;
      if (tid == 0) { n_inl[pair] = 0; winner[pair] = -1; }
    }
    return;
  }
  for (int i = tid; i < n; i += HG_THREADS) { s_src[i] = src[(size_t)pair * max_n + i]; s_dst[i] = dst[(size_t)pair * max_n + i]; }
  __syncthreads();
  const double t2 = __dmul_rn((double)thresh, (double)thresh);
  const int h0 = part * HG_PER_CTA;
  if (tid < HG_PER_CTA) {
    int idx[4];
    double h[9];
    const bool ok = hg_draw4(seed, h0 + tid, n, idx) && hg_solve(s_src, s_dst, idx, h);
    s_ok[tid] = ok ? 1 : 0;
    if (ok)
      for (int k = 0; k < 9; ++k) s_h[tid][k] = h[k];
  }
  __syncthreads();
  for (int j = warp; j < HG_PER_CTA; j += HG_THREADS / 32) {
    if (!s_ok[j]) continue;                            // warp-uniform
    double h[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) h[k] = s_h[j][k];
    int c = 0;
    for (int i = lane; i < n; i += 32) c += hg_inlier(h, s_src[i], s_dst[i], t2) ? 1 : 0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    // most inliers, then the smaller hypothesis index: key = (count + 1) << 16 | (0xFFFF - hyp)
    if (lane == 0) atomicMax(&g_key[pair], ((unsigned)(c + 1) << 16) | (unsigned)(0xFFFF - (h0 + j)));
  }
  __threadfence();
  __syncthreads();
  if (tid == 0) s_last = (atomicAdd(&g_ticket[pair], 1u) == HG_SPLIT - 1);
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  const unsigned best = *reinterpret_cast<volatile unsigned int*>(&g_key[pair]);
  __syncthreads();
  if (tid == 0) { g_key[pair] = 0u; g_ticket[pair] = 0u; }      // ready for the next launch on this scratch
  if (best == 0u) {                                    // every hypothesis degenerate
    for (int i = tid; i < max_n; i += HG_THREADS) mk[i] = 0;
    if (tid == 0) { n_inl[pair] = 0; winner[pair] = -1; }
    return;
  }
  const int hw = 0xFFFF - (int)(best & 0xFFFFu);
  int idx[4];
  double h[9];
  hg_draw4(seed, hw, n, idx);                          // identical arithmetic: every thread rebuilds the winner
  hg_solve(s_src, s_dst, idx, h);
  for (int i = tid; i < max_n; i += HG_THREADS) mk[i] = (i < n && hg_inlier(h, s_src[i], s_dst[i], t2)) ? 1 : 0;
  if (tid == 0) { n_inl[pair] = (int)(best >> 16) - 1; winner[pair] = hw; }
}

osb_status homography_ransac_device(const float* src_dev, const float* dst_dev, const int32_t* n_dev, int n_pairs, int max_n,
                                    float thresh, uint32_t seed, uint8_t* mask_dev, int32_t* n_inl_dev, int32_t* winner_dev,
                                    cudaStream_t st, unsigned int* scratch) {
  if (n_pairs <= 0) return OSB_OK;
  OSB_REQUIRE(max_n > 0 && max_n <= HG_MAXN, "homography: max_n out of range (1..256)");
  OSB_REQUIRE(scratch != nullptr, "homography: no scratch");
  OSB_LAUNCH(homography_ransac_kernel, dim3(n_pairs, HG_SPLIT), HG_THREADS, 0, st, reinterpret_cast<const float2*>(src_dev),
             reinterpret_cast<const float2*>(dst_dev), n_dev, max_n, thresh, seed, mask_dev, n_inl_dev, winner_dev, scratch,
             scratch + n_pairs);
  OSB_CHECK_LAUNCH();
  return OSB_OK;
}

}  // namespace osb

using namespace osb;

extern "C" osb_status osb_homography_ransac_dev(const float* src_dev, const float* dst_dev, const int32_t* n_dev,
                                                int n_pairs, int max_n, float thresh, uint32_t seed, uint8_t* mask_dev,
                                                int32_t* n_inliers_dev, int32_t* winner_dev, void* stream) {
  OSB_REQUIRE(src_dev && dst_dev && n_dev && mask_dev && n_inliers_dev && winner_dev, "null argument");
  osb_status s = require_device();
  if (s != OSB_OK) return s;
  // per-call scratch (key + ticket per pair) from the stream-ordered allocator: no process-wide state, no synchronisation,
  // safe for concurrent callers on different streams (the reference's nodelet is multi-threaded)
  cudaStream_t st = (cudaStream_t)stream;
  unsigned int* scratch = nullptr;
  OSB_CUDA(cudaMallocAsync(&scratch, 2 * (size_t)n_pairs * sizeof(unsigned int), st));
  const cudaError_t e = cudaMemsetAsync(scratch, 0, 2 * (size_t)n_pairs * sizeof(unsigned int), st);
  if (e == cudaSuccess)
    s = homography_ransac_device(src_dev, dst_dev, n_dev, n_pairs, max_n, thresh, seed, mask_dev, n_inliers_dev, winner_dev,
                                 st, scratch);
  cudaFreeAsync(scratch, st);
  OSB_CUDA(e);
  return s;
}

// host buffers in / out (allocates its scratch per call: a convenience for tests and small callers)
extern "C" osb_status osb_homography_ransac(const float* src, const float* dst, const int32_t* n, int n_pairs, int max_n,
                                            float thresh, uint32_t seed, uint8_t* mask, int32_t* n_inliers,
                                            int32_t* winner) {
  OSB_REQUIRE(src && dst && n && mask && n_inliers && n_pairs > 0 && max_n > 0, "bad argument");
  OSB_TRY(require_device());
  const size_t pts = (size_t)n_pairs * max_n;
  Resources res;
  float *d_src = nullptr, *d_dst = nullptr;
  unsigned int* d_scratch = nullptr;
  int32_t *d_n = nullptr, *d_inl = nullptr, *d_win = nullptr;
  uint8_t* d_mask = nullptr;
  OSB_TRY(res.upload(&d_src, src, pts * 2));
  OSB_TRY(res.upload(&d_dst, dst, pts * 2));
  OSB_TRY(res.upload(&d_n, n, n_pairs));
  OSB_TRY(res.alloc(&d_inl, n_pairs));
  OSB_TRY(res.alloc(&d_win, n_pairs));
  OSB_TRY(res.alloc(&d_mask, pts));
  OSB_TRY(res.alloc(&d_scratch, 2 * (size_t)n_pairs));
  OSB_CUDA(cudaMemset(d_scratch, 0, 2 * (size_t)n_pairs * sizeof(unsigned int)));
  OSB_TRY(homography_ransac_device(d_src, d_dst, d_n, n_pairs, max_n, thresh, seed, d_mask, d_inl, d_win, nullptr, d_scratch));
  OSB_CUDA(cudaMemcpy(mask, d_mask, pts, cudaMemcpyDeviceToHost));
  OSB_CUDA(cudaMemcpy(n_inliers, d_inl, n_pairs * sizeof(int32_t), cudaMemcpyDeviceToHost));
  if (winner) OSB_CUDA(cudaMemcpy(winner, d_win, n_pairs * sizeof(int32_t), cudaMemcpyDeviceToHost));
  return OSB_OK;
}
