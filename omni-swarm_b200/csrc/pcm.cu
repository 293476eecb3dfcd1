// pcm.cu -- pairwise-consistency (PCM) outlier rejection of the loop edges of one drone pair, on the device.
//
// Replaces SwarmLocalOutlierRejection::OutlierRejectionLoopEdgesPCM
// (swarm_localization/src/swarm_outlier_rejection/swarm_outlier_rejection.cpp:173-297 of the reference), the stage
// immediately upstream of the pose-graph solve (SURVEY.md section 8f-2):
//   1. pcm_consistency_kernel -- for every pair of loops: err = odom_a * p_edge2 * odom_b^-1 * p_edge1^-1 (:227), its 6-D
//      log map (:228) and the squared Mahalanobis distance against cov_1 + cov_2 + cov(odom_a) + cov(odom_b)
//      (:193,212,224,229); consistency-graph edge iff smd < pcm_thres (:231-235).  O(L^2) independent fp64 evaluations:
//      one thread per (row, 32-column word) writes one word of the adjacency BIT matrix -- no atomics, each unordered pair
//      is evaluated from both rows with the same (edge1 = later loop, edge2 = earlier loop) roles, so the matrix is symmetric
//      by construction.
//   2. pcm_max_clique_kernel -- FMC::maxCliqueHeu (third_party/fast_max-clique_finder/src/findCliqueHeu.cpp:120-244),
//      literally: candidates in index order with prunings 1/3/5, S shrunk by the adjacency of its LAST element (:185).  The
//      candidate loop is sequential by definition (maxClq feeds the prunings), so ONE warp runs it with S, the degree mask
//      and the adjacency rows as bitsets: an iteration is "highest set bit" + a 128-bit AND per lane, warp shuffles only.
// Swarm::Pose / log_map / get_covariance / get_relative_pose_by_ts come from HKUST-Swarm/swarm_msgs, which is not in the
// reference tree: they are defined in oracle/pcm_ref.py and restated here (covariances and ego-motion poses are inputs).
#include "common.cuh"
#include "kernels.cuh"
#include "pose_algebra.cuh"

namespace osb {

constexpr int PCM_MAX_N = 4096;
constexpr int PCM_MAX_W = PCM_MAX_N / 32;

// squared Mahalanobis consistency error of (e1 = the LATER loop, e2 = the earlier one); +inf for another drone pair
__device__ double pcm_pair_smd(const osb_loop_edge* __restrict__ e1, const osb_loop_edge* __restrict__ e2, double pos_cov,
                               double ang_cov) {
  int srp = 0;                                                      // LoopEdge::same_robot_pair
  if (e1->id_a == e2->id_a && e1->id_b == e2->id_b) srp = 1;
  else if (e1->id_a == e2->id_b && e1->id_b == e2->id_a) srp = 2;
  if (srp == 0) return INFINITY;
  PoseD p2 = load_pose(e2->rel_pose);
  const double *a2 = e2->odom_a, *b2 = e2->odom_b;
  double la2 = e2->len_a, lb2 = e2->len_b;
  if (srp == 2) {                                                   // edge2 runs b -> a (:214-224)
    p2 = pose_inv(p2);
    a2 = e2->odom_b; b2 = e2->odom_a; la2 = e2->len_b; lb2 = e2->len_a;
  }
  const PoseD odom_a = pose_mul(pose_inv(load_pose(e1->odom_a)), load_pose(a2));
  const PoseD odom_b = pose_mul(pose_inv(load_pose(e1->odom_b)), load_pose(b2));
  const double dl = fabs(la2 - e1->len_a) + fabs(lb2 - e1->len_b);
  const PoseD err = pose_mul(pose_mul(pose_mul(odom_a, p2), pose_inv(odom_b)), pose_inv(load_pose(e1->rel_pose)));   // :227
  double v[6];
  pose_log(err, v);
  // C = cov_1 + cov_2 + (|dlen_a| + |dlen_b|) * diag(pos x3, ang x3); smd = v^T C^-1 v by an unpivoted Cholesky
  double C[36];
#pragma unroll
  for (int i = 0; i < 36; ++i) C[i] = e1->cov[i] + e2->cov[i];
#pragma unroll
  for (int j = 0; j < 6; ++j) C[j * 6 + j] += dl * (j < 3 ? pos_cov : ang_cov);
  return smd6(v, C);
}

// adjacency bit matrix: thread = (row i, word w) -> bits of columns 32w .. 32w+31
__global__ void __launch_bounds__(128)
pcm_consistency_kernel(const osb_loop_edge* __restrict__ edges, int n, int W, double thres, double pos_cov, double ang_cov,
                       uint32_t* __restrict__ bits /*[n][W]*/, double* __restrict__ smd_out /*[n][n] or null*/) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * W) return;
  const int i = idx / W, w = idx - i * W;
  uint32_t word = 0;
  for (int b = 0; b < 32; ++b) {
    const int j = w * 32 + b;
    if (j >= n) break;
    double smd = INFINITY;
    if (j != i) smd = (i > j) ? pcm_pair_smd(edges + i, edges + j, pos_cov, ang_cov)
                              : pcm_pair_smd(edges + j, edges + i, pos_cov, ang_cov);
    if (smd < thres) word |= 1u << b;
    if (smd_out) smd_out[(size_t)i * n + j] = smd;
  }
  bits[idx] = word;
}

// FMC::maxCliqueHeu on the bit matrix: one warp, lane l owns words l, l+32, l+64, l+96 of every bitset
__global__ void __launch_bounds__(32, 1)
pcm_max_clique_kernel(const uint32_t* __restrict__ bits, int n, int W, int32_t* __restrict__ deg_scratch /*[n]*/,
                      int32_t* __restrict__ inter_scratch /*[n]*/, int32_t* __restrict__ clique_out /*[n]*/,
                      int32_t* __restrict__ clique_size, uint8_t* __restrict__ adj_out /*[n][n] or null*/) {
  extern __shared__ uint32_t s_rows[];          // the whole bit matrix when it fits, else unused
  const int lane = threadIdx.x;
  const bool in_smem = (size_t)n * W * 4 <= 200 * 1024;
  if (in_smem)
    for (int i = lane; i < n * W; i += 32) s_rows[i] = bits[i];
  __syncwarp();
  const uint32_t* rows = in_smem ? s_rows : bits;
  // degrees (CGraphIO::CalculateVertexDegrees) and, optionally, the byte adjacency matrix for the caller
  for (int v = lane; v < n; v += 32) {
    int d = 0;
    for (int w = 0; w < W; ++w) d += __popc(bits[(size_t)v * W + w]);
    deg_scratch[v] = d;
  }
  if (adj_out)
    for (size_t e = lane; e < (size_t)n * n; e += 32) {
      const int i = (int)(e / n), j = (int)(e % n);
      adj_out[e] = (bits[(size_t)i * W + (j >> 5)] >> (j & 31)) & 1u;
    }
  __syncwarp();
  int max_clq = -1, best_len = 0;
  uint32_t dm[4];                               // degree mask {u : maxClq <= deg(u)}; all ones while maxClq = -1
  auto rebuild_mask = [&]() {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int w = lane + 32 * k;
      uint32_t m = 0;
      if (w < W)
        for (int b = 0; b < 32; ++b) {
          const int u = w * 32 + b;
          if (u < n && max_clq <= deg_scratch[u]) m |= 1u << b;
        }
      dm[k] = m;
    }
  };
  rebuild_mask();
  for (int v = 0; v < n; ++v) {
    if (max_clq > deg_scratch[v]) continue;                        // pruning 1 (:149), warp-uniform
    uint32_t S[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {                                  // S = {v} + neighbours passing pruning 3 (:156-165)
      const int w = lane + 32 * k;
      S[k] = (w < W) ? (rows[(size_t)v * W + w] & dm[k]) : 0u;
      if (w == (v >> 5)) S[k] |= 1u << (v & 31);
    }
    int len = 1, icc = 0;
    if (lane == 0) inter_scratch[0] = v;                           // :174
    while (true) {
      // imdv = last element of S (:185): S = [v, ascending neighbours], so the largest member other than v, else v
      int hi = -1;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int w = lane + 32 * k;
        uint32_t s = S[k];
        if (w == (v >> 5)) s &= ~(1u << (v & 31));
        if (s) hi = max(hi, w * 32 + 31 - __clz(s));
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, o));
      const int imdv = hi >= 0 ? hi : v;
      ++icc;
      uint32_t any = 0;
#pragma unroll
      for (int k = 0; k < 4; ++k) {                                // S1 = S & adj(imdv) & pruning 5 (:190-203)
        const int w = lane + 32 * k;
        S[k] = (w < W) ? (S[k] & rows[(size_t)imdv * W + w] & dm[k]) : 0u;
        any |= S[k];
      }
      any = __ballot_sync(0xffffffffu, any != 0);
      if (!any) break;                                             // (S1 empty: nothing pushed, loop ends, :218-232)
      if (lane == 0) inter_scratch[len] = imdv;
      ++len;
    }
    if (max_clq < icc) {                                           // :236-239
      max_clq = icc;
      best_len = len;
      __syncwarp();
      for (int i = lane; i < len; i += 32) clique_out[i] = inter_scratch[i];
      __syncwarp();
      rebuild_mask();
    }
  }
  if (lane == 0) *clique_size = best_len;
}

osb_status pcm_device(const osb_loop_edge* edges_dev, int n, double thres, double pos_cov, double ang_cov, uint32_t* bits,
                      int32_t* deg, int32_t* inter, int32_t* clique_dev, int32_t* size_dev, uint8_t* adj_dev, double* smd_dev,
                      cudaStream_t st) {
  const int W = (n + 31) / 32;
  OSB_LAUNCH(pcm_consistency_kernel, cdiv(n * W, 128), 128, 0, st, edges_dev, n, W, thres, pos_cov, ang_cov, bits, smd_dev);
  OSB_CHECK_LAUNCH();
  const size_t need = (size_t)n * W * 4;
  const size_t smem = need <= 200 * 1024 ? need : 0;
  OSB_SMEM_OPT_IN(pcm_max_clique_kernel, 200 * 1024);
  OSB_LAUNCH(pcm_max_clique_kernel, 1, 32, smem, st, bits, n, W, deg, inter, clique_dev, size_dev, adj_dev);
  OSB_CHECK_LAUNCH();
  return OSB_OK;
}

}  // namespace osb

using namespace osb;

static_assert(sizeof(osb_loop_edge) == 8 + 59 * 8, "osb_loop_edge layout");

extern "C" osb_status osb_pcm_dev(const osb_loop_edge* edges_dev, int n, double pcm_thres, double odom_pos_cov_per_m,
                                  double odom_ang_cov_per_m, int32_t* clique_dev, int32_t* clique_size_dev, uint8_t* adj_dev,
                                  double* smd_dev, void* stream) {
  OSB_REQUIRE(edges_dev && clique_dev && clique_size_dev, "null argument");
  OSB_REQUIRE(n > 0 && n <= PCM_MAX_N, "number of loop edges must be in 1..4096");
  osb_status s = require_device();
  if (s != OSB_OK) return s;
  cudaStream_t st = (cudaStream_t)stream;
  const int W = (n + 31) / 32;
  uint32_t* bits = nullptr;
  int32_t* scratch = nullptr;
  OSB_CUDA(cudaMallocAsync(&bits, (size_t)n * W * sizeof(uint32_t), st));
  const cudaError_t e = cudaMallocAsync(&scratch, (size_t)2 * n * sizeof(int32_t), st);
  if (e == cudaSuccess) {
    s = pcm_device(edges_dev, n, pcm_thres, odom_pos_cov_per_m, odom_ang_cov_per_m, bits, scratch, scratch + n, clique_dev,
                   clique_size_dev, adj_dev, smd_dev, st);
    cudaFreeAsync(scratch, st);
  }
  cudaFreeAsync(bits, st);
  OSB_CUDA(e);
  return s;
}

extern "C" osb_status osb_pcm(const osb_loop_edge* edges, int n, double pcm_thres, double odom_pos_cov_per_m,
                              double odom_ang_cov_per_m, int32_t* clique, int32_t* clique_size, uint8_t* adj, double* smd) {
  OSB_REQUIRE(edges && clique && clique_size, "null argument");
  OSB_REQUIRE(n > 0 && n <= PCM_MAX_N, "number of loop edges must be in 1..4096");
  OSB_TRY(require_device());
  Resources res;
  osb_loop_edge* d_e = nullptr;
  int32_t* d_c = nullptr;
  uint8_t* d_adj = nullptr;
  double* d_smd = nullptr;
  OSB_TRY(res.upload(&d_e, edges, n));
  OSB_TRY(res.alloc(&d_c, (size_t)n + 1));
  if (adj) OSB_TRY(res.alloc(&d_adj, (size_t)n * n));
  if (smd) OSB_TRY(res.alloc(&d_smd, (size_t)n * n));
  OSB_TRY(osb_pcm_dev(d_e, n, pcm_thres, odom_pos_cov_per_m, odom_ang_cov_per_m, d_c, d_c + n, d_adj, d_smd, nullptr));
  OSB_CUDA(cudaMemcpy(clique, d_c, (size_t)n * sizeof(int32_t), cudaMemcpyDeviceToHost));
  OSB_CUDA(cudaMemcpy(clique_size, d_c + n, sizeof(int32_t), cudaMemcpyDeviceToHost));
  if (adj) OSB_CUDA(cudaMemcpy(adj, d_adj, (size_t)n * n, cudaMemcpyDeviceToHost));
  if (smd) OSB_CUDA(cudaMemcpy(smd, d_smd, (size_t)n * n * sizeof(double), cudaMemcpyDeviceToHost));
  return OSB_OK;
}
