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
// osb_pcm_state keeps what the reference keeps between solves (OutlierRejectionLoopEdges, :98-167): every drone pair's
// loops and bit matrix live in a device slot, pcm_grow_kernel computes only the rows and boundary words a call adds, for
// all changed pairs in one launch, and pcm_max_clique_kernel runs one CTA per changed pair.
// Swarm::Pose / log_map / get_covariance / get_relative_pose_by_ts come from HKUST-Swarm/swarm_msgs, which is not in the
// reference tree: they are defined in oracle/pcm_ref.py and restated here (covariances and ego-motion poses are inputs).
#include "common.cuh"
#include "kernels.cuh"
#include "pose_algebra.cuh"

#include <map>
#include <set>
#include <unordered_set>

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

// one word of the adjacency bit matrix: bits of columns 32w .. 32w+31 of row i, the later loop always in the role of e1.
// Loop j is edges_lo[j] below m and edges_hi[j - m] from m on (the resident state reads its new loops from the staging copy).
__device__ __forceinline__ uint32_t pcm_consistency_word(const osb_loop_edge* __restrict__ edges_lo,
                                                         const osb_loop_edge* __restrict__ edges_hi, int m, int n, int i,
                                                         int w, double thres, double pos_cov, double ang_cov,
                                                         double* __restrict__ smd_row /*[n] or null*/) {
  const osb_loop_edge* ei = i < m ? edges_lo + i : edges_hi + (i - m);
  uint32_t word = 0;
  for (int b = 0; b < 32; ++b) {
    const int j = w * 32 + b;
    if (j >= n) break;
    const osb_loop_edge* ej = j < m ? edges_lo + j : edges_hi + (j - m);
    double smd = INFINITY;
    if (j != i) smd = (i > j) ? pcm_pair_smd(ei, ej, pos_cov, ang_cov) : pcm_pair_smd(ej, ei, pos_cov, ang_cov);
    if (smd < thres) word |= 1u << b;
    if (smd_row) smd_row[j] = smd;
  }
  return word;
}

// adjacency bit matrix: thread = (row i, word w) -> bits of columns 32w .. 32w+31
__global__ void __launch_bounds__(128)
pcm_consistency_kernel(const osb_loop_edge* __restrict__ edges, int n, int W, double thres, double pos_cov, double ang_cov,
                       uint32_t* __restrict__ bits /*[n][W]*/, double* __restrict__ smd_out /*[n][n] or null*/) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * W) return;
  const int i = idx / W, w = idx - i * W;
  bits[idx] = pcm_consistency_word(edges, edges, n, n, i, w, thres, pos_cov, ang_cov,
                                   smd_out ? smd_out + (size_t)i * n : nullptr);
}

// One drone pair as the kernels see it.  osb_pcm_dev passes one by value (its own buffers, stride = ceil(n/32)); the
// resident state (osb_pcm_state) uploads one per pair that gained loops, pointing into the pair's slot.
struct PcmPairJob {
  osb_loop_edge* edges;        // [cap] the pair's loops in insertion order (state only)
  uint32_t* bits;              // [n][stride] adjacency bit matrix
  int32_t* deg;                // [n] clique scratch
  int32_t* inter;              // [n]
  int32_t m, n;                // rows before / after this call (state: rows [m, n) are new)
  int32_t staged;              // state: the new loops are staged[staged .. staged + n - m)
  int32_t first_item;          // state: the pair's first (row, word) work item of pcm_grow_kernel
};

// FMC::maxCliqueHeu on the bit matrix: one warp per pair (CTA b runs jobs[b], or `one` when jobs is null), lane l owns
// words l, l+32, l+64, l+96 of every bitset.  Rows are `stride` words apart in global memory and W = ceil(n/32) apart in
// the shared copy.  CTA b writes clique_out + b * out_step and clique_size[b * out_step].
__global__ void __launch_bounds__(32, 1)
pcm_max_clique_kernel(const PcmPairJob* __restrict__ jobs, PcmPairJob one, int stride, int32_t* __restrict__ clique_out,
                      int32_t* __restrict__ clique_size, int out_step, uint8_t* __restrict__ adj_out /*[n][n] or null*/) {
  extern __shared__ uint32_t s_rows[];          // the whole bit matrix when it fits, else unused
  const PcmPairJob job = jobs ? jobs[blockIdx.x] : one;
  const uint32_t* __restrict__ bits = job.bits;
  int32_t* __restrict__ deg_scratch = job.deg;
  int32_t* __restrict__ inter_scratch = job.inter;
  clique_out += (size_t)blockIdx.x * out_step;
  clique_size += (size_t)blockIdx.x * out_step;
  const int n = job.n, W = (n + 31) / 32;
  const int lane = threadIdx.x;
  const bool in_smem = (size_t)n * W * 4 <= 200 * 1024;
  if (in_smem)
    for (int i = lane; i < n * W; i += 32) s_rows[i] = bits[(size_t)(i / W) * stride + i % W];
  __syncwarp();
  const uint32_t* rows = in_smem ? s_rows : bits;
  const int rs = in_smem ? W : stride;
  // degrees (CGraphIO::CalculateVertexDegrees) and, optionally, the byte adjacency matrix for the caller
  for (int v = lane; v < n; v += 32) {
    int d = 0;
    for (int w = 0; w < W; ++w) d += __popc(bits[(size_t)v * stride + w]);
    deg_scratch[v] = d;
  }
  if (adj_out)
    for (size_t e = lane; e < (size_t)n * n; e += 32) {
      const int i = (int)(e / n), j = (int)(e % n);
      adj_out[e] = (bits[(size_t)i * stride + (j >> 5)] >> (j & 31)) & 1u;
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
      S[k] = (w < W) ? (rows[(size_t)v * rs + w] & dm[k]) : 0u;
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
        S[k] = (w < W) ? (S[k] & rows[(size_t)imdv * rs + w] & dm[k]) : 0u;
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
  const PcmPairJob one{nullptr, bits, deg, inter, 0, n, 0, 0};
  OSB_LAUNCH(pcm_max_clique_kernel, 1, 32, smem, st, nullptr, one, W, clique_dev, size_dev, 0, adj_dev);
  OSB_CHECK_LAUNCH();
  return OSB_OK;
}

// Incremental consistency of every pair that gained loops, in one launch.  Job k owns the work items
// [first_item, first_item + m * (W - m/32) + (n - m) * W): for the old rows [0, m) the words from floor(m/32) on, then every
// word of the new rows [m, n).  The boundary word of an old row is recomputed whole: pcm_pair_smd is a pure function of the
// two loops and their order, so its old bits come back unchanged and the matrix equals pcm_consistency_kernel's on the
// pair's whole insertion-ordered list.  The thread of word 0 of a new row also moves that loop from the staging copy into
// the slot; nothing else in this launch reads slot rows >= m.
__global__ void __launch_bounds__(128)
pcm_grow_kernel(const PcmPairJob* __restrict__ jobs, int n_jobs, int n_items, const osb_loop_edge* __restrict__ staged,
                int stride, double thres, double pos_cov, double ang_cov) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_items) return;
  int lo = 0, hi = n_jobs - 1;                                     // the last job with first_item <= t
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (jobs[mid].first_item <= t) lo = mid; else hi = mid - 1;
  }
  const PcmPairJob job = jobs[lo];
  const int m = job.m, n = job.n, W = (n + 31) / 32, old_words = W - (m >> 5);
  int r = t - job.first_item, i, w;
  if (r < m * old_words) {
    i = r / old_words;
    w = (m >> 5) + r % old_words;
  } else {
    r -= m * old_words;
    i = m + r / W;
    w = r % W;
  }
  const osb_loop_edge* fresh = staged + job.staged;
  job.bits[(size_t)i * stride + w] = pcm_consistency_word(job.edges, fresh, m, n, i, w, thres, pos_cov, ang_cov, nullptr);
  if (i >= m && w == 0) job.edges[i] = fresh[i - m];
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

// =============================================================================================================
// C ABI: osb_pcm_state -- SwarmLocalOutlierRejection's persistent PCM state (swarm_outlier_rejection.cpp:37-56, 98-297)
// =============================================================================================================
struct osb_pcm_state {
  Resources res;
  int device = 0;
  osb_pcm_state_params p{};
  int stride = 0;                       // words per bit-matrix row: ceil(pair_capacity / 32), fixed so rows never move
  size_t jobs_bytes = 0;                // the staging buffers hold [max_pairs] PcmPairJob, then the call's new loops
  unsigned char* h_stage = nullptr;     // pinned
  unsigned char* d_stage = nullptr;
  int32_t* h_out = nullptr;             // [max_pairs][1 + pair_capacity]: clique size, clique (pinned)
  int32_t* d_out = nullptr;
  cudaStream_t stream = nullptr;
  std::mutex mu;
  struct Pair {                         // loop_pcm_graph[a][b] + all_loops[a][b] on the device, ids and clique here
    osb_loop_edge* edges;
    uint32_t* bits;
    int32_t* deg;
    int32_t* inter;
    std::vector<int64_t> ids;           // insertion order
    std::vector<int32_t> clique;        // the last maxCliqueHeu result, in its order
  };
  std::vector<Pair> pairs;
  std::map<std::pair<int32_t, int32_t>, int> index;                    // unordered pair (lo, hi) -> pairs[]
  std::unordered_set<int64_t> seen;                                    // all_loops_set
  std::map<std::pair<int32_t, int32_t>, std::set<int64_t>> good;       // good_loops_set, one entry per unordered pair
};

namespace {

std::pair<int32_t, int32_t> pair_key(int32_t a, int32_t b) { return {std::min(a, b), std::max(a, b)}; }

bool pcm_routed(const osb_pcm_state* s, std::pair<int32_t, int32_t> k) {   // :122-139
  return s->p.redundant || k.first == s->p.self_id || k.second == s->p.self_id;
}

// the one device slot of a pair: loops [cap], bit matrix [cap][stride], degree and clique scratch [cap] each
osb_status pcm_acquire_slot(osb_pcm_state* s, osb_pcm_state::Pair* P) {
  const size_t cap = (size_t)s->p.pair_capacity;
  unsigned char* base = nullptr;
  OSB_TRY(s->res.alloc(&base, cap * sizeof(osb_loop_edge) + cap * s->stride * sizeof(uint32_t) + 2 * cap * sizeof(int32_t)));
  P->edges = (osb_loop_edge*)base;
  P->bits = (uint32_t*)(base + cap * sizeof(osb_loop_edge));
  P->deg = (int32_t*)(P->bits + cap * s->stride);
  P->inter = P->deg + cap;
  return OSB_OK;
}

// appends the routed new loops (`fresh`: pair -> input indices in call order) and reruns maxCliqueHeu on every pair that
// gained any: one copy up, two launches, one copy down, one synchronisation.  The host record changes only on success.
osb_status pcm_state_grow(osb_pcm_state* s, const std::map<std::pair<int32_t, int32_t>, std::vector<int>>& fresh,
                          const osb_loop_edge* edges, const int64_t* ids) {
  for (const auto& kv : fresh)
    if (!s->index.count(kv.first)) {
      osb_pcm_state::Pair P{};
      OSB_TRY(pcm_acquire_slot(s, &P));
      s->index[kv.first] = (int)s->pairs.size();
      s->pairs.push_back(std::move(P));
    }
  PcmPairJob* jobs = (PcmPairJob*)s->h_stage;
  osb_loop_edge* staged = (osb_loop_edge*)(s->h_stage + s->jobs_bytes);
  int k = 0, n_staged = 0;
  long long items = 0;
  size_t smem = 0;
  std::vector<int> changed;
  for (const auto& kv : fresh) {
    const int pi = s->index[kv.first];
    osb_pcm_state::Pair& P = s->pairs[pi];
    const int m = (int)P.ids.size(), n = m + (int)kv.second.size(), W = (n + 31) / 32;
    jobs[k++] = PcmPairJob{P.edges, P.bits, P.deg, P.inter, m, n, n_staged, (int32_t)items};
    for (int i : kv.second) staged[n_staged++] = edges[i];
    items += (long long)m * (W - (m >> 5)) + (long long)(n - m) * W;
    const size_t need = (size_t)n * W * 4;
    if (need <= 200 * 1024) smem = std::max(smem, need);
    changed.push_back(pi);
    OSB_REQUIRE(items < (1ll << 31), "too many pair checks in one call");
  }
  cudaStream_t st = s->stream;
  OSB_CUDA(cudaMemcpyAsync(s->d_stage, s->h_stage, s->jobs_bytes + (size_t)n_staged * sizeof(osb_loop_edge),
                           cudaMemcpyHostToDevice, st));
  const PcmPairJob* d_jobs = (const PcmPairJob*)s->d_stage;
  OSB_LAUNCH(pcm_grow_kernel, cdiv((int)items, 128), 128, 0, st, d_jobs, k, (int)items,
             (const osb_loop_edge*)(s->d_stage + s->jobs_bytes), s->stride, s->p.pcm_thres, s->p.odom_pos_cov_per_m,
             s->p.odom_ang_cov_per_m);
  OSB_CHECK_LAUNCH();
  OSB_SMEM_OPT_IN(pcm_max_clique_kernel, 200 * 1024);
  const int out_step = 1 + s->p.pair_capacity;
  OSB_LAUNCH(pcm_max_clique_kernel, k, 32, smem, st, d_jobs, PcmPairJob{}, s->stride, s->d_out + 1, s->d_out, out_step,
             (uint8_t*)nullptr);
  OSB_CHECK_LAUNCH();
  OSB_CUDA(cudaMemcpyAsync(s->h_out, s->d_out, (size_t)k * out_step * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  OSB_CUDA(cudaStreamSynchronize(st));
  k = 0;
  for (const auto& kv : fresh) {                                   // :271-272, 292-297
    osb_pcm_state::Pair& P = s->pairs[changed[k]];
    for (int i : kv.second) P.ids.push_back(ids[i]);
    const int32_t* out = s->h_out + (size_t)k * out_step;
    P.clique.assign(out + 1, out + 1 + out[0]);
    std::set<int64_t>& g = s->good[kv.first];
    g.clear();
    for (int32_t c : P.clique) g.insert(P.ids[c]);
    for (int i : kv.second) s->seen.insert(ids[i]);
    ++k;
  }
  return OSB_OK;
}

}  // namespace

extern "C" osb_status osb_pcm_state_create(osb_pcm_state** out, const osb_pcm_state_params* p) {
  OSB_REQUIRE(out != nullptr && p != nullptr, "null argument");
  OSB_REQUIRE(p->max_pairs > 0 && p->max_pairs <= 65536, "max_pairs must be in 1..65536");
  OSB_REQUIRE(p->pair_capacity > 0 && p->pair_capacity <= PCM_MAX_N, "pair_capacity must be in 1..4096");
  OSB_TRY(require_device());
  std::unique_ptr<osb_pcm_state> s(new osb_pcm_state());
  s->device = current_device();
  s->p = *p;
  s->p.redundant = p->redundant ? 1 : 0;
  s->stride = (p->pair_capacity + 31) / 32;
  s->jobs_bytes = (size_t)p->max_pairs * sizeof(PcmPairJob);
  const size_t stage = s->jobs_bytes + (size_t)p->max_pairs * p->pair_capacity * sizeof(osb_loop_edge);
  const size_t outs = (size_t)p->max_pairs * (1 + p->pair_capacity);
  OSB_TRY(s->res.stream(&s->stream));
  OSB_TRY(s->res.host_alloc(&s->h_stage, stage, cudaHostAllocDefault));
  OSB_TRY(s->res.alloc(&s->d_stage, stage));
  OSB_TRY(s->res.host_alloc(&s->h_out, outs, cudaHostAllocDefault));
  OSB_TRY(s->res.alloc(&s->d_out, outs));
  *out = s.release();
  return OSB_OK;
}

extern "C" osb_status osb_pcm_state_destroy(osb_pcm_state* s) {
  delete s;
  return OSB_OK;
}

extern "C" osb_status osb_pcm_state_reject(osb_pcm_state* s, const osb_loop_edge* edges, const int64_t* ids, int n,
                                           uint8_t* keep) {
  OSB_REQUIRE(s != nullptr && n >= 0, "null state or negative count");
  OSB_REQUIRE(n == 0 || (edges && ids && keep), "null argument");
  std::lock_guard<std::mutex> lk(s->mu);
  DeviceGuard dg(s->device);
  // :106-120: a loop is new unless an earlier call stored its id; the routing of :122-139 decides whether it is stored
  std::map<std::pair<int32_t, int32_t>, std::vector<int>> fresh;
  for (int i = 0; i < n; ++i) {
    if (s->seen.count(ids[i])) continue;
    const auto k = pair_key(edges[i].id_a, edges[i].id_b);
    if (pcm_routed(s, k)) fresh[k].push_back(i);
  }
  size_t new_pairs = 0;
  for (const auto& kv : fresh) {
    const auto it = s->index.find(kv.first);
    const size_t have = it == s->index.end() ? 0 : s->pairs[it->second].ids.size();
    new_pairs += it == s->index.end();
    if (have + kv.second.size() > (size_t)s->p.pair_capacity) {
      set_error(__func__, "a drone pair would exceed pair_capacity loop edges");
      return OSB_ERR_CAPACITY;
    }
  }
  if (s->pairs.size() + new_pairs > (size_t)s->p.max_pairs) {
    set_error(__func__, "the state would exceed max_pairs drone pairs");
    return OSB_ERR_CAPACITY;
  }
  if (!fresh.empty()) OSB_TRY(pcm_state_grow(s, fresh, edges, ids));
  for (int i = 0; i < n; ++i) {                                    // :141-157
    const auto it = s->good.find(pair_key(edges[i].id_a, edges[i].id_b));
    keep[i] = it == s->good.end() || it->second.count(ids[i]) ? 1 : 0;
  }
  return OSB_OK;
}

extern "C" osb_status osb_pcm_state_inliers(osb_pcm_state* s, int32_t id_a, int32_t id_b, int64_t* ids, int cap,
                                            int32_t* n) {
  OSB_REQUIRE(s != nullptr && n != nullptr && cap >= 0, "null argument or negative capacity");
  std::lock_guard<std::mutex> lk(s->mu);
  const auto it = s->good.find(pair_key(id_a, id_b));
  if (it == s->good.end()) {
    *n = -1;
    return OSB_OK;
  }
  *n = (int32_t)it->second.size();
  if (ids == nullptr) return OSB_OK;
  if ((size_t)cap < it->second.size()) {
    set_error(__func__, "the pair's inlier set is larger than cap");
    return OSB_ERR_CAPACITY;
  }
  std::copy(it->second.begin(), it->second.end(), ids);
  return OSB_OK;
}

extern "C" osb_status osb_pcm_state_set_inliers(osb_pcm_state* s, int32_t id_a, int32_t id_b, const int64_t* ids, int n) {
  OSB_REQUIRE(s != nullptr && n >= 0 && (n == 0 || ids != nullptr), "null argument or negative count");
  std::lock_guard<std::mutex> lk(s->mu);
  if (id_a == s->p.self_id || id_b == s->p.self_id) return OSB_OK;    // :40-43
  s->good[pair_key(id_a, id_b)] = std::set<int64_t>(ids, ids + n);
  return OSB_OK;
}

extern "C" osb_status osb_pcm_state_pair(osb_pcm_state* s, int32_t id_a, int32_t id_b, int32_t* n, int64_t* ids,
                                         uint8_t* adj, int32_t* clique, int32_t* clique_size) {
  OSB_REQUIRE(s != nullptr && n != nullptr, "null argument");
  std::lock_guard<std::mutex> lk(s->mu);
  DeviceGuard dg(s->device);
  const auto it = s->index.find(pair_key(id_a, id_b));
  if (it == s->index.end()) {
    *n = 0;
    if (clique_size) *clique_size = 0;
    return OSB_OK;
  }
  const osb_pcm_state::Pair& P = s->pairs[it->second];
  const int m = (int)P.ids.size(), W = (m + 31) / 32;
  *n = m;
  if (ids) std::copy(P.ids.begin(), P.ids.end(), ids);
  if (clique) std::copy(P.clique.begin(), P.clique.end(), clique);
  if (clique_size) *clique_size = (int32_t)P.clique.size();
  if (adj && m > 0) {
    std::vector<uint32_t> rows((size_t)m * W);
    OSB_CUDA(cudaMemcpy2DAsync(rows.data(), W * sizeof(uint32_t), P.bits, s->stride * sizeof(uint32_t),
                               W * sizeof(uint32_t), m, cudaMemcpyDeviceToHost, s->stream));
    OSB_CUDA(cudaStreamSynchronize(s->stream));
    for (int i = 0; i < m; ++i)
      for (int j = 0; j < m; ++j) adj[(size_t)i * m + j] = (rows[(size_t)i * W + (j >> 5)] >> (j & 31)) & 1u;
  }
  return OSB_OK;
}
