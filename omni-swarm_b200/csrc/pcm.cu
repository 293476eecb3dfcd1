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

#include <cstddef>
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
// `hi(k)` is loop m + k.
template <class Hi>
__device__ __forceinline__ uint32_t pcm_consistency_word(const osb_loop_edge* __restrict__ edges_lo, Hi hi, int m, int n,
                                                         int i, int w, double thres, double pos_cov, double ang_cov,
                                                         double* __restrict__ smd_row /*[n] or null*/) {
  const osb_loop_edge* ei = i < m ? edges_lo + i : hi(i - m);
  uint32_t word = 0;
  for (int b = 0; b < 32; ++b) {
    const int j = w * 32 + b;
    if (j >= n) break;
    const osb_loop_edge* ej = j < m ? edges_lo + j : hi(j - m);
    double smd = INFINITY;
    if (j != i) smd = (i > j) ? pcm_pair_smd(ei, ej, pos_cov, ang_cov) : pcm_pair_smd(ej, ei, pos_cov, ang_cov);
    if (smd < thres) word |= 1u << b;
    if (smd_row) smd_row[j] = smd;
  }
  return word;
}

struct PcmContiguous {                                              // loop k at p + k
  const osb_loop_edge* p;
  __device__ const osb_loop_edge* operator()(int k) const { return p + k; }
};

// adjacency bit matrix: thread = (row i, word w) -> bits of columns 32w .. 32w+31
__global__ void __launch_bounds__(128)
pcm_consistency_kernel(const osb_loop_edge* __restrict__ edges, int n, int W, double thres, double pos_cov, double ang_cov,
                       uint32_t* __restrict__ bits /*[n][W]*/, double* __restrict__ smd_out /*[n][n] or null*/) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * W) return;
  const int i = idx / W, w = idx - i * W;
  bits[idx] = pcm_consistency_word(edges, PcmContiguous{edges}, n, n, i, w, thres, pos_cov, ang_cov,
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
  int32_t staged;              // state: the new loops are fresh entries staged .. staged + n - m
  int32_t first_item;          // state: the pair's first (row, word) work item of pcm_grow_kernel
  int64_t* ids;                // state: [cap] the pair's loop ids in insertion order (the device record)
  int32_t slot, reserved;      // state: the pair's slot
};

// Device counters of the resident state.  The anchored path plans on the device, so the grow and clique launches read
// their job count and work-item count here instead of taking them from the host.
struct PcmMeta {
  int32_t status;              // the last reject_anchored call: OSB_OK or OSB_ERR_CAPACITY
  int32_t n_slots, n_dir;      // slots in use, directory entries in use
  int32_t n_jobs, n_items;     // the last anchored call's grow / clique work (0 after a refused call)
  int32_t seen_min;            // INT64_MIN (the hash's empty key) is in the seen set
};

// all_loops_set on the device: open addressing over a power-of-two table, linear probing, empty = INT64_MIN
constexpr unsigned long long PCM_EMPTY = 0x8000000000000000ull;
__host__ __device__ inline unsigned long long pcm_hash(int64_t id) {          // splitmix64's finaliser
  unsigned long long z = (unsigned long long)id + 0x9e3779b97f4a7c15ull;
  z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
  z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
  return z ^ (z >> 31);
}
struct PcmSeen {
  unsigned long long* table;   // null until the first anchored call builds it
  unsigned long long mask;
  PcmMeta* meta;
  __device__ bool has(int64_t id) const {
    if ((unsigned long long)id == PCM_EMPTY) return meta->seen_min != 0;
    for (unsigned long long h = pcm_hash(id) & mask;; h = (h + 1) & mask) {
      const unsigned long long k = table[h];
      if (k == (unsigned long long)id) return true;
      if (k == PCM_EMPTY) return false;
    }
  }
  __device__ void insert(int64_t id) const {
    if ((unsigned long long)id == PCM_EMPTY) { meta->seen_min = 1; return; }
    for (unsigned long long h = pcm_hash(id) & mask;; h = (h + 1) & mask) {
      const unsigned long long k = atomicCAS(table + h, PCM_EMPTY, (unsigned long long)id);
      if (k == PCM_EMPTY || k == (unsigned long long)id) return;
    }
  }
};

// Where a grow launch reads its new loops: fresh entry e is row r = index ? index[e] : e, its edge at
// edge_base + r * edge_stride and its id at id_base + r * id_stride.  The host path stages packed edges and ids; the
// anchored path reads osb_anchor_result rows in place through the planned order.
struct PcmFresh {
  const unsigned char* edge_base;
  const unsigned char* id_base;
  const int32_t* index;
  long long edge_stride, id_stride;
  __device__ long long row(int e) const { return index ? index[e] : e; }
  __device__ const osb_loop_edge* edge(int e) const {
    return reinterpret_cast<const osb_loop_edge*>(edge_base + row(e) * edge_stride);
  }
  __device__ int64_t id(int e) const { return *reinterpret_cast<const int64_t*>(id_base + row(e) * id_stride); }
};
struct PcmFreshAt {                                                // loop m + k of a job = fresh entry first + k
  PcmFresh f;
  int first;
  __device__ const osb_loop_edge* operator()(int k) const { return f.edge(first + k); }
};

// FMC::maxCliqueHeu on the bit matrix: one warp per pair (CTA b runs jobs[b], or `one` when jobs is null), lane l owns
// words l, l+32, l+64, l+96 of every bitset.  Rows are `stride` words apart in global memory and W = ceil(n/32) apart in
// the shared copy.  CTA b writes clique_out + b * out_step and clique_size[b * out_step].  With n_jobs_dev the grid is one
// CTA per possible pair and CTA b exits unless b < *n_jobs_dev (a job list built on the device).
__global__ void __launch_bounds__(32, 1)
pcm_max_clique_kernel(const PcmPairJob* __restrict__ jobs, PcmPairJob one, int stride, int32_t* __restrict__ clique_out,
                      int32_t* __restrict__ clique_size, int out_step, uint8_t* __restrict__ adj_out /*[n][n] or null*/,
                      const int32_t* __restrict__ n_jobs_dev /*or null*/) {
  extern __shared__ uint32_t s_rows[];          // the whole bit matrix when it fits, else unused
  if (n_jobs_dev && (int)blockIdx.x >= *n_jobs_dev) return;
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
  OSB_LAUNCH(pcm_max_clique_kernel, 1, 32, smem, st, nullptr, one, W, clique_dev, size_dev, 0, adj_dev,
             (const int32_t*)nullptr);
  OSB_CHECK_LAUNCH();
  return OSB_OK;
}

// Incremental consistency of every pair that gained loops, in one launch.  Job k owns the work items
// [first_item, first_item + m * (W - m/32) + (n - m) * W): for the old rows [0, m) the words from floor(m/32) on, then every
// word of the new rows [m, n).  The boundary word of an old row is recomputed whole: pcm_pair_smd is a pure function of the
// two loops and their order, so its old bits come back unchanged and the matrix equals pcm_consistency_kernel's on the
// pair's whole insertion-ordered list.  The thread of word 0 of a new row also moves that loop (and its id) from the fresh
// source into the slot and marks the id as seen; nothing else in this launch reads slot rows >= m.  With meta the job and
// item counts come from the device (a device-built job list) and the grid strides over them.
__global__ void __launch_bounds__(128)
pcm_grow_kernel(const PcmPairJob* __restrict__ jobs, int n_jobs, int n_items, const PcmMeta* __restrict__ meta /*or null*/,
                PcmFresh fresh, PcmSeen seen, int stride, double thres, double pos_cov, double ang_cov) {
  if (meta) {
    n_jobs = meta->n_jobs;
    n_items = meta->n_items;
  }
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < n_items; t += gridDim.x * blockDim.x) {
    int lo = 0, hi = n_jobs - 1;                                   // the last job with first_item <= t
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
    const PcmFreshAt at{fresh, job.staged};
    job.bits[(size_t)i * stride + w] = pcm_consistency_word(job.edges, at, m, n, i, w, thres, pos_cov, ang_cov, nullptr);
    if (i >= m && w == 0) {
      job.edges[i] = *at(i - m);
      const int64_t id = fresh.id(job.staged + i - m);
      job.ids[i] = id;
      if (seen.table) seen.insert(id);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// The anchored path: osb_anchor_result rows -> routing, de-duplication, append plan, grow, clique, inlier sets, keep mask,
// all stream-ordered on the device.  Pair keys are (lo << 32) | hi of the unordered drone pair.
// ---------------------------------------------------------------------------------------------------------------------
__host__ __device__ inline int64_t pcm_key(int32_t a, int32_t b) {
  const int32_t lo = a < b ? a : b, hi = a < b ? b : a;
  return (int64_t)(((unsigned long long)(uint32_t)lo << 32) | (uint32_t)hi);
}

struct PcmSlot {               // a pair's device storage (one allocation)
  osb_loop_edge* edges;        // [cap]
  uint32_t* bits;              // [cap][stride]
  int32_t *deg, *inter;        // [cap] each
  int64_t* ids;                // [cap]
  int32_t* clique;             // [1 + cap]: size, then the indices in maxCliqueHeu order
  int64_t* good;               // [cap]: the inlier ids of the last clique, ascending
};
struct PcmDir {                // good_loops_set of one unordered pair (a pair with a slot, or one set_inliers named)
  int64_t key;
  int64_t* gptr;               // ascending ids [gn] (duplicates allowed)
  int32_t slot;                // -1: the pair has no loops
  int32_t gn;                  // -1: the pair has no set
  int32_t gcap, reserved;
};

struct PcmRows {               // the anchored call's rows and the routing rule
  const osb_anchor_result* rows;
  int n;
  int32_t self_id, redundant;
  PcmSeen seen;
  // a row is routed to the state iff OK, its pair is processed (:122-139) and no earlier call stored its id (:106-120)
  __device__ bool fresh(int i) const {
    const osb_anchor_result& r = rows[i];
    if (r.status != OSB_ANCHOR_OK) return false;
    if (!(redundant || r.edge.id_a == self_id || r.edge.id_b == self_id)) return false;
    return !seen.has(r.id);
  }
  __device__ void range(int c, int G, int* lo, int* hi) const {
    *lo = (int)((long long)n * c / G);
    *hi = (int)((long long)n * (c + 1) / G);
  }
};

// block of 256: exclusive rank of each flagged thread in the block and the block's total
__device__ __forceinline__ int pcm_block_rank(bool flag, int* total, int* s_warp) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const unsigned b = __ballot_sync(0xffffffffu, flag);
  __syncthreads();
  if (lane == 0) s_warp[wid] = __popc(b);
  __syncthreads();
  int before = 0, all = 0;
  for (int k = 0; k < (int)(blockDim.x >> 5); ++k) {
    if (k < wid) before += s_warp[k];
    all += s_warp[k];
  }
  *total = all;
  return before + __popc(b & ((1u << lane) - 1));
}

// pass 1: CTA c counts the fresh rows of its contiguous row range
__global__ void __launch_bounds__(256) pcm_anchored_count_kernel(PcmRows v, int32_t* __restrict__ cnt) {
  int lo, hi;
  v.range(blockIdx.x, gridDim.x, &lo, &hi);
  int c = 0;
  for (int base = lo; base < hi; base += 256) {
    const int i = base + threadIdx.x;
    c += __syncthreads_count(i < hi && v.fresh(i));
  }
  if (threadIdx.x == 0) cnt[blockIdx.x] = c;
}

// pass 2: CTA c writes its fresh rows' indices, in row order, from the sum of the counts before it on (a deterministic
// compaction: no atomics).  Entries past cand_cap are dropped; the plan refuses the call then.
__global__ void __launch_bounds__(256)
pcm_anchored_collect_kernel(PcmRows v, const int32_t* __restrict__ cnt, int32_t* __restrict__ cand, int cand_cap) {
  __shared__ int s_warp[8];
  __shared__ int s_off;
  if (threadIdx.x == 0) {
    int o = 0;
    for (int k = 0; k < (int)blockIdx.x; ++k) o += cnt[k];
    s_off = o;
  }
  __syncthreads();
  int off = s_off, lo, hi;
  v.range(blockIdx.x, gridDim.x, &lo, &hi);
  for (int base = lo; base < hi; base += 256) {
    const int i = base + threadIdx.x;
    const bool f = i < hi && v.fresh(i);
    int total;
    const int r = pcm_block_rank(f, &total, s_warp);
    if (f && off + r < cand_cap) cand[off + r] = i;
    off += total;
  }
}

struct PcmPlan {
  const osb_anchor_result* rows;
  const int32_t* cnt;          // [G] pass-1 counts
  int G;
  const int32_t* cand;         // [cand_cap] fresh row indices, row order
  int32_t *cand_slot, *cand_rank;
  int cand_cap;
  int32_t* order;              // [cand_cap] fresh row indices grouped by job, row order within a pair
  int64_t* slot_key;           // [max_pairs]
  int32_t *slot_n, *slot_dir;  // [max_pairs]
  const PcmSlot* slots;        // [max_pairs]
  PcmDir* dir;
  PcmMeta* meta;
  int32_t *pcnt, *poff;        // [max_pairs] scratch
  PcmPairJob* jobs;            // [max_pairs]
  int max_pairs, cap;
};

// warp-inclusive scan of v
__device__ __forceinline__ long long pcm_warp_scan(long long v) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const long long u = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += u;
  }
  return v;
}

// One warp plans the call: finds (or appends, in order of first appearance) each fresh row's pair slot, ranks the row
// within its pair in row order, checks pair_capacity / max_pairs / the work-item bound BEFORE anything of the state is
// written, and only then commits: slot counts, new slots and their directory entries, the dense job list in slot order and
// the fresh rows in job order.  A refused call sets status = OSB_ERR_CAPACITY and zero jobs, and changes nothing else.
__global__ void __launch_bounds__(32, 1) pcm_anchored_plan_kernel(PcmPlan p) {
  const int lane = threadIdx.x;
  const unsigned lt = (1u << lane) - 1u;
  PcmMeta* meta = p.meta;
  long long c_sum = 0;
  for (int c = lane; c < p.G; c += 32) c_sum += p.cnt[c];
  c_sum = __shfl_sync(0xffffffffu, pcm_warp_scan(c_sum), 31);
  const int ns0 = meta->n_slots;
  int ns = ns0;
  bool err = c_sum > p.cand_cap;
  const int C = (int)min(c_sum, (long long)p.cand_cap);
  for (int s = lane; s < p.max_pairs; s += 32) p.pcnt[s] = 0;
  __syncwarp();
  for (int base = 0; base < C && !err; base += 32) {
    const int k = base + lane;
    const bool on = k < C;
    int64_t key = 0;
    int s = -1;
    if (on) {
      const osb_loop_edge& e = p.rows[p.cand[k]].edge;
      key = pcm_key(e.id_a, e.id_b);
      for (int q = 0; q < ns; ++q)
        if (p.slot_key[q] == key) { s = q; break; }
    }
    const bool need = on && s < 0;
    const unsigned needm = __ballot_sync(0xffffffffu, need);
    if (needm) {                                                   // new pairs take slots in order of first appearance
      const unsigned peers = __match_any_sync(0xffffffffu, (unsigned long long)key) & needm;
      const int leader = need ? __ffs(peers) - 1 : lane;
      const bool lead = need && leader == lane;
      const unsigned leads = __ballot_sync(0xffffffffu, lead);
      const int mine = ns + __popc(leads & lt);
      if (lead && mine < p.max_pairs) p.slot_key[mine] = key;      // past n_slots: not state until committed
      const int got = __shfl_sync(0xffffffffu, mine, leader);
      if (need) s = got;
      ns += __popc(leads);
      err = ns > p.max_pairs;
      __syncwarp();
      if (err) break;
    }
    const unsigned onm = __ballot_sync(0xffffffffu, on);
    const unsigned peers = __match_any_sync(0xffffffffu, s) & onm;
    const int rank = on ? p.pcnt[s] + __popc(peers & lt) : 0;
    __syncwarp();
    if (on && __ffs(peers) - 1 == lane) p.pcnt[s] += __popc(peers);
    __syncwarp();
    if (on) {
      p.cand_slot[k] = s;
      p.cand_rank[k] = rank;
    }
  }
  // capacity and work-item checks (dry run of the job list)
  long long items = 0;
  if (!err)
    for (int b = 0; b < ns; b += 32) {
      const int s = b + lane;
      long long it = 0;
      bool over = false;
      if (s < ns) {
        const int add = p.pcnt[s], m = s < ns0 ? p.slot_n[s] : 0, n = m + add, W = (n + 31) / 32;
        over = n > p.cap;
        if (add > 0) it = (long long)m * (W - (m >> 5)) + (long long)add * W;
      }
      err |= __any_sync(0xffffffffu, over);
      items += __shfl_sync(0xffffffffu, pcm_warp_scan(it), 31);
    }
  err |= items >= (1ll << 31);
  if (err) {
    if (lane == 0) {
      meta->status = OSB_ERR_CAPACITY;
      meta->n_jobs = 0;
      meta->n_items = 0;
    }
    return;
  }
  // commit
  int nj = 0, off = 0;
  items = 0;
  for (int b = 0; b < ns; b += 32) {
    const int s = b + lane;
    const int add = s < ns ? p.pcnt[s] : 0;
    const int m = (s < ns0) ? p.slot_n[s] : 0, n = m + add, W = (n + 31) / 32;
    const long long it = add > 0 ? (long long)m * (W - (m >> 5)) + (long long)add * W : 0;
    const long long inc_j = pcm_warp_scan(add > 0 ? 1 : 0), inc_a = pcm_warp_scan(add), inc_i = pcm_warp_scan(it);
    if (add > 0) {
      const PcmSlot& sl = p.slots[s];
      PcmPairJob j;
      j.edges = sl.edges; j.bits = sl.bits; j.deg = sl.deg; j.inter = sl.inter;
      j.m = m; j.n = n;
      j.staged = off + (int)(inc_a - add);
      j.first_item = (int32_t)(items + inc_i - it);
      j.ids = sl.ids; j.slot = s; j.reserved = 0;
      p.jobs[nj + (int)(inc_j - 1)] = j;
      p.poff[s] = j.staged;
      p.slot_n[s] = n;
    }
    nj += (int)__shfl_sync(0xffffffffu, inc_j, 31);
    off += (int)__shfl_sync(0xffffffffu, inc_a, 31);
    items += __shfl_sync(0xffffffffu, inc_i, 31);
  }
  if (lane == 0) {
    int nd = meta->n_dir;
    for (int s = ns0; s < ns; ++s) {                               // a new slot joins its pair's directory entry
      const int64_t key = p.slot_key[s];
      int e = 0;
      while (e < nd && p.dir[e].key != key) ++e;
      if (e == nd) {
        p.dir[e].key = key; p.dir[e].gptr = nullptr; p.dir[e].gn = -1; p.dir[e].gcap = 0; p.dir[e].reserved = 0;
        ++nd;
      }
      p.dir[e].slot = s;
      p.slot_dir[s] = e;
    }
    meta->n_dir = nd;
    meta->n_slots = ns;
    meta->n_jobs = nj;
    meta->n_items = (int32_t)items;
    meta->status = OSB_OK;
  }
  __syncwarp();
  for (int k = lane; k < C; k += 32) p.order[p.poff[p.cand_slot[k]] + p.cand_rank[k]] = p.cand[k];
}

// After the clique launch: CTA b < n_jobs copies job b's clique into its slot and replaces the pair's inlier set with the
// clique's ids, sorted ascending (bitonic sort in shared memory), through the pair's directory entry (:271-272, 292-297).
constexpr int PCM_FINISH_THREADS = 512;
__global__ void __launch_bounds__(PCM_FINISH_THREADS)
pcm_anchored_finish_kernel(const PcmPairJob* __restrict__ jobs, const PcmMeta* __restrict__ meta,
                           const int32_t* __restrict__ out, int out_step, const PcmSlot* __restrict__ slots,
                           const int32_t* __restrict__ slot_dir, PcmDir* __restrict__ dir, int cap) {
  __shared__ int64_t s_ids[PCM_MAX_N];
  if ((int)blockIdx.x >= meta->n_jobs) return;
  const PcmPairJob job = jobs[blockIdx.x];
  const PcmSlot sl = slots[job.slot];
  const int32_t* o = out + (size_t)blockIdx.x * out_step;
  const int size = o[0];
  int P = 1;
  while (P < size) P <<= 1;
  for (int k = threadIdx.x; k < P; k += blockDim.x) {
    if (k < size) {
      const int c = o[1 + k];
      sl.clique[1 + k] = c;
      s_ids[k] = job.ids[c];
    } else {
      s_ids[k] = INT64_MAX;
    }
  }
  if (threadIdx.x == 0) sl.clique[0] = size;
  __syncthreads();
  for (int len = 2; len <= P; len <<= 1)
    for (int j = len >> 1; j > 0; j >>= 1) {
      for (int k = threadIdx.x; k < P; k += blockDim.x) {
        const int q = k ^ j;
        if (q > k) {
          const bool up = (k & len) == 0;
          const int64_t a = s_ids[k], b = s_ids[q];
          if ((a > b) == up) { s_ids[k] = b; s_ids[q] = a; }
        }
      }
      __syncthreads();
    }
  for (int k = threadIdx.x; k < size; k += blockDim.x) sl.good[k] = s_ids[k];
  if (threadIdx.x == 0) {
    PcmDir& d = dir[slot_dir[job.slot]];
    d.gptr = sl.good;
    d.gn = size;
    d.gcap = cap;
  }
}

// keep[i] (:141-157): OK rows whose pair has no inlier set or whose id is in it; 0 for every other row.  Not written when
// the plan refused the call.
__global__ void __launch_bounds__(256)
pcm_anchored_keep_kernel(const osb_anchor_result* __restrict__ rows, int n, const PcmDir* __restrict__ dir,
                         const PcmMeta* __restrict__ meta, uint8_t* __restrict__ keep) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || meta->status != OSB_OK) return;
  const osb_anchor_result& r = rows[i];
  uint8_t k = 0;
  if (r.status == OSB_ANCHOR_OK) {
    const int64_t key = pcm_key(r.edge.id_a, r.edge.id_b), id = r.id;
    const int nd = meta->n_dir;
    int e = 0;
    while (e < nd && dir[e].key != key) ++e;
    k = 1;
    if (e < nd && dir[e].gn >= 0) {
      const int64_t* g = dir[e].gptr;
      int lo = 0, hi = dir[e].gn;                                  // first g[x] >= id
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (g[mid] < id) lo = mid + 1; else hi = mid;
      }
      k = (lo < dir[e].gn && g[lo] == id) ? 1 : 0;
    }
  }
  keep[i] = k;
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
  size_t jobs_bytes = 0;                // the staging buffers hold [max_pairs] PcmPairJob, the call's new loops, their ids
  size_t edges_bytes = 0;               // [max_pairs][pair_capacity] loops
  unsigned char* h_stage = nullptr;     // pinned
  unsigned char* d_stage = nullptr;
  int32_t* h_out = nullptr;             // [max_pairs][1 + pair_capacity]: clique size, clique (pinned)
  int32_t* d_out = nullptr;
  cudaStream_t stream = nullptr;
  std::mutex mu;
  struct Pair {                         // the host record of slots[i]: loop_pcm_graph[a][b] + all_loops[a][b] on the device
    std::pair<int32_t, int32_t> key;
    std::vector<int64_t> ids;           // insertion order
    std::vector<int32_t> clique;        // the last maxCliqueHeu result, in its order
  };
  std::vector<Pair> pairs;              // pairs[i] lives in slots[i]
  std::vector<PcmSlot> slots;           // [max_pairs]; edges == null until acquired
  std::map<std::pair<int32_t, int32_t>, int> index;                    // unordered pair (lo, hi) -> pairs[]
  std::unordered_set<int64_t> seen;                                    // all_loops_set
  std::map<std::pair<int32_t, int32_t>, std::set<int64_t>> good;       // good_loops_set, one entry per unordered pair
  // The device copy of the whole state, which reject_anchored reads and writes.  The first reject_anchored builds it from
  // the host record; from then on every host-side call that changes the state writes it through, and the first host-side
  // call after an anchored call synchronises once and refreshes the host record from it.
  bool dev = false;
  bool dev_ahead = false;               // an anchored call ran since the host record was refreshed
  bool ev_valid = false;
  osb_status last_anchored = OSB_OK;    // what status() reports
  osb_status pending = OSB_OK;          // reported once by the next host-side call
  cudaEvent_t ev = nullptr;             // recorded after each anchored call (not while its stream is being captured)
  PcmSlot* d_slots = nullptr;           // [max_pairs]
  int64_t* d_slot_key = nullptr;
  int32_t *d_slot_n = nullptr, *d_slot_dir = nullptr;
  PcmDir* d_dir = nullptr;
  int dir_cap = 0;
  std::vector<PcmDir> hdir;             // the directory as the host last wrote or read it
  std::vector<int64_t*> own;            // [dir] the entry's own buffer for a set_inliers set (or null)
  std::vector<int> own_cap;
  PcmMeta* d_meta = nullptr;
  unsigned long long* d_seen = nullptr;
  unsigned long long seen_mask = 0;
  int G = 0;                            // CTAs of the two row passes
  int cand_cap = 0;                     // max_pairs x pair_capacity: more fresh rows cannot fit
  int32_t *d_cnt = nullptr, *d_cand = nullptr, *d_cand_slot = nullptr, *d_cand_rank = nullptr, *d_order = nullptr;
  int32_t *d_pcnt = nullptr, *d_poff = nullptr;
  PcmPairJob* d_jobs = nullptr;
};

namespace {

std::pair<int32_t, int32_t> pair_key(int32_t a, int32_t b) { return {std::min(a, b), std::max(a, b)}; }

bool pcm_routed(const osb_pcm_state* s, std::pair<int32_t, int32_t> k) {   // :122-139
  return s->p.redundant || k.first == s->p.self_id || k.second == s->p.self_id;
}

size_t pcm_align(size_t b) { return (b + 15) & ~(size_t)15; }

// the one device slot of pair i: loops [cap], bit matrix [cap][stride], degree and clique scratch [cap] each, ids [cap],
// clique [1 + cap], inlier ids [cap]
osb_status pcm_acquire_slot(osb_pcm_state* s, int i) {
  PcmSlot& sl = s->slots[i];
  if (sl.edges) return OSB_OK;
  const size_t cap = (size_t)s->p.pair_capacity;
  const size_t o_bits = pcm_align(cap * sizeof(osb_loop_edge));
  const size_t o_deg = pcm_align(o_bits + cap * s->stride * sizeof(uint32_t));
  const size_t o_ids = pcm_align(o_deg + 2 * cap * sizeof(int32_t));
  const size_t o_clq = pcm_align(o_ids + cap * sizeof(int64_t));
  const size_t o_good = pcm_align(o_clq + (cap + 1) * sizeof(int32_t));
  unsigned char* base = nullptr;
  OSB_TRY(s->res.alloc(&base, o_good + cap * sizeof(int64_t)));
  sl.edges = (osb_loop_edge*)base;
  sl.bits = (uint32_t*)(base + o_bits);
  sl.deg = (int32_t*)(base + o_deg);
  sl.inter = sl.deg + cap;
  sl.ids = (int64_t*)(base + o_ids);
  sl.clique = (int32_t*)(base + o_clq);
  sl.good = (int64_t*)(base + o_good);
  return OSB_OK;
}

int pcm_dir_entry(osb_pcm_state* s, std::pair<int32_t, int32_t> k) {   // find or append
  const int64_t key = pcm_key(k.first, k.second);
  for (size_t e = 0; e < s->hdir.size(); ++e)
    if (s->hdir[e].key == key) return (int)e;
  s->hdir.push_back(PcmDir{key, nullptr, -1, -1, 0, 0});
  s->own.push_back(nullptr);
  s->own_cap.push_back(0);
  return (int)s->hdir.size() - 1;
}

// writes a good_loops_set to the device: into the slot's buffer when it fits, else into the entry's own buffer
osb_status pcm_upload_set(osb_pcm_state* s, int e, const std::set<int64_t>& g) {
  const std::vector<int64_t> v(g.begin(), g.end());
  PcmDir& d = s->hdir[e];
  const int n = (int)v.size();
  if (d.slot >= 0 && n <= s->p.pair_capacity) {
    d.gptr = s->slots[d.slot].good;
    d.gcap = s->p.pair_capacity;
  } else {
    if (s->own_cap[e] < std::max(n, 1)) {
      if (s->own[e]) s->res.release(s->own[e]);
      s->own[e] = nullptr;
      s->own_cap[e] = 0;
      OSB_TRY(s->res.alloc(&s->own[e], (size_t)std::max(n, 1)));
      s->own_cap[e] = std::max(n, 1);
    }
    d.gptr = s->own[e];
    d.gcap = s->own_cap[e];
  }
  d.gn = n;
  if (n > 0)
    OSB_CUDA(cudaMemcpyAsync(d.gptr, v.data(), (size_t)n * sizeof(int64_t), cudaMemcpyHostToDevice, s->stream));
  return OSB_OK;
}

// pair i's clique and inlier set to the device (after a host-side grow)
osb_status pcm_push_pair(osb_pcm_state* s, int i) {
  const osb_pcm_state::Pair& P = s->pairs[i];
  std::vector<int32_t> c(1 + P.clique.size());
  c[0] = (int32_t)P.clique.size();
  std::copy(P.clique.begin(), P.clique.end(), c.begin() + 1);
  OSB_CUDA(cudaMemcpyAsync(s->slots[i].clique, c.data(), c.size() * sizeof(int32_t), cudaMemcpyHostToDevice, s->stream));
  const int e = pcm_dir_entry(s, P.key);
  s->hdir[e].slot = i;
  const auto it = s->good.find(P.key);
  if (it != s->good.end()) OSB_TRY(pcm_upload_set(s, e, it->second));
  return OSB_OK;
}

// slot table, directory and counters to the device, then one synchronisation: the device copy is complete when a
// host-side call returns.  The directory keeps room for every pair without loops plus max_pairs more.
osb_status pcm_push_tables(osb_pcm_state* s) {
  const int np = (int)s->pairs.size();
  std::vector<int64_t> key(np);
  std::vector<int32_t> n(np), dir(np);
  int slotless = 0;
  for (const PcmDir& d : s->hdir) slotless += d.slot < 0;
  for (size_t e = 0; e < s->hdir.size(); ++e)
    if (s->hdir[e].slot >= 0) dir[s->hdir[e].slot] = (int32_t)e;
  for (int i = 0; i < np; ++i) {
    key[i] = pcm_key(s->pairs[i].key.first, s->pairs[i].key.second);
    n[i] = (int32_t)s->pairs[i].ids.size();
  }
  const int need = slotless + s->p.max_pairs;
  if (need > s->dir_cap) {
    if (s->d_dir) {
      OSB_CUDA(cudaStreamSynchronize(s->stream));
      s->res.release(s->d_dir);
      s->d_dir = nullptr;
    }
    s->dir_cap = 0;
    OSB_TRY(s->res.alloc(&s->d_dir, (size_t)need + 16));
    s->dir_cap = need + 16;
  }
  cudaStream_t st = s->stream;
  if (np > 0) {
    OSB_CUDA(cudaMemcpyAsync(s->d_slot_key, key.data(), np * sizeof(int64_t), cudaMemcpyHostToDevice, st));
    OSB_CUDA(cudaMemcpyAsync(s->d_slot_n, n.data(), np * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    OSB_CUDA(cudaMemcpyAsync(s->d_slot_dir, dir.data(), np * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  }
  if (!s->hdir.empty())
    OSB_CUDA(cudaMemcpyAsync(s->d_dir, s->hdir.data(), s->hdir.size() * sizeof(PcmDir), cudaMemcpyHostToDevice, st));
  const PcmMeta m{OSB_OK, np, (int32_t)s->hdir.size(), 0, 0, s->seen.count(INT64_MIN) ? 1 : 0};
  OSB_CUDA(cudaMemcpyAsync(s->d_meta, &m, sizeof(m), cudaMemcpyHostToDevice, st));
  OSB_CUDA(cudaStreamSynchronize(st));
  return OSB_OK;
}

// the first reject_anchored: every slot, the tables, the seen hash and the scratch of the anchored launches, filled from
// the host record
osb_status pcm_dev_init(osb_pcm_state* s) {
  const int P = s->p.max_pairs, cap = s->p.pair_capacity;
  Resources& R = s->res;
  cudaStream_t st = s->stream;
  for (int i = 0; i < P; ++i) OSB_TRY(pcm_acquire_slot(s, i));
  OSB_TRY(R.alloc(&s->d_slots, (size_t)P));
  OSB_TRY(R.alloc(&s->d_slot_key, (size_t)P));
  OSB_TRY(R.alloc(&s->d_slot_n, (size_t)P));
  OSB_TRY(R.alloc(&s->d_slot_dir, (size_t)P));
  OSB_TRY(R.alloc(&s->d_meta, 1));
  size_t H = 1024;
  while (H < 2 * (size_t)P * cap) H <<= 1;
  OSB_TRY(R.alloc(&s->d_seen, H));
  s->seen_mask = H - 1;
  s->G = num_sms();
  s->cand_cap = P * cap;
  OSB_TRY(R.alloc(&s->d_cnt, (size_t)s->G));
  OSB_TRY(R.alloc(&s->d_cand, (size_t)s->cand_cap));
  OSB_TRY(R.alloc(&s->d_cand_slot, (size_t)s->cand_cap));
  OSB_TRY(R.alloc(&s->d_cand_rank, (size_t)s->cand_cap));
  OSB_TRY(R.alloc(&s->d_order, (size_t)s->cand_cap));
  OSB_TRY(R.alloc(&s->d_pcnt, (size_t)P));
  OSB_TRY(R.alloc(&s->d_poff, (size_t)P));
  OSB_TRY(R.alloc(&s->d_jobs, (size_t)P));
  OSB_TRY(R.event(&s->ev, cudaEventDisableTiming));
  OSB_CUDA(cudaMemcpyAsync(s->d_slots, s->slots.data(), P * sizeof(PcmSlot), cudaMemcpyHostToDevice, st));
  std::vector<unsigned long long> table(H, PCM_EMPTY);
  for (int64_t id : s->seen) {
    if ((unsigned long long)id == PCM_EMPTY) continue;
    unsigned long long h = pcm_hash(id) & s->seen_mask;
    while (table[h] != PCM_EMPTY) h = (h + 1) & s->seen_mask;
    table[h] = (unsigned long long)id;
  }
  OSB_CUDA(cudaMemcpyAsync(s->d_seen, table.data(), H * sizeof(unsigned long long), cudaMemcpyHostToDevice, st));
  s->dev = true;
  for (int i = 0; i < (int)s->pairs.size(); ++i) OSB_TRY(pcm_push_pair(s, i));
  for (const auto& kv : s->good)
    if (!s->index.count(kv.first)) OSB_TRY(pcm_upload_set(s, pcm_dir_entry(s, kv.first), kv.second));
  return pcm_push_tables(s);
}

// after an anchored call: one synchronisation, then the host record is rebuilt from the device copy
osb_status pcm_refresh(osb_pcm_state* s) {
  if (!s->dev_ahead) return OSB_OK;
  DeviceGuard dg(s->device);
  cudaStream_t st = s->stream;
  if (s->ev_valid) OSB_CUDA(cudaEventSynchronize(s->ev));
  PcmMeta m{};
  OSB_CUDA(cudaMemcpyAsync(&m, s->d_meta, sizeof(m), cudaMemcpyDeviceToHost, st));
  OSB_CUDA(cudaStreamSynchronize(st));
  std::vector<int64_t> key(m.n_slots);
  std::vector<int32_t> n(m.n_slots);
  s->hdir.assign(m.n_dir, PcmDir{});
  if (m.n_slots > 0) {
    OSB_CUDA(cudaMemcpyAsync(key.data(), s->d_slot_key, m.n_slots * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    OSB_CUDA(cudaMemcpyAsync(n.data(), s->d_slot_n, m.n_slots * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  }
  if (m.n_dir > 0)
    OSB_CUDA(cudaMemcpyAsync(s->hdir.data(), s->d_dir, m.n_dir * sizeof(PcmDir), cudaMemcpyDeviceToHost, st));
  OSB_CUDA(cudaStreamSynchronize(st));
  s->pairs.resize(m.n_slots);
  s->index.clear();
  s->seen.clear();
  std::vector<int32_t> c(1 + s->p.pair_capacity);
  for (int i = 0; i < m.n_slots; ++i) {
    osb_pcm_state::Pair& P = s->pairs[i];
    P.key = {(int32_t)(key[i] >> 32), (int32_t)(uint32_t)key[i]};
    P.ids.resize(n[i]);
    if (n[i] > 0)
      OSB_CUDA(cudaMemcpyAsync(P.ids.data(), s->slots[i].ids, n[i] * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    OSB_CUDA(cudaMemcpyAsync(c.data(), s->slots[i].clique, c.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    OSB_CUDA(cudaStreamSynchronize(st));
    P.clique.assign(c.begin() + 1, c.begin() + 1 + c[0]);
    s->index[P.key] = i;
    s->seen.insert(P.ids.begin(), P.ids.end());
  }
  s->good.clear();
  s->own.resize(m.n_dir, nullptr);
  s->own_cap.resize(m.n_dir, 0);
  for (const PcmDir& d : s->hdir) {
    if (d.gn < 0) continue;
    std::vector<int64_t> g(d.gn);
    if (d.gn > 0) {
      OSB_CUDA(cudaMemcpyAsync(g.data(), d.gptr, d.gn * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
      OSB_CUDA(cudaStreamSynchronize(st));
    }
    s->good[{(int32_t)(d.key >> 32), (int32_t)(uint32_t)d.key}] = std::set<int64_t>(g.begin(), g.end());
  }
  s->last_anchored = s->pending = (osb_status)m.status;
  s->dev_ahead = false;
  return OSB_OK;
}

// every host-side call starts here: refresh after an anchored call, and report a refused anchored call once
osb_status pcm_host_entry(osb_pcm_state* s) {
  OSB_TRY(pcm_refresh(s));
  if (s->pending != OSB_OK) {
    const osb_status st = s->pending;
    s->pending = OSB_OK;
    set_error("osb_pcm_state", "the last reject_anchored call would exceed pair_capacity or max_pairs and changed nothing");
    return st;
  }
  return OSB_OK;
}

// appends the routed new loops (`fresh`: pair -> input indices in call order) and reruns maxCliqueHeu on every pair that
// gained any: one copy up, two launches, one copy down, one synchronisation.  The host record changes only on success.
osb_status pcm_state_grow(osb_pcm_state* s, const std::map<std::pair<int32_t, int32_t>, std::vector<int>>& fresh,
                          const osb_loop_edge* edges, const int64_t* ids) {
  for (const auto& kv : fresh)
    if (!s->index.count(kv.first)) {
      const int pi = (int)s->pairs.size();
      OSB_TRY(pcm_acquire_slot(s, pi));
      s->index[kv.first] = pi;
      osb_pcm_state::Pair P{};
      P.key = kv.first;
      s->pairs.push_back(std::move(P));
    }
  PcmPairJob* jobs = (PcmPairJob*)s->h_stage;
  osb_loop_edge* staged = (osb_loop_edge*)(s->h_stage + s->jobs_bytes);
  int64_t* staged_ids = (int64_t*)(s->h_stage + s->jobs_bytes + s->edges_bytes);
  int k = 0, n_staged = 0;
  long long items = 0;
  size_t smem = 0;
  std::vector<int> changed;
  for (const auto& kv : fresh) {
    const int pi = s->index[kv.first];
    osb_pcm_state::Pair& P = s->pairs[pi];
    const PcmSlot& sl = s->slots[pi];
    const int m = (int)P.ids.size(), n = m + (int)kv.second.size(), W = (n + 31) / 32;
    jobs[k] = PcmPairJob{sl.edges, sl.bits, sl.deg, sl.inter, m, n, n_staged, (int32_t)items};
    jobs[k].ids = sl.ids;
    jobs[k++].slot = pi;
    for (int i : kv.second) {
      staged_ids[n_staged] = ids[i];
      staged[n_staged++] = edges[i];
    }
    items += (long long)m * (W - (m >> 5)) + (long long)(n - m) * W;
    const size_t need = (size_t)n * W * 4;
    if (need <= 200 * 1024) smem = std::max(smem, need);
    changed.push_back(pi);
    OSB_REQUIRE(items < (1ll << 31), "too many pair checks in one call");
  }
  cudaStream_t st = s->stream;
  OSB_CUDA(cudaMemcpyAsync(s->d_stage, s->h_stage, s->jobs_bytes + (size_t)n_staged * sizeof(osb_loop_edge),
                           cudaMemcpyHostToDevice, st));
  OSB_CUDA(cudaMemcpyAsync(s->d_stage + s->jobs_bytes + s->edges_bytes, staged_ids, (size_t)n_staged * sizeof(int64_t),
                           cudaMemcpyHostToDevice, st));
  const PcmPairJob* d_jobs = (const PcmPairJob*)s->d_stage;
  const PcmFresh f{s->d_stage + s->jobs_bytes, s->d_stage + s->jobs_bytes + s->edges_bytes, nullptr,
                   (long long)sizeof(osb_loop_edge), (long long)sizeof(int64_t)};
  const PcmSeen seen{s->d_seen, s->seen_mask, s->d_meta};         // null table until the device copy exists
  OSB_LAUNCH(pcm_grow_kernel, cdiv((int)items, 128), 128, 0, st, d_jobs, k, (int)items, (const PcmMeta*)nullptr, f, seen,
             s->stride, s->p.pcm_thres, s->p.odom_pos_cov_per_m, s->p.odom_ang_cov_per_m);
  OSB_CHECK_LAUNCH();
  OSB_SMEM_OPT_IN(pcm_max_clique_kernel, 200 * 1024);
  const int out_step = 1 + s->p.pair_capacity;
  OSB_LAUNCH(pcm_max_clique_kernel, k, 32, smem, st, d_jobs, PcmPairJob{}, s->stride, s->d_out + 1, s->d_out, out_step,
             (uint8_t*)nullptr, (const int32_t*)nullptr);
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
  if (s->dev) {
    for (int pi : changed) OSB_TRY(pcm_push_pair(s, pi));
    OSB_TRY(pcm_push_tables(s));
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
  s->edges_bytes = (size_t)p->max_pairs * p->pair_capacity * sizeof(osb_loop_edge);
  const size_t stage = s->jobs_bytes + s->edges_bytes + (size_t)p->max_pairs * p->pair_capacity * sizeof(int64_t);
  const size_t outs = (size_t)p->max_pairs * (1 + p->pair_capacity);
  s->slots.assign(p->max_pairs, PcmSlot{});
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
  OSB_TRY(pcm_host_entry(s));
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

extern "C" osb_status osb_pcm_state_reject_anchored(osb_pcm_state* s, const osb_anchor_result* rows_dev, int n,
                                                    uint8_t* keep_dev, void* stream) {
  OSB_REQUIRE(s != nullptr && n >= 0, "null state or negative count");
  OSB_REQUIRE(n == 0 || (rows_dev && keep_dev), "null argument");
  if (n == 0) return OSB_OK;
  std::lock_guard<std::mutex> lk(s->mu);
  DeviceGuard dg(s->device);
  if (!s->dev) {
    OSB_TRY(pcm_refresh(s));
    OSB_TRY(pcm_dev_init(s));
  }
  cudaStream_t st = (cudaStream_t)stream;
  const PcmSeen seen{s->d_seen, s->seen_mask, s->d_meta};
  const PcmRows v{rows_dev, n, s->p.self_id, s->p.redundant, seen};
  OSB_LAUNCH(pcm_anchored_count_kernel, s->G, 256, 0, st, v, s->d_cnt);
  OSB_CHECK_LAUNCH();
  OSB_LAUNCH(pcm_anchored_collect_kernel, s->G, 256, 0, st, v, s->d_cnt, s->d_cand, s->cand_cap);
  OSB_CHECK_LAUNCH();
  const PcmPlan plan{rows_dev, s->d_cnt, s->G, s->d_cand, s->d_cand_slot, s->d_cand_rank, s->cand_cap, s->d_order,
                     s->d_slot_key, s->d_slot_n, s->d_slot_dir, s->d_slots, s->d_dir, s->d_meta, s->d_pcnt, s->d_poff,
                     s->d_jobs, s->p.max_pairs, s->p.pair_capacity};
  OSB_LAUNCH(pcm_anchored_plan_kernel, 1, 32, 0, st, plan);
  OSB_CHECK_LAUNCH();
  const unsigned char* base = reinterpret_cast<const unsigned char*>(rows_dev);
  const PcmFresh f{base + offsetof(osb_anchor_result, edge), base + offsetof(osb_anchor_result, id), s->d_order,
                   (long long)sizeof(osb_anchor_result), (long long)sizeof(osb_anchor_result)};
  OSB_LAUNCH(pcm_grow_kernel, 4 * s->G, 128, 0, st, s->d_jobs, 0, 0, s->d_meta, f, seen, s->stride, s->p.pcm_thres,
             s->p.odom_pos_cov_per_m, s->p.odom_ang_cov_per_m);
  OSB_CHECK_LAUNCH();
  OSB_SMEM_OPT_IN(pcm_max_clique_kernel, 200 * 1024);
  const int out_step = 1 + s->p.pair_capacity;
  OSB_LAUNCH(pcm_max_clique_kernel, s->p.max_pairs, 32, 200 * 1024, st, s->d_jobs, PcmPairJob{}, s->stride, s->d_out + 1,
             s->d_out, out_step, (uint8_t*)nullptr, (const int32_t*)&s->d_meta->n_jobs);
  OSB_CHECK_LAUNCH();
  OSB_LAUNCH(pcm_anchored_finish_kernel, s->p.max_pairs, PCM_FINISH_THREADS, 0, st, s->d_jobs, s->d_meta, s->d_out,
             out_step, s->d_slots, s->d_slot_dir, s->d_dir, s->p.pair_capacity);
  OSB_CHECK_LAUNCH();
  OSB_LAUNCH(pcm_anchored_keep_kernel, cdiv(n, 256), 256, 0, st, rows_dev, n, s->d_dir, s->d_meta, keep_dev);
  OSB_CHECK_LAUNCH();
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  OSB_CUDA(cudaStreamIsCapturing(st, &cs));
  s->ev_valid = cs == cudaStreamCaptureStatusNone;
  if (s->ev_valid) OSB_CUDA(cudaEventRecord(s->ev, st));
  s->dev_ahead = true;
  return OSB_OK;
}

extern "C" osb_status osb_pcm_state_status(osb_pcm_state* s, osb_status* last) {
  OSB_REQUIRE(s != nullptr && last != nullptr, "null argument");
  std::lock_guard<std::mutex> lk(s->mu);
  OSB_TRY(pcm_refresh(s));
  *last = s->last_anchored;
  return *last;
}

extern "C" osb_status osb_pcm_state_inliers(osb_pcm_state* s, int32_t id_a, int32_t id_b, int64_t* ids, int cap,
                                            int32_t* n) {
  OSB_REQUIRE(s != nullptr && n != nullptr && cap >= 0, "null argument or negative capacity");
  std::lock_guard<std::mutex> lk(s->mu);
  OSB_TRY(pcm_host_entry(s));
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
  OSB_TRY(pcm_host_entry(s));
  if (id_a == s->p.self_id || id_b == s->p.self_id) return OSB_OK;    // :40-43
  const auto k = pair_key(id_a, id_b);
  s->good[k] = std::set<int64_t>(ids, ids + n);
  if (s->dev) {
    DeviceGuard dg(s->device);
    OSB_TRY(pcm_upload_set(s, pcm_dir_entry(s, k), s->good[k]));
    OSB_TRY(pcm_push_tables(s));
  }
  return OSB_OK;
}

extern "C" osb_status osb_pcm_state_pair(osb_pcm_state* s, int32_t id_a, int32_t id_b, int32_t* n, int64_t* ids,
                                         uint8_t* adj, int32_t* clique, int32_t* clique_size) {
  OSB_REQUIRE(s != nullptr && n != nullptr, "null argument");
  std::lock_guard<std::mutex> lk(s->mu);
  DeviceGuard dg(s->device);
  OSB_TRY(pcm_host_entry(s));
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
    OSB_CUDA(cudaMemcpy2DAsync(rows.data(), W * sizeof(uint32_t), s->slots[it->second].bits, s->stride * sizeof(uint32_t),
                               W * sizeof(uint32_t), m, cudaMemcpyDeviceToHost, s->stream));
    OSB_CUDA(cudaStreamSynchronize(s->stream));
    for (int i = 0; i < m; ++i)
      for (int j = 0; j < m; ++j) adj[(size_t)i * m + j] = (rows[(size_t)i * W + (j >> 5)] >> (j & 31)) & 1u;
  }
  return OSB_OK;
}
