// anchor.cu -- re-anchoring of every loop and detection onto the sliding window, on the device (SURVEY.md 8f-4).
//
// Replaces the walk of SwarmLocalizationSolver::find_available_loops_detections (swarm_localization_solver.cpp:1594-1666)
// that every solve() makes over all_loops and all_detections_6d: loop_from_src_loop_connection (:1464-1553) with
// find_node_frame_for_measurement_2drones (:1429-1462), and the factor choice of setup_problem_with_loops_and_detections
// (:1064-1100).  anchor_kernel runs one warp per measurement:
//   1. the lanes scan drone a's and drone b's vo_available window entries (a per-drone index built by set_window, frame
//      order) and a warp arg-min on (|stamp difference|, frame) finds each anchor -- the reference's strict `<` over frames
//      in order keeps the earliest frame of equal differences;
//   2. four lanes run the four nearest-sample binary searches of the trajectory look-ups at once;
//   3. lane 0 does the fp64 pose algebra and the 4x4 sqrt-information of the factor row into shared memory, and the warp
//      stores the row coalesced.
// The trajectories, measurements and window stay on the device between runs; only what a call adds crosses PCIe.
// DroneTrajectory / NodeFrame / LoopEdge arithmetic is defined in oracle/anchor_ref.py (swarm_msgs is not in the tree).
// Built with -fmad=false (Makefile) so every product is rounded as the oracle rounds it.
#include <climits>

#include "common.cuh"
#include "pose_algebra.cuh"

namespace osb {

constexpr int ANCHOR_MAX_DRONES = 256;
constexpr int ANCHOR_WARPS = 8;                                    // warps (= measurements) per CTA
constexpr int64_t ANCHOR_MAX_ERR_NS = 10000ll * 1000000000ll;      // min_ts_err's start, 10000 s (:1436-1437)
constexpr int MEAS_WORDS = (int)(sizeof(osb_measurement) / 8);
constexpr int RESULT_WORDS = (int)(sizeof(osb_anchor_result) / 8);

struct AnchorView {
  const osb_measurement* meas;     // [max_measurements] in arrival order
  const int32_t* loop_slot;        // all_loops[i] = meas[loop_slot[i]]
  const int32_t* det_slot;         // all_detections_6d[i] = meas[det_slot[i]]
  int n_loops, n_total;
  const int32_t* counts;           // [2] loops, detections on the device while a device append may be in flight (then
                                   // n_loops / n_total are unused), else null
  int n_bound;                     // rows written: n_total, or the host's bound of it; rows n_total.. are OSB_ANCHOR_VOID
  const int64_t* traj_stamp;       // [max_drones][max_samples]
  const double* traj_pose;         // [max_drones][max_samples][7]
  const double* traj_len;          // [max_drones][max_samples]
  const int32_t* traj_n;           // [max_drones]
  int max_samples, max_drones;
  const int32_t* drone_first;      // [max_drones + 1]: drone d's vo_available entries are [drone_first[d], drone_first[d+1])
  const int64_t* win_stamp;
  const int32_t* win_frame;
  const int32_t* win_block;
  const double* win_pose;          // [n][7]
  int n_frames;
  int64_t frame0_stamp, begin_dt_ns;
  double dpos_thres, pos_cov, ang_cov;
  int huber;
  uint64_t yaw_obs[ANCHOR_MAX_DRONES / 64];
};

// warp arg-min over drone d's entries of (|stamp - t|, entry); only differences below 10000 s count.  -> entry or -1
__device__ __forceinline__ int anchor_search(const AnchorView& v, int d, int64_t t, int64_t* err_out) {
  const int lane = threadIdx.x & 31;
  int64_t best = ANCHOR_MAX_ERR_NS;
  int idx = INT_MAX;
  if (d >= 0 && d < v.max_drones) {
    const int lo = v.drone_first[d], hi = v.drone_first[d + 1];
    for (int k = lo + lane; k < hi; k += 32) {                    // k ascends, so the first hit of a lane is its earliest
      const int64_t diff = v.win_stamp[k] - t;
      const int64_t e = diff < 0 ? -diff : diff;
      if (e < best) { best = e; idx = k; }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const int64_t eo = __shfl_xor_sync(0xffffffffu, best, o);
    const int io = __shfl_xor_sync(0xffffffffu, idx, o);
    if (eo < best || (eo == best && io < idx)) { best = eo; idx = io; }
  }
  *err_out = best;
  return idx == INT_MAX ? -1 : idx;
}

// DroneTrajectory look-up: the sample nearest to t, ties to the earlier one, clamped to the first / last sample
__device__ __forceinline__ int nearest_sample(const int64_t* __restrict__ s, int n, int64_t t) {
  int lo = 0, hi = n;                                              // first k with s[k] >= t
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (s[mid] < t) lo = mid + 1; else hi = mid;
  }
  if (lo == 0) return 0;
  if (lo == n) return n - 1;
  return (t - s[lo - 1]) <= (s[lo] - t) ? lo - 1 : lo;
}

// RelativePoseFactor4d::CreateCov6d: S = sqrt|inv(blkdiag(cov[0:3,0:3], cov[5,5]))|, Gauss-Jordan with partial pivoting
__device__ void sqrt_information_4d(const double* cov, double* S) {
  double A[4][8];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) A[i][j] = (j == i + 4) ? 1.0 : 0.0;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) A[i][j] = cov[i * 6 + j];
  A[3][3] = cov[35];
  for (int c = 0; c < 4; ++c) {
    int p = c;
    for (int r = c + 1; r < 4; ++r)
      if (fabs(A[r][c]) > fabs(A[p][c])) p = r;
    if (p != c)
      for (int j = 0; j < 8; ++j) { const double x = A[c][j]; A[c][j] = A[p][j]; A[p][j] = x; }
    const double piv = A[c][c];
    for (int j = 0; j < 8; ++j) A[c][j] /= piv;
    for (int r = 0; r < 4; ++r) {
      if (r == c) continue;
      const double f = A[r][c];
      for (int j = 0; j < 8; ++j) A[r][j] -= f * A[c][j];
    }
  }
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) S[i * 4 + j] = sqrt(fabs(A[i][4 + j]));
}

__device__ __forceinline__ void store_pose(double* dst, const PoseD& p) {
  dst[0] = p.t[0]; dst[1] = p.t[1]; dst[2] = p.t[2]; dst[3] = p.q[0]; dst[4] = p.q[1]; dst[5] = p.q[2]; dst[6] = p.q[3];
}

__global__ void __launch_bounds__(ANCHOR_WARPS * 32)
anchor_kernel(const AnchorView v, osb_anchor_result* __restrict__ out) {
  __shared__ double s_meas[ANCHOR_WARPS][MEAS_WORDS];
  __shared__ double s_out[ANCHOR_WARPS][RESULT_WORDS];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i = blockIdx.x * ANCHOR_WARPS + w;
  if (i >= v.n_bound) return;                                      // warp-uniform
  const int n_loops = v.counts ? v.counts[0] : v.n_loops;
  const int n_total = v.counts ? n_loops + v.counts[1] : v.n_total;
  for (int k = lane; k < RESULT_WORDS; k += 32) s_out[w][k] = 0.0;
  if (i >= n_total) {                                              // past the true count: a VOID row, skipped downstream
    __syncwarp();
    if (lane == 0) {
      osb_anchor_result& r = *reinterpret_cast<osb_anchor_result*>(s_out[w]);
      r.status = OSB_ANCHOR_VOID;
      r.skip = 1;
    }
    __syncwarp();
    double* dst = reinterpret_cast<double*>(out + i);
    for (int j = lane; j < RESULT_WORDS; j += 32) dst[j] = s_out[w][j];
    return;
  }
  const int slot = i < n_loops ? v.loop_slot[i] : v.det_slot[i - n_loops];
  const double* src = reinterpret_cast<const double*>(v.meas + slot);
  for (int k = lane; k < MEAS_WORDS; k += 32) s_meas[w][k] = src[k];
  __syncwarp();
  const osb_measurement& m = *reinterpret_cast<const osb_measurement*>(s_meas[w]);
  osb_anchor_result& r = *reinterpret_cast<osb_anchor_result*>(s_out[w]);

  int status = OSB_ANCHOR_OK;
  int ea = -1, eb = -1;
  int64_t err_a = ANCHOR_MAX_ERR_NS, err_b = ANCHOR_MAX_ERR_NS;
  if (v.n_frames == 0) status = OSB_ANCHOR_EMPTY_WINDOW;                                       // :1479-1482
  else if (v.frame0_stamp - m.stamp_a > v.begin_dt_ns) status = OSB_ANCHOR_BEFORE_WINDOW;      // :1484
  else {
    ea = anchor_search(v, m.id_a, m.stamp_a, &err_a);                                          // :1440-1452
    eb = anchor_search(v, m.id_b, m.stamp_b, &err_b);
    if (ea < 0 || eb < 0) status = OSB_ANCHOR_NO_FRAME;                                        // :1456-1461
    else if (v.traj_n[m.id_a] == 0 || v.traj_n[m.id_b] == 0) status = OSB_ANCHOR_NO_TRAJECTORY;
  }
  // the four trajectory look-ups of :1507-1527, one per lane: a at (anchor a, stamp_a), b at (anchor b, stamp_b)
  int k = 0;
  if (status == OSB_ANCHOR_OK && lane < 4) {
    const int d = lane < 2 ? m.id_a : m.id_b;
    const int64_t t = lane == 0 ? v.win_stamp[ea] : lane == 1 ? m.stamp_a : lane == 2 ? v.win_stamp[eb] : m.stamp_b;
    k = nearest_sample(v.traj_stamp + (size_t)d * v.max_samples, v.traj_n[d], t);
  }
  const int k_nfa = __shfl_sync(0xffffffffu, k, 0), k_a = __shfl_sync(0xffffffffu, k, 1);
  const int k_nfb = __shfl_sync(0xffffffffu, k, 2), k_b = __shfl_sync(0xffffffffu, k, 3);

  if (lane == 0) {
    r.id = m.id;
    r.type = m.type;
    r.frame_a = r.frame_b = r.node_a = r.node_b = -1;
    r.ia = r.ib = -1;
    r.factor_type = OSB_FACTOR_RELPOSE;
    r.huber = v.huber;
    if (status != OSB_ANCHOR_EMPTY_WINDOW && status != OSB_ANCHOR_BEFORE_WINDOW) {
      r.dt_err_ns = err_a + err_b;
      if (ea >= 0) { r.frame_a = v.win_frame[ea]; r.node_a = v.win_block[ea]; r.stamp_a = v.win_stamp[ea]; }
      if (eb >= 0) { r.frame_b = v.win_frame[eb]; r.node_b = v.win_block[eb]; r.stamp_b = v.win_stamp[eb]; }
      r.ia = r.node_a;
      r.ib = r.node_b;
    }
    if (status == OSB_ANCHOR_OK) {
      const size_t ba = (size_t)m.id_a * v.max_samples, bb = (size_t)m.id_b * v.max_samples;
      const double len_nfa = v.traj_len[ba + k_nfa], len_nfb = v.traj_len[bb + k_nfb];
      const double da = fabs(v.traj_len[ba + k_a] - len_nfa);     // covariance_between_appro_ts / trajectory_length_by_appro_ts
      const double db = fabs(v.traj_len[bb + k_b] - len_nfb);
      PoseD self_a = load_pose(m.self_pose_a), self_b = load_pose(m.self_pose_b);
      if (m.type != OSB_MEAS_LOOP) {                                                           // :1510-1517
        self_a = load_pose(v.traj_pose + (ba + k_a) * 7);
        self_b = load_pose(v.traj_pose + (bb + k_b) * 7);
        if (m.type == OSB_MEAS_DET4D) { self_a = pose_yaw_only(self_a); self_b = pose_yaw_only(self_b); }
      }
      const PoseD nfa = load_pose(v.win_pose + (size_t)ea * 7), nfb = load_pose(v.win_pose + (size_t)eb * 7);
      const PoseD loop = pose_mul(pose_mul(delta_pose4(nfa, self_a), load_pose(m.relative_pose)),   // :1519-1522
                                  delta_pose4(self_b, nfb));
      r.dpos = da + db;                                                                        // :1524-1532
      if (r.dpos > v.dpos_thres) status = OSB_ANCHOR_DPOS;
      osb_loop_edge& e = r.edge;
      e.id_a = m.id_a;
      e.id_b = m.id_b;
      store_pose(e.rel_pose, loop);
      for (int j = 0; j < 36; ++j) {                                                           // :1548
        const double per_m = (j % 7 == 0) ? (j < 21 ? v.pos_cov : v.ang_cov) : 0.0;
        e.cov[j] = m.cov[j] + (da * per_m + db * per_m);
      }
      store_pose(e.odom_a, nfa);
      store_pose(e.odom_b, nfb);
      e.len_a = len_nfa;
      e.len_b = len_nfb;
      r.payload[0] = loop.t[0];
      r.payload[1] = loop.t[1];
      r.payload[2] = loop.t[2];
      r.payload[3] = quat_yaw(loop.q);
      sqrt_information_4d(e.cov, r.payload + 4);
    }
    r.status = status;
    const bool observable = status == OSB_ANCHOR_OK && ((v.yaw_obs[m.id_a >> 6] >> (m.id_a & 63)) & 1ull) &&
                            ((v.yaw_obs[m.id_b >> 6] >> (m.id_b & 63)) & 1ull);
    r.skip = (observable && r.node_a != r.node_b) ? 0 : 1;                                     // :1066-1073
  }
  __syncwarp();
  double* dst = reinterpret_cast<double*>(out + i);
  for (int j = lane; j < RESULT_WORDS; j += 32) dst[j] = s_out[w][j];
}

// setup_problem_with_loops_and_detections on the device: the rows with skip == 0 (and keep[i]) become the solver's SoA in
// row order.  One CTA streams the rows in tiles of COMPACT_THREADS x COMPACT_ROWS; thread t owns COMPACT_ROWS consecutive
// rows of a tile and a block scan of the per-thread counts gives each kept row its output index (no atomics, so the order
// and the bytes are the same on every run).
constexpr int COMPACT_THREADS = 1024, COMPACT_ROWS = 4;
__global__ void __launch_bounds__(COMPACT_THREADS)
anchor_compact_kernel(const osb_anchor_result* __restrict__ rows, int n, const uint8_t* __restrict__ keep,
                      int32_t* __restrict__ type, int32_t* __restrict__ ia, int32_t* __restrict__ ib,
                      double* __restrict__ payload, uint8_t* __restrict__ huber, int32_t* __restrict__ count) {
  __shared__ int s_warp[COMPACT_THREADS / 32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int out_base = 0;
  for (int base = 0; base < n; base += COMPACT_THREADS * COMPACT_ROWS) {
    const int first = base + threadIdx.x * COMPACT_ROWS;
    bool sel[COMPACT_ROWS];
    int mine = 0;
#pragma unroll
    for (int r = 0; r < COMPACT_ROWS; ++r) {
      const int i = first + r;
      sel[r] = i < n && rows[i].skip == 0 && (keep == nullptr || keep[i] != 0);
      mine += sel[r];
    }
    int inc = mine;                                                // warp-inclusive scan, then across warps
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += u;
    }
    if (lane == 31) s_warp[wid] = inc;
    __syncthreads();
    if (wid == 0) {
      int t = s_warp[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int u = __shfl_up_sync(0xffffffffu, t, o);
        if (lane >= o) t += u;
      }
      s_warp[lane] = t;
    }
    __syncthreads();
    int k = out_base + (wid > 0 ? s_warp[wid - 1] : 0) + inc - mine;
    const int total = s_warp[COMPACT_THREADS / 32 - 1];
#pragma unroll
    for (int r = 0; r < COMPACT_ROWS; ++r) {
      if (!sel[r]) continue;
      const osb_anchor_result& row = rows[first + r];
      type[k] = row.factor_type;
      ia[k] = row.ia;
      ib[k] = row.ib;
      huber[k] = (uint8_t)(row.huber != 0);
      for (int j = 0; j < OSB_PAYLOAD_LEN; ++j) payload[(size_t)k * OSB_PAYLOAD_LEN + j] = row.payload[j];
      ++k;
    }
    out_base += total;
    __syncthreads();                                               // s_warp is rewritten by the next tile
  }
  if (threadIdx.x == 0) *count = out_base;
}

// Row-count feedback of the device append, written into mapped pinned host memory as the front-end's FeFeedback is: the last
// append that has run reports the true counts, its status and how much had been charged to the host's bound when it was
// enqueued, so bound = count + what was charged since.  seq_begin / seq_end make a torn read detectable.
struct AnchorFeedback {
  volatile long long seq_begin;
  volatile long long n_loops, n_dets, charged, status;
  volatile long long seq_end;
};

// add_new_loop_connection / add_new_detection for rows [0, *count) of a device buffer (solver.cpp:558-588): one CTA.
// Pass 1 validates every row and counts what the distance gate keeps; a refused call writes nothing but the feedback.
// Pass 2 appends tile by tile: a block scan of (kept loop, kept detection) per thread gives each row its arrival slot and
// its place in the loop or detection list, in row order (no atomics).
constexpr int APPEND_THREADS = 256;

// exclusive block scan over APPEND_THREADS threads; *total = the block's sum.  Ends with a barrier, so it can be called again.
__device__ __forceinline__ int append_block_scan(int v, int* total) {
  __shared__ int s_warp[APPEND_THREADS / 32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int u = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += u;
  }
  if (lane == 31) s_warp[wid] = inc;
  __syncthreads();
  int base = 0, sum = 0;
#pragma unroll
  for (int w = 0; w < APPEND_THREADS / 32; ++w) { if (w < wid) base += s_warp[w]; sum += s_warp[w]; }
  __syncthreads();
  *total = sum;
  return base + inc - v;
}

// the reference's gate: relative_pose.pos().norm() > loop_outlier_distance_threshold drops a loop; detections pass
__device__ __forceinline__ bool append_keeps(const osb_measurement& r, float thres) {
  if (r.type != OSB_MEAS_LOOP) return true;
  const double* p = r.relative_pose;
  const double d = sqrt(__dadd_rn(__dadd_rn(__dmul_rn(p[0], p[0]), __dmul_rn(p[1], p[1])), __dmul_rn(p[2], p[2])));
  return !(d > (double)thres);
}

__global__ void __launch_bounds__(APPEND_THREADS)
anchor_append_kernel(const osb_measurement* __restrict__ m, const int32_t* __restrict__ count_dev, int max_n, float thres,
                     int max_drones, int max_meas, osb_measurement* __restrict__ meas, int32_t* __restrict__ loop_slot,
                     int32_t* __restrict__ det_slot, int32_t* __restrict__ counts, AnchorFeedback* __restrict__ fb,
                     long long seq, long long charged) {
  __shared__ int s_bad;
  const int tid = threadIdx.x;
  const int n = *count_dev;
  const int have_l = counts[0], have_d = counts[1];               // thread 0 rewrites them after the last barrier
  if (tid == 0) s_bad = 0;
  __syncthreads();
  int status = (n < 0 || n > max_n) ? OSB_ERR_INVALID : OSB_OK;
  int kept = 0;
  if (status == OSB_OK)
#pragma unroll 1
    for (int i = tid; i < n; i += APPEND_THREADS) {
      const osb_measurement& r = m[i];
      const bool ok = (r.type == OSB_MEAS_LOOP || r.type == OSB_MEAS_DET4D || r.type == OSB_MEAS_DET6D) &&
                      r.id_a >= 0 && r.id_a < max_drones && r.id_b >= 0 && r.id_b < max_drones;
      if (!ok) s_bad = 1;
      else kept += append_keeps(r, thres);
    }
  int total;
  append_block_scan(kept, &total);                                 // its barriers also publish s_bad
  if (status == OSB_OK && s_bad) status = OSB_ERR_INVALID;
  if (status == OSB_OK && (long long)have_l + have_d + total > max_meas) status = OSB_ERR_CAPACITY;
  int nl = 0, nd = 0;                                              // kept loops / detections of the tiles before
  if (status == OSB_OK)
#pragma unroll 1
    for (int base = 0; base < n; base += APPEND_THREADS) {
      const int i = base + tid;
      const bool kept_i = i < n && append_keeps(m[i], thres);
      const int loop = kept_i && m[i].type == OSB_MEAS_LOOP, det = kept_i && m[i].type != OSB_MEAS_LOOP;
      int tile;
      const int ex = append_block_scan(loop | (det << 16), &tile);   // a tile's counts fit 16 bits each
      if (loop | det) {
        const int el = ex & 0xffff, ed = ex >> 16;
        const int slot = have_l + have_d + nl + nd + el + ed;     // arrival order
        const double* src = reinterpret_cast<const double*>(m + i);
        double* dst = reinterpret_cast<double*>(meas + slot);
        for (int k = 0; k < MEAS_WORDS; ++k) dst[k] = src[k];
        if (loop) loop_slot[have_l + nl + el] = slot;
        else det_slot[have_d + nd + ed] = slot;
      }
      nl += tile & 0xffff;
      nd += tile >> 16;
    }
  if (tid != 0) return;
  if (status == OSB_OK) { counts[0] = have_l + nl; counts[1] = have_d + nd; }
  fb->seq_begin = seq;
  __threadfence_system();
  fb->n_loops = status == OSB_OK ? have_l + nl : have_l;
  fb->n_dets = status == OSB_OK ? have_d + nd : have_d;
  fb->charged = charged;
  fb->status = status;
  __threadfence_system();
  fb->seq_end = seq;
}

}  // namespace osb

using namespace osb;

static_assert(sizeof(osb_measurement) == 496, "osb_measurement layout");
static_assert(sizeof(osb_window_entry) == 80, "osb_window_entry layout");
static_assert(sizeof(osb_anchor_result) == 760, "osb_anchor_result layout");

struct osb_anchor {
  Resources res;
  int device = 0;
  osb_anchor_params p{};
  int64_t begin_dt_ns = 0;
  cudaStream_t stream = nullptr;
  cudaEvent_t last_run = nullptr;     // recorded after every run: updates wait for it before they overwrite state
  std::mutex mu;
  // device state
  osb_measurement* d_meas = nullptr;
  int32_t *d_loop_slot = nullptr, *d_det_slot = nullptr;
  int64_t* d_traj_stamp = nullptr;
  double *d_traj_pose = nullptr, *d_traj_len = nullptr;
  int32_t* d_traj_n = nullptr;
  int32_t* d_drone_first = nullptr;
  int64_t* d_win_stamp = nullptr;
  int32_t *d_win_frame = nullptr, *d_win_block = nullptr;
  double* d_win_pose = nullptr;
  osb_anchor_result* d_out = nullptr;
  // device appends (osb_anchor_add_measurements_dev), acquired by the first one: the counts on the device, their feedback
  // (mapped pinned memory + its device alias) and an event recorded after every append
  int32_t* d_counts = nullptr;                    // [2] loops, detections
  AnchorFeedback* fb_host = nullptr;
  AnchorFeedback* fb_dev = nullptr;
  cudaEvent_t last_append = nullptr;
  bool append_pending = false;                    // an append may not have run: n_loops / n_dets are stale, `upper` bounds them
  long long append_seq = 0, fb_min_seq = 1;       // feedback older than fb_min_seq carries nothing new
  long long charged = 0;                          // max_n summed over every device append
  long long upper = 0;                            // bound of n_loops + n_dets while append_pending
  osb_status last_status = OSB_OK;                // the last device append's, once synchronised
  // host record
  int n_loops = 0, n_dets = 0;
  std::vector<int32_t> traj_n;
  std::vector<int64_t> last_stamp;
  std::vector<double> last_pos, last_len;     // [max_drones][3], [max_drones]
  int n_frames = 0;
  int64_t frame0_stamp = 0;
  // set_window staging (sized at create)
  std::vector<int32_t> h_drone_first, h_win_frame, h_win_block, h_slot;
  std::vector<int64_t> h_win_stamp;
  std::vector<double> h_win_pose, h_len;
};

namespace {

osb_status anchor_wait_last_run(osb_anchor* h) {
  OSB_CUDA(cudaStreamWaitEvent(h->stream, h->last_run, 0));
  return OSB_OK;
}

bool drone_ok(const osb_anchor* h, int32_t d) { return d >= 0 && d < h->p.max_drones; }

// wait for the last device append and take its exact counts and status (every synchronising call starts with this)
osb_status anchor_settle(osb_anchor* h) {
  if (!h->append_pending) return OSB_OK;
  OSB_CUDA(cudaEventSynchronize(h->last_append));
  const AnchorFeedback* fb = h->fb_host;
  h->n_loops = (int)fb->n_loops;
  h->n_dets = (int)fb->n_dets;
  h->last_status = (osb_status)fb->status;
  h->upper = h->n_loops + h->n_dets;
  h->append_pending = false;
  h->fb_min_seq = h->append_seq + 1;
  return OSB_OK;
}

// lower the bound with what the most recent append that has RUN reported (no synchronisation)
void anchor_tighten(osb_anchor* h) {
  const AnchorFeedback* fb = h->fb_host;
  const long long e = fb->seq_end;
  std::atomic_thread_fence(std::memory_order_acquire);
  const long long nl = fb->n_loops, nd = fb->n_dets, ch = fb->charged;
  std::atomic_thread_fence(std::memory_order_acquire);
  const long long b = fb->seq_begin;
  if (b != e || e < h->fb_min_seq) return;
  h->upper = std::min(h->upper, nl + nd + (h->charged - ch));
}

}  // namespace

extern "C" osb_status osb_anchor_create(osb_anchor** out, const osb_anchor_params* p) {
  OSB_REQUIRE(out != nullptr && p != nullptr, "null argument");
  OSB_REQUIRE(p->max_drones > 0 && p->max_drones <= ANCHOR_MAX_DRONES, "max_drones must be in 1..256");
  OSB_REQUIRE(p->max_traj_samples > 0 && p->max_measurements > 0 && p->max_window_entries > 0, "capacities must be positive");
  OSB_REQUIRE((long long)p->max_drones * p->max_traj_samples < (1ll << 31), "max_drones x max_traj_samples too large");
  OSB_REQUIRE(p->begin_min_loop_dt_s >= 0.0 && p->begin_min_loop_dt_s < 9.0e9, "begin_min_loop_dt_s out of range");
  OSB_TRY(require_device());
  std::unique_ptr<osb_anchor> h(new osb_anchor());
  h->device = current_device();
  h->p = *p;
  h->p.huber = p->huber ? 1 : 0;
  h->begin_dt_ns = llround(p->begin_min_loop_dt_s * 1e9);
  const size_t D = (size_t)p->max_drones, S = (size_t)p->max_traj_samples, M = (size_t)p->max_measurements,
               E = (size_t)p->max_window_entries;
  Resources& R = h->res;
  OSB_TRY(R.stream(&h->stream));
  OSB_TRY(R.event(&h->last_run, cudaEventDisableTiming));
  OSB_TRY(R.alloc(&h->d_meas, M));
  OSB_TRY(R.alloc(&h->d_loop_slot, M));
  OSB_TRY(R.alloc(&h->d_det_slot, M));
  OSB_TRY(R.alloc(&h->d_traj_stamp, D * S));
  OSB_TRY(R.alloc(&h->d_traj_pose, D * S * 7));
  OSB_TRY(R.alloc(&h->d_traj_len, D * S));
  OSB_TRY(R.alloc(&h->d_traj_n, D));
  OSB_TRY(R.alloc(&h->d_drone_first, D + 1));
  OSB_TRY(R.alloc(&h->d_win_stamp, E));
  OSB_TRY(R.alloc(&h->d_win_frame, E));
  OSB_TRY(R.alloc(&h->d_win_block, E));
  OSB_TRY(R.alloc(&h->d_win_pose, E * 7));
  OSB_TRY(R.alloc(&h->d_out, M));
  OSB_CUDA(cudaMemsetAsync(h->d_traj_n, 0, D * sizeof(int32_t), h->stream));
  OSB_CUDA(cudaMemsetAsync(h->d_drone_first, 0, (D + 1) * sizeof(int32_t), h->stream));
  OSB_CUDA(cudaEventRecord(h->last_run, h->stream));
  OSB_CUDA(cudaStreamSynchronize(h->stream));
  h->traj_n.assign(D, 0);
  h->last_stamp.assign(D, 0);
  h->last_pos.assign(D * 3, 0.0);
  h->last_len.assign(D, 0.0);
  h->h_drone_first.resize(D + 1);
  h->h_win_frame.resize(E);
  h->h_win_block.resize(E);
  h->h_win_stamp.resize(E);
  h->h_win_pose.resize(E * 7);
  h->h_len.reserve(S);
  h->h_slot.reserve(M);
  *out = h.release();
  return OSB_OK;
}

extern "C" osb_status osb_anchor_destroy(osb_anchor* h) {
  delete h;
  return OSB_OK;
}

extern "C" osb_status osb_anchor_push_odometry(osb_anchor* h, int32_t drone, int n, const int64_t* stamps_ns,
                                               const double* poses) {
  OSB_REQUIRE(h != nullptr && n >= 0 && (n == 0 || (stamps_ns && poses)), "null argument or negative count");
  OSB_REQUIRE(drone_ok(h, drone), "drone id outside 0..max_drones-1");
  std::lock_guard<std::mutex> lk(h->mu);
  OSB_TRY(anchor_settle(h));
  const int have = h->traj_n[drone];
  for (int i = 0; i < n; ++i) {
    const int64_t prev = i > 0 ? stamps_ns[i - 1] : h->last_stamp[drone];
    OSB_REQUIRE((have == 0 && i == 0) || stamps_ns[i] > prev, "odometry stamps must increase strictly");
  }
  if ((long long)have + n > h->p.max_traj_samples) {
    set_error(__func__, "the drone's trajectory would exceed max_traj_samples");
    return OSB_ERR_CAPACITY;
  }
  if (n == 0) return OSB_OK;
  DeviceGuard dg(h->device);
  // length[k] = length[k-1] + |p_k - p_(k-1)|, summed in sample order
  h->h_len.resize(n);
  double len = h->last_len[drone];
  const double* prev = &h->last_pos[(size_t)drone * 3];
  for (int i = 0; i < n; ++i) {
    const double* p = poses + (size_t)i * 7;
    if (have > 0 || i > 0) {
      const double dx = p[0] - prev[0], dy = p[1] - prev[1], dz = p[2] - prev[2];
      len = len + sqrt(dx * dx + dy * dy + dz * dz);
    }
    h->h_len[i] = len;
    prev = p;
  }
  const size_t base = (size_t)drone * h->p.max_traj_samples + have;
  const int32_t new_n = have + n;
  OSB_TRY(anchor_wait_last_run(h));
  cudaStream_t st = h->stream;
  OSB_CUDA(cudaMemcpyAsync(h->d_traj_stamp + base, stamps_ns, (size_t)n * sizeof(int64_t), cudaMemcpyHostToDevice, st));
  OSB_CUDA(cudaMemcpyAsync(h->d_traj_pose + base * 7, poses, (size_t)n * 7 * sizeof(double), cudaMemcpyHostToDevice, st));
  OSB_CUDA(cudaMemcpyAsync(h->d_traj_len + base, h->h_len.data(), (size_t)n * sizeof(double), cudaMemcpyHostToDevice, st));
  OSB_CUDA(cudaMemcpyAsync(h->d_traj_n + drone, &new_n, sizeof(int32_t), cudaMemcpyHostToDevice, st));
  OSB_CUDA(cudaStreamSynchronize(st));
  h->traj_n[drone] = new_n;
  h->last_stamp[drone] = stamps_ns[n - 1];
  for (int j = 0; j < 3; ++j) h->last_pos[(size_t)drone * 3 + j] = poses[(size_t)(n - 1) * 7 + j];
  h->last_len[drone] = len;
  return OSB_OK;
}

extern "C" osb_status osb_anchor_add_measurements(osb_anchor* h, int n, const osb_measurement* m) {
  OSB_REQUIRE(h != nullptr && n >= 0 && (n == 0 || m), "null argument or negative count");
  for (int i = 0; i < n; ++i) {
    OSB_REQUIRE(m[i].type == OSB_MEAS_LOOP || m[i].type == OSB_MEAS_DET4D || m[i].type == OSB_MEAS_DET6D,
                "unknown measurement type");
    OSB_REQUIRE(drone_ok(h, m[i].id_a) && drone_ok(h, m[i].id_b), "drone id outside 0..max_drones-1");
  }
  std::lock_guard<std::mutex> lk(h->mu);
  OSB_TRY(anchor_settle(h));
  const int have = h->n_loops + h->n_dets;
  if ((long long)have + n > h->p.max_measurements) {
    set_error(__func__, "the handle would exceed max_measurements");
    return OSB_ERR_CAPACITY;
  }
  if (n == 0) return OSB_OK;
  DeviceGuard dg(h->device);
  // storage keeps arrival order; the loop and detection slot lists give the reference's output order
  std::vector<int32_t>& slot = h->h_slot;
  slot.clear();
  for (int i = 0; i < n; ++i)
    if (m[i].type == OSB_MEAS_LOOP) slot.push_back(have + i);
  const int new_loops = (int)slot.size();
  for (int i = 0; i < n; ++i)
    if (m[i].type != OSB_MEAS_LOOP) slot.push_back(have + i);
  OSB_TRY(anchor_wait_last_run(h));
  cudaStream_t st = h->stream;
  OSB_CUDA(cudaMemcpyAsync(h->d_meas + have, m, (size_t)n * sizeof(osb_measurement), cudaMemcpyHostToDevice, st));
  if (new_loops > 0)
    OSB_CUDA(cudaMemcpyAsync(h->d_loop_slot + h->n_loops, slot.data(), (size_t)new_loops * sizeof(int32_t),
                             cudaMemcpyHostToDevice, st));
  if (n > new_loops)
    OSB_CUDA(cudaMemcpyAsync(h->d_det_slot + h->n_dets, slot.data() + new_loops, (size_t)(n - new_loops) * sizeof(int32_t),
                             cudaMemcpyHostToDevice, st));
  const int32_t counts[2] = {h->n_loops + new_loops, h->n_dets + n - new_loops};
  if (h->d_counts)                                                 // device appends continue from here
    OSB_CUDA(cudaMemcpyAsync(h->d_counts, counts, sizeof(counts), cudaMemcpyHostToDevice, st));
  OSB_CUDA(cudaStreamSynchronize(st));
  h->n_loops += new_loops;
  h->n_dets += n - new_loops;
  return OSB_OK;
}

extern "C" osb_status osb_anchor_size(osb_anchor* h, int32_t* n_loops, int32_t* n_detections) {
  OSB_REQUIRE(h != nullptr && n_loops != nullptr && n_detections != nullptr, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  OSB_TRY(anchor_settle(h));
  *n_loops = h->n_loops;
  *n_detections = h->n_dets;
  return OSB_OK;
}

extern "C" osb_status osb_anchor_set_window(osb_anchor* h, int n_frames, const int64_t* frame_stamps_ns,
                                            const int32_t* frame_first, const osb_window_entry* entries) {
  OSB_REQUIRE(h != nullptr && n_frames >= 0, "null handle or negative frame count");
  OSB_REQUIRE(n_frames == 0 || (frame_stamps_ns && frame_first), "null argument");
  const int n_entries = n_frames == 0 ? 0 : frame_first[n_frames];
  if (n_frames > 0) {
    OSB_REQUIRE(frame_first[0] == 0, "frame_first[0] must be 0");
    for (int f = 0; f < n_frames; ++f) OSB_REQUIRE(frame_first[f + 1] >= frame_first[f], "frame_first must not decrease");
    OSB_REQUIRE(n_entries == 0 || entries != nullptr, "null entries");
  }
  std::lock_guard<std::mutex> lk(h->mu);
  OSB_TRY(anchor_settle(h));
  if (n_entries > h->p.max_window_entries) {
    set_error(__func__, "the window would exceed max_window_entries");
    return OSB_ERR_CAPACITY;
  }
  for (int f = 0; f < n_frames; ++f)                               // SwarmFrame::id2nodeframe holds a drone once
    for (int a = frame_first[f]; a < frame_first[f + 1]; ++a) {
      OSB_REQUIRE(drone_ok(h, entries[a].drone_id), "drone id outside 0..max_drones-1");
      for (int b = frame_first[f]; b < a; ++b) OSB_REQUIRE(entries[b].drone_id != entries[a].drone_id, "a drone twice in one frame");
    }
  DeviceGuard dg(h->device);
  // per-drone index of the vo_available entries in frame order (a counting sort by drone)
  const int D = h->p.max_drones;
  std::vector<int32_t>& first = h->h_drone_first;
  std::fill(first.begin(), first.end(), 0);
  for (int e = 0; e < n_entries; ++e)
    if (entries[e].vo_available) ++first[entries[e].drone_id + 1];
  for (int d = 0; d < D; ++d) first[d + 1] += first[d];
  std::vector<int32_t> fill(first.begin(), first.end() - 1);
  for (int f = 0; f < n_frames; ++f)
    for (int e = frame_first[f]; e < frame_first[f + 1]; ++e) {
      if (!entries[e].vo_available) continue;
      const int k = fill[entries[e].drone_id]++;
      h->h_win_stamp[k] = entries[e].stamp;
      h->h_win_frame[k] = f;
      h->h_win_block[k] = entries[e].block;
      std::copy(entries[e].self_pose, entries[e].self_pose + 7, h->h_win_pose.begin() + (size_t)k * 7);
    }
  const int n_vo = first[D];
  OSB_TRY(anchor_wait_last_run(h));
  cudaStream_t st = h->stream;
  OSB_CUDA(cudaMemcpyAsync(h->d_drone_first, first.data(), (size_t)(D + 1) * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  if (n_vo > 0) {
    OSB_CUDA(cudaMemcpyAsync(h->d_win_stamp, h->h_win_stamp.data(), (size_t)n_vo * sizeof(int64_t), cudaMemcpyHostToDevice, st));
    OSB_CUDA(cudaMemcpyAsync(h->d_win_frame, h->h_win_frame.data(), (size_t)n_vo * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    OSB_CUDA(cudaMemcpyAsync(h->d_win_block, h->h_win_block.data(), (size_t)n_vo * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    OSB_CUDA(cudaMemcpyAsync(h->d_win_pose, h->h_win_pose.data(), (size_t)n_vo * 7 * sizeof(double), cudaMemcpyHostToDevice, st));
  }
  OSB_CUDA(cudaStreamSynchronize(st));
  h->n_frames = n_frames;
  h->frame0_stamp = n_frames > 0 ? frame_stamps_ns[0] : 0;
  return OSB_OK;
}

namespace {

osb_status anchor_launch(osb_anchor* h, const uint8_t* yaw_observable, osb_anchor_result* out_dev, int32_t* n_out,
                         cudaStream_t st) {
  AnchorView v{};
  v.meas = h->d_meas;
  v.loop_slot = h->d_loop_slot;
  v.det_slot = h->d_det_slot;
  v.n_loops = h->n_loops;
  v.n_total = h->n_loops + h->n_dets;
  v.traj_stamp = h->d_traj_stamp;
  v.traj_pose = h->d_traj_pose;
  v.traj_len = h->d_traj_len;
  v.traj_n = h->d_traj_n;
  v.max_samples = h->p.max_traj_samples;
  v.max_drones = h->p.max_drones;
  v.drone_first = h->d_drone_first;
  v.win_stamp = h->d_win_stamp;
  v.win_frame = h->d_win_frame;
  v.win_block = h->d_win_block;
  v.win_pose = h->d_win_pose;
  v.n_frames = h->n_frames;
  v.frame0_stamp = h->frame0_stamp;
  v.begin_dt_ns = h->begin_dt_ns;
  v.dpos_thres = h->p.det_dpos_thres;
  v.pos_cov = h->p.odom_pos_cov_per_m;
  v.ang_cov = h->p.odom_ang_cov_per_m;
  v.huber = h->p.huber;
  for (int d = 0; d < h->p.max_drones; ++d)
    if (yaw_observable[d]) v.yaw_obs[d >> 6] |= 1ull << (d & 63);
  v.counts = nullptr;
  v.n_bound = v.n_total;
  if (h->append_pending) {                      // the counts are the device's; the grid covers the host's bound of them
    anchor_tighten(h);
    OSB_CUDA(cudaStreamWaitEvent(st, h->last_append, 0));
    v.counts = h->d_counts;
    v.n_bound = (int)h->upper;
  }
  *n_out = v.n_bound;
  if (v.n_bound == 0) return OSB_OK;
  OSB_LAUNCH(anchor_kernel, cdiv(v.n_bound, ANCHOR_WARPS), ANCHOR_WARPS * 32, 0, st, v, out_dev);
  OSB_CHECK_LAUNCH();
  OSB_CUDA(cudaEventRecord(h->last_run, st));
  return OSB_OK;
}

}  // namespace

extern "C" osb_status osb_anchor_run_dev(osb_anchor* h, const uint8_t* yaw_observable, osb_anchor_result* out_dev,
                                         int32_t* n_out, void* stream) {
  OSB_REQUIRE(h != nullptr && yaw_observable != nullptr && out_dev != nullptr && n_out != nullptr, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  return anchor_launch(h, yaw_observable, out_dev, n_out, (cudaStream_t)stream);
}

extern "C" osb_status osb_anchor_compact_factors_dev(const osb_anchor_result* rows_dev, int n, const uint8_t* keep_dev,
                                                     int32_t* type, int32_t* ia, int32_t* ib, double* payload,
                                                     uint8_t* huber, int32_t* count_dev, void* stream) {
  OSB_REQUIRE(n >= 0 && count_dev != nullptr, "negative count or null count");
  OSB_REQUIRE(n == 0 || (rows_dev && type && ia && ib && payload && huber), "null argument");
  OSB_TRY(require_device());
  OSB_LAUNCH(anchor_compact_kernel, 1, COMPACT_THREADS, 0, (cudaStream_t)stream, rows_dev, n, keep_dev, type, ia, ib,
             payload, huber, count_dev);
  OSB_CHECK_LAUNCH();
  return OSB_OK;
}

extern "C" osb_status osb_anchor_run(osb_anchor* h, const uint8_t* yaw_observable, osb_anchor_result* out, int32_t* n_out) {
  OSB_REQUIRE(h != nullptr && yaw_observable != nullptr && n_out != nullptr, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  OSB_TRY(anchor_settle(h));                                       // exact counts: run writes no VOID row
  OSB_REQUIRE(out != nullptr || h->n_loops + h->n_dets == 0, "null output");
  DeviceGuard dg(h->device);
  OSB_TRY(anchor_launch(h, yaw_observable, h->d_out, n_out, h->stream));
  if (*n_out > 0)
    OSB_CUDA(cudaMemcpyAsync(out, h->d_out, (size_t)*n_out * sizeof(osb_anchor_result), cudaMemcpyDeviceToHost, h->stream));
  OSB_CUDA(cudaStreamSynchronize(h->stream));
  return OSB_OK;
}

namespace {

// the first device append acquires the device counts (seeded with the host's exact ones), the feedback and the event
osb_status anchor_dev_init(osb_anchor* h) {
  if (h->d_counts) return OSB_OK;
  Resources& R = h->res;
  OSB_TRY(R.alloc(&h->d_counts, 2));
  OSB_TRY(R.host_alloc(&h->fb_host, 1, cudaHostAllocMapped));
  memset((void*)h->fb_host, 0, sizeof(AnchorFeedback));
  OSB_CUDA(cudaHostGetDevicePointer((void**)&h->fb_dev, (void*)h->fb_host, 0));
  OSB_TRY(R.event(&h->last_append, cudaEventDisableTiming));
  const int32_t counts[2] = {h->n_loops, h->n_dets};
  OSB_CUDA(cudaMemcpyAsync(h->d_counts, counts, sizeof(counts), cudaMemcpyHostToDevice, h->stream));
  OSB_CUDA(cudaStreamSynchronize(h->stream));
  return OSB_OK;
}

}  // namespace

extern "C" osb_status osb_anchor_add_measurements_dev(osb_anchor* h, const osb_measurement* m_dev, const int32_t* count_dev,
                                                      int max_n, float loop_outlier_distance_threshold, void* stream) {
  OSB_REQUIRE(h != nullptr && m_dev != nullptr && count_dev != nullptr, "null argument");
  OSB_REQUIRE(max_n >= 0, "negative max_n");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  cudaStream_t st = (cudaStream_t)stream;
  OSB_TRY(anchor_dev_init(h));
  // the append rewrites the counts a run reads and follows the previous append, whichever streams those ran on
  OSB_CUDA(cudaStreamWaitEvent(st, h->last_run, 0));
  if (h->append_pending) {
    OSB_CUDA(cudaStreamWaitEvent(st, h->last_append, 0));
    anchor_tighten(h);
  } else {
    h->upper = h->n_loops + h->n_dets;
  }
  const long long seq = h->append_seq + 1, charged = h->charged + max_n;
  OSB_LAUNCH(anchor_append_kernel, 1, APPEND_THREADS, 0, st, m_dev, count_dev, max_n, loop_outlier_distance_threshold,
             h->p.max_drones, h->p.max_measurements, h->d_meas, h->d_loop_slot, h->d_det_slot, h->d_counts, h->fb_dev, seq,
             charged);
  OSB_CHECK_LAUNCH();
  OSB_CUDA(cudaEventRecord(h->last_append, st));
  h->append_seq = seq;
  h->charged = charged;
  h->upper = std::min<long long>(h->upper + max_n, h->p.max_measurements);
  h->append_pending = true;
  return OSB_OK;
}

extern "C" osb_status osb_anchor_status(osb_anchor* h, osb_status* last) {
  OSB_REQUIRE(h != nullptr && last != nullptr, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  OSB_TRY(anchor_settle(h));
  *last = h->last_status;
  return h->last_status;
}
