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
#include <cmath>

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

// PRED (osb_anchor_run_dev_if): predicated on a device word, 0 writes nothing
template <bool PRED>
__global__ void __launch_bounds__(ANCHOR_WARPS * 32)
anchor_kernel(const AnchorView v, osb_anchor_result* __restrict__ out, const int32_t* __restrict__ pred) {
  if constexpr (PRED) {
    if (*pred == 0) return;
  }
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
                     int max_drones, int anon_min, int max_meas, osb_measurement* __restrict__ meas, int32_t* __restrict__ loop_slot,
                     int32_t* __restrict__ det_slot, int32_t* __restrict__ counts, CountRecord* __restrict__ fb,
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
                      r.id_a >= 0 && r.id_a < max_drones && r.id_b >= 0 &&
                      (r.id_b < max_drones || (r.type != OSB_MEAS_LOOP && anon_min > 0 && r.id_b >= anon_min));
                                                                                                  // anon_min 0: no DA
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
  fb->publish(seq, status == OSB_OK ? have_l + nl : have_l, status == OSB_OK ? have_d + nd : have_d, status, charged);
}

// estimate_observability (swarm_localization_solver.cpp:1336-1427) from the rows of this solve: three launches.
// observe_edges_kernel ORs the drone pair of every OK row into a bit matrix (row d: drone d's neighbours, 256 bits);
// observe_state_kernel, one CTA, takes the matrix (and clears it for the next call), walks it from self_id a frontier of
// four 64-bit words at a time, applies the rules to the persistent state and writes the record; observe_skip_kernel
// rewrites each row's skip from the record's yaw.
constexpr int OBS_THREADS = 256;                                  // = ANCHOR_MAX_DRONES: thread d owns drone d
constexpr int OBS_WORDS = ANCHOR_MAX_DRONES / 64;                 // 64-bit words of a drone set
constexpr int OBS_ROW32 = ANCHOR_MAX_DRONES / 32;                 // 32-bit words of a matrix row
constexpr double THRES_YAW_OBSER_XY = 1.0;                        // :49
constexpr int SINGLE_DRONE_SFS_THRES = 3;                         // :62

// what observe takes from the window, derived by set_window on the host
struct ObserveWindow {
  double ext[ANCHOR_MAX_DRONES][3];   // boundingbox_sldwin's max - min per axis (-2000 for a drone without an entry)
  uint64_t nodes[OBS_WORDS];          // all_nodes: every drone of every window since create
  int32_t n_frames, n_nodes;
};

// observe_dev's three launches; the PRED instantiations (observe_dev_if) are predicated on a device word, 0 writes nothing
template <bool PRED>
__global__ void __launch_bounds__(OBS_THREADS)
observe_edges_kernel(const osb_anchor_result* __restrict__ rows, int n, int max_drones, unsigned* __restrict__ adj,
                     const int32_t* __restrict__ pred) {
  if constexpr (PRED) {
    if (*pred == 0) return;
  }
  __shared__ unsigned s_adj[ANCHOR_MAX_DRONES * OBS_ROW32];
  volatile unsigned* vs = s_adj;
  for (int k = threadIdx.x; k < max_drones * OBS_ROW32; k += OBS_THREADS) s_adj[k] = 0;
  __syncthreads();
  for (int i = blockIdx.x * OBS_THREADS + threadIdx.x; i < n; i += gridDim.x * OBS_THREADS) {
    if (rows[i].status != OSB_ANCHOR_OK) continue;
    const int a = rows[i].edge.id_a, b = rows[i].edge.id_b;
    if ((unsigned)a >= (unsigned)max_drones || (unsigned)b >= (unsigned)max_drones) continue;
    const int ab = a * OBS_ROW32 + (b >> 5), ba = b * OBS_ROW32 + (a >> 5);
    const unsigned bit_b = 1u << (b & 31), bit_a = 1u << (a & 31);
    if (!(vs[ab] & bit_b)) atomicOr(&s_adj[ab], bit_b);          // most rows repeat a pair already set
    if (!(vs[ba] & bit_a)) atomicOr(&s_adj[ba], bit_a);
  }
  __syncthreads();
  for (int k = threadIdx.x; k < max_drones * OBS_ROW32; k += OBS_THREADS)
    if (s_adj[k]) atomicOr(adj + k, s_adj[k]);
}

// PRED keeps motion_new: motion_new |= the record's (the second observe of a solve)
template <bool PRED>
__global__ void __launch_bounds__(OBS_THREADS)
observe_state_kernel(unsigned long long* __restrict__ adj, const ObserveWindow* __restrict__ win, int max_drones,
                     int self_id, float xy_thres, float z_thres, osb_observability* __restrict__ obs,
                     const int32_t* __restrict__ pred) {
  if constexpr (PRED) {
    if (*pred == 0) return;
  }
  __shared__ unsigned long long s_adj[ANCHOR_MAX_DRONES][OBS_WORDS];
  __shared__ unsigned long long s_seen[OBS_WORDS], s_front[OBS_WORDS], s_next[OBS_WORDS];
  __shared__ int s_more;
  const int d = threadIdx.x;
  for (int k = d; k < max_drones * OBS_WORDS; k += OBS_THREADS) {
    s_adj[k / OBS_WORDS][k % OBS_WORDS] = adj[k];
    adj[k] = 0;
  }
  if (d < OBS_WORDS) {
    s_seen[d] = s_front[d] = d == (self_id >> 6) ? 1ull << (self_id & 63) : 0ull;
    s_next[d] = 0;
  }
  __syncthreads();
  if (win->n_nodes > 1) {                                          // loop_observable_set's BFS, one level per pass
    for (;;) {
      if (d < max_drones && ((s_front[d >> 6] >> (d & 63)) & 1ull))
        for (int w = 0; w < OBS_WORDS; ++w)
          if (s_adj[d][w]) atomicOr(&s_next[w], s_adj[d][w]);
      __syncthreads();
      if (d == 0) {
        int more = 0;
        for (int w = 0; w < OBS_WORDS; ++w) {
          const unsigned long long f = s_next[w] & ~s_seen[w];
          s_front[w] = f;
          s_seen[w] |= f;
          s_next[w] = 0;
          more |= f != 0;
        }
        s_more = more;
      }
      __syncthreads();
      if (!s_more) break;
    }
  }
  const bool live = d < max_drones;
  const bool node = live && ((win->nodes[d >> 6] >> (d & 63)) & 1ull);
  const bool in_l = live && ((s_seen[d >> 6] >> (d & 63)) & 1ull);
  bool pos = live && obs->pos[d], enable = live && obs->enable[d], yaw = false, to_init = false, fresh = false;
  if (in_l) {                                                      // :1369-1379
    to_init = !pos;
    pos = yaw = enable = true;
  }
  const double* se = win->ext[self_id];                            // :1381-1403
  const bool motion = se[0] > (double)xy_thres && se[1] > (double)xy_thres && se[2] > (double)z_thres;
  if (motion && node) {
    if (!pos) fresh = to_init = true;
    pos = enable = true;
  }
  if (node && (win->ext[d][0] > THRES_YAW_OBSER_XY || win->ext[d][1] > THRES_YAW_OBSER_XY)) yaw = true;   // :1413-1422
  if (d == self_id) enable = true;                                 // :640
  const int other = __syncthreads_or(in_l && d != self_id);
  const int motion_new = __syncthreads_or(fresh);
  obs->nodes[d] = node;
  obs->yaw[d] = yaw;
  obs->pos[d] = pos;
  obs->enable[d] = enable;
  obs->to_init[d] = to_init;
  if (d == 0) {
    const bool single = win->n_frames > SINGLE_DRONE_SFS_THRES && win->n_nodes == 1;   // :1364-1367
    obs->solve_master = obs->solve_master || single || other || motion;
    obs->motion = motion;
    obs->motion_new = motion_new || (PRED && obs->motion_new);
    obs->reserved = 0;
  }
}

template <bool PRED>
__global__ void __launch_bounds__(OBS_THREADS)
observe_skip_kernel(osb_anchor_result* __restrict__ rows, int n, int max_drones, const osb_observability* __restrict__ obs,
                    const int32_t* __restrict__ pred) {
  if constexpr (PRED) {
    if (*pred == 0) return;
  }
  const int i = blockIdx.x * OBS_THREADS + threadIdx.x;
  if (i >= n) return;
  bool use = rows[i].status == OSB_ANCHOR_OK;                      // anchor_kernel's rule (:1066-1073) with this yaw
  if (use) {
    const int a = rows[i].edge.id_a, b = rows[i].edge.id_b;
    use = (unsigned)a < (unsigned)max_drones && (unsigned)b < (unsigned)max_drones && obs->yaw[a] && obs->yaw[b] &&
          rows[i].node_a != rows[i].node_b;
  }
  rows[i].skip = use ? 0 : 1;
}

// random_init_pose's choice of blocks (swarm_localization_solver.cpp:204-216) from the last observe's to_init: thread b
// masks block b iff its drone is to be initialised and is not self_id, and gives it the odometry yaw of its latest frame
__global__ void init_mask_kernel(const int32_t* __restrict__ blk_drone, const double* __restrict__ blk_q,
                                 const int32_t* __restrict__ n_blk, int n_nodes, int self_id,
                                 const osb_observability* __restrict__ obs, uint8_t* __restrict__ mask,
                                 double* __restrict__ yaw) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= n_nodes) return;
  const int d = b < *n_blk ? blk_drone[b] : -1;
  const bool m = d >= 0 && d != self_id && obs->to_init[d];
  mask[b] = m ? 1 : 0;
  yaw[b] = m ? quat_yaw(blk_q + 4 * (size_t)b) : 0.0;
}

// sync_est_poses (swarm_localization_solver.cpp:962-1057) and PredictSwarm (:673-765): three launches per sync.
// sync_gate_kernel (one CTA, thread d = drone d) decides whether the solver's last device call is accepted and the window
// has odometry for every drone, then writes the path counts and the prediction record; sync_kf_kernel writes one keyframe
// path sample per window entry; sync_full_kernel strides over every (drone, 10th odometry sample) of the capacities.
constexpr int SYNC_THREADS = 256;                                  // = ANCHOR_MAX_DRONES
constexpr int FULL_PATH_STEP = 10;                                 // :66

// what sync reads of the window, derived by set_window on the host: every entry, vo_available or not, ordered by
// (drone, frame) -- drone d's are [first[d], first[d+1]) -- and the stamp a steady sync pushes
struct SyncWindow {
  int32_t first[ANCHOR_MAX_DRONES + 1];
  int32_t n_frames, reserved;
  int64_t push_stamp;                 // the last frame that has entries (the reference's last_ts)
};
struct SyncRecord {                   // est_poses_tsid_saved[ts][d] of the last pushed frame ts holding d
  int64_t stamp;
  int32_t valid;
  int32_t estimated;                  // d had a window entry at an applied sync (estimated_nodes, :996-997); sticky
  double saved[4];                    // the solved block pose, x y z yaw
  double vo[7];                       // the entry's self_pose (all_sf[ts].id2nodeframe[d].pose())
};
struct SyncOutcome { int32_t applied, status; };

struct SyncView {
  const SyncWindow* win;
  const int64_t* w_stamp;             // [E] the entry's frame stamp
  const int32_t *w_drone, *w_block;   // [E]
  const double* w_pose;               // [E][7] self_pose
  int max_entries, max_drones, max_samples, max_full;
  const int64_t* traj_stamp;
  const double* traj_pose;
  const int32_t* traj_n;
  // the solver's last device call
  const double* poses;
  const int32_t* word;
  const osb_solve_summary* summary;
  const int32_t* chosen;
  int trials, base_res, normalise, window_size, full_path;
  double acpt_cost;
  // outputs
  SyncOutcome* outcome;
  SyncRecord* rec;
  int32_t* kf_first;                  // [D + 1] the paths' (snapshot of win->first)
  int64_t* kf_stamp;                  // [E]
  double* kf_pose;                    // [E][7]
  int32_t* full_n;                    // [D], -1: none
  int64_t* full_stamp;                // [D][max_full]
  double* full_pose;                  // [D][max_full][7]
};

__device__ __forceinline__ PoseD pose_from4(const double* p) {   // Pose(double[4], true)
  PoseD o;
  o.t[0] = p[0]; o.t[1] = p[1]; o.t[2] = p[2];
  const double rv[3] = {0.0, 0.0, p[3]};
  quat_from_rotvec(rv, o.q);
  return o;
}
// AngleAxis(-yaw(ego), Z) * att(ego)
__device__ __forceinline__ void att_no_yaw(const PoseD& ego, double* q) {
  double qy[4];
  const double rv[3] = {0.0, 0.0, -quat_yaw(ego.q)};
  quat_from_rotvec(rv, qy);
  q_mul(qy, ego.q, q);
}
__device__ __forceinline__ PoseD ego_at(const SyncView& v, int d, int64_t t) {
  const size_t base = (size_t)d * v.max_samples;
  return load_pose(v.traj_pose + (base + nearest_sample(v.traj_stamp + base, v.traj_n[d], t)) * 7);
}

__global__ void __launch_bounds__(SYNC_THREADS) sync_gate_kernel(const SyncView v) {
  __shared__ int s_ok;
  const int d = threadIdx.x;
  const SyncWindow& w = *v.win;
  if (d == 0) {
    bool ok;
    if (v.trials > 0) {
      ok = __ldcg(v.chosen) >= 0;                                  // solve_with_multiple_init's finish_init
    } else {
      const double c = __ldcg(&v.summary->final_cost);
      const int n_res = v.base_res + __ldcg(v.word + 3);
      const double e = v.normalise ? sqrt(c) / (double)n_res / (double)v.window_size : c;
      ok = __ldcg(v.word) == OSB_OK && !(e > v.acpt_cost);         // :947-951
    }
    s_ok = ok;
  }
  const bool live = d < v.max_drones;
  const int lo = live ? w.first[d] : 0, hi = live ? w.first[d + 1] : 0;
  __syncthreads();
  const bool accepted = s_ok != 0;
  const bool no_odom = __syncthreads_or(accepted && hi > lo && v.traj_n[d] == 0);
  if (d == 0) {
    v.outcome->applied = accepted && !no_odom;
    v.outcome->status = no_odom ? OSB_ERR_INVALID : OSB_OK;
  }
  if (!accepted || no_odom || !live) return;
  v.kf_first[d] = lo;
  if (d == v.max_drones - 1) v.kf_first[d + 1] = hi;
  v.full_n[d] = (v.full_path && hi > lo) ? (v.traj_n[d] + FULL_PATH_STEP - 1) / FULL_PATH_STEP : -1;
  SyncRecord& r = v.rec[d];
  if (hi > lo) r.estimated = 1;
  int k = -1;
  if (hi > lo && (v.trials > 0 || v.win->push_stamp == v.w_stamp[hi - 1])) {
    k = hi - 1;                                                    // a pushed frame holds d: the last of them
  } else if (r.valid) {
    for (int j = lo; j < hi; ++j)                                  // its frame is still in the window: rewritten
      if (v.w_stamp[j] == r.stamp) { k = j; break; }
  }
  if (k < 0) return;
  r.stamp = v.w_stamp[k];
  r.valid = 1;
  const double* p = v.poses + 4 * (size_t)v.w_block[k];
  for (int j = 0; j < 4; ++j) r.saved[j] = p[j];
  for (int j = 0; j < 7; ++j) r.vo[j] = v.w_pose[(size_t)k * 7 + j];
}

__global__ void sync_kf_kernel(const SyncView v) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= v.max_entries || !v.outcome->applied || k >= v.win->first[v.max_drones]) return;
  const int d = v.w_drone[k];
  const int64_t t = v.w_stamp[k];
  PoseD p = pose_from4(v.poses + 4 * (size_t)v.w_block[k]);
  double q[4], qa[4];
  att_no_yaw(ego_at(v, d, t), qa);
  q_mul(p.q, qa, q);
  for (int j = 0; j < 4; ++j) p.q[j] = q[j];
  v.kf_stamp[k] = t;
  store_pose(v.kf_pose + (size_t)k * 7, p);
}

__global__ void sync_full_kernel(const SyncView v) {
  if (!v.outcome->applied) return;
  const long long total = (long long)v.max_drones * v.max_full;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int d = (int)(i / v.max_full), j = (int)(i % v.max_full);
    if (j >= v.full_n[d]) continue;
    const int lo = v.kf_first[d], hi = v.kf_first[d + 1];
    const size_t s = (size_t)d * v.max_samples + (size_t)j * FULL_PATH_STEP;
    const int64_t ts_vo = v.traj_stamp[s];
    const int k = lo + nearest_sample(v.kf_stamp + lo, hi - lo, ts_vo);   // the walk of :1034-1040
    PoseD p = pose_mul(load_pose(v.kf_pose + (size_t)k * 7),
                       delta_pose4(load_pose(v.w_pose + (size_t)k * 7), load_pose(v.traj_pose + s * 7)));
    double q[4], qa[4];
    att_no_yaw(ego_at(v, d, v.kf_stamp[k]), qa);
    q_mul(p.q, qa, q);
    for (int c = 0; c < 4; ++c) p.q[c] = q[c];
    const size_t o = (size_t)d * v.max_full + j;
    v.full_stamp[o] = ts_vo;
    store_pose(v.full_pose + o * 7, p);
  }
}

__global__ void predict_kernel(int n, const int32_t* __restrict__ drones, const double* __restrict__ vo_now,
                               const SyncRecord* __restrict__ rec, const osb_observability* __restrict__ obs, int self_id,
                               osb_predict_result* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int d = drones[i];
  const SyncRecord& r = rec[d];
  osb_predict_result o = {};
  if (r.valid) {
    const PoseD est = pose_from4(r.saved), vo = load_pose(r.vo);
    const PoseD vo4 = pose_yaw_only(vo);
    if (d == self_id || (obs != nullptr && obs->enable[d])) {      // :676-678
      o.node_valid = 1;
      store_pose(o.node_pose, pose_mul(est, pose_mul(pose_inv(vo4), load_pose(vo_now + (size_t)i * 7))));   // :691
    }
    o.base_valid = 1;
    store_pose(o.base_pose, pose_mul(pose_yaw_only(est), pose_inv(vo4)));                                   // :708-715
  }
  out[i] = o;
}

// add_as_keyframe's values (swarm_localization_solver.cpp:272-339, :408-515): one CTA, thread i owns node i for the
// initial poses, then the threads stride over the keyframe's distances for the flags and the store.
constexpr int KF_THREADS = 256;                                    // = ANCHOR_MAX_DRONES
constexpr double RAND_INIT_XY = 5.0;                               // :51
constexpr int KF_STAGING = 4;                                      // pinned input slots

struct KeyframeView {
  const osb_keyframe_node* nodes;     // the call's inputs (mapped pinned staging)
  const osb_keyframe_distance* dists;
  int n_nodes, n_dists, max_drones, max_dists;
  int64_t stamp;
  int self_id, finish_init, enable_distance;
  double thr, elev, min_d;            // the float parameters, widened
  uint64_t seed;
  double* poses;                      // the solver's resident poses, [block][4]
  int slot, prev_slot;                // the store slot written and the last keyframe's (-1: none)
  int64_t* st_stamp;                  // [K]
  int32_t* st_n;                      // [K] node count, -1: empty
  osb_keyframe_node* st_node;         // [K][max_drones]
  int32_t* st_first;                  // [K][max_drones + 1] distance offsets
  osb_keyframe_distance* st_dist;     // [K][max_dists]
  int8_t* st_flag;                    // [K][max_dists]
};

__device__ __forceinline__ double kf_draw(uint64_t seed, int64_t stamp, int drone, int comp) {
  return counter_draw(seed, splitmix64((uint64_t)stamp) ^ (((uint64_t)(uint32_t)drone << 2) | (uint64_t)comp), RAND_INIT_XY);
}
__device__ __forceinline__ void store_pose4(double* dst, const double* t, double yaw) {   // to_vector_xyzyaw
  dst[0] = t[0]; dst[1] = t[1]; dst[2] = t[2]; dst[3] = yaw;
}
// the node whose distances hold index k: the last i with first[i] <= k
__device__ __forceinline__ int kf_owner(const int* first, int n, int k) {
  int lo = 0, hi = n;                                              // first[lo] <= k < first[hi]
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (first[mid] <= k) lo = mid; else hi = mid;
  }
  return lo;
}

__global__ void __launch_bounds__(KF_THREADS) keyframe_kernel(const KeyframeView v) {
  __shared__ int s_node[ANCHOR_MAX_DRONES];                        // drone -> its node here, -1
  __shared__ int s_last[ANCHOR_MAX_DRONES];                        // drone in the last keyframe: -1 absent, 0 no VO, 1 VO
  __shared__ int s_first[ANCHOR_MAX_DRONES + 1];
  __shared__ int s_stop;                                           // the node whose `return` ends the flag walk
  const int t = threadIdx.x;
  s_node[t] = -1;
  s_last[t] = -1;
  if (t == 0) {
    s_stop = INT_MAX;
    int acc = 0;
    for (int i = 0; i < v.n_nodes; ++i) { s_first[i] = acc; acc += v.nodes[i].n_distances; }
    s_first[v.n_nodes] = acc;
  }
  __syncthreads();
  const bool mine = t < v.n_nodes;
  if (v.prev_slot >= 0 && t < v.st_n[v.prev_slot]) {               // read before the slot is written: with one slot
    const osb_keyframe_node& pn = v.st_node[(size_t)v.prev_slot * v.max_drones + t];   // the two are the same
    s_last[pn.drone_id] = pn.vo_available ? 1 : 0;
  }
  __syncthreads();
  osb_keyframe_node nd{};
  if (mine) {
    nd = v.nodes[t];
    s_node[nd.drone_id] = t;
    v.st_node[(size_t)v.slot * v.max_drones + t] = nd;
  }
  if (mine && nd.new_block) {                                      // a. the new block's initial pose
    const PoseD vo = load_pose(nd.pose);
    double* dst = v.poses + 4 * (size_t)nd.block;
    const bool dynamic_predict = !nd.is_static && (nd.drone_id != v.self_id || v.finish_init) && nd.prev_block >= 0;
    const bool self_vo = !nd.is_static && nd.drone_id == v.self_id && !v.finish_init;
    if (dynamic_predict) {                                         // :279-298
      const PoseD est_last = pose_from4(v.poses + 4 * (size_t)nd.prev_block);
      const PoseD p = pose_mul(est_last, delta_pose4(load_pose(nd.prev_pose), vo));
      store_pose4(dst, p.t, quat_yaw(p.q));
    } else if (self_vo) {                                          // :306-310
      store_pose4(dst, vo.t, quat_yaw(vo.q));
    } else {                                                       // :300-305, :329-335
      double p[3];
      for (int c = 0; c < 3; ++c) p[c] = __dadd_rn(vo.t[c], kf_draw(v.seed, v.stamp, nd.drone_id, c));
      store_pose4(dst, p, quat_yaw(vo.q));
    }
  }
  __syncthreads();                                                 // s_last is complete, the new poses are visible
  if (mine && v.finish_init && s_last[nd.drone_id] == 0) atomicMin(&s_stop, t);
  for (int i = t; i <= v.n_nodes; i += KF_THREADS) v.st_first[(size_t)v.slot * (v.max_drones + 1) + i] = s_first[i];
  __syncthreads();
  for (int k = t; k < v.n_dists; k += KF_THREADS) {                // b. and c.
    const int i = kf_owner(s_first, v.n_nodes, k);
    const osb_keyframe_node* here = v.st_node + (size_t)v.slot * v.max_drones;   // written above, read from the device
    const osb_keyframe_node& a = here[i];
    const osb_keyframe_distance dk = v.dists[k];
    const int jn = s_node[dk.peer];
    int flag = -1;
    if (jn >= 0 && here[jn].vo_available) {
      const osb_keyframe_node& b = here[jn];
      const double dis = dk.distance;
      if (!v.finish_init) {                                        // :427-438
        const double dh = __dadd_rn(b.pose[2], -a.pose[2]);
        flag = (fabs(asin(dh / dis)) > v.elev || !v.enable_distance) ? 1 : 0;
      } else if (i < s_stop && s_last[a.drone_id] == 1) {          // :454-460, then :489-507
        const double* pa = v.poses + 4 * (size_t)a.block;
        const double* pb = v.poses + 4 * (size_t)b.block;
        const double dx = __dadd_rn(pb[0], -pa[0]), dy = __dadd_rn(pb[1], -pa[1]), dz = __dadd_rn(pb[2], -pa[2]);
        const double est = sqrt(__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)));
        flag = (fabs(__dadd_rn(dis, -est)) > v.thr || dis < v.min_d || fabs(asin(dz / dis)) > v.elev ||
                !v.enable_distance) ? 1 : 0;
      }
    }
    const size_t o = (size_t)v.slot * v.max_dists + k;
    v.st_dist[o] = dk;
    v.st_flag[o] = (int8_t)flag;
  }
  if (t == 0) {
    v.st_stamp[v.slot] = v.stamp;
    v.st_n[v.slot] = v.n_nodes;
  }
}

// setup_problem_with_sferror of every window frame (:1102-1154): one CTA walks the frames in order; per frame a block
// scan over the stored distances gives each kept one its row, in (a, b) order (no atomics).
constexpr int DF_THREADS = 1024, DF_WARPS = DF_THREADS / 32;

struct DistanceView {
  const int64_t* w_stamp;             // the window: frame stamps, frame_first, each entry's drone and block
  const int32_t *w_first, *w_drone, *w_block, *w_n;
  const int64_t* st_stamp;
  const int32_t* st_n;
  const osb_keyframe_node* st_node;
  const int32_t* st_first;
  const osb_keyframe_distance* st_dist;
  const int8_t* st_flag;
  int slots, max_drones, max_dists;
  const osb_observability* obs;
  int self_id, enable_distance, huber;
  double sqrt_inf;
  int32_t *type, *ia, *ib;
  double* payload;
  uint8_t* hub;
  int32_t* count;
  int max_tail;
};

__global__ void __launch_bounds__(DF_THREADS) distance_factors_kernel(const DistanceView v) {
  __shared__ int s_blk[ANCHOR_MAX_DRONES];                         // drone -> its block in the frame, -1
  __shared__ int s_first[ANCHOR_MAX_DRONES + 1];
  __shared__ int s_warp[DF_WARPS];
  __shared__ int s_slot;
  const int t = threadIdx.x, lane = t & 31, wid = t >> 5;
  const int base = *v.count;
  __syncthreads();                                                 // every thread has read it before thread 0 rewrites it
  if (base < 0) return;                                            // the tail is refused already
  const int nf = *v.w_n;
  int out = base;
  for (int f = 0; f < nf; ++f) {
    if (t < ANCHOR_MAX_DRONES) s_blk[t] = -1;
    if (t == 0) s_slot = -1;
    __syncthreads();
    const int64_t ts = v.w_stamp[f];
    for (int s = t; s < v.slots; s += DF_THREADS)                  // stamps are unique among the stored keyframes
      if (v.st_n[s] >= 0 && v.st_stamp[s] == ts) s_slot = s;
    for (int e = v.w_first[f] + t; e < v.w_first[f + 1]; e += DF_THREADS) s_blk[v.w_drone[e]] = v.w_block[e];
    __syncthreads();
    const int slot = s_slot;
    const int nn = slot >= 0 ? v.st_n[slot] : 0;
    if (slot >= 0)
      for (int i = t; i <= nn; i += DF_THREADS) s_first[i] = v.st_first[(size_t)slot * (v.max_drones + 1) + i];
    __syncthreads();
    const int nd = slot >= 0 ? s_first[nn] : 0;
    for (int k0 = 0; k0 < nd; k0 += DF_THREADS) {
      const int k = k0 + t;
      bool sel = false;
      int ba = 0, bb = 0;
      double dis = 0.0;
      if (k < nd) {
        const osb_keyframe_node& a = v.st_node[(size_t)slot * v.max_drones + kf_owner(s_first, nn, k)];
        const size_t o = (size_t)slot * v.max_dists + k;
        const int ida = a.drone_id, idb = v.st_dist[o].peer;
        dis = v.st_dist[o].distance;
        sel = v.enable_distance && a.frame_available && a.dists_available && idb < ida && v.st_flag[o] != 1 &&
              (ida == v.self_id || v.obs->enable[ida]);
        if (sel) {
          ba = s_blk[ida];
          bb = s_blk[idb];
          sel = ba >= 0 && bb >= 0;
        }
      }
      int inc = sel ? 1 : 0;                                       // block scan of the kept distances
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int u = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += u;
      }
      if (lane == 31) s_warp[wid] = inc;
      __syncthreads();
      if (wid == 0) {
        int w = s_warp[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const int u = __shfl_up_sync(0xffffffffu, w, o);
          if (lane >= o) w += u;
        }
        s_warp[lane] = w;
      }
      __syncthreads();
      const int row = out + (wid > 0 ? s_warp[wid - 1] : 0) + inc - (sel ? 1 : 0);
      const int total = s_warp[DF_WARPS - 1];
      if (sel && row < v.max_tail) {
        v.type[row] = OSB_FACTOR_DISTANCE;
        v.ia[row] = ba;
        v.ib[row] = bb;
        v.hub[row] = (uint8_t)v.huber;
        double* pl = v.payload + (size_t)row * OSB_PAYLOAD_LEN;
        pl[0] = dis;
        pl[1] = v.sqrt_inf;
        for (int j = 2; j < OSB_PAYLOAD_LEN; ++j) pl[j] = 0.0;
      }
      out += total;
      __syncthreads();                                             // s_warp is rewritten by the next tile
    }
  }
  if (t == 0) *v.count = out > v.max_tail ? -1 : out;
}

// The loop map of OutlierRejectionLoopEdges (swarm_outlier_rejection.cpp:106-120): all_loop_map as open addressing over
// H + 1 records (a power of two H, linear probing, empty key -1; the id -1 itself lives in record H) and
// all_loops_set_by_pair as each ordered pair's smallest id.  Two launches per call: record_claim_kernel inserts the key of
// every OK row whose id is not recorded yet, takes the smallest row index of each such id by atomicMin and lowers its
// pairs' minima; record_write_kernel lets each id's first row write the record.  Only record_write_kernel sets
// `recorded`, and only the winner reads its own, so no outcome depends on the order of atomics.
constexpr int LM_THREADS = 256;
constexpr int64_t LM_EMPTY = -1;
constexpr unsigned long long LM_NONE = ~0ull;                     // a pair without an id (the id INT64_MAX maps to it)
struct LoopRec {
  osb_loop_record r;                  // r.id is the key
  uint32_t claim;                     // the smallest row of this call that holds the id, UINT32_MAX: none
  uint32_t recorded;                  // 1: the values are written
};
// order-preserving map of an int64 id onto the unsigned pair minima
__device__ __forceinline__ unsigned long long lm_order(int64_t id) { return (unsigned long long)id ^ (1ull << 63); }

__device__ __forceinline__ int lm_find(const LoopRec* t, int H, int64_t id) {
  if (id == LM_EMPTY) return H;
  unsigned long long h = splitmix64((uint64_t)id) & (unsigned long long)(H - 1);
  for (int p = 0; p < H; ++p, h = (h + 1) & (unsigned long long)(H - 1)) {
    const int64_t k = *(volatile const int64_t*)&t[h].r.id;
    if (k == id) return (int)h;
    if (k == LM_EMPTY) return -1;
  }
  return -1;
}
__device__ __forceinline__ int lm_insert(LoopRec* t, int H, int64_t id) {   // -> the id's record, -1: the table is full
  if (id == LM_EMPTY) return H;
  unsigned long long h = splitmix64((uint64_t)id) & (unsigned long long)(H - 1);
  for (int p = 0; p < H; ++p, h = (h + 1) & (unsigned long long)(H - 1)) {
    unsigned long long* k = reinterpret_cast<unsigned long long*>(&t[h].r.id);
    unsigned long long cur = *(volatile unsigned long long*)k;
    if (cur == (unsigned long long)LM_EMPTY) cur = atomicCAS(k, (unsigned long long)LM_EMPTY, (unsigned long long)id);
    if (cur == (unsigned long long)LM_EMPTY || cur == (unsigned long long)id) return (int)h;
  }
  return -1;
}

struct LoopMapView {
  LoopRec* tab;                       // [H + 1]
  unsigned long long* pair;           // [D][D] lm_order(smallest id), LM_NONE
  int32_t* meta;                      // [0] the map overflowed (sticky), [1] the last init_by_loops' status
  int H, max_drones;
};

__global__ void __launch_bounds__(LM_THREADS)
record_claim_kernel(const osb_anchor_result* __restrict__ rows, int n, const LoopMapView v) {
  for (int i = blockIdx.x * LM_THREADS + threadIdx.x; i < n; i += gridDim.x * LM_THREADS) {
    if (rows[i].status != OSB_ANCHOR_OK) continue;
    const int64_t id = rows[i].id;
    const int s = lm_insert(v.tab, v.H, id);
    if (s < 0) { v.meta[0] = 1; continue; }
    if (v.tab[s].recorded == 1u) continue;                         // only record_write_kernel writes it
    atomicMin(&v.tab[s].claim, (uint32_t)i);
    const int a = rows[i].edge.id_a, b = rows[i].edge.id_b;
    if ((unsigned)a >= (unsigned)v.max_drones || (unsigned)b >= (unsigned)v.max_drones) continue;
    atomicMin(v.pair + (size_t)a * v.max_drones + b, lm_order(id));
    atomicMin(v.pair + (size_t)b * v.max_drones + a, lm_order(id));
  }
}

__global__ void __launch_bounds__(LM_THREADS)
record_write_kernel(const osb_anchor_result* __restrict__ rows, int n, const LoopMapView v) {
  for (int i = blockIdx.x * LM_THREADS + threadIdx.x; i < n; i += gridDim.x * LM_THREADS) {
    if (rows[i].status != OSB_ANCHOR_OK) continue;
    const int s = lm_find(v.tab, v.H, rows[i].id);
    if (s < 0 || v.tab[s].recorded == 1u || v.tab[s].claim != (uint32_t)i) continue;
    osb_loop_record& r = v.tab[s].r;
    r.id_a = rows[i].edge.id_a;
    r.id_b = rows[i].edge.id_b;
    r.stamp_a = rows[i].stamp_a;
    r.stamp_b = rows[i].stamp_b;
    for (int j = 0; j < 7; ++j) r.rel_pose[j] = rows[i].edge.rel_pose[j];
    v.tab[s].recorded = 1u;
  }
}

// init_pose_by_loops (swarm_localization_solver.cpp:218-269): one CTA, thread d decides drone d -- its id2, its loop and
// the prefix pose0 * odoma * rel -- then every thread strides over the window entries (ordered by drone, frame) and writes
// prefix * odomb into the entry's block.  A refusal anywhere leaves every pose as it was.
constexpr int IBL_THREADS = 256;                                   // = ANCHOR_MAX_DRONES

struct InitLoopsView {
  const osb_observability* obs;
  const PcmDir* dir;
  const int32_t* n_dir;
  LoopMapView lm;
  const SyncWindow* win;              // every window entry by (drone, frame): frame stamp and block
  const int64_t* w_stamp;
  const int32_t* w_block;
  const int32_t* kf_first;            // the keyframe paths of the last applied sync
  const int64_t* kf_stamp;
  const double* kf_pose;
  const SyncRecord* rec;              // rec[d].estimated
  const int64_t* traj_stamp;
  const double* traj_pose;
  const int32_t* traj_n;
  int max_samples, max_drones, self_id;
  double* poses;                      // the solver's resident poses, [block][4]
};

__device__ __forceinline__ PoseD ibl_ego(const InitLoopsView& v, int d, int64_t t, int64_t* t_out) {
  const size_t base = (size_t)d * v.max_samples;
  const int k = nearest_sample(v.traj_stamp + base, v.traj_n[d], t);
  if (t_out) *t_out = v.traj_stamp[base + k];
  return load_pose(v.traj_pose + (base + k) * 7);
}
// get_relative_pose_by_appro_ts(t1, t2) = pose(t1)^-1 pose(t2), nearest samples
__device__ __forceinline__ PoseD ibl_rel(const InitLoopsView& v, int d, int64_t t1, int64_t t2) {
  return pose_mul(pose_inv(ibl_ego(v, d, t1, nullptr)), ibl_ego(v, d, t2, nullptr));
}

__global__ void __launch_bounds__(IBL_THREADS) init_by_loops_kernel(const InitLoopsView v) {
  __shared__ double s_pre[ANCHOR_MAX_DRONES][7];
  __shared__ int64_t s_tb[ANCHOR_MAX_DRONES];
  __shared__ int s_id2[ANCHOR_MAX_DRONES];
  const int d = threadIdx.x;
  const int D = v.max_drones;
  const SyncWindow& w = *v.win;
  const int n_ent = w.first[D];
  const bool self_kf = w.first[v.self_id + 1] > w.first[v.self_id];
  int id2 = -1, status = v.lm.meta[0] ? OSB_ERR_CAPACITY : OSB_OK;
  int64_t lid = 0;
  if (d < D && v.obs->to_init[d] && status == OSB_OK) {
    const int nd = *v.n_dir;
    bool good = false;                                             // good_loops_set.find(_id) (:221-224)
    for (int e = 0; e < nd && !good; ++e) {
      const int64_t key = v.dir[e].key;
      good = v.dir[e].gn >= 0 && ((int)(key >> 32) == d || (int)(uint32_t)key == d);
    }
    const int n_cand = good ? nd : D;
    for (int c = 0; c < n_cand; ++c) {                             // each qualifying pair in turn (:225-232)
      int j;
      int64_t id;
      if (good) {
        const PcmDir& e = v.dir[c];
        const int lo = (int)(e.key >> 32), hi = (int)(uint32_t)e.key;
        if (e.gn <= 0 || (lo != d && hi != d)) continue;
        j = lo == d ? hi : lo;
        id = e.gptr[0];
      } else {
        j = c;
        const unsigned long long m = v.lm.pair[(size_t)d * D + c];
        if (m == LM_NONE) continue;
        id = (int64_t)(m ^ (1ull << 63));
      }
      if ((unsigned)j >= (unsigned)D || !(v.rec[j].estimated || (j == v.self_id && self_kf))) continue;
      const int s = lm_find(v.lm.tab, v.lm.H, id);                  // all_loop_map.at() and ego_motion_trajs.at()
      const bool has_path = v.kf_first[j + 1] > v.kf_first[j];
      if (s < 0 || v.lm.tab[s].recorded != 1u ||
          (v.traj_n[j] == 0 && (n_ent > 0 || (j == v.self_id && !has_path)))) {
        status = OSB_ERR_INVALID;
        break;
      }
      if (j > id2) { id2 = j; lid = id; }                           // the last pair in ascending id2 order wins
    }
  }
  const int bad = __syncthreads_or(status != OSB_OK);
  if (bad) {
    const int first_bad = __syncthreads_or(status == OSB_ERR_CAPACITY);
    if (d == 0) v.lm.meta[1] = first_bad ? OSB_ERR_CAPACITY : OSB_ERR_INVALID;
    return;
  }
  if (d < ANCHOR_MAX_DRONES) s_id2[d] = -1;
  if (id2 >= 0 && v.traj_n[id2] > 0) {                             // init_pose_by_loop (:236-268)
    const osb_loop_record& r = v.lm.tab[lm_find(v.lm.tab, v.lm.H, lid)].r;
    int64_t ta = r.stamp_a, tb = r.stamp_b;
    PoseD rel = load_pose(r.rel_pose);
    if (r.id_a != id2) {                                           // invert_loop
      ta = r.stamp_b;
      tb = r.stamp_a;
      rel = pose_inv(rel);
    }
    int64_t t0 = ta;
    PoseD pose0;
    pose0.t[0] = pose0.t[1] = pose0.t[2] = 0.0;
    pose0.q[0] = 1.0; pose0.q[1] = pose0.q[2] = pose0.q[3] = 0.0;
    const int lo = v.kf_first[id2], hi = v.kf_first[id2 + 1];
    if (hi > lo) {
      const int k = lo + nearest_sample(v.kf_stamp + lo, hi - lo, t0);
      t0 = v.kf_stamp[k];
      pose0 = load_pose(v.kf_pose + (size_t)k * 7);
    } else if (id2 == v.self_id) {
      pose0 = ibl_ego(v, id2, ta, &t0);
    }
    const PoseD pre = pose_mul(pose_mul(pose0, ibl_rel(v, id2, t0, ta)), rel);
    store_pose(s_pre[d], pre);
    s_tb[d] = tb;
    s_id2[d] = id2;
  }
  __syncthreads();
  for (int k = d; k < n_ent; k += IBL_THREADS) {
    const int dr = kf_owner(w.first, D, k);                        // the entry's drone: the last d with first[d] <= k
    const int j2 = s_id2[dr];
    if (j2 < 0) continue;
    const int blk = v.w_block[k];
    bool later = false;                                            // a later frame of the drone shares the block
    for (int k2 = k + 1; k2 < w.first[dr + 1] && !later; ++k2) later = v.w_block[k2] == blk;
    if (later) continue;
    const PoseD p = pose_mul(load_pose(s_pre[dr]), ibl_rel(v, j2, s_tb[dr], v.w_stamp[k]));
    store_pose4(v.poses + 4 * (size_t)blk, p.t, quat_yaw(p.q));
  }
  if (d == 0) v.lm.meta[1] = OSB_OK;
}

// LocalizationDAInit::try_data_association (localization_DA_init.cpp:29-90) and its DFS (:153-272) for the call site at
// swarm_localization_solver.cpp:893-916.  One CTA: the threads gather the unidentified ids (ascending, by repeated block
// minima, so the order is the reference's std::set and no result depends on atomics' order), their detections and the
// starting estimates; thread 0 then walks the DFS with an explicit stack in the reference's order, and on success the
// threads rename the store's anonymous rows.
constexpr int DA_THREADS = 256;                                    // = ANCHOR_MAX_DRONES
constexpr int DA_MAX_IDS = 32;
constexpr int DA_WORDS = ANCHOR_MAX_DRONES / 64;

struct DaResult {                     // the device record data_association_result reads; applied is the predicate word
  int32_t applied, status, n, reserved;
  int64_t nodes;                      // DFS calls of the last search
  int32_t anon[DA_MAX_IDS], guess[DA_MAX_IDS];
};

struct DaView {
  const osb_observability* obs;
  const osb_measurement* meas;
  const int32_t* det_slot;
  const int32_t* counts;              // [2] loops, detections
  const int64_t* traj_stamp;
  const double* traj_pose;
  const int32_t* traj_n;
  const int32_t* kf_first;
  const int64_t* kf_stamp;
  const double* kf_pose;
  int max_samples, max_drones, self_id, anon_min, max_nodes;
  double thres;
  DaResult* res;
  osb_measurement* meas_w;            // = meas: the rows renamed in place
};

__device__ __forceinline__ PoseD da_ego(const DaView& v, int d, int64_t t, int64_t* t_out) {
  const size_t base = (size_t)d * v.max_samples;
  const int k = nearest_sample(v.traj_stamp + base, v.traj_n[d], t);
  if (t_out) *t_out = v.traj_stamp[base + k];
  return load_pose(v.traj_pose + (base + k) * 7);
}
__device__ __forceinline__ PoseD da_rel(const DaView& v, int d, int64_t t1, int64_t t2) {   // pose(t1)^-1 pose(t2)
  return pose_mul(pose_inv(da_ego(v, d, t1, nullptr)), da_ego(v, d, t2, nullptr));
}
__device__ __forceinline__ bool bit_of(const unsigned long long* m, int d) { return (m[d >> 6] >> (d & 63)) & 1ull; }
__device__ __forceinline__ int da_index(const int* ids, int n, int id) {   // the unidentified id's index, -1: none
  for (int k = 0; k < n; ++k)
    if (ids[k] == id) return k;
  return -1;
}

__global__ void __launch_bounds__(DA_THREADS) data_association_kernel(const DaView v) {
  __shared__ double s_est[ANCHOR_MAX_DRONES][7];
  __shared__ unsigned long long s_has[DA_WORDS], s_avail[DA_WORDS], s_need[DA_WORDS];
  __shared__ int s_ids[DA_MAX_IDS + 1], s_n, s_min;
  __shared__ int s_last[DA_MAX_IDS], s_det_min[DA_MAX_IDS], s_first[DA_MAX_IDS];
  __shared__ int s_guess[DA_MAX_IDS];
  __shared__ unsigned long long s_t0;
  __shared__ int s_orphan, s_status, s_ok;
  const int t = threadIdx.x;
  const int D = v.max_drones;
  DaResult& R = *v.res;
  if (t == 0) { R.applied = 0; R.status = OSB_OK; R.n = 0; R.nodes = 0; }
  // the gate (:893-900): a node not enabled, more than one node, a detection in the store
  const bool node = t < D && v.obs->nodes[t];
  const int not_inited = __syncthreads_or(node && !v.obs->enable[t]);
  const int n_nodes = __syncthreads_count(node);
  const int n_det = v.counts[1];
  if (!not_inited || n_nodes <= 1 || n_det <= 0) return;
  // unidentified, ascending: repeated block minima of the anonymous ids above the last one found
  if (t == 0) s_n = 0;
  if (t < DA_WORDS) { s_has[t] = s_avail[t] = s_need[t] = 0ull; }
  if (t < DA_MAX_IDS) { s_last[t] = -1; s_det_min[t] = INT_MAX; s_first[t] = INT_MAX; }
  if (t == 0) { s_t0 = 0ull; s_orphan = 0; s_status = OSB_OK; s_ok = 0; }
  __syncthreads();
  for (int prev = INT_MIN;;) {
    if (t == 0) s_min = INT_MAX;
    __syncthreads();
    int mine = INT_MAX;
    for (int i = t; i < n_det; i += DA_THREADS) {
      const osb_measurement& m = v.meas[v.det_slot[i]];
      if (m.id_b >= v.anon_min && m.id_b > prev && v.traj_n[m.id_a] > 0 && m.id_b < mine) mine = m.id_b;
    }
    if (mine != INT_MAX) atomicMin(&s_min, mine);
    __syncthreads();
    const int found = s_min;
    __syncthreads();
    if (found == INT_MAX) break;
    if (t == 0) s_ids[s_n] = found;
    if (t == 0) ++s_n;
    __syncthreads();
    if (s_n > DA_MAX_IDS) break;
    prev = found;
  }
  const int n_u = s_n;
  if (n_u == 0) return;                                            // :46-48
  // per id: its last detection (raw_dets, uniden_detector), its detectors, the first row of its smallest detector
  for (int i = t; i < n_det; i += DA_THREADS) {
    const osb_measurement& m = v.meas[v.det_slot[i]];
    if (m.id_b < v.anon_min) continue;
    const int k = da_index(s_ids, min(n_u, DA_MAX_IDS), m.id_b);
    if (k < 0) { s_orphan = 1; continue; }                          // no detector with odometry: guess.at() throws
    if (v.traj_n[m.id_a] == 0) continue;
    atomicMax(&s_last[k], i);
    atomicMin(&s_det_min[k], m.id_a);
    atomicOr(&s_need[m.id_a >> 6], 1ull << (m.id_a & 63));        // verify() reads every detector's estimate
  }
  __syncthreads();
  for (int i = t; i < n_det; i += DA_THREADS) {
    const osb_measurement& m = v.meas[v.det_slot[i]];
    if (m.id_b < v.anon_min) continue;
    const int k = da_index(s_ids, min(n_u, DA_MAX_IDS), m.id_b);
    if (k >= 0 && m.id_a == s_det_min[k]) atomicMin(&s_first[k], i);
  }
  // available_nodes and t0 = the largest first odometry stamp (:56-65)
  const bool avail = t < D && v.traj_n[t] > 0;
  if (avail) {
    atomicOr(&s_avail[t >> 6], 1ull << (t & 63));
    atomicMax(&s_t0, (unsigned long long)v.traj_stamp[(size_t)t * v.max_samples] ^ (1ull << 63));
  }
  __syncthreads();
  if (!bit_of(s_avail, v.self_id)) return;                         // :53-55
  const int64_t t0 = (int64_t)(s_t0 ^ (1ull << 63));
  // est_poses_t0 (:67-76): self from its odometry, then every drone with a keyframe path (self overwritten)
  if (t == v.self_id) {
    store_pose(s_est[t], da_ego(v, t, t0, nullptr));
    atomicOr(&s_has[t >> 6], 1ull << (t & 63));
  }
  __syncthreads();
  bool bad = false;
  if (t < D && v.kf_first[t + 1] > v.kf_first[t]) {
    if (!avail) {
      bad = true;                                                  // ego_motions.at() throws
    } else {
      const int lo = v.kf_first[t], hi = v.kf_first[t + 1];
      const int k = lo + nearest_sample(v.kf_stamp + lo, hi - lo, t0);
      store_pose(s_est[t], pose_mul(load_pose(v.kf_pose + (size_t)k * 7), da_rel(v, t, v.kf_stamp[k], t0)));
      atomicOr(&s_has[t >> 6], 1ull << (t & 63));
    }
  }
  if (__syncthreads_or(bad)) {
    if (t == 0) R.status = OSB_ERR_INVALID;
    return;
  }
  if (n_u > DA_MAX_IDS) {
    if (t == 0) R.status = OSB_ERR_CAPACITY;
    return;
  }
  if (t == 0) {
    // the DFS with an explicit stack; frame l holds the remaining ids, the id and candidate it is at, whether a candidate
    // of that id succeeded, and what its candidate changed in est (to undo on return)
    uint32_t rem[DA_MAX_IDS + 1];
    int u_at[DA_MAX_IDS + 1], c_at[DA_MAX_IDS + 1], g[DA_MAX_IDS + 1];
    bool found[DA_MAX_IDS + 1], had[DA_MAX_IDS + 1];
    double old[DA_MAX_IDS + 1][7];
    int lvl = 0, status = OSB_OK;
    long long nodes = 0;
    bool recorded = false, ret = false;
    rem[0] = n_u == 32 ? 0xffffffffu : ((1u << n_u) - 1u);
    enum { ENTER, NEXT_U, NEXT_C, RETURN } step = ENTER;
    for (;;) {
      if (step == ENTER) {
        if (++nodes > v.max_nodes) { status = OSB_ERR_CAPACITY; break; }
        if (rem[lvl] == 0u) {                                      // a leaf (:166-181)
          unsigned long long need[DA_WORDS];
          for (int w = 0; w < DA_WORDS; ++w) need[w] = s_need[w];
          for (int l = 0; l < lvl; ++l) need[g[l] >> 6] |= 1ull << (g[l] & 63);
          bool miss = false, all = true;
          for (int w = 0; w < DA_WORDS; ++w) {
            miss = miss || (need[w] & ~s_has[w]) != 0ull;          // verify()'s est_pathes.at() throws
            all = all && s_has[w] == s_avail[w];
          }
          if (miss) { status = OSB_ERR_INVALID; break; }
          ret = v.thres > 0.0 && all;                              // verify() is 0: cost in [0, thres) iff thres > 0
          if (ret && !recorded) {
            for (int l = 0; l < lvl; ++l) s_guess[u_at[l]] = g[l];
            recorded = true;
          }
          step = RETURN;
          continue;
        }
        u_at[lvl] = -1;
        step = NEXT_U;
        continue;
      }
      if (step == RETURN) {
        if (lvl == 0) break;
        --lvl;
        const int c = c_at[lvl];
        if (c > 0) {                                               // undo this candidate's est entry
          if (had[lvl]) for (int j = 0; j < 7; ++j) s_est[c][j] = old[lvl][j];
          else s_has[c >> 6] &= ~(1ull << (c & 63));
        }
        found[lvl] = found[lvl] || ret;
        step = NEXT_C;
        continue;
      }
      if (step == NEXT_U) {                                        // the next id whose detector has an estimate
        int u = u_at[lvl] + 1;
        while (u < n_u && (!((rem[lvl] >> u) & 1u) || !bit_of(s_has, v.meas[v.det_slot[s_last[u]]].id_a))) ++u;
        if (u >= n_u) { ret = false; step = RETURN; continue; }
        u_at[lvl] = u;
        c_at[lvl] = -1;
        found[lvl] = false;
        step = NEXT_C;
        continue;
      }
      // NEXT_C: the next candidate drone of id u_at[lvl]
      const int u = u_at[lvl];
      const osb_measurement& last = v.meas[v.det_slot[s_last[u]]];
      int c = c_at[lvl] + 1;
      while (c < D && (!bit_of(s_avail, c) || c == last.id_a)) ++c;
      if (c >= D) {
        if (found[lvl]) { ret = true; step = RETURN; }             // the first success of this id is kept (:259-263)
        else step = NEXT_U;                                        // on to the next id
        continue;
      }
      c_at[lvl] = c;
      had[lvl] = false;
      if (c > 0) {                                                 // estimate_path (:277-289) and the Mahalanobis gate
        const osb_measurement& e = v.meas[v.det_slot[s_first[u]]];
        if (!bit_of(s_has, e.id_a)) { status = OSB_ERR_INVALID; break; }   // est_poses_t0.at(edge.id_a)
        const PoseD pose = pose_mul(pose_mul(pose_mul(load_pose(s_est[e.id_a]), da_rel(v, e.id_a, t0, e.stamp_a)),
                                             load_pose(e.relative_pose)), da_rel(v, c, e.stamp_b, t0));
        had[lvl] = bit_of(s_has, c);
        if (had[lvl]) {
          double lg[6];
          pose_log(pose_mul(pose_inv(load_pose(s_est[c])), pose), lg);
          if (!(smd6(lg, last.cov) < v.thres)) { c_at[lvl] = c; continue; }   // skip the candidate (step stays NEXT_C)
          for (int j = 0; j < 7; ++j) old[lvl][j] = s_est[c][j];
        }
        store_pose(s_est[c], pose);
        s_has[c >> 6] |= 1ull << (c & 63);
      }
      g[lvl] = c;
      rem[lvl + 1] = rem[lvl] & ~(1u << u);
      ++lvl;
      step = ENTER;
    }
    R.nodes = nodes;
    if (status == OSB_OK && ret && s_orphan) status = OSB_ERR_INVALID;   // guess.at() of a row left out of the search
    s_status = status;
    s_ok = status == OSB_OK && ret;
  }
  __syncthreads();
  if (!s_ok) {
    if (t == 0) R.status = s_status;
    return;
  }
  for (int i = t; i < n_det; i += DA_THREADS) {                    // :84-88, in place
    osb_measurement& m = v.meas_w[v.det_slot[i]];
    if (m.id_b >= v.anon_min) m.id_b = s_guess[da_index(s_ids, n_u, m.id_b)];
  }
  if (t < n_u) { R.anon[t] = s_ids[t]; R.guess[t] = s_guess[t]; }
  if (t == 0) { R.n = n_u; R.applied = 1; }
}

}  // namespace osb

using namespace osb;

static_assert(sizeof(osb_measurement) == 496, "osb_measurement layout");
static_assert(sizeof(osb_window_entry) == 80, "osb_window_entry layout");
static_assert(sizeof(osb_anchor_result) == 760, "osb_anchor_result layout");
static_assert(sizeof(osb_observability) == 5 * 256 + 16, "osb_observability layout");
static_assert(sizeof(osb_predict_result) == 128, "osb_predict_result layout");
static_assert(sizeof(osb_loop_record) == 88, "osb_loop_record layout");
static_assert(sizeof(osb_sync_params) == 24, "osb_sync_params layout");

// The parts of a handle's device state, one bit each.  A device call waits for the last call that touched (read or wrote)
// each part it touches, on any stream, and then becomes that part's last toucher: the touchers of a part form one chain,
// so one event per part orders them.  The trajectories, the run's window and init_mask's block table are written only by
// the synchronising updates (push_odometry, add_measurements, set_window), which wait for every part.
enum AnchorPart : unsigned {
  STORE = 1u << 0,        // measurements, loop and detection slots, device counts
  OBSERVE = 1u << 1,      // drone-pair matrix, observe window record, osb_observability record
  SYNC = 1u << 2,         // sync window table, keyframe and full paths, prediction records, outcome
  KEYFRAMES = 1u << 3,    // keyframe ring and its frame table
  LOOPS = 1u << 4,        // loop map, pair minima, meta words
  DA = 1u << 5,           // data association result, the applied word included
};
constexpr int ANCHOR_PARTS = 6;
constexpr unsigned ALL_PARTS = (1u << ANCHOR_PARTS) - 1;

struct osb_anchor {
  Resources res;
  int device = 0;
  osb_anchor_params p{};
  int64_t begin_dt_ns = 0;
  cudaStream_t stream = nullptr;
  cudaEvent_t last[ANCHOR_PARTS] = {};   // [k]: recorded after the last call that touched part 1 << k, on its stream
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
  // device appends (osb_anchor_add_measurements_dev), acquired by the first one: the counts on the device and their feedback
  // (each append charges its max_n and publishes the loop and detection counts and its status)
  int32_t* d_counts = nullptr;                    // [2] loops, detections
  CountFeedback fb;                               // fb.pending: an append may not have run, n_loops / n_dets are stale
  long long upper = 0;                            // bound of n_loops + n_dets while fb.pending
  osb_status last_status = OSB_OK;                // the last device append's, once synchronised
  // observe_dev, acquired by the first one: the drone-pair matrix (zero between calls), the window record and the
  // persistent state, which is also the outcome osb_anchor_observability reads
  unsigned* d_adj = nullptr;                      // [max_drones][8] 32-bit words
  ObserveWindow* d_obs_win = nullptr;
  osb_observability* d_obs = nullptr;
  ObserveWindow obs_win{};                        // the host's, kept by set_window whether or not observe ever ran
  // init_mask_dev: every window block's drone (-1: no entry) and its latest frame's self_pose quaternion, derived by
  // set_window on the host; the first init_mask_dev acquires the device copy (and its length), set_window keeps it current
  std::vector<int32_t> blk_drone;
  std::vector<double> blk_q;                      // [block][4] qw qx qy qz
  bool blk_negative = false;                      // a window entry with block < 0
  int32_t* d_blk_drone = nullptr;                 // [blk_cap], then the table's length
  double* d_blk_q = nullptr;
  size_t blk_cap = 0;
  // sync_dev, acquired by the first one: the window table (set_window keeps it current after that), the paths, the
  // prediction record and the outcome; predict's query and result buffers
  SyncWindow sync_win{};                          // the host's, kept by set_window whether or not a sync ever ran
  std::vector<int64_t> sw_stamp;
  std::vector<int32_t> sw_drone, sw_block;
  std::vector<double> sw_pose;
  int sw_max_block = -1;                          // the window's largest block id (-1: none)
  SyncWindow* d_sync_win = nullptr;
  int64_t* d_sw_stamp = nullptr;
  int32_t *d_sw_drone = nullptr, *d_sw_block = nullptr;
  double* d_sw_pose = nullptr;
  SyncOutcome* d_outcome = nullptr;
  SyncRecord* d_rec = nullptr;
  int32_t *d_kf_first = nullptr, *d_full_n = nullptr;
  int64_t *d_kf_stamp = nullptr, *d_full_stamp = nullptr;
  double *d_kf_pose = nullptr, *d_full_pose = nullptr;
  int max_full = 0;                               // ceil(max_traj_samples / 10)
  int32_t* d_pred_drone = nullptr;
  double* d_pred_vo = nullptr;
  osb_predict_result* d_pred_out = nullptr;
  // the keyframe store (osb_anchor_add_keyframe_dev / distance_factors_dev), acquired by the first of them: a ring of
  // max_keyframes slots, the window's frame table (set_window keeps it current after that), the pinned staging ring
  int64_t* d_st_stamp = nullptr;
  int32_t *d_st_n = nullptr, *d_st_first = nullptr;
  osb_keyframe_node* d_st_node = nullptr;
  osb_keyframe_distance* d_st_dist = nullptr;
  int8_t* d_st_flag = nullptr;
  std::vector<int64_t> st_stamp;                  // the host's record of the ring: each slot's stamp
  std::vector<int32_t> st_count;                  // ... its distance count, -1: empty
  long long kf_seq = 0;                           // keyframes added
  int kf_last_slot = -1;
  char* kf_stage[KF_STAGING] = {};                // pinned, mapped: nodes [max_drones] then dists [max_dists]
  char* kf_stage_dev[KF_STAGING] = {};
  cudaEvent_t kf_stage_ev[KF_STAGING] = {};
  std::vector<int64_t> kw_stamp;                  // the window's frames (set_window), host side
  std::vector<int32_t> kw_first, kw_drone, kw_block;
  int64_t* d_kw_stamp = nullptr;
  int32_t *d_kw_first = nullptr, *d_kw_drone = nullptr, *d_kw_block = nullptr, *d_kw_n = nullptr;
  int64_t kf_evicted = INT64_MIN;                 // the largest stamp whose slot a later keyframe took
  // the loop map (record_loops_dev, init_by_loops_dev), acquired by the first of them: H + 1 records, the pair minima,
  // the overflow flag and init_by_loops' status
  LoopRec* d_lm = nullptr;
  unsigned long long* d_lm_pair = nullptr;
  int32_t* d_lm_meta = nullptr;
  int lm_H = 0;
  // data association (set_data_association, data_association_dev): 0 until the setter, and then >= max_drones >= 1;
  // 0 makes no id_b anonymous
  int32_t da_anon_min = 0;
  osb_da_params da{};
  DaResult* d_da = nullptr;                       // acquired by the setter
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

// orders `st` after the last toucher of each part in `parts` (an external wait inside a capture)
osb_status anchor_wait(osb_anchor* h, unsigned parts, cudaStream_t st) {
  for (int k = 0; k < ANCHOR_PARTS; ++k)
    if (parts & (1u << k)) OSB_CUDA(wait_event_capturable(st, h->last[k]));
  return OSB_OK;
}

// makes the work enqueued on `st` so far the last toucher of each part in `parts` (an external record inside a capture,
// so the calls after a replay wait for the replayed work)
osb_status anchor_record(osb_anchor* h, unsigned parts, cudaStream_t st) {
  for (int k = 0; k < ANCHOR_PARTS; ++k)
    if (parts & (1u << k)) OSB_CUDA(record_event_capturable(h->last[k], st));
  return OSB_OK;
}

// the window's frame table of distance_factors_dev to the device, on the handle's stream (the caller synchronises)
osb_status upload_kf_window(osb_anchor* h) {
  const size_t nf = h->kw_stamp.size();           // <= max_window_entries: set_window keeps the frames with entries
  cudaStream_t st = h->stream;
  const int32_t n = (int32_t)nf;
  const size_t ne = h->kw_drone.size();
  OSB_CUDA(cudaMemcpyAsync(h->d_kw_n, &n, sizeof(n), cudaMemcpyHostToDevice, st));
  OSB_CUDA(cudaMemcpyAsync(h->d_kw_first, h->kw_first.data(), (nf + 1) * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  if (nf > 0) OSB_CUDA(cudaMemcpyAsync(h->d_kw_stamp, h->kw_stamp.data(), nf * sizeof(int64_t), cudaMemcpyHostToDevice, st));
  if (ne > 0) {
    OSB_CUDA(cudaMemcpyAsync(h->d_kw_drone, h->kw_drone.data(), ne * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    OSB_CUDA(cudaMemcpyAsync(h->d_kw_block, h->kw_block.data(), ne * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  }
  return OSB_OK;
}

// the window's part of sync: every entry ordered by (drone, frame), with its frame's stamp (a counting sort by drone)
void sync_window(osb_anchor* h, int n_frames, const int64_t* frame_stamps, const int32_t* frame_first,
                 const osb_window_entry* entries) {
  const int D = h->p.max_drones, n = n_frames == 0 ? 0 : frame_first[n_frames];
  SyncWindow& w = h->sync_win;
  std::fill(w.first, w.first + ANCHOR_MAX_DRONES + 1, 0);
  for (int e = 0; e < n; ++e) ++w.first[entries[e].drone_id + 1];
  for (int d = 0; d < D; ++d) w.first[d + 1] += w.first[d];
  for (int d = D + 1; d <= ANCHOR_MAX_DRONES; ++d) w.first[d] = w.first[D];
  w.n_frames = n_frames;
  w.push_stamp = 0;
  h->sw_stamp.resize(n); h->sw_drone.resize(n); h->sw_block.resize(n); h->sw_pose.resize((size_t)n * 7);
  std::vector<int32_t> fill(w.first, w.first + D);
  h->sw_max_block = -1;
  for (int f = 0; f < n_frames; ++f) {
    if (frame_first[f + 1] > frame_first[f]) w.push_stamp = frame_stamps[f];
    for (int e = frame_first[f]; e < frame_first[f + 1]; ++e) {
      const int k = fill[entries[e].drone_id]++;
      h->sw_stamp[k] = frame_stamps[f];
      h->sw_drone[k] = entries[e].drone_id;
      h->sw_block[k] = entries[e].block;
      std::copy(entries[e].self_pose, entries[e].self_pose + 7, h->sw_pose.begin() + (size_t)k * 7);
      h->sw_max_block = std::max(h->sw_max_block, entries[e].block);
    }
  }
}

// the sync's window table to the device, on the handle's stream (the caller synchronises)
osb_status upload_sync_window(osb_anchor* h) {
  cudaStream_t st = h->stream;
  const size_t n = h->sw_stamp.size();
  OSB_CUDA(cudaMemcpyAsync(h->d_sync_win, &h->sync_win, sizeof(SyncWindow), cudaMemcpyHostToDevice, st));
  if (n > 0) {
    OSB_CUDA(cudaMemcpyAsync(h->d_sw_stamp, h->sw_stamp.data(), n * sizeof(int64_t), cudaMemcpyHostToDevice, st));
    OSB_CUDA(cudaMemcpyAsync(h->d_sw_drone, h->sw_drone.data(), n * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    OSB_CUDA(cudaMemcpyAsync(h->d_sw_block, h->sw_block.data(), n * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    OSB_CUDA(cudaMemcpyAsync(h->d_sw_pose, h->sw_pose.data(), n * 7 * sizeof(double), cudaMemcpyHostToDevice, st));
  }
  return OSB_OK;
}

// the window's part of observe: all_nodes grows by every drone of the window; each drone's box spans its vo_available
// entries, from max = -1000 and min = +1000 per axis (boundingbox_sldwin, swarm_localization_solver.cpp:848-878)
void observe_window(ObserveWindow& w, int max_drones, int n_frames, int n_entries, const osb_window_entry* entries) {
  double lo[ANCHOR_MAX_DRONES][3], hi[ANCHOR_MAX_DRONES][3];
  for (int d = 0; d < max_drones; ++d)
    for (int j = 0; j < 3; ++j) { hi[d][j] = -1000.0; lo[d][j] = 1000.0; }
  for (int e = 0; e < n_entries; ++e) {
    const int d = entries[e].drone_id;
    w.nodes[d >> 6] |= 1ull << (d & 63);
    if (!entries[e].vo_available) continue;
    for (int j = 0; j < 3; ++j) {
      const double x = entries[e].self_pose[j];
      if (x > hi[d][j]) hi[d][j] = x;
      if (x < lo[d][j]) lo[d][j] = x;
    }
  }
  for (int d = 0; d < max_drones; ++d)
    for (int j = 0; j < 3; ++j) w.ext[d][j] = hi[d][j] - lo[d][j];
  int n_nodes = 0;
  for (int k = 0; k < OBS_WORDS; ++k) n_nodes += __builtin_popcountll(w.nodes[k]);
  w.n_frames = n_frames;
  w.n_nodes = n_nodes;
}

bool drone_ok(const osb_anchor* h, int32_t d) { return d >= 0 && d < h->p.max_drones; }

// wait for the last device append and take its exact counts and status (every synchronising call starts with this)
osb_status anchor_settle(osb_anchor* h) {
  if (!h->fb.pending) return OSB_OK;
  OSB_CUDA(cudaEventSynchronize(h->fb.ev));
  const CountRecord* r = h->fb.host;
  h->n_loops = (int)r->count[0];
  h->n_dets = (int)r->count[1];
  h->last_status = (osb_status)r->status;
  h->upper = h->n_loops + h->n_dets;
  h->fb.pending = false;
  h->fb.exact();
  return OSB_OK;
}

// the block table to the device: acquired at max_window_entries blocks (or the window's, if more), replaced by a larger one
// only when the window's block ids outgrow it.  The handle's stream is idle: the callers have waited for every part and
// synchronised.
osb_status upload_blocks(osb_anchor* h) {
  const size_t n_blk = h->blk_drone.size();
  if (!h->d_blk_drone || n_blk > h->blk_cap) {
    const size_t cap = std::max(n_blk, (size_t)h->p.max_window_entries);
    int32_t* drone = nullptr;
    double* q = nullptr;
    OSB_TRY(h->res.alloc(&drone, cap + 1));
    OSB_TRY(h->res.alloc(&q, 4 * cap));
    if (h->d_blk_drone) { h->res.release(h->d_blk_drone); h->res.release(h->d_blk_q); }
    h->d_blk_drone = drone; h->d_blk_q = q; h->blk_cap = cap;
  }
  const int32_t len = (int32_t)n_blk;
  cudaStream_t st = h->stream;
  if (n_blk > 0) {
    OSB_CUDA(cudaMemcpyAsync(h->d_blk_drone, h->blk_drone.data(), n_blk * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    OSB_CUDA(cudaMemcpyAsync(h->d_blk_q, h->blk_q.data(), 4 * n_blk * sizeof(double), cudaMemcpyHostToDevice, st));
  }
  OSB_CUDA(cudaMemcpyAsync(h->d_blk_drone + h->blk_cap, &len, sizeof(len), cudaMemcpyHostToDevice, st));
  OSB_CUDA(cudaStreamSynchronize(st));
  return OSB_OK;
}

}  // namespace

extern "C" osb_status osb_anchor_create(osb_anchor** out, const osb_anchor_params* p) {
  OSB_REQUIRE(out != nullptr && p != nullptr, "null argument");
  OSB_REQUIRE(p->max_drones > 0 && p->max_drones <= ANCHOR_MAX_DRONES, "max_drones must be in 1..256");
  OSB_REQUIRE(p->max_traj_samples > 0 && p->max_measurements > 0 && p->max_window_entries > 0, "capacities must be positive");
  OSB_REQUIRE((long long)p->max_drones * p->max_traj_samples < (1ll << 31), "max_drones x max_traj_samples too large");
  OSB_REQUIRE(p->begin_min_loop_dt_s >= 0.0 && p->begin_min_loop_dt_s < 9.0e9, "begin_min_loop_dt_s out of range");
  OSB_REQUIRE(p->max_keyframes >= 0 && (p->max_keyframes == 0 || p->max_keyframe_distances > 0),
              "max_keyframes must be >= 0, and max_keyframe_distances positive when it is not");
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
  for (cudaEvent_t& e : h->last) OSB_TRY(R.event(&e, cudaEventDisableTiming));
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
  OSB_TRY(anchor_record(h.get(), ALL_PARTS, h->stream));
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
  observe_window(h->obs_win, p->max_drones, 0, 0, nullptr);
  sync_window(h.get(), 0, nullptr, nullptr, nullptr);
  h->kw_first.assign(1, 0);
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
  OSB_TRY(anchor_wait(h, ALL_PARTS, h->stream));
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
  std::lock_guard<std::mutex> lk(h->mu);
  for (int i = 0; i < n; ++i) {
    OSB_REQUIRE(m[i].type == OSB_MEAS_LOOP || m[i].type == OSB_MEAS_DET4D || m[i].type == OSB_MEAS_DET6D,
                "unknown measurement type");
    const bool anon = m[i].type != OSB_MEAS_LOOP && h->da_anon_min > 0 && m[i].id_b >= h->da_anon_min;
    OSB_REQUIRE(drone_ok(h, m[i].id_a) && (drone_ok(h, m[i].id_b) || anon), "drone id outside 0..max_drones-1");
  }
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
  OSB_TRY(anchor_wait(h, ALL_PARTS, h->stream));
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
  if (h->d_kw_n)                                                   // a keyframe whose slot was taken has no rows left
    for (int f = 0; f < n_frames; ++f) {
      if (frame_first[f + 1] == frame_first[f] || frame_stamps_ns[f] > h->kf_evicted) continue;
      bool stored = false;
      for (int k = 0; k < h->p.max_keyframes && !stored; ++k) stored = h->st_count[k] >= 0 && h->st_stamp[k] == frame_stamps_ns[f];
      if (!stored) {
        set_error(__func__, "a window frame's keyframe has left the store: max_keyframes does not cover the window");
        return OSB_ERR_CAPACITY;
      }
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
  observe_window(h->obs_win, D, n_frames, n_entries, entries);
  // every entry, vo_available or not; frames in order, so a shared block keeps its latest frame's pose
  int n_blk = 0;
  h->blk_negative = false;
  for (int e = 0; e < n_entries; ++e) {
    h->blk_negative = h->blk_negative || entries[e].block < 0;
    n_blk = std::max(n_blk, entries[e].block + 1);
  }
  h->blk_drone.assign(n_blk, -1);
  h->blk_q.assign(4 * (size_t)n_blk, 0.0);
  for (int e = 0; e < n_entries; ++e) {
    const int b = entries[e].block;
    if (b < 0) continue;
    h->blk_drone[b] = entries[e].drone_id;
    std::copy(entries[e].self_pose + 3, entries[e].self_pose + 7, h->blk_q.begin() + 4 * (size_t)b);
  }
  OSB_TRY(anchor_wait(h, ALL_PARTS, h->stream));
  cudaStream_t st = h->stream;
  OSB_CUDA(cudaMemcpyAsync(h->d_drone_first, first.data(), (size_t)(D + 1) * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  if (h->d_obs_win)
    OSB_CUDA(cudaMemcpyAsync(h->d_obs_win, &h->obs_win, sizeof(ObserveWindow), cudaMemcpyHostToDevice, st));
  if (n_vo > 0) {
    OSB_CUDA(cudaMemcpyAsync(h->d_win_stamp, h->h_win_stamp.data(), (size_t)n_vo * sizeof(int64_t), cudaMemcpyHostToDevice, st));
    OSB_CUDA(cudaMemcpyAsync(h->d_win_frame, h->h_win_frame.data(), (size_t)n_vo * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    OSB_CUDA(cudaMemcpyAsync(h->d_win_block, h->h_win_block.data(), (size_t)n_vo * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    OSB_CUDA(cudaMemcpyAsync(h->d_win_pose, h->h_win_pose.data(), (size_t)n_vo * 7 * sizeof(double), cudaMemcpyHostToDevice, st));
  }
  sync_window(h, n_frames, frame_stamps_ns, frame_first, entries);
  if (h->d_sync_win) OSB_TRY(upload_sync_window(h));
  h->kw_stamp.clear();                                             // the frames that hold entries: no other has rows
  h->kw_first.assign(1, 0);
  for (int f = 0; f < n_frames; ++f)
    if (frame_first[f + 1] > frame_first[f]) { h->kw_stamp.push_back(frame_stamps_ns[f]); h->kw_first.push_back(frame_first[f + 1]); }
  h->kw_drone.resize(n_entries);
  h->kw_block.resize(n_entries);
  for (int e = 0; e < n_entries; ++e) { h->kw_drone[e] = entries[e].drone_id; h->kw_block[e] = entries[e].block; }
  if (h->d_kw_n) OSB_TRY(upload_kf_window(h));
  OSB_CUDA(cudaStreamSynchronize(st));
  if (h->d_blk_drone) OSB_TRY(upload_blocks(h));
  h->n_frames = n_frames;
  h->frame0_stamp = n_frames > 0 ? frame_stamps_ns[0] : 0;
  return OSB_OK;
}

namespace {

// pred: null for run / run_dev, the device word of run_dev_if, which also touches DA
osb_status anchor_launch(osb_anchor* h, const uint8_t* yaw_observable, osb_anchor_result* out_dev, int32_t* n_out,
                         cudaStream_t st, const int32_t* pred = nullptr) {
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
  if (h->fb.pending) {                          // the counts are the device's; the grid covers the host's bound of them
    long long n[2], since;                      // lowered by what the last append that has RUN reported
    if (h->fb.read(n, &since)) h->upper = std::min(h->upper, n[0] + n[1] + since);
    v.counts = h->d_counts;
    v.n_bound = (int)h->upper;
  }
  *n_out = v.n_bound;
  if (v.n_bound == 0) return OSB_OK;
  const unsigned parts = pred ? STORE | DA : STORE;
  const auto kernel = pred ? anchor_kernel<true> : anchor_kernel<false>;
  OSB_TRY(anchor_wait(h, parts, st));
  OSB_LAUNCH(kernel, cdiv(v.n_bound, ANCHOR_WARPS), ANCHOR_WARPS * 32, 0, st, v, out_dev, pred);
  OSB_CHECK_LAUNCH();
  return anchor_record(h, parts, st);
}

}  // namespace

extern "C" osb_status osb_anchor_run_dev(osb_anchor* h, const uint8_t* yaw_observable, osb_anchor_result* out_dev,
                                         int32_t* n_out, void* stream) {
  OSB_REQUIRE(h != nullptr && yaw_observable != nullptr && out_dev != nullptr && n_out != nullptr, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  return anchor_launch(h, yaw_observable, out_dev, n_out, (cudaStream_t)stream);
}

extern "C" osb_status osb_anchor_run_dev_if(osb_anchor* h, const uint8_t* yaw_observable, osb_anchor_result* out_dev,
                                            int32_t* n_out, const int32_t* pred_dev, void* stream) {
  OSB_REQUIRE(h != nullptr && yaw_observable != nullptr && out_dev != nullptr && n_out != nullptr && pred_dev != nullptr,
              "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  return anchor_launch(h, yaw_observable, out_dev, n_out, (cudaStream_t)stream, pred_dev);
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

// the first device append acquires the device counts (seeded with the host's exact ones) and the feedback
osb_status anchor_dev_init(osb_anchor* h) {
  if (h->d_counts) return OSB_OK;
  OSB_TRY(h->res.alloc(&h->d_counts, 2));
  OSB_TRY(h->fb.init(h->res));
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
  OSB_TRY(anchor_wait(h, STORE, st));
  if (h->fb.pending) {
    long long n[2], since;
    if (h->fb.read(n, &since)) h->upper = std::min(h->upper, n[0] + n[1] + since);
  } else {
    h->upper = h->n_loops + h->n_dets;
  }
  const long long seq = h->fb.charge(max_n);
  OSB_LAUNCH(anchor_append_kernel, 1, APPEND_THREADS, 0, st, m_dev, count_dev, max_n, loop_outlier_distance_threshold,
             h->p.max_drones, h->da_anon_min, h->p.max_measurements, h->d_meas, h->d_loop_slot, h->d_det_slot, h->d_counts, h->fb.dev, seq,
             h->fb.charged);
  OSB_CHECK_LAUNCH();
  OSB_TRY(anchor_record(h, STORE, st));
  OSB_CUDA(h->fb.record(st));
  h->upper = std::min<long long>(h->upper + max_n, h->p.max_measurements);
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

namespace {

// the first observe acquires the matrix (zeroed), the window record (the host's) and the state (zeroed)
osb_status observe_init(osb_anchor* h) {
  if (h->d_obs) return OSB_OK;
  const size_t D = (size_t)h->p.max_drones;
  OSB_TRY(h->res.alloc(&h->d_adj, D * OBS_ROW32));
  OSB_TRY(h->res.alloc(&h->d_obs_win, 1));
  osb_observability* obs = nullptr;
  OSB_TRY(h->res.alloc(&obs, 1));
  OSB_CUDA(cudaMemsetAsync(h->d_adj, 0, D * OBS_ROW32 * sizeof(unsigned), h->stream));
  OSB_CUDA(cudaMemsetAsync(obs, 0, sizeof(osb_observability), h->stream));
  OSB_CUDA(cudaMemcpyAsync(h->d_obs_win, &h->obs_win, sizeof(ObserveWindow), cudaMemcpyHostToDevice, h->stream));
  OSB_CUDA(cudaStreamSynchronize(h->stream));
  h->d_obs = obs;                                                  // set last: a failed first call is tried again
  return OSB_OK;
}

// pred: null for observe_dev, the device word of observe_dev_if, which also touches DA
osb_status observe_launch(osb_anchor* h, const osb_observe_params* p, osb_anchor_result* rows_dev, int n, cudaStream_t st,
                          const int32_t* pred = nullptr) {
  OSB_TRY(observe_init(h));
  const int D = h->p.max_drones;
  const int blocks = cdiv(std::max(n, 1), OBS_THREADS);
  const unsigned parts = pred ? OBSERVE | DA : OBSERVE;
  const auto edges = pred ? observe_edges_kernel<true> : observe_edges_kernel<false>;
  const auto state = pred ? observe_state_kernel<true> : observe_state_kernel<false>;
  const auto skip = pred ? observe_skip_kernel<true> : observe_skip_kernel<false>;
  OSB_TRY(anchor_wait(h, parts, st));
  OSB_LAUNCH(edges, std::min(blocks, 4 * num_sms()), OBS_THREADS, 0, st, rows_dev, n, D, h->d_adj, pred);
  OSB_CHECK_LAUNCH();
  OSB_LAUNCH(state, 1, OBS_THREADS, 0, st, reinterpret_cast<unsigned long long*>(h->d_adj), h->d_obs_win, D, p->self_id,
             p->init_xy_movement, p->init_z_movement, h->d_obs, pred);
  OSB_CHECK_LAUNCH();
  OSB_LAUNCH(skip, blocks, OBS_THREADS, 0, st, rows_dev, n, D, h->d_obs, pred);
  OSB_CHECK_LAUNCH();
  return anchor_record(h, parts, st);
}

}  // namespace

extern "C" osb_status osb_anchor_observe_dev(osb_anchor* h, const osb_observe_params* p, osb_anchor_result* rows_dev, int n,
                                             void* stream) {
  OSB_REQUIRE(h != nullptr && p != nullptr && rows_dev != nullptr, "null argument");
  OSB_REQUIRE(n >= 0, "negative row count");
  OSB_REQUIRE(drone_ok(h, p->self_id), "self_id outside 0..max_drones-1");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  return observe_launch(h, p, rows_dev, n, (cudaStream_t)stream);
}

extern "C" osb_status osb_anchor_observe_dev_if(osb_anchor* h, const osb_observe_params* p, osb_anchor_result* rows_dev,
                                                int n, const int32_t* pred_dev, void* stream) {
  OSB_REQUIRE(h != nullptr && p != nullptr && rows_dev != nullptr && pred_dev != nullptr, "null argument");
  OSB_REQUIRE(n >= 0, "negative row count");
  OSB_REQUIRE(drone_ok(h, p->self_id), "self_id outside 0..max_drones-1");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  return observe_launch(h, p, rows_dev, n, (cudaStream_t)stream, pred_dev);
}

extern "C" osb_status osb_anchor_observability(osb_anchor* h, osb_observability* out) {
  OSB_REQUIRE(h != nullptr && out != nullptr, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  if (!h->d_obs) {
    memset(out, 0, sizeof(*out));
    return OSB_OK;
  }
  DeviceGuard dg(h->device);
  OSB_TRY(anchor_wait(h, OBSERVE, h->stream));
  OSB_CUDA(cudaMemcpyAsync(out, h->d_obs, sizeof(*out), cudaMemcpyDeviceToHost, h->stream));
  OSB_CUDA(cudaStreamSynchronize(h->stream));
  return OSB_OK;
}

extern "C" osb_status osb_anchor_init_mask_dev(osb_anchor* h, int32_t self_id, int n_nodes, uint8_t* mask_dev,
                                               double* yaw_dev, void* stream) {
  OSB_REQUIRE(h != nullptr && mask_dev != nullptr && yaw_dev != nullptr, "null argument");
  OSB_REQUIRE(n_nodes >= 1, "n_nodes must be >= 1");
  OSB_REQUIRE(drone_ok(h, self_id), "self_id outside 0..max_drones-1");
  std::lock_guard<std::mutex> lk(h->mu);
  OSB_REQUIRE(h->d_obs != nullptr, "no osb_anchor_observe_dev call on this handle: to_init is not set");
  OSB_REQUIRE(!h->blk_negative && h->blk_drone.size() <= (size_t)n_nodes, "a window block outside 0..n_nodes-1");
  DeviceGuard dg(h->device);
  if (!h->d_blk_drone) {                                          // the first call acquires the table
    OSB_TRY(anchor_wait(h, ALL_PARTS, h->stream));
    OSB_TRY(upload_blocks(h));
  }
  cudaStream_t st = (cudaStream_t)stream;
  OSB_TRY(anchor_wait(h, OBSERVE, st));
  OSB_LAUNCH(init_mask_kernel, cdiv(n_nodes, 256), 256, 0, st, h->d_blk_drone, h->d_blk_q, h->d_blk_drone + h->blk_cap,
             n_nodes, self_id, h->d_obs, mask_dev, yaw_dev);
  OSB_CHECK_LAUNCH();
  return anchor_record(h, OBSERVE, st);
}

namespace {

// the first sync acquires the window table (the host's), the paths (no drone has one), the records (none valid) and the
// outcome (nothing applied)
osb_status sync_init(osb_anchor* h) {
  if (h->d_outcome) return OSB_OK;
  const size_t D = (size_t)h->p.max_drones, E = (size_t)h->p.max_window_entries;
  h->max_full = (int)cdiv64(h->p.max_traj_samples, FULL_PATH_STEP);
  const size_t F = D * (size_t)h->max_full;
  Resources& R = h->res;
  OSB_TRY(R.alloc(&h->d_sync_win, 1));
  OSB_TRY(R.alloc(&h->d_sw_stamp, E));
  OSB_TRY(R.alloc(&h->d_sw_drone, E));
  OSB_TRY(R.alloc(&h->d_sw_block, E));
  OSB_TRY(R.alloc(&h->d_sw_pose, E * 7));
  OSB_TRY(R.alloc(&h->d_kf_first, D + 1));
  OSB_TRY(R.alloc(&h->d_kf_stamp, E));
  OSB_TRY(R.alloc(&h->d_kf_pose, E * 7));
  OSB_TRY(R.alloc(&h->d_full_n, D));
  OSB_TRY(R.alloc(&h->d_full_stamp, F));
  OSB_TRY(R.alloc(&h->d_full_pose, F * 7));
  OSB_TRY(R.alloc(&h->d_rec, D));
  SyncOutcome* outcome = nullptr;
  OSB_TRY(R.alloc(&outcome, 1));
  cudaStream_t st = h->stream;
  OSB_CUDA(cudaMemsetAsync(h->d_kf_first, 0, (D + 1) * sizeof(int32_t), st));
  OSB_CUDA(cudaMemsetAsync(h->d_full_n, 0xff, D * sizeof(int32_t), st));
  OSB_CUDA(cudaMemsetAsync(h->d_rec, 0, D * sizeof(SyncRecord), st));
  OSB_CUDA(cudaMemsetAsync(outcome, 0, sizeof(SyncOutcome), st));
  OSB_TRY(upload_sync_window(h));
  OSB_CUDA(cudaStreamSynchronize(st));
  h->d_outcome = outcome;                                          // set last: a failed first call is tried again
  return OSB_OK;
}

}  // namespace

extern "C" osb_status osb_anchor_sync_dev(osb_anchor* h, osb_solver* s, const osb_sync_params* p, void* stream) {
  OSB_REQUIRE(h != nullptr && s != nullptr && p != nullptr, "null argument");
  OSB_REQUIRE(drone_ok(h, p->self_id), "self_id outside 0..max_drones-1");
  OSB_REQUIRE(!p->normalise || p->window_size >= 1, "window_size must be >= 1 when normalise is set");
  OSB_REQUIRE(!std::isnan(p->acpt_cost), "acpt_cost is NaN");
  SolverDeviceCall c{};
  OSB_TRY(solver_device_call(s, &c));
  std::lock_guard<std::mutex> lk(h->mu);
  OSB_REQUIRE(c.device == h->device, "the anchor and the solver are on different devices");
  OSB_REQUIRE(!h->blk_negative && h->sw_max_block < c.n_nodes, "a window block outside 0 .. the solver's node count - 1");
  DeviceGuard dg(h->device);
  OSB_TRY(sync_init(h));
  cudaStream_t st = (cudaStream_t)stream;
  SyncView v{};
  v.win = h->d_sync_win;
  v.w_stamp = h->d_sw_stamp; v.w_drone = h->d_sw_drone; v.w_block = h->d_sw_block; v.w_pose = h->d_sw_pose;
  v.max_entries = h->p.max_window_entries; v.max_drones = h->p.max_drones; v.max_samples = h->p.max_traj_samples;
  v.max_full = h->max_full;
  v.traj_stamp = h->d_traj_stamp; v.traj_pose = h->d_traj_pose; v.traj_n = h->d_traj_n;
  v.poses = c.poses; v.word = c.word; v.summary = c.summary; v.chosen = c.chosen;
  v.trials = c.trials; v.base_res = c.base_res;
  v.normalise = p->normalise ? 1 : 0; v.window_size = p->window_size; v.full_path = p->full_path ? 1 : 0;
  v.acpt_cost = p->acpt_cost;
  v.outcome = h->d_outcome; v.rec = h->d_rec;
  v.kf_first = h->d_kf_first; v.kf_stamp = h->d_kf_stamp; v.kf_pose = h->d_kf_pose;
  v.full_n = h->d_full_n; v.full_stamp = h->d_full_stamp; v.full_pose = h->d_full_pose;
  OSB_CUDA(wait_event_capturable(st, c.done));                    // the solved poses and the call's outcome
  OSB_TRY(anchor_wait(h, SYNC, st));
  OSB_LAUNCH(sync_gate_kernel, 1, SYNC_THREADS, 0, st, v);
  OSB_CHECK_LAUNCH();
  OSB_LAUNCH(sync_kf_kernel, cdiv(v.max_entries, 256), 256, 0, st, v);
  OSB_CHECK_LAUNCH();
  const long long work = (long long)v.max_drones * v.max_full;
  OSB_LAUNCH(sync_full_kernel, (int)std::min<long long>(cdiv64(work, 256), 8LL * num_sms()), 256, 0, st, v);
  OSB_CHECK_LAUNCH();
  return anchor_record(h, SYNC, st);
}

extern "C" osb_status osb_anchor_sync_result(osb_anchor* h, int32_t* applied, osb_status* last) {
  OSB_REQUIRE(h != nullptr && applied != nullptr && last != nullptr, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  *applied = 0;
  *last = OSB_OK;
  if (!h->d_outcome) return OSB_OK;
  DeviceGuard dg(h->device);
  SyncOutcome o;
  OSB_TRY(anchor_wait(h, SYNC, h->stream));
  OSB_CUDA(cudaMemcpyAsync(&o, h->d_outcome, sizeof(o), cudaMemcpyDeviceToHost, h->stream));
  OSB_CUDA(cudaStreamSynchronize(h->stream));
  *applied = o.applied;
  *last = (osb_status)o.status;
  return OSB_OK;
}

extern "C" osb_status osb_anchor_paths(osb_anchor* h, int full, int32_t drone, int64_t* stamps, double* poses7, int cap,
                                       int32_t* n) {
  OSB_REQUIRE(h != nullptr && n != nullptr && cap >= 0 && (cap == 0 || (stamps && poses7)), "null argument or negative cap");
  OSB_REQUIRE(drone_ok(h, drone), "drone id outside 0..max_drones-1");
  std::lock_guard<std::mutex> lk(h->mu);
  *n = -1;
  if (!h->d_outcome) return OSB_OK;
  DeviceGuard dg(h->device);
  cudaStream_t st = h->stream;
  OSB_TRY(anchor_wait(h, SYNC, st));
  int32_t cnt[2];
  const int64_t* src_stamp;
  const double* src_pose;
  if (full) {
    OSB_CUDA(cudaMemcpyAsync(cnt, h->d_full_n + drone, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    OSB_CUDA(cudaStreamSynchronize(st));
    const size_t o = (size_t)drone * h->max_full;
    src_stamp = h->d_full_stamp + o;
    src_pose = h->d_full_pose + o * 7;
  } else {
    OSB_CUDA(cudaMemcpyAsync(cnt, h->d_kf_first + drone, 2 * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    OSB_CUDA(cudaStreamSynchronize(st));
    src_stamp = h->d_kf_stamp + cnt[0];
    src_pose = h->d_kf_pose + (size_t)cnt[0] * 7;
    cnt[0] = cnt[1] > cnt[0] ? cnt[1] - cnt[0] : -1;
  }
  *n = cnt[0];
  const int k = std::min(cnt[0], cap);
  if (k > 0) {
    OSB_CUDA(cudaMemcpyAsync(stamps, src_stamp, (size_t)k * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    OSB_CUDA(cudaMemcpyAsync(poses7, src_pose, (size_t)k * 7 * sizeof(double), cudaMemcpyDeviceToHost, st));
    OSB_CUDA(cudaStreamSynchronize(st));
  }
  return OSB_OK;
}

extern "C" osb_status osb_anchor_predict(osb_anchor* h, const osb_predict_params* p, int n, const int32_t* drones,
                                         const double* vo_poses7, osb_predict_result* out) {
  OSB_REQUIRE(h != nullptr && p != nullptr, "null argument");
  OSB_REQUIRE(n >= 0 && n <= h->p.max_drones, "n outside 0..max_drones");
  OSB_REQUIRE(n == 0 || (drones && vo_poses7 && out), "null argument");
  OSB_REQUIRE(drone_ok(h, p->self_id), "self_id outside 0..max_drones-1");
  for (int i = 0; i < n; ++i) OSB_REQUIRE(drone_ok(h, drones[i]), "drone id outside 0..max_drones-1");
  std::lock_guard<std::mutex> lk(h->mu);
  if (n > 0) memset(out, 0, (size_t)n * sizeof(osb_predict_result));
  if (n == 0 || !p->finish_init || !h->d_outcome) return OSB_OK;   // :738-741; no sync: no record
  DeviceGuard dg(h->device);
  const size_t D = (size_t)h->p.max_drones;
  if (!h->d_pred_out) {
    OSB_TRY(h->res.alloc(&h->d_pred_drone, D));
    OSB_TRY(h->res.alloc(&h->d_pred_vo, D * 7));
    OSB_TRY(h->res.alloc(&h->d_pred_out, D));
  }
  cudaStream_t st = h->stream;
  OSB_TRY(anchor_wait(h, SYNC | OBSERVE, st));
  OSB_CUDA(cudaMemcpyAsync(h->d_pred_drone, drones, (size_t)n * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  OSB_CUDA(cudaMemcpyAsync(h->d_pred_vo, vo_poses7, (size_t)n * 7 * sizeof(double), cudaMemcpyHostToDevice, st));
  OSB_LAUNCH(predict_kernel, cdiv(n, 128), 128, 0, st, n, h->d_pred_drone, h->d_pred_vo, h->d_rec, h->d_obs, p->self_id,
             h->d_pred_out);
  OSB_CHECK_LAUNCH();
  OSB_CUDA(cudaMemcpyAsync(out, h->d_pred_out, (size_t)n * sizeof(osb_predict_result), cudaMemcpyDeviceToHost, st));
  OSB_CUDA(cudaStreamSynchronize(st));
  return OSB_OK;
}

namespace {

// the first keyframe or distance_factors_dev call acquires the store (every slot empty), the window's frame table (the
// host's) and the staging ring with its events
osb_status kf_init(osb_anchor* h) {
  if (h->d_kw_n) return OSB_OK;
  const size_t K = (size_t)h->p.max_keyframes, D = (size_t)h->p.max_drones, M = (size_t)h->p.max_keyframe_distances;
  const size_t E = (size_t)h->p.max_window_entries;
  Resources& R = h->res;
  OSB_TRY(R.alloc(&h->d_st_stamp, K));
  OSB_TRY(R.alloc(&h->d_st_n, K));
  OSB_TRY(R.alloc(&h->d_st_node, K * D));
  OSB_TRY(R.alloc(&h->d_st_first, K * (D + 1)));
  OSB_TRY(R.alloc(&h->d_st_dist, K * M));
  OSB_TRY(R.alloc(&h->d_st_flag, K * M));
  OSB_TRY(R.alloc(&h->d_kw_drone, E));
  OSB_TRY(R.alloc(&h->d_kw_stamp, E));
  OSB_TRY(R.alloc(&h->d_kw_first, E + 1));
  OSB_TRY(R.alloc(&h->d_kw_block, E));
  const size_t stage = D * sizeof(osb_keyframe_node) + M * sizeof(osb_keyframe_distance);
  for (int k = 0; k < KF_STAGING; ++k) {
    OSB_TRY(R.host_alloc(&h->kf_stage[k], stage, cudaHostAllocMapped));
    OSB_CUDA(cudaHostGetDevicePointer((void**)&h->kf_stage_dev[k], h->kf_stage[k], 0));
    OSB_TRY(R.event(&h->kf_stage_ev[k], cudaEventDisableTiming));
  }
  cudaStream_t st = h->stream;
  OSB_CUDA(cudaMemsetAsync(h->d_st_n, 0xff, K * sizeof(int32_t), st));
  int32_t* n = nullptr;
  OSB_TRY(R.alloc(&n, 1));
  h->d_kw_n = n;
  const osb_status s = upload_kf_window(h);
  if (s != OSB_OK) { h->d_kw_n = nullptr; return s; }
  for (int k = 0; k < KF_STAGING; ++k) OSB_CUDA(cudaEventRecord(h->kf_stage_ev[k], st));
  cudaError_t e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) { h->d_kw_n = nullptr; OSB_CUDA(e); }      // a failed first call is tried again
  h->st_stamp.assign(K, 0);
  h->st_count.assign(K, -1);
  return OSB_OK;
}

}  // namespace

extern "C" osb_status osb_anchor_add_keyframe_dev(osb_anchor* h, osb_solver* s, int64_t stamp_ns, int n_nodes,
                                                  const osb_keyframe_node* nodes, int n_distances,
                                                  const osb_keyframe_distance* dists, const osb_keyframe_params* p,
                                                  void* stream) {
  OSB_REQUIRE(h != nullptr && s != nullptr && p != nullptr && nodes != nullptr, "null argument");
  OSB_REQUIRE(n_distances >= 0 && (n_distances == 0 || dists != nullptr), "null dists or negative count");
  OSB_REQUIRE(h->p.max_keyframes > 0, "the handle was created with max_keyframes == 0");
  OSB_REQUIRE(n_nodes >= 1 && n_nodes <= h->p.max_drones, "n_nodes outside 1..max_drones");
  OSB_REQUIRE(drone_ok(h, p->self_id), "self_id outside 0..max_drones-1");
  long long total = 0;
  for (int i = 0; i < n_nodes; ++i) {
    OSB_REQUIRE(drone_ok(h, nodes[i].drone_id), "drone id outside 0..max_drones-1");
    OSB_REQUIRE(i == 0 || nodes[i].drone_id > nodes[i - 1].drone_id, "nodes must be in ascending drone id");
    OSB_REQUIRE(nodes[i].n_distances >= 0 && nodes[i].n_distances <= h->p.max_drones, "n_distances outside 0..max_drones");
    total += nodes[i].n_distances;
  }
  OSB_REQUIRE(total == n_distances, "the nodes' n_distances do not sum to n_distances");
  for (int i = 0, k = 0; i < n_nodes; ++i)
    for (int j = 0; j < nodes[i].n_distances; ++j, ++k) {
      OSB_REQUIRE(drone_ok(h, dists[k].peer), "peer id outside 0..max_drones-1");
      OSB_REQUIRE(j == 0 || dists[k].peer > dists[k - 1].peer, "a node's peers must be in ascending id");
    }
  if (n_distances > h->p.max_keyframe_distances) {
    set_error(__func__, "the keyframe has more distances than max_keyframe_distances");
    return OSB_ERR_CAPACITY;
  }
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  OSB_TRY(kf_init(h));
  for (int k = 0; k < h->p.max_keyframes; ++k)
    OSB_REQUIRE(h->st_count[k] < 0 || h->st_stamp[k] != stamp_ns, "a keyframe with this stamp is already stored");
  cudaStream_t st = (cudaStream_t)stream;
  SolverPoseWrite w{};
  {
    int solver_dev = 0;
    const int n_blocks = solver_node_count(s, &solver_dev);   // checked before anything is enqueued
    OSB_REQUIRE(solver_dev == h->device, "the anchor and the solver are on different devices");
    for (int i = 0; i < n_nodes; ++i) {
      const osb_keyframe_node& nd = nodes[i];
      OSB_REQUIRE(nd.block >= 0 && nd.block < n_blocks, "a block outside 0 .. the solver's node count - 1");
      const bool uses_prev = nd.new_block && !nd.is_static && (nd.drone_id != p->self_id || p->finish_init);
      OSB_REQUIRE(!uses_prev || (nd.prev_block >= -1 && nd.prev_block < n_blocks),
                  "a prev_block outside -1 .. the solver's node count - 1");
    }
  }
  const int slot = (int)(h->kf_seq % h->p.max_keyframes), stage = (int)(h->kf_seq % KF_STAGING);
  if (h->st_count[slot] >= 0)
    for (const int64_t ts : h->kw_stamp)
      if (ts == h->st_stamp[slot]) {
        set_error(__func__, "the oldest stored keyframe is still in the window: max_keyframes does not cover it");
        return OSB_ERR_CAPACITY;
      }
  OSB_TRY(solver_pose_write(s, st, &w));
  OSB_CUDA(cudaEventSynchronize(h->kf_stage_ev[stage]));           // the call KF_STAGING before has read its inputs
  const size_t D = (size_t)h->p.max_drones;
  memcpy(h->kf_stage[stage], nodes, (size_t)n_nodes * sizeof(osb_keyframe_node));
  char* dist_stage = h->kf_stage[stage] + D * sizeof(osb_keyframe_node);
  if (n_distances > 0) memcpy(dist_stage, dists, (size_t)n_distances * sizeof(osb_keyframe_distance));
  KeyframeView v{};
  v.nodes = reinterpret_cast<const osb_keyframe_node*>(h->kf_stage_dev[stage]);
  v.dists = reinterpret_cast<const osb_keyframe_distance*>(h->kf_stage_dev[stage] + D * sizeof(osb_keyframe_node));
  v.n_nodes = n_nodes; v.n_dists = n_distances; v.max_drones = h->p.max_drones; v.max_dists = h->p.max_keyframe_distances;
  v.stamp = stamp_ns;
  v.self_id = p->self_id; v.finish_init = p->finish_init ? 1 : 0; v.enable_distance = p->enable_distance ? 1 : 0;
  const bool no_rej = p->debug_no_rejection != 0;                  // :89-96
  v.thr = (double)(no_rej ? 1e8f : p->outlier_threshold);
  v.elev = (double)(no_rej ? 1e8f : p->elevation_threshold);
  v.min_d = (double)(no_rej ? -1.0f : p->minimum_distance);
  v.seed = p->seed;
  v.poses = w.poses;
  v.slot = slot; v.prev_slot = h->kf_last_slot;
  v.st_stamp = h->d_st_stamp; v.st_n = h->d_st_n; v.st_node = h->d_st_node; v.st_first = h->d_st_first;
  v.st_dist = h->d_st_dist; v.st_flag = h->d_st_flag;
  OSB_TRY(anchor_wait(h, KEYFRAMES, st));
  OSB_LAUNCH(keyframe_kernel, 1, KF_THREADS, 0, st, v);
  OSB_CHECK_LAUNCH();
  OSB_CUDA(record_event_capturable(w.written, st));
  OSB_CUDA(record_event_capturable(h->kf_stage_ev[stage], st));
  OSB_TRY(anchor_record(h, KEYFRAMES, st));
  if (h->st_count[slot] >= 0) h->kf_evicted = std::max(h->kf_evicted, h->st_stamp[slot]);
  h->st_stamp[slot] = stamp_ns;
  h->st_count[slot] = n_distances;
  h->kf_last_slot = slot;
  ++h->kf_seq;
  return OSB_OK;
}

extern "C" osb_status osb_anchor_keyframe_flags(osb_anchor* h, int64_t stamp_ns, int8_t* flags, int cap, int32_t* n) {
  OSB_REQUIRE(h != nullptr && n != nullptr && cap >= 0 && (cap == 0 || flags != nullptr), "null argument or negative cap");
  std::lock_guard<std::mutex> lk(h->mu);
  *n = -1;
  if (!h->d_kw_n) return OSB_OK;
  int slot = -1;
  for (int k = 0; k < h->p.max_keyframes; ++k)
    if (h->st_count[k] >= 0 && h->st_stamp[k] == stamp_ns) slot = k;
  if (slot < 0) return OSB_OK;
  *n = h->st_count[slot];
  const int m = std::min(*n, cap);
  if (m == 0) return OSB_OK;
  DeviceGuard dg(h->device);
  cudaStream_t st = h->stream;
  OSB_TRY(anchor_wait(h, KEYFRAMES, st));
  OSB_CUDA(cudaMemcpyAsync(flags, h->d_st_flag + (size_t)slot * h->p.max_keyframe_distances, (size_t)m,
                           cudaMemcpyDeviceToHost, st));
  OSB_CUDA(cudaStreamSynchronize(st));
  return OSB_OK;
}

extern "C" osb_status osb_anchor_distance_factors_dev(osb_anchor* h, const osb_distance_params* p, int32_t* type,
                                                      int32_t* ia, int32_t* ib, double* payload, uint8_t* huber,
                                                      int32_t* count_dev, int max_tail, void* stream) {
  OSB_REQUIRE(h != nullptr && p != nullptr && type && ia && ib && payload && huber && count_dev, "null argument");
  OSB_REQUIRE(max_tail >= 0, "max_tail must be >= 0");
  OSB_REQUIRE(drone_ok(h, p->self_id), "self_id outside 0..max_drones-1");
  OSB_REQUIRE(h->p.max_keyframes > 0, "the handle was created with max_keyframes == 0");
  std::lock_guard<std::mutex> lk(h->mu);
  OSB_REQUIRE(h->d_obs != nullptr, "no osb_anchor_observe_dev call on this handle: enable is not set");
  DeviceGuard dg(h->device);
  OSB_TRY(kf_init(h));
  DistanceView v{};
  v.w_stamp = h->d_kw_stamp; v.w_first = h->d_kw_first; v.w_drone = h->d_kw_drone; v.w_block = h->d_kw_block;
  v.w_n = h->d_kw_n;
  v.st_stamp = h->d_st_stamp; v.st_n = h->d_st_n; v.st_node = h->d_st_node; v.st_first = h->d_st_first;
  v.st_dist = h->d_st_dist; v.st_flag = h->d_st_flag;
  v.slots = h->p.max_keyframes; v.max_drones = h->p.max_drones; v.max_dists = h->p.max_keyframe_distances;
  v.obs = h->d_obs;
  v.self_id = p->self_id; v.enable_distance = p->enable_distance ? 1 : 0; v.huber = p->debug_no_rejection ? 0 : 1;
  v.sqrt_inf = 1.0 / sqrt((double)p->distance_measurement_cov);
  v.type = type; v.ia = ia; v.ib = ib; v.payload = payload; v.hub = huber; v.count = count_dev; v.max_tail = max_tail;
  cudaStream_t st = (cudaStream_t)stream;
  OSB_TRY(anchor_wait(h, OBSERVE | KEYFRAMES, st));
  OSB_LAUNCH(distance_factors_kernel, 1, DF_THREADS, 0, st, v);
  OSB_CHECK_LAUNCH();
  return anchor_record(h, OBSERVE | KEYFRAMES, st);
}

namespace {

// the first record_loops_dev or init_by_loops_dev acquires the map (no id recorded, no pair, no overflow)
osb_status loops_init(osb_anchor* h) {
  if (h->d_lm_meta) return OSB_OK;
  int H = 1;
  while (H < 2 * h->p.max_measurements) H <<= 1;
  const size_t D = (size_t)h->p.max_drones;
  Resources& R = h->res;
  OSB_TRY(R.alloc(&h->d_lm, (size_t)H + 1));
  OSB_TRY(R.alloc(&h->d_lm_pair, D * D));
  int32_t* meta = nullptr;
  OSB_TRY(R.alloc(&meta, 2));
  cudaStream_t st = h->stream;
  OSB_CUDA(cudaMemsetAsync(h->d_lm, 0xff, ((size_t)H + 1) * sizeof(LoopRec), st));   // key -1, claim none, not recorded
  OSB_CUDA(cudaMemsetAsync(h->d_lm_pair, 0xff, D * D * sizeof(unsigned long long), st));
  OSB_CUDA(cudaMemsetAsync(meta, 0, 2 * sizeof(int32_t), st));
  OSB_CUDA(cudaStreamSynchronize(st));
  h->lm_H = H;
  h->d_lm_meta = meta;                                             // set last: a failed first call is tried again
  return OSB_OK;
}

LoopMapView loop_map_view(const osb_anchor* h) {
  return LoopMapView{h->d_lm, h->d_lm_pair, h->d_lm_meta, h->lm_H, h->p.max_drones};
}

}  // namespace

extern "C" osb_status osb_anchor_record_loops_dev(osb_anchor* h, const osb_anchor_result* rows_dev, int n, void* stream) {
  OSB_REQUIRE(h != nullptr && n >= 0 && (n == 0 || rows_dev != nullptr), "null argument or negative count");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  OSB_TRY(loops_init(h));
  cudaStream_t st = (cudaStream_t)stream;
  const LoopMapView v = loop_map_view(h);
  const int blocks = std::min(cdiv(std::max(n, 1), LM_THREADS), 4 * num_sms());
  OSB_TRY(anchor_wait(h, LOOPS, st));
  OSB_LAUNCH(record_claim_kernel, blocks, LM_THREADS, 0, st, rows_dev, n, v);
  OSB_CHECK_LAUNCH();
  OSB_LAUNCH(record_write_kernel, blocks, LM_THREADS, 0, st, rows_dev, n, v);
  OSB_CHECK_LAUNCH();
  return anchor_record(h, LOOPS, st);
}

extern "C" osb_status osb_anchor_init_by_loops_dev(osb_anchor* h, osb_pcm_state* pcm, osb_solver* s, int32_t self_id,
                                                   void* stream) {
  OSB_REQUIRE(h != nullptr && pcm != nullptr && s != nullptr, "null argument");
  OSB_REQUIRE(drone_ok(h, self_id), "self_id outside 0..max_drones-1");
  PcmDeviceDir pd{};
  OSB_TRY(pcm_device_dir(pcm, &pd));
  int solver_dev = 0;
  const int n_blocks = solver_node_count(s, &solver_dev);
  std::lock_guard<std::mutex> lk(h->mu);
  OSB_REQUIRE(pd.device == h->device && solver_dev == h->device, "the handles are on different devices");
  OSB_REQUIRE(h->d_obs != nullptr, "no osb_anchor_observe_dev call on this handle: to_init is not set");
  OSB_REQUIRE(!h->blk_negative && h->sw_max_block < n_blocks, "a window block outside 0 .. the solver's node count - 1");
  DeviceGuard dg(h->device);
  OSB_TRY(loops_init(h));
  OSB_TRY(sync_init(h));
  cudaStream_t st = (cudaStream_t)stream;
  SolverPoseWrite w{};
  OSB_TRY(solver_pose_write(s, st, &w));
  InitLoopsView v{};
  v.obs = h->d_obs;
  v.dir = pd.dir;
  v.n_dir = pd.n_dir;
  v.lm = loop_map_view(h);
  v.win = h->d_sync_win; v.w_stamp = h->d_sw_stamp; v.w_block = h->d_sw_block;
  v.kf_first = h->d_kf_first; v.kf_stamp = h->d_kf_stamp; v.kf_pose = h->d_kf_pose;
  v.rec = h->d_rec;
  v.traj_stamp = h->d_traj_stamp; v.traj_pose = h->d_traj_pose; v.traj_n = h->d_traj_n;
  v.max_samples = h->p.max_traj_samples; v.max_drones = h->p.max_drones; v.self_id = self_id;
  v.poses = w.poses;
  if (pd.done) OSB_CUDA(wait_event_capturable(st, pd.done));     // the inlier sets of the last anchored PCM call
  OSB_TRY(anchor_wait(h, OBSERVE | SYNC | LOOPS, st));
  OSB_LAUNCH(init_by_loops_kernel, 1, IBL_THREADS, 0, st, v);
  OSB_CHECK_LAUNCH();
  OSB_CUDA(record_event_capturable(w.written, st));
  return anchor_record(h, OBSERVE | SYNC | LOOPS, st);
}

extern "C" osb_status osb_anchor_init_by_loops_result(osb_anchor* h, osb_status* last) {
  OSB_REQUIRE(h != nullptr && last != nullptr, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  *last = OSB_OK;
  if (!h->d_lm_meta) return OSB_OK;
  DeviceGuard dg(h->device);
  int32_t st = 0;
  OSB_TRY(anchor_wait(h, LOOPS, h->stream));
  OSB_CUDA(cudaMemcpyAsync(&st, h->d_lm_meta + 1, sizeof(st), cudaMemcpyDeviceToHost, h->stream));
  OSB_CUDA(cudaStreamSynchronize(h->stream));
  *last = (osb_status)st;
  return OSB_OK;
}

extern "C" osb_status osb_anchor_loop_map(osb_anchor* h, osb_loop_record* out, int cap, int32_t* n, int64_t* pair_min,
                                          uint8_t* estimated) {
  OSB_REQUIRE(h != nullptr && n != nullptr && cap >= 0 && (cap == 0 || out != nullptr), "null argument or negative cap");
  std::lock_guard<std::mutex> lk(h->mu);
  const size_t D = (size_t)h->p.max_drones;
  *n = 0;
  if (pair_min) std::fill(pair_min, pair_min + D * D, INT64_MAX);
  if (estimated) memset(estimated, 0, D);
  DeviceGuard dg(h->device);
  cudaStream_t st = h->stream;
  OSB_TRY(anchor_wait(h, LOOPS | SYNC, st));
  if (h->d_lm_meta) {
    std::vector<LoopRec> tab((size_t)h->lm_H + 1);
    std::vector<unsigned long long> pair(D * D);
    OSB_CUDA(cudaMemcpyAsync(tab.data(), h->d_lm, tab.size() * sizeof(LoopRec), cudaMemcpyDeviceToHost, st));
    OSB_CUDA(cudaMemcpyAsync(pair.data(), h->d_lm_pair, D * D * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    OSB_CUDA(cudaStreamSynchronize(st));
    std::vector<osb_loop_record> recs;
    for (const LoopRec& r : tab)
      if (r.recorded == 1u) recs.push_back(r.r);
    std::sort(recs.begin(), recs.end(), [](const osb_loop_record& a, const osb_loop_record& b) { return a.id < b.id; });
    *n = (int32_t)recs.size();
    std::copy(recs.begin(), recs.begin() + std::min((size_t)cap, recs.size()), out);
    if (pair_min)
      for (size_t k = 0; k < D * D; ++k)
        if (pair[k] != LM_NONE) pair_min[k] = (int64_t)(pair[k] ^ (1ull << 63));
  }
  if (estimated && h->d_rec) {
    std::vector<SyncRecord> rec(D);
    OSB_CUDA(cudaMemcpyAsync(rec.data(), h->d_rec, D * sizeof(SyncRecord), cudaMemcpyDeviceToHost, st));
    OSB_CUDA(cudaStreamSynchronize(st));
    for (size_t d = 0; d < D; ++d) estimated[d] = rec[d].estimated ? 1 : 0;
  }
  return OSB_OK;
}

extern "C" osb_status osb_anchor_set_data_association(osb_anchor* h, const osb_da_params* p) {
  OSB_REQUIRE(h != nullptr && p != nullptr, "null argument");
  OSB_REQUIRE(p->anon_min >= h->p.max_drones, "anon_min must be >= max_drones: an anonymous id is no drone id");
  OSB_REQUIRE(p->max_nodes >= 1, "max_nodes must be >= 1");
  OSB_REQUIRE(!std::isnan(p->accept_thres), "accept_thres is NaN");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  if (!h->d_da) {                                                  // the first call acquires the result
    DaResult* r = nullptr;
    OSB_TRY(h->res.alloc(&r, 1));
    OSB_CUDA(cudaMemsetAsync(r, 0, sizeof(DaResult), h->stream));
    OSB_CUDA(cudaStreamSynchronize(h->stream));
    h->d_da = r;
  }
  h->da = *p;
  h->da_anon_min = p->anon_min;
  return OSB_OK;
}

extern "C" osb_status osb_anchor_data_association_dev(osb_anchor* h, int32_t self_id, void* stream) {
  OSB_REQUIRE(h != nullptr, "null argument");
  OSB_REQUIRE(drone_ok(h, self_id), "self_id outside 0..max_drones-1");
  std::lock_guard<std::mutex> lk(h->mu);
  OSB_REQUIRE(h->d_da != nullptr, "no osb_anchor_set_data_association call on this handle");
  OSB_REQUIRE(h->d_obs != nullptr, "no osb_anchor_observe_dev call on this handle: the node set is not known");
  DeviceGuard dg(h->device);
  OSB_TRY(anchor_dev_init(h));
  OSB_TRY(sync_init(h));
  cudaStream_t st = (cudaStream_t)stream;
  DaView v{};
  v.obs = h->d_obs;
  v.meas = h->d_meas; v.meas_w = h->d_meas;
  v.det_slot = h->d_det_slot;
  v.counts = h->d_counts;
  v.traj_stamp = h->d_traj_stamp; v.traj_pose = h->d_traj_pose; v.traj_n = h->d_traj_n;
  v.kf_first = h->d_kf_first; v.kf_stamp = h->d_kf_stamp; v.kf_pose = h->d_kf_pose;
  v.max_samples = h->p.max_traj_samples; v.max_drones = h->p.max_drones; v.self_id = self_id;
  v.anon_min = h->da.anon_min; v.max_nodes = h->da.max_nodes;
  v.thres = (double)h->da.accept_thres;
  v.res = h->d_da;
  OSB_TRY(anchor_wait(h, STORE | OBSERVE | SYNC | DA, st));
  OSB_LAUNCH(data_association_kernel, 1, DA_THREADS, 0, st, v);
  OSB_CHECK_LAUNCH();
  return anchor_record(h, STORE | OBSERVE | SYNC | DA, st);
}

extern "C" osb_status osb_anchor_data_association_result(osb_anchor* h, int32_t* applied, osb_status* status,
                                                         osb_da_guess* guess, int cap, int32_t* n) {
  OSB_REQUIRE(h != nullptr && applied != nullptr && status != nullptr && n != nullptr && cap >= 0 &&
              (cap == 0 || guess != nullptr), "null argument or negative cap");
  std::lock_guard<std::mutex> lk(h->mu);
  *applied = 0;
  *status = OSB_OK;
  *n = 0;
  if (!h->d_da) return OSB_OK;
  DeviceGuard dg(h->device);
  DaResult r{};
  OSB_TRY(anchor_wait(h, DA, h->stream));
  OSB_CUDA(cudaMemcpyAsync(&r, h->d_da, sizeof(r), cudaMemcpyDeviceToHost, h->stream));
  OSB_CUDA(cudaStreamSynchronize(h->stream));
  *applied = r.applied;
  *status = (osb_status)r.status;
  *n = r.applied ? r.n : 0;
  for (int k = 0; k < std::min(cap, (int)*n); ++k) guess[k] = osb_da_guess{r.anon[k], r.guess[k]};
  return OSB_OK;
}

extern "C" osb_status osb_anchor_data_association_word(osb_anchor* h, const int32_t** applied_dev) {
  OSB_REQUIRE(h != nullptr && applied_dev != nullptr, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  OSB_REQUIRE(h->d_da != nullptr, "no osb_anchor_set_data_association call on this handle");
  *applied_dev = &h->d_da->applied;
  return OSB_OK;
}
