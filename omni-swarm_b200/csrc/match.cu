// match.cu -- keyframe database (exact inner-product top-k) and local-descriptor cross-check matcher.
//
// Replaces faiss::IndexFlatIP::{add,search} (swarm_loop/src/loop_detector.cpp:166-169,213) and
// cv::BFMatcher(NORM_L2, crossCheck=true).match (swarm_loop/src/loop_cam.cpp:147-150,
// swarm_loop/src/loop_detector.cpp:564-567).
//
// db_scan_kernel is the HBM-roofline kernel of the front-end: it streams the [N][4096] f32 database exactly
// once (algorithmic bytes = N * 16384 B per search batch, SURVEY.md section 8d) and keeps a per-CTA top-k so
// that only grid*k candidates reach the merge kernel.
#include "common.cuh"
#include "kernels.cuh"

namespace osb {

constexpr int DB_THREADS = 512;
constexpr int DB_CHUNK_MAX = 512;  // rows per CTA

// ---- shared tail of the scan kernels ----------------------------------------------------------------------------
// (1) the CTA emits the top-k of its own rows by rank counting (score desc, row id asc);
// (2) fused merge: the LAST CTA to finish (ticket counter) merges the per-CTA lists of each query in shared memory
//     (64-bit keys = inverted order-preserving score bits : row id) and writes the final k results -- no second
//     launch, which at 10 k rows was a third of the search time.  Used when k <= DB_FUSE_KMAX and grid <= DB_MERGE_MAX;
//     otherwise the host launches db_merge_kernel.
constexpr int DB_MERGE_MAX = 3584;       // heads + k*k candidate keys must fit the 32 KB key buffer
constexpr int DB_FUSE_KMAX = 16;
constexpr size_t DB_SCAN_SMEM = 200 * 1024;   // db_scan_kernel's dynamic shared-memory opt-in: Q x (dim + DB_CHUNK_MAX) floats

__device__ __forceinline__ unsigned long long db_key(float s, int64_t id) {
  if (id < 0) return ~0ull;
  s += 0.0f;                                                   // -0 -> +0 (they tie as floats)
  unsigned u = __float_as_uint(s);
  u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);              // ascending unsigned order == ascending float order
  return ((unsigned long long)(~u) << 32) | (unsigned long long)(unsigned)id;   // ascending key: score desc, id asc
}
__device__ __forceinline__ float db_key_score(unsigned long long key) {
  const unsigned o = ~(unsigned)(key >> 32);
  return __uint_as_float((o & 0x80000000u) ? (o & 0x7fffffffu) : ~o);
}

// the one row loader of both scan kernels: V is a group of 4 consecutive row elements, ld() returns them as fp32.  An fp16
// row is read at the same group (float4 column) index as an fp32 one, 8 bytes instead of 16, so every lane's fmaf chain is
// the fp32 kernel's own and an fp16 store scores exactly like an fp32 store holding the same rows already rounded to fp16.
template <typename T> struct DbRow4;
template <> struct DbRow4<float> {
  using V = float4;
  static __device__ __forceinline__ float4 ld(const V* p) { return ld_stream_f4(p); }
};
template <> struct DbRow4<__half> {
  using V = uint2;
  static __device__ __forceinline__ float4 ld(const V* p) { return ld_stream_h4(reinterpret_cast<const __half*>(p)); }
};

__device__ void db_emit_and_merge(const float* ss, int ss_stride, int nrows, int64_t row0, int nq, int k,
                                  float* __restrict__ part_scores, int64_t* __restrict__ part_ids,
                                  float* __restrict__ out_scores, int64_t* __restrict__ out_ids, unsigned int* done,
                                  int fuse, unsigned long long* keys) {
  const int tid = threadIdx.x, nthr = blockDim.x;
  for (int qq = 0; qq < nq; ++qq) {
    const float* s = ss + qq * ss_stride;
    float* ps = part_scores + ((size_t)qq * gridDim.x + blockIdx.x) * k;
    int64_t* pi = part_ids + ((size_t)qq * gridDim.x + blockIdx.x) * k;
    for (int i = tid; i < k; i += nthr)
      if (i >= nrows) { ps[i] = -INFINITY; pi[i] = -1; }
    for (int i = tid; i < nrows; i += nthr) {
      const float si = s[i];
      int rank = 0;
      for (int j = 0; j < nrows; ++j) {
        const float sj = s[j];
        rank += (sj > si) || (sj == si && j < i);
      }
      if (rank < k) { ps[rank] = si; pi[rank] = row0 + i; }
    }
  }
  if (!fuse) return;
  __shared__ int s_last;
  __threadfence();
  __syncthreads();
  if (tid == 0) s_last = (atomicAdd(done, 1u) == gridDim.x - 1);
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  // Every CTA's list is already in final order, so the global top-k can only come from the lists whose HEAD is among
  // the k best heads: rank the G heads (G^2 / 512 comparisons per thread, shared-memory broadcasts), pull those <= k
  // lists (k^2 candidates) and rank them.  Keys are unique (row ids are), so ranks are slots.
  const int G = gridDim.x;
  unsigned long long* heads = keys;                 // [G]
  unsigned long long* cand = keys + G;              // [k*k]
  __shared__ int s_sel[DB_FUSE_KMAX];
  __shared__ int s_nsel;
  for (int qq = 0; qq < nq; ++qq) {
    const float* ps = part_scores + (size_t)qq * G * k;
    const int64_t* pi = part_ids + (size_t)qq * G * k;
    __syncthreads();
    if (tid == 0) s_nsel = 0;
    for (int b = tid; b < G; b += nthr) heads[b] = db_key(__ldcg(ps + (size_t)b * k), __ldcg(pi + (size_t)b * k));
    __syncthreads();
    for (int b = tid; b < G; b += nthr) {
      const unsigned long long kb = heads[b];
      if (kb == ~0ull) continue;
      int rank = 0;
      for (int j = 0; j < G; ++j) rank += heads[j] < kb;
      if (rank < k) { s_sel[rank] = b; atomicMax(&s_nsel, rank + 1); }
    }
    __syncthreads();
    const int nsel = s_nsel, nc = nsel * k;
    for (int i = tid; i < nc; i += nthr) {
      const size_t src = (size_t)s_sel[i / k] * k + (i % k);
      cand[i] = db_key(__ldcg(ps + src), __ldcg(pi + src));
    }
    for (int i = tid; i < k; i += nthr) { out_scores[qq * k + i] = -INFINITY; out_ids[qq * k + i] = -1; }
    __syncthreads();
    for (int i = tid; i < nc; i += nthr) {
      const unsigned long long ki = cand[i];
      if (ki == ~0ull) continue;
      int rank = 0;
      for (int j = 0; j < nc; ++j) rank += cand[j] < ki;
      if (rank < k) {
        out_scores[qq * k + rank] = db_key_score(ki);
        out_ids[qq * k + rank] = (int64_t)(unsigned)(ki & 0xffffffffull);
      }
    }
  }
  if (tid == 0) *done = 0;                                     // ready for the next search on this scratch
}

// -------------------------------------------------------------------------------------------------------------
// db_scan_coop_kernel<T,Q>: small databases (<= DB_COOP_CHUNK rows per CTA, i.e. <= ~19 k rows; dim = 4096).  With few
// rows per CTA the warp-per-row scheme leaves half the warps idle (10 k rows / 296 CTAs = 34 rows = 9 groups of 4 for
// 16 warps) and too few bytes in flight.  Here ALL 16 warps share every row: warp w owns float4 columns
// [64w, 64w+64) -- its slice of the queries lives in registers (no shared-memory query copy at all), each lane has
// R x 2 independent 16-byte streaming loads in flight, and the 16 partial sums per row are added in fixed warp order
// (deterministic).
// -------------------------------------------------------------------------------------------------------------
constexpr int DB_COOP_CHUNK = 64;
constexpr int DB_COOP_DIM = 4096;

template <typename T, int Q>
__global__ void __launch_bounds__(DB_THREADS, (Q <= 2) ? 2 : 1)
db_scan_coop_kernel(const T* __restrict__ db, int64_t n_val, const int64_t* __restrict__ n_dev,
                    const float* __restrict__ q, int nq, int k, float* __restrict__ part_scores,
                    int64_t* __restrict__ part_ids, float* __restrict__ out_scores, int64_t* __restrict__ out_ids,
                    unsigned int* done, int fuse) {
  constexpr int DIM4 = DB_COOP_DIM / 4, NW = DB_THREADS / 32, C = DIM4 / (NW * 32), R = 4, CH = DB_COOP_CHUNK;
  static_assert(C == 2, "column slice");
  extern __shared__ __align__(16) float smem[];
  float* partial = smem;                        // [NW][CH][Q]
  float* ss = smem + NW * CH * Q;               // [Q][CH]
  if (!fuse && blockIdx.x == 0)
    for (int i = threadIdx.x; i < nq * k; i += DB_THREADS) { out_scores[i] = -INFINITY; out_ids[i] = -1; }
  const int64_t n = n_dev ? *n_dev : n_val;
  const int64_t chunk = (n + gridDim.x - 1) / gridDim.x;         // <= CH: the grid was sized for an upper bound of n
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t row0 = (int64_t)blockIdx.x * chunk;
  const int64_t row1 = min(n, row0 + chunk);
  // the grid was sized from a HOST upper bound of n; should the device count ever exceed it, rows beyond the chunk are
  // dropped rather than written past the shared arrays (the front-end keeps the bound exact, see fe_refresh_counts)
  const int nrows = (int)min((int64_t)CH, max((int64_t)0, row1 - row0));
  const int col = warp * (C * 32) + lane;
  float4 wq[Q][C];
#pragma unroll
  for (int qq = 0; qq < Q; ++qq)
#pragma unroll
    for (int c = 0; c < C; ++c)
      wq[qq][c] = (qq < nq) ? __ldg(reinterpret_cast<const float4*>(q) + (size_t)qq * DIM4 + col + c * 32)
                            : make_float4(0.f, 0.f, 0.f, 0.f);
  using V = typename DbRow4<T>::V;
  const V* base = reinterpret_cast<const V*>(db) + row0 * DIM4 + col;
#pragma unroll 2
  for (int r0 = 0; r0 < nrows; r0 += R) {
    float4 v[R][C];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const int row = min(r0 + r, nrows - 1);                      // clamped: the surplus loads hit a valid row
#pragma unroll
      for (int c = 0; c < C; ++c) v[r][c] = DbRow4<T>::ld(base + (size_t)row * DIM4 + c * 32);
    }
#pragma unroll
    for (int r = 0; r < R; ++r)
#pragma unroll
      for (int qq = 0; qq < Q; ++qq) {
        float a = 0.f;
#pragma unroll
        for (int c = 0; c < C; ++c) {
          a = fmaf(v[r][c].x, wq[qq][c].x, a);
          a = fmaf(v[r][c].y, wq[qq][c].y, a);
          a = fmaf(v[r][c].z, wq[qq][c].z, a);
          a = fmaf(v[r][c].w, wq[qq][c].w, a);
        }
        a = warp_sum(a);
        if (lane == 0 && r0 + r < nrows) partial[(warp * CH + r0 + r) * Q + qq] = a;
      }
  }
  __syncthreads();
  for (int i = tid; i < nrows * Q; i += DB_THREADS) {
    const int row = i / Q, qq = i % Q;
    float a = 0.f;
#pragma unroll
    for (int w = 0; w < NW; ++w) a += partial[(w * CH + row) * Q + qq];
    ss[qq * CH + row] = a;
  }
  __syncthreads();
  db_emit_and_merge(ss, CH, nrows, row0, nq, k, part_scores, part_ids, out_scores, out_ids, done, fuse,
                    reinterpret_cast<unsigned long long*>(smem));
}

// -------------------------------------------------------------------------------------------------------------
// db_scan_kernel<T,Q,R>: each warp owns R consecutive rows at a time and dots them with Q queries held in shared
// memory; a lane streams float4 columns lane, lane+32, ... of all R rows (R independent 16-byte loads in flight,
// 512 contiguous bytes per row per warp instruction).  Scores of the CTA's row chunk are parked in shared memory
// and the CTA emits its own top-k by rank counting (score desc, row id asc: the library's documented tie rule).
// -------------------------------------------------------------------------------------------------------------

template <typename T, int Q, int R>
__global__ void __launch_bounds__(DB_THREADS)
db_scan_kernel(const T* __restrict__ db, int64_t n_val, const int64_t* __restrict__ n_dev, int dim,
               const float* __restrict__ q, int nq, int k, float* __restrict__ part_scores,
               int64_t* __restrict__ part_ids, float* __restrict__ out_scores, int64_t* __restrict__ out_ids,
               unsigned int* done, int fuse) {
  if (!fuse && blockIdx.x == 0)   // final rows start as "no result" (faiss: -inf / -1); the merge kernel overwrites the hits
    for (int i = threadIdx.x; i < nq * k; i += DB_THREADS) { out_scores[i] = -INFINITY; out_ids[i] = -1; }
  // the row count may live on the device (keyframe front-end: rows are appended without a host round trip);
  // the launch grid was sized for an upper bound, the chunk is derived from the true count.
  const int64_t n = n_dev ? *n_dev : n_val;
  const int64_t chunk = (n + gridDim.x - 1) / gridDim.x;
  extern __shared__ __align__(16) float smem[];
  float* sq = smem;                         // [Q][dim]
  float* ss = smem + (size_t)Q * dim;       // [Q][DB_CHUNK_MAX]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = DB_THREADS / 32;
  const int dim4 = dim >> 2;
  for (int i = tid; i < Q * dim4; i += DB_THREADS) {
    int qq = i / dim4;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (qq < nq) v = reinterpret_cast<const float4*>(q)[i];
    reinterpret_cast<float4*>(sq)[i] = v;
  }
  __syncthreads();
  const int64_t row0 = (int64_t)blockIdx.x * chunk;
  const int64_t row1 = min(n, row0 + chunk);
  const int nrows = (int)min((int64_t)DB_CHUNK_MAX, max((int64_t)0, row1 - row0));   // (same guard as the cooperative kernel)
  const int ngroups = (nrows + R - 1) / R;
  for (int g = warp; g < ngroups; g += nwarps) {
    const int64_t r0 = row0 + (int64_t)g * R;
    using V = typename DbRow4<T>::V;
    const V* rp[R];
    bool valid[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      valid[r] = (r0 + r) < row0 + nrows;
      rp[r] = reinterpret_cast<const V*>(db + (valid[r] ? (r0 + r) : r0) * (int64_t)dim);
    }
    float acc[R][Q];
#pragma unroll
    for (int r = 0; r < R; ++r)
#pragma unroll
      for (int qq = 0; qq < Q; ++qq) acc[r][qq] = 0.f;
#pragma unroll 2
    for (int j = lane; j < dim4; j += 32) {
      float4 v[R];
#pragma unroll
      for (int r = 0; r < R; ++r) v[r] = DbRow4<T>::ld(rp[r] + j);
#pragma unroll
      for (int qq = 0; qq < Q; ++qq) {
        const float4 w = reinterpret_cast<const float4*>(sq + (size_t)qq * dim)[j];
#pragma unroll
        for (int r = 0; r < R; ++r) {
          acc[r][qq] = fmaf(v[r].x, w.x, acc[r][qq]);
          acc[r][qq] = fmaf(v[r].y, w.y, acc[r][qq]);
          acc[r][qq] = fmaf(v[r].z, w.z, acc[r][qq]);
          acc[r][qq] = fmaf(v[r].w, w.w, acc[r][qq]);
        }
      }
    }
#pragma unroll
    for (int r = 0; r < R; ++r)
#pragma unroll
      for (int qq = 0; qq < Q; ++qq) {
        float s = warp_sum(acc[r][qq]);
        if (lane == 0 && valid[r]) ss[qq * DB_CHUNK_MAX + g * R + r] = s;
      }
  }
  __syncthreads();
  db_emit_and_merge(ss, DB_CHUNK_MAX, nrows, row0, nq, k, part_scores, part_ids, out_scores, out_ids, done, fuse,
                    reinterpret_cast<unsigned long long*>(smem));
}

// merge: rank counting over the grid*k partial candidates, spread over many CTAs: CTA (x, q) ranks candidates
// [32x, 32x+32) of query q -- one candidate per warp, the 32 lanes split the comparison range and a shuffle reduction
// adds the partial counts.  A candidate whose rank is < k writes itself to its final slot (ranks are unique: ids are).
// The output rows are pre-filled with (-inf, -1) by block 0 of the scan kernel.
__global__ void __launch_bounds__(1024)
db_merge_kernel(const float* __restrict__ part_scores, const int64_t* __restrict__ part_ids, int ncand, int k,
                float* __restrict__ out_scores, int64_t* __restrict__ out_ids) {
  const int qq = blockIdx.y;
  const float* ps = part_scores + (size_t)qq * ncand;
  const int64_t* pi = part_ids + (size_t)qq * ncand;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int i = blockIdx.x * 32 + warp;
  if (i >= ncand) return;
  const int64_t idi = __ldg(pi + i);
  if (idi < 0) return;                       // warp-uniform
  const float si = __ldg(ps + i);
  int rank = 0;
  for (int j = lane; j < ncand; j += 32) {
    const int64_t idj = __ldg(pi + j);
    const float sj = __ldg(ps + j);
    rank += (idj >= 0) && ((sj > si) || (sj == si && idj < idi));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) rank += __shfl_xor_sync(0xffffffffu, rank, o);
  if (lane == 0 && rank < k) { out_scores[qq * k + rank] = si; out_ids[qq * k + rank] = idi; }
}

template <int Q, typename T>
static osb_status launch_scan(const T* db, int64_t n, const int64_t* n_dev, int dim, const float* q, int nq,
                              int k, int grid, bool coop, float* ps, int64_t* pi, float* os, int64_t* oi,
                              unsigned int* done, int fuse, cudaStream_t st) {
  constexpr int R = 4;
  const size_t merge_bytes = fuse ? (size_t)(DB_MERGE_MAX + DB_FUSE_KMAX * DB_FUSE_KMAX) * sizeof(unsigned long long) : 0;
  if (coop) {
    const size_t smem = std::max(merge_bytes, (size_t)(DB_THREADS / 32 + 1) * DB_COOP_CHUNK * Q * sizeof(float));
    OSB_SMEM_OPT_IN((db_scan_coop_kernel<T, Q>), 64 * 1024);
    OSB_LAUNCH((db_scan_coop_kernel<T, Q>), grid, DB_THREADS, smem, st, db, n, n_dev, q, nq, k, ps, pi, os, oi, done, fuse);
    OSB_CHECK_LAUNCH();
    return OSB_OK;
  }
  const size_t smem = std::max(merge_bytes, ((size_t)Q * dim + (size_t)Q * DB_CHUNK_MAX) * sizeof(float));
  OSB_SMEM_OPT_IN((db_scan_kernel<T, Q, R>), DB_SCAN_SMEM);
  OSB_LAUNCH((db_scan_kernel<T, Q, R>), grid, DB_THREADS, smem, st, db, n, n_dev, dim, q, nq, k, ps, pi, os, oi, done, fuse);
  OSB_CHECK_LAUNCH();
  return OSB_OK;
}

// largest grid any search over <= n rows uses (scratch sizing)
int db_scan_grid(int64_t n, int64_t* chunk_out) {
  // two CTAs (2 x 16 warps) per SM
  int grid = 2 * num_sms();
  int64_t chunk = cdiv64(n > 0 ? n : 1, grid);
  if (chunk > DB_CHUNK_MAX) {
    chunk = DB_CHUNK_MAX;
    grid = (int)cdiv64(n, chunk);
  }
  *chunk_out = chunk;
  return grid;
}

// device-side search of up to 8 queries per pass; the scratch holds 8*grid_max*k floats / int64 and one ticket counter
// (zero between searches).  n is an upper bound of *n_dev when n_dev is given.  rows are float or, with
// storage == OSB_DB_STORAGE_FP16, __half; the grid, kernel choice, passes and merge do not depend on the storage.
osb_status db_search_device(const void* rows, int storage, int64_t n, const int64_t* n_dev, int dim, const float* q_dev, int nq,
                            int k, float* part_scores, int64_t* part_ids, unsigned int* done, float* scores_dev,
                            int64_t* ids_dev, cudaStream_t st) {
  int64_t chunk;
  int grid = db_scan_grid(n, &chunk);
  // small databases: every warp of a CTA shares each row (db_scan_coop_kernel); a CTA never gets more than 64 rows
  const bool coop = (dim == DB_COOP_DIM) && chunk <= DB_COOP_CHUNK;
  if (coop) grid = (int)std::max<int64_t>(1, std::min<int64_t>(grid, n));
  const int fuse = (done != nullptr && k <= DB_FUSE_KMAX && grid <= DB_MERGE_MAX) ? 1 : 0;
  // queries per pass: 8 while db_scan_kernel<8,4>'s query slab and score rows fit its shared memory (dim <= 5888),
  // else 4, which fits up to dim 12288
  const int pass = (8 * ((size_t)dim + DB_CHUNK_MAX) * sizeof(float) <= DB_SCAN_SMEM) ? 8 : 4;
  for (int q0 = 0; q0 < nq; q0 += pass) {
    const int nb = min(pass, nq - q0);
    const float* qp = q_dev + (size_t)q0 * dim;
    float* os = scores_dev + (size_t)q0 * k;
    int64_t* oi = ids_dev + (size_t)q0 * k;
    auto scan = [&](auto* r) {
      if (nb == 1) return launch_scan<1>(r, n, n_dev, dim, qp, nb, k, grid, coop, part_scores, part_ids, os, oi, done, fuse, st);
      if (nb == 2) return launch_scan<2>(r, n, n_dev, dim, qp, nb, k, grid, coop, part_scores, part_ids, os, oi, done, fuse, st);
      if (nb <= 4) return launch_scan<4>(r, n, n_dev, dim, qp, nb, k, grid, coop, part_scores, part_ids, os, oi, done, fuse, st);
      return launch_scan<8>(r, n, n_dev, dim, qp, nb, k, grid, coop, part_scores, part_ids, os, oi, done, fuse, st);
    };
    const osb_status s = storage == OSB_DB_STORAGE_FP16 ? scan(static_cast<const __half*>(rows))
                                                        : scan(static_cast<const float*>(rows));
    if (s != OSB_OK) return s;
    if (!fuse) {
      OSB_LAUNCH(db_merge_kernel, dim3(cdiv(grid * k, 32), nb), 1024, 0, st, part_scores, part_ids, grid * k, k, os, oi);
      OSB_CHECK_LAUNCH();
    }
  }
  return OSB_OK;
}

// -------------------------------------------------------------------------------------------------------------
// cross-check matcher
// -------------------------------------------------------------------------------------------------------------
constexpr int BF_ROWS = 16;   // query rows per CTA
constexpr int BF_DIM = 64;

// dist[pair][i][j] = sqrt(sum_k (q_ik - t_jk)^2), accumulated k = 0..63 with separately rounded sub/mul/add
// (no FMA contraction) so that the distances are bit-identical to the oracle's scalar order.
__global__ void __launch_bounds__(256)
bf_dist_kernel(const float* const* __restrict__ qptr, const int32_t* __restrict__ nq,
               const float* const* __restrict__ tptr, const int32_t* __restrict__ nt, int max_n,
               float* __restrict__ dist) {
  __shared__ __align__(16) float sq[BF_ROWS][BF_DIM];
  const int pair = blockIdx.y;
  const int n_q = nq[pair], n_t = nt[pair];
  const int i0 = blockIdx.x * BF_ROWS;
  if (i0 >= n_q) return;
  const float* qp = qptr[pair];
  const float* tp = tptr[pair];
  for (int e = threadIdx.x; e < BF_ROWS * BF_DIM / 4; e += blockDim.x) {
    const int r = e / (BF_DIM / 4);
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (i0 + r < n_q) v = reinterpret_cast<const float4*>(qp + (size_t)(i0 + r) * BF_DIM)[e % (BF_DIM / 4)];
    reinterpret_cast<float4*>(&sq[0][0])[e] = v;
  }
  __syncthreads();
  const int j = threadIdx.x;
  if (j >= n_t) return;
  float tv[BF_DIM];
#pragma unroll
  for (int k4 = 0; k4 < BF_DIM / 4; ++k4) {
    const float4 v = reinterpret_cast<const float4*>(tp + (size_t)j * BF_DIM)[k4];
    tv[4 * k4] = v.x; tv[4 * k4 + 1] = v.y; tv[4 * k4 + 2] = v.z; tv[4 * k4 + 3] = v.w;
  }
  float acc[BF_ROWS];
#pragma unroll
  for (int r = 0; r < BF_ROWS; ++r) acc[r] = 0.f;
#pragma unroll
  for (int k4 = 0; k4 < BF_DIM / 4; ++k4) {
#pragma unroll
    for (int r = 0; r < BF_ROWS; ++r) {
      const float4 qv = reinterpret_cast<const float4*>(&sq[r][0])[k4];
      float d;
      d = __fsub_rn(qv.x, tv[4 * k4]);     acc[r] = __fadd_rn(acc[r], __fmul_rn(d, d));
      d = __fsub_rn(qv.y, tv[4 * k4 + 1]); acc[r] = __fadd_rn(acc[r], __fmul_rn(d, d));
      d = __fsub_rn(qv.z, tv[4 * k4 + 2]); acc[r] = __fadd_rn(acc[r], __fmul_rn(d, d));
      d = __fsub_rn(qv.w, tv[4 * k4 + 3]); acc[r] = __fadd_rn(acc[r], __fmul_rn(d, d));
    }
  }
  float* dp = dist + (size_t)pair * max_n * max_n;
#pragma unroll
  for (int r = 0; r < BF_ROWS; ++r)
    if (i0 + r < n_q) dp[(size_t)(i0 + r) * max_n + j] = __fsqrt_rn(acc[r]);
}

// one CTA per pair: forward / backward argmin (first minimum wins), mutual test, ordered compaction.
// ONE coalesced pass over the distance matrix with 32 warps: warp w owns rows w, w+32, ...; a lane holds columns lane,
// lane+32, ... of the row.  Row minimum = lane-local scan (ascending j, strict <) + shuffle reduction (ties -> smaller
// j).  Column minimum = min over 64-bit keys (distance bits : row) -- distances are >= +0, so their bit patterns order
// like the floats and a tie resolves to the smaller row: per-lane running key, then one shared-memory atomicMin per
// (warp, column).  Both reproduce "first minimum wins" of the sequential scan exactly.
constexpr int BF_MAXN = 256;                       // max_n <= 256 (one thread per query row in the compaction)
constexpr int BF_CC_THREADS = 1024;
__global__ void __launch_bounds__(BF_CC_THREADS)
bf_crosscheck_kernel(const float* __restrict__ dist, const int32_t* __restrict__ nq, const int32_t* __restrict__ nt,
                     int max_n, int out_stride, int group, size_t group_stride, int32_t* __restrict__ qi,
                     int32_t* __restrict__ ti, float* __restrict__ dout, int32_t* __restrict__ n_out,
                     int32_t* __restrict__ map_out) {
  __shared__ int fwd[BF_MAXN];
  __shared__ float fdist[BF_MAXN];
  __shared__ unsigned long long ckey[BF_MAXN];
  __shared__ int warp_cnt[8];
  const int pair = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  constexpr int NW = BF_CC_THREADS / 32, CPL = BF_MAXN / 32;
  const int n_q = nq[pair], n_t = nt[pair];
  const float* dp = dist + (size_t)pair * max_n * max_n;
  // pair = group * g + s writes its lists at g * group_stride + s * out_stride and its count at g * group_stride + s
  const size_t gbase = (size_t)(pair / group) * group_stride, obase = gbase + (size_t)(pair % group) * out_stride;
  if (tid < BF_MAXN) ckey[tid] = ~0ull;
  __syncthreads();
  unsigned long long cbest[CPL];
#pragma unroll
  for (int c = 0; c < CPL; ++c) cbest[c] = ~0ull;
#pragma unroll 2
  for (int i = warp; i < n_q; i += NW) {
    float v[CPL];
#pragma unroll
    for (int c = 0; c < CPL; ++c) {
      const int j = lane + 32 * c;
      v[c] = (j < n_t) ? dp[(size_t)i * max_n + j] : INFINITY;
    }
    float best = INFINITY;
    int bj = 0x7fffffff;
#pragma unroll
    for (int c = 0; c < CPL; ++c) {
      const int j = lane + 32 * c;
      if (j < n_t) {
        if (v[c] < best || bj == 0x7fffffff) { best = v[c]; bj = j; }
        const unsigned long long key = ((unsigned long long)__float_as_uint(v[c]) << 32) | (unsigned)i;
        cbest[c] = min(cbest[c], key);
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
      if (oj != 0x7fffffff && (bj == 0x7fffffff || ob < best || (ob == best && oj < bj))) { best = ob; bj = oj; }
    }
    if (lane == 0 && n_t > 0) { fwd[i] = bj; fdist[i] = best; }
  }
#pragma unroll
  for (int c = 0; c < CPL; ++c)
    if (cbest[c] != ~0ull) atomicMin(&ckey[lane + 32 * c], cbest[c]);
  __syncthreads();
  const bool keep = (tid < n_q) && (n_t > 0) && ((int)(unsigned)(ckey[fwd[tid]] & 0xffffffffull) == tid);
  const unsigned bal = __ballot_sync(0xffffffffu, keep);
  if (lane == 0 && warp < 8) warp_cnt[warp] = __popc(bal);
  __syncthreads();
  int base = 0, total = 0;
  for (int w = 0; w < 8; ++w) { if (w < warp) base += warp_cnt[w]; total += warp_cnt[w]; }
  if (keep) {
    const int pos = base + __popc(bal & ((1u << lane) - 1u));
    qi[obase + pos] = tid;
    ti[obase + pos] = fwd[tid];
    dout[obase + pos] = fdist[tid];
  }
  if (map_out != nullptr && tid < max_n) map_out[obase + tid] = keep ? fwd[tid] : -1;
  if (tid == 0) n_out[gbase + pair % group] = total;
}

osb_status db_rows_alloc(Resources& m, void** rows, size_t n, int storage) {
  if (storage == OSB_DB_STORAGE_FP16) {
    __half* p = nullptr;
    OSB_TRY(m.alloc(&p, n));
    *rows = p;
  } else {
    float* p = nullptr;
    OSB_TRY(m.alloc(&p, n));
    *rows = p;
  }
  return OSB_OK;
}

__global__ void db_rows_to_half_kernel(__half2* __restrict__ dst, const float4* __restrict__ src, size_t n4) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
    const float4 v = src[i];
    dst[2 * i] = __floats2half2_rn(v.x, v.y);
    dst[2 * i + 1] = __floats2half2_rn(v.z, v.w);
  }
}

osb_status db_rows_to_half(__half* dst, const float* src, size_t n, cudaStream_t st) {
  const size_t n4 = n / 4;
  if (n4 == 0) return OSB_OK;
  const int grid = (int)std::min<size_t>(cdiv64((int64_t)n4, 256), (size_t)8 * num_sms());
  OSB_LAUNCH(db_rows_to_half_kernel, grid, 256, 0, st, reinterpret_cast<__half2*>(dst),
             reinterpret_cast<const float4*>(src), n4);
  OSB_CHECK_LAUNCH();
  return OSB_OK;
}

osb_status bf_match_device(int n_pairs, int max_n, int out_stride, const float* const* q, const int32_t* nq,
                           const float* const* t,
                           const int32_t* nt, float* dist_scratch, int32_t* qi, int32_t* ti, float* dout,
                           int32_t* n_out, int32_t* map_out, cudaStream_t st, int group, size_t group_stride) {
  if (n_pairs <= 0) return OSB_OK;
  if (group <= 0) { group = n_pairs; group_stride = 0; }     // one group: pair p at p * out_stride, count at p
  dim3 g1(cdiv(max_n, BF_ROWS), n_pairs);
  OSB_LAUNCH(bf_dist_kernel, g1, 256, 0, st, q, nq, t, nt, max_n, dist_scratch);
  OSB_CHECK_LAUNCH();
  OSB_LAUNCH(bf_crosscheck_kernel, n_pairs, BF_CC_THREADS, 0, st, dist_scratch, nq, nt, max_n, out_stride, group,
             group_stride, qi, ti, dout, n_out, map_out);
  OSB_CHECK_LAUNCH();
  return OSB_OK;
}

}  // namespace osb

// =============================================================================================================
// C ABI: osb_db
// =============================================================================================================
using namespace osb;

struct osb_db {
  Resources res;
  int device = 0;
  int dim = 0;
  int64_t cap = 0, ntotal = 0;
  int storage = OSB_DB_STORAGE_FP32;
  void* rows = nullptr;             // [cap][dim] float, or __half in OSB_DB_STORAGE_FP16
  float* part_scores = nullptr;
  int64_t* part_ids = nullptr;
  unsigned int* done = nullptr;     // ticket counter of the fused merge
  float *d_q = nullptr, *d_scores = nullptr;
  int64_t* d_ids = nullptr;
  int kmax = 64, qmax = 64;
  int grid_max = 0;
  cudaStream_t stream = nullptr;
  std::mutex mu;
};

extern "C" osb_status osb_db_create_storage(osb_db** out, int dim, int64_t capacity, int storage) {
  OSB_REQUIRE(out != nullptr && dim > 0 && dim % 4 == 0 && dim <= 8192 && capacity > 0, "bad dim/capacity");
  OSB_REQUIRE(storage == OSB_DB_STORAGE_FP32 || storage == OSB_DB_STORAGE_FP16,
              "storage must be OSB_DB_STORAGE_FP32 or OSB_DB_STORAGE_FP16");
  OSB_TRY(require_device());
  std::unique_ptr<osb_db> h(new osb_db());
  h->device = current_device();
  h->dim = dim; h->cap = capacity; h->storage = storage;
  int64_t chunk;
  h->grid_max = db_scan_grid(capacity, &chunk);
  OSB_TRY(h->res.stream(&h->stream));
  OSB_TRY(db_rows_alloc(h->res, &h->rows, (size_t)capacity * dim, storage));
  OSB_TRY(h->res.alloc(&h->part_scores, (size_t)8 * h->grid_max * h->kmax));
  OSB_TRY(h->res.alloc(&h->part_ids, (size_t)8 * h->grid_max * h->kmax));
  OSB_TRY(h->res.alloc(&h->done, 1));
  OSB_CUDA(cudaMemset(h->done, 0, sizeof(unsigned int)));
  OSB_TRY(h->res.alloc(&h->d_q, (size_t)h->qmax * dim));
  OSB_TRY(h->res.alloc(&h->d_scores, (size_t)h->qmax * h->kmax));
  OSB_TRY(h->res.alloc(&h->d_ids, (size_t)h->qmax * h->kmax));
  *out = h.release();
  return OSB_OK;
}

extern "C" osb_status osb_db_create(osb_db** out, int dim, int64_t capacity) {
  return osb_db_create_storage(out, dim, capacity, OSB_DB_STORAGE_FP32);
}

extern "C" osb_status osb_db_destroy(osb_db* h) {
  delete h;
  return OSB_OK;
}

extern "C" int64_t osb_db_size(osb_db* h) { return h ? h->ntotal : -1; }

extern "C" osb_status osb_db_reset(osb_db* h) {
  OSB_REQUIRE(h != nullptr, "null handle");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  h->ntotal = 0;
  return OSB_OK;
}

static osb_status db_add_impl(osb_db* h, int64_t n, const float* x, int64_t* first_id, cudaMemcpyKind kind,
                              cudaStream_t st, bool sync) {
  OSB_REQUIRE(h != nullptr && n >= 0 && (x != nullptr || n == 0), "bad arguments");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  if (h->ntotal + n > h->cap) { set_error("osb_db_add", "capacity exceeded"); return OSB_ERR_CAPACITY; }
  const size_t off = (size_t)h->ntotal * h->dim;
  if (n > 0 && h->storage == OSB_DB_STORAGE_FP32) {
    OSB_CUDA(cudaMemcpyAsync(static_cast<float*>(h->rows) + off, x, (size_t)n * h->dim * sizeof(float), kind, st));
  } else if (n > 0 && kind == cudaMemcpyDeviceToDevice) {
    OSB_TRY(db_rows_to_half(static_cast<__half*>(h->rows) + off, x, (size_t)n * h->dim, st));
  } else if (n > 0) {
    // host rows: staged through the query buffer d_q, qmax rows at a time (stream order protects its reuse)
    for (int64_t r0 = 0; r0 < n; r0 += h->qmax) {
      const size_t e = (size_t)std::min<int64_t>(h->qmax, n - r0) * h->dim;
      OSB_CUDA(cudaMemcpyAsync(h->d_q, x + (size_t)r0 * h->dim, e * sizeof(float), kind, st));
      OSB_TRY(db_rows_to_half(static_cast<__half*>(h->rows) + off + (size_t)r0 * h->dim, h->d_q, e, st));
    }
  }
  if (first_id) *first_id = h->ntotal;
  h->ntotal += n;
  if (sync) OSB_CUDA(cudaStreamSynchronize(st));
  return OSB_OK;
}

extern "C" osb_status osb_db_add(osb_db* h, int64_t n, const float* x, int64_t* first_id) {
  OSB_REQUIRE(h != nullptr, "null handle");
  return db_add_impl(h, n, x, first_id, cudaMemcpyHostToDevice, h->stream, true);
}

extern "C" osb_status osb_db_add_dev(osb_db* h, int64_t n, const float* x_dev, int64_t* first_id, void* stream) {
  OSB_REQUIRE(h != nullptr, "null handle");
  return db_add_impl(h, n, x_dev, first_id, cudaMemcpyDeviceToDevice, (cudaStream_t)stream, false);
}

extern "C" osb_status osb_db_search_dev(osb_db* h, int64_t nq, const float* q_dev, int k, float* scores_dev,
                                        int64_t* ids_dev, void* stream) {
  OSB_REQUIRE(h != nullptr && q_dev && scores_dev && ids_dev, "null argument");
  OSB_REQUIRE(k > 0 && k <= h->kmax && nq > 0, "k must be in 1..64 and nq > 0");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  return db_search_device(h->rows, h->storage, h->ntotal, nullptr, h->dim, q_dev, (int)nq, k, h->part_scores, h->part_ids, h->done, scores_dev,
                          ids_dev, (cudaStream_t)stream);
}

// candidate lists of several database shards -> global top-k (same order rule as the scan: score descending, ties by
// ascending id).  Used by the row-sharded search (SURVEY.md section 8e): every rank scans its shard, the k candidates
// per query are all-gathered, and each rank merges world*k candidates.  id_offset[l] is added to the ids of list l
// (shard-local row -> global row); ids < 0 are padding.
__global__ void topk_fill_offset_kernel(float* __restrict__ out_scores, int64_t* __restrict__ out_ids, int n_out,
                                        int64_t* __restrict__ cand_ids, int64_t n_cand_total, int ncand, int list_len,
                                        const int64_t* __restrict__ id_offset) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_out) { out_scores[i] = -INFINITY; out_ids[i] = -1; }
  if (i < n_cand_total && id_offset) {
    const int64_t id = cand_ids[i];
    if (id >= 0) cand_ids[i] = id + id_offset[(i % ncand) / list_len];
  }
}

extern "C" osb_status osb_topk_merge_dev(int nq, int n_lists, int k, const float* cand_scores_dev, int64_t* cand_ids_dev,
                                         const int64_t* id_offset_dev, float* scores_dev, int64_t* ids_dev,
                                         void* stream) {
  OSB_REQUIRE(cand_scores_dev && cand_ids_dev && scores_dev && ids_dev, "null argument");
  OSB_REQUIRE(nq > 0 && n_lists > 0 && k > 0 && k <= 64, "bad nq / n_lists / k");
  osb_status s = require_device();
  if (s != OSB_OK) return s;
  cudaStream_t st = (cudaStream_t)stream;
  const int ncand = n_lists * k;
  const int64_t total = (int64_t)nq * ncand;
  OSB_LAUNCH(topk_fill_offset_kernel, (unsigned)cdiv64(total, 256), 256, 0, st, scores_dev, ids_dev, nq * k, cand_ids_dev,
             total, ncand, k, id_offset_dev);
  OSB_CHECK_LAUNCH();
  OSB_LAUNCH(db_merge_kernel, dim3(cdiv(ncand, 32), nq), 1024, 0, st, cand_scores_dev, cand_ids_dev, ncand, k,
             scores_dev, ids_dev);
  OSB_CHECK_LAUNCH();
  return OSB_OK;
}

extern "C" osb_status osb_db_search(osb_db* h, int64_t nq, const float* q, int k, float* scores, int64_t* ids) {
  OSB_REQUIRE(h != nullptr && q && scores && ids, "null argument");
  OSB_REQUIRE(k > 0 && k <= h->kmax && nq > 0, "k must be in 1..64 and nq > 0");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  for (int64_t q0 = 0; q0 < nq; q0 += h->qmax) {
    const int nb = (int)std::min<int64_t>(h->qmax, nq - q0);
    OSB_CUDA(cudaMemcpyAsync(h->d_q, q + (size_t)q0 * h->dim, (size_t)nb * h->dim * sizeof(float),
                             cudaMemcpyHostToDevice, h->stream));
    osb_status s = db_search_device(h->rows, h->storage, h->ntotal, nullptr, h->dim, h->d_q, nb, k, h->part_scores, h->part_ids, h->done,
                                    h->d_scores, h->d_ids, h->stream);
    if (s != OSB_OK) return s;
    OSB_CUDA(cudaMemcpyAsync(scores + (size_t)q0 * k, h->d_scores, (size_t)nb * k * sizeof(float),
                             cudaMemcpyDeviceToHost, h->stream));
    OSB_CUDA(cudaMemcpyAsync(ids + (size_t)q0 * k, h->d_ids, (size_t)nb * k * sizeof(int64_t),
                             cudaMemcpyDeviceToHost, h->stream));
    OSB_CUDA(cudaStreamSynchronize(h->stream));
  }
  return OSB_OK;
}

// =============================================================================================================
// C ABI: osb_matcher
// =============================================================================================================
struct osb_matcher {
  Resources res;
  int device = 0;
  int max_pairs = 0, max_n = 0, dim = 0;
  float *d_q = nullptr, *d_t = nullptr, *d_dist = nullptr, *d_dout = nullptr;
  int32_t *d_nq = nullptr, *d_nt = nullptr, *d_qi = nullptr, *d_ti = nullptr, *d_nout = nullptr;
  const float** d_ptrs = nullptr;   // [2][max_pairs] pointer tables (query, train)
  cudaStream_t stream = nullptr;
  std::mutex mu;
};

static osb_status matcher_tables(osb_matcher* h, int n_pairs, const float* q, const float* t, cudaStream_t st) {
  std::vector<const float*> tab(2 * (size_t)h->max_pairs, nullptr);
  for (int p = 0; p < n_pairs; ++p) {
    tab[p] = q + (size_t)p * h->max_n * h->dim;
    tab[h->max_pairs + p] = t + (size_t)p * h->max_n * h->dim;
  }
  OSB_CUDA(cudaMemcpyAsync(h->d_ptrs, tab.data(), tab.size() * sizeof(float*), cudaMemcpyHostToDevice, st));
  OSB_CUDA(cudaStreamSynchronize(st));   // `tab` is a stack-lifetime staging buffer
  return OSB_OK;
}

extern "C" osb_status osb_matcher_create(osb_matcher** out, int max_pairs, int max_n, int dim) {
  OSB_REQUIRE(out != nullptr && max_pairs > 0 && max_n > 0 && max_n <= 256 && dim == BF_DIM,
              "max_n must be <= 256 and dim == 64");
  OSB_TRY(require_device());
  std::unique_ptr<osb_matcher> h(new osb_matcher());
  h->device = current_device();
  h->max_pairs = max_pairs; h->max_n = max_n; h->dim = dim;
  const size_t pn = (size_t)max_pairs * max_n;
  OSB_TRY(h->res.stream(&h->stream));
  OSB_TRY(h->res.alloc(&h->d_q, pn * dim));
  OSB_TRY(h->res.alloc(&h->d_t, pn * dim));
  OSB_TRY(h->res.alloc(&h->d_dist, pn * max_n));
  OSB_TRY(h->res.alloc(&h->d_dout, pn));
  OSB_TRY(h->res.alloc(&h->d_qi, pn));
  OSB_TRY(h->res.alloc(&h->d_ti, pn));
  OSB_TRY(h->res.alloc(&h->d_nq, max_pairs));
  OSB_TRY(h->res.alloc(&h->d_nt, max_pairs));
  OSB_TRY(h->res.alloc(&h->d_nout, max_pairs));
  OSB_TRY(h->res.alloc(&h->d_ptrs, 2 * (size_t)max_pairs));
  *out = h.release();
  return OSB_OK;
}

extern "C" osb_status osb_matcher_destroy(osb_matcher* h) {
  delete h;
  return OSB_OK;
}

extern "C" osb_status osb_matcher_match_dev(osb_matcher* h, int n_pairs, const float* q_dev, const int32_t* nq_dev,
                                            const float* t_dev, const int32_t* nt_dev, int32_t* qi_dev,
                                            int32_t* ti_dev, float* dist_dev, int32_t* n_out_dev, void* stream) {
  OSB_REQUIRE(h != nullptr && n_pairs >= 0 && n_pairs <= h->max_pairs, "n_pairs out of range");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  osb_status s = matcher_tables(h, n_pairs, q_dev, t_dev, (cudaStream_t)stream);
  if (s != OSB_OK) return s;
  return bf_match_device(n_pairs, h->max_n, h->max_n, h->d_ptrs, nq_dev, h->d_ptrs + h->max_pairs, nt_dev, h->d_dist, qi_dev,
                         ti_dev, dist_dev, n_out_dev, nullptr, (cudaStream_t)stream);
}

extern "C" osb_status osb_matcher_match(osb_matcher* h, int n_pairs, const float* q, const int32_t* nq,
                                        const float* t, const int32_t* nt, int32_t* qi, int32_t* ti, float* dist,
                                        int32_t* n_out) {
  OSB_REQUIRE(h != nullptr && n_pairs >= 0 && n_pairs <= h->max_pairs, "n_pairs out of range");
  OSB_REQUIRE(q && nq && t && nt && qi && ti && dist && n_out, "null argument");
  for (int p = 0; p < n_pairs; ++p)
    OSB_REQUIRE(nq[p] >= 0 && nq[p] <= h->max_n && nt[p] >= 0 && nt[p] <= h->max_n, "row count out of range");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  const size_t pn = (size_t)n_pairs * h->max_n;
  cudaStream_t st = h->stream;
  OSB_CUDA(cudaMemcpyAsync(h->d_q, q, pn * h->dim * sizeof(float), cudaMemcpyHostToDevice, st));
  OSB_CUDA(cudaMemcpyAsync(h->d_t, t, pn * h->dim * sizeof(float), cudaMemcpyHostToDevice, st));
  OSB_CUDA(cudaMemcpyAsync(h->d_nq, nq, n_pairs * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  OSB_CUDA(cudaMemcpyAsync(h->d_nt, nt, n_pairs * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  osb_status s = matcher_tables(h, n_pairs, h->d_q, h->d_t, st);
  if (s != OSB_OK) return s;
  s = bf_match_device(n_pairs, h->max_n, h->max_n, h->d_ptrs, h->d_nq, h->d_ptrs + h->max_pairs, h->d_nt, h->d_dist, h->d_qi,
                      h->d_ti, h->d_dout, h->d_nout, nullptr, st);
  if (s != OSB_OK) return s;
  OSB_CUDA(cudaMemcpyAsync(qi, h->d_qi, pn * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  OSB_CUDA(cudaMemcpyAsync(ti, h->d_ti, pn * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  OSB_CUDA(cudaMemcpyAsync(dist, h->d_dout, pn * sizeof(float), cudaMemcpyDeviceToHost, st));
  OSB_CUDA(cudaMemcpyAsync(n_out, h->d_nout, n_pairs * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  OSB_CUDA(cudaStreamSynchronize(st));
  return OSB_OK;
}
