// postproc.cu -- SuperPoint head epilogues and the keypoint / descriptor post-processing that the reference runs
// on the CPU after every engine call (swarm_loop/src/superpoint_tensorrt.cpp:164-310):
//   getKeyPoints (threshold + findNonZero)  :164-189
//   NMS2 (order-dependent greedy 9x9 suppression, sort by confidence, top max_num)  :237-310
//   computeDescriptors (grid_sampler bilinear, per-channel norm over keypoints, PCA)  :192-230
// All integer outputs (candidate set, survivors, keypoint order) are bit-exact restatements; see SURVEY.md A.2/A.3.
#include "common.cuh"
#include "kernels.cuh"

namespace osb {

// -------------------------------------------------------------------------------------------------------------
// detector head epilogue: softmax over 65 logits per cell, drop the dustbin, 8x8 pixel shuffle
// (superpoint.ipynb:190-198).  One thread per cell.
// -------------------------------------------------------------------------------------------------------------
__global__ void sp_softmax_shuffle_kernel(const float* __restrict__ logits, int cstride, float* __restrict__ semi,
                                          int Hc, int Wc, int64_t cells) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= cells) return;
  const int cx = (int)(i % Wc);
  const int cy = (int)((i / Wc) % Hc);
  const int b = (int)(i / ((int64_t)Wc * Hc));
  const float* l = logits + (size_t)i * cstride;
  float v[65];
  float m = -INFINITY;
#pragma unroll
  for (int c = 0; c < 65; ++c) { v[c] = l[c]; m = fmaxf(m, v[c]); }
  float s = 0.f;
#pragma unroll
  for (int c = 0; c < 65; ++c) { v[c] = expf(v[c] - m); s += v[c]; }
  const int W = Wc * 8;
  float* out = semi + ((size_t)b * Hc * 8 + cy * 8) * W + cx * 8;
#pragma unroll
  for (int r = 0; r < 8; ++r) {
    float4 a = make_float4(v[r * 8 + 0] / s, v[r * 8 + 1] / s, v[r * 8 + 2] / s, v[r * 8 + 3] / s);
    float4 c = make_float4(v[r * 8 + 4] / s, v[r * 8 + 5] / s, v[r * 8 + 6] / s, v[r * 8 + 7] / s);
    reinterpret_cast<float4*>(out + (size_t)r * W)[0] = a;
    reinterpret_cast<float4*>(out + (size_t)r * W)[1] = c;
  }
}

osb_status sp_softmax_shuffle(const float* logits, int cstride, float* semi, int B, int Hc, int Wc, cudaStream_t st) {
  const int64_t cells = (int64_t)B * Hc * Wc;
  OSB_LAUNCH(sp_softmax_shuffle_kernel, (unsigned)cdiv64(cells, 128), 128, 0, st, logits, cstride, semi, Hc, Wc, cells);
  OSB_CHECK_LAUNCH();
  return OSB_OK;
}

// ||p||_2 over C channels, by one warp (every lane gets it); the sparse descriptor head divides by the same value
__device__ __forceinline__ float cell_norm(const float* p, int C, int lane) {
  float s = 0.f;
  for (int c = lane; c < C; c += 32) { const float v = p[c]; s = fmaf(v, v, s); }
  s = warp_sum(s);
  return sqrtf(s);
}

// descriptor head epilogue: desc /= ||desc||_2 over channels (superpoint.ipynb:187-188); one warp per cell
__global__ void l2norm_cells_kernel(float* __restrict__ x, int64_t cells, int C) {
  const int64_t cell = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (cell >= cells) return;
  float* p = x + (size_t)cell * C;
  const float n = cell_norm(p, C, lane);
  for (int c = lane; c < C; c += 32) p[c] = p[c] / n;
}

osb_status l2norm_cells(float* x, int64_t cells, int C, cudaStream_t st) {
  OSB_LAUNCH(l2norm_cells_kernel, (unsigned)cdiv64(cells * 32, 256), 256, 0, st, x, cells, C);
  OSB_CHECK_LAUNCH();
  return OSB_OK;
}

// -------------------------------------------------------------------------------------------------------------
// Keypoint extraction: ONE CTA PER IMAGE (the batch gives the parallelism; each stage is latency bound).
//
//  phase 1  ordered compaction of {L : prob[L] > thres} (raster order = cv::findNonZero order) into cand[],
//           state plane: 0 not a candidate, 1 undecided, 2 active, 3 suppressed.
//  phase 2  NMS2's raster-order greedy loop resolved by dependency: candidate p is ACTIVE iff no earlier-visited
//           ACTIVE candidate in its 9x9 flat-address window has strictly larger confidence.  A candidate can be
//           decided as soon as all earlier, stronger neighbours are decided; iterate to the fixpoint (the
//           earliest undecided candidate is always decidable, so every round makes progress).
//  phase 3  survivor = ACTIVE and no later-visited ACTIVE neighbour with strictly larger confidence
//           (that neighbour would have overwritten its grid value 2 with 0, superpoint_tensorrt.cpp:278-280).
//  phase 4  sort survivors by (confidence desc, raster index asc) -- the oracle's defined tie rule for the
//           reference's unstable std::sort -- and emit the first max_num.  Keys are (~conf_bits << 32 | L).
//  The flat-address window reproduces cv::Mat::at's unchecked column wrap; addresses outside the plane are
//  skipped.  The u16 index plane (inds, :246,:260) is reproduced: survivor coordinates are those of candidate
//  (rank & 0xFFFF).
// -------------------------------------------------------------------------------------------------------------
constexpr int KP_THREADS = 1024;
constexpr int KP_SORT_CAP = 8192;  // survivors sortable in shared memory (64 KB of keys)
constexpr int KP_RANK_CAP = 128;   // tiny survivor sets: rank counting (no barriers); otherwise bitonic sort in smem

// 9 consecutive state bytes starting at flat address `start` (may be negative / beyond the plane: those read as 0,
// "not a candidate") through two aligned 64-bit L2 loads
__device__ __forceinline__ void load_state9(const uint8_t* __restrict__ state, int start, int HW, uint8_t (&out)[9]) {
  const int a0 = (start >> 3) << 3;                      // floor to a multiple of 8 (arithmetic shift: works below 0)
  const unsigned long long lo = (a0 >= 0 && a0 + 8 <= HW) ? __ldcg(reinterpret_cast<const unsigned long long*>(state + a0)) : 0ull;
  const unsigned long long hi = (a0 + 8 >= 0 && a0 + 16 <= HW) ? __ldcg(reinterpret_cast<const unsigned long long*>(state + a0 + 8)) : 0ull;
  const int sh = start - a0;
#pragma unroll
  for (int i = 0; i < 9; ++i) {
    const int bpos = i + sh;
    out[i] = (uint8_t)((bpos < 8 ? (lo >> (8 * bpos)) : (hi >> (8 * (bpos - 8)))) & 0xff);
  }
}

// the same 9-byte window kept packed: bytes 0..7 in `w`, byte 8 in `b8` (no per-byte arrays -> no local memory)
__device__ __forceinline__ void load_state9p(const uint8_t* __restrict__ state, int start, int HW, unsigned long long& w,
                                             unsigned& b8) {
  const int a0 = (start >> 3) << 3;
  const unsigned long long lo = (a0 >= 0 && a0 + 8 <= HW) ? __ldcg(reinterpret_cast<const unsigned long long*>(state + a0)) : 0ull;
  const unsigned long long hi = (a0 + 8 >= 0 && a0 + 16 <= HW) ? __ldcg(reinterpret_cast<const unsigned long long*>(state + a0 + 8)) : 0ull;
  const int sh = 8 * (start - a0);
  w = sh ? ((lo >> sh) | (hi << (64 - sh))) : lo;
  b8 = (unsigned)((hi >> sh) & 0xffull);
}
// 9-bit mask of the window positions whose state byte equals `val`
__device__ __forceinline__ unsigned window_eq(unsigned long long w, unsigned b8, unsigned val) {
  unsigned m = 0;
#pragma unroll
  for (int j = 0; j < 8; ++j) m |= (unsigned)(((w >> (8 * j)) & 0xffull) == val) << j;
  m |= (unsigned)(b8 == val) << 8;
  return m;
}

__device__ __forceinline__ int block_exclusive_scan(int v, int* warp_sums, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int n = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += n;
  }
  if (lane == 31) warp_sums[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    int w = (lane < KP_THREADS / 32) ? warp_sums[lane] : 0;
    int winc = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int n = __shfl_up_sync(0xffffffffu, winc, o);
      if (lane >= o) winc += n;
    }
    warp_sums[lane] = winc - w;  // exclusive
    if (lane == 31) *total = winc;
  }
  __syncthreads();
  const int r = warp_sums[warp] + inc - v;
  __syncthreads();
  return r;
}

__global__ void __launch_bounds__(KP_THREADS)
sp_keypoints_kernel(const float* __restrict__ semi, int H, int W, float thres, int max_num, uint8_t* __restrict__ state_,
                    uint8_t* __restrict__ surv_, int32_t* __restrict__ cand_, unsigned long long* __restrict__ skey_,
                    unsigned long long* __restrict__ cmask_, int write_surv, int32_t* __restrict__ counts, int32_t* __restrict__ n_kpts, float* __restrict__ kpts,
                    float* __restrict__ conf) {
  extern __shared__ __align__(16) unsigned long long skeys[];  // KP_SORT_CAP keys
  __shared__ int warp_sums[32];
  __shared__ int s_total, s_undecided, s_nsurv;
  const int b = blockIdx.x, tid = threadIdx.x;
  const int HW = H * W;
  const float* prob = semi + (size_t)b * HW;
  uint8_t* state = state_ + (size_t)b * HW;
  uint8_t* surv = surv_ + (size_t)b * HW;
  int32_t* cand = cand_ + (size_t)b * HW;
  unsigned long long* skey = skey_ + (size_t)b * HW;
  unsigned long long* cmask = cmask_ + (size_t)b * 2 * HW;

  const long long t_start = clock64();
  // ---- phase 1: ordered compaction.  Warp w owns the contiguous pixel range [w*seg, (w+1)*seg): pass A counts its
  // candidates, one block scan turns the 32 warp totals into offsets, pass B rescans and writes cand[] in raster
  // order with a shuffle scan per 128-pixel row of lanes (no block barrier inside the loops).
  const int lane = tid & 31, warp = tid >> 5;
  const int seg = ((HW / 4 + 31) / 32) * 4;          // pixels per warp, multiple of 4
  const int wp0 = warp * seg, wp1 = min(HW, wp0 + seg);
  int wcount = 0;
  for (int q0 = wp0; q0 < wp1; q0 += 8 * 128) {           // 8 guarded, independent 16-byte loads in flight per lane
    float4 vv[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int p = q0 + u * 128 + lane * 4;
      vv[u] = (p < wp1) ? *reinterpret_cast<const float4*>(prob + p) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int u = 0; u < 8; ++u)
      wcount += (vv[u].x > thres) + (vv[u].y > thres) + (vv[u].z > thres) + (vv[u].w > thres);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) wcount += __shfl_xor_sync(0xffffffffu, wcount, o);
  const int wbase = block_exclusive_scan(lane == 0 ? wcount : 0, warp_sums, &s_total);
  // (only lane 0 contributed, so the exclusive prefix seen by lane 0 of warp w is the sum of earlier warps)
  int base = __shfl_sync(0xffffffffu, wbase, 0);
  const int M = s_total;
  for (int q0 = wp0; q0 < wp1; q0 += 4 * 128) {           // batches of 4 rows of 128 pixels: loads first, scans after
    float4 vv[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int p = q0 + u * 128 + lane * 4;
      vv[u] = (p < wp1) ? *reinterpret_cast<const float4*>(prob + p) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int p = q0 + u * 128 + lane * 4;
      const float4 v = vv[u];
      const int f0 = (p < wp1) && (v.x > thres), f1 = (p < wp1) && (v.y > thres);
      const int f2 = (p < wp1) && (v.z > thres), f3 = (p < wp1) && (v.w > thres);
      const int cnt = f0 + f1 + f2 + f3;
      int inc = cnt;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int n = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += n;
      }
      if (p < wp1) {
        int o = base + inc - cnt;
        if (f0) cand[o++] = p;
        if (f1) cand[o++] = p + 1;
        if (f2) cand[o++] = p + 2;
        if (f3) cand[o++] = p + 3;
        *reinterpret_cast<uchar4*>(state + p) = make_uchar4(f0, f1, f2, f3);
        if (write_surv) *reinterpret_cast<uchar4*>(surv + p) = make_uchar4(0, 0, 0, 0);
      }
      base += __shfl_sync(0xffffffffu, inc, 31);
    }
  }
  __syncthreads();

  const long long t_p1 = clock64();
  // ---- phase 2a: per candidate, WHICH of the 40 earlier-visited / 40 later-visited window positions hold a candidate
  // with strictly larger confidence (bit q = row*9 + col of the 5x9 window).  Confidences are compared once, here;
  // the fixpoint rounds below then only look at state bytes.
  for (int i = tid; i < M; i += KP_THREADS) {
    const int L = cand[i];
    const float c = prob[L];
    unsigned long long we[5], wl[5];
    unsigned be[5], bl[5];
#pragma unroll
    for (int k = 0; k < 5; ++k) {
      load_state9p(state, L + (k - 4) * W - 4, HW, we[k], be[k]);
      load_state9p(state, L + k * W - 4, HW, wl[k], bl[k]);
    }
    unsigned long long me = 0ull, ml = 0ull;
#pragma unroll
    for (int k = 0; k < 5; ++k) {
      // candidate positions (state != 0) of the row, restricted to the earlier / later half of the window
      unsigned ce = 0x1ffu & ~window_eq(we[k], be[k], 0u), cl = 0x1ffu & ~window_eq(wl[k], bl[k], 0u);
      if (k == 4) ce &= 0x00fu;                       // row of L itself: only the 4 pixels to the left are earlier
      if (k == 0) cl &= 0x1e0u;                       // ... and only the 4 pixels to the right are later
      while (ce) { const int j = __ffs(ce) - 1; ce &= ce - 1; if (prob[L + (k - 4) * W + (j - 4)] > c) me |= 1ull << (k * 9 + j); }
      while (cl) { const int j = __ffs(cl) - 1; cl &= cl - 1; if (prob[L + k * W + (j - 4)] > c) ml |= 1ull << (k * 9 + j); }
    }
    cmask[i] = me;
    cmask[HW + i] = ml;
  }
  __syncthreads();
  // ---- phase 2: resolve ACTIVE by dependency order ----
  int rounds = 0;
  while (true) {
    if (tid == 0) s_undecided = 0;
    __syncthreads();
    int local_undecided = 0;
    for (int i = tid; i < M; i += KP_THREADS) {
      const int L = cand[i];
      if (__ldcg(state + L) != 1) continue;
      const unsigned long long me = cmask[i];
      unsigned long long act = 0ull, und = 0ull;             // positions whose candidate is ACTIVE / still undecided
#pragma unroll
      for (int k = 0; k < 5; ++k) {
        unsigned long long w; unsigned b8;
        load_state9p(state, L + (k - 4) * W - 4, HW, w, b8);
        act |= (unsigned long long)window_eq(w, b8, 2u) << (k * 9);
        und |= (unsigned long long)window_eq(w, b8, 1u) << (k * 9);
      }
      if (me & act) __stcg(state + L, (uint8_t)3);           // an earlier, stronger, active neighbour zeroed it
      else if (!(me & und)) __stcg(state + L, (uint8_t)2);   // every earlier stronger neighbour is decided inactive
      else local_undecided = 1;
    }
    if (local_undecided) atomicOr(&s_undecided, 1);
    __syncthreads();
    ++rounds;
    const int u = s_undecided;
    __syncthreads();
    if (!u) break;
  }

  const long long t_p2 = clock64();
  // ---- phase 3: survivors ----
  if (tid == 0) s_nsurv = 0;
  __syncthreads();
  for (int i = tid; i < M; i += KP_THREADS) {
    const int L = cand[i];
    if (__ldcg(state + L) != 2) continue;
    const unsigned long long ml = cmask[HW + i];
    unsigned long long act = 0ull;
#pragma unroll
    for (int k = 0; k < 5; ++k) {
      unsigned long long w; unsigned b8;
      load_state9p(state, L + k * W - 4, HW, w, b8);
      act |= (unsigned long long)window_eq(w, b8, 2u) << (k * 9);
    }
    if (!(ml & act)) {                                       // no later, stronger, active neighbour overwrote its 2
      if (write_surv) surv[L] = 1;
      const int pos = atomicAdd(&s_nsurv, 1);
      skey[pos] = ((unsigned long long)(~__float_as_uint(prob[L])) << 32) | (unsigned)L;
    }
  }
  __syncthreads();
  const int S = s_nsurv;
  const int n_out = min(S, max_num);

  const long long t_p3 = clock64();
  // ---- phase 4: order by (conf desc, raster asc), keep the first max_num ----
  if (S <= KP_RANK_CAP) {
    // rank counting over the keys in shared memory: the key's rank IS its output slot (keys are unique)
    for (int i = tid; i < S; i += KP_THREADS) skeys[KP_RANK_CAP + i] = skey[i];
    __syncthreads();
    for (int i = tid; i < S; i += KP_THREADS) {
      const unsigned long long ki = skeys[KP_RANK_CAP + i];
      int rank = 0;
      for (int j = 0; j < S; ++j) rank += skeys[KP_RANK_CAP + j] < ki;
      if (rank < n_out) skeys[rank] = ki;
    }
    __syncthreads();
  } else if (S <= KP_SORT_CAP) {
    int n2 = 32;
    while (n2 < S) n2 <<= 1;
    for (int i = tid; i < n2; i += KP_THREADS) skeys[i] = (i < S) ? skey[i] : ~0ull;
    __syncthreads();
    for (int size = 2; size <= n2; size <<= 1) {
      for (int stride = size >> 1; stride > 0; stride >>= 1) {
        for (int i = tid; i < (n2 >> 1); i += KP_THREADS) {
          const int lo = 2 * i - (i & (stride - 1));
          const int hi = lo + stride;
          const bool up = ((lo & size) == 0);
          const unsigned long long a = skeys[lo], c2 = skeys[hi];
          if ((a > c2) == up) { skeys[lo] = c2; skeys[hi] = a; }
        }
        __syncthreads();
      }
    }
  } else {
    // rare path (more than KP_SORT_CAP survivors, e.g. large plateaus of equal confidence): max_num rounds of
    // block-wide minimum over the keys in global memory.
    __shared__ unsigned long long s_best[32];
    for (int r = 0; r < n_out; ++r) {
      unsigned long long best = ~0ull;
      for (int i = tid; i < S; i += KP_THREADS) best = min(best, skey[i]);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) best = min(best, __shfl_xor_sync(0xffffffffu, best, o));
      if ((tid & 31) == 0) s_best[tid >> 5] = best;
      __syncthreads();
      if (tid < 32) {
        best = s_best[tid];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) best = min(best, __shfl_xor_sync(0xffffffffu, best, o));
        if (tid == 0) { s_best[0] = best; skeys[r] = best; }
      }
      __syncthreads();
      best = s_best[0];
      for (int i = tid; i < S; i += KP_THREADS)
        if (skey[i] == best) skey[i] = ~0ull;   // keys are unique (L is unique)
      __syncthreads();
    }
  }
  for (int i = tid; i < n_out; i += KP_THREADS) {
    const unsigned long long key = skeys[i];
    int L = (int)(key & 0xffffffffull);
    const float c = __uint_as_float(~(unsigned)(key >> 32));
    if (M > 65536) {
      // inds plane is CV_16UC1 (superpoint_tensorrt.cpp:246,260): the stored candidate index wraps
      int lo = 0, hi = M - 1;
      while (lo < hi) { const int mid = (lo + hi) >> 1; if (cand[mid] < L) lo = mid + 1; else hi = mid; }
      L = cand[lo & 0xFFFF];
    }
    kpts[((size_t)b * max_num + i) * 2 + 0] = (float)(L % W);
    kpts[((size_t)b * max_num + i) * 2 + 1] = (float)(L / W);
    conf[(size_t)b * max_num + i] = c;
  }
  if (tid == 0) {
    n_kpts[b] = n_out;
    const long long t_end = clock64();
    counts[b * 8 + 0] = M; counts[b * 8 + 1] = S; counts[b * 8 + 2] = rounds; counts[b * 8 + 3] = 0;
    counts[b * 8 + 4] = (int)(t_p1 - t_start); counts[b * 8 + 5] = (int)(t_p2 - t_p1);   // SM cycles per phase
    counts[b * 8 + 6] = (int)(t_p3 - t_p2); counts[b * 8 + 7] = (int)(t_end - t_p3);
  }
}

osb_status sp_keypoints(const float* semi, int B, int H, int W, float thres, int max_num, KeypointScratch& ks,
                        int32_t* n_kpts, float* kpts, float* conf, cudaStream_t st) {
  OSB_REQUIRE((H * W) % 8 == 0, "H*W must be a multiple of 8");
  const size_t smem = (size_t)KP_SORT_CAP * sizeof(unsigned long long);
  OSB_SMEM_OPT_IN(sp_keypoints_kernel, smem);
  OSB_LAUNCH(sp_keypoints_kernel, B, KP_THREADS, smem, st, semi, H, W, thres, max_num, ks.state, ks.surv, ks.cand,
             ks.skey, ks.cmask, ks.write_surv ? 1 : 0, ks.counts, n_kpts, kpts, conf);
  OSB_CHECK_LAUNCH();
  return OSB_OK;
}

// -------------------------------------------------------------------------------------------------------------
// Descriptors (superpoint_tensorrt.cpp:192-230).  desc is NHWC [Hc][Wc][256] (already channel-normalised).
// bilinear tap arithmetic follows ATen's grid_sampler_2d (align_corners=false, zeros padding) in f32.
// -------------------------------------------------------------------------------------------------------------
struct Taps { int x0, y0; float nw, ne, sw, se; };

__device__ __forceinline__ Taps bilinear_taps(float kx, float ky, int W, int H, int Wc, int Hc) {
  // grid = 2*x/W - 1 (superpoint_tensorrt.cpp:204-205), then unnormalise: ((g + 1) * size - 1) / 2
  const float gx = __fsub_rn(__fdiv_rn(__fmul_rn(2.0f, kx), (float)W), 1.0f);
  const float gy = __fsub_rn(__fdiv_rn(__fmul_rn(2.0f, ky), (float)H), 1.0f);
  const float ix = __fdiv_rn(__fsub_rn(__fmul_rn(__fadd_rn(gx, 1.0f), (float)Wc), 1.0f), 2.0f);
  const float iy = __fdiv_rn(__fsub_rn(__fmul_rn(__fadd_rn(gy, 1.0f), (float)Hc), 1.0f), 2.0f);
  const float fx = floorf(ix), fy = floorf(iy);
  Taps t;
  t.x0 = (int)fx; t.y0 = (int)fy;
  const float ex = __fadd_rn(fx, 1.0f), ey = __fadd_rn(fy, 1.0f);
  t.nw = __fmul_rn(__fsub_rn(ex, ix), __fsub_rn(ey, iy));
  t.ne = __fmul_rn(__fsub_rn(ix, fx), __fsub_rn(ey, iy));
  t.sw = __fmul_rn(__fsub_rn(ex, ix), __fsub_rn(iy, fy));
  t.se = __fmul_rn(__fsub_rn(ix, fx), __fsub_rn(iy, fy));
  return t;
}

// SLOT: d holds convDb's output at the listed cells only, row slot[y][x] for cell (y, x) of the image (sp_cell_gather), not
// yet normalised: the value is d / nrm[row - row0], what l2norm_cells stores.  Else d is the image's normalised dense
// [Hc][Wc][256] map.
template <bool SLOT = false>
__device__ __forceinline__ float sample_channel(const float* __restrict__ d, const int32_t* __restrict__ slot,
                                                const float* nrm, int row0, const Taps& t, int Wc, int Hc, int ch) {
  auto at = [&](int y, int x) {
    if constexpr (SLOT) {
      const int row = slot[y * Wc + x];
      return d[(size_t)row * 256 + ch] / nrm[row - row0];
    } else {
      return d[((size_t)y * Wc + x) * 256 + ch];
    }
  };
  float r = 0.f;
  const bool x0 = t.x0 >= 0 && t.x0 < Wc, x1 = t.x0 + 1 >= 0 && t.x0 + 1 < Wc;
  const bool y0 = t.y0 >= 0 && t.y0 < Hc, y1 = t.y0 + 1 >= 0 && t.y0 + 1 < Hc;
  if (y0 && x0) r = __fadd_rn(r, __fmul_rn(at(t.y0, t.x0), t.nw));
  if (y0 && x1) r = __fadd_rn(r, __fmul_rn(at(t.y0, t.x0 + 1), t.ne));
  if (y1 && x0) r = __fadd_rn(r, __fmul_rn(at(t.y0 + 1, t.x0), t.sw));
  if (y1 && x1) r = __fadd_rn(r, __fmul_rn(at(t.y0 + 1, t.x0 + 1), t.se));
  return r;
}

// -------------------------------------------------------------------------------------------------------------
// Sparse descriptor head: the cells the selected keypoints sample, and their convDa input as a 1x1 layer's
// -------------------------------------------------------------------------------------------------------------
// Grid (image, CL_SPLIT).  Every CTA marks the in-range taps of the image's keypoints (sample_channel's conditions) and
// numbers them row-major in shared memory: rank r of the image is row b * seg + r, and the image's rows past its cells are
// padding (-1).  CTA 0 of the image writes slot [b][Hc][Wc] (-1 for an unsampled cell).  Then each CTA gathers its share of
// the image's rows: convDa's input at the cell as the input of a 1x1 layer of 9 x 128 channels, channel slab
// (kx * 2 + s) * 3 + ky holding channels 64 s .. 64 s + 63 of the cell's (ky, kx) neighbour in x ([B][Hc][Wc][128] split
// planes), zero outside the image or for a padding row.  That slab order is conv_stream_t_kernel's K order (kx, slab, ky)
// of the 3x3 layer.  Work unit = (row, tap, 16-byte chunk of the 128 channels).
constexpr int CL_THREADS = KP_THREADS;             // block_exclusive_scan's block
constexpr int CL_SPLIT = 16;
template <bool FP16>
__global__ void __launch_bounds__(CL_THREADS)
sp_cell_gather_kernel(int H, int W, const int32_t* __restrict__ n_kpts, const float* __restrict__ kpts, int max_num, int seg,
                      int32_t* __restrict__ slot, const __half* __restrict__ x_hi, const __half* __restrict__ x_lo,
                      __half* __restrict__ col_hi, __half* __restrict__ col_lo) {
  extern __shared__ int32_t list[];                    // [seg], then the marks [Hc * Wc] as bytes
  __shared__ int wsum[32], total;
  const int b = blockIdx.x, tid = threadIdx.x, Hc = H / 8, Wc = W / 8, cells = Hc * Wc;
  uint8_t* mark = reinterpret_cast<uint8_t*>(list + seg);
  for (int c = tid; c < cells; c += CL_THREADS) mark[c] = 0;
  __syncthreads();
  const int N = n_kpts[b];
  for (int n = tid; n < N; n += CL_THREADS) {
    const Taps t = bilinear_taps(kpts[((size_t)b * max_num + n) * 2], kpts[((size_t)b * max_num + n) * 2 + 1], W, H, Wc, Hc);
    for (int dy = 0; dy < 2; ++dy)
      for (int dx = 0; dx < 2; ++dx) {
        const int y = t.y0 + dy, x = t.x0 + dx;
        if (y >= 0 && y < Hc && x >= 0 && x < Wc) mark[y * Wc + x] = 1;
      }
  }
  __syncthreads();
  // each thread numbers a contiguous run of cells: its count, a block-wide exclusive scan, then the run
  const int per = (cells + CL_THREADS - 1) / CL_THREADS, c0 = tid * per, c1 = min(c0 + per, cells);
  int cnt = 0;
  for (int c = c0; c < c1; ++c) cnt += mark[c];
  int rank = block_exclusive_scan(cnt, wsum, &total);
  const bool writer = blockIdx.y == 0;
  for (int c = c0; c < c1; ++c) {
    if (mark[c]) {
      if (writer) slot[(size_t)b * cells + c] = b * seg + rank;
      list[rank++] = c;
    } else if (writer) {
      slot[(size_t)b * cells + c] = -1;
    }
  }
  for (int r = total + tid; r < seg; r += CL_THREADS) list[r] = -1;
  __syncthreads();
  for (int e = blockIdx.y * CL_THREADS + tid; e < seg * 144; e += CL_SPLIT * CL_THREADS) {
    const int i = e / 144, r = e % 144, tap = r / 16, j = r % 16, ky = tap / 3, kx = tap % 3, s = j / 8;
    const int c = list[i];
    uint4 h = make_uint4(0, 0, 0, 0), l = h;
    if (c >= 0) {
      const int y = c / Wc + ky - 1, xx = c % Wc + kx - 1;
      if (y >= 0 && y < Hc && xx >= 0 && xx < Wc) {
        const size_t src = (((size_t)b * Hc + y) * Wc + xx) * 128 + j * 8;
        h = *reinterpret_cast<const uint4*>(x_hi + src);
        if constexpr (!FP16) l = *reinterpret_cast<const uint4*>(x_lo + src);
      }
    }
    const size_t dst = ((size_t)b * seg + i) * 1152 + ((kx * 2 + s) * 3 + ky) * 64 + (j % 8) * 8;
    *reinterpret_cast<uint4*>(col_hi + dst) = h;
    if constexpr (!FP16) *reinterpret_cast<uint4*>(col_lo + dst) = l;
  }
}

osb_status sp_cell_gather(int B, int H, int W, const int32_t* n_kpts, const float* kpts, int max_num, int seg, int32_t* slot,
                          const __half* x_hi, const __half* x_lo, __half* col_hi, __half* col_lo, bool fp16,
                          cudaStream_t st) {
  const int smem = seg * 4 + (H / 8) * (W / 8);
  OSB_REQUIRE(smem <= 48 * 1024, "sparse descriptor head: too many cells per image");
  const dim3 grid(B, CL_SPLIT);
  if (fp16)
    OSB_LAUNCH(sp_cell_gather_kernel<true>, grid, CL_THREADS, smem, st, H, W, n_kpts, kpts, max_num, seg, slot, x_hi, x_lo,
               col_hi, col_lo);
  else
    OSB_LAUNCH(sp_cell_gather_kernel<false>, grid, CL_THREADS, smem, st, H, W, n_kpts, kpts, max_num, seg, slot, x_hi, x_lo,
               col_hi, col_lo);
  OSB_CHECK_LAUNCH();
  return OSB_OK;
}

// per-channel L2 norm over the keypoints of an image (torch::norm(desc, 2, 1) on [256,N], :214).
// The kernel is a chain of dependent L2 round trips (keypoint -> 4 taps), so it is spread wide: CTA = (image, 64-channel
// slab), 1024 threads = 16 keypoint groups x 64 channels; group g sums keypoints g, g+16, ... (two in flight per
// iteration) and the 16 partial sums are combined in a fixed order.
// SLOT (here and in sp_desc_pca_kernel): desc holds the listed cells only, found through slot [B][Hc][Wc] (sample_channel)
constexpr int DN_GROUPS = 16, DN_CH = 64;
template <bool SLOT = false>
__global__ void __launch_bounds__(DN_GROUPS * DN_CH)
sp_desc_norm_kernel(const float* __restrict__ desc, const int32_t* __restrict__ slot, int seg, float* __restrict__ cell_n,
                    int H, int W, const int32_t* __restrict__ n_kpts, const float* __restrict__ kpts, int max_num,
                    float* __restrict__ cnorm) {
  __shared__ float part[DN_GROUPS][DN_CH];
  extern __shared__ float nrm[];                       // SLOT: [seg] the norms of the image's rows
  const int b = blockIdx.x, c = threadIdx.x % DN_CH, g = threadIdx.x / DN_CH;
  const int ch = blockIdx.y * DN_CH + c;
  const int Hc = H / 8, Wc = W / 8;
  const float* d = SLOT ? desc : desc + (size_t)b * Hc * Wc * 256;
  const int32_t* sl = SLOT ? slot + (size_t)b * Hc * Wc : nullptr;
  if constexpr (SLOT) {
    // every row's L2 norm, one warp per row as l2norm_cells; the image's first CTA also keeps them for sp_desc_pca_kernel
    const int lane = threadIdx.x & 31;
    for (int r = threadIdx.x >> 5; r < seg; r += DN_GROUPS * DN_CH / 32) {
      const float n = cell_norm(desc + ((size_t)b * seg + r) * 256, 256, lane);
      if (lane == 0) {
        nrm[r] = n;
        if (blockIdx.y == 0) cell_n[(size_t)b * seg + r] = n;
      }
    }
    __syncthreads();
  }
  const float* kp = kpts + (size_t)b * max_num * 2;
  const int N = n_kpts[b];
  float s = 0.f;
  for (int n = g; n < N; n += 2 * DN_GROUPS) {
    const int n2 = n + DN_GROUPS;
    const Taps t0 = bilinear_taps(kp[2 * n], kp[2 * n + 1], W, H, Wc, Hc);
    const Taps t1 = bilinear_taps(kp[2 * min(n2, N - 1)], kp[2 * min(n2, N - 1) + 1], W, H, Wc, Hc);
    const float v0 = sample_channel<SLOT>(d, sl, nrm, b * seg, t0, Wc, Hc, ch);
    const float v1 = sample_channel<SLOT>(d, sl, nrm, b * seg, t1, Wc, Hc, ch);
    s = fmaf(v0, v0, s);
    if (n2 < N) s = fmaf(v1, v1, s);
  }
  part[g][c] = s;
  __syncthreads();
  if (g == 0) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < DN_GROUPS; ++i) t += part[i][c];
    cnorm[b * 256 + ch] = sqrtf(t);
  }
}

// (S^T / cnorm - mean) @ comp^T  (:215-221).  CTA = 8 keypoints of one image, 256 threads.
constexpr int DP_KP = 8;
template <bool SLOT = false>
__global__ void __launch_bounds__(256)
sp_desc_pca_kernel(const float* __restrict__ desc, const int32_t* __restrict__ slot, const float* __restrict__ cell_n,
                   int H, int W, const int32_t* __restrict__ n_kpts,
                   const float* __restrict__ kpts, int max_num, const float* __restrict__ cnorm,
                   const float* __restrict__ pca_compT, const float* __restrict__ pca_mean, float* __restrict__ out) {
  __shared__ float sv[DP_KP][256];
  const int b = blockIdx.y, n0 = blockIdx.x * DP_KP, tid = threadIdx.x;
  const int N = n_kpts[b];
  if (n0 >= N) return;
  const int Hc = H / 8, Wc = W / 8;
  const float* d = SLOT ? desc : desc + (size_t)b * Hc * Wc * 256;
  const int32_t* sl = SLOT ? slot + (size_t)b * Hc * Wc : nullptr;
  const float cn = cnorm[b * 256 + tid], mu = pca_mean[tid];
#pragma unroll
  for (int i = 0; i < DP_KP; ++i) {                       // unrolled: the 8 x 4 tap loads are independent L2 round trips
    const int n = n0 + i;
    float v = 0.f;
    if (n < N) {
      const Taps t = bilinear_taps(kpts[((size_t)b * max_num + n) * 2], kpts[((size_t)b * max_num + n) * 2 + 1], W, H, Wc, Hc);
      v = __fsub_rn(__fdiv_rn(sample_channel<SLOT>(d, sl, cell_n, 0, t, Wc, Hc, tid), cn), mu);
    }
    sv[i][tid] = v;
  }
  __syncthreads();
  // 8 keypoints x 64 outputs = 512 dot products of length 256; thread -> (kp = tid/32 .., o = ...)
  const int o = tid & 63, kq = tid >> 6;  // kq in 0..3 -> keypoints kq and kq+4
  float a0 = 0.f, a1 = 0.f;
#pragma unroll 8
  for (int c = 0; c < 256; ++c) {
    const float w = __ldg(pca_compT + c * 64 + o);   // transposed [256][64]: coalesced across o
    a0 = fmaf(sv[kq][c], w, a0);
    a1 = fmaf(sv[kq + 4][c], w, a1);
  }
  if (n0 + kq < N) out[((size_t)b * max_num + n0 + kq) * 64 + o] = a0;
  if (n0 + kq + 4 < N) out[((size_t)b * max_num + n0 + kq + 4) * 64 + o] = a1;
}

osb_status sp_descriptors(const float* desc_nhwc, int B, int H, int W, const int32_t* n_kpts, const float* kpts,
                          int max_num, const float* pca_compT, const float* pca_mean, float* cnorm, float* out,
                          cudaStream_t st, const int32_t* slot, int seg, float* cell_n) {
  const dim3 gn(B, 256 / DN_CH), gp(cdiv(max_num, DP_KP), B);
  if (slot) {
    OSB_REQUIRE(seg * 4 <= 48 * 1024 && cell_n, "sparse descriptor head: too many rows per image");
    OSB_LAUNCH(sp_desc_norm_kernel<true>, gn, DN_GROUPS * DN_CH, seg * 4, st, desc_nhwc, slot, seg, cell_n, H, W, n_kpts,
               kpts, max_num, cnorm);
    OSB_CHECK_LAUNCH();
    OSB_LAUNCH(sp_desc_pca_kernel<true>, gp, 256, 0, st, desc_nhwc, slot, cell_n, H, W, n_kpts, kpts, max_num, cnorm,
               pca_compT, pca_mean, out);
  } else {
    OSB_LAUNCH(sp_desc_norm_kernel<false>, gn, DN_GROUPS * DN_CH, 0, st, desc_nhwc, slot, 0, cell_n, H, W, n_kpts, kpts,
               max_num, cnorm);
    OSB_CHECK_LAUNCH();
    OSB_LAUNCH(sp_desc_pca_kernel<false>, gp, 256, 0, st, desc_nhwc, slot, cell_n, H, W, n_kpts, kpts, max_num, cnorm,
               pca_compT, pca_mean, out);
  }
  OSB_CHECK_LAUNCH();
  return OSB_OK;
}

// -------------------------------------------------------------------------------------------------------------
// layout helpers (used by the parity hooks only)
// -------------------------------------------------------------------------------------------------------------
__global__ void nchw_to_nhwc_kernel(const float* __restrict__ in, float* __restrict__ out, int C, int hw, int64_t total) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c = (int)(i % C);
  const int64_t p = (i / C) % hw;
  const int64_t b = i / ((int64_t)C * hw);
  out[i] = in[(b * C + c) * hw + p];
}
__global__ void nhwc_to_nchw_kernel(const float* __restrict__ in, float* __restrict__ out, int C, int hw, int64_t total) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int64_t p = i % hw;
  const int c = (int)((i / hw) % C);
  const int64_t b = i / ((int64_t)C * hw);
  out[i] = in[(b * hw + p) * C + c];
}
osb_status nchw_to_nhwc(const float* in, float* out, int B, int C, int h, int w, cudaStream_t st) {
  const int64_t total = (int64_t)B * C * h * w;
  OSB_LAUNCH(nchw_to_nhwc_kernel, (unsigned)cdiv64(total, 256), 256, 0, st, in, out, C, h * w, total);
  OSB_CHECK_LAUNCH();
  return OSB_OK;
}
osb_status nhwc_to_nchw(const float* in, float* out, int B, int C, int h, int w, cudaStream_t st) {
  const int64_t total = (int64_t)B * C * h * w;
  OSB_LAUNCH(nhwc_to_nchw_kernel, (unsigned)cdiv64(total, 256), 256, 0, st, in, out, C, h * w, total);
  OSB_CHECK_LAUNCH();
  return OSB_OK;
}

}  // namespace osb
