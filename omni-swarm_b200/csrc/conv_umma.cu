// conv_umma.cu -- SuperPoint / NetVLAD convolutions on the Hopper tensor cores (wgmma + TMA + mbarrier), sm_90a.
//
// Layers: swarm_loop/superpoint.ipynb:143-158 of the reference (3x3 pad 1 and 1x1 convolutions, NHWC here).
//
// Implicit GEMM, one CTA tile = 8 x 16 output pixels (M = 128) x N output channels (conv_umma_kernel: N = 64 or 80; the
// 128-channel layers, and those of 256 / 512 channels as 2 / 4 work items of 128 channels per tile, run transposed in
// conv_stream_t_kernel, below):
//   * A operand: for every horizontal filter tap kx and every 64-channel slab, ONE TMA box {64 ch, 16 x, 8 + 2 y, 1 image}
//     fetched at the kx-shifted coordinate; out-of-image elements are zero-filled by the TMA unit, which is the
//     convolution's zero padding.  The box lands in shared memory as one 128-byte row per pixel with the 128-byte swizzle,
//     i.e. exactly the canonical K-major SWIZZLE_128B wgmma layout (im2col staging is done by the copy engine).  The three
//     vertical taps ky read the same box from pixel row ky on: + ky * 2048 bytes, a multiple of the 1024-byte swizzle atom.
//   * B operand: the weight slab [N][64] of the same tap, K-major SWIZZLE_128B, by TMA.
//   * D: fp32 accumulators in the registers of two consumer warpgroups, 64 pixels each.  Warpgroup g reads the 8-pixel core
//     matrices at columns 8g .. 8g+7 of the eight tile rows (descriptor stride = one pixel row), so the two accumulator
//     rows a thread holds are vertically adjacent pixels of one column: the fused 2x2 max-pool is one max in the thread
//     and one shuffle.
// Precision: parity with the fp32 oracle needs ~1e-6 relative error, which fp16/bf16 operands cannot give.  Every
// fp32 operand x is carried as TWO fp16 planes  hi = fp16(s*x), lo = fp16(s*x - hi)  (s a power of two, exact), and
// each K step computes the three products  hi*hi + lo*hi + hi*lo  (the dropped lo*lo term is 2^-22 relative): hi*hi goes
// to a MAIN accumulator, the two cross products to a CROSS accumulator whose magnitude -- and rounding error -- is 2^-11
// of the main one; the epilogue adds them in fp32.  The weight slot is [W_hi (N rows) | W_lo (N rows)]; per K step three
// MMAs of width N write two register fragments of the same shape (hi*hi -> main, hi*lo and lo*hi -> cross), disjoint so
// that the compiler keeps the wgmma pipeline asynchronous.  Both planes together are 4 bytes per element -- the same
// HBM/L2 footprint as fp32 activations.  Measured against the oracle: see tests/test_gpu_superpoint.py.
// Warp roles (384 threads): warpgroups 0-1 = MMA + epilogue, warpgroup 2 = producer (one elected thread issues the TMA
// copies).  Persistent over tiles; the producer runs up to two A boxes and the weight ring ahead of the MMAs.
//
// The 64 -> 64 channel 3x3 layers (conv1b, conv2a, conv2b: 65 % of the network's MACs) run in conv_res64_kernel instead:
// the 9 taps' weights stay resident in shared memory, and the GEMM is transposed, D[64 oc][128 px] = W * X^T, so that each
// MMA is m64n128k16 with the weight slab as the 64-row operand and the whole tile's A box as the 128-column one (three
// such MMAs read 18 KB of shared memory per 192 tensor clocks, where six m64n64k16 of the form above read 24 KB).  Each
// consumer warpgroup computes whole tiles, alternating with the other, so that one's epilogue runs under the other's MMAs.
#include <cuda.h>
#include <cuda_fp16.h>
#include <cmath>
#include "common.cuh"
#include "kernels.cuh"
#include "conv_umma.cuh"
#include "umma_ptx.cuh"

namespace osb {

constexpr int UM_TH = 8, UM_TW = 16;            // output tile (pixels)
constexpr int UM_KC = 64;                       // fp16 channels per K slab (= 128 bytes = one swizzle row)
constexpr int UM_ROW = UM_TW * 128;             // bytes of one pixel row of an A box (2 swizzle atoms)

// Shared-memory plan.  For a 3x3 layer ONE A box per (kx, 64-channel slab) carries 10 rows (tile + vertical halo), read
// by the three vertical taps; that cuts the activation traffic from 9 to 3.75 tile-loads per tile.  The weights of each
// tap stream through their own ring.
constexpr int UM_A_SLOT = (UM_TH + 2) * UM_ROW;        // 20 KB per plane: 10 rows x 16 px x 128 B
constexpr int UM_A_SLOTS = 2;
// threads: warpgroups 0 and 1 issue the MMAs and run the epilogue, warpgroup 2 is the producer.  Launched at 168 registers
// per thread; the producer hands registers to the MMA warpgroups with setmaxnreg (producer 40 -> consumers 232), so that a
// 128-register accumulator fragment fits with the MMA pipeline in flight.
constexpr int UM_CONSUMERS = 256;
constexpr int UM_THREADS = UM_CONSUMERS + 128;
constexpr int UM_PRODUCER_REGS = 40, UM_CONSUMER_REGS = 232;
static_assert(128 * UM_PRODUCER_REGS + UM_CONSUMERS * UM_CONSUMER_REGS <= 65536, "register file");
// FP16 = true is the plain-fp16 form of every kernel below (OSB_PRECISION_FP16): only the hi planes are read and written,
// one MMA per K step.  Its slots hold one plane, so the same 80 KB ring carries four A boxes and the weight ring twice
// the slots of the split form (B_SLOT = B_BYTES).
template <int N, bool FP16 = false>
struct UmmaCfg {
  static_assert(N == 64 || N == 80, "128-channel layers run in conv_stream_t_kernel");
  static constexpr int PLANES = FP16 ? 1 : 2;
  static constexpr int A_SLOTS = FP16 ? 4 : UM_A_SLOTS;
  static constexpr int A_RING = A_SLOTS * PLANES * UM_A_SLOT;    // 80 KB either way
  static constexpr int B_BYTES = N * 128;                        // one weight plane of one tap / slab
  static constexpr int B_SLOT = PLANES * B_BYTES;                // hi (+ lo)
  static constexpr int B_SLOTS = FP16 ? ((N <= 64) ? 12 : 10) : ((N <= 64) ? 6 : 5);
  static constexpr int SMEM_BYTES = A_RING + B_SLOTS * B_SLOT + 1024 /*alignment slack*/ + 256 /*barriers*/;
  static_assert(SMEM_BYTES <= 227 * 1024, "shared-memory plan exceeds the 227 KB of an H100 block");
  static_assert(2 * (A_SLOTS + B_SLOTS) * 8 <= 256, "barriers exceed their 256 bytes");
};
// conv_res64_kernel: the 9 taps' weight planes (9 x 16 KB, or 9 x 8 KB of W_hi in fp16) stay resident in shared memory
// for the CTA's whole life.  The fp16 form spends the freed 72 KB on a ring of six hi boxes (120 KB): with three boxes per
// tile, warpgroup 0's tiles always land in slots 0-2 and warpgroup 1's in slots 3-5, so the producer fills a warpgroup's
// next tile while the other warpgroup still holds its own.
template <bool FP16 = false>
struct R64Cfg {
  static constexpr int PLANES = FP16 ? 1 : 2;
  static constexpr int A_SLOTS = FP16 ? 6 : UM_A_SLOTS;
  static constexpr int A_RING = A_SLOTS * PLANES * UM_A_SLOT;
  static constexpr int W_PLANE = 64 * 128;                       // [64 oc][64 ch] fp16
  static constexpr int W_SLOT = PLANES * W_PLANE;                // W_hi (| W_lo) of one tap
  static constexpr int SMEM_BYTES = A_RING + 9 * W_SLOT + 1024 /*alignment slack*/ + 256 /*barriers*/;
  static_assert(SMEM_BYTES <= 227 * 1024, "shared-memory plan exceeds the 227 KB of an H100 block");
  static_assert((3 * A_SLOTS + 9) * 8 <= 256, "barriers exceed their 256 bytes");
};
// conv_stream_t_kernel: a ring of A boxes read by both consumer warpgroups, and per warpgroup a ring of weight HALF slots
// (the 64 rows [64g, 64g + 64) of the item's 128-row slab; hi (+ lo)).  Split: 3 boxes of 40 KB + 2 x 3 half slots of
// 16 KB = 216 KB; fp16: 6 boxes of 20 KB + 2 x 6 half slots of 8 KB = 216 KB.  With the commit-group release rule a
// warpgroup holds at most two boxes and two of its half slots, so any ring of at least 3 boxes and 3 half slots runs,
// with room for one warpgroup to run ahead of the other.
template <bool FP16 = false>
struct StreamTCfg {
  static constexpr int PLANES = FP16 ? 1 : 2;
  static constexpr int A_SLOTS = FP16 ? 6 : 3;
  static constexpr int A_RING = A_SLOTS * PLANES * UM_A_SLOT;    // 120 KB either way
  static constexpr int W_PLANE = 64 * 128;                       // [64 oc][64 ch] fp16
  static constexpr int W_SLOT = PLANES * W_PLANE;                // W_hi (| W_lo) of one half
  static constexpr int W_SLOTS = FP16 ? 6 : 3;                   // per warpgroup
  static constexpr int SMEM_BYTES = A_RING + 2 * W_SLOTS * W_SLOT + 1024 /*alignment slack*/ + 512 /*barriers*/;
  static_assert(A_SLOTS >= 3 && W_SLOTS >= 3, "the rings need three slots each for the two warpgroups to run apart");
  static_assert(SMEM_BYTES <= 227 * 1024, "shared-memory plan exceeds the 227 KB of an H100 block");
  static_assert(2 * (A_SLOTS + 2 * W_SLOTS) * 8 <= 512, "barriers exceed their 512 bytes");
};

struct UmmaArgs {
  const float* bias;       // [N]
  __half* out_hi;          // NHWC planes of the next layer (or null)
  __half* out_lo;
  float* out_f32;          // fp32 output [pixels][out_cstride] (or null)
  int H, W, B;
  int ks;                  // 1 or 3
  int cin_slabs;           // Cin / 64
  int out_c;               // channels stored per pixel (<= N)
  int out_cstride;         // channel stride of the destination
  float inv_scale;         // 1 / (act_scale * w_scale)
  float out_scale;         // scale of the stored fp16 planes
  int relu;                // 0 none, 1 ReLU, 2 ReLU6
  int n_off;               // first output channel of this launch
  int pool;                // 1: fused 2x2 max-pool, the planes written are [B][H/2][W/2][C]
  int n_split;             // a layer wider than the kernel's N runs as n_split work items per tile (N channels each)
  int epi;                 // 0: bias/act/pool + store; 1: detector head -- softmax over 65 logits, drop the dustbin,
                           //    8x8 pixel shuffle straight into the heat map `out_f32` ([B][8H][8W])
  TileRect band;           // BAND kernels: these tiles of every image are stored as the constant band_hi / band_lo
  const __half* band_hi;   // [out_c] each
  const __half* band_lo;
};

// BAND kernels: the launch's work items are the tiles outside the band, compacted in tile order; image b's items follow
// image b - 1's.  Producer and consumers map an item to its tile here.
__device__ __forceinline__ int band_tile(int item, int tiles_x, int tiles_y, const UmmaArgs& P) {
  const int bh = P.band.y1 - P.band.y0, bw = P.band.x1 - P.band.x0, m = tiles_x - bw;   // m: computed tiles per band row
  const int per = tiles_x * tiles_y - bh * bw;
  const int b = item / per;
  int k = item - b * per, t;
  const int head = P.band.y0 * tiles_x;
  if (k < head) {
    t = k;
  } else if ((k -= head) < bh * m) {
    const int row = k / m, c = k - row * m;
    t = (P.band.y0 + row) * tiles_x + (c < P.band.x0 ? c : c + bw);
  } else {
    t = P.band.y1 * tiles_x + (k - bh * m);
  }
  return b * tiles_x * tiles_y + t;
}

// BAND kernels: the band's outputs (after the pool, if any), 8 channels of one pixel per 16-byte store of each plane.  The
// CTAs of the launch share the work; thread t of the CTA's nt filling threads.
template <bool FP16>
__device__ void band_fill(const UmmaArgs& P, int t, int nt) {
  const int sh = P.pool ? 1 : 0;
  const int Ho = P.H >> sh, Wo = P.W >> sh;
  const int y0 = (P.band.y0 * UM_TH) >> sh, x0 = (P.band.x0 * UM_TW) >> sh;
  const int bh = ((P.band.y1 - P.band.y0) * UM_TH) >> sh, bw = ((P.band.x1 - P.band.x0) * UM_TW) >> sh;
  const int c8 = P.out_c / 8, total = P.B * bh * bw * c8;              // < 2^31: checked on the host
  const uint4* chi = reinterpret_cast<const uint4*>(P.band_hi);
  const uint4* clo = reinterpret_cast<const uint4*>(P.band_lo);
  for (int e = blockIdx.x * nt + t; e < total; e += gridDim.x * nt) {
    const int c = e % c8, p = e / c8, x = p % bw, y = (p / bw) % bh, b = p / (bw * bh);
    const size_t o = (((size_t)b * Ho + y0 + y) * Wo + x0 + x) * P.out_cstride + P.n_off + 8 * c;
    *reinterpret_cast<uint4*>(P.out_hi + o) = __ldg(chi + c);
    if constexpr (!FP16) *reinterpret_cast<uint4*>(P.out_lo + o) = __ldg(clo + c);
  }
}

// 4 x 4 transpose of 32-bit words across the four lanes of a quad (t4 = lane % 4): on return v[k] is the word v[t4] of
// quad lane k.  Round r takes word (t4 - r) % 4 from lane (t4 + r) % 4; all indices stay compile-time after unrolling.
__device__ __forceinline__ void quad_transpose(uint32_t (&v)[4], int t4) {
  uint32_t o[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) o[k] = (k == t4) ? v[k] : 0u;
#pragma unroll
  for (int r = 1; r < 4; ++r) {
    const int send = (t4 - r) & 3, from = (t4 + r) & 3;
    uint32_t s = v[0];
#pragma unroll
    for (int k = 1; k < 4; ++k) s = (send == k) ? v[k] : s;
    const uint32_t got = __shfl_sync(0xffffffffu, s, (threadIdx.x & 28) | from);
#pragma unroll
    for (int k = 0; k < 4; ++k) o[k] = (from == k) ? got : o[k];
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) v[k] = o[k];
}

// FP16: the plain-fp16 form (UmmaCfg): tm_a_lo / tm_w_lo and P.out_lo are not used
template <int N, bool FP16 = false>
__global__ void __launch_bounds__(UM_THREADS, 1)
conv_umma_kernel(const __grid_constant__ CUtensorMap tm_a_hi, const __grid_constant__ CUtensorMap tm_a_lo,
                 const __grid_constant__ CUtensorMap tm_w_hi, const __grid_constant__ CUtensorMap tm_w_lo, UmmaArgs P) {
  using Cfg = UmmaCfg<N, FP16>;
  constexpr int AS = Cfg::A_SLOTS, BS = Cfg::B_SLOTS, A_STRIDE = Cfg::PLANES * UM_A_SLOT;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t b_base = smem_base + Cfg::A_RING;
  const uint32_t bar_base = b_base + BS * Cfg::B_SLOT;                   // 8-byte barriers
  auto a_full = [&](int s) { return bar_base + 8u * s; };
  auto a_empty = [&](int s) { return bar_base + 8u * (AS + s); };
  auto b_full = [&](int s) { return bar_base + 8u * (2 * AS + s); };
  auto b_empty = [&](int s) { return bar_base + 8u * (2 * AS + BS + s); };

  const int lane = threadIdx.x & 31;
  const int tiles_x = (P.W + UM_TW - 1) / UM_TW, tiles_y = (P.H + UM_TH - 1) / UM_TH;
  const int n_tiles = P.B * tiles_x * tiles_y;
  const int halo = P.ks / 2;
  const uint32_t a_box_bytes = (uint32_t)(UM_TH + 2 * halo) * UM_ROW;   // bytes of one A plane box

  if (threadIdx.x == 0) {
    // the empty barriers count one arrival per consumer warpgroup
    for (int s = 0; s < AS; ++s) { mbar_init(a_full(s), 1); mbar_init(a_empty(s), 2); }
    for (int s = 0; s < BS; ++s) { mbar_init(b_full(s), 1); mbar_init(b_empty(s), 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  // programmatic dependent launch: the next layer's CTAs may be scheduled as ours retire (they still wait for this whole
  // grid in their own griddepcontrol.wait before touching activations)
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

  if (threadIdx.x >= UM_CONSUMERS) {
    const int pt = threadIdx.x - UM_CONSUMERS;             // producer thread
    setmaxnreg_dec<UM_PRODUCER_REGS>();
    // the activations are the previous kernel's output: wait for the whole grid we depend on (no-op without PDL)
    asm volatile("griddepcontrol.wait;" ::: "memory");
    if (pt < 32 && elect_one()) {
      // ===================== TMA producer =====================
      int as = 0; uint32_t aph = 0;
      int bs = 0; uint32_t bph = 0;
      for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int tx = tile % tiles_x, ty = (tile / tiles_x) % tiles_y, b = tile / (tiles_x * tiles_y);
        const int x0 = tx * UM_TW, y0 = ty * UM_TH;
        for (int kx = 0; kx < P.ks; ++kx) {
          for (int cs = 0; cs < P.cin_slabs; ++cs) {
            // activation box: tile rows + vertical halo at the kx-shifted column, shared by the ks vertical taps
            mbar_wait(a_empty(as), aph ^ 1);
            const uint32_t sa = smem_base + as * A_STRIDE;
            mbar_expect_tx(a_full(as), Cfg::PLANES * a_box_bytes);
            tma_load_4d(sa, &tm_a_hi, a_full(as), cs * UM_KC, x0 + kx - halo, y0 - halo, b);
            if constexpr (!FP16) tma_load_4d(sa + UM_A_SLOT, &tm_a_lo, a_full(as), cs * UM_KC, x0 + kx - halo, y0 - halo, b);
            if (++as == AS) { as = 0; aph ^= 1; }
            for (int ky = 0; ky < P.ks; ++ky) {
              mbar_wait(b_empty(bs), bph ^ 1);
              const uint32_t sb = b_base + bs * Cfg::B_SLOT;
              mbar_expect_tx(b_full(bs), Cfg::B_SLOT);
              tma_load_3d(sb, &tm_w_hi, b_full(bs), cs * UM_KC, P.n_off, ky * P.ks + kx);
              if constexpr (!FP16) tma_load_3d(sb + Cfg::B_BYTES, &tm_w_lo, b_full(bs), cs * UM_KC, P.n_off, ky * P.ks + kx);
              if (++bs == BS) { bs = 0; bph ^= 1; }
            }
          }
        }
      }
    }
  } else {
    // ===================== MMA + epilogue (two warpgroups, 64 pixels each) =====================
    setmaxnreg_inc<UM_CONSUMER_REGS>();
    const int cw = threadIdx.x >> 7;                         // warpgroup: tile columns 8cw .. 8cw+7
    const int wq = (threadIdx.x >> 5) & 3;                   // warp of the warpgroup: tile rows 2wq, 2wq+1
    const int col = lane >> 2, t4 = lane & 3;                // pixel column in the core matrix, channel pair in a group of 8
    const bool signaller = (threadIdx.x & 127) == 0;
    int as = 0; uint32_t aph = 0;
    int bs = 0; uint32_t bph = 0;
    // buffers are released once the MMAs that read them have retired: one warpgroup arrival on each empty barrier.  The MMAs
    // of one vertical tap form one commit group, and a group's buffers (its weight slot; the A box after its last tap) are
    // released when the NEXT group has been issued and this one has completed -- so a warpgroup holds at most two weight
    // slots and two A boxes at any time, whatever the ring sizes.
    auto release = [&](int a_slot, int b_slot) {
      if (!signaller) return;
      if (a_slot >= 0) mbar_arrive(a_empty(a_slot));
      if (b_slot >= 0) mbar_arrive(b_empty(b_slot));
    };
    const int n_off = P.n_off;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
      // two fragments of the same shape (N/2 registers each): main = hi*hi, cross = hi*lo + lo*hi.  Disjoint register sets --
      // an MMA into part of another MMA's fragment would make the compiler serialize the wgmma pipeline.  fp16: main only
      float acc[N / 2], cross[FP16 ? 1 : N / 2];
#pragma unroll
      for (int i = 0; i < N / 2; ++i) { acc[i] = 0.f; if constexpr (!FP16) cross[i] = 0.f; }
      uint32_t scale_d = 0;
      int pend_a = -1, pend_b = -1;                          // buffers of the last committed group
      for (int kx = 0; kx < P.ks; ++kx) {
        for (int cs = 0; cs < P.cin_slabs; ++cs) {
          mbar_wait(a_full(as), aph);
          const uint32_t sa = smem_base + as * A_STRIDE + cw * 1024;
          for (int ky = 0; ky < P.ks; ++ky) {
            mbar_wait(b_full(bs), bph);
            const uint32_t sb = b_base + bs * Cfg::B_SLOT;
            const int b_slot = bs;
            if (++bs == BS) { bs = 0; bph ^= 1; }
            // vertical tap ky reads the box from pixel row ky on; core matrices one pixel row (2048 B) apart
            const uint64_t a_hi = wgmma_desc_sw128(sa + ky * UM_ROW, UM_ROW);
            const uint64_t a_lo = wgmma_desc_sw128(sa + UM_A_SLOT + ky * UM_ROW, UM_ROW);
            const uint64_t b_hi = wgmma_desc_sw128(sb, 1024), b_lo = wgmma_desc_sw128(sb + Cfg::B_BYTES, 1024);
            // the warpgroup is converged again after the barrier waits: fence the accumulators here, right before the
            // tap's MMAs, so that no compiler-inserted fence lands on a divergent path and serializes the MMA pipeline
#pragma unroll
            for (int i = 0; i < N / 2; ++i) { fence_operand(acc[i]); if constexpr (!FP16) fence_operand(cross[i]); }
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < UM_KC / 16; ++k) {
              const uint64_t adv = (uint64_t)(k * 32 >> 4);     // advance 16 fp16 = 32 bytes inside the swizzle row
              Wgmma<N>::mma(acc, a_hi + adv, b_hi + adv, scale_d);        // hi*hi -> main
              if constexpr (!FP16) {
                Wgmma<N>::mma(cross, a_hi + adv, b_lo + adv, scale_d);    // hi*lo -> cross
                Wgmma<N>::mma(cross, a_lo + adv, b_hi + adv, 1u);         // lo*hi -> cross
              }
              scale_d = 1;
            }
            wgmma_commit();
#pragma unroll
            for (int i = 0; i < N / 2; ++i) { fence_operand(acc[i]); if constexpr (!FP16) fence_operand(cross[i]); }
            wgmma_wait<1>();                                 // the previous group has retired
            release(pend_a, pend_b);
            pend_a = (ky == P.ks - 1) ? as : -1;
            pend_b = b_slot;
          }
          if (++as == AS) { as = 0; aph ^= 1; }
        }
      }
      wgmma_wait<0>();
      release(pend_a, pend_b);
#pragma unroll
      for (int i = 0; i < N / 2; ++i) { fence_operand(acc[i]); if constexpr (!FP16) fence_operand(cross[i]); }

      // ---- epilogue: registers [4j, 4j+1] hold channels 8j + 2*t4 + {0,1} of pixel (y, x), [4j+2, 4j+3] of (y+1, x) ----
      const int tx = tile % tiles_x, ty = (tile / tiles_x) % tiles_y, b = tile / (tiles_x * tiles_y);
      const int x = tx * UM_TW + cw * 8 + col, y = ty * UM_TH + 2 * wq;
      const bool in0 = y < P.H && x < P.W, in1 = y + 1 < P.H && x < P.W;
      const size_t pix0 = ((size_t)b * P.H + y) * P.W + x, pix1 = pix0 + P.W;
      auto value = [&](int r, int c) {                       // r = register index of the main accumulator
        if constexpr (FP16) return fmaf(acc[r], P.inv_scale, __ldg(P.bias + n_off + c));
        else return fmaf(acc[r] + cross[r], P.inv_scale, __ldg(P.bias + n_off + c));
      };
      if (P.epi == 1) {
        // fused detector head (superpoint.ipynb:190-198): softmax over the 65 logits of a cell, which four lanes of a quad
        // hold, then the dustbin is dropped and the 64 probabilities are pixel-shuffled into the heat map
        const int W8 = P.W * 8;
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          float mx = -INFINITY;
#pragma unroll
          for (int j = 0; j < 9; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e)
              if (8 * j + 2 * t4 + e < 65) mx = fmaxf(mx, value(4 * j + 2 * r + e, 8 * j + 2 * t4 + e));
          mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
          mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
          float sum = 0.f;
#pragma unroll
          for (int j = 0; j < 9; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e)
              if (8 * j + 2 * t4 + e < 65) sum += expf(value(4 * j + 2 * r + e, 8 * j + 2 * t4 + e) - mx);
          sum += __shfl_xor_sync(0xffffffffu, sum, 1);
          sum += __shfl_xor_sync(0xffffffffu, sum, 2);
          if (!(r ? in1 : in0)) continue;
          float* out = P.out_f32 + ((size_t)b * P.H * 8 + (size_t)(y + r) * 8) * W8 + (size_t)x * 8 + 2 * t4;
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float e0 = expf(value(4 * j + 2 * r, 8 * j + 2 * t4) - mx) / sum;
            const float e1 = expf(value(4 * j + 2 * r + 1, 8 * j + 2 * t4 + 1) - mx) / sum;
            *reinterpret_cast<float2*>(out + (size_t)j * W8) = make_float2(e0, e1);
          }
        }
      } else {
        // fused 2x2 max-pool: the pooled pixel of (even y, even x) is the max over this thread's two rows and the lane
        // holding column x + 1 (lane + 4); writer lanes hold even columns
        const int py = ty * (UM_TH / 2) + wq, px = tx * (UM_TW / 2) + cw * 4 + (col >> 1);
        const bool pool_writer = !(col & 1) && py < (P.H >> 1) && px < (P.W >> 1);
        const size_t ppix = ((size_t)b * (P.H >> 1) + py) * (P.W >> 1) + px;
        auto store = [&](size_t pix, int c, float v0, float v1) {
          if (P.out_f32) {
            *reinterpret_cast<float2*>(P.out_f32 + pix * P.out_cstride + n_off + c) = make_float2(v0, v1);
          } else {
            const float s0 = v0 * P.out_scale, s1 = v1 * P.out_scale;
            // packed conversions (cvt.rn.f16x2.f32: the roundings of two scalar conversions)
            const __half2 hp = __floats2half2_rn(s0, s1);
            if constexpr (FP16) {
              *reinterpret_cast<__half2*>(P.out_hi + pix * P.out_cstride + n_off + c) = hp;
            } else {
              const float2 hf = __half22float2(hp);
              const __half2 lp = __floats2half2_rn(s0 - hf.x, s1 - hf.y);
              *reinterpret_cast<__half2*>(P.out_hi + pix * P.out_cstride + n_off + c) = hp;
              *reinterpret_cast<__half2*>(P.out_lo + pix * P.out_cstride + n_off + c) = lp;
            }
          }
        };
        if (N % 32 == 0 && !P.pool && !P.out_f32) {
          // planes without pooling: the quad holds 8 channels (16 bytes) of its pixel for every block j.  Four blocks are
          // transposed across the quad at a time so that each lane stores one block whole: one 16-byte store where the
          // loop below issues four 4-byte ones
#pragma unroll
          for (int q = 0; q < N / 32; ++q) {
            if (n_off - P.n_off + 32 * q >= P.out_c) continue;           // warp-uniform
            uint32_t h[2][4], l[2][4];                                   // [pixel row][block 4q + k]
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              const int j = 4 * q + k, c = 8 * j + 2 * t4;
#pragma unroll
              for (int r = 0; r < 2; ++r) {
                float a0 = value(4 * j + 2 * r, c), a1 = value(4 * j + 2 * r + 1, c + 1);
                if (P.relu) { a0 = fmaxf(a0, 0.f); a1 = fmaxf(a1, 0.f); }
                if (P.relu == 2) { a0 = fminf(a0, 6.f); a1 = fminf(a1, 6.f); }
                const float s0 = a0 * P.out_scale, s1 = a1 * P.out_scale;
                const __half2 hp = __floats2half2_rn(s0, s1);        // the roundings of `store` below
                if constexpr (FP16) {
                  h[r][k] = *reinterpret_cast<const uint32_t*>(&hp);
                } else {
                  const float2 hf = __half22float2(hp);
                  const __half2 lp = __floats2half2_rn(s0 - hf.x, s1 - hf.y);
                  h[r][k] = *reinterpret_cast<const uint32_t*>(&hp);
                  l[r][k] = *reinterpret_cast<const uint32_t*>(&lp);
                }
              }
            }
#pragma unroll
            for (int r = 0; r < 2; ++r) { quad_transpose(h[r], t4); if constexpr (!FP16) quad_transpose(l[r], t4); }
            const int cb = n_off + 8 * (4 * q + t4);                     // the block this lane stores
            if (cb - P.n_off >= P.out_c) continue;
            if (in0) {
              *reinterpret_cast<uint4*>(P.out_hi + pix0 * P.out_cstride + cb) = make_uint4(h[0][0], h[0][1], h[0][2], h[0][3]);
              if constexpr (!FP16)
                *reinterpret_cast<uint4*>(P.out_lo + pix0 * P.out_cstride + cb) = make_uint4(l[0][0], l[0][1], l[0][2], l[0][3]);
            }
            if (in1) {
              *reinterpret_cast<uint4*>(P.out_hi + pix1 * P.out_cstride + cb) = make_uint4(h[1][0], h[1][1], h[1][2], h[1][3]);
              if constexpr (!FP16)
                *reinterpret_cast<uint4*>(P.out_lo + pix1 * P.out_cstride + cb) = make_uint4(l[1][0], l[1][1], l[1][2], l[1][3]);
            }
          }
          continue;
        }
#pragma unroll
        for (int j = 0; j < N / 8; ++j) {
          if (n_off - P.n_off + 8 * j >= P.out_c) continue;            // warp-uniform
          const int c = 8 * j + 2 * t4;
          float f[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            float a = value(4 * j + i, c + (i & 1));
            if (P.relu) a = fmaxf(a, 0.f);
            if (P.relu == 2) a = fminf(a, 6.f);
            f[i] = a;
          }
          if (P.pool) {
            float m0 = fmaxf(f[0], f[2]), m1 = fmaxf(f[1], f[3]);
            m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 4));
            m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 4));
            if (pool_writer) store(ppix, c, m0, m1);
          } else {
            if (in0) store(pix0, c, f[0], f[1]);
            if (in1) store(pix1, c, f[2], f[3]);
          }
        }
      }
    }
  }
}

// --------------------------------------------------------------------------------------------------------------
// 64 -> 64 channel 3x3 layers: weights resident, D[64 oc][128 px] = W * X^T, one warpgroup per tile
// --------------------------------------------------------------------------------------------------------------
// Per K step three wgmma m64n128k16: W_hi*X_hi -> main, W_lo*X_hi -> cross, W_hi*X_lo -> cross (the products and the
// accumulators they go to of conv_umma_kernel, with M and N swapped).
//   * M operand: the tap's weight slab [64 oc][64 ch] of a resident slot (K-major SWIZZLE_128B, 8-row groups 1024 B apart).
//   * N operand: the whole 8 x 16 tile from the A box, one 128-byte row per pixel in row-major order, so the 16 8-pixel
//     core-matrix groups are 1024 B apart; vertical tap ky starts at + ky * 2048 B as before.
//   * D: warp w of a warpgroup holds output channels 16w + lane/4 and + 8; fragment register 4j + 2h + e is channel
//     16w + 8h + lane/4 of pixel (j / 2, 8 (j & 1) + 2 (lane & 3) + e) of the tile: row y + 1 is n-group j + 2, so the
//     fused 2x2 max-pool is all in the thread.
// Tiles: the CTA's i-th tile belongs to warpgroup i & 1.  The producer fills one ring of two A boxes (hi + lo) in tile
// order, three boxes per tile.  Each slot has one full barrier per warpgroup, so that a warpgroup's parity sequence counts
// only its own boxes, and one empty barrier on which the single reader of a box arrives.
// FP16: one wgmma W_hi*X_hi per K step on hi-only boxes and resident W_hi (R64Cfg); tm_a_lo / tm_w_lo are not used.
//
// tr_epilogue: bias, ReLU / ReLU6, optional 2x2 max-pool and the stores of one warpgroup's D[64 oc][128 px] fragment of
// this layout (conv_res64_kernel and conv_stream_t_kernel).  c_abs is the output channel of fragment row 0, c_rel the
// same channel counted from the launch's first one (P.n_off; compared with P.out_c); bias[h] is channel
// c_abs + 16w + 8h + lane/4.  NHWC outputs want channel-contiguous stores, so the split planes and the fp32 values are
// transposed across the warp in registers (movmatrix): afterwards a quad holds one pixel's 8-channel block.
template <bool FP16>
__device__ __forceinline__ void tr_epilogue(const float (&acc)[64], const float (&cross)[FP16 ? 1 : 64],
                                            const float (&bias)[2], int c_abs, int c_rel, int tile, int tiles_x,
                                            int tiles_y, const UmmaArgs& P, int w, int r, int t4) {
  if (c_rel + 16 * w >= P.out_c) return;                     // warp-uniform; out_c is a multiple of 16
  const int tx = tile % tiles_x, ty = (tile / tiles_x) % tiles_y, b = tile / (tiles_x * tiles_y);
  const int x0 = tx * UM_TW, y0 = ty * UM_TH;
  auto value = [&](int k, int h) {                           // fragment register k, channel half h
    float a;
    if constexpr (FP16) a = fmaf(acc[k], P.inv_scale, bias[h]);
    else a = fmaf(acc[k] + cross[k], P.inv_scale, bias[h]);
    if (P.relu) a = fmaxf(a, 0.f);
    if (P.relu == 2) a = fminf(a, 6.f);
    return a;
  };
  // split a channel's values of two pixels into the planes and transpose the 8 x 8 (channel x pixel) blocks of the
  // warp: afterwards lane l holds channels 2 (l % 4), + 1 of pixel l / 4, so a quad holds 16 contiguous bytes.
  // fp16: the hi plane only (tl is not written)
  auto split_t = [&](float v0, float v1, uint32_t& th, uint32_t& tl) {
    const float s0 = v0 * P.out_scale, s1 = v1 * P.out_scale;
    const __half2 hp = __floats2half2_rn(s0, s1);            // packed conversions: the roundings of two scalar ones
    if constexpr (FP16) {
      th = movmatrix_trans(*reinterpret_cast<const uint32_t*>(&hp));
    } else {
      const float2 hf = __half22float2(hp);
      const __half2 lp = __floats2half2_rn(s0 - hf.x, s1 - hf.y);
      th = movmatrix_trans(*reinterpret_cast<const uint32_t*>(&hp));
      tl = movmatrix_trans(*reinterpret_cast<const uint32_t*>(&lp));
    }
  };
  if (!P.pool && !P.out_f32) {
    // unpooled planes: the four blocks (n-group 2y + k / 2, channel half k % 2) of tile row y are transposed across the
    // quad as well, so that lane t4 holds block t4 whole and writes it with one 16-byte store: column 8 (t4 / 2) + r,
    // channels c_abs + 16w + 8 (t4 % 2) .. + 7
#pragma unroll
    for (int y = 0; y < UM_TH; ++y) {
      uint32_t th[4], tl[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int j = 2 * y + (k >> 1), h = k & 1;
        split_t(value(4 * j + 2 * h, h), value(4 * j + 2 * h + 1, h), th[k], tl[k]);
      }
      quad_transpose(th, t4);
      if constexpr (!FP16) quad_transpose(tl, t4);
      const int gy = y0 + y, gx = x0 + 8 * (t4 >> 1) + r;
      if (gy < P.H && gx < P.W) {
        const size_t o = (((size_t)b * P.H + gy) * P.W + gx) * P.out_cstride + c_abs + 16 * w + 8 * (t4 & 1);
        *reinterpret_cast<uint4*>(P.out_hi + o) = make_uint4(th[0], th[1], th[2], th[3]);
        if constexpr (!FP16) *reinterpret_cast<uint4*>(P.out_lo + o) = make_uint4(tl[0], tl[1], tl[2], tl[3]);
      }
    }
    return;
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int cb = 16 * w + 8 * h;                           // first channel of the warp's 8-channel block
    const int c_own = c_abs + cb + r, c_st = c_abs + cb + 2 * t4;
    if (P.pool) {
      // pooled row py of the tile, pooled column 4k + t4 from n-groups j = 4py + k and j + 2
      const int Hp = P.H >> 1, Wp = P.W >> 1;
#pragma unroll
      for (int py = 0; py < UM_TH / 2; ++py) {
        float m[2];
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          const int j = 4 * py + k;
          m[k] = fmaxf(fmaxf(value(4 * j + 2 * h, h), value(4 * (j + 2) + 2 * h, h)),
                       fmaxf(value(4 * j + 2 * h + 1, h), value(4 * (j + 2) + 2 * h + 1, h)));
        }
        const int gpy = ty * (UM_TH / 2) + py;
        if (P.out_f32) {
#pragma unroll
          for (int k = 0; k < 2; ++k) {
            const int gpx = tx * (UM_TW / 2) + 4 * k + t4;
            if (gpy < Hp && gpx < Wp) P.out_f32[(((size_t)b * Hp + gpy) * Wp + gpx) * P.out_cstride + c_own] = m[k];
          }
        } else {
          // column 2 t4 + k of the block is pooled pixel 4k + t4: after the transpose lane l holds pixel
          // 4 ((l / 4) & 1) + (l / 4) / 2
          uint32_t th, tl;
          split_t(m[0], m[1], th, tl);
          const int gpx = tx * (UM_TW / 2) + 4 * (r & 1) + (r >> 1);
          if (gpy < Hp && gpx < Wp) {
            const size_t o = (((size_t)b * Hp + gpy) * Wp + gpx) * P.out_cstride + c_st;
            *reinterpret_cast<uint32_t*>(P.out_hi + o) = th;
            if constexpr (!FP16) *reinterpret_cast<uint32_t*>(P.out_lo + o) = tl;
          }
        }
      }
    } else {
      // fp32: the low and the high 16 bits of each value are transposed as two b16 blocks and put back together, so
      // that lane l holds channels c_st, c_st + 1 of pixel column 8 (j & 1) + l / 4 for one 8-byte store
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const uint32_t u0 = __float_as_uint(value(4 * j + 2 * h, h)), u1 = __float_as_uint(value(4 * j + 2 * h + 1, h));
        const uint32_t tlo = movmatrix_trans(__byte_perm(u0, u1, 0x5410)), thi = movmatrix_trans(__byte_perm(u0, u1, 0x7632));
        const int gy = y0 + (j >> 1), gx = x0 + 8 * (j & 1) + r;
        if (gy < P.H && gx < P.W)
          *reinterpret_cast<float2*>(P.out_f32 + (((size_t)b * P.H + gy) * P.W + gx) * P.out_cstride + c_st) =
              make_float2(__uint_as_float(__byte_perm(tlo, thi, 0x5410)), __uint_as_float(__byte_perm(tlo, thi, 0x7632)));
      }
    }
  }
}

// BAND: the tiles of P.band are not computed: the items are the other tiles (band_tile), and producer warps 1-3, idle
// otherwise, store the band's constant (band_fill) while the MMAs run.
template <bool FP16 = false, bool BAND = false>
__global__ void __launch_bounds__(UM_THREADS, 1)
conv_res64_kernel(const __grid_constant__ CUtensorMap tm_a_hi, const __grid_constant__ CUtensorMap tm_a_lo,
                  const __grid_constant__ CUtensorMap tm_w_hi, const __grid_constant__ CUtensorMap tm_w_lo, UmmaArgs P) {
  using Cfg = R64Cfg<FP16>;
  constexpr int AS = Cfg::A_SLOTS, A_STRIDE = Cfg::PLANES * UM_A_SLOT;
  constexpr int R64_W_PLANE = Cfg::W_PLANE, R64_W_SLOT = Cfg::W_SLOT;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t w_base = smem_base + Cfg::A_RING;
  const uint32_t bar_base = w_base + 9 * R64_W_SLOT;                     // 8-byte barriers
  auto a_full = [&](int g, int s) { return bar_base + 8u * (g * AS + s); };
  auto a_empty = [&](int s) { return bar_base + 8u * (2 * AS + s); };
  auto w_full = [&](int t) { return bar_base + 8u * (3 * AS + t); };

  const int lane = threadIdx.x & 31;
  const int tiles_x = (P.W + UM_TW - 1) / UM_TW, tiles_y = (P.H + UM_TH - 1) / UM_TH;
  const int n_tiles = P.B * (tiles_x * tiles_y - (BAND ? (P.band.y1 - P.band.y0) * (P.band.x1 - P.band.x0) : 0));
  auto tile_of = [&](int item) { return BAND ? band_tile(item, tiles_x, tiles_y, P) : item; };

  if (threadIdx.x == 0) {
    for (int s = 0; s < AS; ++s) { mbar_init(a_full(0, s), 1); mbar_init(a_full(1, s), 1); mbar_init(a_empty(s), 1); }
    for (int t = 0; t < 9; ++t) mbar_init(w_full(t), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

  if (threadIdx.x >= UM_CONSUMERS) {
    const int pt = threadIdx.x - UM_CONSUMERS;
    setmaxnreg_dec<UM_PRODUCER_REGS>();
    if (pt < 32 && elect_one()) {
      // all 9 taps once: slot t holds tap t.  Issued BEFORE the dependency wait: weights are constants, so under
      // programmatic dependent launch they stream in while the previous layer is still draining.
      for (int t = 0; t < 9; ++t) {
        const uint32_t sw = w_base + t * R64_W_SLOT;
        mbar_expect_tx(w_full(t), R64_W_SLOT);
        tma_load_3d(sw, &tm_w_hi, w_full(t), 0, P.n_off, t);
        if constexpr (!FP16) tma_load_3d(sw + R64_W_PLANE, &tm_w_lo, w_full(t), 0, P.n_off, t);
      }
    }
    asm volatile("griddepcontrol.wait;" ::: "memory");
    if constexpr (BAND) if (pt >= 32) band_fill<FP16>(P, pt - 32, 96);
    if (pt < 32 && elect_one()) {
      int as = 0; uint32_t aph = 0;
      for (int i = 0, item = blockIdx.x; item < n_tiles; ++i, item += gridDim.x) {
        const int tile = tile_of(item);
        const int tx = tile % tiles_x, ty = (tile / tiles_x) % tiles_y, b = tile / (tiles_x * tiles_y);
        const int x0 = tx * UM_TW, y0 = ty * UM_TH;
        for (int kx = 0; kx < 3; ++kx) {
          mbar_wait(a_empty(as), aph ^ 1);
          const uint32_t sa = smem_base + as * A_STRIDE;
          const uint32_t full = a_full(i & 1, as);
          mbar_expect_tx(full, A_STRIDE);
          tma_load_4d(sa, &tm_a_hi, full, 0, x0 + kx - 1, y0 - 1, b);
          if constexpr (!FP16) tma_load_4d(sa + UM_A_SLOT, &tm_a_lo, full, 0, x0 + kx - 1, y0 - 1, b);
          if (++as == AS) { as = 0; aph ^= 1; }
        }
      }
    }
  } else {
    setmaxnreg_inc<UM_CONSUMER_REGS>();
    const int g = threadIdx.x >> 7;                          // warpgroup: the CTA's tiles of parity g
    const int w = (threadIdx.x >> 5) & 3;                    // warp: output channels 16w .. 16w + 15
    const int r = lane >> 2, t4 = lane & 3;
    const bool signaller = (threadIdx.x & 127) == 0;
    for (int t = 0; t < 9; ++t) mbar_wait(w_full(t), 0);
    const float bias[2] = {__ldg(P.bias + P.n_off + 16 * w + r), __ldg(P.bias + P.n_off + 16 * w + 8 + r)};
    uint32_t fph = 0;                                        // bit s: parity of this warpgroup's next box in slot s
    for (int i = g, item = blockIdx.x + g * gridDim.x; item < n_tiles; i += 2, item += 2 * gridDim.x) {
      const int tile = tile_of(item);
      // disjoint fragments (64 registers each): main = hi*hi, cross = lo*hi + hi*lo.  fp16: main only
      float acc[64], cross[FP16 ? 1 : 64];
#pragma unroll
      for (int k = 0; k < 64; ++k) { acc[k] = 0.f; if constexpr (!FP16) cross[k] = 0.f; }
      uint32_t scale_d = 0;
      int pend = -1;                                         // box to release once the last group that reads it retires
      for (int kx = 0; kx < 3; ++kx) {
        const int as = (3 * i + kx) % AS;                    // box kx of the CTA's i-th tile is the ring's (3i + kx)-th
        mbar_wait(a_full(g, as), (fph >> as) & 1u);
        fph ^= 1u << as;
        const uint32_t sa = smem_base + as * A_STRIDE;
        for (int ky = 0; ky < 3; ++ky) {
          const uint32_t sw = w_base + (ky * 3 + kx) * R64_W_SLOT;
          const uint64_t w_hi = wgmma_desc_sw128(sw, 1024), w_lo = wgmma_desc_sw128(sw + R64_W_PLANE, 1024);
          const uint64_t x_hi = wgmma_desc_sw128(sa + ky * UM_ROW, 1024);
          const uint64_t x_lo = wgmma_desc_sw128(sa + UM_A_SLOT + ky * UM_ROW, 1024);
#pragma unroll
          for (int k = 0; k < 64; ++k) { fence_operand(acc[k]); if constexpr (!FP16) fence_operand(cross[k]); }
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < UM_KC / 16; ++k) {
            const uint64_t adv = (uint64_t)(k * 32 >> 4);
            Wgmma<128>::mma(acc, w_hi + adv, x_hi + adv, scale_d);       // hi*hi -> main
            if constexpr (!FP16) {
              Wgmma<128>::mma(cross, w_lo + adv, x_hi + adv, scale_d);   // lo*hi -> cross
              Wgmma<128>::mma(cross, w_hi + adv, x_lo + adv, 1u);        // hi*lo -> cross
            }
            scale_d = 1;
          }
          wgmma_commit();
#pragma unroll
          for (int k = 0; k < 64; ++k) { fence_operand(acc[k]); if constexpr (!FP16) fence_operand(cross[k]); }
          wgmma_wait<1>();
          if (signaller && pend >= 0) mbar_arrive(a_empty(pend));
          pend = (ky == 2) ? as : -1;
        }
      }
      wgmma_wait<0>();
      if (signaller) mbar_arrive(a_empty(pend));
#pragma unroll
      for (int k = 0; k < 64; ++k) { fence_operand(acc[k]); if constexpr (!FP16) fence_operand(cross[k]); }

      tr_epilogue<FP16>(acc, cross, bias, P.n_off, 0, tile, tiles_x, tiles_y, P, w, r, t4);
    }
  }
}

// --------------------------------------------------------------------------------------------------------------
// 128-channel layers (and 256 / 512 as 2 / 4 work items of 128 channels): streamed weights, D[64 oc][128 px] = W * X^T
// --------------------------------------------------------------------------------------------------------------
// The MMAs of conv_res64_kernel on conv_umma_kernel's pipeline.  Both consumer warpgroups work on the same item: warpgroup
// g owns output channels [64g, 64g + 64) of it across all 128 pixels of the tile, reads every A box (the empty barrier
// counts both readers) and only its own 64 weight rows, which producer warp 1 + g streams through the warpgroup's own
// ring of half slots (StreamTCfg), so that every weight row still crosses L2 once per item and a warpgroup that runs
// ahead never waits on the other's weights.  Producer warp 0 loads the A boxes.  Per K step (kx, then slab, then ky,
// then the four k16 steps, as conv_umma_kernel) three wgmma m64n128k16: W_hi*X_hi -> main, W_lo*X_hi -> cross,
// W_hi*X_lo -> cross.
// Skew: warpgroup 1 starts once warpgroup 0 has issued the MMAs of its first box.  From then on the two run a box apart,
// so that each one's epilogue overlaps the other's MMAs instead of leaving the tensor pipe idle.
// FP16: one wgmma W_hi*X_hi per K step on hi-only boxes and W_hi-only half slots; tm_a_lo / tm_w_lo are not used.
// BAND (not with SPLIT): the tiles of P.band are not computed (conv_res64_kernel); producer warp 3 stores their constant.
template <bool SPLIT, bool FP16 = false, bool BAND = false>
__global__ void __launch_bounds__(UM_THREADS, 1)
conv_stream_t_kernel(const __grid_constant__ CUtensorMap tm_a_hi, const __grid_constant__ CUtensorMap tm_a_lo,
                     const __grid_constant__ CUtensorMap tm_w_hi, const __grid_constant__ CUtensorMap tm_w_lo, UmmaArgs P) {
  using Cfg = StreamTCfg<FP16>;
  constexpr int AS = Cfg::A_SLOTS, WS = Cfg::W_SLOTS, A_STRIDE = Cfg::PLANES * UM_A_SLOT;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t w_base = smem_base + Cfg::A_RING;                       // warpgroup g's half slots at + g * WS * W_SLOT
  const uint32_t bar_base = w_base + 2 * WS * Cfg::W_SLOT;               // 8-byte barriers
  auto a_full = [&](int s) { return bar_base + 8u * s; };
  auto a_empty = [&](int s) { return bar_base + 8u * (AS + s); };
  auto w_full = [&](int g, int s) { return bar_base + 8u * (2 * AS + g * WS + s); };
  auto w_empty = [&](int g, int s) { return bar_base + 8u * (2 * AS + 2 * WS + g * WS + s); };

  const int lane = threadIdx.x & 31;
  const int tiles_x = (P.W + UM_TW - 1) / UM_TW, tiles_y = (P.H + UM_TH - 1) / UM_TH;
  // work item = (tile, 128-channel block): items of one tile are adjacent, so concurrent CTAs share its activations in L2
  static_assert(!(SPLIT && BAND), "a band is not taken by the layers of more than 128 channels");
  const int n_split = SPLIT ? P.n_split : 1;          // compile-time 1 for ordinary layers: no div / mod per item
  const int n_items =
      P.B * (tiles_x * tiles_y - (BAND ? (P.band.y1 - P.band.y0) * (P.band.x1 - P.band.x0) : 0)) * n_split;
  auto tile_of = [&](int item) { return SPLIT ? item / n_split : BAND ? band_tile(item, tiles_x, tiles_y, P) : item; };
  const int halo = P.ks / 2;
  const uint32_t a_box_bytes = (uint32_t)(UM_TH + 2 * halo) * UM_ROW;   // bytes of one A plane box

  if (threadIdx.x == 0) {
    for (int s = 0; s < AS; ++s) { mbar_init(a_full(s), 1); mbar_init(a_empty(s), 2); }
    for (int s = 0; s < 2 * WS; ++s) { mbar_init(w_full(0, s), 1); mbar_init(w_empty(0, s), 1); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

  if (threadIdx.x >= UM_CONSUMERS) {
    const int pw = (threadIdx.x - UM_CONSUMERS) >> 5;      // producer warp: 0 A boxes, 1 + g weight rows of warpgroup g
    setmaxnreg_dec<UM_PRODUCER_REGS>();
    asm volatile("griddepcontrol.wait;" ::: "memory");
    if constexpr (BAND) if (pw == 3) band_fill<FP16>(P, lane, 32);
    if (pw < 3 && elect_one()) {
      const int g = pw - 1;
      int s = 0; uint32_t ph = 0;
      for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
        const int tile = tile_of(item), n_off = SPLIT ? P.n_off + (item % n_split) * 128 : P.n_off;
        const int tx = tile % tiles_x, ty = (tile / tiles_x) % tiles_y, b = tile / (tiles_x * tiles_y);
        for (int kx = 0; kx < P.ks; ++kx) {
          for (int cs = 0; cs < P.cin_slabs; ++cs) {
            if (pw == 0) {
              mbar_wait(a_empty(s), ph ^ 1);
              const uint32_t sa = smem_base + s * A_STRIDE;
              const int xa = tx * UM_TW + kx - halo, ya = ty * UM_TH - halo;
              mbar_expect_tx(a_full(s), Cfg::PLANES * a_box_bytes);
              tma_load_4d(sa, &tm_a_hi, a_full(s), cs * UM_KC, xa, ya, b);
              if constexpr (!FP16) tma_load_4d(sa + UM_A_SLOT, &tm_a_lo, a_full(s), cs * UM_KC, xa, ya, b);
              if (++s == AS) { s = 0; ph ^= 1; }
              continue;
            }
            for (int ky = 0; ky < P.ks; ++ky) {
              mbar_wait(w_empty(g, s), ph ^ 1);
              const uint32_t sw = w_base + (g * WS + s) * Cfg::W_SLOT;
              mbar_expect_tx(w_full(g, s), Cfg::W_SLOT);
              tma_load_3d(sw, &tm_w_hi, w_full(g, s), cs * UM_KC, n_off + 64 * g, ky * P.ks + kx);
              if constexpr (!FP16)
                tma_load_3d(sw + Cfg::W_PLANE, &tm_w_lo, w_full(g, s), cs * UM_KC, n_off + 64 * g, ky * P.ks + kx);
              if (++s == WS) { s = 0; ph ^= 1; }
            }
          }
        }
      }
    }
  } else {
    setmaxnreg_inc<UM_CONSUMER_REGS>();
    const int g = threadIdx.x >> 7;                          // warpgroup: output channels [64g, 64g + 64) of every item
    const int w = (threadIdx.x >> 5) & 3;                    // warp: output channels 64g + 16w .. + 15
    const int r = lane >> 2, t4 = lane & 3;
    const bool signaller = (threadIdx.x & 127) == 0;
    const uint32_t w_ring = w_base + g * WS * Cfg::W_SLOT;
    bool skew_set = g == 1;                                  // warpgroup 0 releases warpgroup 1 once
    if (g == 1) named_bar_sync(1, 256);
    // buffers are released once the MMAs that read them have retired (conv_umma_kernel's commit-group rule): one arrival
    // per warpgroup on the box's empty barrier, the reader's on its half slot's
    auto release = [&](int a_slot, int w_slot) {
      if (!signaller) return;
      if (a_slot >= 0) mbar_arrive(a_empty(a_slot));
      if (w_slot >= 0) mbar_arrive(w_empty(g, w_slot));
    };
    int as = 0; uint32_t aph = 0;
    int ws = 0; uint32_t wph = 0;
    for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
      const int tile = tile_of(item), n_off = SPLIT ? P.n_off + (item % n_split) * 128 : P.n_off;
      const int c_abs = n_off + 64 * g;
      const float bias[2] = {__ldg(P.bias + c_abs + 16 * w + r), __ldg(P.bias + c_abs + 16 * w + 8 + r)};
      // disjoint fragments (64 registers each): main = hi*hi, cross = lo*hi + hi*lo.  fp16: main only
      float acc[64], cross[FP16 ? 1 : 64];
#pragma unroll
      for (int k = 0; k < 64; ++k) { acc[k] = 0.f; if constexpr (!FP16) cross[k] = 0.f; }
      uint32_t scale_d = 0;
      int pend_a = -1, pend_w = -1;                          // buffers of the last committed group
      for (int kx = 0; kx < P.ks; ++kx) {
        for (int cs = 0; cs < P.cin_slabs; ++cs) {
          mbar_wait(a_full(as), aph);
          const uint32_t sa = smem_base + as * A_STRIDE;
          for (int ky = 0; ky < P.ks; ++ky) {
            mbar_wait(w_full(g, ws), wph);
            const uint32_t sw = w_ring + ws * Cfg::W_SLOT;
            const int w_slot = ws;
            if (++ws == WS) { ws = 0; wph ^= 1; }
            const uint64_t w_hi = wgmma_desc_sw128(sw, 1024), w_lo = wgmma_desc_sw128(sw + Cfg::W_PLANE, 1024);
            const uint64_t x_hi = wgmma_desc_sw128(sa + ky * UM_ROW, 1024);
            const uint64_t x_lo = wgmma_desc_sw128(sa + UM_A_SLOT + ky * UM_ROW, 1024);
#pragma unroll
            for (int k = 0; k < 64; ++k) { fence_operand(acc[k]); if constexpr (!FP16) fence_operand(cross[k]); }
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < UM_KC / 16; ++k) {
              const uint64_t adv = (uint64_t)(k * 32 >> 4);
              Wgmma<128>::mma(acc, w_hi + adv, x_hi + adv, scale_d);       // hi*hi -> main
              if constexpr (!FP16) {
                Wgmma<128>::mma(cross, w_lo + adv, x_hi + adv, scale_d);   // lo*hi -> cross
                Wgmma<128>::mma(cross, w_hi + adv, x_lo + adv, 1u);        // hi*lo -> cross
              }
              scale_d = 1;
            }
            wgmma_commit();
#pragma unroll
            for (int k = 0; k < 64; ++k) { fence_operand(acc[k]); if constexpr (!FP16) fence_operand(cross[k]); }
            wgmma_wait<1>();
            release(pend_a, pend_w);
            pend_a = (ky == P.ks - 1) ? as : -1;
            pend_w = w_slot;
          }
          if (++as == AS) { as = 0; aph ^= 1; }
          if (!skew_set) { named_bar_arrive(1, 256); skew_set = true; }
        }
      }
      wgmma_wait<0>();
      release(pend_a, pend_w);
#pragma unroll
      for (int k = 0; k < 64; ++k) { fence_operand(acc[k]); if constexpr (!FP16) fence_operand(cross[k]); }
      tr_epilogue<FP16>(acc, cross, bias, c_abs, c_abs - P.n_off, tile, tiles_x, tiles_y, P, w, r, t4);
    }
  }
}

// --------------------------------------------------------------------------------------------------------------
// first layer (Cin = 1) and 2x2 max-pool on split planes, re-split after the fp32 op
// --------------------------------------------------------------------------------------------------------------
// FP16 (here and in the three kernels below): the fp32 arithmetic is the same, only the hi plane is written
template <bool FP16>
__device__ __forceinline__ void split_store8(__half* hi, __half* lo, const float* f, float scale) {
  uint32_t h[4], l[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float s0 = f[2 * i] * scale, s1 = f[2 * i + 1] * scale;
    const __half h0 = __float2half_rn(s0), h1 = __float2half_rn(s1);
    h[i] = (uint32_t)__half_as_ushort(h0) | ((uint32_t)__half_as_ushort(h1) << 16);
    if constexpr (!FP16) {
      const __half l0 = __float2half_rn(s0 - __half2float(h0)), l1 = __float2half_rn(s1 - __half2float(h1));
      l[i] = (uint32_t)__half_as_ushort(l0) | ((uint32_t)__half_as_ushort(l1) << 16);
    }
  }
  *reinterpret_cast<uint4*>(hi) = make_uint4(h[0], h[1], h[2], h[3]);
  if constexpr (!FP16) *reinterpret_cast<uint4*>(lo) = make_uint4(l[0], l[1], l[2], l[3]);
}

// conv1a (Cin = 1) + bias + ReLU -> split fp16 planes.  Thread = (8 output channels, one pixel column of a 32 x 8 tile):
// the 72 weights of its channels live in registers for the whole tile, the inputs (after the u8 -> f32 LUT) are staged
// once per CTA in shared memory and slide down the column through registers (3 broadcast LDS per pixel instead of one
// LDS per FMA pair), and the 8 threads of a pixel write its 128-byte channel vector as eight adjacent 16-byte chunks --
// a warp stores 4 pixels x 128 B contiguously per plane, no staging of the output.  The plane scale (a power of two) is
// folded into weights and bias, and the 9 taps (ky-major) accumulate onto the bias.  The pixels of `skip` (those no
// computed tile of the next layer reads) are neither computed nor written.
constexpr int CF_TW = 32, CF_TH = 8;
template <bool FP16 = false>
__global__ void __launch_bounds__(256)
conv_first_split_kernel(const float* __restrict__ w, const float* __restrict__ bias, const float* __restrict__ lut,
                        const uint8_t* __restrict__ img, __half* __restrict__ out_hi, __half* __restrict__ out_lo,
                        int H, int W, float out_scale, TileRect skip) {
  __shared__ float sin_[CF_TH + 2][CF_TW + 2];
  const int tid = threadIdx.x, b = blockIdx.z, x0 = blockIdx.x * CF_TW, y0 = blockIdx.y * CF_TH;
  if (y0 >= skip.y0 && y0 + CF_TH <= skip.y1 && x0 >= skip.x0 && x0 + CF_TW <= skip.x1) return;   // the whole block
  const uint8_t* ib = img + (size_t)b * H * W;
  for (int e = tid; e < (CF_TH + 2) * (CF_TW + 2); e += 256) {
    const int r = e / (CF_TW + 2), c = e % (CF_TW + 2);
    const int gy = y0 + r - 1, gx = x0 + c - 1;
    sin_[r][c] = (gy >= 0 && gy < H && gx >= 0 && gx < W) ? __ldg(lut + ib[(size_t)gy * W + gx]) : 0.f;
  }
  const int cg = tid & 7, px = tid >> 3;
  float wr[9][8], br[8];
#pragma unroll
  for (int t = 0; t < 9; ++t) {
    const float4 w0 = __ldg(reinterpret_cast<const float4*>(w + t * 64 + cg * 8));
    const float4 w1 = __ldg(reinterpret_cast<const float4*>(w + t * 64 + cg * 8 + 4));
    wr[t][0] = w0.x; wr[t][1] = w0.y; wr[t][2] = w0.z; wr[t][3] = w0.w;
    wr[t][4] = w1.x; wr[t][5] = w1.y; wr[t][6] = w1.z; wr[t][7] = w1.w;
#pragma unroll
    for (int j = 0; j < 8; ++j) wr[t][j] *= out_scale;          // power of two: exact, commutes with every rounding below
  }
  {
    const float4 b0 = __ldg(reinterpret_cast<const float4*>(bias + cg * 8));
    const float4 b1 = __ldg(reinterpret_cast<const float4*>(bias + cg * 8 + 4));
    br[0] = b0.x; br[1] = b0.y; br[2] = b0.z; br[3] = b0.w; br[4] = b1.x; br[5] = b1.y; br[6] = b1.z; br[7] = b1.w;
#pragma unroll
    for (int j = 0; j < 8; ++j) br[j] *= out_scale;
  }
  __syncthreads();
  const int x = x0 + px;
  float in[3][3];
#pragma unroll
  for (int k = 0; k < 3; ++k) { in[0][k] = sin_[0][px + k]; in[1][k] = sin_[1][px + k]; }
#pragma unroll
  for (int r = 0; r < CF_TH; ++r) {
#pragma unroll
    for (int k = 0; k < 3; ++k) in[2][k] = sin_[r + 2][px + k];
    const int y = y0 + r;
    if (y < H && x < W && !(y >= skip.y0 && y < skip.y1 && x >= skip.x0 && x < skip.x1)) {
      uint32_t h[4], l[4];
#pragma unroll
      for (int j2 = 0; j2 < 4; ++j2) {
        float a0 = br[2 * j2], a1 = br[2 * j2 + 1];                // bias first: 9 taps accumulate onto it
#pragma unroll
        for (int t = 0; t < 9; ++t) {
          a0 = fmaf(in[t / 3][t % 3], wr[t][2 * j2], a0);
          a1 = fmaf(in[t / 3][t % 3], wr[t][2 * j2 + 1], a1);
        }
        const float s0 = fmaxf(a0, 0.f), s1 = fmaxf(a1, 0.f);
        const __half h0 = __float2half_rn(s0), h1 = __float2half_rn(s1);
        h[j2] = (uint32_t)__half_as_ushort(h0) | ((uint32_t)__half_as_ushort(h1) << 16);
        if constexpr (!FP16) {
          const __half l0 = __float2half_rn(s0 - __half2float(h0)), l1 = __float2half_rn(s1 - __half2float(h1));
          l[j2] = (uint32_t)__half_as_ushort(l0) | ((uint32_t)__half_as_ushort(l1) << 16);
        }
      }
      const size_t chunk = (((size_t)b * H + y) * W + x) * 8 + cg;          // 16-byte chunk index inside the plane
      reinterpret_cast<uint4*>(out_hi)[chunk] = make_uint4(h[0], h[1], h[2], h[3]);
      if constexpr (!FP16) reinterpret_cast<uint4*>(out_lo)[chunk] = make_uint4(l[0], l[1], l[2], l[3]);
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) { in[0][k] = in[1][k]; in[1][k] = in[2][k]; }
  }
}

// --------------------------------------------------------------------------------------------------------------
// host side
// --------------------------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = (PFN_encodeTiled)p;
  }
  return fn;
}

osb_status umma_make_tmap(CUtensorMap* tm, void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                          const uint32_t* box) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) { set_error("conv_umma", "cuTensorMapEncodeTiled entry point not available"); return OSB_ERR_CUDA; }
  cuuint64_t gd[5]; cuuint64_t gs[4]; cuuint32_t bx[5]; cuuint32_t es[5];
  for (int i = 0; i < rank; ++i) { gd[i] = dims[i]; bx[i] = box[i]; es[i] = 1; }
  for (int i = 0; i < rank - 1; ++i) gs[i] = strides_bytes[i];
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank, base, gd, gs, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char buf[128];
    snprintf(buf, sizeof(buf), "cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
    set_error("conv_umma", buf);
    return OSB_ERR_CUDA;
  }
  return OSB_OK;
}

osb_status umma_layer_upload(Resources& res, UmmaLayer* L, const float* w_oihw, const float* bias, int cin, int cout,
                             int ks, float w_scale) {
  L->cin = cin; L->cout = cout; L->ks = ks; L->taps = ks * ks; L->w_scale = w_scale;
  L->n_pad = (cout <= 64) ? 64 : (cout <= 80) ? 80 : (cout <= 128) ? 128 : (cout <= 256) ? 256 : 512;
  OSB_REQUIRE(cin % UM_KC == 0 && cout <= 512, "tensor-core conv: Cin must be a multiple of 64 and Cout <= 512");
  const size_t n = (size_t)L->taps * L->n_pad * cin;
  std::vector<__half> hi(n, __float2half(0.f)), lo(n, __float2half(0.f));
  std::vector<float> bp(L->n_pad, 0.f);
  for (int o = 0; o < cout; ++o) {
    bp[o] = bias[o];
    for (int c = 0; c < cin; ++c)
      for (int t = 0; t < L->taps; ++t) {
        const float s = w_oihw[((size_t)o * cin + c) * L->taps + t] * w_scale;
        const __half h = __float2half_rn(s);
        if (!std::isfinite(__half2float(h))) {
          char buf[192];
          snprintf(buf, sizeof(buf), "weight %g (output %d, input %d, tap %d) is outside the split-fp16 range: "
                   "|w| * %g must be below 65520", (double)w_oihw[((size_t)o * cin + c) * L->taps + t], o, c, t,
                   (double)w_scale);
          set_error("umma_layer_upload", buf);
          return OSB_ERR_INVALID;
        }
        const size_t idx = ((size_t)t * L->n_pad + o) * cin + c;
        hi[idx] = h;
        lo[idx] = __float2half_rn(s - __half2float(h));
      }
  }
  OSB_TRY(res.upload(&L->w_hi, hi.data(), n));
  OSB_TRY(res.upload(&L->w_lo, lo.data(), n));
  OSB_TRY(res.upload(&L->bias, bp.data(), L->n_pad));
  const uint64_t dims[3] = {(uint64_t)cin, (uint64_t)L->n_pad, (uint64_t)L->taps};
  const uint64_t strides[2] = {(uint64_t)cin * 2, (uint64_t)cin * L->n_pad * 2};
  // one box = the 80 rows of the detector head, else 64 rows: a whole slab of the N = 64 kernels, one warpgroup's half
  // of a 128-channel work item in conv_stream_t_kernel
  const uint32_t box[3] = {UM_KC, (uint32_t)(L->n_pad == 80 ? 80 : 64), 1};
  OSB_TRY(umma_make_tmap(&L->tm_hi, L->w_hi, 3, dims, strides, box));
  OSB_TRY(umma_make_tmap(&L->tm_lo, L->w_lo, 3, dims, strides, box));
  return OSB_OK;
}

osb_status umma_act_maps(CUtensorMap* hi, CUtensorMap* lo, __half* p_hi, __half* p_lo, int B, int H, int W, int C,
                         int ks) {
  const uint64_t dims[4] = {(uint64_t)C, (uint64_t)W, (uint64_t)H, (uint64_t)B};
  const uint64_t strides[3] = {(uint64_t)C * 2, (uint64_t)W * C * 2, (uint64_t)H * W * C * 2};
  // the box carries the vertical halo of the layer that READS these planes (ks x ks filter)
  const uint32_t box[4] = {UM_KC, UM_TW, (uint32_t)(UM_TH + 2 * (ks / 2)), 1};
  osb_status s;
  if ((s = umma_make_tmap(hi, p_hi, 4, dims, strides, box)) != OSB_OK) return s;
  return umma_make_tmap(lo, p_lo, 4, dims, strides, box);
}

// OSB_CONV_PDL=1 launches the convolutions with programmatic dependent launch.  Off by default: the dependent layer's CTAs
// take the SMs the concurrent NetVLAD stream of the front-end would otherwise fill.
static const bool g_conv_pdl = [] { const char* e = getenv("OSB_CONV_PDL"); return e && atoi(e) != 0; }();

// one instantiation per kernel: the shared-memory opt-in is remembered per instantiation
template <auto kernel>
static osb_status launch_persistent(int smem_bytes, const CUtensorMap& a_hi, const CUtensorMap& a_lo,
                                    const CUtensorMap& w_hi, const CUtensorMap& w_lo, const UmmaArgs& P, cudaStream_t st,
                                    int max_ctas) {
  OSB_SMEM_OPT_IN(kernel, smem_bytes);
  // work items: the tiles outside the band.  Every CTA must get one: conv_stream_t_kernel's warpgroup 1 waits for
  // warpgroup 0 to start its first item
  const int band_tiles = (P.band.y1 - P.band.y0) * (P.band.x1 - P.band.x0);
  const int tiles = P.B * (cdiv(P.W, UM_TW) * cdiv(P.H, UM_TH) - (P.band.empty() ? 0 : band_tiles)) * P.n_split;
  // persistent CTAs, one per SM; `max_ctas` leaves SMs free for a kernel running beside this one on another stream
  const int grid = std::max(1, std::min(tiles, persistent_ctas(max_ctas)));
  cudaLaunchConfig_t cfg = {};
  cudaLaunchAttribute attr[1];
  cfg.gridDim = dim3(grid); cfg.blockDim = dim3(UM_THREADS); cfg.dynamicSmemBytes = smem_bytes; cfg.stream = st;
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = g_conv_pdl ? 1 : 0;
  cfg.attrs = attr; cfg.numAttrs = 1;
  OSB_CUDA(cudaLaunchKernelEx(&cfg, kernel, a_hi, a_lo, w_hi, w_lo, P));
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return OSB_OK;
}

template <int N, bool FP16 = false>
static osb_status launch_umma(const CUtensorMap& a_hi, const CUtensorMap& a_lo, const UmmaLayer& L, const UmmaArgs& P,
                              cudaStream_t st, int max_ctas) {
  return launch_persistent<conv_umma_kernel<N, FP16>>(UmmaCfg<N, FP16>::SMEM_BYTES, a_hi, a_lo, L.tm_hi, L.tm_lo, P, st,
                                                      max_ctas);
}

template <bool SPLIT, bool FP16, bool BAND = false>
static osb_status launch_stream_t(const CUtensorMap& a_hi, const CUtensorMap& a_lo, const UmmaLayer& L, const UmmaArgs& P,
                                  cudaStream_t st, int max_ctas) {
  return launch_persistent<conv_stream_t_kernel<SPLIT, FP16, BAND>>(StreamTCfg<FP16>::SMEM_BYTES, a_hi, a_lo, L.tm_hi,
                                                                    L.tm_lo, P, st, max_ctas);
}

static bool precision_fp16(int precision) { return precision == OSB_PRECISION_FP16; }

void band_geometry(int H, int W, int r0, const BandLayer* layers, int n, TileRect* px, TileRect* tiles,
                   TileRect* first_skip) {
  // the constant input of the first layer: the zero rows
  TileRect in;
  if (r0 >= 0 && r0 < H) in = TileRect{r0, H, 0, W};
  int h = H, w = W;
  for (int l = 0; l < n; ++l) {
    const int halo = layers[l].ks / 2;
    // outputs whose window lies in the image and in the constant input
    TileRect o{std::max(in.y0 + halo, halo), std::min(in.y1 - halo, h - halo), std::max(in.x0 + halo, halo),
               std::min(in.x1 - halo, w - halo)};
    if (in.empty() || o.empty()) o = TileRect{};
    TileRect t{cdiv(o.y0, UM_TH), o.y1 / UM_TH, cdiv(o.x0, UM_TW), o.x1 / UM_TW};     // tiles inside o (never ragged)
    tiles[l] = (o.empty() || t.empty()) ? TileRect{} : t;
    if (layers[l].pool) {
      // a pooled pixel is constant when its whole 2 x 2 window is
      o = TileRect{cdiv(o.y0, 2), o.y1 / 2, cdiv(o.x0, 2), o.x1 / 2};
      if (o.empty()) o = TileRect{};
      h /= 2; w /= 2;
    }
    px[l] = in = o;
  }
  // a computed tile of the second layer reads its rows and columns plus the halo
  *first_skip = TileRect{};
  if (n > 1 && !tiles[1].empty()) {
    const int halo = layers[1].ks / 2;
    const TileRect& t = tiles[1];
    const TileRect s{t.y0 * UM_TH + halo, t.y1 * UM_TH - halo, t.x0 * UM_TW + halo, t.x1 * UM_TW - halo};
    if (!s.empty()) *first_skip = s;
  }
}

// the arguments that follow from the layer and its input; the caller adds the output and the epilogue
static UmmaArgs umma_args(const UmmaLayer& L, int B, int H, int W, float act_scale) {
  UmmaArgs P = {};
  P.bias = L.bias; P.H = H; P.W = W; P.B = B; P.ks = L.ks; P.cin_slabs = L.cin / UM_KC;
  P.inv_scale = 1.0f / (act_scale * L.w_scale); P.n_split = 1;
  return P;
}

template <bool FP16>
static osb_status umma_conv_launch(const UmmaLayer& L, const CUtensorMap& a_hi, const CUtensorMap& a_lo, UmmaArgs& P,
                                   cudaStream_t st, int max_ctas) {
  const bool band = !P.band.empty();
  const bool res64 = L.n_pad == 64 && L.ks == 3 && L.cin == UM_KC;
  // conv_umma_kernel and the split layers have no band form
  OSB_REQUIRE(!band || res64 || L.n_pad == 128, "a constant band needs a 64 -> 64 3x3 or a 128-channel layer");
  switch (L.n_pad) {
    case 64:
      if (res64) {                                // weights resident, transposed GEMM
        if (band)
          return launch_persistent<conv_res64_kernel<FP16, true>>(R64Cfg<FP16>::SMEM_BYTES, a_hi, a_lo, L.tm_hi, L.tm_lo,
                                                                  P, st, max_ctas);
        return launch_persistent<conv_res64_kernel<FP16>>(R64Cfg<FP16>::SMEM_BYTES, a_hi, a_lo, L.tm_hi, L.tm_lo, P, st,
                                                          max_ctas);
      }
      return launch_umma<64, FP16>(a_hi, a_lo, L, P, st, max_ctas);
    case 80: return launch_umma<80, FP16>(a_hi, a_lo, L, P, st, max_ctas);
    case 128:
      if (band) return launch_stream_t<false, FP16, true>(a_hi, a_lo, L, P, st, max_ctas);
      return launch_stream_t<false, FP16>(a_hi, a_lo, L, P, st, max_ctas);
    case 256:                                     // 2 / 4 items of 128 channels per tile (a 256-wide accumulator pair
    case 512:                                     // would not fit a warpgroup's registers)
      P.n_split = L.n_pad / 128;
      return launch_stream_t<true, FP16>(a_hi, a_lo, L, P, st, max_ctas);
  }
  set_error("umma_conv_forward", "unsupported N");
  return OSB_ERR_INVALID;
}

osb_status umma_conv_forward(const UmmaLayer& L, const CUtensorMap& a_hi, const CUtensorMap& a_lo, int B, int H, int W,
                             float act_scale, __half* out_hi, __half* out_lo, float* out_f32, int out_c, int out_cstride,
                             float out_scale, int relu, int pool, cudaStream_t st, int max_ctas, int precision,
                             const ConvBand* band) {
  OSB_REQUIRE(!pool || (H % 2 == 0 && W % 2 == 0), "fused max-pool needs even H and W");
  OSB_REQUIRE(out_c % 16 == 0 && out_c <= L.n_pad && out_cstride % 8 == 0, "tensor-core conv: bad output channel layout");
  UmmaArgs P = umma_args(L, B, H, W, act_scale);
  P.out_hi = out_hi; P.out_lo = out_lo; P.out_f32 = out_f32; P.out_c = out_c; P.out_cstride = out_cstride;
  P.out_scale = out_scale; P.relu = relu; P.pool = pool;
  if (band && !band->tiles.empty()) {
    const TileRect& t = band->tiles;
    OSB_REQUIRE(out_hi && !out_f32 && band->hi && (band->lo || precision_fp16(precision)),
                "a constant band is stored into split planes");
    OSB_REQUIRE(t.y0 >= 0 && t.x0 >= 0 && t.y1 * UM_TH <= H && t.x1 * UM_TW <= W, "band tiles outside the image");
    OSB_REQUIRE((int64_t)B * t.y1 * UM_TH * t.x1 * UM_TW * (out_c / 8) < INT32_MAX, "band too large");
    P.band = t; P.band_hi = band->hi; P.band_lo = band->lo;
  }
  return precision_fp16(precision) ? umma_conv_launch<true>(L, a_hi, a_lo, P, st, max_ctas)
                                   : umma_conv_launch<false>(L, a_hi, a_lo, P, st, max_ctas);
}

// detector head: convPb (256 -> 65, 1x1) with the softmax + 8x8 pixel shuffle fused into the epilogue; `semi` is the heat
// map [B][8H][8W]
osb_status umma_conv_softmax_forward(const UmmaLayer& L, const CUtensorMap& a_hi, const CUtensorMap& a_lo, int B, int H, int W,
                                     float act_scale, float* semi, cudaStream_t st, int max_ctas, int precision) {
  OSB_REQUIRE(L.n_pad == 80 && L.cout == 65 && L.ks == 1, "fused detector head expects the 65-logit 1x1 layer");
  UmmaArgs P = umma_args(L, B, H, W, act_scale);
  P.out_f32 = semi; P.out_c = 80; P.out_cstride = 80; P.out_scale = 1.f; P.epi = 1;
  return precision_fp16(precision) ? launch_umma<80, true>(a_hi, a_lo, L, P, st, max_ctas)
                                   : launch_umma<80>(a_hi, a_lo, L, P, st, max_ctas);
}

// depthwise 3x3 (pad 1, stride s) + bias + ReLU6 on fp32 NHWC input, output as split fp16 planes for the pointwise
// tensor-core conv that follows; one thread per (output pixel, 8 channels)
template <bool FP16 = false>
__global__ void dwconv3x3_split_kernel(const float* __restrict__ w, const float* __restrict__ bias,
                                       const float* __restrict__ x, __half* __restrict__ out_hi,
                                       __half* __restrict__ out_lo, int H, int W, int Ho, int Wo, int C, int stride,
                                       float out_scale, int64_t total) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int C8 = C >> 3;
  const int c = (int)(i % C8) * 8;
  int64_t p = i / C8;
  const int ox = (int)(p % Wo); p /= Wo;
  const int oy = (int)(p % Ho);
  const int b = (int)(p / Ho);
  float a[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) a[j] = 0.f;
#pragma unroll
  for (int ky = 0; ky < 3; ++ky)
#pragma unroll
    for (int kx = 0; kx < 3; ++kx) {
      const int gy = oy * stride + ky - 1, gx = ox * stride + kx - 1;
      if (gy < 0 || gy >= H || gx < 0 || gx >= W) continue;
      const float4* xp = reinterpret_cast<const float4*>(x + (((size_t)b * H + gy) * W + gx) * C + c);
      const float4* wp = reinterpret_cast<const float4*>(w + (size_t)(ky * 3 + kx) * C + c);
      const float4 v0 = xp[0], v1 = xp[1], w0 = wp[0], w1 = wp[1];
      a[0] = fmaf(v0.x, w0.x, a[0]); a[1] = fmaf(v0.y, w0.y, a[1]); a[2] = fmaf(v0.z, w0.z, a[2]); a[3] = fmaf(v0.w, w0.w, a[3]);
      a[4] = fmaf(v1.x, w1.x, a[4]); a[5] = fmaf(v1.y, w1.y, a[5]); a[6] = fmaf(v1.z, w1.z, a[6]); a[7] = fmaf(v1.w, w1.w, a[7]);
    }
#pragma unroll
  for (int j = 0; j < 8; ++j) a[j] = fminf(fmaxf(a[j] + bias[c + j], 0.f), 6.f);
  split_store8<FP16>(out_hi + (size_t)i * 8, out_lo + (size_t)i * 8, a, out_scale);
}

// stride-1 variant: one thread per (4 consecutive output pixels of a row, 8 channels).  The 3 x 6 input window is read
// once (36 float4 instead of 72 for four single-pixel threads) and the 9 x 8 weights once per thread; same tap order per
// output as the kernel above, so the planes are bit-identical.
template <bool FP16 = false>
__global__ void dwconv3x3_split_s1x4_kernel(const float* __restrict__ w, const float* __restrict__ bias,
                                            const float* __restrict__ x, __half* __restrict__ out_hi,
                                            __half* __restrict__ out_lo, int H, int W, int C, float out_scale,
                                            int64_t total) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int C8 = C >> 3, Wg = (W + 3) >> 2;
  const int c = (int)(i % C8) * 8;
  int64_t p = i / C8;
  const int ox0 = (int)(p % Wg) * 4; p /= Wg;
  const int oy = (int)(p % H);
  const int b = (int)(p / H);
  float4 wv[9][2];
#pragma unroll
  for (int t = 0; t < 9; ++t) {
    const float4* wp = reinterpret_cast<const float4*>(w + (size_t)t * C + c);
    wv[t][0] = __ldg(wp); wv[t][1] = __ldg(wp + 1);
  }
  float a[4][8];
#pragma unroll
  for (int q = 0; q < 4; ++q)
#pragma unroll
    for (int j = 0; j < 8; ++j) a[q][j] = 0.f;
#pragma unroll
  for (int ky = 0; ky < 3; ++ky) {
    const int gy = oy + ky - 1;
    if (gy < 0 || gy >= H) continue;
    float4 v[6][2];
#pragma unroll
    for (int cx = 0; cx < 6; ++cx) {
      const int gx = ox0 + cx - 1;
      if (gx >= 0 && gx < W) {
        const float4* xp = reinterpret_cast<const float4*>(x + (((size_t)b * H + gy) * W + gx) * C + c);
        v[cx][0] = xp[0]; v[cx][1] = xp[1];
      } else {
        v[cx][0] = v[cx][1] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
#pragma unroll
    for (int q = 0; q < 4; ++q)
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const int gx = ox0 + q + kx - 1;
        if (gx < 0 || gx >= W) continue;              // (skipped like the single-pixel kernel: no +0 added)
        const float4 v0 = v[q + kx][0], v1 = v[q + kx][1], w0 = wv[ky * 3 + kx][0], w1 = wv[ky * 3 + kx][1];
        a[q][0] = fmaf(v0.x, w0.x, a[q][0]); a[q][1] = fmaf(v0.y, w0.y, a[q][1]);
        a[q][2] = fmaf(v0.z, w0.z, a[q][2]); a[q][3] = fmaf(v0.w, w0.w, a[q][3]);
        a[q][4] = fmaf(v1.x, w1.x, a[q][4]); a[q][5] = fmaf(v1.y, w1.y, a[q][5]);
        a[q][6] = fmaf(v1.z, w1.z, a[q][6]); a[q][7] = fmaf(v1.w, w1.w, a[q][7]);
      }
  }
  float bb[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) bb[j] = __ldg(bias + c + j);
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int ox = ox0 + q;
    if (ox >= W) break;
#pragma unroll
    for (int j = 0; j < 8; ++j) a[q][j] = fminf(fmaxf(a[q][j] + bb[j], 0.f), 6.f);
    const size_t o = ((((size_t)b * H + oy) * W + ox) * C8 + (c >> 3)) * 8;
    split_store8<FP16>(out_hi + o, out_lo + o, a[q], out_scale);
  }
}

osb_status umma_dwconv_forward(const float* w_tap_c, const float* bias, const float* x, __half* out_hi, __half* out_lo,
                               int B, int H, int W, int C, int stride, float out_scale, cudaStream_t st, bool s1x4,
                               int precision) {
  const int Ho = H / stride, Wo = W / stride;
  const bool fp16 = precision_fp16(precision);
  if (stride == 1 && s1x4) {
    const int64_t total4 = (int64_t)B * H * ((W + 3) / 4) * (C / 8);
    const auto kernel = fp16 ? dwconv3x3_split_s1x4_kernel<true> : dwconv3x3_split_s1x4_kernel<false>;
    OSB_LAUNCH(kernel, (unsigned)cdiv64(total4, 128), 128, 0, st, w_tap_c, bias, x, out_hi, out_lo, H, W, C, out_scale,
               total4);
    OSB_CHECK_LAUNCH();
    return OSB_OK;
  }
  const int64_t total = (int64_t)B * Ho * Wo * (C / 8);
  const auto kernel = fp16 ? dwconv3x3_split_kernel<true> : dwconv3x3_split_kernel<false>;
  OSB_LAUNCH(kernel, (unsigned)cdiv64(total, 256), 256, 0, st, w_tap_c, bias, x, out_hi, out_lo, H, W, Ho, Wo, C, stride,
             out_scale, total);
  OSB_CHECK_LAUNCH();
  return OSB_OK;
}

osb_status umma_first_forward(const float* w_tap_cout, const float* bias, const float* lut, const uint8_t* img,
                              __half* out_hi, __half* out_lo, int B, int H, int W, float out_scale, cudaStream_t st,
                              int precision, TileRect skip) {
  dim3 grid(cdiv(W, CF_TW), cdiv(H, CF_TH), B);
  const auto kernel = precision_fp16(precision) ? conv_first_split_kernel<true> : conv_first_split_kernel<false>;
  OSB_LAUNCH(kernel, grid, 256, 0, st, w_tap_cout, bias, lut, img, out_hi, out_lo, H, W, out_scale, skip);
  OSB_CHECK_LAUNCH();
  return OSB_OK;
}

}  // namespace osb

// --------------------------------------------------------------------------------------------------------------
// parity hooks: one layer of the networks' tensor-core path on caller-supplied operands (tests only)
// --------------------------------------------------------------------------------------------------------------
using namespace osb;

// the hooks below share these bodies; in plain fp16 (OSB_PRECISION_FP16) in_lo / out_lo are never read or written, and
// the lo activation map is made over the hi plane
static osb_status conv_layer_hook(const float* w, const float* bias, int cin, int cout, int ks, float w_scale,
                                  const void* in_hi, const void* in_lo, int batch, int height, int width, float act_scale,
                                  int relu, int pool, int out_c, int out_cstride, int max_ctas, int mode, float* out_f32,
                                  void* out_hi, void* out_lo, float out_scale, void* stream, int precision) {
  OSB_TRY(require_device());
  const cudaStream_t st = (cudaStream_t)stream;
  Resources res;
  res.sync_before_release(st);
  UmmaLayer L;
  CUtensorMap a_hi, a_lo;
  OSB_TRY(umma_layer_upload(res, &L, w, bias, cin, cout, ks, w_scale));
  OSB_TRY(umma_act_maps(&a_hi, &a_lo, (__half*)in_hi, (__half*)in_lo, batch, height, width, cin, ks));
  if (mode == 2)
    OSB_TRY(umma_conv_softmax_forward(L, a_hi, a_lo, batch, height, width, act_scale, out_f32, st, max_ctas, precision));
  else
    OSB_TRY(umma_conv_forward(L, a_hi, a_lo, batch, height, width, act_scale, mode == 1 ? (__half*)out_hi : nullptr,
                              mode == 1 ? (__half*)out_lo : nullptr, mode == 0 ? out_f32 : nullptr, out_c, out_cstride,
                              out_scale, relu, pool, st, max_ctas, precision));
  OSB_CUDA(cudaStreamSynchronize(st));
  return OSB_OK;
}

static osb_status conv_first_hook(const float* w1a, const float* b1a, const uint8_t* images_dev, int batch, int height,
                                  int width, float act_scale, void* out_hi, void* out_lo, void* stream, int precision) {
  OSB_TRY(require_device());
  const cudaStream_t st = (cudaStream_t)stream;
  Resources res;
  res.sync_before_release(st);
  float *wd = nullptr, *bd = nullptr, *lut = nullptr;
  std::vector<float> l(256);
  for (int v = 0; v < 256; ++v) l[v] = (float)v * (float)(1.0 / 255.0);
  OSB_TRY(upload_tap_major(res, &wd, w1a, 64));
  OSB_TRY(res.upload(&bd, b1a, 64));
  OSB_TRY(res.upload(&lut, l.data(), 256));
  OSB_TRY(umma_first_forward(wd, bd, lut, images_dev, (__half*)out_hi, (__half*)out_lo, batch, height, width, act_scale, st,
                             precision));
  OSB_CUDA(cudaStreamSynchronize(st));
  return OSB_OK;
}

static osb_status dwconv_hook(const float* w, const float* bias, const float* x_dev, int batch, int height, int width,
                              int channels, int stride, int generic, float out_scale, void* out_hi, void* out_lo,
                              void* stream, int precision) {
  OSB_REQUIRE(batch > 0 && height > 0 && width > 0 && channels > 0 && channels % 8 == 0 && (stride == 1 || stride == 2),
              "bad geometry (channels must be a multiple of 8, stride 1 or 2)");
  OSB_TRY(require_device());
  const cudaStream_t st = (cudaStream_t)stream;
  Resources res;
  res.sync_before_release(st);
  float *wd = nullptr, *bd = nullptr;
  OSB_TRY(upload_tap_major(res, &wd, w, channels));
  OSB_TRY(res.upload(&bd, bias, channels));
  OSB_TRY(umma_dwconv_forward(wd, bd, x_dev, (__half*)out_hi, (__half*)out_lo, batch, height, width, channels, stride,
                              out_scale, st, !generic, precision));
  OSB_CUDA(cudaStreamSynchronize(st));
  return OSB_OK;
}

extern "C" osb_status osb_conv_layer_parity(const float* w, const float* bias, int cin, int cout, int ks, float w_scale,
                                            const void* in_hi, const void* in_lo, int batch, int height, int width,
                                            float act_scale, int relu, int pool, int out_c, int out_cstride, int max_ctas,
                                            int mode, float* out_f32, void* out_hi, void* out_lo, float out_scale,
                                            void* stream) {
  OSB_REQUIRE(w && bias && in_hi && in_lo, "null argument");
  OSB_REQUIRE(batch > 0 && height > 0 && width > 0 && (ks == 1 || ks == 3), "bad geometry");
  OSB_REQUIRE(relu >= 0 && relu <= 2 && mode >= 0 && mode <= 2, "relu must be 0..2, mode 0 (fp32), 1 (planes) or 2 (softmax)");
  OSB_REQUIRE(mode == 1 ? (out_hi && out_lo) : (out_f32 != nullptr), "null output");
  return conv_layer_hook(w, bias, cin, cout, ks, w_scale, in_hi, in_lo, batch, height, width, act_scale, relu, pool, out_c,
                         out_cstride, max_ctas, mode, out_f32, out_hi, out_lo, out_scale, stream, OSB_PRECISION_SPLIT_FP16);
}

extern "C" osb_status osb_conv_layer_fp16_parity(const float* w, const float* bias, int cin, int cout, int ks,
                                                 float w_scale, const void* in_hi, int batch, int height, int width,
                                                 float act_scale, int relu, int pool, int out_c, int out_cstride,
                                                 int max_ctas, int mode, float* out_f32, void* out_hi, float out_scale,
                                                 void* stream) {
  OSB_REQUIRE(w && bias && in_hi, "null argument");
  OSB_REQUIRE(batch > 0 && height > 0 && width > 0 && (ks == 1 || ks == 3), "bad geometry");
  OSB_REQUIRE(relu >= 0 && relu <= 2 && mode >= 0 && mode <= 2, "relu must be 0..2, mode 0 (fp32), 1 (planes) or 2 (softmax)");
  OSB_REQUIRE(mode == 1 ? (out_hi != nullptr) : (out_f32 != nullptr), "null output");
  return conv_layer_hook(w, bias, cin, cout, ks, w_scale, in_hi, in_hi, batch, height, width, act_scale, relu, pool, out_c,
                         out_cstride, max_ctas, mode, out_f32, out_hi, nullptr, out_scale, stream, OSB_PRECISION_FP16);
}

extern "C" osb_status osb_conv_first_parity(const float* w1a, const float* b1a, const uint8_t* images_dev, int batch,
                                            int height, int width, float act_scale, void* out_hi, void* out_lo,
                                            void* stream) {
  OSB_REQUIRE(w1a && b1a && images_dev && out_hi && out_lo, "null argument");
  OSB_REQUIRE(batch > 0 && height > 0 && width > 0, "bad geometry");
  return conv_first_hook(w1a, b1a, images_dev, batch, height, width, act_scale, out_hi, out_lo, stream,
                         OSB_PRECISION_SPLIT_FP16);
}

extern "C" osb_status osb_conv_first_fp16_parity(const float* w1a, const float* b1a, const uint8_t* images_dev, int batch,
                                                 int height, int width, float act_scale, void* out_hi, void* stream) {
  OSB_REQUIRE(w1a && b1a && images_dev && out_hi, "null argument");
  OSB_REQUIRE(batch > 0 && height > 0 && width > 0, "bad geometry");
  return conv_first_hook(w1a, b1a, images_dev, batch, height, width, act_scale, out_hi, nullptr, stream, OSB_PRECISION_FP16);
}

extern "C" osb_status osb_dwconv_parity(const float* w, const float* bias, const float* x_dev, int batch, int height,
                                        int width, int channels, int stride, int generic, float out_scale, void* out_hi,
                                        void* out_lo, void* stream) {
  OSB_REQUIRE(w && bias && x_dev && out_hi && out_lo, "null argument");
  return dwconv_hook(w, bias, x_dev, batch, height, width, channels, stride, generic, out_scale, out_hi, out_lo, stream,
                     OSB_PRECISION_SPLIT_FP16);
}

extern "C" osb_status osb_dwconv_fp16_parity(const float* w, const float* bias, const float* x_dev, int batch, int height,
                                             int width, int channels, int stride, int generic, float out_scale,
                                             void* out_hi, void* stream) {
  OSB_REQUIRE(w && bias && x_dev && out_hi, "null argument");
  return dwconv_hook(w, bias, x_dev, batch, height, width, channels, stride, generic, out_scale, out_hi, nullptr, stream,
                     OSB_PRECISION_FP16);
}
