// netvlad.cu -- osb_netvlad: replacement of class MobileNetVLADTensorRT
// (swarm_loop/include/swarm_loop/mobilenetvlad_tensorrt.h:10-21, swarm_loop/src/mobilenetvlad_tensorrt.cpp:4-15).
// The reference only fixes the I/O contract (HxW float 0..255 in, 4096 floats out); the hfnet MobileNetVLAD
// architecture is not in the repository.  The stand-in pinned here (and in oracle/frontend_ref.py::netvlad_net):
//   conv0 3x3 s2 1->32 ReLU6 | 7 x [depthwise 3x3 (s) ReLU6 + pointwise 1x1 ReLU6] -> 512 ch at 1/16 resolution |
//   1x1 projection to D=128, per-image centring (x - mean over locations), per-location L2 norm | NetVLAD K=32: soft-assign (1x1 conv + softmax),
//   residual aggregation, intra-normalisation, flatten (K*D = 4096), L2 norm.
#include "superpoint.cuh"
#include <stdlib.h>

namespace osb {

constexpr float NV_ACT_SCALE = 16.f;     // ReLU6 activations (<= 6) as split fp16 planes
constexpr float NV_W_SCALE = 1024.f;

static const int NVB_CIN[7] = {32, 64, 128, 128, 256, 256, 512};
static const int NVB_COUT[7] = {64, 128, 128, 256, 256, 512, 512};
static const int NVB_STRIDE[7] = {1, 2, 1, 2, 1, 2, 1};
constexpr int NV_K = 32, NV_D = 128;

size_t nv_expected_weights() {
  size_t n = 32 * 9 + 32;
  for (int i = 0; i < 7; ++i) n += (size_t)NVB_CIN[i] * 9 + NVB_CIN[i] + (size_t)NVB_COUT[i] * NVB_CIN[i] + NVB_COUT[i];
  n += (size_t)NV_D * 512 + NV_D + (size_t)NV_K * NV_D + NV_K + (size_t)NV_K * NV_D;
  return n;
}

// softmax over K=32 assignment logits of every location, in place; one thread per location
__global__ void nv_softmax_kernel(float* __restrict__ a, int64_t locs) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= locs) return;
  float* p = a + (size_t)i * NV_K;
  float v[NV_K];
  float m = -INFINITY;
#pragma unroll
  for (int k = 0; k < NV_K; ++k) { v[k] = p[k]; m = fmaxf(m, v[k]); }
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < NV_K; ++k) { v[k] = expf(v[k] - m); s += v[k]; }
#pragma unroll
  for (int k = 0; k < NV_K; ++k) p[k] = v[k] / s;
}

// per-image, per-channel mean of the projected features over all locations (instance centring): thread = channel
__global__ void __launch_bounds__(NV_D)
nv_colmean_kernel(const float* __restrict__ x, int P, float* __restrict__ mu) {
  const int b = blockIdx.x, ch = threadIdx.x;
  const float* xb = x + (size_t)b * P * NV_D;
  float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
  int p = 0;
  for (; p + 3 < P; p += 4) {
    s0 += xb[(size_t)p * NV_D + ch]; s1 += xb[(size_t)(p + 1) * NV_D + ch];
    s2 += xb[(size_t)(p + 2) * NV_D + ch]; s3 += xb[(size_t)(p + 3) * NV_D + ch];
  }
  for (; p < P; ++p) s0 += xb[(size_t)p * NV_D + ch];
  mu[b * NV_D + ch] = ((s0 + s1) + (s2 + s3)) / (float)P;
}

// x <- (x - mu[image]) / ||x - mu[image]||_2 per location; one warp per location, lane = 4 channels
__global__ void nv_center_norm_kernel(float* __restrict__ x, const float* __restrict__ mu, int P, int64_t locs) {
  const int64_t loc = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (loc >= locs) return;
  const int b = (int)(loc / P);
  float4 v = reinterpret_cast<float4*>(x + (size_t)loc * NV_D)[lane];
  const float4 m = reinterpret_cast<const float4*>(mu + (size_t)b * NV_D)[lane];
  v.x -= m.x; v.y -= m.y; v.z -= m.z; v.w -= m.w;
  float s = v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  s = warp_sum(s);
  const float n = fmaxf(sqrtf(s), 1e-12f);       // eps as in F.normalize: a blank image centres to exactly zero
  v.x /= n; v.y /= n; v.z /= n; v.w /= n;
  reinterpret_cast<float4*>(x + (size_t)loc * NV_D)[lane] = v;
}

// VLAD aggregation, stage 1: grid (image, slice); warp = cluster k, lane = 4 dims; partial sums over a slice of the
// locations (fixed partition -> deterministic), written to part[b][slice][k][d] and psum[b][slice][k]
constexpr int NV_SLICES = 8;
__global__ void __launch_bounds__(1024)
nv_vlad_partial_kernel(const float* __restrict__ x, const float* __restrict__ a, int P, float* __restrict__ part,
                       float* __restrict__ psum) {
  const int b = blockIdx.x, sl = blockIdx.y, k = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int per = (P + NV_SLICES - 1) / NV_SLICES;
  const int p0 = sl * per, p1 = min(P, p0 + per);
  const float* xb = x + (size_t)b * P * NV_D;
  const float* ab = a + (size_t)b * P * NV_K;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  float asum = 0.f;
#pragma unroll 4
  for (int p = p0; p < p1; ++p) {
    const float w = __ldg(ab + (size_t)p * NV_K + k);
    const float4 v = __ldg(reinterpret_cast<const float4*>(xb + (size_t)p * NV_D) + lane);
    acc.x = fmaf(w, v.x, acc.x); acc.y = fmaf(w, v.y, acc.y);
    acc.z = fmaf(w, v.z, acc.z); acc.w = fmaf(w, v.w, acc.w);
    asum += w;
  }
  reinterpret_cast<float4*>(part + (((size_t)b * NV_SLICES + sl) * NV_K + k) * NV_D)[lane] = acc;
  if (lane == 0) psum[((size_t)b * NV_SLICES + sl) * NV_K + k] = asum;
}

// stage 2: sum the slices, subtract asum * centroid, intra-normalise, flatten, L2-normalise; one CTA per image
__global__ void __launch_bounds__(1024)
nv_vlad_final_kernel(const float* __restrict__ part, const float* __restrict__ psum, const float* __restrict__ cent,
                     float* __restrict__ out) {
  __shared__ float red[32];
  const int b = blockIdx.x, k = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  float asum = 0.f;
  for (int sl = 0; sl < NV_SLICES; ++sl) {
    const float4 v = reinterpret_cast<const float4*>(part + (((size_t)b * NV_SLICES + sl) * NV_K + k) * NV_D)[lane];
    acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    asum += psum[((size_t)b * NV_SLICES + sl) * NV_K + k];
  }
  const float4 c = reinterpret_cast<const float4*>(cent + (size_t)k * NV_D)[lane];
  acc.x -= asum * c.x; acc.y -= asum * c.y; acc.z -= asum * c.z; acc.w -= asum * c.w;
  float s = acc.x * acc.x + acc.y * acc.y + acc.z * acc.z + acc.w * acc.w;
  s = warp_sum(s);
  const float n = fmaxf(sqrtf(s), 1e-12f);
  acc.x /= n; acc.y /= n; acc.z /= n; acc.w /= n;                  // intra-normalisation
  float t = acc.x * acc.x + acc.y * acc.y + acc.z * acc.z + acc.w * acc.w;
  t = warp_sum(t);
  if (lane == 0) red[k] = t;
  __syncthreads();
  float tot = red[lane];
  tot = warp_sum(tot);
  const float g = fmaxf(sqrtf(tot), 1e-12f);
  acc.x /= g; acc.y /= g; acc.z /= g; acc.w /= g;
  reinterpret_cast<float4*>(out + (size_t)b * NV_K * NV_D + (size_t)k * NV_D)[lane] = acc;
}

// Block 0 fused: depthwise 3x3 (32 ch, stride 1) + ReLU6 -> pointwise 32 -> 64 + ReLU6, fp32 in / fp32 out.
// The pointwise layer has K = 32, half a tensor-core slab, and as a generic tiled GEMM it was the slowest launch of the
// network (75 us for 1.3 GFLOP); fused, the depthwise output never leaves shared memory.  CTA = 8 x 16 pixels:
// (1) input tile + halo -> shared memory, (2) depthwise: thread = (4 channels, pixel), its 9 x 4 weights in registers,
// (3) pointwise: thread = 4 pixels x 8 output channels, K = 32 from shared memory (padded rows, broadcast reads).
constexpr int F0_TW = 16, F0_TH = 8, F0_C = 32, F0_OC = 64, F0_PX = F0_TW * F0_TH;
constexpr int F0_SMEM = ((F0_TH + 2) * (F0_TW + 2) * F0_C + F0_PX * (F0_C + 1) + F0_C * F0_OC) * (int)sizeof(float);
__global__ void __launch_bounds__(256)
nv_block0_fused_kernel(const float* __restrict__ x, const float* __restrict__ dw_w, const float* __restrict__ dw_b,
                       const float* __restrict__ pw_kc, const float* __restrict__ pw_b, float* __restrict__ y, int H,
                       int W) {
  extern __shared__ __align__(16) float f0_smem[];
  float* s_in = f0_smem;                                               // [TH+2][TW+2][32]
  float* s_dw = s_in + (F0_TH + 2) * (F0_TW + 2) * F0_C;               // [128][33]
  float* s_w = s_dw + F0_PX * (F0_C + 1);                              // [32][64]
  const int tid = threadIdx.x, b = blockIdx.z, x0 = blockIdx.x * F0_TW, y0 = blockIdx.y * F0_TH;
  const float* xb = x + (size_t)b * H * W * F0_C;
  for (int e = tid; e < (F0_TH + 2) * (F0_TW + 2) * (F0_C / 4); e += 256) {
    const int c4 = e % (F0_C / 4), pc = (e / (F0_C / 4)) % (F0_TW + 2), pr = e / ((F0_C / 4) * (F0_TW + 2));
    const int gy = y0 + pr - 1, gx = x0 + pc - 1;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (gy >= 0 && gy < H && gx >= 0 && gx < W) v = __ldg(reinterpret_cast<const float4*>(xb + ((size_t)gy * W + gx) * F0_C) + c4);
    reinterpret_cast<float4*>(s_in)[e] = v;
  }
  for (int e = tid; e < F0_C * F0_OC / 4; e += 256) reinterpret_cast<float4*>(s_w)[e] = __ldg(reinterpret_cast<const float4*>(pw_kc) + e);
  // depthwise weights of this thread's 4 channels
  const int cg = tid & 7, slot = tid >> 3;
  float4 wd[9];
#pragma unroll
  for (int t = 0; t < 9; ++t) wd[t] = __ldg(reinterpret_cast<const float4*>(dw_w + t * F0_C) + cg);
  const float4 bd = __ldg(reinterpret_cast<const float4*>(dw_b) + cg);
  __syncthreads();
#pragma unroll
  for (int j = 0; j < F0_PX / 32; ++j) {
    const int px = slot + 32 * j, r = px / F0_TW, c = px % F0_TW;
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int ky = 0; ky < 3; ++ky)
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const float4 v = reinterpret_cast<const float4*>(s_in + ((r + ky) * (F0_TW + 2) + c + kx) * F0_C)[cg];
        const float4 ww = wd[ky * 3 + kx];
        a.x = fmaf(v.x, ww.x, a.x); a.y = fmaf(v.y, ww.y, a.y); a.z = fmaf(v.z, ww.z, a.z); a.w = fmaf(v.w, ww.w, a.w);
      }
    float* d = s_dw + px * (F0_C + 1) + cg * 4;
    d[0] = fminf(fmaxf(a.x + bd.x, 0.f), 6.f); d[1] = fminf(fmaxf(a.y + bd.y, 0.f), 6.f);
    d[2] = fminf(fmaxf(a.z + bd.z, 0.f), 6.f); d[3] = fminf(fmaxf(a.w + bd.w, 0.f), 6.f);
  }
  __syncthreads();
  // pointwise: 4 pixels x 8 output channels per thread
  const int ocg = tid & 7, pxg = tid >> 3;
  float acc[4][8];
#pragma unroll
  for (int j = 0; j < 4; ++j)
#pragma unroll
    for (int o = 0; o < 8; ++o) acc[j][o] = 0.f;
#pragma unroll 8
  for (int k = 0; k < F0_C; ++k) {
    const float4 w0 = reinterpret_cast<const float4*>(s_w + k * F0_OC + ocg * 8)[0];
    const float4 w1 = reinterpret_cast<const float4*>(s_w + k * F0_OC + ocg * 8)[1];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float av = s_dw[(pxg * 4 + j) * (F0_C + 1) + k];
      acc[j][0] = fmaf(av, w0.x, acc[j][0]); acc[j][1] = fmaf(av, w0.y, acc[j][1]);
      acc[j][2] = fmaf(av, w0.z, acc[j][2]); acc[j][3] = fmaf(av, w0.w, acc[j][3]);
      acc[j][4] = fmaf(av, w1.x, acc[j][4]); acc[j][5] = fmaf(av, w1.y, acc[j][5]);
      acc[j][6] = fmaf(av, w1.z, acc[j][6]); acc[j][7] = fmaf(av, w1.w, acc[j][7]);
    }
  }
  const float4 b0v = __ldg(reinterpret_cast<const float4*>(pw_b + ocg * 8)), b1v = __ldg(reinterpret_cast<const float4*>(pw_b + ocg * 8) + 1);
  const float bb[8] = {b0v.x, b0v.y, b0v.z, b0v.w, b1v.x, b1v.y, b1v.z, b1v.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int px = pxg * 4 + j, gy = y0 + px / F0_TW, gx = x0 + px % F0_TW;
    if (gy >= H || gx >= W) continue;
    float o[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) o[q] = fminf(fmaxf(acc[j][q] + bb[q], 0.f), 6.f);
    float4* dst = reinterpret_cast<float4*>(y + (((size_t)b * H + gy) * W + gx) * F0_OC + ocg * 8);
    dst[0] = make_float4(o[0], o[1], o[2], o[3]);
    dst[1] = make_float4(o[4], o[5], o[6], o[7]);
  }
}

static osb_status copy_dev(float* dst, const float* src, size_t n, cudaStream_t st) {
  OSB_CUDA(cudaMemcpyAsync(dst, src, n * sizeof(float), cudaMemcpyDeviceToDevice, st));
  return OSB_OK;
}

static osb_status nv_block0_prepare() {
  OSB_CUDA(cudaFuncSetAttribute(nv_block0_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, F0_SMEM));
  return OSB_OK;
}

// block 0 of the tensor-core path: x fp32 [B][h][w][32] -> y fp32 [B][h][w][64]; dw_tap_c [9][32], pw_kc [32][64]
static osb_status nv_block0_forward(const float* x, const float* dw_tap_c, const float* dw_b, const float* pw_kc,
                                    const float* pw_b, float* y, int B, int h, int w, cudaStream_t st) {
  dim3 grid(cdiv(w, F0_TW), cdiv(h, F0_TH), B);
  OSB_LAUNCH(nv_block0_fused_kernel, grid, 256, F0_SMEM, st, x, dw_tap_c, dw_b, pw_kc, pw_b, y, h, w);
  OSB_CHECK_LAUNCH();
  return OSB_OK;
}

// The head, from the projected features x fp32 [B][h][w][D]: per-image mean mu [B][D]; x centred and L2-normalised per
// location IN PLACE; soft-assignment a [B][h][w][K] (logits, then softmax in place; when logits_copy is not null the
// logits are copied there first); VLAD partial sums part / psum, and the 4096-vector out [B][K*D].
static osb_status nv_head_forward(const ConvLayer& assign, const float* centroids, float* x, int B, int h, int w,
                                  float* mu, float* a, float* part, float* psum, float* out, cudaStream_t st,
                                  float* logits_copy = nullptr) {
  const int P = h * w;
  const int64_t locs = (int64_t)B * P;
  OSB_LAUNCH(nv_colmean_kernel, B, NV_D, 0, st, x, P, mu);
  OSB_CHECK_LAUNCH();
  OSB_LAUNCH(nv_center_norm_kernel, (unsigned)cdiv64(locs * 32, 256), 256, 0, st, x, mu, P, locs);
  OSB_CHECK_LAUNCH();
  osb_status s = conv_forward(assign, x, a, B, h, w, NV_K, ACT_NONE, st);
  if (s != OSB_OK) return s;
  if (logits_copy && (s = copy_dev(logits_copy, a, (size_t)locs * NV_K, st)) != OSB_OK) return s;
  OSB_LAUNCH(nv_softmax_kernel, (unsigned)cdiv64(locs, 128), 128, 0, st, a, locs);
  OSB_CHECK_LAUNCH();
  OSB_LAUNCH(nv_vlad_partial_kernel, dim3(B, NV_SLICES), 1024, 0, st, x, a, P, part, psum);
  OSB_CHECK_LAUNCH();
  OSB_LAUNCH(nv_vlad_final_kernel, B, 1024, 0, st, part, psum, centroids, out);
  OSB_CHECK_LAUNCH();
  return OSB_OK;
}

osb_status NetVLAD::init(const float* weights, size_t n_weights, int width, int height, int max_batch_) {
  OSB_REQUIRE(weights != nullptr, "null weights");
  OSB_REQUIRE(n_weights == nv_expected_weights(), "weight blob has the wrong length (expected 607968 floats)");
  OSB_REQUIRE(width % 16 == 0 && height % 16 == 0 && width > 0 && height > 0, "width/height must be multiples of 16");
  W = width; H = height; max_batch = max_batch_;
  OSB_TRY(res.stream(&stream));
  {
    const char* e = getenv("OSB_SP_CONV");      // same debug switch as SuperPoint: ffma = fp32 CUDA-core pointwise convs
    use_umma = !(e && strcmp(e, "ffma") == 0);
  }
  const float* p = weights;
  {
    std::vector<float> w9(9 * 32);
    for (int o = 0; o < 32; ++o)
      for (int t = 0; t < 9; ++t) w9[t * 32 + o] = p[o * 9 + t];
    OSB_TRY(res.upload(&w0, w9.data(), 9 * 32));
    OSB_TRY(res.upload(&b0, p + 32 * 9, 32));
    p += 32 * 9 + 32;
  }
  for (int i = 0; i < 7; ++i) {
    const int ci = NVB_CIN[i], co = NVB_COUT[i];
    blk[i].cin = ci; blk[i].cout = co; blk[i].stride = NVB_STRIDE[i];
    std::vector<float> dw((size_t)9 * ci);
    for (int c = 0; c < ci; ++c)
      for (int t = 0; t < 9; ++t) dw[(size_t)t * ci + c] = p[(size_t)c * 9 + t];
    OSB_TRY(res.upload(&blk[i].dw, dw.data(), dw.size()));
    p += (size_t)ci * 9;
    OSB_TRY(res.upload(&blk[i].dwb, p, ci));
    p += ci;
    OSB_TRY(conv_layer_upload(res, &blk[i].pw, p, p + (size_t)co * ci, ci, co, 1));
    if (i == 0) {                                  // block 0 fused kernel: pointwise weights as [k][oc]
      std::vector<float> kc((size_t)ci * co);
      for (int o = 0; o < co; ++o)
        for (int k = 0; k < ci; ++k) kc[(size_t)k * co + o] = p[(size_t)o * ci + k];
      OSB_TRY(res.upload(&pw0_kc, kc.data(), kc.size()));
      OSB_TRY(res.upload(&pw0_b, p + (size_t)co * ci, co));
      OSB_TRY(nv_block0_prepare());
    }
    if (use_umma && i >= 1) OSB_TRY(umma_layer_upload(res, &upw[i], p, p + (size_t)co * ci, ci, co, 1, NV_W_SCALE));
    p += (size_t)co * ci + co;
  }
  OSB_TRY(conv_layer_upload(res, &proj, p, p + (size_t)NV_D * 512, 512, NV_D, 1));
  if (use_umma) OSB_TRY(umma_layer_upload(res, &uproj, p, p + (size_t)NV_D * 512, 512, NV_D, 1, NV_W_SCALE));
  p += (size_t)NV_D * 512 + NV_D;
  OSB_TRY(conv_layer_upload(res, &assign, p, p + (size_t)NV_K * NV_D, NV_D, NV_K, 1));
  p += (size_t)NV_K * NV_D + NV_K;
  OSB_TRY(res.upload(&centroids, p, (size_t)NV_K * NV_D));
  {
    // engine input is the u8 image converted to float UNSCALED (mobilenetvlad_tensorrt.cpp:8-10); the stand-in
    // network's first op multiplies by 1/255 in f32.
    std::vector<float> l(256);
    const float sc = (float)(1.0 / 255.0);
    for (int v = 0; v < 256; ++v) l[v] = (float)v * sc;
    OSB_TRY(res.upload(&lut, l.data(), 256));
  }
  const size_t B = max_batch;
  const size_t act = B * (H / 2) * (W / 2) * 64;   // largest activation: block 0 output (64 ch at 1/2 res)
  OSB_TRY(res.alloc(&d_img, B * H * W));
  OSB_TRY(res.alloc(&actA, act));
  OSB_TRY(res.alloc(&actB, act));
  OSB_TRY(res.alloc(&d_assign, B * (H / 16) * (W / 16) * NV_K));
  OSB_TRY(res.alloc(&d_out, B * NV_K * NV_D));
  OSB_TRY(res.alloc(&d_mu, B * NV_D));
  OSB_TRY(res.alloc(&d_part, B * NV_SLICES * NV_K * NV_D));
  OSB_TRY(res.alloc(&d_psum, B * NV_SLICES * NV_K));
  if (use_umma) {
    // planes of the pointwise inputs: blocks 1..6 (depthwise outputs) and the projection (block 6 output); all share
    // one buffer sized for the largest (they are live one at a time, except block 6 -> projection: two halves)
    size_t maxe = 0;
    int h = H / 2, w = W / 2;
    int gh[8], gw[8], gc[8];
    for (int i = 0; i < 7; ++i) {
      h /= blk[i].stride; w /= blk[i].stride;
      gh[i] = h; gw[i] = w; gc[i] = blk[i].cin;
      if (i >= 1) maxe = std::max(maxe, (size_t)B * h * w * blk[i].cin);
    }
    gh[7] = h; gw[7] = w; gc[7] = 512;
    maxe = std::max(maxe, (size_t)B * h * w * 512);
    OSB_TRY(res.alloc(&planes, 4 * maxe));      // two regions of (hi, lo)
    for (int i = 1; i < 8; ++i) {
      __half* base = planes + ((i & 1) ? 0 : 2 * maxe);                 // alternate regions: block 6 (even) vs proj (7, odd)
      pl_hi[i] = base; pl_lo[i] = base + (size_t)B * gh[i] * gw[i] * gc[i];
      OSB_TRY(umma_act_maps(&tmA[i], &tmB[i], pl_hi[i], pl_lo[i], (int)B, gh[i], gw[i], gc[i], 1));
    }
  }
  return OSB_OK;
}

osb_status NetVLAD::infer_dev(const uint8_t* img_dev, int B, float* out_dev, cudaStream_t st) {
  OSB_REQUIRE(B > 0 && B <= max_batch, "batch out of range");
  int h = H / 2, w = W / 2;
  OSB_TRY(conv_first_forward(w0, b0, lut, img_dev, actA, B, H, W, 32, 2, ACT_RELU6, st));
  float* cur = actA;                 // fp32 activations of the previous block
  for (int i = 0; i < 7; ++i) {
    if (use_umma && i == 0) {
      OSB_TRY(nv_block0_forward(cur, blk[0].dw, blk[0].dwb, pw0_kc, pw0_b, actB, B, h, w, st));
      cur = actB;
    } else if (use_umma) {
      // depthwise (fp32 -> split planes) then pointwise on the tensor cores (planes -> fp32, or planes for the projection)
      OSB_TRY(umma_dwconv_forward(blk[i].dw, blk[i].dwb, cur, pl_hi[i], pl_lo[i], B, h, w, blk[i].cin, blk[i].stride,
                                  NV_ACT_SCALE, st, true, precision));
      h /= blk[i].stride; w /= blk[i].stride;
      if (i < 6) {
        OSB_TRY(umma_conv_forward(upw[i], tmA[i], tmB[i], B, h, w, NV_ACT_SCALE, nullptr, nullptr, actA, blk[i].cout,
                                  blk[i].cout, 1.f, 2, 0, st, 0, precision));
        cur = actA;
      } else {
        OSB_TRY(umma_conv_forward(upw[i], tmA[i], tmB[i], B, h, w, NV_ACT_SCALE, pl_hi[7], pl_lo[7], nullptr, blk[i].cout,
                                  blk[i].cout, NV_ACT_SCALE, 2, 0, st, 0, precision));
      }
    } else {
      OSB_TRY(dwconv3x3_forward(blk[i].dw, blk[i].dwb, actA, actB, B, h, w, blk[i].cin, blk[i].stride, ACT_RELU6, st));
      h /= blk[i].stride; w /= blk[i].stride;
      OSB_TRY(conv_forward(blk[i].pw, actB, actA, B, h, w, blk[i].cout, ACT_RELU6, st));
    }
  }
  if (use_umma)
    OSB_TRY(umma_conv_forward(uproj, tmA[7], tmB[7], B, h, w, NV_ACT_SCALE, nullptr, nullptr, actB, NV_D, NV_D, 1.f, 0, 0, st,
                              0, precision));
  else
    OSB_TRY(conv_forward(proj, actA, actB, B, h, w, NV_D, ACT_NONE, st));
  OSB_TRY(nv_head_forward(assign, centroids, actB, B, h, w, d_mu, d_assign, d_part, d_psum, out_dev, st));
  return OSB_OK;
}

}  // namespace osb

using namespace osb;

struct osb_netvlad {
  int device = 0;
  NetVLAD nv;
  std::mutex mu;
};

extern "C" osb_status osb_netvlad_create(osb_netvlad** out, const float* weights, size_t n_weights, int width,
                                         int height, int max_batch) {
  OSB_REQUIRE(out != nullptr && max_batch > 0, "bad arguments");
  OSB_TRY(require_device());
  std::unique_ptr<osb_netvlad> h(new osb_netvlad());
  h->device = current_device();
  OSB_TRY(h->nv.init(weights, n_weights, width, height, max_batch));
  *out = h.release();
  return OSB_OK;
}

extern "C" osb_status osb_netvlad_destroy(osb_netvlad* h) {
  delete h;
  return OSB_OK;
}

extern "C" osb_status osb_netvlad_infer_dev(osb_netvlad* h, const uint8_t* images_dev, int batch, float* out_dev,
                                            void* stream) {
  OSB_REQUIRE(h && images_dev && out_dev, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  return h->nv.infer_dev(images_dev, batch, out_dev, (cudaStream_t)stream);
}

extern "C" osb_status osb_netvlad_set_precision(osb_netvlad* h, int precision) {
  OSB_REQUIRE(h != nullptr, "null handle");
  std::lock_guard<std::mutex> lk(h->mu);
  return h->nv.set_precision(precision);
}

extern "C" osb_status osb_netvlad_infer(osb_netvlad* h, const uint8_t* images, int batch, float* out) {
  OSB_REQUIRE(h && images && out, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  NetVLAD& nv = h->nv;
  OSB_REQUIRE(batch > 0 && batch <= nv.max_batch, "batch out of range");
  cudaStream_t st = nv.stream;
  OSB_CUDA(cudaMemcpyAsync(nv.d_img, images, (size_t)batch * nv.H * nv.W, cudaMemcpyHostToDevice, st));
  osb_status s = nv.infer_dev(nv.d_img, batch, nv.d_out, st);
  if (s != OSB_OK) return s;
  OSB_CUDA(cudaMemcpyAsync(out, nv.d_out, (size_t)batch * NV_K * NV_D * sizeof(float), cudaMemcpyDeviceToHost, st));
  OSB_CUDA(cudaStreamSynchronize(st));
  return OSB_OK;
}

// --------------------------------------------------------------------------------------------------------------
// parity hooks: block 0 and the head of the network, run by the host functions infer_dev calls (tests only)
// --------------------------------------------------------------------------------------------------------------
extern "C" osb_status osb_nv_block0_parity(const float* dw_w, const float* dw_b, const float* pw_w, const float* pw_b,
                                           const float* x_dev, int batch, int height, int width, float* y_dev,
                                           void* stream) {
  OSB_REQUIRE(dw_w && dw_b && pw_w && pw_b && x_dev && y_dev, "null argument");
  OSB_REQUIRE(batch > 0 && height > 0 && width > 0, "bad geometry");
  OSB_TRY(require_device());
  const cudaStream_t st = (cudaStream_t)stream;
  Resources res;
  res.sync_before_release(st);
  std::vector<float> kc(F0_C * F0_OC);
  for (int o = 0; o < F0_OC; ++o)
    for (int k = 0; k < F0_C; ++k) kc[k * F0_OC + o] = pw_w[o * F0_C + k];
  float *dwd = nullptr, *dbd = nullptr, *kcd = nullptr, *pbd = nullptr;
  OSB_TRY(upload_tap_major(res, &dwd, dw_w, F0_C));
  OSB_TRY(res.upload(&dbd, dw_b, F0_C));
  OSB_TRY(res.upload(&kcd, kc.data(), kc.size()));
  OSB_TRY(res.upload(&pbd, pw_b, F0_OC));
  OSB_TRY(nv_block0_prepare());
  OSB_TRY(nv_block0_forward(x_dev, dwd, dbd, kcd, pbd, y_dev, batch, height, width, st));
  OSB_CUDA(cudaStreamSynchronize(st));
  return OSB_OK;
}

extern "C" osb_status osb_nv_head_parity(const float* assign_w, const float* assign_b, const float* centroids,
                                         const float* x_dev, int batch, int height, int width, float* mu_dev,
                                         float* xn_dev, float* logits_dev, float* assign_dev, float* out_dev,
                                         void* stream) {
  OSB_REQUIRE(assign_w && assign_b && centroids && x_dev && mu_dev && xn_dev && logits_dev && assign_dev && out_dev,
              "null argument");
  OSB_REQUIRE(batch > 0 && height > 0 && width > 0, "bad geometry");
  OSB_TRY(require_device());
  const cudaStream_t st = (cudaStream_t)stream;
  Resources res;
  res.sync_before_release(st);
  const size_t locs = (size_t)batch * height * width;
  ConvLayer L;
  float *cd = nullptr, *part = nullptr, *psum = nullptr;
  OSB_TRY(conv_layer_upload(res, &L, assign_w, assign_b, NV_D, NV_K, 1));
  OSB_TRY(res.upload(&cd, centroids, (size_t)NV_K * NV_D));
  OSB_TRY(res.alloc(&part, (size_t)batch * NV_SLICES * NV_K * NV_D));
  OSB_TRY(res.alloc(&psum, (size_t)batch * NV_SLICES * NV_K));
  OSB_TRY(copy_dev(xn_dev, x_dev, locs * NV_D, st));  // the head centres and normalises in place
  OSB_TRY(nv_head_forward(L, cd, xn_dev, batch, height, width, mu_dev, assign_dev, part, psum, out_dev, st, logits_dev));
  OSB_CUDA(cudaStreamSynchronize(st));
  return OSB_OK;
}
