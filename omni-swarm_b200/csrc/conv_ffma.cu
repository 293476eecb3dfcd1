// conv_ffma.cu -- fp32 CUDA-core convolution kernels (NHWC).
//
// These are the full-precision implicit-GEMM kernels of the SuperPoint / NetVLAD networks
// (network definition: swarm_loop/superpoint.ipynb:135-205 of the reference).  They accumulate in fp32 with FFMA
// and are what the parity tests pin the tensor-core path against; conv_umma.cu holds the tensor-core (wgmma) kernels.
#include "common.cuh"
#include "kernels.cuh"

namespace osb {

// -------------------------------------------------------------------------------------------------------------
// Dense conv, stride 1, "same" padding, KS in {1,3}.
// CTA = 256 threads = 32 pixel-threads x 8 channel-groups; CTA tile = 8 rows x 32 px x 64 output channels;
// thread tile = 1 row x 8 px x 8 oc (64 fp32 accumulators).  K is consumed in chunks of 8 input channels:
// the halo'd input tile sits in shared memory as [c][y][x] with pitch 41 (conflict-free: see index math below)
// and the weight chunk as [tap][c][64].
// -------------------------------------------------------------------------------------------------------------
constexpr int CV_TH = 8, CV_TW = 32, CV_TC = 64, CV_KC = 8;
constexpr int CV_PITCH = 41;  // >= CV_TW + 2 and == 1 (mod 8): bank = 9*row + 8*colgroup -> 32 distinct banks

template <int KS>
__global__ void __launch_bounds__(256)
conv_ffma_kernel(const float* __restrict__ x, const float* __restrict__ wp, const float* __restrict__ bias,
                 float* __restrict__ y, int H, int W, int Cin, int Cout, int Cout_pad, int out_cstride, int act,
                 int tiles_x) {
  constexpr int HALO = KS / 2;
  constexpr int IH = CV_TH + 2 * HALO, IW = CV_TW + 2 * HALO;
  constexpr int TAPS = KS * KS;
  __shared__ float sin_[CV_KC][IH][CV_PITCH];
  __shared__ __align__(16) float sw[TAPS][CV_KC][CV_TC];

  const int tid = threadIdx.x;
  const int pt = tid & 31, ot = tid >> 5;
  const int ty = pt >> 2, tx = pt & 3;           // thread's row in the tile, 8-px column group
  const int tile_y = blockIdx.x / tiles_x, tile_x = blockIdx.x % tiles_x;
  const int y0 = tile_y * CV_TH, x0 = tile_x * CV_TW;
  const int co0 = blockIdx.y * CV_TC;
  const int b = blockIdx.z;
  const float* xb = x + (size_t)b * H * W * Cin;

  float acc[8][8];
#pragma unroll
  for (int p = 0; p < 8; ++p)
#pragma unroll
    for (int o = 0; o < 8; ++o) acc[p][o] = 0.f;

  for (int c0 = 0; c0 < Cin; c0 += CV_KC) {
    // ---- stage input chunk: IH*IW pixels x 8 channels (two float4 per pixel) ----
    for (int e = tid; e < IH * IW * 2; e += 256) {
      const int half = e & 1, px = e >> 1;
      const int iy = px / IW, ix = px % IW;
      const int gy = y0 + iy - HALO, gx = x0 + ix - HALO;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (gy >= 0 && gy < H && gx >= 0 && gx < W)
        v = *reinterpret_cast<const float4*>(xb + ((size_t)gy * W + gx) * Cin + c0 + 4 * half);
      sin_[4 * half + 0][iy][ix] = v.x;
      sin_[4 * half + 1][iy][ix] = v.y;
      sin_[4 * half + 2][iy][ix] = v.z;
      sin_[4 * half + 3][iy][ix] = v.w;
    }
    // ---- stage weight chunk: [tap][8][64] from wp[(tap*Cin + c)*Cout_pad + co] ----
    for (int e = tid; e < TAPS * CV_KC * (CV_TC / 4); e += 256) {
      const int o4 = e % (CV_TC / 4);
      const int c = (e / (CV_TC / 4)) % CV_KC;
      const int tap = e / (CV_TC / 4 * CV_KC);
      const float4 v = *reinterpret_cast<const float4*>(wp + ((size_t)tap * Cin + c0 + c) * Cout_pad + co0 + 4 * o4);
      *reinterpret_cast<float4*>(&sw[tap][c][4 * o4]) = v;
    }
    __syncthreads();
#pragma unroll
    for (int c = 0; c < CV_KC; ++c) {
#pragma unroll
      for (int ky = 0; ky < KS; ++ky) {
        float in[8 + 2 * HALO];
#pragma unroll
        for (int i = 0; i < 8 + 2 * HALO; ++i) in[i] = sin_[c][ty + ky][tx * 8 + i];
#pragma unroll
        for (int kx = 0; kx < KS; ++kx) {
          const float4 w0 = *reinterpret_cast<const float4*>(&sw[ky * KS + kx][c][ot * 8]);
          const float4 w1 = *reinterpret_cast<const float4*>(&sw[ky * KS + kx][c][ot * 8 + 4]);
          const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
          for (int p = 0; p < 8; ++p)
#pragma unroll
            for (int o = 0; o < 8; ++o) acc[p][o] = fmaf(in[p + kx], wv[o], acc[p][o]);
        }
      }
    }
    __syncthreads();
  }
  // ---- epilogue ----
  const int co = co0 + ot * 8;
  if (co >= out_cstride) return;
  float bv[8];
#pragma unroll
  for (int o = 0; o < 8; ++o) bv[o] = bias[co + o];
  const int gy = y0 + ty;
  if (gy >= H) return;
  float* yb = y + ((size_t)b * H + gy) * W * out_cstride;
#pragma unroll
  for (int p = 0; p < 8; ++p) {
    const int gx = x0 + tx * 8 + p;
    if (gx >= W) continue;
    float r[8];
#pragma unroll
    for (int o = 0; o < 8; ++o) {
      float v = acc[p][o] + bv[o];
      if (act == ACT_RELU) v = fmaxf(v, 0.f);
      else if (act == ACT_RELU6) v = fminf(fmaxf(v, 0.f), 6.f);
      r[o] = v;
    }
    float4* dst = reinterpret_cast<float4*>(yb + (size_t)gx * out_cstride + co);
    dst[0] = make_float4(r[0], r[1], r[2], r[3]);
    dst[1] = make_float4(r[4], r[5], r[6], r[7]);
  }
}

osb_status conv_layer_upload(Resources& res, ConvLayer* L, const float* w_oihw, const float* bias, int cin, int cout,
                             int ks) {
  L->cin = cin; L->cout = cout; L->ks = ks;
  L->cout_pad = cdiv(cout, CV_TC) * CV_TC;
  const int taps = ks * ks;
  std::vector<float> wp((size_t)taps * cin * L->cout_pad, 0.f), bp(L->cout_pad, 0.f);
  for (int o = 0; o < cout; ++o) {
    bp[o] = bias[o];
    for (int c = 0; c < cin; ++c)
      for (int t = 0; t < taps; ++t) wp[((size_t)t * cin + c) * L->cout_pad + o] = w_oihw[((size_t)o * cin + c) * taps + t];
  }
  OSB_TRY(res.upload(&L->w, wp.data(), wp.size()));
  return res.upload(&L->b, bp.data(), bp.size());
}

osb_status upload_tap_major(Resources& res, float** dst, const float* w_oihw, int cout) {
  std::vector<float> t(9 * (size_t)cout);
  for (int o = 0; o < cout; ++o)
    for (int k = 0; k < 9; ++k) t[(size_t)k * cout + o] = w_oihw[(size_t)o * 9 + k];
  return res.upload(dst, t.data(), t.size());
}

osb_status conv_forward(const ConvLayer& L, const float* x, float* y, int B, int H, int W, int out_cstride,
                        int act, cudaStream_t st) {
  OSB_REQUIRE(L.cin % CV_KC == 0 && out_cstride % 8 == 0 && out_cstride <= L.cout_pad && out_cstride >= L.cout,
              "conv_forward: Cin must be a multiple of 8 and out_cstride a multiple of 8 in [Cout, Cout_pad]");
  const int tiles_x = cdiv(W, CV_TW), tiles_y = cdiv(H, CV_TH);
  dim3 grid(tiles_x * tiles_y, L.cout_pad / CV_TC, B);
  if (L.ks == 3)
    OSB_LAUNCH(conv_ffma_kernel<3>, grid, 256, 0, st, x, L.w, L.b, y, H, W, L.cin, L.cout, L.cout_pad, out_cstride,
               act, tiles_x);
  else
    OSB_LAUNCH(conv_ffma_kernel<1>, grid, 256, 0, st, x, L.w, L.b, y, H, W, L.cin, L.cout, L.cout_pad, out_cstride,
               act, tiles_x);
  OSB_CHECK_LAUNCH();
  return OSB_OK;
}

// -------------------------------------------------------------------------------------------------------------
// First layer: single-channel u8 image, 3x3, pad 1, stride 1 or 2 -> COUT channels.  Store-bandwidth bound
// (COUT*4 bytes written per 1 byte read): one thread per output pixel, weights broadcast from shared memory.
// The u8 -> f32 conversion (cv::Mat::convertTo, superpoint_tensorrt.cpp:127 / mobilenetvlad_tensorrt.cpp:10)
// is a 256-entry LUT computed on the host.
// -------------------------------------------------------------------------------------------------------------
template <int COUT>
__global__ void __launch_bounds__(128)
conv_first_kernel(const float* __restrict__ w, const float* __restrict__ bias, const float* __restrict__ lut,
                  const uint8_t* __restrict__ img, float* __restrict__ y, int H, int W, int Ho, int Wo, int stride,
                  int act) {
  __shared__ __align__(16) float sw[9][COUT];
  __shared__ __align__(16) float sb[COUT];
  __shared__ float slut[256];
  for (int e = threadIdx.x; e < 9 * COUT; e += blockDim.x) (&sw[0][0])[e] = w[e];
  for (int e = threadIdx.x; e < COUT; e += blockDim.x) sb[e] = bias[e];
  for (int e = threadIdx.x; e < 256; e += blockDim.x) slut[e] = lut[e];
  __syncthreads();
  const int b = blockIdx.y;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= Ho * Wo) return;
  const int oy = p / Wo, ox = p % Wo;
  const uint8_t* ib = img + (size_t)b * H * W;
  float in[9];
#pragma unroll
  for (int ky = 0; ky < 3; ++ky)
#pragma unroll
    for (int kx = 0; kx < 3; ++kx) {
      const int gy = oy * stride + ky - 1, gx = ox * stride + kx - 1;
      in[ky * 3 + kx] = (gy >= 0 && gy < H && gx >= 0 && gx < W) ? slut[ib[(size_t)gy * W + gx]] : 0.f;
    }
  float4* dst = reinterpret_cast<float4*>(y + ((size_t)b * Ho * Wo + p) * COUT);
#pragma unroll 4
  for (int o4 = 0; o4 < COUT / 4; ++o4) {
    float r[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float a = 0.f;
#pragma unroll
      for (int t = 0; t < 9; ++t) a = fmaf(in[t], sw[t][4 * o4 + j], a);
      a += sb[4 * o4 + j];
      if (act == ACT_RELU) a = fmaxf(a, 0.f);
      else if (act == ACT_RELU6) a = fminf(fmaxf(a, 0.f), 6.f);
      r[j] = a;
    }
    dst[o4] = make_float4(r[0], r[1], r[2], r[3]);
  }
}

osb_status conv_first_forward(const float* w_tap_cout, const float* bias, const float* lut, const uint8_t* img,
                              float* y, int B, int H, int W, int cout, int stride, int act, cudaStream_t st) {
  const int Ho = H / stride, Wo = W / stride;
  dim3 grid(cdiv(Ho * Wo, 128), B);
  if (cout == 64)
    OSB_LAUNCH(conv_first_kernel<64>, grid, 128, 0, st, w_tap_cout, bias, lut, img, y, H, W, Ho, Wo, stride, act);
  else if (cout == 32)
    OSB_LAUNCH(conv_first_kernel<32>, grid, 128, 0, st, w_tap_cout, bias, lut, img, y, H, W, Ho, Wo, stride, act);
  else {
    set_error("conv_first_forward", "cout must be 32 or 64");
    return OSB_ERR_INVALID;
  }
  OSB_CHECK_LAUNCH();
  return OSB_OK;
}

// -------------------------------------------------------------------------------------------------------------
// 2x2 max pool, NHWC, one thread per (output pixel, 4 channels)
// -------------------------------------------------------------------------------------------------------------
__global__ void maxpool2x2_kernel(const float4* __restrict__ x, float4* __restrict__ y, int H, int W, int C4,
                                  int64_t total) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int Ho = H / 2, Wo = W / 2;
  const int c = (int)(i % C4);
  int64_t p = i / C4;
  const int ox = (int)(p % Wo); p /= Wo;
  const int oy = (int)(p % Ho);
  const int b = (int)(p / Ho);
  const float4* xb = x + (((size_t)b * H + 2 * oy) * W + 2 * ox) * C4 + c;
  const float4 a = xb[0], bb = xb[C4], cc = xb[(size_t)W * C4], d = xb[(size_t)W * C4 + C4];
  float4 r;
  r.x = fmaxf(fmaxf(a.x, bb.x), fmaxf(cc.x, d.x));
  r.y = fmaxf(fmaxf(a.y, bb.y), fmaxf(cc.y, d.y));
  r.z = fmaxf(fmaxf(a.z, bb.z), fmaxf(cc.z, d.z));
  r.w = fmaxf(fmaxf(a.w, bb.w), fmaxf(cc.w, d.w));
  y[i] = r;
}

osb_status maxpool2x2_forward(const float* x, float* y, int B, int H, int W, int C, cudaStream_t st) {
  const int64_t total = (int64_t)B * (H / 2) * (W / 2) * (C / 4);
  OSB_LAUNCH(maxpool2x2_kernel, (unsigned)cdiv64(total, 256), 256, 0, st, reinterpret_cast<const float4*>(x),
             reinterpret_cast<float4*>(y), H, W, C / 4, total);
  OSB_CHECK_LAUNCH();
  return OSB_OK;
}

// -------------------------------------------------------------------------------------------------------------
// depthwise 3x3, pad 1, stride s, NHWC; one thread per (output pixel, 4 channels); HBM bound
// -------------------------------------------------------------------------------------------------------------
__global__ void dwconv3x3_kernel(const float4* __restrict__ w, const float4* __restrict__ bias,
                                 const float4* __restrict__ x, float4* __restrict__ y, int H, int W, int Ho, int Wo,
                                 int C4, int stride, int act, int64_t total) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c = (int)(i % C4);
  int64_t p = i / C4;
  const int ox = (int)(p % Wo); p /= Wo;
  const int oy = (int)(p % Ho);
  const int b = (int)(p / Ho);
  float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int ky = 0; ky < 3; ++ky)
#pragma unroll
    for (int kx = 0; kx < 3; ++kx) {
      const int gy = oy * stride + ky - 1, gx = ox * stride + kx - 1;
      if (gy < 0 || gy >= H || gx < 0 || gx >= W) continue;
      const float4 v = x[(((size_t)b * H + gy) * W + gx) * C4 + c];
      const float4 ww = w[(size_t)(ky * 3 + kx) * C4 + c];
      a.x = fmaf(v.x, ww.x, a.x); a.y = fmaf(v.y, ww.y, a.y);
      a.z = fmaf(v.z, ww.z, a.z); a.w = fmaf(v.w, ww.w, a.w);
    }
  const float4 bb = bias[c];
  a.x += bb.x; a.y += bb.y; a.z += bb.z; a.w += bb.w;
  if (act == ACT_RELU) { a.x = fmaxf(a.x, 0.f); a.y = fmaxf(a.y, 0.f); a.z = fmaxf(a.z, 0.f); a.w = fmaxf(a.w, 0.f); }
  else if (act == ACT_RELU6) {
    a.x = fminf(fmaxf(a.x, 0.f), 6.f); a.y = fminf(fmaxf(a.y, 0.f), 6.f);
    a.z = fminf(fmaxf(a.z, 0.f), 6.f); a.w = fminf(fmaxf(a.w, 0.f), 6.f);
  }
  y[i] = a;
}

osb_status dwconv3x3_forward(const float* w_tap_c, const float* bias, const float* x, float* y, int B, int H, int W,
                             int C, int stride, int act, cudaStream_t st) {
  const int Ho = H / stride, Wo = W / stride;
  const int64_t total = (int64_t)B * Ho * Wo * (C / 4);
  OSB_LAUNCH(dwconv3x3_kernel, (unsigned)cdiv64(total, 256), 256, 0, st, reinterpret_cast<const float4*>(w_tap_c),
             reinterpret_cast<const float4*>(bias), reinterpret_cast<const float4*>(x), reinterpret_cast<float4*>(y),
             H, W, Ho, Wo, C / 4, stride, act, total);
  OSB_CHECK_LAUNCH();
  return OSB_OK;
}

}  // namespace osb

// --------------------------------------------------------------------------------------------------------------
// parity hooks: one fp32 layer, run by the host functions above on caller-supplied operands (tests only)
// --------------------------------------------------------------------------------------------------------------
using namespace osb;

extern "C" osb_status osb_conv_ffma_parity(const float* w, const float* bias, int cin, int cout, int ks,
                                           const float* x_dev, int batch, int height, int width, int act,
                                           int out_cstride, float* y_dev, void* stream) {
  OSB_REQUIRE(w && bias && x_dev && y_dev, "null argument");
  OSB_REQUIRE(batch > 0 && height > 0 && width > 0 && cin > 0 && cout > 0 && (ks == 1 || ks == 3) && act >= 0 &&
              act <= 2, "bad geometry (ks 1 or 3, act 0..2)");
  OSB_TRY(require_device());
  const cudaStream_t st = (cudaStream_t)stream;
  Resources res;
  res.sync_before_release(st);
  ConvLayer L;
  OSB_TRY(conv_layer_upload(res, &L, w, bias, cin, cout, ks));
  OSB_TRY(conv_forward(L, x_dev, y_dev, batch, height, width, out_cstride, act, st));
  OSB_CUDA(cudaStreamSynchronize(st));
  return OSB_OK;
}

extern "C" osb_status osb_conv_first_ffma_parity(const float* w, const float* bias, int cout, int stride, int act,
                                                 const uint8_t* images_dev, int batch, int height, int width,
                                                 float* y_dev, void* stream) {
  OSB_REQUIRE(w && bias && images_dev && y_dev, "null argument");
  OSB_REQUIRE(batch > 0 && height > 0 && width > 0 && (stride == 1 || stride == 2) && act >= 0 && act <= 2,
              "bad geometry (stride 1 or 2, act 0..2)");
  OSB_TRY(require_device());
  const cudaStream_t st = (cudaStream_t)stream;
  Resources res;
  res.sync_before_release(st);
  float *wd = nullptr, *bd = nullptr, *lut = nullptr;
  std::vector<float> l(256);
  for (int v = 0; v < 256; ++v) l[v] = (float)v * (float)(1.0 / 255.0);
  if (cout == 32 || cout == 64) {
    OSB_TRY(upload_tap_major(res, &wd, w, cout));
    OSB_TRY(res.upload(&bd, bias, cout));
    OSB_TRY(res.upload(&lut, l.data(), 256));
  }
  OSB_TRY(conv_first_forward(wd, bd, lut, images_dev, y_dev, batch, height, width, cout, stride, act, st));
  OSB_CUDA(cudaStreamSynchronize(st));
  return OSB_OK;
}

extern "C" osb_status osb_dwconv_ffma_parity(const float* w, const float* bias, const float* x_dev, int batch,
                                             int height, int width, int channels, int stride, int act, float* y_dev,
                                             void* stream) {
  OSB_REQUIRE(w && bias && x_dev && y_dev, "null argument");
  OSB_REQUIRE(batch > 0 && height > 0 && width > 0 && channels > 0 && channels % 4 == 0 && (stride == 1 || stride == 2) &&
              act >= 0 && act <= 2, "bad geometry (channels a multiple of 4, stride 1 or 2, act 0..2)");
  OSB_TRY(require_device());
  const cudaStream_t st = (cudaStream_t)stream;
  Resources res;
  res.sync_before_release(st);
  float *wd = nullptr, *bd = nullptr;
  OSB_TRY(upload_tap_major(res, &wd, w, channels));
  OSB_TRY(res.upload(&bd, bias, channels));
  OSB_TRY(dwconv3x3_forward(wd, bd, x_dev, y_dev, batch, height, width, channels, stride, act, st));
  OSB_CUDA(cudaStreamSynchronize(st));
  return OSB_OK;
}

extern "C" osb_status osb_maxpool_parity(const float* x_dev, int batch, int height, int width, int channels,
                                         float* y_dev, void* stream) {
  OSB_REQUIRE(x_dev && y_dev, "null argument");
  OSB_REQUIRE(batch > 0 && height > 1 && width > 1 && channels > 0 && channels % 4 == 0,
              "bad geometry (channels a multiple of 4)");
  osb_status s = require_device();
  if (s != OSB_OK) return s;
  const cudaStream_t st = (cudaStream_t)stream;
  s = maxpool2x2_forward(x_dev, y_dev, batch, height, width, channels, st);
  const cudaError_t e = cudaStreamSynchronize(st);
  if (s == OSB_OK) OSB_CUDA(e);
  return s;
}
