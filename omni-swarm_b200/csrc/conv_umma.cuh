// conv_umma.cuh -- host-side interface of the tensor-core (wgmma) convolution path (conv_umma.cu)
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include "common.cuh"

namespace osb {

// Range of the split planes: an operand x is stored as hi = fp16(scale * x), lo = fp16(scale * x - hi), and fp16 rounds
// |v| >= 65520 to infinity, so x is representable only for |x| < 65520 / scale: activations below 4095 at the networks'
// x16, weights below 63.984375 at x1024.  umma_layer_upload rejects weights outside that range (OSB_ERR_INVALID).  An
// ACTIVATION beyond it is written as hi = +-inf, lo = -+inf; the next layer's sums are then NaN, which a following ReLU
// (fmaxf) or max-pool turns into a finite value, so that overflow is silent (pinned by tests/test_gpu_conv_layers.py).
// weights of one conv layer as two fp16 planes [tap][n_pad][Cin] (K-major rows) + their TMA descriptors
struct UmmaLayer {
  int cin = 0, cout = 0, n_pad = 0, ks = 1, taps = 1;
  float w_scale = 1.f;
  __half *w_hi = nullptr, *w_lo = nullptr;
  float* bias = nullptr;
  CUtensorMap tm_hi, tm_lo;           // boxes of 64 rows (80 for the 80-row detector head)
};

// Blanked band: when every image of a batch is zero from row r0 down, an output pixel whose receptive field lies in the
// zero rows and touches no padding has the same value everywhere: the layer's constant.  A tile whose 8 x 16 outputs are
// all such pixels is not computed; it receives the constant as plain stores.
struct TileRect {                     // [y0, y1) x [x0, x1)
  int y0 = 0, y1 = 0, x0 = 0, x1 = 0;
  bool empty() const { return y0 >= y1 || x0 >= x1; }
};
struct BandLayer { int ks, pool; };   // a layer of a chain: kernel size, fused 2x2 max-pool of its output
// The chain's first layer reads the H x W images, each later one the previous one's output.  For every layer: px[l], its
// output pixels (after the pool) that equal the layer's constant, and tiles[l], its 8 x 16 output tiles (before the pool)
// that are constant throughout.  first_skip: the first layer's output pixels that only constant tiles of the second read.
// A pixel counts as constant only when its whole window lies inside the image and inside the constant input (the zero
// rows for the first layer), so padding never enters; ragged tiles never qualify.
void band_geometry(int H, int W, int r0, const BandLayer* layers, int n, TileRect* px, TileRect* tiles,
                   TileRect* first_skip);
// the constant tiles of one launch and the layer's constant output (out_c channels per plane; lo unused in plain fp16)
struct ConvBand {
  TileRect tiles;
  const __half* hi = nullptr;
  const __half* lo = nullptr;
};

// the weight planes and bias belong to `res`
osb_status umma_layer_upload(Resources& res, UmmaLayer* L, const float* w_oihw, const float* bias, int cin, int cout,
                             int ks, float w_scale);
// TMA descriptors of an activation tensor stored as two fp16 NHWC planes [B][H][W][C]
osb_status umma_act_maps(CUtensorMap* hi, CUtensorMap* lo, __half* p_hi, __half* p_lo, int B, int H, int W, int C,
                         int ks);
// relu: 0 none, 1 ReLU, 2 ReLU6.  y = act(conv(x) + b), optionally followed by a fused 2x2 max-pool (pool = 1: output is [B][H/2][W/2][C]);
// output either as split fp16 planes (out_hi/out_lo, scaled by out_scale) or as fp32.
// precision (these four functions): OSB_PRECISION_SPLIT_FP16 (default) reads and writes both planes, OSB_PRECISION_FP16
// only the hi planes (one MMA per K step; out_lo and the lo input planes are not touched).  The weights are the same.
// band (optional): tiles of every image that are stored as its constant instead of computed; only the 64 -> 64 3x3 and the
// 128-channel layers take one, with split planes as output.
osb_status umma_conv_forward(const UmmaLayer& L, const CUtensorMap& a_hi, const CUtensorMap& a_lo, int B, int H, int W,
                             float act_scale, __half* out_hi, __half* out_lo, float* out_f32, int out_c, int out_cstride,
                             float out_scale, int relu, int pool, cudaStream_t st, int max_ctas = 0,
                             int precision = OSB_PRECISION_SPLIT_FP16, const ConvBand* band = nullptr);
osb_status umma_conv_softmax_forward(const UmmaLayer& L, const CUtensorMap& a_hi, const CUtensorMap& a_lo, int B, int H, int W,
                                     float act_scale, float* semi, cudaStream_t st, int max_ctas = 0,
                                     int precision = OSB_PRECISION_SPLIT_FP16);
osb_status umma_first_forward(const float* w_tap_cout, const float* bias, const float* lut, const uint8_t* img,
                              __half* out_hi, __half* out_lo, int B, int H, int W, float out_scale, cudaStream_t st,
                              int precision = OSB_PRECISION_SPLIT_FP16, TileRect skip = {});   // skip: pixels not written
osb_status umma_make_tmap(CUtensorMap* tm, void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                          const uint32_t* box);
// depthwise 3x3 + bias + ReLU6, fp32 NHWC in, split fp16 planes out (feeds a pointwise tensor-core conv).  Stride 1 runs
// the four-pixel kernel unless s1x4 = false (the generic kernel; the planes are bit-identical)
osb_status umma_dwconv_forward(const float* w_tap_c, const float* bias, const float* x, __half* out_hi, __half* out_lo,
                               int B, int H, int W, int C, int stride, float out_scale, cudaStream_t st, bool s1x4 = true,
                               int precision = OSB_PRECISION_SPLIT_FP16);
}  // namespace osb
