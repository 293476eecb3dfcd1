// superpoint.cu -- osb_superpoint: the device-resident replacement of class SuperPointTensorRT
// (swarm_loop/include/swarm_loop/superpoint_tensorrt.h:20-28, swarm_loop/src/superpoint_tensorrt.cpp:91-230).
// Network: swarm_loop/superpoint.ipynb:135-205.  Everything from the u8 image to {keypoints, 64-d descriptors}
// stays in HBM; the reference copied 1.2 MB + 4.9 MB per image back to the host and post-processed on the CPU
// (swarm_loop/src/tensorrt_generic.cpp:58-75).
#include "superpoint.cuh"
#include <stdlib.h>

namespace osb {

static const int SP_CIN[12] = {1, 64, 64, 64, 64, 128, 128, 128, 128, 256, 128, 256};
static const int SP_COUT[12] = {64, 64, 64, 64, 128, 128, 128, 128, 256, 65, 256, 256};
static const int SP_KS[12] = {3, 3, 3, 3, 3, 3, 3, 3, 3, 1, 3, 1};
// power-of-two scales of the split-fp16 planes (exact): activations (post-ReLU, O(1)) x 16, weights (O(0.05)) x 1024
constexpr float SP_ACT_SCALE = 16.f;
constexpr float SP_W_SCALE = 1024.f;
// the trunk conv1a .. conv4b as the chain of band_geometry (trunk layer i is layer i above); the layers after it read
// conv4b's output, which no geometry the front-end runs leaves a constant tile in
constexpr int SP_TRUNK = 8;
static const BandLayer SP_TRUNK_LAYERS[SP_TRUNK] = {{3, 0}, {3, 1}, {3, 0}, {3, 1}, {3, 0}, {3, 1}, {3, 0}, {3, 0}};
constexpr int SP_BAND_C = 128;         // channel stride of band_c (the widest trunk layer)

static void sp_band_geometry(int H, int W, int zero_row, TileRect* px, TileRect* tiles, TileRect* first_skip) {
  band_geometry(H, W, zero_row, SP_TRUNK_LAYERS, SP_TRUNK, px, tiles, first_skip);
}

static size_t band_offset(int prec, int layer, int plane) {
  const int p = prec == OSB_PRECISION_FP16 ? 1 : 0;
  return ((size_t)(p * SP_TRUNK + layer) * 2 + plane) * SP_BAND_C;
}

const __half* SuperPoint::band_const(int prec, int layer, int plane) const {
  return band_c + band_offset(prec, layer, plane);
}

// Every trunk layer's constant from its own kernel: a zero image (one, of the handle's size) through conv1a .. conv4b with
// nothing skipped, and the output pixel of each layer read off inside its constant region (band_geometry with zero_row
// 0).  Interior pixels run the same K order, accumulators and epilogue wherever they sit, so the pixel is bit-exact for
// every constant tile of that layer.
osb_status SuperPoint::band_init() {
  if (!use_umma || band_c) return OSB_OK;
  TileRect px[SP_TRUNK], tiles[SP_TRUNK], skip;
  sp_band_geometry(H, W, 0, px, tiles, &skip);
  __half* c = nullptr;
  OSB_TRY(res.alloc(&c, (size_t)2 * SP_TRUNK * 2 * SP_BAND_C));
  OSB_CUDA(cudaMemsetAsync(d_img, 0, (size_t)H * W, stream));
  for (const int prec : {OSB_PRECISION_SPLIT_FP16, OSB_PRECISION_FP16}) {
    OSB_TRY(umma_first_forward(w1a, b1a, lut, d_img, in_hi[1], in_lo[1], 1, H, W, SP_ACT_SCALE, stream, prec));
    int h = H, w = W;
    for (int i = 1; i < SP_TRUNK; ++i) {
      const int pool = SP_TRUNK_LAYERS[i].pool;
      OSB_TRY(umma_conv_forward(UL[i], tmA[i], tmB[i], 1, h, w, SP_ACT_SCALE, in_hi[i + 1], in_lo[i + 1], nullptr,
                                SP_COUT[i], SP_COUT[i], SP_ACT_SCALE, 1, pool, stream, 0, prec));
      if (pool) { h /= 2; w /= 2; }
      if (px[i].empty()) continue;                   // then no geometry of this size has a constant tile here
      const size_t at = ((size_t)px[i].y0 * w + px[i].x0) * SP_COUT[i], bytes = SP_COUT[i] * sizeof(__half);
      OSB_CUDA(cudaMemcpyAsync(c + band_offset(prec, i, 0), in_hi[i + 1] + at, bytes, cudaMemcpyDeviceToDevice, stream));
      if (prec == OSB_PRECISION_SPLIT_FP16)
        OSB_CUDA(cudaMemcpyAsync(c + band_offset(prec, i, 1), in_lo[i + 1] + at, bytes, cudaMemcpyDeviceToDevice, stream));
    }
  }
  OSB_CUDA(cudaStreamSynchronize(stream));
  band_c = c;
  return OSB_OK;
}

osb_status SuperPoint::sparse_init() {
  if (const char* e = getenv("OSB_SP_SPARSE_HEAD")) if (atoi(e) == 0) return OSB_OK;
  if (!use_umma || sparse_head) return OSB_OK;
  seg = cdiv(std::min(4 * max_num, Hc * Wc), 128) * 128;
  const size_t rows = (size_t)max_batch * seg;
  OSB_TRY(res.alloc(&cell_slot, (size_t)max_batch * Hc * Wc));
  OSB_TRY(res.alloc(&cell_n, rows));
  OSB_TRY(res.alloc(&col_hi, rows * 1152));
  OSB_TRY(res.alloc(&col_lo, rows * 1152));
  OSB_TRY(res.alloc(&da_hi, rows * 256));
  OSB_TRY(res.alloc(&da_lo, rows * 256));
  OSB_TRY(res.alloc(&desc_c, rows * 256));
  // the rows as images of one 8 x 16 tile (the tensor-core kernels' tile), which a 1x1 layer reads without a halo
  const int tiles = (int)(rows / 128);
  OSB_TRY(umma_act_maps(&tm_col[0], &tm_col[1], col_hi, col_lo, tiles, 8, 16, 1152, 1));
  OSB_TRY(umma_act_maps(&tm_da[0], &tm_da[1], da_hi, da_lo, tiles, 8, 16, 256, 1));
  sparse_head = true;
  return OSB_OK;
}

osb_status SuperPoint::sparse_desc_head(int B, const KpJob& kp, cudaStream_t st) {
  const float SA = SP_ACT_SCALE;
  const int tiles = B * seg / 128;
  OSB_TRY(sp_cell_gather(B, H, W, kp.nk, kp.kpts, max_num, seg, cell_slot, in_hi[10], in_lo[10], col_hi, col_lo,
                         precision == OSB_PRECISION_FP16, st));
  OSB_TRY(umma_conv_forward(UDa_col, tm_col[0], tm_col[1], tiles, 8, 16, SA, da_hi, da_lo, nullptr, 256, 256, SA, 1, 0, st,
                            0, precision));                                                   // convDa
  // convDb; the L2 norm of each row is taken inside the descriptor kernels (sp_descriptors)
  return umma_conv_forward(UL[11], tm_da[0], tm_da[1], tiles, 8, 16, SA, nullptr, nullptr, desc_c, 256, 256, 1.f, 0, 0, st,
                           0, precision);
}

size_t sp_expected_weights() {
  size_t n = 0;
  for (int i = 0; i < 12; ++i) n += (size_t)SP_COUT[i] * SP_CIN[i] * SP_KS[i] * SP_KS[i] + SP_COUT[i];
  return n;
}

osb_status SuperPoint::init(const float* weights, size_t n_weights, int width, int height, float thres_, int max_num_,
                            const float* pca_comp, const float* pca_mean, int max_batch_) {
  OSB_REQUIRE(weights && pca_comp && pca_mean, "null weights / pca");
  OSB_REQUIRE(n_weights == sp_expected_weights(), "weight blob has the wrong length (expected 1300865 floats)");
  OSB_REQUIRE(width > 0 && height > 0 && width % 8 == 0 && height % 8 == 0, "width/height must be multiples of 8");
  OSB_REQUIRE(max_num_ > 0 && max_num_ <= 8192 && max_batch_ > 0, "bad max_num / max_batch");
  W = width; H = height; thres = thres_; max_num = max_num_; max_batch = max_batch_;
  Hc = H / 8; Wc = W / 8;
  OSB_TRY(res.stream(&stream));
  {
    int least = 0, greatest = 0;
    OSB_CUDA(cudaDeviceGetStreamPriorityRange(&least, &greatest));
    OSB_TRY(res.stream(&kp_stream, greatest));
  }
  OSB_TRY(res.event(&ev_semi, cudaEventDisableTiming));
  OSB_TRY(res.event(&ev_kp, cudaEventDisableTiming));
  if (const char* e = getenv("OSB_SP_OVERLAP")) overlap_kp = atoi(e) != 0;
  if (const char* e = getenv("OSB_SP_FUSED_SOFTMAX")) fused_softmax = atoi(e) != 0;
  // ---- weights ----
  const float* p = weights;
  {
    // conv1a: [64][1][3][3] -> [tap][64]
    std::vector<float> w9(9 * 64);
    for (int o = 0; o < 64; ++o)
      for (int t = 0; t < 9; ++t) w9[t * 64 + o] = p[o * 9 + t];
    OSB_TRY(res.upload(&w1a, w9.data(), 9 * 64));
    OSB_TRY(res.upload(&b1a, p + 64 * 9, 64));
    p += 64 * 9 + 64;
  }
  {
    // OSB_SP_CONV=ffma selects the fp32 CUDA-core convolutions (debug / A-B parity); default = tensor-core path
    const char* e = getenv("OSB_SP_CONV");
    use_umma = !(e && strcmp(e, "ffma") == 0);
  }
  for (int i = 1; i < 12; ++i) {
    const size_t nw = (size_t)SP_COUT[i] * SP_CIN[i] * SP_KS[i] * SP_KS[i];
    OSB_TRY(conv_layer_upload(res, &L[i], p, p + nw, SP_CIN[i], SP_COUT[i], SP_KS[i]));
    if (use_umma) OSB_TRY(umma_layer_upload(res, &UL[i], p, p + nw, SP_CIN[i], SP_COUT[i], SP_KS[i], SP_W_SCALE));
    if (use_umma && i == 10) {
      // convDa as a 1x1 layer of 9 x 128 inputs: input slab (kx * 2 + s) * 3 + ky is channel slab s of tap (ky, kx), the
      // 3x3 layer's K order (sp_cell_gather)
      std::vector<float> wc((size_t)256 * 1152);
      for (int o = 0; o < 256; ++o)
        for (int c = 0; c < 128; ++c)
          for (int t = 0; t < 9; ++t) {
            const int ky = t / 3, kx = t % 3, slab = (kx * 2 + c / 64) * 3 + ky;
            wc[(size_t)o * 1152 + slab * 64 + c % 64] = p[((size_t)o * 128 + c) * 9 + t];
          }
      OSB_TRY(umma_layer_upload(res, &UDa_col, wc.data(), p + nw, 1152, 256, 1, SP_W_SCALE));
    }
    p += nw + SP_COUT[i];
  }
  {
    // u8 -> f32 * (1/255): cv::Mat::convertTo(CV_32F, 1/255.0) computes (float)v * (float)alpha
    // (superpoint_tensorrt.cpp:127)
    std::vector<float> l(256);
    const float alpha = (float)(1.0 / 255.0);
    for (int v = 0; v < 256; ++v) l[v] = (float)v * alpha;
    OSB_TRY(res.upload(&lut, l.data(), 256));
  }
  {
    std::vector<float> ct(256 * 64);
    for (int o = 0; o < 64; ++o)
      for (int c = 0; c < 256; ++c) ct[c * 64 + o] = pca_comp[o * 256 + c];
    OSB_TRY(res.upload(&pca_compT, ct.data(), 256 * 64));
    OSB_TRY(res.upload(&pca_mean_d, pca_mean, 256));
  }
  // ---- activations ----
  const size_t B = max_batch, HW = (size_t)H * W;
  OSB_TRY(res.alloc(&d_img, B * HW));
  OSB_TRY(res.alloc(&actA, B * HW * 64));
  OSB_TRY(res.alloc(&actB, B * HW * 64));
  OSB_TRY(res.alloc(&d_logits, B * Hc * Wc * 80));
  if (use_umma) {
    // input geometry of every conv layer: which ping-pong buffer it reads and its [H][W][C]
    // (layer order: 1 conv1b 2 conv2a 3 conv2b 4 conv3a 5 conv3b 6 conv4a 7 conv4b 8 convPa 9 convPb 10 convDa 11 convDb)
    // with the pools fused into the conv epilogues the layers simply alternate between the two buffers;
    // conv4b's output x (layer 8 input) stays in B while convPa writes A, so convDa (10) reads B, convDb (11) reads A
    const int in_buf[12] = {-1, 0, 1, 0, 1, 0, 1, 0, 1, 0, 1, 0};      // 0 = actA, 1 = actB
    const int in_div[12] = {0, 1, 2, 2, 4, 4, 8, 8, 8, 8, 8, 8};
    for (int i = 1; i < 12; ++i) {
      const int h = H / in_div[i], w = W / in_div[i], c = SP_CIN[i];
      __half* base = reinterpret_cast<__half*>(in_buf[i] == 0 ? actA : actB);
      in_hi[i] = base;
      in_lo[i] = base + (size_t)max_batch * h * w * c;
      OSB_TRY(umma_act_maps(&tmA[i], &tmB[i], in_hi[i], in_lo[i], max_batch, h, w, c, SP_KS[i]));
    }
  }
  OSB_TRY(res.alloc(&d_semi, B * HW));
  OSB_TRY(res.alloc(&d_desc, B * Hc * Wc * 256));
  OSB_TRY(res.alloc(&ks.state, B * HW));
  OSB_TRY(res.alloc(&ks.surv, B * HW));
  OSB_TRY(res.alloc(&ks.cand, B * HW));
  OSB_TRY(res.alloc(&ks.skey, B * HW));
  OSB_TRY(res.alloc(&ks.cmask, B * 2 * HW));
  OSB_TRY(res.alloc(&ks.counts, B * 8));
  OSB_TRY(res.alloc(&ks.cnorm, B * 256));
  OSB_TRY(res.alloc(&d_nk, B));
  OSB_TRY(res.alloc(&d_kpts, B * max_num * 2));
  OSB_TRY(res.alloc(&d_conf, B * max_num));
  OSB_TRY(res.alloc(&d_out, B * max_num * 64));
  OSB_CUDA(cudaMemset(d_nk, 0, B * sizeof(int32_t)));
  OSB_CUDA(cudaMemset(ks.surv, 0, B * HW));
  return OSB_OK;
}

// tensor-core network: every activation is a pair of fp16 planes (hi, lo) scaled by SP_ACT_SCALE; the planes of a
// layer's output live in the ping-pong buffer the next layer's TMA descriptors point at.
osb_status SuperPoint::network_umma(const uint8_t* img_dev, int B, cudaStream_t st, const KpJob* kp, int zero_row) {
  const float SA = SP_ACT_SCALE;
  n_lev = 0;
  mark(st);
  // blanked band: the trunk's constant tiles are stored, not computed, and conv1a skips the pixels only they would read
  TileRect band_px[SP_TRUNK], band_tiles[SP_TRUNK], first_skip;
  const bool banded = zero_row >= 0 && band_c;
  if (banded) sp_band_geometry(H, W, zero_row, band_px, band_tiles, &first_skip);
  // conv layer i at resolution h x w; its output (optionally 2x2 max-pooled in the epilogue) becomes the input planes
  // of layer `out_layer`
  auto conv = [&](int i, int h, int w, int out_layer, int pool) {
    ConvBand band;
    if (banded && i < SP_TRUNK)
      band = ConvBand{band_tiles[i], band_const(precision, i, 0), band_const(precision, i, 1)};
    return umma_conv_forward(UL[i], tmA[i], tmB[i], B, h, w, SA, in_hi[out_layer], in_lo[out_layer], nullptr,
                             SP_COUT[i], SP_COUT[i], SA, 1, pool, st, 0, precision, &band);
  };
  OSB_TRY(umma_first_forward(w1a, b1a, lut, img_dev, in_hi[1], in_lo[1], B, H, W, SA, st, precision,
                             banded ? first_skip : TileRect{}));                               // conv1a -> A
  mark(st);
  OSB_TRY(conv(1, H, W, 2, 1));                                                               // conv1b + pool     -> B
  mark(st);
  OSB_TRY(conv(2, H / 2, W / 2, 3, 0));                                                       // conv2a            -> A
  mark(st);
  OSB_TRY(conv(3, H / 2, W / 2, 4, 1));                                                       // conv2b + pool     -> B
  mark(st);
  OSB_TRY(conv(4, H / 4, W / 4, 5, 0));                                                       // conv3a            -> A
  mark(st);
  OSB_TRY(conv(5, H / 4, W / 4, 6, 1));                                                       // conv3b + pool     -> B
  mark(st);
  OSB_TRY(conv(6, Hc, Wc, 7, 0));                                                             // conv4a            -> A
  mark(st);
  OSB_TRY(conv(7, Hc, Wc, 8, 0));                                                             // conv4b            -> B (x)
  mark(st);
  OSB_TRY(conv(8, Hc, Wc, 9, 0));                                                             // convPa            -> A
  mark(st);
  if (fused_softmax) {
    OSB_TRY(umma_conv_softmax_forward(UL[9], tmA[9], tmB[9], B, Hc, Wc, SA, d_semi, st, 0, precision));   // convPb + softmax + pixel shuffle
    mark(st);
  } else {
    OSB_TRY(umma_conv_forward(UL[9], tmA[9], tmB[9], B, Hc, Wc, SA, nullptr, nullptr, d_logits, 80, 80, 1.f, 0, 0, st, 0,
                              precision));   // convPb
    mark(st);
    OSB_TRY(sp_softmax_shuffle(d_logits, 80, d_semi, B, Hc, Wc, st));
  }
  // sparse head: the keypoints first, then the descriptor head at the cells they sample only
  sparse_ran = sparse_head && kp && !layer_prof;
  if (sparse_ran) {
    OSB_TRY(keypoints(B, *kp, st));
    return sparse_desc_head(B, *kp, st);
  }
  // the keypoint kernel (one CTA per image, latency-bound) runs beside the descriptor head, which leaves it B SMs
  const bool fork = kp && overlap_kp && !layer_prof && kp_stream;
  int head_ctas = 0;
  if (fork) {
    OSB_CUDA(cudaEventRecord(ev_semi, st));
    OSB_CUDA(cudaStreamWaitEvent(kp_stream, ev_semi, 0));
    OSB_TRY(keypoints(B, *kp, kp_stream));
    OSB_CUDA(cudaEventRecord(ev_kp, kp_stream));
    head_ctas = std::max(1, persistent_ctas() - B);
  }
  OSB_TRY(umma_conv_forward(UL[10], tmA[10], tmB[10], B, Hc, Wc, SA, in_hi[11], in_lo[11], nullptr, SP_COUT[10], SP_COUT[10],
                            SA, 1, 0, st, head_ctas, precision));                             // convDa (reads B)  -> A
  mark(st);
  OSB_TRY(umma_conv_forward(UL[11], tmA[11], tmB[11], B, Hc, Wc, SA, nullptr, nullptr, d_desc, 256, 256, 1.f, 0, 0, st,
                            head_ctas, precision));                                           // convDb
  mark(st);
  OSB_TRY(l2norm_cells(d_desc, (int64_t)B * Hc * Wc, 256, st));
  if (fork) OSB_CUDA(cudaStreamWaitEvent(st, ev_kp, 0));
  else if (kp) OSB_TRY(keypoints(B, *kp, st));
  return OSB_OK;
}

// the network: u8 images (device) -> d_semi, d_desc
osb_status SuperPoint::network(const uint8_t* img_dev, int B, cudaStream_t st, const KpJob* kp, int zero_row) {
  sparse_ran = false;
  if (use_umma) return network_umma(img_dev, B, st, kp, zero_row);
  OSB_TRY(conv_first_forward(w1a, b1a, lut, img_dev, actA, B, H, W, 64, 1, ACT_RELU, st));  // conv1a
  OSB_TRY(conv_forward(L[1], actA, actB, B, H, W, 64, ACT_RELU, st));                        // conv1b
  OSB_TRY(maxpool2x2_forward(actB, actA, B, H, W, 64, st));
  OSB_TRY(conv_forward(L[2], actA, actB, B, H / 2, W / 2, 64, ACT_RELU, st));                // conv2a
  OSB_TRY(conv_forward(L[3], actB, actA, B, H / 2, W / 2, 64, ACT_RELU, st));                // conv2b
  OSB_TRY(maxpool2x2_forward(actA, actB, B, H / 2, W / 2, 64, st));
  OSB_TRY(conv_forward(L[4], actB, actA, B, H / 4, W / 4, 128, ACT_RELU, st));               // conv3a
  OSB_TRY(conv_forward(L[5], actA, actB, B, H / 4, W / 4, 128, ACT_RELU, st));               // conv3b
  OSB_TRY(maxpool2x2_forward(actB, actA, B, H / 4, W / 4, 128, st));
  OSB_TRY(conv_forward(L[6], actA, actB, B, Hc, Wc, 128, ACT_RELU, st));                     // conv4a
  OSB_TRY(conv_forward(L[7], actB, actA, B, Hc, Wc, 128, ACT_RELU, st));                     // conv4b
  OSB_TRY(conv_forward(L[8], actA, actB, B, Hc, Wc, 256, ACT_RELU, st));                     // convPa
  OSB_TRY(conv_forward(L[9], actB, d_logits, B, Hc, Wc, 72, ACT_NONE, st));                  // convPb (65 -> stride 72)
  OSB_TRY(conv_forward(L[10], actA, actB, B, Hc, Wc, 256, ACT_RELU, st));                    // convDa
  OSB_TRY(conv_forward(L[11], actB, d_desc, B, Hc, Wc, 256, ACT_NONE, st));                  // convDb
  OSB_TRY(l2norm_cells(d_desc, (int64_t)B * Hc * Wc, 256, st));
  OSB_TRY(sp_softmax_shuffle(d_logits, 72, d_semi, B, Hc, Wc, st));
  if (kp) OSB_TRY(keypoints(B, *kp, st));
  return OSB_OK;
}

osb_status SuperPoint::keypoints(int B, const KpJob& kp, cudaStream_t st) {
  return sp_keypoints(d_semi, B, H, W, thres, max_num, ks, kp.nk, kp.kpts, kp.conf, st);
}

osb_status SuperPoint::descriptors(int B, const KpJob& kp, float* out, cudaStream_t st) {
  if (sparse_ran)
    return sp_descriptors(desc_c, B, H, W, kp.nk, kp.kpts, max_num, pca_compT, pca_mean_d, ks.cnorm, out, st, cell_slot, seg,
                          cell_n);
  return sp_descriptors(d_desc, B, H, W, kp.nk, kp.kpts, max_num, pca_compT, pca_mean_d, ks.cnorm, out, st);
}

osb_status SuperPoint::postprocess(int B, int32_t* nk, float* kpts, float* conf, float* out, cudaStream_t st) {
  sparse_ran = false;                   // the caller's map is in d_desc
  const KpJob kp{nk, kpts, conf};
  osb_status s = keypoints(B, kp, st);
  if (s != OSB_OK) return s;
  return descriptors(B, kp, out, st);
}

osb_status SuperPoint::forward(const uint8_t* img_dev, int B, int32_t* nk, float* kpts, float* conf, float* out,
                               cudaStream_t st) {
  OSB_REQUIRE(B > 0 && B <= max_batch, "batch out of range");
  const KpJob kp{nk, kpts, conf};
  osb_status s = network(img_dev, B, st, &kp);
  if (s != OSB_OK) return s;
  last_batch = B;
  return descriptors(B, kp, out, st);
}

osb_status SuperPoint::infer_dev(const uint8_t* img_dev, int B, int32_t* nk, float* kpts, float* out, cudaStream_t st) {
  return forward(img_dev, B, nk, kpts, d_conf, out, st);
}

}  // namespace osb

using namespace osb;

struct osb_superpoint {
  int device = 0;
  SuperPoint sp;
  std::mutex mu;
};

extern "C" osb_status osb_superpoint_create(osb_superpoint** out, const float* weights, size_t n_weights, int width,
                                            int height, float thres, int max_num, const float* pca_comp,
                                            const float* pca_mean, int max_batch) {
  OSB_REQUIRE(out != nullptr, "null out");
  OSB_TRY(require_device());
  std::unique_ptr<osb_superpoint> h(new osb_superpoint());
  h->device = current_device();
  OSB_TRY(h->sp.init(weights, n_weights, width, height, thres, max_num, pca_comp, pca_mean, max_batch));
  *out = h.release();
  return OSB_OK;
}

extern "C" osb_status osb_superpoint_destroy(osb_superpoint* h) {
  delete h;
  return OSB_OK;
}

static osb_status sp_copy_out(SuperPoint& sp, int B, int32_t* n_kpts, float* kpts, float* desc, cudaStream_t st) {
  OSB_CUDA(cudaMemcpyAsync(n_kpts, sp.d_nk, B * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  OSB_CUDA(cudaMemcpyAsync(kpts, sp.d_kpts, (size_t)B * sp.max_num * 2 * sizeof(float), cudaMemcpyDeviceToHost, st));
  OSB_CUDA(cudaMemcpyAsync(desc, sp.d_out, (size_t)B * sp.max_num * 64 * sizeof(float), cudaMemcpyDeviceToHost, st));
  OSB_CUDA(cudaStreamSynchronize(st));
  return OSB_OK;
}

extern "C" osb_status osb_superpoint_infer(osb_superpoint* h, const uint8_t* images, int batch, int32_t* n_kpts,
                                           float* kpts, float* desc) {
  OSB_REQUIRE(h && images && n_kpts && kpts && desc, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  SuperPoint& sp = h->sp;
  OSB_REQUIRE(batch > 0 && batch <= sp.max_batch, "batch out of range");
  cudaStream_t st = sp.stream;
  OSB_CUDA(cudaMemcpyAsync(sp.d_img, images, (size_t)batch * sp.H * sp.W, cudaMemcpyHostToDevice, st));
  osb_status s = sp.infer_dev(sp.d_img, batch, sp.d_nk, sp.d_kpts, sp.d_out, st);
  if (s != OSB_OK) return s;
  return sp_copy_out(sp, batch, n_kpts, kpts, desc, st);
}

extern "C" osb_status osb_superpoint_infer_dev(osb_superpoint* h, const uint8_t* images_dev, int batch,
                                               int32_t* n_kpts_dev, float* kpts_dev, float* desc_dev, void* stream) {
  OSB_REQUIRE(h && images_dev && n_kpts_dev && kpts_dev && desc_dev, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  return h->sp.infer_dev(images_dev, batch, n_kpts_dev, kpts_dev, desc_dev, (cudaStream_t)stream);
}

extern "C" osb_status osb_superpoint_postprocess(osb_superpoint* h, const float* semi, const float* desc_nchw,
                                                 int batch, int32_t* n_kpts, float* kpts, float* desc) {
  OSB_REQUIRE(h && semi && desc_nchw && n_kpts && kpts && desc, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  SuperPoint& sp = h->sp;
  OSB_REQUIRE(batch > 0 && batch <= sp.max_batch, "batch out of range");
  cudaStream_t st = sp.stream;
  const size_t HW = (size_t)sp.H * sp.W, dn = (size_t)256 * sp.Hc * sp.Wc;
  OSB_CUDA(cudaMemcpyAsync(sp.d_semi, semi, batch * HW * sizeof(float), cudaMemcpyHostToDevice, st));
  OSB_CUDA(cudaMemcpyAsync(sp.actA, desc_nchw, batch * dn * sizeof(float), cudaMemcpyHostToDevice, st));
  osb_status s = nchw_to_nhwc(sp.actA, sp.d_desc, batch, 256, sp.Hc, sp.Wc, st);
  if (s != OSB_OK) return s;
  sp.last_batch = batch;
  s = sp.postprocess(batch, sp.d_nk, sp.d_kpts, sp.d_conf, sp.d_out, st);
  if (s != OSB_OK) return s;
  return sp_copy_out(sp, batch, n_kpts, kpts, desc, st);
}

extern "C" osb_status osb_superpoint_set_profiling(osb_superpoint* h, int enable) {
  OSB_REQUIRE(h != nullptr, "null handle");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  h->sp.layer_prof = enable != 0;
  h->sp.n_lev = 0;
  return OSB_OK;
}

extern "C" osb_status osb_superpoint_set_precision(osb_superpoint* h, int precision) {
  OSB_REQUIRE(h != nullptr, "null handle");
  std::lock_guard<std::mutex> lk(h->mu);
  return h->sp.set_precision(precision);
}

extern "C" osb_status osb_superpoint_layer_ms(osb_superpoint* h, float* ms, int n) {
  OSB_REQUIRE(h != nullptr && ms != nullptr && n >= 12, "need room for 12 layer times");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  SuperPoint& sp = h->sp;
  OSB_CUDA(cudaStreamSynchronize(sp.stream));
  for (int i = 0; i < n; ++i) ms[i] = 0.f;
  for (int i = 0; i + 1 < sp.n_lev && i < n; ++i) {
    float t = 0.f;
    if (cudaEventElapsedTime(&t, sp.lev[i], sp.lev[i + 1]) == cudaSuccess) ms[i] = t; else cudaGetLastError();
  }
  return OSB_OK;
}

extern "C" osb_status osb_superpoint_band_geometry(int height, int width, int zero_row, int32_t* out) {
  OSB_REQUIRE(out != nullptr, "null out");
  OSB_REQUIRE(height > 0 && width > 0 && height % 8 == 0 && width % 8 == 0, "width/height must be multiples of 8");
  TileRect px[SP_TRUNK], tiles[SP_TRUNK], skip;
  sp_band_geometry(height, width, zero_row, px, tiles, &skip);
  auto put = [&](int32_t* o, const TileRect& r) { o[0] = r.y0; o[1] = r.y1; o[2] = r.x0; o[3] = r.x1; };
  for (int l = 0; l < SP_TRUNK; ++l) { put(out + 8 * l, px[l]); put(out + 8 * l + 4, tiles[l]); }
  put(out + 8 * SP_TRUNK, skip);
  return OSB_OK;
}

extern "C" osb_status osb_superpoint_read(osb_superpoint* h, int what, int image, float* out, size_t n_floats) {
  OSB_REQUIRE(h && out, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  SuperPoint& sp = h->sp;
  OSB_REQUIRE(image >= 0 && image < sp.max_batch, "image index out of range");
  cudaStream_t st = sp.stream;
  const size_t HW = (size_t)sp.H * sp.W, dn = (size_t)256 * sp.Hc * sp.Wc;
  if (what == 0) {
    OSB_REQUIRE(n_floats == HW, "semi needs H*W floats");
    OSB_CUDA(cudaMemcpyAsync(out, sp.d_semi + image * HW, HW * sizeof(float), cudaMemcpyDeviceToHost, st));
  } else if (what == 1) {
    OSB_REQUIRE(n_floats == dn, "desc needs 256*H/8*W/8 floats");
    osb_status s = nhwc_to_nchw(sp.d_desc + image * dn, sp.actB, 1, 256, sp.Hc, sp.Wc, st);
    if (s != OSB_OK) return s;
    OSB_CUDA(cudaMemcpyAsync(out, sp.actB, dn * sizeof(float), cudaMemcpyDeviceToHost, st));
  } else if (what == 2) {
    OSB_REQUIRE(n_floats == (size_t)sp.max_num, "conf needs max_num floats");
    OSB_CUDA(cudaMemcpyAsync(out, sp.d_conf + (size_t)image * sp.max_num, sp.max_num * sizeof(float),
                             cudaMemcpyDeviceToHost, st));
  } else if (what == 3) {
    OSB_REQUIRE(n_floats == HW, "survivor plane needs H*W floats");
    std::vector<uint8_t> tmp(HW);
    OSB_CUDA(cudaMemcpyAsync(tmp.data(), sp.ks.surv + image * HW, HW, cudaMemcpyDeviceToHost, st));
    OSB_CUDA(cudaStreamSynchronize(st));
    for (size_t i = 0; i < HW; ++i) out[i] = (float)tmp[i];
    return OSB_OK;
  } else if (what == 4) {
    OSB_REQUIRE(n_floats == 8, "counts needs 8 floats");
    int32_t c[8];
    OSB_CUDA(cudaMemcpyAsync(c, sp.ks.counts + image * 8, sizeof(c), cudaMemcpyDeviceToHost, st));
    OSB_CUDA(cudaStreamSynchronize(st));
    for (int i = 0; i < 8; ++i) out[i] = (float)c[i];
    return OSB_OK;
  } else {
    set_error("osb_superpoint_read", "unknown `what`");
    return OSB_ERR_INVALID;
  }
  OSB_CUDA(cudaStreamSynchronize(st));
  return OSB_OK;
}
