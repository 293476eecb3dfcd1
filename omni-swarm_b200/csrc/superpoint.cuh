// superpoint.cuh -- internal SuperPoint / NetVLAD objects (shared by the C-ABI wrappers and the keyframe front-end)
#pragma once
#include "common.cuh"
#include "kernels.cuh"
#include "conv_umma.cuh"

namespace osb {

size_t sp_expected_weights();
size_t nv_expected_weights();

// a network's precision switch: OSB_PRECISION_FP16 needs the tensor-core path (not OSB_SP_CONV=ffma)
inline osb_status umma_set_precision(bool use_umma, int* precision, int p) {
  OSB_REQUIRE(p == OSB_PRECISION_SPLIT_FP16 || p == OSB_PRECISION_FP16,
              "precision must be OSB_PRECISION_SPLIT_FP16 or OSB_PRECISION_FP16");
  OSB_REQUIRE(use_umma || p == OSB_PRECISION_SPLIT_FP16,
              "plain fp16 needs the tensor-core convolutions (the handle was created under OSB_SP_CONV=ffma)");
  *precision = p;
  return OSB_OK;
}

struct SuperPoint {
  Resources res;                   // every buffer, stream and event below
  int W = 0, H = 0, Wc = 0, Hc = 0, max_num = 0, max_batch = 0, last_batch = 0;
  float thres = 0.f;
  cudaStream_t stream = nullptr;
  // weights
  float *w1a = nullptr, *b1a = nullptr, *lut = nullptr, *pca_compT = nullptr, *pca_mean_d = nullptr;
  ConvLayer L[12];
  // activations / outputs (device)
  uint8_t* d_img = nullptr;
  float *actA = nullptr, *actB = nullptr, *d_logits = nullptr, *d_semi = nullptr, *d_desc = nullptr;
  KeypointScratch ks;
  int32_t* d_nk = nullptr;
  float *d_kpts = nullptr, *d_conf = nullptr, *d_out = nullptr;

  // tensor-core path (conv_umma.cu): weights as split fp16 planes, one pair of TMA descriptors per conv input
  bool use_umma = true;
  int precision = OSB_PRECISION_SPLIT_FP16;   // of the tensor-core path; fp16 reads and writes the hi planes only
  UmmaLayer UL[12];
  CUtensorMap tmA[12], tmB[12];     // [layer] -> (hi, lo) descriptors of that layer's INPUT planes
  __half *in_hi[12] = {}, *in_lo[12] = {};
  // blanked band (network's zero_row): per precision and trunk layer (conv1a .. conv4b), the hi and lo planes of the
  // layer's constant output, 128 channels apart.  Null until band_init; while it is null, network ignores zero_row.
  __half* band_c = nullptr;
  const __half* band_const(int prec, int layer, int plane) const;
  // computes band_c with each layer's own kernel on a zero image (both precisions); synchronizes `stream`
  osb_status band_init();
  // sparse descriptor head (front-end only, after sparse_init): convDa and convDb at the cells the keypoints' bilinear
  // taps read (sp_cell_gather), the L2 norm inside the descriptor kernels.  convDa runs as a 1x1 layer (UDa_col: 9 x 128
  // inputs in the 3x3 layer's K order) over those cells' gathered neighbourhoods, so each computed cell is bit-identical to
  // the dense map's.  Rows of image b: b * seg .. b * seg + seg - 1, seg a multiple of the 128-cell tile.
  // OSB_SP_SPARSE_HEAD=0 keeps the dense head.
  UmmaLayer UDa_col;
  bool sparse_head = false, sparse_ran = false;      // sparse_ran: the last network() left desc_c + cell_slot, not d_desc
  int seg = 0;
  int32_t* cell_slot = nullptr;
  __half *col_hi = nullptr, *col_lo = nullptr, *da_hi = nullptr, *da_lo = nullptr;
  float *desc_c = nullptr, *cell_n = nullptr;
  CUtensorMap tm_col[2], tm_da[2];
  osb_status sparse_init();
  // per-layer timing (debug / bench): ev[i] is recorded after launch i of the network when `layer_prof` is set
  bool layer_prof = false;
  cudaEvent_t lev[20] = {};
  int n_lev = 0;
  void mark(cudaStream_t st) { if (layer_prof && n_lev < 20) { if (!lev[n_lev]) res.event(&lev[n_lev]); cudaEventRecord(lev[n_lev++], st); } }

  osb_status init(const float* weights, size_t n_weights, int width, int height, float thres, int max_num,
                  const float* pca_comp, const float* pca_mean, int max_batch);
  osb_status set_precision(int p) { return umma_set_precision(use_umma, &precision, p); }
  // keypoint extraction needs only the detector head: when a KpJob is passed, the network launches it on `kp_stream`
  // as soon as the heat map exists and runs the descriptor head beside it (on B fewer SMs); `st` re-joins before return
  struct KpJob { int32_t* nk; float* kpts; float* conf; };
  osb_status sparse_desc_head(int B, const KpJob& kp, cudaStream_t st);
  cudaStream_t kp_stream = nullptr;
  cudaEvent_t ev_semi = nullptr, ev_kp = nullptr;
  bool overlap_kp = true;
  bool fused_softmax = true;       // detector-head softmax + pixel shuffle in convPb's epilogue (OSB_SP_FUSED_SOFTMAX=0: two kernels)
  // zero_row >= 0: rows zero_row .. H - 1 of every image are zero, so the tensor-core trunk skips the tiles whose output is
  // the layer's constant (after band_init; DESIGN.md section 3)
  osb_status network(const uint8_t* img_dev, int B, cudaStream_t st, const KpJob* kp = nullptr, int zero_row = -1);
  osb_status network_umma(const uint8_t* img_dev, int B, cudaStream_t st, const KpJob* kp, int zero_row);
  osb_status keypoints(int B, const KpJob& kp, cudaStream_t st);
  osb_status descriptors(int B, const KpJob& kp, float* out, cudaStream_t st);
  // network + keypoints + descriptors (what inference() is)
  osb_status forward(const uint8_t* img_dev, int B, int32_t* nk, float* kpts, float* conf, float* out, cudaStream_t st);
  osb_status postprocess(int B, int32_t* nk, float* kpts, float* conf, float* out, cudaStream_t st);
  osb_status infer_dev(const uint8_t* img_dev, int B, int32_t* nk, float* kpts, float* out, cudaStream_t st);
};

struct NetVLAD {
  Resources res;                   // every buffer and the stream below
  int W = 0, H = 0, max_batch = 0;
  cudaStream_t stream = nullptr;
  float *w0 = nullptr, *b0 = nullptr, *lut = nullptr, *pw0_kc = nullptr, *pw0_b = nullptr;
  struct Block { float *dw = nullptr, *dwb = nullptr; ConvLayer pw; int cin = 0, cout = 0, stride = 1; } blk[7];
  ConvLayer proj, assign;
  float* centroids = nullptr;
  uint8_t* d_img = nullptr;
  float *actA = nullptr, *actB = nullptr, *d_assign = nullptr, *d_out = nullptr;
  float *d_mu = nullptr, *d_part = nullptr, *d_psum = nullptr;
  // tensor-core pointwise path: blocks 1..6 and the projection read split fp16 planes written by the depthwise kernel
  bool use_umma = true;
  int precision = OSB_PRECISION_SPLIT_FP16;
  UmmaLayer upw[7], uproj;
  CUtensorMap tmA[8], tmB[8];           // [block] (7 = projection) descriptors of the pointwise conv's input planes
  __half *pl_hi[8] = {}, *pl_lo[8] = {};
  __half* planes = nullptr;

  osb_status init(const float* weights, size_t n_weights, int width, int height, int max_batch);
  osb_status set_precision(int p) { return umma_set_precision(use_umma, &precision, p); }
  osb_status infer_dev(const uint8_t* img_dev, int B, float* out_dev, cudaStream_t st);
};

}  // namespace osb
