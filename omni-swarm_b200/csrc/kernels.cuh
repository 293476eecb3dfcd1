// kernels.cuh -- internal (non-ABI) launchers shared between the translation units of libomniswarm_b200.
#pragma once
#include "common.cuh"

namespace osb {

// ---- match.cu ------------------------------------------------------------------------------------------------
int db_scan_grid(int64_t n, int64_t* chunk_out);
// rows: [n][dim] float, or __half with storage == OSB_DB_STORAGE_FP16 (the queries stay fp32)
// n_dev (optional): true row count in device memory, n is then an upper bound used to size the grid
osb_status db_search_device(const void* rows, int storage, int64_t n, const int64_t* n_dev, int dim, const float* q_dev,
                            int nq, int k, float* part_scores, int64_t* part_ids, unsigned int* done, float* scores_dev,
                            int64_t* ids_dev, cudaStream_t st);
// the row plane of a database: n elements of float, or of __half for OSB_DB_STORAGE_FP16, owned by `m`
osb_status db_rows_alloc(Resources& m, void** rows, size_t n, int storage);
// dst[i] = __float2half_rn(src[i]) for n elements (n a multiple of 4) of device memory, on `st`
osb_status db_rows_to_half(__half* dst, const float* src, size_t n, cudaStream_t st);
// q/t: device tables of n_pairs pointers to [<=max_n][64] descriptor blocks
// outputs (qi/ti/dout/map_out) are [n_pairs][out_stride] and n_out [n_pairs] -- or, with group > 0, pair p = group * g + s
// writes them at g * group_stride + s * out_stride and g * group_stride + s (elements): the pairs of record g land in the
// g-th of an array of structs
osb_status bf_match_device(int n_pairs, int max_n, int out_stride, const float* const* q, const int32_t* nq,
                           const float* const* t,
                           const int32_t* nt, float* dist_scratch, int32_t* qi, int32_t* ti, float* dout,
                           int32_t* n_out, int32_t* map_out, cudaStream_t st, int group = 0, size_t group_stride = 0);

// ---- conv_ffma.cu --------------------------------------------------------------------------------------------
enum Act { ACT_NONE = 0, ACT_RELU = 1, ACT_RELU6 = 2 };

// Weights of one dense conv layer repacked for the FFMA kernel: [tap][Cin][Cout_pad] + bias[Cout_pad].
struct ConvLayer {
  int cin = 0, cout = 0, cout_pad = 0, ks = 1;
  float* w = nullptr;     // device
  float* b = nullptr;     // device
};
// the weight buffers belong to `res`
osb_status conv_layer_upload(Resources& res, ConvLayer* L, const float* w_oihw, const float* bias, int cin, int cout, int ks);
// 3x3 one-input-channel weights [cout][9] (OIHW) -> new device buffer of `res` as [9][cout]
osb_status upload_tap_major(Resources& res, float** dst, const float* w_oihw, int cout);

// y[B][H][W][out_cstride] = act(conv_ks(x[B][H][W][Cin]) + b)   (NHWC, stride 1, "same" padding)
osb_status conv_forward(const ConvLayer& L, const float* x, float* y, int B, int H, int W, int out_cstride,
                        int act, cudaStream_t st);
// first layer: u8 image [B][H][W] -> [B][H/stride][W/stride][COUT], 3x3 pad 1, input value LUT (256 floats, device)
osb_status conv_first_forward(const float* w_tap_cout /*[9][cout]*/, const float* bias, const float* lut,
                              const uint8_t* img, float* y, int B, int H, int W, int cout, int stride, int act,
                              cudaStream_t st);
osb_status maxpool2x2_forward(const float* x, float* y, int B, int H, int W, int C, cudaStream_t st);
// depthwise 3x3 pad 1 stride s: w [9][C], NHWC
osb_status dwconv3x3_forward(const float* w_tap_c, const float* bias, const float* x, float* y, int B, int H, int W,
                             int C, int stride, int act, cudaStream_t st);

// ---- postproc.cu ---------------------------------------------------------------------------------------------
// detector head: logits [B][Hc][Wc][cstride>=65] -> semi [B][Hc*8][Wc*8]  (softmax over 65, drop dustbin, 8x8 shuffle)
osb_status sp_softmax_shuffle(const float* logits, int cstride, float* semi, int B, int Hc, int Wc, cudaStream_t st);
// descriptor head: in-place L2 normalisation over `C` channels of every cell of [cells][C]
osb_status l2norm_cells(float* x, int64_t cells, int C, cudaStream_t st);

struct KeypointScratch {   // per handle, sized for max_batch images
  uint8_t* state = nullptr;     // [B][H*W]
  uint8_t* surv = nullptr;      // [B][H*W]
  int32_t* cand = nullptr;      // [B][H*W]
  unsigned long long* skey = nullptr;  // [B][H*W]
  unsigned long long* cmask = nullptr; // [B][2][H*W] earlier / later stronger-neighbour bit masks per candidate
  bool write_surv = true;              // maintain the survivor plane (parity hook `read(3)`); off in the front-end
  int32_t* counts = nullptr;    // [B][8]: M candidates, S survivors, rounds, reserved, SM cycles of phases 1..4
  float* cnorm = nullptr;       // [B][256]
};
osb_status sp_keypoints(const float* semi, int B, int H, int W, float thres, int max_num, KeypointScratch& ks,
                        int32_t* n_kpts, float* kpts, float* conf, cudaStream_t st);
// desc_nhwc [B][Hc][Wc][256]; kpts [B][max_num][2]; out [B][max_num][64].  With `slot` ([B][Hc][Wc], sp_cell_gather)
// desc_nhwc is convDb's output at the listed cells only, [B * seg][256] and not yet L2-normalised: the kernels divide each
// tap by its row's norm (kept in cell_n [B * seg]), the value l2norm_cells would have stored
osb_status sp_descriptors(const float* desc_nhwc, int B, int H, int W, const int32_t* n_kpts, const float* kpts,
                          int max_num, const float* pca_compT /*[256][64]*/, const float* pca_mean, float* cnorm, float* out,
                          cudaStream_t st, const int32_t* slot = nullptr, int seg = 0, float* cell_n = nullptr);
// sparse descriptor head: the cells the keypoints' bilinear taps read, numbered row-major per image into segments of
// `seg` rows (slot [B][Hc][Wc], -1 where unsampled), and convDa's input at them: x [B][Hc][Wc][128] split planes ->
// col [B * seg][1152] (9 taps x 128 channels in conv_stream_t_kernel's K order, zero for padding rows)
osb_status sp_cell_gather(int B, int H, int W, const int32_t* n_kpts, const float* kpts, int max_num, int seg, int32_t* slot,
                          const __half* x_hi, const __half* x_lo, __half* col_hi, __half* col_lo, bool fp16,
                          cudaStream_t st);
// layout helper: [B][C][h][w] -> [B][h][w][C]
osb_status nchw_to_nhwc(const float* in, float* out, int B, int C, int h, int w, cudaStream_t st);
osb_status nhwc_to_nchw(const float* in, float* out, int B, int C, int h, int w, cudaStream_t st);

// ---- geom.cu ---------------------------------------------------------------------------------------------------
// homography-RANSAC inlier masks of n_pairs correspondence sets ([n_pairs][max_n] float2 old / new points)
// stereo triangulation of the matched up/down keypoints of n_dirs directions (lift.cu; loop_cam.cpp:393-432); down_main:
// the points go to the down keypoints' slots (LOWER_CAM_AS_MAIN)
osb_status stereo_lift_device(const float* kp_up, const float* kp_down, const int32_t* match, const int32_t* n_up,
                              const int32_t* n_down, int n_dirs, int max_n, const double* K, const double* pose_up,
                              const double* pose_down, double triangle_thres, int min_pts, float* pts3d, uint8_t* flag_up,
                              uint8_t* flag_down, cudaStream_t st, bool down_main = false);
// depth look-up lift of the keypoints of n_dirs directions (lift.cu; loop_cam.cpp:276-302)
osb_status depth_lift_device(const float* kp, const int32_t* n_kp, int n_dirs, int max_n, const uint16_t* depth_mm, int H,
                             int W, const double* K, const double* pose_cam, double near_thres, double far_thres,
                             int min_pts, float* pts3d, uint8_t* flag, cudaStream_t st);
osb_status homography_ransac_device(const float* src_dev, const float* dst_dev, const int32_t* n_dev, int n_pairs, int max_n,
                                    float thresh, uint32_t seed, uint8_t* mask_dev, int32_t* n_inl_dev, int32_t* winner_dev,
                                    cudaStream_t st, unsigned int* scratch /* 2 * n_pairs words, zero between launches */);

// ---- pnp.cu ----------------------------------------------------------------------------------------------------
// deterministic PnP-RANSAC + the reference's checks, one CTA of PNP_THREADS per candidate (osb_pnp_ransac_dev; also launched
// by osb_frontend_compute_loop on the correspondences it assembles).  max_n <= PNP_MAXN.
constexpr int PNP_THREADS = 256;
constexpr int PNP_MAXN = 1024;
__global__ void __launch_bounds__(PNP_THREADS)
pnp_ransac_kernel(const float* __restrict__ pts3d, const float* __restrict__ pts2d, const int32_t* __restrict__ n_pts, int max_n,
                  const osb_pnp_params* __restrict__ params, uint8_t* __restrict__ mask_out, osb_pnp_result* __restrict__ results);

}  // namespace osb
