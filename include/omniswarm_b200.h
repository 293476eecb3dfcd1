/*
 * omniswarm_b200.h -- C ABI of libomniswarm_b200.so
 *
 * H100-native (sm_90a) replacement for the ONE compute-heavy path of HKUST-Aerial-Robotics/Omni-swarm:
 * the swarm_loop keyframe front-end and the swarm_localization pose-graph solve.  The reference has no
 * plugin ABI for this path (the boundary is C++ member calls inside one process, SURVEY.md section 8b);
 * every entry point below names the reference call site it replaces (paths relative to /root/reference).
 * INTEGRATION.md shows the thin C++ adapter classes a maintainer adds so that loop_cam.cpp /
 * loop_detector.cpp / swarm_localization_solver.cpp keep their signatures.
 *
 * Conventions
 *   - plain C types only; every function returns an osb_status (0 = OK) and never throws;
 *   - "host" entry points take HOST pointers and do their own H2D/D2H (the drop-in calls);
 *     "_dev" entry points take DEVICE pointers plus a cudaStream_t (passed as void*) and never synchronise:
 *     they exist so that a caller that already owns device memory (bench.py, the multi-GPU keyframe exchange)
 *     can keep everything resident;
 *   - all device memory is owned by the opaque handles for their lifetime (as the reference's
 *     TensorRTInferenceGeneric does, swarm_loop/src/tensorrt_generic.cpp:99-120).  destroy() releases every
 *     buffer, stream and event that create() and later calls acquired; a create() that fails leaves nothing
 *     behind, and so does a host entry point that fails;
 *   - handles are internally serialised (one stream + one mutex per handle): the reference calls
 *     LoopDetector from the ROS thread and the LCM thread without a lock (SURVEY.md section 3.1);
 *   - there is NO CPU fallback: without a CUDA device every create() returns OSB_ERR_NO_DEVICE.
 */
#ifndef OMNISWARM_B200_H
#define OMNISWARM_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef int osb_status;
#define OSB_OK 0
#define OSB_ERR_INVALID 1    /* bad argument (null pointer, size mismatch, batch > max_batch ...) */
#define OSB_ERR_CUDA 2       /* a CUDA call failed; osb_last_error() has the text */
#define OSB_ERR_CAPACITY 3   /* database / solver capacity exceeded */
#define OSB_ERR_NO_DEVICE 4  /* no CUDA device: this library has no CPU path */

#define OSB_SP_DESC_RAW_LEN 256   /* SP_DESC_RAW_LEN, swarm_loop/include/swarm_loop/loop_defines.h */
#define OSB_FEATURE_DESC_SIZE 64  /* FEATURE_DESC_SIZE, loop_defines.h:67 */
#define OSB_DEEP_DESC_SIZE 4096   /* DEEP_DESC_SIZE,    loop_defines.h:30 */
#define OSB_MAX_DIRS 4            /* MAX_DIRS for STEREO_FISHEYE, swarm_loop/src/swarm_loop.cpp:277-278 */
#define OSB_MAX_KPTS 200          /* superpoint_max_num, swarm_loop/launch/nodelet-sfisheye.launch:30 */
#define OSB_REMOTE_MAGIN_NUMBER 1000000  /* REMOTE_MAGIN_NUMBER, swarm_loop/include/swarm_loop/loop_detector.h:22 */

const char* osb_last_error(void);          /* thread-local text of the last failure */
const char* osb_version(void);
int osb_device_count(void);                /* 0 when no CUDA device is visible */

/* ------------------------------------------------------------------------------------------------------------
 * SuperPoint  -- replaces class SuperPointTensorRT (swarm_loop/include/swarm_loop/superpoint_tensorrt.h:20-28,
 *               constructed at swarm_loop/src/loop_cam.cpp:26, called at loop_cam.cpp:542).
 * `weights`: float32 blob, for each layer of swarm_loop/superpoint.ipynb:143-158 in definition order
 *            (conv1a,conv1b,conv2a,conv2b,conv3a,conv3b,conv4a,conv4b,convPa,convPb,convDa,convDb):
 *            weight in PyTorch OIHW order, then bias.  1 300 865 floats.  (Replaces the .trt engine path:
 *            TensorRT engine binaries are device-specific and not portable.)
 * `pca_comp` [64][256] row-major = components_.csv, `pca_mean` [256] = mean_.csv (superpoint_tensorrt.cpp:110-111).
 * infer():   images  [batch][height][width] uint8 (the reference asserts the size, superpoint_tensorrt.cpp:122)
 *            n_kpts  [batch]                          number of keypoints per image (<= max_num)
 *            kpts    [batch][max_num][2] float (x,y)  ordered by descending confidence (NMS2, :304-308)
 *            desc    [batch][max_num][64] float       PCA-projected descriptors (:221)
 *            rows >= n_kpts[b] are left untouched.
 * -----------------------------------------------------------------------------------------------------------*/
typedef struct osb_superpoint osb_superpoint;
osb_status osb_superpoint_create(osb_superpoint** out, const float* weights, size_t n_weights, int width,
                                 int height, float thres, int max_num, const float* pca_comp,
                                 const float* pca_mean, int max_batch);
osb_status osb_superpoint_destroy(osb_superpoint* h);
osb_status osb_superpoint_infer(osb_superpoint* h, const uint8_t* images, int batch, int32_t* n_kpts,
                                float* kpts, float* desc);
osb_status osb_superpoint_infer_dev(osb_superpoint* h, const uint8_t* images_dev, int batch, int32_t* n_kpts_dev,
                                    float* kpts_dev, float* desc_dev, void* stream);
/* Stage-wise parity hooks (tests only; not used by the reference call sites):
 *  set_heatmap: upload a caller-supplied `semi` [batch][H][W] and `desc` [batch][256][H/8][W/8] (the two engine
 *               outputs, superpoint_tensorrt.cpp:139-140) and run ONLY getKeyPoints+NMS2+computeDescriptors.
 *  read:        copy an intermediate of the last infer() back: what = 0 semi [H][W], 1 desc [256][H/8][W/8],
 *               2 confidences of the returned keypoints [max_num], 3 NMS survivor plane as float [H][W],
 *               4 keypoint kernel counters [8]: candidates, survivors, NMS rounds, 0, SM cycles of its 4 phases. */
osb_status osb_superpoint_postprocess(osb_superpoint* h, const float* semi, const float* desc_nchw, int batch,
                                      int32_t* n_kpts, float* kpts, float* desc);
osb_status osb_superpoint_read(osb_superpoint* h, int what, int image, float* out, size_t n_floats);
/* per-layer device time of the last infer() (bench / profiling aid; tensor-core path only): enable, run infer(), then
 * layer_ms fills ms[0..11] = conv1a, conv1b(+pool), conv2a, conv2b(+pool), conv3a, conv3b(+pool), conv4a, conv4b, convPa,
 * convPb, convDa, convDb in milliseconds (CUDA events on the handle's stream). */
osb_status osb_superpoint_set_profiling(osb_superpoint* h, int enable);
osb_status osb_superpoint_layer_ms(osb_superpoint* h, float* ms, int n);
/* Network precision of the tensor-core path (SuperPoint, NetVLAD, and both networks of the front-end):
 *  OSB_PRECISION_SPLIT_FP16 (the default): every operand is carried as two fp16 planes and each K step computes three
 *    products, which matches an fp32 network to ~1e-6 relative;
 *  OSB_PRECISION_FP16: plain fp16 operands (the precision of the reference's fp16 TensorRT engines): the hi planes only,
 *    one product per K step, fp32 accumulation.  Heat-map and descriptors move by ~1e-3 (DESIGN.md section 3).
 * The weights are uploaded once and both precisions read them; switching acquires nothing and is serialised with the
 * handle's other calls, and switching back gives the outputs of a handle that never switched.  A handle created under
 * OSB_SP_CONV=ffma (fp32 CUDA cores) accepts only OSB_PRECISION_SPLIT_FP16 (OSB_ERR_INVALID otherwise).  Everything
 * outside the convolutions (conv1a's arithmetic, softmax, L2 norms, keypoints, NetVLAD's head) stays fp32. */
#define OSB_PRECISION_SPLIT_FP16 0
#define OSB_PRECISION_FP16 1
osb_status osb_superpoint_set_precision(osb_superpoint* h, int precision);
/* Geometry of the blanked band (tests only; no device needed): for images of height x width whose rows >= zero_row are
 * zero, the front-end's SuperPoint skips the trunk's (conv1a .. conv4b) tiles whose output is the layer's constant.
 * out [68] int32: for each trunk layer l, out[8l .. 8l+3] = its constant output pixels (after the pool) and
 * out[8l+4 .. 8l+7] = its constant 8 x 16 output tiles (before the pool), each as y0, y1, x0, x1 of [y0, y1) x [x0, x1);
 * out[64 .. 67] = the conv1a pixels that no computed conv1b tile reads.  An empty set has y0 >= y1 or x0 >= x1. */
osb_status osb_superpoint_band_geometry(int height, int width, int zero_row, int32_t* out);

/* Convolution parity hooks (tests only): ONE layer of the tensor-core path, run by the same host functions and kernels
 * as the SuperPoint / NetVLAD networks, on caller-supplied operands.  Weights and biases are HOST fp32, OIHW; activation
 * operands are DEVICE pointers; every call synchronises `stream` (a cudaStream_t as void*, 0 = default stream).
 * Split planes are fp16 NHWC [batch][H][W][C] pairs hi = fp16(s * x), lo = fp16(s * x - hi) with s a power of two.
 *  conv_layer:  w [cout][cin][ks][ks] (cin a multiple of 64, cout <= 512, ks 1 or 3) split at w_scale (the networks use
 *               1024); in_hi/in_lo the input planes at act_scale.  relu 0 none / 1 ReLU / 2 ReLU6, pool 1 = fused 2x2
 *               max-pool (even H and W), out_c channels stored (a multiple of 16), max_ctas 0 = one CTA per SM.
 *               mode 0: out_f32 [batch*Ho*Wo][out_cstride]; mode 1: planes out_hi/out_lo [batch][Ho][Wo][out_cstride] at
 *               out_scale; mode 2: the detector head (cout 65, ks 1): softmax, dustbin dropped, 8x8 pixel shuffle into
 *               out_f32 = heat map [batch][8H][8W].
 *  conv_first:  SuperPoint conv1a (w1a [64][1][3][3]) + ReLU on u8 images [batch][H][W] (scaled by 1/255) -> the conv1a
 *               planes [batch][H][W][64] at act_scale.
 *  dwconv:      depthwise 3x3 (w [C][1][3][3], pad 1, stride 1 or 2) + bias + ReLU6 on fp32 NHWC x [batch][H][W][C]
 *               -> planes [batch][H/stride][W/stride][C] at out_scale; generic = 1 runs the one-pixel kernel at stride 1
 *               instead of the four-pixel one. */
osb_status osb_conv_layer_parity(const float* w, const float* bias, int cin, int cout, int ks, float w_scale,
                                 const void* in_hi, const void* in_lo, int batch, int height, int width, float act_scale,
                                 int relu, int pool, int out_c, int out_cstride, int max_ctas, int mode, float* out_f32,
                                 void* out_hi, void* out_lo, float out_scale, void* stream);
osb_status osb_conv_first_parity(const float* w1a, const float* b1a, const uint8_t* images_dev, int batch, int height,
                                 int width, float act_scale, void* out_hi, void* out_lo, void* stream);
osb_status osb_dwconv_parity(const float* w, const float* bias, const float* x_dev, int batch, int height, int width,
                             int channels, int stride, int generic, float out_scale, void* out_hi, void* out_lo,
                             void* stream);
/* The same three in OSB_PRECISION_FP16: one fp16 plane in_hi = fp16(s * x) in, one plane out_hi out (no lo planes). */
osb_status osb_conv_layer_fp16_parity(const float* w, const float* bias, int cin, int cout, int ks, float w_scale,
                                      const void* in_hi, int batch, int height, int width, float act_scale, int relu,
                                      int pool, int out_c, int out_cstride, int max_ctas, int mode, float* out_f32,
                                      void* out_hi, float out_scale, void* stream);
osb_status osb_conv_first_fp16_parity(const float* w1a, const float* b1a, const uint8_t* images_dev, int batch,
                                      int height, int width, float act_scale, void* out_hi, void* stream);
osb_status osb_dwconv_fp16_parity(const float* w, const float* bias, const float* x_dev, int batch, int height,
                                  int width, int channels, int stride, int generic, float out_scale, void* out_hi,
                                  void* stream);
/* The same for the fp32 CUDA-core path (OSB_SP_CONV=ffma, and the layers both paths run in fp32); fp32 NHWC device
 * operands, act 0 none / 1 ReLU / 2 ReLU6:
 *  conv_ffma:       w [cout][cin][ks][ks] (cin a multiple of 8, ks 1 or 3), x [batch][H][W][cin] ->
 *                   y [batch][H][W][out_cstride] (out_cstride a multiple of 8 in [cout, cout rounded up to 64]; the
 *                   channels in [cout, out_cstride) are stored as 0).
 *  conv_first_ffma: w [cout][1][3][3] (cout 32 or 64) on u8 images [batch][H][W] (scaled by 1/255), pad 1, stride 1 or 2
 *                   -> y [batch][H/stride][W/stride][cout].
 *  dwconv_ffma:     depthwise 3x3, w [C][1][3][3], pad 1, stride 1 or 2 -> y [batch][H/stride][W/stride][C].
 *  maxpool:         2x2 max-pool, x [batch][H][W][C] (C a multiple of 4) -> y [batch][H/2][W/2][C]. */
osb_status osb_conv_ffma_parity(const float* w, const float* bias, int cin, int cout, int ks, const float* x_dev,
                                int batch, int height, int width, int act, int out_cstride, float* y_dev, void* stream);
osb_status osb_conv_first_ffma_parity(const float* w, const float* bias, int cout, int stride, int act,
                                      const uint8_t* images_dev, int batch, int height, int width, float* y_dev,
                                      void* stream);
osb_status osb_dwconv_ffma_parity(const float* w, const float* bias, const float* x_dev, int batch, int height, int width,
                                  int channels, int stride, int act, float* y_dev, void* stream);
osb_status osb_maxpool_parity(const float* x_dev, int batch, int height, int width, int channels, float* y_dev,
                              void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * NetVLAD global descriptor -- replaces class MobileNetVLADTensorRT
 *   (swarm_loop/include/swarm_loop/mobilenetvlad_tensorrt.h:10-21, loop_cam.cpp:27 ctor, loop_cam.cpp:554 call).
 * images [batch][H][W] uint8 (converted to float UNSCALED, mobilenetvlad_tensorrt.cpp:8-10) -> out [batch][4096].
 * The hfnet MobileNetVLAD architecture is not part of the reference; DESIGN.md pins the stand-in whose weight
 * blob layout is omniswarm_b200/synth.py::netvlad_layer_table().
 * -----------------------------------------------------------------------------------------------------------*/
typedef struct osb_netvlad osb_netvlad;
osb_status osb_netvlad_create(osb_netvlad** out, const float* weights, size_t n_weights, int width, int height,
                              int max_batch);
osb_status osb_netvlad_destroy(osb_netvlad* h);
osb_status osb_netvlad_infer(osb_netvlad* h, const uint8_t* images, int batch, float* out);
osb_status osb_netvlad_infer_dev(osb_netvlad* h, const uint8_t* images_dev, int batch, float* out_dev, void* stream);
/* OSB_PRECISION_SPLIT_FP16 / OSB_PRECISION_FP16 of the pointwise convolutions (see osb_superpoint_set_precision) */
osb_status osb_netvlad_set_precision(osb_netvlad* h, int precision);
/* NetVLAD parity hooks (tests only): two parts of the network run by the host functions osb_netvlad_infer_dev calls,
 * conventions as the convolution hooks above (host OIHW weights, device fp32 NHWC activations, one synchronise):
 *  nv_block0: block 0 of the default path, depthwise 3x3 (dw_w [32][1][3][3]) + ReLU6 -> pointwise pw_w [64][32][1][1] +
 *             ReLU6, x [batch][H][W][32] -> y [batch][H][W][64].
 *  nv_head:   from the projected features x [batch][H][W][128]: mu [batch][128] (per-image mean), xn = (x - mu) / ||x - mu||
 *             per location, logits [batch][H][W][32] of assign_w [32][128][1][1], their softmax `assign`, and the
 *             4096-vector out [batch][32*128] (VLAD with centroids [32][128], intra- and global L2 normalisation). */
osb_status osb_nv_block0_parity(const float* dw_w, const float* dw_b, const float* pw_w, const float* pw_b,
                                const float* x_dev, int batch, int height, int width, float* y_dev, void* stream);
osb_status osb_nv_head_parity(const float* assign_w, const float* assign_b, const float* centroids, const float* x_dev,
                              int batch, int height, int width, float* mu_dev, float* xn_dev, float* logits_dev,
                              float* assign_dev, float* out_dev, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Keyframe database -- replaces faiss::IndexFlatIP(4096) (swarm_loop/include/swarm_loop/loop_detector.h:27-29;
 *   add: loop_detector.cpp:166,169; search: loop_detector.cpp:213; ntotal: loop_detector.cpp:291).
 * Exact float32 inner product, top-k by descending score, ties by ascending row id, ids = -1 and
 * scores = -inf where fewer than k rows exist.  Rows live in HBM, row-major [capacity][dim].
 *
 * Row storage (osb_db_create_storage, osb_frontend_set_db_storage):
 *  OSB_DB_STORAGE_FP32 (the default, osb_db_create): rows as given -- faiss::IndexFlatIP's semantics.
 *  OSB_DB_STORAGE_FP16: every row element is stored as __float2half_rn(x) (round to nearest even, overflow to +-inf;
 *   numpy's astype(float16)), on the device, whichever call adds it.  Half the HBM per row and half the bytes per scan.
 *   Queries stay fp32: a score is the fp32 inner product of the query with the row converted exactly to fp32, so a search
 *   returns byte-identical ids and scores to a search of an fp32 database holding the rows already rounded to fp16.  For
 *   unit-norm rows of dim 4096 a score moves by at most 2^-11 sum|q_i x_i| + 2^-25 sum|q_i| (<= 4.9e-4 + 1.9e-6 for a
 *   unit query); results near a threshold or a tie can change.
 * -----------------------------------------------------------------------------------------------------------*/
typedef struct osb_db osb_db;
#define OSB_DB_STORAGE_FP32 0
#define OSB_DB_STORAGE_FP16 1
osb_status osb_db_create(osb_db** out, int dim, int64_t capacity);       /* = osb_db_create_storage(..., OSB_DB_STORAGE_FP32) */
/* capacity x dim elements of the storage's type; OSB_ERR_INVALID for any other storage value.  add / add_dev convert on the
 * device (the host form stages through the handle's own 64-row buffer); capacity errors, reset and size as for fp32. */
osb_status osb_db_create_storage(osb_db** out, int dim, int64_t capacity, int storage);
osb_status osb_db_destroy(osb_db* h);
osb_status osb_db_add(osb_db* h, int64_t n, const float* x, int64_t* first_id);
osb_status osb_db_add_dev(osb_db* h, int64_t n, const float* x_dev, int64_t* first_id, void* stream);
osb_status osb_db_search(osb_db* h, int64_t nq, const float* q, int k, float* scores, int64_t* ids);
osb_status osb_db_search_dev(osb_db* h, int64_t nq, const float* q_dev, int k, float* scores_dev,
                             int64_t* ids_dev, void* stream);
int64_t osb_db_size(osb_db* h);
osb_status osb_db_reset(osb_db* h);        /* ntotal = 0 (rows stay allocated) */
/* Row-sharded search (SURVEY.md section 8e, alternative for the 50 k-row sweep): each GPU scans its shard with
 * osb_db_search_dev, the per-shard top-k lists are all-gathered, and this call merges n_lists lists of k candidates per
 * query (cand_* are [nq][n_lists][k], ids < 0 = padding) into the global top-k with faiss::IndexFlatIP's order
 * (loop_detector.cpp:213): score descending, ties by ascending id.  id_offset_dev[l] (may be null) is added IN PLACE to the
 * ids of list l (shard-local row -> global row). */
osb_status osb_topk_merge_dev(int nq, int n_lists, int k, const float* cand_scores_dev, int64_t* cand_ids_dev,
                              const int64_t* id_offset_dev, float* scores_dev, int64_t* ids_dev, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Local descriptor matcher -- replaces cv::BFMatcher(cv::NORM_L2, crossCheck = true).match(query, train)
 *   (swarm_loop/src/loop_cam.cpp:147-150 stereo up/down; swarm_loop/src/loop_detector.cpp:564-567 loop pairs).
 * For every query row the nearest train row by L2 (first minimum wins), kept only if mutual; output sorted by
 * query index.  Batched over `n_pairs` independent (query, train) pairs:
 *   q [n_pairs][max_n][dim], t [n_pairs][max_n][dim], nq/nt [n_pairs] valid row counts,
 *   out: qi/ti/dist [n_pairs][max_n], n_out [n_pairs].   max_n <= 256, dim == 64.
 * -----------------------------------------------------------------------------------------------------------*/
typedef struct osb_matcher osb_matcher;
osb_status osb_matcher_create(osb_matcher** out, int max_pairs, int max_n, int dim);
osb_status osb_matcher_destroy(osb_matcher* h);
osb_status osb_matcher_match(osb_matcher* h, int n_pairs, const float* q, const int32_t* nq, const float* t,
                             const int32_t* nt, int32_t* qi, int32_t* ti, float* dist, int32_t* n_out);
osb_status osb_matcher_match_dev(osb_matcher* h, int n_pairs, const float* q_dev, const int32_t* nq_dev,
                                 const float* t_dev, const int32_t* nt_dev, int32_t* qi_dev, int32_t* ti_dev,
                                 float* dist_dev, int32_t* n_out_dev, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Pose-graph solve -- replaces the body of SwarmLocalizationSolver::solve_once
 *   (swarm_localization/src/swarm_localization_solver.cpp:1668-1725): the three setup_problem_with_* walks
 *   (:1064-1214) become a flat factor list built by the adapter, ceres::Solve (:1712) becomes a GPU
 *   Levenberg-Marquardt with a block-Jacobi preconditioned CG on the 4x4-block normal equations.
 * poses   [n_nodes][4] double (x,y,z,yaw) in/out  -- the 4-vectors of EstimatePoses (swarm_localization_solver.hpp:46-50)
 * fixed   [n_nodes] 1 = SetParameterBlockConstant (solver.cpp:1196-1206)
 * type/ia/ib [n_factors]: factor kind and the two pose blocks
 * huber   [n_factors] 1 = ceres::HuberLoss(1.0) (solver.cpp:1077-1082,1138-1141), 0 = no loss (ego motion :1178)
 * payload [n_factors][OSB_PAYLOAD_LEN] double:
 *   OSB_FACTOR_DISTANCE  (DistanceMeasurementFactor, swarm_localization_factors.hpp:203-224): [d, sqrt_inf]
 *   OSB_FACTOR_RELPOSE   (RelativePoseFactor4d, :226-271): [meas x,y,z,yaw, sqrt_inf 4x4 row-major]
 *   OSB_FACTOR_DETECTION (DroneDetection4dFactor, :273-367): [dir 3, tan_base 2x3, inv_dep, flags, extrinsic_z,
 *                         dposea 4, dposeb 4, DETECTION_SPHERE_STD, DETECTION_INV_DEP_STD]; flags bit0 enable_depth,
 *                         bit1 enable_dpose
 * -----------------------------------------------------------------------------------------------------------*/
#define OSB_FACTOR_DISTANCE 0
#define OSB_FACTOR_RELPOSE 1
#define OSB_FACTOR_DETECTION 2
#define OSB_PAYLOAD_LEN 24

typedef struct {
  int32_t max_iterations;        /* ceres max_num_iterations = 1000 (solver.cpp:1697) */
  int32_t max_pcg_iterations;    /* per LM step */
  double max_time_s;             /* max_solver_time_in_seconds (solver.cpp:1702); <= 0 disables */
  double function_tolerance;     /* Ceres default 1e-6 */
  double gradient_tolerance;     /* Ceres default 1e-10 */
  double parameter_tolerance;    /* Ceres default 1e-8 */
  double pcg_tolerance;          /* relative residual of the inner solve */
  double initial_trust_radius;   /* Ceres default 1e4 */
  int32_t preconditioner;        /* OSB_PRECOND_AUTO (chain block-tridiagonal when the graph fits the one-cluster fast
                                    path, else block-Jacobi) or OSB_PRECOND_BLOCK_JACOBI */
  int32_t inner_precision;       /* arithmetic INSIDE the PCG (Jacobian blocks, direction/residual vectors, preconditioner):
                                    OSB_INNER_AUTO = fp32 when pcg_tolerance >= 1e-4 (LM only needs an inexact step), else
                                    fp64.  Residuals, costs, gradient, poses and all LM decisions are always fp64. */
} osb_solve_options;
#define OSB_PRECOND_AUTO 0
#define OSB_PRECOND_BLOCK_JACOBI 1
#define OSB_INNER_AUTO 0
#define OSB_INNER_FP64 1
#define OSB_INNER_FP32 2

typedef struct {
  double initial_cost;           /* 1/2 sum rho(|r|^2), as ceres Summary::initial_cost */
  double final_cost;             /* Summary::final_cost (solver.cpp:1721) */
  double solve_ms;               /* device time of the solve kernel(s), CUDA events */
  int32_t iterations;            /* LM iterations taken (accepted + rejected) */
  int32_t pcg_iterations;        /* total inner iterations */
  int32_t n_residuals;           /* problem.NumResiduals() (solver.cpp:1724) */
  int32_t termination;           /* 0 converged (function tol), 1 gradient tol, 2 parameter tol, 3 max iterations,
                                    4 time limit, 5 failure (non-finite cost) */
} osb_solve_summary;

typedef struct osb_solver osb_solver;
void osb_solve_default_options(osb_solve_options* o);
osb_status osb_solver_create(osb_solver** out, int max_nodes, int max_factors);
osb_status osb_solver_destroy(osb_solver* h);
osb_status osb_solver_solve(osb_solver* h, int n_nodes, double* poses, const uint8_t* fixed, int n_factors,
                            const int32_t* type, const int32_t* ia, const int32_t* ib, const double* payload,
                            const uint8_t* huber, const osb_solve_options* opt, osb_solve_summary* summary);
/* Random-restart initialisation -- solve_with_multiple_init (swarm_localization_solver.cpp:781-845, called at :925):
 * n_trials solves of the same graph, all in ONE launch (one thread-block cluster per trial when the graph fits the
 * one-cluster path; otherwise the trials run one after another as cooperative grids).  Trial t starts from `poses` with
 * every node whose init_mask[node] is set and that is not fixed scattered as random_init_pose (:204-216) does: x, y
 * uniform in [-rand_xy, rand_xy), z in [-rand_z, rand_z), yaw kept (the adapter supplies the odometry yaw there, :212).
 * The draws are a counter hash of (seed, t, node, component) (oracle/multistart_ref.py: multistart_initial_poses).
 * Each trial runs exactly the arithmetic of osb_solver_solve from its starting poses.  Then, as :783-831:
 *   equv_t = normalise ? sqrt(final_cost_t) / n_residuals / window_size : final_cost_t      (:1721-1725)
 *   best = acpt_cost; trial t is chosen iff equv_t < best (strictly; the first of equal minima wins, NaN never does).
 * poses is overwritten with the chosen trial's result; when no trial is accepted *chosen = -1 and poses is untouched.
 * trial_summaries[t] is filled for every trial; their solve_ms is the device time of the whole batch.
 * Unlike the reference, every trial starts from the caller's poses (its trial i starts from trial i-1's solution for the
 * nodes it does not scatter), and the draws are hashed instead of rand().
 * Memory: the solves of a handle share one arena, which osb_solver_create sizes for one solve at the handle's capacity.
 *   This call grows it to n_trials blocks of at most 704 n + 512 m + 64 G + 5 KB bytes (n nodes, m factors, G CTAs per
 *   solve: <= 16 on the cluster path, <= the SM count otherwise), plus 128 m (fp32 inner) / 256 m (fp64) when the
 *   Jacobians do not fit shared memory, and keeps it until osb_solver_destroy.  A failed allocation returns
 *   OSB_ERR_CUDA and leaves the handle as it was. */
typedef struct {
  int32_t n_trials;      /* INIT_TRIAL = 3 (solver.cpp:54); 1 ... 256 */
  int32_t normalise;     /* 1: equv_cost = sqrt(final_cost)/n_residuals/window_size (the reference's num_res_blks > 1) */
  int32_t window_size;   /* sliding_window_size() (solver.cpp:1724); >= 1 when normalise */
  uint64_t seed;
  double rand_xy, rand_z;   /* RAND_INIT_XY = 5, RAND_INIT_Z = 1 (solver.cpp:51-52); finite, >= 0 */
  double acpt_cost;         /* max_accept_cost (swarm_localization_node.cpp:470); not NaN */
} osb_multistart_options;
osb_status osb_solver_solve_multistart(osb_solver* h, int n_nodes, double* poses, const uint8_t* fixed,
                                       const uint8_t* init_mask, int n_factors, const int32_t* type, const int32_t* ia,
                                       const int32_t* ib, const double* payload, const uint8_t* huber,
                                       const osb_solve_options* opt, const osb_multistart_options* ms,
                                       osb_solve_summary* trial_summaries /*[n_trials]*/, double* equv_costs /*[n_trials]*/,
                                       int32_t* chosen);
/* Resident graph (SURVEY.md 8f-4): instead of re-flattening the whole window for every solve (the reference rebuilds its
 * ceres::Problem each time: setup_problem_with_sferror / _loops_and_detections / _ego_motion,
 * swarm_localization_solver.cpp:1064-1214), the adapter appends what add_new_swarm_frame / add_new_loop_connection
 * (swarm_localization_solver.hpp:197-214) bring.  The factor list stays in device memory, only new factors cross PCIe,
 * and the poses persist between solves like the reference's est_poses.  Node ids are append order; drop_oldest renumbers
 * (sliding window, solver.cpp:186-202).  osb_solver_solve and the resident graph can be mixed on one handle. */
osb_status osb_solver_graph_clear(osb_solver* h);
osb_status osb_solver_graph_add_nodes(osb_solver* h, int n, const double* poses /*[n][4]*/, const uint8_t* fixed /*[n] or NULL*/,
                                      int32_t* first_id);
osb_status osb_solver_graph_add_factors(osb_solver* h, int m, const int32_t* type, const int32_t* ia, const int32_t* ib,
                                        const double* payload, const uint8_t* huber);
osb_status osb_solver_graph_set_fixed(osb_solver* h, int node, int fixed);
osb_status osb_solver_graph_set_poses(osb_solver* h, int first, int n, const double* poses);
osb_status osb_solver_graph_get_poses(osb_solver* h, int first, int n, double* poses);
osb_status osb_solver_graph_size(osb_solver* h, int32_t* n_nodes, int32_t* n_factors);
osb_status osb_solver_graph_drop_oldest(osb_solver* h, int n_nodes);
osb_status osb_solver_solve_resident(osb_solver* h, const osb_solve_options* opt, osb_solve_summary* summary);
/* The resident graph plus a device-side tail: each solve's loop and detection rows, straight from
 * osb_anchor_compact_factors_dev's buffers (type / ia / ib / payload / huber in its layout, *count_dev rows), are solved
 * after the resident factors without reaching the host.  ia / ib are resident node ids (append order, renumbered by
 * drop_oldest): the adapter numbers the anchor window's `block` ids as resident node ids and passes the renumbered window
 * to osb_anchor_set_window after a drop.  The tail is not stored; the next call brings its own.
 *   Numbering: the chain plan is built from the resident factors alone (on the host, cached by topology); tail rows never
 *   join a path.  A tail row enters the chain preconditioner as a coupling when its two internal ids are consecutive and
 *   linked, otherwise through its diagonal blocks -- as osb_solver_solve would place it under that plan.  The index
 *   tables of (resident, tail) are built on the device in a fixed number of launches, deterministically.
 *   max_tail picks the launch shape: it is osb_solver_solve's for (n, m + max_tail), and the solve reads m + k from the
 *   device.  A call is bit-identical to osb_solver_solve of the concatenated list whenever both pick the same shape and
 *   the same plan.  Size max_tail to the window, not to max_measurements: on the fp32 cluster path, m + max_tail <= 25 600
 *   keeps the Jacobians in shared memory and <= 12 288 keeps the chain fast path.
 *   Poses stay on the device: the call starts from a device copy of the resident poses and writes the solution back to it.
 *   The first host-side solver call afterwards (graph_get_poses, graph_set_poses, graph_add_nodes, graph_drop_oldest,
 *   solve_resident, solve, last_summary, ...) synchronises once and refreshes the host copy.  When the call was captured,
 *   every host-side call re-reads what the last replay left, so the caller synchronises a replay before such a call;
 *   this lasts until a host-side change of the poses or the graph.  Host-side pose changes are uploaded by the next
 *   device call.
 *   Refused on the device: a tail row with an unknown type, a node id outside [0, n), ia == ib, or *count_dev < 0
 *   (OSB_ERR_INVALID) or > max_tail (OSB_ERR_CAPACITY): nothing is solved, poses and graph stay unchanged, and
 *   osb_solver_last_summary returns the code.  Refused at once, with nothing enqueued: null pointers, max_tail < 0
 *   (OSB_ERR_INVALID), m + max_tail > max_factors (OSB_ERR_CAPACITY), an empty resident graph (OSB_ERR_INVALID).
 *   Stream capture: the call needs no host work when the topology and the poses have not changed on the host since the
 *   previous device call, no factor is waiting to be uploaded and the options and max_tail are the previous call's.  Such
 *   a call on the cluster path can be captured.  Under capture, a call that would need host work or would run on the
 *   cooperative path returns OSB_ERR_INVALID before it enqueues anything.
 *   Everything runs on `stream` (a cudaStream_t; consecutive device calls of a handle on one stream), after the handle's
 *   host-side calls, which end in a synchronisation.  Six launches per call.
 *   Memory: the first call acquires the device pose copy, the resident plan's tables and the per-call scratch (about
 *   60 n + 36 m + 8 n ceil(m / 256) bytes at the handle's capacity n nodes, m factors); later calls acquire nothing. */
osb_status osb_solver_solve_resident_dev(osb_solver* h, int max_tail, const int32_t* type_dev, const int32_t* ia_dev,
                                         const int32_t* ib_dev, const double* payload_dev, const uint8_t* huber_dev,
                                         const int32_t* count_dev, const osb_solve_options* opt, void* stream);
/* synchronises with the last osb_solver_solve_resident_dev call -> its status; on OSB_OK its summary (n_residuals =
 * resident + tail; solve_ms from CUDA events, 0 when the call was captured).  After an
 * osb_solver_solve_multistart_resident_dev call it returns OSB_ERR_INVALID: osb_solver_last_multistart reads that call. */
osb_status osb_solver_last_summary(osb_solver* h, osb_solve_summary* summary);
/* Random-restart initialisation on the device chain -- solve_with_multiple_init (swarm_localization_solver.cpp:781-845)
 * of the resident window plus a device tail, the branch solve() takes at start-up, when a drone appears and after a solve
 * whose equv_cost exceeds acpt_cost (:880-960).  Takes osb_solver_solve_resident_dev's arguments, plus:
 *   init_mask_dev [n] (caller's node ids, device): the nodes to scatter, e.g. what osb_anchor_init_mask_dev wrote;
 *   init_yaw_dev [n] (device) or NULL: a scattered node's yaw (the odometry yaw of random_init_pose, :212); NULL keeps
 *   the node's yaw; ms: as osb_solver_solve_multistart.
 *   Rule: osb_solver_solve_multistart of the concatenated list (resident factors, then the *count_dev tail rows) under the
 *   resident plan, started from the resident device poses: the same draws keyed (seed, trial, caller's node id,
 *   component), the same ranking (equv, strict < against acpt_cost, first of equal minima), with n_residuals (for
 *   normalise) = resident + tail residuals counted on the device.  A trial's arithmetic is osb_solver_solve_resident_dev's
 *   from its starting poses, so every trial, equv and the choice are bit-identical to osb_solver_solve_multistart of the
 *   concatenated list whenever both pick the same shape and plan.  The chosen trial's poses go into the resident device
 *   pose copy; with no trial accepted (chosen = -1) that copy is left as it was (osb_solver_solve_multistart's documented
 *   deviation, not the reference's "last trial's poses").  The host copy is refreshed as after osb_solver_solve_resident_dev.
 *   Launches: the shape is osb_solver_solve's for (n, m + max_tail); the four tail-table launches (built once, shared by
 *   the trials), one scatter, the trials, one selection: 7 launches on the cluster path (all trials in one launch, one
 *   cluster each), 6 + n_trials on the cooperative path (the trials in turn, each keeping its own summary).
 *   Refused on the device as osb_solver_solve_resident_dev (every trial leaves before its first barrier): chosen = -1, poses
 *   and graph unchanged, osb_solver_last_multistart returns the code.  Refused at once with nothing enqueued: its refusals,
 *   a null init_mask_dev or ms, and osb_solver_solve_multistart's checks of ms (n_trials outside 1 ... 256, normalise with
 *   window_size < 1, rand_xy / rand_z negative or not finite, acpt_cost NaN).
 *   Memory: the first call acquires what osb_solver_solve_resident_dev's first call does; the arena grows to n_trials solves
 *   as in osb_solver_solve_multistart.  Growing it is host work: under stream capture a call that would need it returns
 *   OSB_ERR_INVALID with nothing enqueued.  Otherwise capture follows osb_solver_solve_resident_dev's rules. */
osb_status osb_solver_solve_multistart_resident_dev(osb_solver* h, int max_tail, const int32_t* type_dev,
                                                    const int32_t* ia_dev, const int32_t* ib_dev, const double* payload_dev,
                                                    const uint8_t* huber_dev, const int32_t* count_dev,
                                                    const uint8_t* init_mask_dev, const double* init_yaw_dev,
                                                    const osb_solve_options* opt, const osb_multistart_options* ms,
                                                    void* stream);
/* synchronises with the last osb_solver_solve_multistart_resident_dev call -> its status; on OSB_OK every trial's summary
 * [n_trials] (n_residuals = resident + tail; solve_ms = the device time of all trials from CUDA events, 0 when the call was
 * captured), equv [n_trials] and chosen (-1: none accepted).  OSB_ERR_INVALID when the last device call was a single solve. */
osb_status osb_solver_last_multistart(osb_solver* h, osb_solve_summary* summaries, double* equv, int32_t* chosen);
/* profiling aid: SM-clock cycles block 0 spent in the phases of the LAST solve, summed over its CG iterations:
 * out[0] factor phase, [1] barrier after it, [2] node phase 1, [3] reduction 1, [4] node phase 2, [5] reduction 2,
 * [6] number of CG iterations, [7] whole kernel; [8] CTAs, [9] 1 = one thread-block cluster (hardware barrier) /
 * 0 = cooperative grid, [10] bit 0 = Jacobians in shared memory, bit 1 = chain preconditioner, bit 2 = fp32 inner
 * arithmetic, [11] threads per CTA. */
osb_status osb_solver_phase_cycles(osb_solver* h, double* out12);
/* profiling aid: SM-clock cycles each warp spent in the chain-preconditioner sweeps of the LAST solve, [16 CTAs][8 warps] */
osb_status osb_solver_chain_cycles(osb_solver* h, double* out128);
/* host-only (no GPU needed): the node numbering the solver uses for its chain preconditioner -- a greedy maximum-weight
 * path cover of the factor graph (on a swarm graph: every drone's odometry chain).  order_out[i] = caller's node id of
 * internal node i; link_out[i] = 1 iff internal node i-1 precedes i on its path and i % 16 != 0. */
osb_status osb_solver_chain_plan(int n_nodes, const uint8_t* fixed, int n_factors, const int32_t* type,
                                 const int32_t* ia, const int32_t* ib, const double* payload, int32_t* order_out,
                                 uint8_t* link_out);
/* residual + analytic Jacobian of every factor at `poses` (parity hook for the factor kernels):
 * r [n_factors][4], Ja/Jb [n_factors][4][4] (rows >= the factor's residual count are zero), un-robustified. */
osb_status osb_solver_linearize(osb_solver* h, int n_nodes, const double* poses, int n_factors,
                                const int32_t* type, const int32_t* ia, const int32_t* ib, const double* payload,
                                double* r, double* Ja, double* Jb);

/* ------------------------------------------------------------------------------------------------------------
 * PCM outlier rejection of loop edges (SURVEY.md 8f-2) -- replaces SwarmLocalOutlierRejection::OutlierRejectionLoopEdgesPCM
 *   (swarm_localization/src/swarm_outlier_rejection/swarm_outlier_rejection.cpp:173-297), the stage that feeds
 *   get_good_loops() to the solve: pairwise consistency of the n loop edges of one drone pair
 *   (err = odom_a * p_edge2 * odom_b^-1 * p_edge1^-1, 6-D log map, squared Mahalanobis distance < pcm_thres, :190-235) and
 *   FMC::maxCliqueHeu on the consistency graph (third_party/fast_max-clique_finder/src/findCliqueHeu.cpp:120-244, restated
 *   literally incl. its prunings and candidate order).
 * osb_loop_edge: what the adapter reads off a Swarm::LoopEdge and the two DroneTrajectory objects (swarm_msgs is not in the
 *   reference tree, so its arithmetic is defined in oracle/pcm_ref.py): relative_pose as (x y z, qw qx qy qz),
 *   get_covariance() 6x6 row-major (translation block first), the ego-motion pose of drone id_a at ts_a and of drone id_b at
 *   ts_b, and the accumulated trajectory length at those stamps.  The odometry between two stamps is pose(ts1)^-1 * pose(ts2)
 *   with covariance |len2 - len1| * diag(odom_pos_cov_per_m x3, odom_ang_cov_per_m x3).
 * Edges are in insertion order (all_loops[id_a][id_b]); edges of another drone pair are never consistent.
 * Outputs: clique [n] = indices of the kept loops in maxCliqueHeu's order (good_loops_set, :291-296), clique_size; optional
 *   adj [n][n] (1 = consistent) and smd [n][n] (squared Mahalanobis distances, +inf where undefined).  n <= 4096. */
typedef struct {
  int32_t id_a, id_b;
  double rel_pose[7];
  double cov[36];
  double odom_a[7];
  double odom_b[7];
  double len_a, len_b;
} osb_loop_edge;
osb_status osb_pcm(const osb_loop_edge* edges, int n, double pcm_thres, double odom_pos_cov_per_m, double odom_ang_cov_per_m,
                   int32_t* clique, int32_t* clique_size, uint8_t* adj, double* smd);
osb_status osb_pcm_dev(const osb_loop_edge* edges_dev, int n, double pcm_thres, double odom_pos_cov_per_m,
                       double odom_ang_cov_per_m, int32_t* clique_dev, int32_t* clique_size_dev, uint8_t* adj_dev,
                       double* smd_dev, void* stream);
/* Clique parity hook (tests only): pcm_max_clique_kernel on caller-given adjacency bit matrices, launched as each of its
 *   callers launches it.  Graph g has n[g] vertices (1..slot_rows); its row i is bits[(g * slot_rows + i) * stride ..] with
 *   bit j of word j / 32 set iff i and j are adjacent (symmetric, zero diagonal, bits past n[g] zero); stride >= the words
 *   of a slot_rows-bit row.  out [n_graphs][1 + slot_rows]: the clique size, then its vertices in maxCliqueHeu's order.
 *   form 0: one graph in one CTA, as osb_pcm_dev (pass stride = ceil(n / 32));
 *   form 1: one CTA per graph from a host job list, with the shared memory of the largest in-smem graph, as
 *           osb_pcm_state_reject;
 *   form 2: n_ctas >= n_graphs CTAs with 200 KiB of shared memory and the job count read from the device, so the CTAs past
 *           it exit, as osb_pcm_state_reject_anchored. */
osb_status osb_pcm_clique_parity(int form, const uint32_t* bits, int n_graphs, const int32_t* n, int slot_rows, int stride,
                                 int n_ctas, int32_t* out);
/* Persistent PCM state -- SwarmLocalOutlierRejection::OutlierRejectionLoopEdges (swarm_outlier_rejection.cpp:98-167, 173-297)
 *   with the state it keeps between solves: the consistency graph and the loops of every drone pair stay on the device, a
 *   call checks only its new loops (O(new x L) pair checks, not O(L^2)) and reruns maxCliqueHeu on the pairs that gained any.
 * reject(): loop edges[i] carries the LoopEdge::id ids[i].  As :106-139:
 *   - a loop whose id an earlier call stored is skipped: the FIRST-seen values of an id are the ones used (the reference
 *     ignores the values re-anchoring gives the same id later);
 *   - routing: a loop belongs to the unordered pair {id_a, id_b}; with `redundant` every pair is processed, else only the
 *     pairs that contain self_id, (self, self) included.  Loops of other pairs are neither stored nor marked as seen, so
 *     they count as new again on the next call;
 *   - a pair's new loops are appended in call order (the same id twice in one call is appended twice), each checked against
 *     every earlier loop of its pair with edge1 = the later loop, so its graph is bit-identical to osb_pcm's on the pair's
 *     whole insertion-ordered list; every pair that gained a loop reruns maxCliqueHeu on its whole graph and its inlier set
 *     becomes the clique's ids, replacing whatever set_inliers wrote;
 *   - keep[i] = 1 iff edge i is in the returned good_loops (:141-157): its pair has no inlier set, or its id is in the set.
 *   A call that would push a pair past pair_capacity or the state past max_pairs returns OSB_ERR_CAPACITY and changes
 *   nothing.  A call that routes nothing new launches no kernel; otherwise it makes one copy up (pinned staging), two
 *   launches, one copy down and one synchronisation on the handle's stream.
 * inliers(): good_loops_set[a][b] in ascending id order (what broadcast_good_loops sends); *n = its size, -1 if the pair has
 *   none; ids may be NULL to query the size, else OSB_ERR_CAPACITY when the set exceeds cap.
 * set_inliers(): good_ids_handle (:37-56): replaces the pair's set with ids[0..n); ignored when the pair contains self_id.
 *   (The reference's handler inserts the indices 0..inlier_id_size-1, not msg->inlier_ids: the adapter decides what to pass.)
 * pair(): read-out for tests: the pair's loop count *n (0 for an unknown pair), its ids in insertion order [n], adjacency
 *   [n][n] (1 = consistent), its last clique in maxCliqueHeu order and its size; every output but n may be NULL.
 * Memory: create holds a stream, max_pairs x (64 + 488 pair_capacity) bytes of pinned and of device staging and
 *   max_pairs x (1 + pair_capacity) x 4 bytes of clique output on each side.  A pair's first loop acquires its slot,
 *   pair_capacity x (508 + 4 ceil(pair_capacity / 32)) bytes + 4 (4.2 MB at 4096), kept until destroy.  The device path
 *   (osb_pcm_state_reject_anchored, after osb_anchor_run_dev below) acquires more on its first call only. */
typedef struct {
  int32_t self_id;
  int32_t redundant;             /* SwarmLocalOutlierRejectionParams::redundant */
  int32_t max_pairs;             /* unordered drone pairs {a,b}, a == b allowed (intra-drone loops) */
  int32_t pair_capacity;         /* edges per pair, 1..4096 (the clique kernel's bitset bound) */
  double pcm_thres, odom_pos_cov_per_m, odom_ang_cov_per_m;
} osb_pcm_state_params;
typedef struct osb_pcm_state osb_pcm_state;
osb_status osb_pcm_state_create(osb_pcm_state** out, const osb_pcm_state_params* p);
osb_status osb_pcm_state_destroy(osb_pcm_state* s);
osb_status osb_pcm_state_reject(osb_pcm_state* s, const osb_loop_edge* edges, const int64_t* ids, int n, uint8_t* keep);
osb_status osb_pcm_state_inliers(osb_pcm_state* s, int32_t id_a, int32_t id_b, int64_t* ids, int cap, int32_t* n);
osb_status osb_pcm_state_set_inliers(osb_pcm_state* s, int32_t id_a, int32_t id_b, const int64_t* ids, int n);
osb_status osb_pcm_state_pair(osb_pcm_state* s, int32_t id_a, int32_t id_b, int32_t* n, int64_t* ids, uint8_t* adj,
                              int32_t* clique, int32_t* clique_size);

/* ------------------------------------------------------------------------------------------------------------
 * Re-anchoring of loops and detections onto the sliding window (SURVEY.md 8f-4) -- replaces the walk of
 *   SwarmLocalizationSolver::find_available_loops_detections (swarm_localization_solver.cpp:1594-1666) over every
 *   measurement ever received: loop_from_src_loop_connection (:1464-1553), find_node_frame_for_measurement_2drones
 *   (:1429-1462), and the factor choice of setup_problem_with_loops_and_detections (:1064-1100).  One launch per run.
 * The handle keeps ego_motion_trajs (push_odometry), all_loops / all_detections_6d (add_measurements) and sf_sld_win
 *   (set_window) on the device.  Stamps are int64 nanoseconds, so every comparison is exact.  DroneTrajectory, NodeFrame and
 *   LoopEdge come from swarm_msgs, which is not in the reference tree; their arithmetic is defined in oracle/anchor_ref.py:
 *   a trajectory's length[k] is the sequential fp64 sum of |p_j - p_(j-1)| for j <= k; a look-up at stamp t uses the nearest
 *   sample (ties to the earlier, clamped at both ends); the odometry covariance between two stamps is
 *   |length(t2) - length(t1)| * diag(odom_pos_cov_per_m x3, odom_ang_cov_per_m x3).
 * run(): for measurement i (all loops in order, then all detections in order) out[i] holds, as :1464-1553:
 *   status: OSB_ANCHOR_EMPTY_WINDOW (no frame), OSB_ANCHOR_BEFORE_WINDOW (frame 0's stamp - stamp_a > begin_min_loop_dt_s,
 *     strictly; stamp_b is not tested), OSB_ANCHOR_NO_FRAME (drone a or b has no vo_available entry in the window closer than
 *     10000 s, strictly), OSB_ANCHOR_NO_TRAJECTORY (drone a or b has no odometry), OSB_ANCHOR_DPOS (dpos > det_dpos_thres),
 *     else OSB_ANCHOR_OK -- tested in this order;
 *   frame_a/b, node_a/b, stamp_a/b: the anchor of each side (the entry of the drone with the smallest |stamp difference|,
 *     the earliest frame on ties), its caller pose-block id and stamp; -1 / -1 / 0 when not found;
 *   dt_err_ns: the two stamp differences summed, 10000 s for a side not found (0 when no search ran: EMPTY_WINDOW,
 *     BEFORE_WINDOW);
 *   dpos and edge (for OK and DPOS): dpos = |len(stamp_a) - len(anchor a)| + the same for b; edge.rel_pose =
 *     DeltaPose(anchor_a.self_pose, self_pose_a, 4-DoF) * relative_pose * DeltaPose(self_pose_b, anchor_b.self_pose, 4-DoF),
 *     where detections take self_pose_a/b from the trajectories at their stamps (DET4D: yaw only); edge.cov = cov + the
 *     odometry covariance of both sides; edge.odom_a/b = the anchors' self poses, edge.len_a/b = the lengths at their stamps:
 *     the edge osb_pcm_state_reject takes;
 *   skip = 1 unless status is OK, both drones are yaw-observable and node_a != node_b;
 *   the solver row (factor_type OSB_FACTOR_RELPOSE, ia = node_a, ib = node_b, huber, payload [x y z yaw, S 4x4]) with
 *     S_ij = sqrt|(cov4^-1)_ij|, cov4 = blkdiag(edge.cov[0:3,0:3], edge.cov[5,5]) (RelativePoseFactor4d::CreateCov6d).
 *   run_dev writes out_dev[*n_out] on `stream` without synchronising; run copies to the host and synchronises.
 *   yaw_observable [max_drones] is read during the call.  Every run is one kernel launch (none when there is no measurement).
 * Errors: a drone id outside 0..max_drones-1, a null pointer, a stamp not after the drone's last one, an unknown type, a
 *   drone twice in one frame or a malformed frame_first give OSB_ERR_INVALID; exceeding a capacity gives OSB_ERR_CAPACITY.
 *   Either way the handle is unchanged.
 * Ordering: the handle's device state is in six parts.  A device call waits for the last call that touched (read or
 *   wrote) each part it touches, on any stream, and then becomes that part's last toucher; so the calls that touch one
 *   part run in the order they were made, whatever streams they are on, also inside a CUDA graph (there the waits and
 *   records are external event nodes).  Reads and writes count alike: two runs on different streams do not overlap.
 *     STORE      measurements, loop and detection slots, device counts: run, run_dev, run_dev_if, add_measurements_dev,
 *                data_association_dev
 *     OBSERVE    drone-pair matrix, observe window record, osb_observability record: observe_dev, observe_dev_if,
 *                init_mask_dev, distance_factors_dev, init_by_loops_dev, data_association_dev
 *     SYNC       sync window table, keyframe and full paths, prediction records, outcome: sync_dev, init_by_loops_dev,
 *                data_association_dev
 *     KEYFRAMES  keyframe ring and its frame table: add_keyframe_dev, distance_factors_dev
 *     LOOPS      loop map, pair minima, overflow flag and init_by_loops' status: record_loops_dev, init_by_loops_dev
 *     DA         data association result, the applied word included: data_association_dev, run_dev_if, observe_dev_if
 *   The synchronising readers (observability, sync_result, paths, predict, keyframe_flags, init_by_loops_result,
 *   loop_map, data_association_result) wait for the parts they read.  The updates (push_odometry, add_measurements,
 *   set_window) alone write the trajectories, the window and init_mask's block table, and wait for every part first.
 *   Work of another handle (the solver's last device call, the PCM state's last anchored call) is waited for where a call
 *   below says so.
 * Memory: create acquires a stream, six events, and the trajectories, measurements, window and run output at their
 *   capacities.  The first call that needs the rest acquires it (each call below gives the sizes): the device counts
 *   (add_measurements_dev, data_association_dev), the observe state (observe_dev, observe_dev_if), the block table
 *   (init_mask_dev), the sync's window table, paths and records (sync_dev, init_by_loops_dev, data_association_dev),
 *   predict's buffers (predict), the keyframe store (add_keyframe_dev, distance_factors_dev), the loop map
 *   (record_loops_dev, init_by_loops_dev) and the data association result (set_data_association). */
#define OSB_MEAS_LOOP 0
#define OSB_MEAS_DET4D 1
#define OSB_MEAS_DET6D 2
#define OSB_ANCHOR_OK 0
#define OSB_ANCHOR_EMPTY_WINDOW 1
#define OSB_ANCHOR_BEFORE_WINDOW 2
#define OSB_ANCHOR_NO_FRAME 3
#define OSB_ANCHOR_NO_TRAJECTORY 4
#define OSB_ANCHOR_DPOS 5
typedef struct {
  int32_t max_drones;            /* drone ids 0 .. max_drones-1; 1..256 */
  int32_t max_traj_samples;      /* odometry samples per drone */
  int32_t max_measurements;      /* loops + detections */
  int32_t max_window_entries;    /* node frames in the window */
  double begin_min_loop_dt_s;    /* BEGIN_MIN_LOOP_DT = 1000 (solver.cpp:56) */
  double det_dpos_thres;
  double odom_pos_cov_per_m, odom_ang_cov_per_m;
  int32_t huber;                 /* 1 = HuberLoss(1.0) on every row (0 = debug_no_rejection) */
  int32_t max_keyframes;         /* keyframes the distance store holds (osb_anchor_add_keyframe_dev); 0: no store */
  int32_t max_keyframe_distances;/* distances of one keyframe, all its nodes together */
  int32_t reserved;
} osb_anchor_params;
typedef struct {                 /* a Swarm::LoopEdge (LOOP) or DroneDetection (DET4D / DET6D) */
  int64_t id;
  int32_t type, id_a, id_b, reserved;
  int64_t stamp_a, stamp_b;      /* ns */
  double relative_pose[7];       /* x y z, qw qx qy qz */
  double cov[36];                /* 6x6 row-major, translation block first */
  double self_pose_a[7], self_pose_b[7];
} osb_measurement;
typedef struct {                 /* a NodeFrame of the window */
  int32_t drone_id, vo_available;
  int32_t block;                 /* the caller's pose-block id (est_poses_idts[id][ts]); shared blocks share an id */
  int32_t reserved;
  int64_t stamp;                 /* ns */
  double self_pose[7];
} osb_window_entry;
typedef struct {
  int64_t id;
  int32_t type, status;
  int32_t frame_a, frame_b, node_a, node_b;
  int64_t stamp_a, stamp_b, dt_err_ns;
  double dpos;
  osb_loop_edge edge;
  int32_t skip, factor_type, ia, ib, huber, reserved;
  double payload[OSB_PAYLOAD_LEN];
} osb_anchor_result;
typedef struct osb_anchor osb_anchor;
osb_status osb_anchor_create(osb_anchor** out, const osb_anchor_params* p);
osb_status osb_anchor_destroy(osb_anchor* h);
/* appends n samples (stamps strictly increasing, also against the drone's last sample); poses [n][7] */
osb_status osb_anchor_push_odometry(osb_anchor* h, int32_t drone, int n, const int64_t* stamps_ns, const double* poses);
osb_status osb_anchor_add_measurements(osb_anchor* h, int n, const osb_measurement* m);
/* n_loops and n_detections held (run() writes n_loops + n_detections results) */
osb_status osb_anchor_size(osb_anchor* h, int32_t* n_loops, int32_t* n_detections);
/* replaces the window: frame f holds entries [frame_first[f], frame_first[f+1]) and was taken at frame_stamps_ns[f] */
osb_status osb_anchor_set_window(osb_anchor* h, int n_frames, const int64_t* frame_stamps_ns, const int32_t* frame_first,
                                 const osb_window_entry* entries);
osb_status osb_anchor_run(osb_anchor* h, const uint8_t* yaw_observable, osb_anchor_result* out, int32_t* n_out);
osb_status osb_anchor_run_dev(osb_anchor* h, const uint8_t* yaw_observable, osb_anchor_result* out_dev, int32_t* n_out,
                              void* stream);
/* osb_anchor_add_measurements_dev(): add_new_loop_connection / add_new_detection (swarm_localization_solver.cpp:558-588) for
 *   rows [0, *count_dev) of a DEVICE buffer, e.g. what osb_frontend_loop_measurements wrote, on `stream` without
 *   synchronising.  A LOOP row is dropped when sqrt((x*x + y*y) + z*z) of its relative_pose, in fp64 without fused
 *   multiply-adds, is > (double)loop_outlier_distance_threshold (a float, as the reference's parameter); detections are not
 *   gated.  The kept rows are stored as osb_anchor_add_measurements stores them, in row order.  A dropped loop has used up
 *   its id, so the ids in the store may have gaps, as in the reference.  One launch (a one-CTA block scan that validates,
 *   gates, appends and updates the counts, which then live on the device).
 *   Refused on the device, leaving the store unchanged: an unknown type or a drone id outside 0..max_drones-1
 *   (OSB_ERR_INVALID), *count_dev outside [0, max_n] (OSB_ERR_INVALID), more kept rows than max_measurements leaves room for
 *   (OSB_ERR_CAPACITY); osb_anchor_status() reports it.  Null pointers and max_n < 0 return OSB_ERR_INVALID at once, with
 *   nothing enqueued.  The first call acquires 8 bytes of device counts, a mapped pinned feedback word and an event.
 *   While an append may not have run, the host keeps a bound of the row count: the count the last executed append reported
 *   plus the max_n of every append enqueued after it, capped at max_measurements.  run_dev launches over that bound, reads
 *   the true counts on the device, writes rows past them as OSB_ANCHOR_VOID (skip = 1, every other field zero: PCM and the
 *   factor compaction pass over them) and returns the bound as *n_out.  Every synchronising call (run, size,
 *   add_measurements, push_odometry, set_window, status) first waits for the last device append, after which the counts are
 *   exact and run returns exactly n_loops + n_detections rows.  A handle that never calls add_measurements_dev behaves as
 *   if it did not exist.  The call can be captured into a CUDA graph (after an uncaptured first call): its event waits
 *   and records are external event nodes, so the synchronising calls after a replay wait for the replayed append.
 * osb_anchor_status(): waits for the last device append and writes its status to *last (OSB_OK when none ran); returns the
 *   same value. */
#define OSB_ANCHOR_VOID 6
osb_status osb_anchor_add_measurements_dev(osb_anchor* h, const osb_measurement* m_dev, const int32_t* count_dev, int max_n,
                                           float loop_outlier_distance_threshold, void* stream);
osb_status osb_anchor_status(osb_anchor* h, osb_status* last);
/* osb_anchor_observe_dev(): SwarmLocalizationSolver::estimate_observability (swarm_localization_solver.cpp:1336-1427) on the
 *   device, from the n rows osb_anchor_run_dev wrote (n = its n_out, VOID tail included), on `stream` without
 *   synchronising.  Goes between run_dev and osb_anchor_compact_factors_dev (before or after osb_pcm_state_reject_anchored,
 *   which reads only status).  With the window's frame count, the node set and the drones' bounding boxes, and the
 *   handle's persistent state (pos, enable, solve_master):
 *   1. E = the unordered pairs (edge.id_a, edge.id_b) of the rows with status == OSB_ANCHOR_OK (loops and detections);
 *   2. L = {self_id}, or its closure over E when the node set holds more than one drone (loop_observable_set, :1299-1334);
 *   3. yaw is cleared; 4. more than 3 frames (SINGLE_DRONE_SFS_THRES) and exactly one node: solve_master;
 *   5. every d in L: to_init if !pos[d]; pos = yaw = enable = 1; solve_master when d != self_id;
 *   6. self_id's box: xmax - xmin > init_xy_movement && ymax - ymin > init_xy_movement && zmax - zmin > init_z_movement
 *      (the float thresholds compared as doubles): solve_master, motion; every node with !pos: motion_new, to_init;
 *      every node: pos = enable = 1;
 *   7. every node whose box's x or y extent is > 1.0 (THRES_YAW_OBSER_XY): yaw;
 *   8. every row: skip = !(status == OK && yaw[edge.id_a] && yaw[edge.id_b] && node_a != node_b), written in place; no
 *      other byte of a row changes.  So the rows become run_dev's with this yaw as its yaw_observable.
 *   A drone's box covers its vo_available entries of the current window, from max = -1000 and min = +1000 per axis
 *   (boundingbox_sldwin, :848-878), in fp64; an empty box has extents of -2000.  The node set (all_nodes) is every drone id
 *   of every set_window entry since create, vo_available or not.  pos and enable start at 0 and only ever become 1, as
 *   does solve_master; enable[self_id] is always 1 (:640).  set_window derives the frame count, the node set and the
 *   boxes on the host, so a captured observe sees the window set before each replay.
 *   Three launches whatever n and the drone count (one pass over the rows sets a drone-pair bit matrix from status,
 *   edge.id_a and edge.id_b; one CTA runs the closure and steps 3-7; one pass rewrites skip).  The first call acquires the
 *   state, the bit matrix and the window record, and synchronises; later calls acquire nothing and can be captured into a
 *   CUDA graph.  Refused at once with nothing enqueued (OSB_ERR_INVALID): a null pointer, n < 0, self_id outside
 *   0..max_drones-1.
 * osb_anchor_observability(): waits for the last observe and writes its outcome: per drone the node set, yaw, the sticky
 *   pos and enable and to_init (ids_to_init), 1 or 0 each; solve_master (enable_to_solve_master, sticky), motion (the self
 *   box test held) and motion_new (it found a node with !pos).  The caller's state machine keeps finish_init and
 *   system_is_initied_by_motion: motion_new means finish_init = 0 and by_motion = 1; motion && !finish_init means
 *   by_motion = 1 (:1392-1402).  All zero before the first observe. */
typedef struct {
  int32_t self_id;
  float init_xy_movement, init_z_movement;   /* the reference's float parameters */
  int32_t reserved;
} osb_observe_params;
typedef struct {
  uint8_t nodes[256], yaw[256], pos[256], enable[256], to_init[256];   /* [drone], 1 or 0; drones >= max_drones are 0 */
  int32_t solve_master, motion, motion_new, reserved;
} osb_observability;
osb_status osb_anchor_observe_dev(osb_anchor* h, const osb_observe_params* p, osb_anchor_result* rows_dev, int n,
                                  void* stream);
osb_status osb_anchor_observability(osb_anchor* h, osb_observability* out);
/* osb_anchor_init_mask_dev(): random_init_pose's choice of blocks (swarm_localization_solver.cpp:204-216) from the window
 *   and the record the last osb_anchor_observe_dev wrote, on the device: mask_dev[b] = 1 iff block b belongs to a window
 *   entry of a drone d with to_init[d] and d != self_id, and yaw_dev[b] = the yaw of that entry's self_pose (NodeFrame::yaw(),
 *   the odometry yaw; quaternion -> yaw as the re-anchoring computes it, oracle/anchor_ref.py).  Every window entry counts,
 *   vo_available or not (add_as_keyframe gives each node frame an est_poses block, :517-540).  A block shared by several
 *   frames takes its latest frame's pose (the reference writes the shared block once per frame, in stamp order).  Every
 *   other element of [0, n_nodes) gets mask 0 and yaw 0.  The output feeds osb_solver_solve_multistart_resident_dev.
 *   set_window derives each block's drone and pose on the host; the first call acquires the device copy (at
 *   max_window_entries blocks, or the window's largest block id + 1 if more) and synchronises, and set_window keeps it
 *   current after that.  to_init is read on the device, so a captured call follows both the window set before each replay
 *   and that replay's observe.  (A set_window whose block ids outgrow the copy replaces it: capture again after it.)
 *   One launch on `stream`.  Refused at once with nothing enqueued (OSB_ERR_INVALID): a null pointer, n_nodes < 1, a
 *   window block outside 0 .. n_nodes-1, self_id outside 0..max_drones-1, or no observe_dev since create. */
osb_status osb_anchor_init_mask_dev(osb_anchor* h, int32_t self_id, int n_nodes, uint8_t* mask_dev, double* yaw_dev,
                                    void* stream);
/* osb_anchor_sync_dev(): SwarmLocalizationSolver::sync_est_poses (swarm_localization_solver.cpp:962-1057) on the device,
 *   after the solver's last device call (osb_solver_solve_resident_dev or osb_solver_solve_multistart_resident_dev), on
 *   `stream` without synchronising.  It is ordered after that call on any stream, also inside a CUDA graph.
 *   Applied only if solve() would accept that call (:925, :947-951), decided on the device:
 *     a single solve when its status is OK and !(equv > acpt_cost), equv = normalise ? sqrt(final_cost) / n_residuals /
 *     window_size : final_cost, n_residuals = the resident factors' residuals + the device tail's;
 *     a multistart when it chose a trial (chosen >= 0); the sync is then an init sync (is_init_solve).
 *   A sync not applied changes no output and no state.  An applied sync, with the window set last and the solved poses
 *   (x y z yaw) of its blocks:
 *   keyframe path of drone d: one sample per window entry of d, in frame order, vo_available or not; stamp = the entry's
 *     FRAME stamp; pose = Pose(block pose, yaw) with att = att * (AngleAxis(-yaw(ego), Z) * att(ego)), ego = d's odometry
 *     at the frame stamp (nearest sample, as the re-anchoring looks it up).  Every path is rebuilt: a drone without a window
 *     entry has none.  A quaternion of yaw y is quat_from_rotvec(0, 0, y), as everywhere in the back-end;
 *   full path (full_path != 0) of every drone with a keyframe path: odometry samples i = 0, 10, 20, ... (FULL_PATH_STEP);
 *     the keyframe sample nearest to the odometry stamp, the earlier one on ties (the reference's forward walk, bounded at
 *     the last sample); pose = kf_pose * DeltaPose(vo_ref, ego_i, 4-DoF), then att = att * att_no_yaw(ego at the
 *     keyframe's stamp), vo_ref = that keyframe entry's self_pose; stamp = the odometry stamp.  full_path == 0: no drone
 *     has one (the reference clears full_trajs);
 *   prediction record (est_poses_tsid_saved / last_saved_est_kf_ts, read by osb_anchor_predict): per drone, the last
 *     pushed frame holding it, with its solved block pose and its entry's self_pose.  An init sync pushes every window
 *     frame in order; a steady sync pushes the last frame that has entries.  A record whose frame is still in the window
 *     is rewritten in place (the reference rewrites est_poses_tsid_saved of every window frame); once its frame has left,
 *     it is frozen.  This equals the reference's reverse scan of last_saved_est_kf_ts as long as a frame stamp keeps the
 *     drones it was first pushed with (a SwarmFrame does).
 *   Refused on the device with every output and all state unchanged: a window drone without odometry (the reference
 *   throws from ego_motion_trajs.at()) -- osb_anchor_sync_result reports OSB_ERR_INVALID.
 *   Refused at once with nothing enqueued (OSB_ERR_INVALID): a null pointer; self_id outside 0..max_drones-1; normalise
 *   with window_size < 1; a NaN acpt_cost; the two handles on different devices; no solver device call since its last
 *   host-side pose or graph change; a window block < 0 or >= the solver's node count.
 *   Work: 3 launches whatever the window, the drone count or the trajectory lengths (one CTA decides, writes the record
 *   and the path counts; one pass over the window entries writes the keyframe paths; a fixed grid-stride pass over
 *   max_drones x ceil(max_traj_samples / 10) writes the full paths).  The trajectory counts and the window are read on the
 *   device, so a captured sync follows push_odometry and set_window made between replays.
 *   Memory: the first call acquires 136 E + 4 (D + 1) bytes of window table and keyframe paths, 64 D S10 + 4 D bytes of
 *   full paths, 104 D bytes of records and about 1 KB of window counts and outcome (E = max_window_entries,
 *   D = max_drones, S10 = ceil(max_traj_samples / 10); 6.5 MB for 5 drones, 2e5 samples and 2048 entries), and
 *   synchronises; set_window keeps the table current after that.
 *   Later calls acquire nothing and can be captured.
 *   self_id is checked only: the sync does not depend on it (the reference's does not either). */
typedef struct {
  int32_t self_id, full_path;
  int32_t normalise, window_size;   /* the equv_cost rule of osb_multistart_options */
  double acpt_cost;
} osb_sync_params;
osb_status osb_anchor_sync_dev(osb_anchor* h, osb_solver* s, const osb_sync_params* p, void* stream);
/* osb_anchor_sync_result(): waits for the last sync -> *applied (1: applied, 0: not accepted, refused, or none ran) and
 *   *last (OSB_OK, or OSB_ERR_INVALID for a window drone without odometry); returns OSB_OK. */
osb_status osb_anchor_sync_result(osb_anchor* h, int32_t* applied, osb_status* last);
/* osb_anchor_paths(): waits for the last sync and copies drone's keyframe path (full == 0) or full path (full != 0):
 *   *n = its sample count, -1 when the drone has none (also before the first applied sync); min(*n, cap) samples of
 *   stamps [ns] and poses7 [x y z qw qx qy qz] are written. */
osb_status osb_anchor_paths(osb_anchor* h, int full, int32_t drone, int64_t* stamps, double* poses7, int cap, int32_t* n);
/* osb_anchor_record_loops_dev(): the loop map of SwarmLocalOutlierRejection::OutlierRejectionLoopEdges
 *   (swarm_outlier_rejection.cpp:106-120), which every solve makes whether or not PCM processes a pair, from the n rows
 *   osb_anchor_run_dev wrote (n = its n_out, VOID tail included), on `stream` without synchronising.  Goes after run_dev,
 *   once per solve.  Every row with status == OSB_ANCHOR_OK (loops and detections) whose id is not yet recorded:
 *     all_loop_map[id] = (id, edge.id_a, edge.id_b, stamp_a, stamp_b, edge.rel_pose) -- the re-anchored edge as first
 *       seen (stamp_a / stamp_b are the anchor node frames' stamps, loc_ret.ts_a / ts_b); when one call holds an id more
 *       than once, the first row in row order wins.  A recorded id keeps its values for good;
 *     all_loops_set_by_pair[a][b] and [b][a] gain the id.  Only the smallest id of a pair is kept (the `.begin()` that
 *       init_pose_by_loops reads); ids are only added, so it only moves down.
 *   Nothing depends on the order of atomics: a 32-bit atomicMin on the row index picks each id's first row, a second
 *   launch writes the winners, and a pair's minimum is a 64-bit atomicMin.  An id of INT64_MAX is recorded but never a
 *   pair's minimum.  Two launches whatever n.  The first call acquires 96 (H + 1) + 8 D^2 bytes (H = the power of two
 *   >= 2 max_measurements, D = max_drones) and synchronises; a handle that never makes it holds none of this.  Later
 *   calls acquire nothing and can be captured.  The map holds at most H distinct ids (the rows of one handle have at most
 *   max_measurements); past that the map is full and osb_anchor_init_by_loops_result reports OSB_ERR_CAPACITY.
 *   Refused at once with nothing enqueued (OSB_ERR_INVALID): a null handle or rows pointer with n > 0, n < 0.
 * osb_anchor_init_by_loops_dev(): SwarmLocalizationSolver::init_pose_by_loops (swarm_localization_solver.cpp:218-269),
 *   the start of the single init trial before the swarm is initialised by motion, on the device, on `stream` without
 *   synchronising.  It reads the last observe's to_init, the PCM state's inlier sets (good_loops_set), the loop map, the
 *   keyframe paths and estimated drones of the last applied sync, the trajectories and the window, and writes the
 *   solver's resident pose copy.  For each drone _id with to_init, ascending:
 *     the candidate pairs are _id's inlier sets when the PCM state holds any set of a pair of _id (a PCM result or a
 *       set_inliers set, empty ones included), else _id's pairs of the loop map -- the whole map is replaced;
 *     pairs go by ascending id2 = the other drone; a pair is skipped when its set is empty or id2 is not estimated; each
 *       later pair overwrites the earlier one, so the largest qualifying id2 decides;
 *     the loop is all_loop_map[smallest id of the set]; when its id_a != id2 it is inverted (drones and stamps swapped,
 *       relative pose inverted);
 *     pose0, t0: id2's keyframe path sample nearest to the loop's stamp_a if id2 has a path; else, for id2 == self_id,
 *       its odometry sample nearest to stamp_a; else identity and t0 = stamp_a;
 *     every window entry of _id, vo_available or not: block pose = to_xyzyaw(pose0 * odoma * rel * odomb), odoma = id2's
 *       relative odometry from t0 to stamp_a, odomb = id2's relative odometry from stamp_b to the entry's FRAME stamp
 *       (both on id2's trajectory, as the reference computes them); relative pose = pose(t1)^-1 pose(t2) of the nearest
 *       samples, 6-DoF.  A block shared by frames takes its latest frame's value.
 *   Estimated drones: every drone that had a window entry at an applied osb_anchor_sync_dev, and self_id while the window
 *   holds an entry of it (it has a keyframe).  self_id is placed like any other drone when to_init holds it.  Blocks
 *   belong to one drone (as add_as_keyframe gives them out).  Keyframes outside the window are not written: the solver
 *   holds only the window.
 *   Refused on the device with every pose unchanged, reported by osb_anchor_init_by_loops_result: a qualifying pair whose
 *   smallest id is not in the loop map, or a qualifying id2 without odometry while the window has entries or its start
 *   needs it (the reference throws from all_loop_map.at() / ego_motion_trajs.at()) -- OSB_ERR_INVALID; a full loop map --
 *   OSB_ERR_CAPACITY.
 *   Refused at once with nothing enqueued (OSB_ERR_INVALID): a null pointer, self_id outside 0..max_drones-1, the handles
 *   on different devices, no observe_dev since create, a PCM state without a device copy (no reject_anchored call yet), a
 *   window block < 0 or >= the solver's node count.
 *   One launch (one CTA: thread d decides drone d, then the threads stride over the window entries).  The first call
 *   acquires the loop map (as record_loops_dev) and the sync's paths (as sync_dev) if they are not there yet, and
 *   synchronises; later calls acquire nothing and can be captured, reading to_init, the PCM directory, the map, the paths
 *   and the trajectories on the device.  Ordered after the solver's last device call and the PCM state's last anchored
 *   call on any stream.
 * osb_anchor_init_by_loops_result(): waits for the last init_by_loops -> *last (OSB_OK when none ran); returns OSB_OK.
 * osb_anchor_loop_map(): waits for the last record_loops and sync -> *n = the number of recorded ids, min(*n, cap)
 *   records ascending by id; pair_min [max_drones][max_drones] (or null): each ordered pair's smallest id, INT64_MAX for
 *   none; estimated [max_drones] (or null): 1 for every drone that had a window entry at an applied sync.  All empty
 *   before the first call that acquires them. */
typedef struct {
  int64_t id;
  int32_t id_a, id_b;
  int64_t stamp_a, stamp_b;
  double rel_pose[7];
} osb_loop_record;
osb_status osb_anchor_record_loops_dev(osb_anchor* h, const osb_anchor_result* rows_dev, int n, void* stream);
osb_status osb_anchor_init_by_loops_dev(osb_anchor* h, osb_pcm_state* pcm, osb_solver* s, int32_t self_id, void* stream);
osb_status osb_anchor_init_by_loops_result(osb_anchor* h, osb_status* last);
osb_status osb_anchor_loop_map(osb_anchor* h, osb_loop_record* out, int cap, int32_t* n, int64_t* pair_min,
                               uint8_t* estimated);
/* Data association of anonymous detections (LocalizationDAInit, localization_DA_init.cpp, called at
 *   swarm_localization_solver.cpp:893-916).  Opt-in: a handle that never calls osb_anchor_set_data_association behaves as
 *   before, byte for byte.
 * osb_anchor_set_data_association(): enables data association with the given parameters (a later call replaces them).
 *   From then on add_measurements and add_measurements_dev also accept DET4D / DET6D rows whose id_b >= anon_min (an
 *   anonymous target; the reference's MAX_DRONE_ID = 1000); id_a must still be a drone id and loops keep both ids in
 *   0..max_drones-1.  Anonymous rows re-anchor as OSB_ANCHOR_NO_FRAME (find_node_frame_for_measurement_2drones finds no
 *   frame of their target).  The first call acquires 280 bytes of device result and synchronises.  Refused
 *   (OSB_ERR_INVALID): a null pointer, anon_min < max_drones, max_nodes < 1, a NaN accept_thres.
 * osb_anchor_data_association_dev(): the DA branch of solve() on the device, on `stream` without synchronising.  One launch
 *   of one CTA.  It runs when all of these hold on the device (else it changes nothing and reports applied = 0, OSB_OK):
 *   the last observe's node set holds a drone with enable == 0 (has_node_not_inited), holds more than one drone, and the
 *   store holds a detection (DET4D or DET6D: add_new_detection pushes both kinds to all_detections_6d).  Then, over the
 *   store in order, the trajectories and the keyframe paths of the last applied osb_anchor_sync_dev:
 *     unidentified = the id_b >= anon_min of the detections whose id_a has odometry; per such id the detector and the
 *       covariance of its LAST such detection, and the FIRST detection of its SMALLEST detector (estimate_path);
 *     no unidentified id, or self_id without odometry: nothing happens;
 *     t0 = the largest first odometry stamp; est[self_id] = self's odometry at t0; then every drone with a keyframe path,
 *       ascending: est[d] = path(d) at t0 (stamp t1) * odom_d(t1)^-1 odom_d(t0) (nearest samples, ties to the earlier);
 *     the reference's DFS, literally (DESIGN.md section 7b): at each level the remaining ids ascending, skipping one whose
 *       detector has no estimate; each drone with odometry other than the detector is tried, ascending; for a candidate
 *       c > 0 the pose est[smallest detector] * odom(t0, ts_a) * relative_pose * odom_c(ts_b, t0) must pass
 *       smd(log(est[c]^-1 pose), cov) < accept_thres when c has an estimate, and becomes est[c]; drone 0 is guessed but
 *       never estimated; a leaf succeeds iff accept_thres > 0 and est covers every drone with odometry; the first
 *       success of a level is kept, every candidate of that level is still searched, and a level whose id finds none
 *       goes on to the next id.
 *   On success every detection with id_b >= anon_min gets id_b = its guess, in place (anyoumos_det_mapper stays empty,
 *   as in the reference) and the word osb_anchor_data_association_word points to becomes 1; else it becomes 0.
 *   Refused on the device with no row renamed (applied = 0), reported by osb_anchor_data_association_result:
 *   OSB_ERR_INVALID where the reference throws (a keyframe-path drone without odometry; estimate_path of a smallest
 *   detector without an estimate; a leaf whose detectors or guessed drones lack an estimate, verify's at(); a success while
 *   an anonymous row's id is not unidentified, guess.at()); OSB_ERR_CAPACITY for more than 32 unidentified ids or more DFS
 *   calls than max_nodes.  Refused at once with nothing enqueued (OSB_ERR_INVALID): a null handle, self_id outside
 *   0..max_drones-1, no set_data_association or no observe_dev since create.  The first call acquires the device counts
 *   (as add_measurements_dev) and the sync's paths (as sync_dev) if they are not there yet, and synchronises; later calls
 *   acquire nothing and can be captured.
 *   The branch, as solve() runs it: run_dev -> observe_dev -> record_loops_dev -> reject_anchored -> data_association_dev
 *   -> run_dev_if -> observe_dev_if -> record_loops_dev -> reject_anchored -> ...  (estimate_observability runs the loop
 *   map and PCM each time; when nothing was applied the second pair sees the same rows and changes nothing).
 *   max_nodes: the search runs on one thread and a search that does not resolve uses its whole budget.  The budget counts
 *   DFS calls, not gate evaluations: one call can gate up to n_u x (D - 1) candidates (8160 at 32 ids and 256 drones), so
 *   a search is bounded by max_nodes x n_u x (D - 1) gates, about 7.5 us each on an H100 80GB HBM3 at 700 W (measured).
 *   At 32 ids and 256 drones that bounds a call by about 61 ms and the bindings' default of 4096 calls by about 250 s
 *   (a measured worst case took about 50 ms a call).  Size max_nodes from the gate bound where latency matters
 *   (DESIGN.md section 5).
 * osb_anchor_data_association_result(): waits for the last data_association_dev -> *applied (1: rows renamed), *status
 *   (OSB_OK, or the refusal), *n = the unidentified ids of an applied call and min(*n, cap) (anonymous id, drone) pairs,
 *   ascending by anonymous id.  All zero before the first call.
 * osb_anchor_data_association_word(): the device address of the applied word (an int32, 0 before the first call), for
 *   osb_anchor_run_dev_if / osb_anchor_observe_dev_if.  OSB_ERR_INVALID before set_data_association.
 * osb_anchor_run_dev_if() / osb_anchor_observe_dev_if(): run_dev and observe_dev with the same launches, predicated on
 *   *pred_dev read on the device: 0 writes nothing (rows, state and record keep every byte), else the call is run_dev's /
 *   observe_dev's, except that observe_dev_if keeps a motion_new the record already holds (motion_new |= this call's), so
 *   the record reflects both observe calls of one solve.  run_dev_if returns the same *n_out as run_dev. */
typedef struct {
  float accept_thres;            /* DA_accept_thres (3.345f), compared as a double */
  int32_t anon_min;              /* MAX_DRONE_ID (1000): detection targets at or above it are anonymous */
  int32_t max_nodes;             /* search budget: DFS calls per data_association_dev */
  int32_t reserved;
} osb_da_params;
typedef struct {
  int32_t anon_id, drone_id;
} osb_da_guess;
osb_status osb_anchor_set_data_association(osb_anchor* h, const osb_da_params* p);
osb_status osb_anchor_data_association_dev(osb_anchor* h, int32_t self_id, void* stream);
osb_status osb_anchor_data_association_result(osb_anchor* h, int32_t* applied, osb_status* status, osb_da_guess* guess,
                                              int cap, int32_t* n);
osb_status osb_anchor_data_association_word(osb_anchor* h, const int32_t** applied_dev);
osb_status osb_anchor_run_dev_if(osb_anchor* h, const uint8_t* yaw_observable, osb_anchor_result* out_dev, int32_t* n_out,
                                 const int32_t* pred_dev, void* stream);
osb_status osb_anchor_observe_dev_if(osb_anchor* h, const osb_observe_params* p, osb_anchor_result* rows_dev, int n,
                                     const int32_t* pred_dev, void* stream);
/* osb_anchor_predict(): PredictSwarm / PredictNode / NodeCooridnateOffset (swarm_localization_solver.cpp:673-765) for one
 *   frame of n drones (distinct ids, vo_poses7 [n][7] their odometry now), from the prediction record of the last applied
 *   sync.  With the drone's record (saved block pose P4, its frame's self_pose vo):
 *     node_pose = Pose(P4, yaw) * DeltaPose(set_yaw_only(vo), vo_now, 6-DoF), valid iff the drone is enabled in the last
 *       observe (osb_anchor_observability; self_id always is);
 *     base_pose = set_yaw_only(Pose(P4, yaw)) * set_yaw_only(vo)^-1.
 *   A drone without a record (no applied sync pushed a frame holding it), or finish_init == 0, gives neither.  One launch,
 *   then a synchronisation (no launch before the first sync or with finish_init == 0); the record never leaves the
 *   device.  Refused (OSB_ERR_INVALID): a null pointer, n outside 0..max_drones, a drone id or self_id outside
 *   0..max_drones-1.  The first call that launches acquires 188 D bytes of query and result buffers. */
typedef struct {
  int32_t self_id, finish_init;
} osb_predict_params;
typedef struct {
  int32_t node_valid, reserved0;
  double node_pose[7];
  int32_t base_valid, reserved1;
  double base_pose[7];
} osb_predict_result;
osb_status osb_anchor_predict(osb_anchor* h, const osb_predict_params* p, int n, const int32_t* drones,
                              const double* vo_poses7, osb_predict_result* out);

/* ------------------------------------------------------------------------------------------------------------
 * The solve's chain from re-anchoring to factor rows on the device: run_dev -> reject_anchored -> compact_factors_dev, all
 *   stream-ordered on one stream, then one copy of the count and of at most that many rows.
 * osb_pcm_state_reject_anchored(): the PCM rejection of the rows osb_anchor_run_dev wrote, read in place.  Equals
 *   osb_pcm_state_reject over (rows[i].edge, rows[i].id) for the rows with status == OSB_ANCHOR_OK, in row order, with every
 *   rule of reject() above; keep_dev[i] = that call's keep for those rows and 0 for every other row.  n is run_dev's n_out.
 *   Work: seven kernel launches whatever n and however many pairs change (none when n == 0): two passes over the rows find
 *   the fresh ones (OK, routed, id not in the device's seen set) and compact their indices in row order; one warp plans the
 *   appends (a pair's new loops keep row order, new pairs take slots in order of first appearance) and checks
 *   pair_capacity and max_pairs before it writes anything; the consistency-graph growth and maxCliqueHeu run from that
 *   device-built job list (one clique CTA per possible pair, exiting early when the pair did not change); the inlier sets
 *   are replaced by the cliques' ids; keep_dev is each OK row's membership in its pair's set.  No host synchronisation and
 *   no allocation after the first call, so the sequence can be captured into a CUDA graph.  Calls on one handle must be
 *   ordered: on one stream, or joined by the caller.
 *   Errors: null pointers or n < 0 return OSB_ERR_INVALID at once.  A call that would exceed pair_capacity or max_pairs is
 *   refused on the device: the state is unchanged and keep_dev is not written; osb_pcm_state_status() then returns
 *   OSB_ERR_CAPACITY, and so does (once) the next host-side call on the handle (reject, inliers, set_inliers, pair) instead
 *   of running.
 *   One state: the host-side calls and the anchored path may be mixed in any order.  The first anchored call builds the
 *   device copy from the host record; host-side calls write their changes through to it before they return, and the first
 *   host-side call after an anchored call synchronises once (on the anchored call's stream; when that call was captured,
 *   the caller must have run and synchronised the graph) and refreshes the host record from the device.
 *   Memory of the first call: the slots of all max_pairs pairs not yet acquired (max_pairs x slot size above, 63 MB for
 *   15 pairs at 4096), a seen table of 8 x 2^ceil(log2(2 max_pairs pair_capacity)) bytes (>= 8 KB; 1 MB for 15 x 4096),
 *   4 x 4 max_pairs pair_capacity bytes of row indices, an event and small tables.  set_inliers may acquire a buffer for a
 *   set larger than pair_capacity or of a pair without loops.
 * osb_pcm_state_status(): synchronises with the last anchored call and writes its status to *last (OSB_OK when none ran);
 *   returns the same value. */
osb_status osb_pcm_state_reject_anchored(osb_pcm_state* s, const osb_anchor_result* rows_dev, int n, uint8_t* keep_dev,
                                         void* stream);
osb_status osb_pcm_state_status(osb_pcm_state* s, osb_status* last);
/* osb_anchor_compact_factors_dev(): the rows with skip == 0 && (keep_dev == NULL || keep_dev[i]), in row order, as the
 *   solver's SoA -- type [k] (OSB_FACTOR_RELPOSE), ia / ib [k] (the rows' pose-block ids), payload [k][OSB_PAYLOAD_LEN],
 *   huber [k] (0/1) -- exactly what osb::add_anchored_factors appends; *count_dev = k.  All pointers are device memory and
 *   the outputs must hold n rows.  One launch (also for n == 0, which writes count 0), a block scan: deterministic. */
osb_status osb_anchor_compact_factors_dev(const osb_anchor_result* rows_dev, int n, const uint8_t* keep_dev,
                                          int32_t* type, int32_t* ia, int32_t* ib, double* payload, uint8_t* huber,
                                          int32_t* count_dev, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * The UWB half of add_new_swarm_frame and of every solve, on the device.
 * osb_anchor_add_keyframe_dev(): add_as_keyframe (swarm_localization_solver.cpp:517-540) for one keyframe the caller has
 *   accepted (judge_is_key_frame, the block assignment, the odometry factors and set_window stay with the caller).  nodes
 *   [n_nodes] in ascending drone id (SwarmFrame::id2nodeframe's order), each followed in `dists` by its n_distances
 *   (peer, metres) pairs in ascending peer id (NodeFrame::dis_map's order).  On `stream`, without synchronising:
 *   a. each node with new_block writes its block's initial pose (x y z yaw) into the solver's resident device poses:
 *      a static node, or a dynamic one with prev_block < 0 that is not self_id before finish_init: the odometry position
 *        plus a draw in [-5, 5) per axis (RAND_INIT_XY), the odometry yaw (:300-305, :329-335);
 *      self_id before finish_init: the odometry pose (:306-310);
 *      otherwise: Pose(prev block, yaw) * DeltaPose(prev_pose, pose, 4-DoF) (Predict_By_VO, :279-298).
 *      A node with new_block == 0 writes nothing (the not-moving merge of :291-294, a static node's first block).  The
 *      draw replaces rand(): splitmix64 of (seed, splitmix64(stamp) ^ (drone << 2 | axis)), as the multistart draws;
 *   b. outlier_distance of each distance to a peer of this keyframe with vo_available (outlier_rejection_frame, :408-515):
 *      before finish_init: |asin((z_peer - z) / d)| > elevation_threshold || !enable_distance, z the odometry heights;
 *      after it: |d - |p_peer - p|| > outlier_threshold || d < minimum_distance || |asin((z_peer - z) / d)| >
 *        elevation_threshold || !enable_distance, p the estimated positions of this keyframe (step a's and the resident
 *        poses of reused blocks); a node absent from the previous keyframe is skipped, and the first node (in id order)
 *        without vo_available there ends the walk -- its flags and those of every later node are not written (the
 *        reference's `return`).  A NaN asin (|dz| > d) compares false.  The float thresholds are compared as doubles;
 *        debug_no_rejection sets both thresholds to 1e8f and minimum_distance to -1 (:89-96);
 *   c. stores the keyframe (its nodes, distances and flags: 1 outlier, 0 not, -1 not written) in the handle's ring of
 *      max_keyframes slots, keyed by stamp; the oldest slot is overwritten.  A call whose slot holds a
 *      keyframe of the window set last, and a set_window with a frame (holding entries) whose keyframe has left the ring,
 *      are refused with OSB_ERR_CAPACITY: max_keyframes must cover the window.
 *   One launch.  The inputs go through a pinned staging ring of 4 slots: a call waits (on the host) only for the call 4
 *   before it.  Ordered after the solver's last device call on any stream.  The solver's host mirror is stale afterwards:
 *   its next host-side call waits for this write and refreshes it, and its next device call starts from the written
 *   poses.
 *   Refused at once with nothing enqueued (OSB_ERR_INVALID): a null pointer, max_keyframes == 0, n_nodes outside
 *   1..max_drones, nodes not in ascending drone id, a drone or peer id outside 0..max_drones-1, peers not ascending, a
 *   block or a used prev_block outside 0 .. the solver's node count - 1, a stamp already stored, the handles on different
 *   devices; more distances than max_keyframe_distances gives OSB_ERR_CAPACITY.  The solver's next device call, on any
 *   stream, waits for the write.  The first call acquires the store
 *   (max_keyframes x (16 + 156 max_drones + 17 max_keyframe_distances) bytes and a frame table of 20 max_window_entries
 *   bytes, sized once), the staging
 *   ring and its events, and synchronises.
 * osb_anchor_keyframe_flags(): waits for the last keyframe and copies the stored flags of the keyframe at stamp_ns, in
 *   `dists` order: *n = their count, -1 when the stamp is not stored; min(*n, cap) are written. */
typedef struct {                 /* one NodeFrame of a keyframe, 152 bytes */
  int32_t drone_id;
  int32_t block;                 /* the pose block the caller assigned (est_poses_idts[id][ts]) */
  int32_t new_block;             /* 1: a new block, its initial pose is written; 0: a reused block */
  int32_t prev_block;            /* new dynamic block: the block of the drone's latest keyframe, -1 when it has none */
  int32_t vo_available, is_static, frame_available, dists_available;
  int32_t n_distances;           /* this node's pairs in the call's dists, following the previous nodes' */
  int32_t reserved;
  double pose[7];                /* odometry x y z qw qx qy qz */
  double prev_pose[7];           /* the odometry at the drone's latest keyframe (read when prev_block is) */
} osb_keyframe_node;
typedef struct {
  int32_t peer, reserved;
  double distance;               /* metres */
} osb_keyframe_distance;
typedef struct {
  int32_t self_id, finish_init, enable_distance, debug_no_rejection;
  float outlier_threshold;       /* distance_measurement_outlier_threshold */
  float elevation_threshold;     /* distance_measurement_outlier_elevation_threshold */
  float minimum_distance;
  int32_t reserved;
  uint64_t seed;
} osb_keyframe_params;
osb_status osb_anchor_add_keyframe_dev(osb_anchor* h, osb_solver* s, int64_t stamp_ns, int n_nodes,
                                       const osb_keyframe_node* nodes, int n_distances, const osb_keyframe_distance* dists,
                                       const osb_keyframe_params* p, void* stream);
osb_status osb_anchor_keyframe_flags(osb_anchor* h, int64_t stamp_ns, int8_t* flags, int cap, int32_t* n);
/* osb_anchor_distance_factors_dev(): setup_problem_with_sferror (swarm_localization_solver.cpp:1102-1154) of every window
 *   frame, appended to the SoA osb_anchor_compact_factors_dev wrote, at row *count_dev.  Goes between compact_factors_dev
 *   and the resident solve (steady or multistart).  For each frame of the window set last whose stamp is stored, each
 *   stored node a that has a window entry in that frame, and each of its distances to a peer b: one OSB_FACTOR_DISTANCE
 *   row iff enable_distance && frame_available && dists_available (of a) && b < a && b has a window entry in the frame &&
 *   the distance is not flagged an outlier (an unwritten flag is not) && (a == self_id || enable[a] of the last
 *   osb_anchor_observe_dev).  Rows in frame order, then a, then b ascending; ia / ib = the window entries' blocks of a
 *   and b; payload [d, 1 / sqrt((double)distance_measurement_cov), 0 ...] (the float parameter widened, then the fp64
 *   square root and division); huber = !debug_no_rejection.  NodeFrame::distance_available (swarm_msgs, not in the
 *   reference tree) is taken as "has a distance to b that is not flagged"; cutting_edges enables every distance
 *   (:1225-1297).  A count that would pass max_tail (the buffers' rows) writes -1 to *count_dev and no row past max_tail,
 *   so the solve refuses the tail; *count_dev < 0 on entry is left as it is.
 *   One launch of one CTA (a block scan per frame: deterministic, no atomics).  Everything is read on the device, so the
 *   call can be captured into a CUDA graph: a replay's rows follow that replay's observe and the window set before it.
 *   Refused at once with nothing enqueued (OSB_ERR_INVALID): a null pointer, max_tail < 0, self_id outside
 *   0..max_drones-1, max_keyframes == 0, or no observe_dev since create.  The first call acquires what the first
 *   add_keyframe_dev does. */
typedef struct {
  int32_t self_id, enable_distance, debug_no_rejection;
  float distance_measurement_cov;
} osb_distance_params;
osb_status osb_anchor_distance_factors_dev(osb_anchor* h, const osb_distance_params* p, int32_t* type, int32_t* ia,
                                           int32_t* ib, double* payload, uint8_t* huber, int32_t* count_dev, int max_tail,
                                           void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Geometric filter of the loop matcher (SURVEY.md 8f-1, first half) -- the inlier mask of
 *   cv::findHomography(old_2d, new_2d, CV_RANSAC, 3, mask)            swarm_loop/src/loop_detector.cpp:589-598
 * for n_pairs correspondence sets at once.  src = old_2d, dst = new_2d, [n_pairs][max_n][2] floats, n[pair] points each
 * (max_n <= 256).  mask [n_pairs][max_n] (1 = inlier), n_inliers [n_pairs], winner [n_pairs] (hypothesis index, -1 if
 * none; may be NULL in the host variant).  Fewer than 4 points: empty mask (the reference rejects the pair, :598-600).
 * OpenCV's RANSAC is randomised; this one is deterministic in (points, seed): 512 hypotheses drawn by a counter-based
 * hash, same 4-point model / error / threshold rule, first best hypothesis wins (oracle/geometry_ref.py, pinned against
 * cv2 on well-separated data).  No process-wide state: the _dev entry point takes its scratch from the stream-ordered
 * allocator of `stream`, so concurrent callers on different streams are safe. */
osb_status osb_homography_ransac(const float* src, const float* dst, const int32_t* n, int n_pairs, int max_n,
                                 float thresh, uint32_t seed, uint8_t* mask, int32_t* n_inliers, int32_t* winner);
osb_status osb_homography_ransac_dev(const float* src_dev, const float* dst_dev, const int32_t* n_dev, int n_pairs,
                                     int max_n, float thresh, uint32_t seed, uint8_t* mask_dev, int32_t* n_inliers_dev,
                                     int32_t* winner_dev, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Keypoints -> 3-D landmarks + landmarks_flag (SURVEY.md 8f-3) -- replaces the per-keypoint loops of
 *   LoopCam::generate_stereo_image_descriptor (swarm_loop/src/loop_cam.cpp:393-432: liftProjective, triangulatePoint :73-106,
 *   err <= TRIANGLE_THRES, in front of the up camera) and generate_gray_depth_image_descriptor (:276-302: depth look-up in
 *   mm, DEPTH_NEAR_THRES < dep < DEPTH_FAR_THRES, lift through pose_cam).  Arrays are [n_dirs][max_n][...]; intrinsics =
 *   fx fy cx cy of the distortion-free flattened pinhole (HOST pointer in both variants); poses are 7 doubles
 *   (x y z, qw qx qy qz), already pose_drone * extrinsic; nothing is lifted when a direction has <= accept_min_3d_pts
 *   keypoints (:385-391, :267).  stereo_match[d][i] = index of the down keypoint matched to up keypoint i, or -1. */
osb_status osb_stereo_lift(const float* kp_up, const float* kp_down, const int32_t* stereo_match, const int32_t* n_up,
                           const int32_t* n_down, int n_dirs, int max_n, const double* intrinsics, const double* pose_up,
                           const double* pose_down, double triangle_thres, int accept_min_3d_pts, float* pts3d,
                           uint8_t* flag_up, uint8_t* flag_down);
osb_status osb_stereo_lift_dev(const float* kp_up_dev, const float* kp_down_dev, const int32_t* stereo_match_dev,
                               const int32_t* n_up_dev, const int32_t* n_down_dev, int n_dirs, int max_n,
                               const double* intrinsics, const double* pose_up_dev, const double* pose_down_dev,
                               double triangle_thres, int accept_min_3d_pts, float* pts3d_dev, uint8_t* flag_up_dev,
                               uint8_t* flag_down_dev, void* stream);
osb_status osb_depth_lift(const float* kp, const int32_t* n, int n_dirs, int max_n, const uint16_t* depth_mm, int height,
                          int width, const double* intrinsics, const double* pose_cam, double near_thres, double far_thres,
                          int accept_min_3d_pts, float* pts3d, uint8_t* flag);
osb_status osb_depth_lift_dev(const float* kp_dev, const int32_t* n_dev, int n_dirs, int max_n, const uint16_t* depth_mm_dev,
                              int height, int width, const double* intrinsics, const double* pose_cam_dev, double near_thres,
                              double far_thres, int accept_min_3d_pts, float* pts3d_dev, uint8_t* flag_dev, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Relative pose of a loop candidate (SURVEY.md 8f-1, second half) -- replaces LoopDetector::compute_relative_pose
 *   (swarm_loop/src/loop_detector.cpp:355-413: cv::solvePnPRansac(matched_3d_now, matched_2d_norm_old, K = I, iterations
 *   100 / 1000 in init mode, reprojection error 3), PnPRestoCamPose, DeltaPose, RPerror :338-351, pnp_result_verify :317-336)
 *   and LoopDetector::check_loop_odometry_consistency (:294-315): everything between the matched landmarks and the LoopEdge.
 * pts3d [n_cand][max_n][3] = matched_3d_now (landmarks in the NEW drone's body frame), pts2d [n_cand][max_n][2] =
 *   matched_2d_norm_old (normalised coordinates in the OLD camera), n [n_cand] valid counts, max_n <= 1024.
 * OpenCV's RANSAC is randomised; this one is deterministic in (points, seed, prior): hypothesis h fits 4 hashed
 *   correspondences by a fixed-schedule Levenberg-Marquardt started from `prior` (the odometry prediction the reference
 *   computes and leaves unused, initial_old_cam_pose :377-382), the first hypothesis with the most inliers
 *   (reprojection error^2 <= thresh^2, no cheirality test, as cv::projectPoints) wins, and the pose is the LM minimiser over
 *   its inliers -- the definition of solvePnPRansac's result (oracle/pnp_ref.py, pinned against cv2.solvePnPRansac).
 * Poses are 7 doubles (x y z, qw qx qy qz); Swarm::Pose / DeltaPose / quat2eulers are defined in oracle/pnp_ref.py
 *   (swarm_msgs is not in the reference tree). */
typedef struct {
  int32_t iterations;            /* 100, or 1000 in init mode (:385-391) */
  float reproj_thresh;           /* 3 (:393) */
  uint32_t seed;
  int32_t is_4dof;               /* DeltaPose(..., is_4dof) (:403) */
  int32_t min_loop_num;          /* MIN_LOOP_NUM, or INIT_MODE_MIN_LOOP_NUM in init mode (:328-332) */
  int32_t same_drone;            /* 1: drone_id_a == drone_id_b, run the odometry-consistency check (:294-298) */
  double rperr_thres;            /* RPERR_THRES */
  double accept_loop_yaw_rad;    /* ACCEPT_LOOP_YAW_RAD */
  double max_loop_dis;           /* MAX_LOOP_DIS */
  double odometry_consistency_threshold;
  double prior[7];               /* initial (R, t) guess, x_cam_old = R X_now + t: (drone_pose_now^-1 drone_pose_old extrinsic)^-1 */
  double extrinsic[7];           /* old camera in the old drone's body frame */
  double drone_pose_now[7];
  double drone_pose_old[7];
  double odom_rel[7];            /* same_drone: ego-motion between the two stamps (get_relative_pose_by_ts) */
  double odom_edge_cov[36];      /* same_drone: odometry covariance + edge covariance, 6x6 row-major (:303) */
} osb_pnp_params;
typedef struct {
  int32_t pnp_success;           /* a model with >= 4 inliers was found */
  int32_t n_inliers;
  int32_t winner;                /* winning hypothesis, -1 if none */
  int32_t verified;              /* pnp_result_verify (:317-336) */
  int32_t odometry_consistent;   /* check_loop_odometry_consistency (:294-315); 1 for inter-drone loops */
  int32_t reserved;
  double rperr;                  /* RPerror (:338-351) */
  double md;                     /* squared Mahalanobis distance of the odometry check */
  double pose_cam[7];            /* (t, q) of the PnP solution: x_cam_old = R X_now + t */
  double dp_old_to_new[4];       /* DP_old_to_new: x y z yaw -- the LoopEdge's relative pose */
} osb_pnp_result;
osb_status osb_pnp_ransac(const float* pts3d, const float* pts2d, const int32_t* n, int n_cand, int max_n,
                          const osb_pnp_params* params, uint8_t* mask /*[n_cand][max_n]*/, osb_pnp_result* results);
osb_status osb_pnp_ransac_dev(const float* pts3d_dev, const float* pts2d_dev, const int32_t* n_dev, int n_cand, int max_n,
                              const osb_pnp_params* params_dev, uint8_t* mask_dev, osb_pnp_result* results_dev, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Keyframe front-end -- the per-keyframe pipeline of LoopCam::on_flattened_images (loop_cam.cpp:178-229 ->
 *   generate_stereo_image_descriptor :341-523) followed by LoopDetector::on_image_recv's database work
 *   (loop_detector.cpp:89-104,150-287) and compute_correspond_features' matcher (loop_detector.cpp:539-587),
 *   kept resident on the GPU.  With the cameras set, the triangulation (or depth look-up) runs inside extract; with the
 *   geometric filter, the homography RANSAC runs inside query; and osb_frontend_compute_loop turns a round's hits into
 *   loop edges (correspondences, PnP-RANSAC and the reference's checks) on the device as well.
 *
 * One keyframe = n_dirs directions x (up image, down image) (STEREO_FISHEYE: n_dirs=4, 8 images).
 * osb_keyframe_record is the fixed-size record every drone contributes to the swarm-wide exchange
 * (replaces LoopNet::broadcast_fisheye_desc, swarm_loop/src/loop_net.cpp:20-120): on the 8-GPU box it is
 * the unit of ONE ncclAllGather.
 * -----------------------------------------------------------------------------------------------------------*/
typedef struct {
  int32_t drone_id;
  int32_t msg_id;
  int32_t n_dirs;
  int32_t reserved;
  /* the image fields below are the up image's; with osb_frontend_set_main_camera(OSB_MAIN_CAMERA_DOWN) the down image's and
     stereo_match the other way round (see there) */
  int32_t n_kpts[OSB_MAX_DIRS];                                        /* landmark_num per direction (up image) */
  int32_t n_kpts_down[OSB_MAX_DIRS];
  float global_desc[OSB_MAX_DIRS][OSB_DEEP_DESC_SIZE];                 /* image_desc */
  float local_desc[OSB_MAX_DIRS][OSB_MAX_KPTS][OSB_FEATURE_DESC_SIZE]; /* feature_descriptor (up image) */
  float kpts[OSB_MAX_DIRS][OSB_MAX_KPTS][2];                           /* landmarks_2d (up image) */
  int32_t stereo_match[OSB_MAX_DIRS][OSB_MAX_KPTS];                    /* down-image keypoint index matched to each
                                                                          up keypoint by the cross-check matcher, or -1 */
  float landmarks_3d[OSB_MAX_DIRS][OSB_MAX_KPTS][3];                   /* landmarks_3d (loop_cam.cpp:405-432): triangulated
                                                                          in the drone's odometry frame; zero without flag */
  int32_t landmarks_flag[OSB_MAX_DIRS][OSB_MAX_KPTS];                  /* landmarks_flag.  With osb_frontend_set_cameras: 1
                                                                          iff the stereo pair triangulates (err <=
                                                                          TRIANGLE_THRES, in front of the camera, :423);
                                                                          without cameras: stereo_match >= 0, a superset */
} osb_keyframe_record;

typedef struct {
  int32_t hit_id;                /* database image id (remote ids + OSB_REMOTE_MAGIN_NUMBER) or -1 */
  int32_t hit_dir;               /* imgid2dir of the hit (direction_old) or -1 */
  float hit_score;               /* `distance` of query_from_database (-1 when untouched) */
  int32_t accepted;              /* id != -1 && distance > -1 (loop_detector.cpp:265) */
  int32_t swapped;               /* 1 when the hit is a remote keyframe and the query keyframe is our own: the reference
                                    then calls compute_loop(old, new) (loop_detector.cpp:113-118), i.e. the DATABASE
                                    frame is the matcher's query side ("new") and the current keyframe the train side */
  int32_t hit_msg_id;            /* msg_id of the matched keyframe = imgid2fisheye[best_image_id], the key of
                                    fisheyeframe_database (loop_detector.cpp:272-275,105-111); -1 without a hit, and for rows
                                    put in with osb_frontend_db_load */
  int32_t hit_drone_id;          /* drone_id of the matched keyframe (fisheyeframe_database[msg_id].drone_id); -1 without a hit */
  int32_t dir_new[OSB_MAX_DIRS]; /* direction pairing of compute_correspond_features (loop_detector.cpp:455-465), */
  int32_t dir_old[OSB_MAX_DIRS]; /* one slot per pair with landmarks on both sides, -1 = unused slot */
  int32_t n_matches[OSB_MAX_DIRS];                 /* cross-check matches new-vs-old per direction pair */
  int32_t match_new[OSB_MAX_DIRS][OSB_MAX_KPTS];   /* queryIdx */
  int32_t match_old[OSB_MAX_DIRS][OSB_MAX_KPTS];   /* trainIdx */
  /* geometric filter (osb_frontend_config::geometric_filter; loop_detector.cpp:569-598): per direction pair, the
   * matches whose NEW landmark has a 3-D flag (stereo_match >= 0) and that pass the homography-RANSAC mask of
   * findHomography(old_2d, new_2d, RANSAC, 3).  geo_valid = 0 when fewer than 4 flagged matches remained (the reference
   * returns false for the pair).  Untouched (zero) when the filter is off. */
  int32_t geo_valid[OSB_MAX_DIRS];
  int32_t n_geo[OSB_MAX_DIRS];
  int32_t geo_new[OSB_MAX_DIRS][OSB_MAX_KPTS];
  int32_t geo_old[OSB_MAX_DIRS][OSB_MAX_KPTS];
} osb_loop_result;

typedef struct osb_frontend osb_frontend;
typedef struct {
  int32_t width, height, n_dirs, max_num;
  float sp_thres;                /* superpoint_thres */
  int32_t self_id;
  int32_t db_capacity;           /* rows per database (local and remote) */
  double inner_product_thres;    /* INNER_PRODUCT_THRES (query_thres) */
  double init_mode_product_thres;/* INIT_MODE_PRODUCT_THRES */
  int32_t match_index_dist;      /* MATCH_INDEX_DIST */
  int32_t query_dir;             /* direction queried: 1 for STEREO_FISHEYE, 0 for pinhole (loop_detector.cpp:249-257) */
  int32_t zero_bottom_quarter;   /* 1 for STEREO_FISHEYE: blank rows [3H/4, H) of every image (loop_cam.cpp:535-538) */
  int32_t accept_min_3d_pts;     /* ACCEPT_MIN_3D_PTS: stereo match skipped when n_kpts <= this (loop_cam.cpp:385-391) */
  int32_t geometric_filter;      /* 1: run the 3-D-flag + homography-RANSAC filter of loop_detector.cpp:569-598 in query */
  int32_t ransac_seed;           /* seed of the deterministic RANSAC (osb_homography_ransac) */
} osb_frontend_config;

osb_status osb_frontend_create(osb_frontend** out, const osb_frontend_config* cfg, const float* sp_weights,
                               size_t n_sp_weights, const float* pca_comp, const float* pca_mean,
                               const float* nv_weights, size_t n_nv_weights);
osb_status osb_frontend_destroy(osb_frontend* h);
/* extract: images_up/down [n_dirs][H][W] uint8 HOST (pinned or pageable) -> record written to `record_dev`
 * (DEVICE pointer, sizeof(osb_keyframe_record)); no synchronisation.  msg_id is stored in the record. */
osb_status osb_frontend_extract(osb_frontend* h, const uint8_t* images_up, const uint8_t* images_down,
                                int32_t msg_id, osb_keyframe_record* record_dev, void* stream);
/* same with images already on the device */
osb_status osb_frontend_extract_dev(osb_frontend* h, const uint8_t* images_up_dev, const uint8_t* images_down_dev,
                                    int32_t msg_id, osb_keyframe_record* record_dev, void* stream);
/* ingest: add `n_records` records (DEVICE array, e.g. the all-gather output; records whose drone_id == self go to the
 * local database, others to the remote one; index `skip` is ignored, pass -1 to ingest all) -- add_to_database. */
osb_status osb_frontend_ingest(osb_frontend* h, const osb_keyframe_record* records_dev, int n_records, int skip,
                               void* stream);
/* the same for ONE record that the caller knows to be this drone's own (the record extract has just written: on_image_recv's
 * add_to_database, loop_detector.cpp:89).  The routing is still by drone_id on the device; what the promise buys is that the
 * host does not have to assume the record might have gone to the remote database, so a drone that has never received a
 * foreign keyframe does not scan an empty remote store on every query. */
osb_status osb_frontend_ingest_own(osb_frontend* h, const osb_keyframe_record* record_dev, void* stream);
/* query: run query_from_database for the keyframe in `record_dev` (must already be ingested if it is an own keyframe,
 * as on_image_recv does) and, on a hit, the per-direction cross-check match against the stored keyframe; the result
 * is written to `result_dev` (DEVICE).  init_mode / nonkeyframe as loop_detector.cpp:176. */
osb_status osb_frontend_query(osb_frontend* h, const osb_keyframe_record* record_dev, int init_mode,
                              int nonkeyframe, osb_loop_result* result_dev, void* stream);
/* query_from_database for keyframes received from other drones (loop_detector.cpp:98-119,191-195), a batch at once,
 * e.g. the all-gather output of a round.  For every r != skip whose drone_id != self_id, results_dev[r] is what
 * osb_frontend_query(h, records_dev + r, init_mode[r], 0, ...) would write at this point of `stream`.  Reads the local
 * store only: the remote store, and whether the records have been ingested yet, do not affect the results.
 * Records r == skip or with drone_id == self_id get the gate-closed result (hit_id -1, hit_score -1, accepted 0, every
 * direction slot -1, n_matches 0; with the geometric filter n_geo 0 and geo_valid 0).  init_mode: HOST array [n_records]
 * of 0/1 or NULL (all 0).  0 <= n_records <= 64 (the ingest limit); n_records == 0 does nothing.  The first call acquires
 * the handle's scratch for 64 records (about 4 * 64 * max_num^2 floats); no later call allocates.  No host
 * synchronisation.  nonkeyframe is not an argument: the reference ignores it for foreign keyframes (:191-195). */
osb_status osb_frontend_query_received(osb_frontend* h, const osb_keyframe_record* records_dev, int n_records, int skip,
                                       const uint8_t* init_mode, osb_loop_result* results_dev, void* stream);
/* the whole single-drone step with HOST buffers: extract + ingest(own) + query, one synchronisation at the end. */
osb_status osb_frontend_process(osb_frontend* h, const uint8_t* images_up, const uint8_t* images_down,
                                int32_t msg_id, osb_keyframe_record* record_host, osb_loop_result* result_host);
/* synchronise `stream` and refresh the host-side row counts (call once per keyframe round when driving the
 * extract / ingest / query stages separately, e.g. around the multi-GPU all-gather) */
osb_status osb_frontend_finish(osb_frontend* h, void* stream);
int64_t osb_frontend_db_size(osb_frontend* h, int remote);
osb_status osb_frontend_db_reset(osb_frontend* h);
/* bulk-load rows into a database without running the networks (benchmark / replay set-up): global descriptors
 * [n][4096] and optional local descriptors [n][max_num][64] + counts [n] (HOST).  In OSB_DB_STORAGE_FP16 the global
 * descriptors are converted on the device through a 4 MB staging buffer acquired by the first such load. */
osb_status osb_frontend_db_load(osb_frontend* h, int remote, int64_t n, const float* global_desc,
                                const float* local_desc, const int32_t* n_kpts);
/* Stereo triangulation inside extract (SURVEY.md 8f-3): with the cameras set, every keyframe's record carries the
 * reference's landmarks_3d / landmarks_flag (loop_cam.cpp:393-432) -- up/down keypoints lifted through the distortion-free
 * pinhole of the flattened images (intrinsics fx fy cx cy), triangulated between pose_drone * left_extrinsic[d] and
 * pose_drone * right_extrinsic[d] (7 doubles each: x y z, qw qx qy qz), kept iff err <= triangle_thres and the point is in
 * front of the up camera.  set_drone_pose gives the pose_drone of the NEXT extract (msg.pose_drone, :394). */
osb_status osb_frontend_set_cameras(osb_frontend* h, const double* intrinsics /*[4]*/, const double* left_extrinsics /*[n_dirs][7]*/,
                                    const double* right_extrinsics /*[n_dirs][7]*/, double triangle_thres);
osb_status osb_frontend_set_drone_pose(osb_frontend* h, const double* pose_drone /*[7]*/);
/* Depth-camera keyframes (PINHOLE_DEPTH, LoopCam::generate_gray_depth_image_descriptor, loop_cam.cpp:231-302): one gray
 * image and one aligned 16-bit depth image (mm) per direction, both of the configured W x H.  extract_depth runs SuperPoint
 * and NetVLAD on the n_dirs gray images (the bottom quarter is never blanked; zero_bottom_quarter is a STEREO_FISHEYE
 * setting) and, when n_kpts > accept_min_3d_pts, lifts every keypoint through the depth look-up of osb_depth_lift with
 * pose_cam = pose_drone * extrinsics[d] (pose_drone from osb_frontend_set_drone_pose): landmarks_flag = 1 iff
 * near_thres < depth / 1000 < far_thres.  There is no stereo match: stereo_match = -1, n_kpts_down = 0.
 * set_depth_camera takes the intrinsics fx fy cx cy of the distortion-free pinhole and allocates the handle's depth buffer;
 * the extracts return OSB_ERR_INVALID until it has been called.  The stereo extract is unaffected by it. */
osb_status osb_frontend_set_depth_camera(osb_frontend* h, const double* intrinsics /*[4]*/,
                                         const double* extrinsics /*[n_dirs][7]*/, double near_thres, double far_thres);
/* images [n_dirs][H][W] uint8 and depth_mm [n_dirs][H][W] uint16, HOST (pinned or pageable) -> record_dev, no synchronisation */
osb_status osb_frontend_extract_depth(osb_frontend* h, const uint8_t* images, const uint16_t* depth_mm, int32_t msg_id,
                                      osb_keyframe_record* record_dev, void* stream);
/* same with images and depth already on the device */
osb_status osb_frontend_extract_depth_dev(osb_frontend* h, const uint8_t* images_dev, const uint16_t* depth_mm_dev,
                                          int32_t msg_id, osb_keyframe_record* record_dev, void* stream);
/* osb_frontend_process for a depth keyframe: extract_depth + ingest(own) + query, one synchronisation at the end */
osb_status osb_frontend_process_depth(osb_frontend* h, const uint8_t* images, const uint16_t* depth_mm, int32_t msg_id,
                                      osb_keyframe_record* record_host, osb_loop_result* result_host);
/* landmarks_2d [n][max_num][2] and stereo_match [n][max_num] (>= 0 <=> landmarks_flag) of rows loaded with
 * osb_frontend_db_load -- what the geometric filter reads when such a row is the loop hit */
osb_status osb_frontend_db_set_geometry(osb_frontend* h, int remote, int64_t first_row, int64_t n, const float* kpts,
                                        const int32_t* stereo_match);
/* stage timing (CUDA events on the caller's stream, recorded only while enabled).  After a synchronising call
 * (process / finish) stage_ms returns the device time of the LAST extract+ingest+query sequence:
 * [0] SuperPoint network  [1] keypoints + descriptors (NetVLAD runs concurrently on a second stream)
 * [2] NetVLAD remainder not hidden behind [1]  [3] stereo match + record pack (depth keyframes: depth lift + record pack)
 * [4] add_to_database  [5] database scans (remote + local)  [6] acceptance rule + per-direction match  [7] unused */
osb_status osb_frontend_set_profiling(osb_frontend* h, int enable);
osb_status osb_frontend_stage_ms(osb_frontend* h, float* ms8);
/* precision of both networks of the front-end (SuperPoint and NetVLAD; see osb_superpoint_set_precision) */
osb_status osb_frontend_set_precision(osb_frontend* h, int precision);
/* Row storage of both keyframe databases' global descriptors (OSB_DB_STORAGE_FP32, the default, or OSB_DB_STORAGE_FP16;
 * see osb_db).  Ingest and osb_frontend_db_load round every global-descriptor element with __float2half_rn in fp16; local
 * descriptors, keypoints, flags and landmarks_3d stay fp32, and queries read the records' fp32 descriptors.  Valid only while
 * both databases are empty (no ingest or db_load since create or osb_frontend_db_reset, even one not yet synchronised);
 * otherwise OSB_ERR_INVALID and the handle is unchanged.  The two [db_capacity][4096] row planes are freed and acquired
 * anew (fp16 holds db_capacity x 8 KB less per database).  osb_frontend_db_reset keeps the storage. */
osb_status osb_frontend_set_db_storage(osb_frontend* h, int storage);
/* Which camera of each stereo pair is the main one (the reference's LOWER_CAM_AS_MAIN, swarm_loop.cpp:243).
 * OSB_MAIN_CAMERA_UP (the default): the record as described above.  OSB_MAIN_CAMERA_DOWN (loop_cam.cpp:341-523): SuperPoint
 * runs on both images as before, NetVLAD on the DOWN images, and direction d of the record is the down image's:
 *   kpts, local_desc, n_kpts, landmarks_3d and landmarks_flag are the down image's; n_kpts_down is the UP count;
 *   stereo_match[d][j] is the up index mutually matched to down keypoint j, or -1;
 *   with set_cameras the pair is triangulated as in UP mode (in-front test on the up camera) and the point and flag land
 *   on the down keypoint; without cameras landmarks_flag = stereo_match >= 0;
 *   when the up count is <= accept_min_3d_pts (the reference returns the up descriptor, which has no global descriptor):
 *   kpts / local_desc / n_kpts are the up image's, n_kpts_down the up count too, stereo_match -1, no flags and a ZERO
 *   global_desc, so the direction still adds its database row and no query can accept it.
 * compute_loop lifts the old frame through the right extrinsics of set_cameras.  Ingest, query and query_received read only
 * the record and are unchanged.  The call allocates nothing and applies from the next extract on.  OSB_ERR_INVALID after
 * set_depth_camera; set_depth_camera and the depth extracts return OSB_ERR_INVALID on a DOWN handle. */
#define OSB_MAIN_CAMERA_UP 0
#define OSB_MAIN_CAMERA_DOWN 1
osb_status osb_frontend_set_main_camera(osb_frontend* h, int which);

/* Loop edges on the device -- LoopDetector::compute_loop + the frame-level compute_correspond_features
 *   (loop_detector.cpp:431-537, 627-836): for every hit of a query, the correspondences of its direction pairs, PnP-RANSAC
 *   (osb_pnp_ransac's kernel), pnp_result_verify and the odometry-consistency check.
 * osb_loop_params: the constants of swarm_loop.cpp:221-256.  osb_loop_candidate: what only the host knows about candidate i
 *   (the poses of the two keyframes, init_mode, and for same-drone loops the ego-motion between the two stamps).
 * Roles (:113-118, :637).  results[i].swapped == 0: new = records[i], old = the local row of the hit, main_dir_new =
 *   query_dir, main_dir_old = hit_dir.  swapped == 1: new = the remote keyframe of the hit (its 3-D landmarks come from the
 *   remote store), old = records[i], and the two main directions are exchanged.  The old frame is always this drone's own, so
 *   its 2-D landmarks are lifted through the handle's camera: the depth camera (set_depth_camera) or the left cameras
 *   (set_cameras; the right ones after osb_frontend_set_main_camera(OSB_MAIN_CAMERA_DOWN)); a handle with neither or both gets OSB_ERR_INVALID, as does one without geometric_filter (the reference
 *   builds with USE_FUNDMENTAL) or without set_loop_params.
 * Correspondences, in the slot order of osb_loop_result (the reference's dirs_new): slot j contributes geo_new / geo_old when
 *   geo_valid[j] == 1; when geo_valid[j] == 0 it contributes the 0-3 matches whose new landmark is flagged (the per-image
 *   function pushes them before it returns false, and the frame-level caller ignores the return value, :488).  The 3-D point
 *   is the new landmark's landmarks_3d; the 2-D point is the old landmark's liftProjective (fp64, rounded to float) rotated
 *   into the old main direction by rotate_pt_norm2d(pt, q_ext_old[main_dir_old]^-1 q_ext_old[dir_old]) (fp64, z clamped to
 *   +-1e-3 as :419-425, rounded to float).  A slot counts towards matched_dir_count when it contributes >= min_match_per_dir.
 * PnP: iterations 100 (1000 in init_mode), min_loop_num (init_mode_min_loop_num in init_mode), extrinsic = the old camera
 *   of main_dir_old, prior = (pose_now^-1 pose_old extrinsic)^-1 evaluated left to right without fused multiply-adds (the
 *   value oracle/loop_ref.py computes), same_drone = drone_id_a == drone_id_b.  These are exactly the osb_pnp_params a host
 *   caller of osb_pnp_ransac would pass.
 * set_loop_params: allocates the remote store's landmarks_3d plane (db_capacity x max_num x 3 floats) on its first call, and
 *   from then on ingest keeps the 3-D landmarks of remote keyframes; OSB_ERR_INVALID once the remote store holds rows.
 *   Without it nothing is allocated and ingest is unchanged.
 * compute_loop: 1 <= n <= 64 candidates; records_dev / results_dev are what osb_frontend_query (n = 1) or
 *   osb_frontend_query_received wrote, with the stores as they are now; cand is a HOST array [n]; out_dev [n] (DEVICE).  The
 *   candidates travel as kernel parameters, so there is no host synchronisation; the first call acquires the scratch for 64
 *   candidates and no later call allocates. */
#define OSB_LOOP_ACCEPTED 0
#define OSB_LOOP_NO_HIT 1                 /* accepted == 0 */
#define OSB_LOOP_NO_FRAME 2               /* the hit is a row put in with db_load (hit_msg_id == -1), or has no 3-D landmarks */
#define OSB_LOOP_FEW_LANDMARKS 3          /* new.landmark_num (sum of n_kpts) < min_loop_num (:632) */
#define OSB_LOOP_CORRESPONDENCE_FAILED 4  /* no correspondence, or matched_dir_count < min_direction_loop (:532) */
#define OSB_LOOP_TOO_FEW_COMMON 5         /* n_corr <= min_loop_num, and not (init_mode and n_corr > init_mode_min_loop_num) (:671) */
#define OSB_LOOP_PNP_FAILED 6             /* no PnP model with >= 4 inliers */
#define OSB_LOOP_NOT_VERIFIED 7           /* pnp_result_verify (:317-336) */
#define OSB_LOOP_ODOMETRY_INCONSISTENT 8  /* check_loop_odometry_consistency (:294-315) */
typedef struct {
  int32_t min_loop_num;            /* MIN_LOOP_NUM (15) */
  int32_t init_mode_min_loop_num;  /* INIT_MODE_MIN_LOOP_NUM (10) */
  int32_t min_match_per_dir;       /* MIN_MATCH_PRE_DIR (15) */
  int32_t min_direction_loop;      /* MIN_DIRECTION_LOOP (3) */
  int32_t is_4dof;
  float reproj_thresh;             /* 3, as the reference passes it (normalised units, :390-391) */
  uint32_t seed;                   /* seed of the deterministic PnP-RANSAC */
  int32_t reserved;
  double rperr_thres;              /* RPERR_THRES */
  double accept_loop_yaw_rad;      /* ACCEPT_LOOP_YAW_RAD */
  double max_loop_dis;             /* MAX_LOOP_DIS */
  double odometry_consistency_threshold;
} osb_loop_params;
typedef struct {
  int32_t init_mode;
  int32_t reserved;
  double pose_query[7];            /* pose_drone of records[i] (x y z, qw qx qy qz) */
  double pose_hit[7];              /* pose_drone of the hit keyframe (results[i].hit_msg_id) */
  double odom_rel[7];              /* same drone only: ego_motion_traj.get_relative_pose_by_ts(ts_a, ts_b) (:302) */
  double odom_edge_cov[36];        /* same drone only: odometry + edge covariance, 6x6 row-major (:303) */
} osb_loop_candidate;
typedef struct {
  int32_t status;                  /* OSB_LOOP_* */
  int32_t drone_id_a, drone_id_b;  /* a = old, b = new (:790-800) */
  int32_t msg_id_a, msg_id_b;
  int32_t main_dir_new, main_dir_old;
  int32_t matched_dir_count;
  int32_t n_corr;                  /* correspondences (new_norm_2d.size()) */
  int32_t reserved;
  osb_pnp_result pnp;              /* the PnP stage as osb_pnp_ransac writes it; zero when no PnP ran */
  double relative_pose[7];         /* DP_old_to_new as to_ros_pose(): x y z, qw qx qy qz; zero when PnP found no model */
  int32_t corr_dir_new[OSB_MAX_DIRS * OSB_MAX_KPTS];   /* index2dirindex_new (:527): direction and landmark index of */
  int32_t corr_idx_new[OSB_MAX_DIRS * OSB_MAX_KPTS];   /* correspondence k, k < n_corr */
  int32_t corr_dir_old[OSB_MAX_DIRS * OSB_MAX_KPTS];   /* index2dirindex_old (:521) */
  int32_t corr_idx_old[OSB_MAX_DIRS * OSB_MAX_KPTS];
  uint8_t inlier[OSB_MAX_DIRS * OSB_MAX_KPTS];          /* PnP inlier mask over the correspondences (0 beyond n_corr) */
} osb_loop_edge_result;
osb_status osb_frontend_set_loop_params(osb_frontend* h, const osb_loop_params* p);
osb_status osb_frontend_compute_loop(osb_frontend* h, const osb_keyframe_record* records_dev, const osb_loop_result* results_dev,
                                     int n, const osb_loop_candidate* cand /*HOST [n]*/, osb_loop_edge_result* out_dev,
                                     void* stream);
/* Loop edges -> the back-end's measurement rows on the device -- the success branch of compute_loop that builds the
 *   LoopEdge (loop_detector.cpp:787-829), for a whole round.  results_dev, edges_dev, cand and n are what the preceding
 *   osb_frontend_compute_loop received or wrote; stamps [n] (HOST) are the two keyframes' stamps of each candidate.
 * Only candidates with status == OSB_LOOP_ACCEPTED give a row, in candidate order (the reference handles a round one keyframe
 *   at a time); *count_dev = the number of rows (a deterministic in-block scan, no atomics).  Row k (out_dev[k]):
 *   id = self_id * 100000000 + loop_count, in int64 (the reference computes it in int, which overflows for self_id >= 22);
 *   type OSB_MEAS_LOOP; id_a / id_b = the edge's drone_id_a / drone_id_b (old / new); relative_pose = the edge's;
 *   stamp_a / self_pose_a the old keyframe's and stamp_b / self_pose_b the new one's, routed by results[i].swapped as
 *   compute_loop routes them (swapped == 1: old = the query record, from stamp_query_ns / pose_query);
 *   cov = diag(loop_cov_pos x3, loop_cov_ang x3), translation block first.
 * Counters, on the device: loop_count (the next id's suffix) grows by one per row; for every row
 *   inter_drone_loop_count[new][old] and [old][new] grow by one each (an intra-drone loop adds 2 to its cell, :826-827).
 *   The pair counts are kept for drone ids 0..255; a row with a drone id outside that range is emitted all the same.
 *   osb_frontend_db_reset leaves both counters as they are (the reference never resets them).
 * 0 <= n <= 64; one launch, no host synchronisation; the host arrays travel as kernel parameters.  The first call acquires
 *   the counters (8 bytes + 256 KB and an event); no later call allocates.  Calls on one handle must be ordered (one stream,
 *   or joined by the caller).
 * osb_frontend_loop_counts(): waits for the last loop_measurements call and reads loop_count and, unless pair_counts is
 *   NULL, inter_drone_loop_count [256][256] row-major ([new][old]); zeros before the first call. */
typedef struct {
  int64_t stamp_query_ns;          /* stamp of records[i] */
  int64_t stamp_hit_ns;            /* stamp of the hit keyframe (results[i].hit_msg_id) */
} osb_loop_stamps;
osb_status osb_frontend_loop_measurements(osb_frontend* h, const osb_loop_result* results_dev,
                                          const osb_loop_edge_result* edges_dev, int n,
                                          const osb_loop_candidate* cand /*HOST [n]*/, const osb_loop_stamps* stamps /*HOST [n]*/,
                                          double loop_cov_pos, double loop_cov_ang, osb_measurement* out_dev /*[n]*/,
                                          int32_t* count_dev, void* stream);
osb_status osb_frontend_loop_counts(osb_frontend* h, int64_t* loop_count, int32_t* pair_counts /*[256][256] or NULL*/);

/* Keyframe metadata on the device -- the pose_drone and timestamp every FisheyeFrameDescriptor_t carries
 *   (fisheyeframe_database, loop_detector.cpp:105-111, 150-173) and the ego-motion trajectory built from them (:27), so that
 *   a round's loop candidates are built without a host read.
 * osb_keyframe_meta travels beside osb_keyframe_record: one meta per record, same index (72 bytes).
 * ingest_meta / ingest_own_meta: exactly osb_frontend_ingest / osb_frontend_ingest_own (the same rows, routing, frame slots,
 *   host bounds and launches), and each meta goes into the frame slot its record took.  A meta whose drone_id or msg_id
 *   differs from its record's is not stored (that frame has no meta) and the call's status is OSB_ERR_INVALID.  Every own
 *   keyframe (drone_id == self_id) ingested with a stored meta appends (stamp_ns, pose_drone) to the ego-motion trajectory in
 *   ingest order; a stamp not after the last sample is not appended (status OSB_ERR_INVALID), nor is a sample beyond
 *   db_capacity samples (OSB_ERR_CAPACITY).  Frames ingested through ingest / ingest_own and rows of db_load have no meta.
 *   The first call acquires the meta tables of both stores (a meta and a flag per frame slot, db_capacity x 76 bytes each) and
 *   the trajectory (db_capacity samples x 72 bytes); osb_frontend_db_reset clears the tables and keeps the trajectory.  Null
 *   pointers give OSB_ERR_INVALID with nothing enqueued.
 * osb_frontend_meta_status(): waits for the last ingest and writes the status of the last meta ingest to *last (OSB_OK
 *   when none ran); returns the same value.
 * Trajectory: length[k] = the sequential fp64 sum of |p_k - p_(k-1)| (sqrt((dx*dx + dy*dy) + dz*dz), no fused multiply-add);
 *   a look-up takes the sample nearest to the stamp (ties to the earlier, clamped at both ends), as osb_anchor's.
 *   relative pose (ts_a, ts_b) = pose(ts_a)^-1 * pose(ts_b); its covariance = |len(ts_b) - len(ts_a)| *
 *   diag(pos_covariance_per_meter x3, yaw_covariance_per_meter x3).  Only own keyframes enter it (the reference also pushes
 *   foreign frames, DESIGN.md section 5).
 * set_candidate_params: inter_drone_init_frames and the covariances of swarm_loop.cpp:227-256. */
typedef struct {
  int32_t drone_id;
  int32_t msg_id;
  int64_t stamp_ns;
  double pose_drone[7];            /* x y z, qw qx qy qz */
} osb_keyframe_meta;
typedef struct {
  int32_t inter_drone_init_frames; /* inter_drone_init_frames (50) */
  int32_t reserved;
  double pos_covariance_per_meter; /* 0.01 */
  double yaw_covariance_per_meter; /* 0.003 */
  double loop_cov_pos;             /* 0.013 */
  double loop_cov_ang;             /* 2.5e-4 */
} osb_candidate_params;
osb_status osb_frontend_ingest_meta(osb_frontend* h, const osb_keyframe_record* records_dev, const osb_keyframe_meta* metas_dev,
                                    int n_records, int skip, void* stream);
osb_status osb_frontend_ingest_own_meta(osb_frontend* h, const osb_keyframe_record* record_dev, const osb_keyframe_meta* meta_dev,
                                        void* stream);
osb_status osb_frontend_meta_status(osb_frontend* h, osb_status* last);
osb_status osb_frontend_set_candidate_params(osb_frontend* h, const osb_candidate_params* p);
/* osb_frontend_init_modes_dev(): init_mode_out_dev[r] (bytes, DEVICE) = the init_mode of on_image_recv (loop_detector.cpp
 *   :65-72) for records r of a received round: 1 iff drone_id != self_id and inter_drone_loop_count[drone_id][self_id] <
 *   inter_drone_init_frames, read from the device's counters (osb_frontend_loop_measurements); 0 for r == skip.  Drone ids
 *   outside 0..255 count 0.  One launch, no synchronisation; 0 <= n_records <= 64; needs set_candidate_params.
 * osb_frontend_query_received_dev(): osb_frontend_query_received with init_mode a DEVICE byte array [n_records] (or NULL, all
 *   0) read by the rule kernel; the same launches and results. */
osb_status osb_frontend_init_modes_dev(osb_frontend* h, const osb_keyframe_record* records_dev, int n_records, int skip,
                                       uint8_t* init_mode_out_dev, void* stream);
osb_status osb_frontend_query_received_dev(osb_frontend* h, const osb_keyframe_record* records_dev, int n_records, int skip,
                                           const uint8_t* init_mode_dev, osb_loop_result* results_dev, void* stream);
/* osb_frontend_loop_candidates_dev(): the osb_loop_candidate and osb_loop_stamps a host caller of compute_loop /
 *   loop_measurements writes (INTEGRATION.md 2.5), built on the device for results_dev [n] of query / query_received,
 *   records_dev [n] and metas_dev [n] (DEVICE), with the stores as they are now.  One launch, one thread per candidate, no
 *   synchronisation; 0 <= n <= 64 (0 does nothing); needs set_candidate_params.  Acquires the meta tables and the loop
 *   counters when no earlier call has.
 *   Query side: metas_dev[i] (pose_query, stamp_query_ns) when its drone_id / msg_id are records[i]'s.  Hit side (accepted
 *   results): the meta of the hit's frame in the store that holds it (pose_hit, stamp_hit_ns).  A missing side is the
 *   identity pose and stamp 0.  init_mode: init_mode_dev[i] when init_mode_dev is not NULL, else the rule of
 *   osb_frontend_init_modes_dev on records[i].drone_id.  Same-drone accepted candidates (drone_id == hit_drone_id):
 *   odom_rel = the trajectory's relative pose (ts_a, ts_b) with a = the old side, b = the new side (results[i].swapped
 *   routes them as compute_loop does), odom_edge_cov = its covariance + diag(loop_cov_pos x3, loop_cov_ang x3); other
 *   candidates: odom_rel identity, odom_edge_cov zero.  Every value is computed in fp64 with each product rounded on its own
 *   (the order of tests/loop_candidates_ref.py).  reserved = 1 marks an accepted candidate whose query or hit has no meta (or
 *   a same-drone one with an empty trajectory): compute_loop_dev gives it OSB_LOOP_NO_FRAME; 0 otherwise.
 * osb_frontend_compute_loop_dev() / osb_frontend_loop_measurements_dev(): osb_frontend_compute_loop /
 *   osb_frontend_loop_measurements with the candidates (and stamps) read from DEVICE arrays [n], e.g. what
 *   loop_candidates_dev wrote; the same launches and, for unmarked candidates, the same bytes.  With them a round from
 *   query_received through osb_anchor_add_measurements_dev enqueues with no host read and can be captured into a CUDA
 *   graph. */
/* osb_frontend_receive_dev(): out_dev[r] = records_dev[r] as this drone's on_image_recv sees it after LoopNet's delivery
 *   (loop_net.cpp:20-93 sends the directions with landmark_num > 0 and of them only the landmarks with landmarks_flag > 0;
 *   :142-166, :230-262 rebuild the frame; loop_detector.cpp:36-65 gate it).  Pass out_dev, unchanged and with the metas at
 *   their indices, to every later call of the round: ingest{,_meta}, init_modes_dev, query_received{,_dev},
 *   loop_candidates_dev, compute_loop{,_dev}, loop_measurements{,_dev}.
 *   Records r == skip and records with drone_id == self_id are copied byte for byte.  A foreign record, per direction
 *   d < n_dirs: the landmarks i < n_kpts[d] with landmarks_flag[d][i] > 0, c_d of them in increasing i, move (kpts,
 *   local_desc, landmarks_3d, landmarks_flag, stereo_match) to slots 0 .. c_d-1; slots from c_d on are zero, stereo_match -1;
 *   n_kpts[d] = c_d, n_kpts_down[d] = 0 (no down image travels); global_desc[d] is kept when c_d > 0 and zero otherwise (a
 *   null image: ingest adds no row for it, and the query gate closes on it).  Directions d >= n_dirs come out as null images.
 *   The foreign record is dropped (on_image_recv's order) when (a) the local + remote store rows at this point of `stream`
 *   are 0, (b) fewer than min_direction_loop directions have c_d > 0, or (c) sum c_d < min_loop_num (set_loop_params).  A
 *   dropped record keeps drone_id, msg_id and n_dirs, so its meta still pairs with it; every other field is zero, so ingest
 *   adds no row for it and query_received gives it the gate-closed result.
 *   Gate (a) is exact for a whole round: a dropped frame adds no row, so no frame of the round changes database_size() for
 *   another.  The caller orders its own keyframe's ingest before or after the call as its callbacks order them in the
 *   reference (the own keyframe is on_image_recv'd before or after the received ones).
 *   0 <= n_records <= 64 (0 does nothing); both buffers 16-byte aligned; OSB_ERR_INVALID with nothing enqueued for a null
 *   pointer, out_dev overlapping records_dev, or a handle without set_loop_params.  One launch, no allocation, no host
 *   synchronisation: the call can be captured into a CUDA graph. */
osb_status osb_frontend_receive_dev(osb_frontend* h, const osb_keyframe_record* records_dev, int n_records, int skip,
                                    osb_keyframe_record* out_dev, void* stream);
osb_status osb_frontend_loop_candidates_dev(osb_frontend* h, const osb_keyframe_record* records_dev,
                                            const osb_keyframe_meta* metas_dev, const osb_loop_result* results_dev, int n,
                                            const uint8_t* init_mode_dev, osb_loop_candidate* cand_out_dev,
                                            osb_loop_stamps* stamps_out_dev, void* stream);
osb_status osb_frontend_compute_loop_dev(osb_frontend* h, const osb_keyframe_record* records_dev,
                                         const osb_loop_result* results_dev, int n, const osb_loop_candidate* cand_dev,
                                         osb_loop_edge_result* out_dev, void* stream);
osb_status osb_frontend_loop_measurements_dev(osb_frontend* h, const osb_loop_result* results_dev,
                                              const osb_loop_edge_result* edges_dev, int n, const osb_loop_candidate* cand_dev,
                                              const osb_loop_stamps* stamps_dev, double loop_cov_pos, double loop_cov_ang,
                                              osb_measurement* out_dev, int32_t* count_dev, void* stream);
/* ------------------------------------------------------------------------------------------------------------
 * Swarm-wide keyframe exchange -- replaces LoopNet::broadcast_fisheye_desc / image_desc_callback
 *   (swarm_loop/src/loop_net.cpp:20-120,142-172; called from swarm_loop/src/swarm_loop.cpp:167): the LCM UDP multicast of
 *   one header + one message per landmark becomes ONE ncclAllGather of the fixed-size osb_keyframe_record per keyframe
 *   round (drone = rank; NVLink on the 8-GPU box).  NCCL is opened with dlopen on first use (no link-time dependency).
 * unique_id: rank 0 creates the 128-byte communicator id and hands it to the other drones over any channel they already
 *            share (a ROS parameter, a file, the LCM channel); every rank then calls init with the same id.
 * exchange:  record_dev (this drone's record) -> gathered_dev[world] in rank order, enqueued on `stream`, no
 *            synchronisation.  osb_frontend_ingest(gathered_dev, world, ...) routes own / foreign records by drone_id.
 * exchange_async + wait: the reference's exchange is asynchronous (loop_net.cpp:142-172), so the collective may run on
 *            the handle's own stream behind an event of `stream` while the next keyframe is extracted; osb_swarm_wait
 *            makes `stream` wait for the LAST exchange_async.  One exchange in flight per handle; the caller
 *            double-buffers record_dev / gathered_dev.   world == 1: a device copy, no NCCL needed.
 *            Transport of exchange_async: when the ranks can map each other's memory (CUDA IPC, one node), every record is
 *            PUSHED into the peers' inboxes by the copy engines over NVLink and completion travels as 32-bit round stamps
 *            that the streams wait on (cuStreamWaitValue32) -- no kernel, no SM, nothing spinning while a peer is late;
 *            otherwise (or with OSB_SWARM_P2P=0) it is the ncclAllGather on the handle's stream.  Every rank must call
 *            exchange_async and wait the same number of times. */
#define OSB_SWARM_ID_BYTES 128
typedef struct osb_swarm osb_swarm;
osb_status osb_swarm_unique_id(uint8_t* id_out /*[OSB_SWARM_ID_BYTES]*/);
osb_status osb_swarm_init(osb_swarm** out, const uint8_t* id /*[OSB_SWARM_ID_BYTES], may be NULL when world == 1*/, int rank,
                          int world);
osb_status osb_swarm_destroy(osb_swarm* h);
osb_status osb_swarm_exchange(osb_swarm* h, const osb_keyframe_record* record_dev, osb_keyframe_record* gathered_dev,
                              void* stream);
osb_status osb_swarm_exchange_async(osb_swarm* h, const osb_keyframe_record* record_dev, osb_keyframe_record* gathered_dev,
                                    void* stream);
osb_status osb_swarm_wait(osb_swarm* h, void* stream);
/* exchange_meta: meta_dev (this drone's osb_keyframe_meta, the one beside its record) -> gathered_dev[world] in rank order:
 *   one ncclAllGather of world x 72 bytes on `stream` (a device copy at world == 1), no synchronisation.  Pair it with
 *   osb_swarm_exchange of the record, so that gathered metas and records share their index. */
osb_status osb_swarm_exchange_meta(osb_swarm* h, const osb_keyframe_meta* meta_dev, osb_keyframe_meta* gathered_dev,
                                   void* stream);
int osb_swarm_transport(osb_swarm* h);     /* what exchange_async uses: 1 = peer-to-peer copy engines (CUDA IPC inboxes, stream
                                              stamps; no SM, no NCCL kernel), 0 = ncclAllGather on the side stream */
int osb_swarm_rank(osb_swarm* h);
int osb_swarm_world(osb_swarm* h);

/* The convolution kernels are persistent (one CTA per SM, statically strided tiles): they run at full speed only when all of
 * their CTAs are resident.  A host that keeps another kernel on the GPU beside the front-end -- the pose-graph solve holds a
 * 16-CTA cluster for milliseconds -- caps them at n_sms (process-wide; 0 = every SM). */
void osb_set_sm_budget(int n_sms);
/* number of kernels launched by this library since it was loaded (all handles), for bench.py's gpu_launches */
int64_t osb_launch_count(void);
/* number of device buffers, pinned host buffers, streams and events the library holds right now (all handles and calls in
 * flight).  Each destroy() returns it to its value before the matching create(); osb_swarm's peer-to-peer inbox is not
 * counted. */
int64_t osb_live_resources(void);

#ifdef __cplusplus
}
#endif
#endif /* OMNISWARM_B200_H */
