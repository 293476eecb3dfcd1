// omniswarm_b200_adapters.hpp -- header-only C++ adapters that keep the reference's class signatures and forward to
// the C ABI of libomniswarm_b200.so.  A maintainer drops these in place of the TensorRT / faiss / OpenCV objects:
//
//   SuperPointTensorRT     (swarm_loop/include/swarm_loop/superpoint_tensorrt.h:20-28)   -> osb::SuperPointB200
//   MobileNetVLADTensorRT  (swarm_loop/include/swarm_loop/mobilenetvlad_tensorrt.h:10-21) -> osb::MobileNetVLADB200
//   faiss::IndexFlatIP     (swarm_loop/include/swarm_loop/loop_detector.h:27-29)          -> osb::IndexFlatIPB200
//   cv::BFMatcher          (swarm_loop/src/loop_cam.cpp:147-150, loop_detector.cpp:564)   -> osb::BFMatcherB200
//   ceres::Solve in solve_once (swarm_localization/src/swarm_localization_solver.cpp:1695-1712) -> osb::FlatPoseGraph
//   find_available_loops_detections (swarm_localization_solver.cpp:1594-1666)    -> osb_anchor_* + add_anchored_factors
//                                                                                   (or add_compacted_factors)
//   on_loop_connection -> add_new_loop_connection (loop_detector.cpp:787-829, swarm_localization_solver.cpp:558-588)
//                                                                                -> osb::hand_loops_to_anchor
//
// The cv::Mat / cv::Point2f / cv::DMatch overloads are compiled when OSB_WITH_OPENCV is defined (the reference build
// has OpenCV; this repository's container does not, so tests/cpp/adapter_smoke.cpp exercises the raw-pointer forms).
// Error style follows the reference: fatal errors print and exit(-1) (e.g. swarm_loop/src/loop_net.cpp:5-8).
#pragma once
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <utility>
#include <unordered_map>
#include <vector>

#include "omniswarm_b200.h"
#ifdef OSB_WITH_OPENCV
#include <opencv2/opencv.hpp>
#endif

namespace osb {

inline void check(osb_status s, const char* what) {
  if (s != OSB_OK) {
    std::fprintf(stderr, "[omniswarm_b200] %s failed (%d): %s\n", what, s, osb_last_error());
    std::exit(-1);
  }
}

// weights: float32 blob (see omniswarm_b200.h); pca_comp [64*256] row-major, pca_mean [256] -- the contents of the
// reference's components_.csv / mean_.csv (superpoint_tensorrt.cpp:110-111).
class SuperPointB200 {
 public:
  SuperPointB200(const std::vector<float>& weights, const std::vector<float>& pca_comp, const std::vector<float>& pca_mean,
                 int _width, int _height, float _thres = 0.015f, int _max_num = 200, bool _enable_perf = false)
      : width(_width), height(_height), max_num(_max_num), enable_perf(_enable_perf) {
    check(osb_superpoint_create(&h_, weights.data(), weights.size(), width, height, _thres, max_num, pca_comp.data(),
                                pca_mean.data(), 8), "osb_superpoint_create");
    n_.resize(8); k_.resize((size_t)8 * max_num * 2); d_.resize((size_t)8 * max_num * OSB_FEATURE_DESC_SIZE);
  }
  ~SuperPointB200() { osb_superpoint_destroy(h_); }
  SuperPointB200(const SuperPointB200&) = delete;
  SuperPointB200& operator=(const SuperPointB200&) = delete;
  // OSB_PRECISION_SPLIT_FP16 (default) or OSB_PRECISION_FP16, the precision of the reference's fp16 engines
  void set_precision(int precision) { check(osb_superpoint_set_precision(h_, precision), "osb_superpoint_set_precision"); }

  // raw form: one 8-bit grey image [height][width]; keypoints as (x,y) pairs ordered by descending confidence
  void inference(const uint8_t* image, std::vector<std::pair<float, float>>& keypoints, std::vector<float>& local_descriptors) {
    keypoints.clear(); local_descriptors.clear();                                   // superpoint_tensorrt.cpp:120-121
    check(osb_superpoint_infer(h_, image, 1, n_.data(), k_.data(), d_.data()), "osb_superpoint_infer");
    for (int i = 0; i < n_[0]; ++i) keypoints.emplace_back(k_[2 * i], k_[2 * i + 1]);
    local_descriptors.assign(d_.begin(), d_.begin() + (size_t)n_[0] * OSB_FEATURE_DESC_SIZE);
  }
#ifdef OSB_WITH_OPENCV
  void inference(const cv::Mat& input, std::vector<cv::Point2f>& keypoints, std::vector<float>& local_descriptors) {
    assert(input.rows == height && input.cols == width && "Input image must have same size with network");   // :122
    cv::Mat grey = input.isContinuous() ? input : input.clone();
    std::vector<std::pair<float, float>> k;
    inference(grey.data, k, local_descriptors);
    keypoints.clear();
    for (auto& p : k) keypoints.emplace_back(p.first, p.second);
  }
#endif
  int width, height, max_num;
  bool enable_perf;

 private:
  osb_superpoint* h_ = nullptr;
  std::vector<int32_t> n_;
  std::vector<float> k_, d_;
};

class MobileNetVLADB200 {
 public:
  MobileNetVLADB200(const std::vector<float>& weights, int _width, int _height, bool _enable_perf = false)
      : width(_width), height(_height) {
    (void)_enable_perf;
    check(osb_netvlad_create(&h_, weights.data(), weights.size(), width, height, 4), "osb_netvlad_create");
  }
  ~MobileNetVLADB200() { osb_netvlad_destroy(h_); }
  void set_precision(int precision) { check(osb_netvlad_set_precision(h_, precision), "osb_netvlad_set_precision"); }
  std::vector<float> inference(const uint8_t* image) {
    std::vector<float> out(OSB_DEEP_DESC_SIZE);
    check(osb_netvlad_infer(h_, image, 1, out.data()), "osb_netvlad_infer");
    return out;
  }
#ifdef OSB_WITH_OPENCV
  std::vector<float> inference(const cv::Mat& input) {
    cv::Mat grey = input.isContinuous() ? input : input.clone();
    return inference(grey.data);
  }
#endif
  int width, height;

 private:
  osb_netvlad* h_ = nullptr;
};

// faiss::IndexFlatIP look-alike (only the members LoopDetector uses)
class IndexFlatIPB200 {
 public:
  typedef int64_t idx_t;
  // use_float16: rows stored as fp16 (faiss GpuIndexFlatConfig::useFloat16; see OSB_DB_STORAGE_FP16)
  explicit IndexFlatIPB200(int d, int64_t capacity = 65536, bool use_float16 = false) : d(d) {
    check(osb_db_create_storage(&h_, d, capacity, use_float16 ? OSB_DB_STORAGE_FP16 : OSB_DB_STORAGE_FP32),
          "osb_db_create_storage");
  }
  ~IndexFlatIPB200() { osb_db_destroy(h_); }
  void add(idx_t n, const float* x) { check(osb_db_add(h_, n, x, nullptr), "osb_db_add"); ntotal = osb_db_size(h_); }
  void search(idx_t n, const float* x, idx_t k, float* distances, idx_t* labels) const {
    check(osb_db_search(h_, n, x, (int)k, distances, labels), "osb_db_search");
  }
  int d;
  idx_t ntotal = 0;

 private:
  osb_db* h_ = nullptr;
};

struct DMatchB200 { int queryIdx, trainIdx; float distance; };

// cv::BFMatcher(cv::NORM_L2, crossCheck = true)
class BFMatcherB200 {
 public:
  explicit BFMatcherB200(int max_n = OSB_MAX_KPTS) : max_n_(max_n) {
    check(osb_matcher_create(&h_, 1, max_n, OSB_FEATURE_DESC_SIZE), "osb_matcher_create");
    q_.resize((size_t)max_n * OSB_FEATURE_DESC_SIZE); t_.resize(q_.size());
    qi_.resize(max_n); ti_.resize(max_n); dist_.resize(max_n);
  }
  ~BFMatcherB200() { osb_matcher_destroy(h_); }
  // query [nq][64], train [nt][64] row-major
  void match(const float* query, int nq, const float* train, int nt, std::vector<DMatchB200>& matches) {
    std::copy(query, query + (size_t)nq * OSB_FEATURE_DESC_SIZE, q_.begin());
    std::copy(train, train + (size_t)nt * OSB_FEATURE_DESC_SIZE, t_.begin());
    int32_t n = 0;
    check(osb_matcher_match(h_, 1, q_.data(), &nq, t_.data(), &nt, qi_.data(), ti_.data(), dist_.data(), &n), "osb_matcher_match");
    matches.clear();
    for (int i = 0; i < n; ++i) matches.push_back({qi_[i], ti_[i], dist_[i]});
  }
#ifdef OSB_WITH_OPENCV
  void match(const cv::Mat& query, const cv::Mat& train, std::vector<cv::DMatch>& matches) {
    std::vector<DMatchB200> m;
    match(query.ptr<float>(), query.rows, train.ptr<float>(), train.rows, m);
    matches.clear();
    for (auto& x : m) matches.emplace_back(x.queryIdx, x.trainIdx, x.distance);
  }
#endif

 private:
  osb_matcher* h_ = nullptr;
  int max_n_;
  std::vector<float> q_, t_, dist_;
  std::vector<int32_t> qi_, ti_;
};

// Flat factor list that replaces ceres::Problem inside solve_once: the three setup_problem_with_* walks
// (swarm_localization_solver.cpp:1064-1214) call add_* instead of problem.AddResidualBlock, `solve` replaces
// ceres::Solve (:1712) and writes the optimised 4-vectors back through the same double* the reference uses.
class FlatPoseGraph {
 public:
  // every distinct pose block (double[4]) gets a node index; shared blocks (not-moving keyframes, :291-294) map once
  int node(double* pose) {                                          // O(1): a C5 window has 2 000 blocks, 24 000 look-ups
    auto it = index_.find(pose);
    if (it != index_.end()) return it->second;
    ptr_.push_back(pose); fixed_.push_back(0);
    index_.emplace(pose, (int)ptr_.size() - 1);
    return (int)ptr_.size() - 1;
  }
  void set_constant(double* pose) { fixed_[node(pose)] = 1; }                       // SetParameterBlockConstant (:1198)
  void add_distance(double* pa, double* pb, double d, double sqrt_inf, bool huber) { // DistanceMeasurementFactor::Create
    if (pa == pb) return;
    double pl[OSB_PAYLOAD_LEN] = {d, sqrt_inf};
    push(OSB_FACTOR_DISTANCE, pa, pb, pl, huber);
  }
  // RelativePoseFactor4d::Create: meas = relative pose (x,y,z,yaw), S = sqrt information 4x4 row-major
  void add_relative_pose(double* pa, double* pb, const double meas[4], const double S[16], bool huber) {
    if (pa == pb) return;                                                            // :1071-1073, :1176
    double pl[OSB_PAYLOAD_LEN] = {0};
    for (int i = 0; i < 4; ++i) pl[i] = meas[i];
    for (int i = 0; i < 16; ++i) pl[4 + i] = S[i];
    push(OSB_FACTOR_RELPOSE, pa, pb, pl, huber);
  }
  // DroneDetection4dFactor::Create (swarm_localization_factors.hpp:273-367; reached at swarm_localization_solver.cpp:1088-1094):
  // dir = unit bearing [3], tan_base = detect_tan_base 2x3 row-major, inv_dep and its flag, the antenna z offset OR the two
  // pre-composed dposes (x y z yaw each), DETECTION_SPHERE_STD / DETECTION_INV_DEP_STD.  Payload layout: omniswarm_b200.h.
  void add_detection(double* pa, double* pb, const double dir[3], const double tan_base[6], double inv_dep, bool enable_depth,
                     double extrinsic_z, const double* dposea /*[4] or null*/, const double* dposeb /*[4] or null*/,
                     double sphere_std, double inv_dep_std, bool huber) {
    if (pa == pb) return;
    double pl[OSB_PAYLOAD_LEN] = {0};
    for (int i = 0; i < 3; ++i) pl[i] = dir[i];
    for (int i = 0; i < 6; ++i) pl[3 + i] = tan_base[i];
    pl[9] = inv_dep;
    const bool dpose = dposea != nullptr && dposeb != nullptr;
    pl[10] = (double)((enable_depth ? 1 : 0) | (dpose ? 2 : 0));
    pl[11] = extrinsic_z;
    if (dpose) for (int i = 0; i < 4; ++i) { pl[12 + i] = dposea[i]; pl[16 + i] = dposeb[i]; }
    pl[20] = sphere_std; pl[21] = inv_dep_std;
    push(OSB_FACTOR_DETECTION, pa, pb, pl, huber);
  }
  osb_solve_summary solve(osb_solver* solver, const osb_solve_options* opt = nullptr) {
    const int n = (int)ptr_.size(), m = (int)type_.size();
    std::vector<double> poses((size_t)n * 4);
    for (int i = 0; i < n; ++i) for (int j = 0; j < 4; ++j) poses[4 * i + j] = ptr_[i][j];
    osb_solve_summary s{};
    check(osb_solver_solve(solver, n, poses.data(), fixed_.data(), m, type_.data(), ia_.data(), ib_.data(), payload_.data(),
                           huber_.data(), opt, &s), "osb_solver_solve");
    for (int i = 0; i < n; ++i) for (int j = 0; j < 4; ++j) ptr_[i][j] = poses[4 * i + j];
    return s;
  }
  // random_init_pose (solver.cpp:204-216): the caller marks every pose block of the drones in ids_to_init except
  // self_id, with the odometry yaw already in pose[3] (:212)
  void mark_for_init(double* pose) {
    const int id = node(pose);
    if (init_mask_.size() <= (size_t)id) init_mask_.resize(id + 1, 0);
    init_mask_[id] = 1;
  }
  // solve_with_multiple_init (:781-845): ms.n_trials solves from random restarts of the marked blocks, one launch.  The
  // pose blocks are written back only when a trial got below ms.acpt_cost; returns that (cost_updated, :844).
  bool solve_with_multiple_init(osb_solver* solver, const osb_multistart_options& ms, const osb_solve_options* opt = nullptr) {
    const int n = (int)ptr_.size(), m = (int)type_.size();
    std::vector<double> poses((size_t)n * 4);
    for (int i = 0; i < n; ++i) for (int j = 0; j < 4; ++j) poses[4 * i + j] = ptr_[i][j];
    init_mask_.resize(n, 0);
    std::vector<osb_solve_summary> summaries(ms.n_trials > 0 ? ms.n_trials : 1);
    std::vector<double> equv(summaries.size());
    int32_t chosen = -1;
    check(osb_solver_solve_multistart(solver, n, poses.data(), fixed_.data(), init_mask_.data(), m, type_.data(), ia_.data(),
                                      ib_.data(), payload_.data(), huber_.data(), opt, &ms, summaries.data(), equv.data(),
                                      &chosen), "osb_solver_solve_multistart");
    if (chosen < 0) return false;
    for (int i = 0; i < n; ++i) for (int j = 0; j < 4; ++j) ptr_[i][j] = poses[4 * i + j];
    cost_now = equv[chosen];
    return true;
  }
  int num_factors() const { return (int)type_.size(); }
  double cost_now = 0.0;             // equv_cost of the trial solve_with_multiple_init accepted last (:809)

 private:
  void push(int type, double* pa, double* pb, const double* pl, bool huber) {
    type_.push_back(type); ia_.push_back(node(pa)); ib_.push_back(node(pb)); huber_.push_back(huber ? 1 : 0);
    payload_.insert(payload_.end(), pl, pl + OSB_PAYLOAD_LEN);
  }
  std::vector<double*> ptr_;
  std::unordered_map<double*, int> index_;
  std::vector<uint8_t> fixed_, huber_, init_mask_;
  std::vector<int32_t> type_, ia_, ib_;
  std::vector<double> payload_;
};

// find_available_loops_detections + setup_problem_with_loops_and_detections (swarm_localization_solver.cpp:1594-1666,
// 1064-1100) on the device: the rows of osb_anchor_run with skip == 0 (and keep[i], e.g. osb_pcm_state_reject's mask over
// the same rows) become RelativePoseFactor4d blocks of `graph`; blocks[id] is the double[4] of the pose-block id the
// window entries carry.  Returns the number of factors added.
inline int add_anchored_factors(FlatPoseGraph& graph, const osb_anchor_result* rows, int n, double* const* blocks,
                                const uint8_t* keep = nullptr) {
  int added = 0;
  for (int i = 0; i < n; ++i) {
    const osb_anchor_result& r = rows[i];
    if (r.skip || (keep && !keep[i])) continue;
    graph.add_relative_pose(blocks[r.ia], blocks[r.ib], r.payload, r.payload + 4, r.huber != 0);
    ++added;
  }
  return added;
}

// LoopDetector::on_loop_connection feeding SwarmLocalizationSolver::add_new_loop_connection, on the device: the accepted
// loop edges of the compute_loop call that took (results_dev, cand, n) and wrote edges_dev become LoopEdge rows
// (osb_frontend_loop_measurements) and pass the solver's distance gate into the anchor's store
// (osb_anchor_add_measurements_dev), stream-ordered, no host copy and no synchronisation.  meas_dev [n] and count_dev
// are the caller's device scratch; the next osb_anchor_run_dev on any stream sees the rows.
inline void hand_loops_to_anchor(osb_frontend* fe, osb_anchor* anchor, const osb_loop_result* results_dev,
                                 const osb_loop_edge_result* edges_dev, int n, const osb_loop_candidate* cand,
                                 const osb_loop_stamps* stamps, double loop_cov_pos, double loop_cov_ang,
                                 float loop_outlier_distance_threshold, osb_measurement* meas_dev, int32_t* count_dev,
                                 void* stream) {
  check(osb_frontend_loop_measurements(fe, results_dev, edges_dev, n, cand, stamps, loop_cov_pos, loop_cov_ang, meas_dev,
                                       count_dev, stream), "osb_frontend_loop_measurements");
  check(osb_anchor_add_measurements_dev(anchor, meas_dev, count_dev, n, loop_outlier_distance_threshold, stream),
        "osb_anchor_add_measurements_dev");
}

// A whole received round on the device, from LoopDetector::on_image_recv to add_new_loop_connection: the init modes from the
// device's inter_drone_loop_count, query_received, the candidates from the keyframe metadata (records_dev / metas_dev [n],
// the all-gather outputs of osb_swarm_exchange and osb_swarm_exchange_meta; the keyframes ingested with
// osb_frontend_ingest_meta), compute_loop, the LoopEdge rows and the anchor's append.  Stream-ordered, no host read and no
// synchronisation, so the sequence can be captured into a CUDA graph.  The DEVICE scratch: init_dev [n], results_dev [n],
// cand_dev [n], stamps_dev [n], edges_dev [n], meas_dev [n] and count_dev.
struct RoundScratch {
  uint8_t* init_dev;
  osb_loop_result* results_dev;
  osb_loop_candidate* cand_dev;
  osb_loop_stamps* stamps_dev;
  osb_loop_edge_result* edges_dev;
  osb_measurement* meas_dev;
  int32_t* count_dev;
};
inline void hand_round_to_anchor_dev(osb_frontend* fe, osb_anchor* anchor, const osb_keyframe_record* records_dev,
                                     const osb_keyframe_meta* metas_dev, int n, int skip, const RoundScratch& s,
                                     double loop_cov_pos, double loop_cov_ang, float loop_outlier_distance_threshold,
                                     void* stream) {
  if (n == 0) return;
  check(osb_frontend_init_modes_dev(fe, records_dev, n, skip, s.init_dev, stream), "osb_frontend_init_modes_dev");
  check(osb_frontend_query_received_dev(fe, records_dev, n, skip, s.init_dev, s.results_dev, stream),
        "osb_frontend_query_received_dev");
  check(osb_frontend_loop_candidates_dev(fe, records_dev, metas_dev, s.results_dev, n, s.init_dev, s.cand_dev, s.stamps_dev,
                                         stream), "osb_frontend_loop_candidates_dev");
  check(osb_frontend_compute_loop_dev(fe, records_dev, s.results_dev, n, s.cand_dev, s.edges_dev, stream),
        "osb_frontend_compute_loop_dev");
  check(osb_frontend_loop_measurements_dev(fe, s.results_dev, s.edges_dev, n, s.cand_dev, s.stamps_dev, loop_cov_pos,
                                           loop_cov_ang, s.meas_dev, s.count_dev, stream),
        "osb_frontend_loop_measurements_dev");
  check(osb_anchor_add_measurements_dev(anchor, s.meas_dev, s.count_dev, n, loop_outlier_distance_threshold, stream),
        "osb_anchor_add_measurements_dev");
}

// The same factors from osb_anchor_compact_factors_dev's SoA after its one copy to the host: count rows of type / ia / ib /
// payload [count][OSB_PAYLOAD_LEN] / huber.  Returns the number of factors added (count).
inline int add_compacted_factors(FlatPoseGraph& graph, int count, const int32_t* ia, const int32_t* ib, const double* payload,
                                 const uint8_t* huber, double* const* blocks) {
  for (int k = 0; k < count; ++k) {
    const double* pl = payload + (size_t)k * OSB_PAYLOAD_LEN;
    graph.add_relative_pose(blocks[ia[k]], blocks[ib[k]], pl, pl + 4, huber[k] != 0);
  }
  return count;
}

// Same interface, but the window lives in the solver between solves (osb_solver_graph_*, SURVEY.md 8f-4): after a solve
// only the pose blocks and factors added since (add_new_swarm_frame / add_new_loop_connection,
// swarm_localization_solver.hpp:197-214) are sent; poses are written back to the caller's double[4] blocks.
class ResidentPoseGraph {
 public:
  explicit ResidentPoseGraph(osb_solver* solver) : solver_(solver) { check(osb_solver_graph_clear(solver_), "osb_solver_graph_clear"); }
  int node(double* pose) {
    auto it = index_.find(pose);
    if (it != index_.end()) return it->second;
    ptr_.push_back(pose);
    new_fixed_.push_back(0);
    index_.emplace(pose, (int)ptr_.size() - 1);
    return (int)ptr_.size() - 1;
  }
  void set_constant(double* pose) {
    const int id = node(pose);
    if (id >= sent_nodes_) new_fixed_[id - sent_nodes_] = 1;
    else check(osb_solver_graph_set_fixed(solver_, id, 1), "osb_solver_graph_set_fixed");
  }
  void add_distance(double* pa, double* pb, double d, double sqrt_inf, bool huber) {
    if (pa == pb) return;
    double pl[OSB_PAYLOAD_LEN] = {d, sqrt_inf};
    push(OSB_FACTOR_DISTANCE, pa, pb, pl, huber);
  }
  void add_relative_pose(double* pa, double* pb, const double meas[4], const double S[16], bool huber) {
    if (pa == pb) return;
    double pl[OSB_PAYLOAD_LEN] = {0};
    for (int i = 0; i < 4; ++i) pl[i] = meas[i];
    for (int i = 0; i < 16; ++i) pl[4 + i] = S[i];
    push(OSB_FACTOR_RELPOSE, pa, pb, pl, huber);
  }
  // DroneDetection4dFactor::Create (swarm_localization_factors.hpp:273-367; reached at swarm_localization_solver.cpp:1088-1094):
  // dir = unit bearing [3], tan_base = detect_tan_base 2x3 row-major, inv_dep and its flag, the antenna z offset OR the two
  // pre-composed dposes (x y z yaw each), DETECTION_SPHERE_STD / DETECTION_INV_DEP_STD.  Payload layout: omniswarm_b200.h.
  void add_detection(double* pa, double* pb, const double dir[3], const double tan_base[6], double inv_dep, bool enable_depth,
                     double extrinsic_z, const double* dposea /*[4] or null*/, const double* dposeb /*[4] or null*/,
                     double sphere_std, double inv_dep_std, bool huber) {
    if (pa == pb) return;
    double pl[OSB_PAYLOAD_LEN] = {0};
    for (int i = 0; i < 3; ++i) pl[i] = dir[i];
    for (int i = 0; i < 6; ++i) pl[3 + i] = tan_base[i];
    pl[9] = inv_dep;
    const bool dpose = dposea != nullptr && dposeb != nullptr;
    pl[10] = (double)((enable_depth ? 1 : 0) | (dpose ? 2 : 0));
    pl[11] = extrinsic_z;
    if (dpose) for (int i = 0; i < 4; ++i) { pl[12 + i] = dposea[i]; pl[16 + i] = dposeb[i]; }
    pl[20] = sphere_std; pl[21] = inv_dep_std;
    push(OSB_FACTOR_DETECTION, pa, pb, pl, huber);
  }
  osb_solve_summary solve(const osb_solve_options* opt = nullptr) {
    flush();
    osb_solve_summary s{};
    check(osb_solver_solve_resident(solver_, opt, &s), "osb_solver_solve_resident");
    std::vector<double> poses(4 * ptr_.size());
    check(osb_solver_graph_get_poses(solver_, 0, (int)ptr_.size(), poses.data()), "osb_solver_graph_get_poses");
    for (size_t i = 0; i < ptr_.size(); ++i) for (int j = 0; j < 4; ++j) ptr_[i][j] = poses[4 * i + j];
    return s;
  }
  // The resident window plus this solve's loop and detection rows where osb_anchor_compact_factors_dev left them (device
  // pointers, *count_dev rows whose ia / ib are this graph's node ids, i.e. the anchor window's `block` ids; see
  // osb_solver_solve_resident_dev).  Sends what was added, solves on `stream`, then waits for the solve and writes the
  // poses back to the caller's double[4] blocks.
  osb_solve_summary solve_with_device_factors(int max_tail, const int32_t* type_dev, const int32_t* ia_dev,
                                              const int32_t* ib_dev, const double* payload_dev, const uint8_t* huber_dev,
                                              const int32_t* count_dev, void* stream, const osb_solve_options* opt = nullptr) {
    flush();
    check(osb_solver_solve_resident_dev(solver_, max_tail, type_dev, ia_dev, ib_dev, payload_dev, huber_dev, count_dev, opt,
                                        stream), "osb_solver_solve_resident_dev");
    osb_solve_summary s{};
    check(osb_solver_last_summary(solver_, &s), "osb_solver_last_summary");
    std::vector<double> poses(4 * ptr_.size());
    check(osb_solver_graph_get_poses(solver_, 0, (int)ptr_.size(), poses.data()), "osb_solver_graph_get_poses");
    for (size_t i = 0; i < ptr_.size(); ++i) for (int j = 0; j < 4; ++j) ptr_[i][j] = poses[4 * i + j];
    return s;
  }
  // solve_with_multiple_init (:781-845) on the device chain: the resident window plus this solve's rows (as
  // solve_with_device_factors), ms.n_trials restarts of the blocks init_mask_dev marks (e.g. osb_anchor_init_mask_dev's
  // output after the solve's osb_anchor_observe_dev), with their yaw from init_yaw_dev (or kept, when null).  Sends what was
  // added, solves on `stream`, waits, and writes the poses back to the caller's double[4] blocks only when a trial got
  // below ms.acpt_cost; returns that (cost_updated, :844) and sets cost_now to the accepted trial's equv_cost.
  bool solve_with_multiple_init_dev(int max_tail, const int32_t* type_dev, const int32_t* ia_dev, const int32_t* ib_dev,
                                    const double* payload_dev, const uint8_t* huber_dev, const int32_t* count_dev,
                                    const uint8_t* init_mask_dev, const double* init_yaw_dev,
                                    const osb_multistart_options& ms, void* stream, const osb_solve_options* opt = nullptr) {
    flush();
    check(osb_solver_solve_multistart_resident_dev(solver_, max_tail, type_dev, ia_dev, ib_dev, payload_dev, huber_dev,
                                                   count_dev, init_mask_dev, init_yaw_dev, opt, &ms, stream),
          "osb_solver_solve_multistart_resident_dev");
    std::vector<osb_solve_summary> summaries(ms.n_trials);
    std::vector<double> equv(ms.n_trials);
    int32_t chosen = -1;
    check(osb_solver_last_multistart(solver_, summaries.data(), equv.data(), &chosen), "osb_solver_last_multistart");
    if (chosen < 0) return false;
    std::vector<double> poses(4 * ptr_.size());
    check(osb_solver_graph_get_poses(solver_, 0, (int)ptr_.size(), poses.data()), "osb_solver_graph_get_poses");
    for (size_t i = 0; i < ptr_.size(); ++i) for (int j = 0; j < 4; ++j) ptr_[i][j] = poses[4 * i + j];
    cost_now = equv[chosen];
    return true;
  }
  // The same before the swarm is initialised by motion (:786-806): one trial that starts from init_pose_by_loops
  // (:218-269) instead of random poses.  osb_anchor_init_by_loops_dev places the blocks of the last observe's to_init
  // drones on the device, from the loop map that osb_anchor_record_loops_dev keeps after each run_dev, the PCM state's
  // inlier sets (pcm: its good_loops_set) and the last applied sync's keyframe paths; then one trial with no block
  // scattered (zero_mask_dev: n_nodes zero bytes on the device).  Nothing between run_dev and this solve reads the host.
  // Sends what was added first, so the window's blocks exist in the solver; returns whether the trial was accepted.
  bool solve_with_loops_init_dev(osb_anchor* anchor, osb_pcm_state* pcm, int32_t self_id, int max_tail,
                                 const int32_t* type_dev, const int32_t* ia_dev, const int32_t* ib_dev,
                                 const double* payload_dev, const uint8_t* huber_dev, const int32_t* count_dev,
                                 const uint8_t* zero_mask_dev, osb_multistart_options ms, void* stream,
                                 const osb_solve_options* opt = nullptr) {
    flush();
    check(osb_anchor_init_by_loops_dev(anchor, pcm, solver_, self_id, stream), "osb_anchor_init_by_loops_dev");
    ms.n_trials = 1;                                 // solve_with_multiple_init's max_number = 1 (:790-792)
    return solve_with_multiple_init_dev(max_tail, type_dev, ia_dev, ib_dev, payload_dev, huber_dev, count_dev,
                                        zero_mask_dev, nullptr, ms, stream, opt);
  }
  // solve()'s data association (:893-916) after the first run -> observe -> record_loops -> reject_anchored, on the
  // device (record_loops_dev and reject_anchored follow it again, as the second estimate_observability runs them): the
  // search and
  // the renaming (osb_anchor_data_association_dev), then estimate_observability again on the renamed store, predicated
  // on the search's applied word (run_dev_if, observe_dev_if), so the launches do not depend on the outcome and the
  // branch can be captured.  rows_dev holds the first run_dev's n rows and gets the second's; returns its row count.
  static int32_t try_data_association_dev(osb_anchor* anchor, const osb_observe_params* obs_params,
                                          const uint8_t* yaw_observable, osb_anchor_result* rows_dev, void* stream) {
    check(osb_anchor_data_association_dev(anchor, obs_params->self_id, stream), "osb_anchor_data_association_dev");
    const int32_t* applied = nullptr;
    check(osb_anchor_data_association_word(anchor, &applied), "osb_anchor_data_association_word");
    int32_t n = 0;
    check(osb_anchor_run_dev_if(anchor, yaw_observable, rows_dev, &n, applied, stream), "osb_anchor_run_dev_if");
    check(osb_anchor_observe_dev_if(anchor, obs_params, rows_dev, n, applied, stream), "osb_anchor_observe_dev_if");
    return n;
  }
  double cost_now = 0.0;             // equv_cost of the trial solve_with_multiple_init_dev accepted last (:809)

 private:
  void flush() {                                     // send what was added since the last solve
    const int n_new = (int)ptr_.size() - sent_nodes_;
    if (n_new > 0) {
      std::vector<double> poses(4 * (size_t)n_new);
      for (int i = 0; i < n_new; ++i) for (int j = 0; j < 4; ++j) poses[4 * i + j] = ptr_[sent_nodes_ + i][j];
      int32_t first = -1;
      check(osb_solver_graph_add_nodes(solver_, n_new, poses.data(), new_fixed_.data(), &first), "osb_solver_graph_add_nodes");
      sent_nodes_ += n_new; new_fixed_.clear();
    }
    if (!type_.empty()) {
      check(osb_solver_graph_add_factors(solver_, (int)type_.size(), type_.data(), ia_.data(), ib_.data(), payload_.data(),
                                         huber_.data()), "osb_solver_graph_add_factors");
      type_.clear(); ia_.clear(); ib_.clear(); huber_.clear(); payload_.clear();
    }
  }
  void push(int type, double* pa, double* pb, const double* pl, bool huber) {
    type_.push_back(type); ia_.push_back(node(pa)); ib_.push_back(node(pb)); huber_.push_back(huber ? 1 : 0);
    payload_.insert(payload_.end(), pl, pl + OSB_PAYLOAD_LEN);
  }
  osb_solver* solver_;
  int sent_nodes_ = 0;
  std::vector<double*> ptr_;
  std::unordered_map<double*, int> index_;
  std::vector<uint8_t> new_fixed_, huber_;
  std::vector<int32_t> type_, ia_, ib_;
  std::vector<double> payload_;
};

}  // namespace osb
