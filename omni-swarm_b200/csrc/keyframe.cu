// keyframe.cu -- osb_frontend: the per-keyframe pipeline kept resident on the GPU.
//
//   extract  = LoopCam::on_flattened_images -> generate_stereo_image_descriptor for every direction
//              (swarm_loop/src/loop_cam.cpp:178-229, 341-523): SuperPoint on the up and down image, NetVLAD on the
//              up image (extractor_img_desc_deepnet :524-585, incl. the STEREO_FISHEYE bottom-quarter blanking
//              :535-538), stereo cross-check match up<->down (match_HFNet_local_features :141-174).  With the lower
//              camera as main (LOWER_CAM_AS_MAIN, osb_frontend_set_main_camera): NetVLAD on the down image and the
//              down image's record (:350-351, :443-444, :517-521).
//   ingest   = LoopDetector::add_to_database (swarm_loop/src/loop_detector.cpp:150-173).
//   query    = query_fisheyeframe_from_database + query_from_database (:176-287, SURVEY.md Appendix A.4) and the
//              per-direction matcher of compute_correspond_features (:431-470, :539-567).
//
// Row counters and the image-id -> (frame, direction) maps live in device memory, so a keyframe is processed with
// a single host synchronisation at the very end (the reference synchronised after every engine call,
// swarm_loop/src/tensorrt_generic.cpp:73).
#include "superpoint.cuh"
#include "pose_algebra.cuh"

namespace osb {

struct DbDev {                 // device-resident counters of a database (one for own keyframes, one for remote ones)
  int64_t ntotal;              // rows (faiss ntotal)
  int nframes;
};

// what the kernels see of one database
struct DbView {
  DbDev* dev;
  int storage;                 // OSB_DB_STORAGE_FP32 / _FP16: the element type of `rows`
  void* rows;                  // [cap][4096] float or __half
  float* ldesc;                // [cap][max_num][64]
  float* kpts;                 // [cap][max_num][2]   landmarks_2d of the row (geometric filter)
  int32_t* lflag;              // [cap][max_num]      landmarks_flag of the row (non-zero = the landmark has a 3-D point)
  int32_t* nk;                 // [cap]
  int32_t* row_frame;          // [cap]
  int32_t* row_dir;            // [cap]
  int32_t* frame_rows;         // [cap][4]
  int32_t* frame_msg;          // [cap]   msg_id of the keyframe (imgid2fisheye -> fisheyeframe_database key)
  int32_t* frame_drone;        // [cap]   drone_id of the keyframe
  float* top_scores;           // [KMAX]
  int64_t* top_ids;            // [KMAX]
  float* l3d;                  // [cap][max_num][3] landmarks_3d of the row: the remote store after osb_frontend_set_loop_params
                               // (the new side of a swapped loop edge); null otherwise
};

// both databases, passed to the kernels by value: db[0] local, db[1] remote (so db[is_remote])
struct FeStores {
  DbView db[2];
};

struct DbStore {
  DbView v{};
  int64_t cap = 0;
  int64_t upper = 0;           // host-side upper bound of ntotal (exact after every synchronising call)
  float* part_scores = nullptr;   // scan scratch
  int64_t* part_ids = nullptr;
  unsigned int* done = nullptr;
};

// the matcher's direction-pair table: per slot the query / train descriptor blocks and their counts, and for the
// geometric filter the 2-D landmarks of both sides and the landmarks_flag of the query side.  S slots: OSB_MAX_DIRS for one
// keyframe; a batch of records uses OSB_MAX_DIRS per record, slot = OSB_MAX_DIRS * record + pair.
template <int S>
struct FePairsT {
  const float* q[S];
  const float* t[S];
  int32_t nq[S], nt[S];
  const float* qk[S];
  const float* tk[S];
  const int32_t* qflag[S];
};
using FePairs = FePairsT<OSB_MAX_DIRS>;

constexpr int FE_KMAX = 32;
constexpr int FE_MAX_RECORDS = 64;     // records per ingest / received-keyframe query (one bit each in a 64-bit mask)
constexpr int FE_LOAD_ROWS = 256;      // rows per staging step of osb_frontend_db_load into an fp16 store (4 MB)
constexpr int FE_RQ_K = 5 + 1;         // SEARCH_NEAREST_NUM + max_index of a received keyframe's query (loop_detector.cpp:191-195)
using FeBatchPairs = FePairsT<OSB_MAX_DIRS * FE_MAX_RECORDS>;

// a pair table of either size as the kernels see it (device pointers to its arrays)
struct FePairView {
  const float** q;
  const float** t;
  int32_t *nq, *nt;
  const float** qk;
  const float** tk;
  const int32_t** qflag;
};
template <int S>
static FePairView fe_pair_view(FePairsT<S>* p) { return FePairView{p->q, p->t, p->nq, p->nt, p->qk, p->tk, p->qflag}; }

// blank the bottom quarter of every image (loop_cam.cpp:535-538): rows rows0 = 3H/4 .. H - 1 (H is a multiple of 8)
__global__ void fe_blank_kernel(uint8_t* __restrict__ img, int H, int W, int n_img, int rows0) {
  const int nrow = H - rows0;
  const size_t per = (size_t)nrow * W;
  const size_t total = per * n_img;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t im = i / per, off = i % per;
    img[im * (size_t)H * W + (size_t)rows0 * W + off] = 0;
  }
}

// assemble the keyframe record from the SuperPoint outputs (batch order: up[0..n_dirs), down[0..n_dirs)).
// stereo_map == null: a depth keyframe (one image per direction, no down side): stereo_match = -1, n_kpts_down = 0.
// DOWN (LOWER_CAM_AS_MAIN, loop_cam.cpp:517-521): the direction is the down image's ides_down -- its keypoints and
// descriptors, stereo_match = the up index matched to each down keypoint (the inverse of stereo_map, built here), and
// n_kpts_down = the up count.  When the up count is <= accept_min_3d_pts the reference returns the up descriptor, which has
// no global descriptor (:385-391): the direction then carries the up keypoints, stereo_match -1 and a zero global row.
template <bool DOWN>
__global__ void fe_pack_kernel(osb_keyframe_record* __restrict__ rec, int drone_id, int msg_id, int n_dirs, int max_num,
                               const int32_t* __restrict__ nk, const float* __restrict__ kpts,
                               const float* __restrict__ desc, const int32_t* __restrict__ stereo_map /*or null*/,
                               int accept_min_3d_pts, const float* __restrict__ l3d /*[n_dirs][max_num][3] or null*/,
                               const uint8_t* __restrict__ lflag /*[n_dirs][max_num] or null*/) {
  const int d = blockIdx.x;
  const int tid = threadIdx.x;
  if (d >= n_dirs) {          // unused directions: zero counts
    if (tid == 0 && d < OSB_MAX_DIRS) { rec->n_kpts[d] = 0; rec->n_kpts_down[d] = 0; }
    return;
  }
  // b: the SuperPoint image the direction's landmarks come from
  int b = d, n = nk[d];
  bool stereo = n > accept_min_3d_pts;                      // the stereo stage runs (loop_cam.cpp:385-391)
  __shared__ int32_t inv[DOWN ? OSB_MAX_KPTS : 1];
  if constexpr (DOWN) {
    const int n_up = n;
    if (stereo) { b = n_dirs + d; n = nk[b]; }
    for (int i = tid; i < OSB_MAX_KPTS; i += blockDim.x) inv[i] = -1;
    __syncthreads();
    // the cross-check pairs are one-to-one: every down index is written by at most one up keypoint
    for (int i = tid; stereo && i < n_up; i += blockDim.x) {
      const int j = stereo_map[(size_t)d * max_num + i];
      if (j >= 0 && j < n) inv[j] = i;
    }
    __syncthreads();
    if (tid == 0) { rec->n_kpts[d] = n; rec->n_kpts_down[d] = n_up; }
    if (!stereo)                                            // the early return: no NetVLAD on the up image
      for (int i = tid; i < OSB_DEEP_DESC_SIZE; i += blockDim.x) rec->global_desc[d][i] = 0.f;
  }
  if (d == 0 && tid == 0) { rec->drone_id = drone_id; rec->msg_id = msg_id; rec->n_dirs = n_dirs; rec->reserved = 0; }
  if (!DOWN && tid == 0) { rec->n_kpts[d] = n; rec->n_kpts_down[d] = stereo_map ? nk[n_dirs + d] : 0; }
  for (int i = tid; i < OSB_MAX_KPTS * OSB_FEATURE_DESC_SIZE; i += blockDim.x) {
    const int r = i / OSB_FEATURE_DESC_SIZE;
    rec->local_desc[d][r][i % OSB_FEATURE_DESC_SIZE] =
        (r < n) ? desc[((size_t)b * max_num + r) * OSB_FEATURE_DESC_SIZE + (i % OSB_FEATURE_DESC_SIZE)] : 0.f;
  }
  for (int i = tid; i < OSB_MAX_KPTS; i += blockDim.x) {
    const bool ok = i < n;
    rec->kpts[d][i][0] = ok ? kpts[((size_t)b * max_num + i) * 2] : 0.f;
    rec->kpts[d][i][1] = ok ? kpts[((size_t)b * max_num + i) * 2 + 1] : 0.f;
    // the stereo match is skipped when landmarks_2d.size() <= ACCEPT_MIN_3D_PTS (loop_cam.cpp:385-391)
    int sm;
    if constexpr (DOWN) sm = (ok && stereo) ? inv[i] : -1;
    else sm = (stereo_map && ok && stereo) ? stereo_map[(size_t)d * max_num + i] : -1;
    rec->stereo_match[d][i] = sm;
    // landmarks_flag / landmarks_3d (loop_cam.cpp:405-432; depth: :276-302): lifted on the device when the cameras are known
    const bool fl = ok && (lflag ? lflag[(size_t)d * max_num + i] != 0 : sm >= 0);
    rec->landmarks_flag[d][i] = fl ? 1 : 0;
#pragma unroll
    for (int k = 0; k < 3; ++k) rec->landmarks_3d[d][i][k] = (fl && l3d) ? l3d[((size_t)d * max_num + i) * 3 + k] : 0.f;
  }
}

// keyframe metadata (osb_frontend_ingest_meta): per store a meta and a stored-flag per frame slot, and the ego-motion
// trajectory of the own keyframes (stamps, poses, sequential lengths) with its sample count and the last call's status
struct FeMetaDev {
  int32_t traj_n;
  int32_t status;
};
struct FeMeta {
  osb_keyframe_meta* meta[2];   // [cap] per store, indexed by frame slot
  int32_t* ok[2];               // [cap] 1 = the slot's meta is stored
  int64_t* t_stamp;             // [t_cap]
  double* t_pose;               // [t_cap][7]
  double* t_len;                // [t_cap]
  int t_cap;
  FeMetaDev* dev;
};

// a product rounded on its own (__dmul_rn is never contracted into an FMA)
__device__ __forceinline__ double lc_mul(double a, double b) { return __dmul_rn(a, b); }

// the meta of the record that has just taken frame slot fs of store is_remote; own keyframes also extend the trajectory.
// Returns the status so far, the first refusal kept.
__device__ int fe_store_meta(const FeMeta& mt, int is_remote, int fs, const osb_keyframe_record* rec,
                             const osb_keyframe_meta& m, int status) {
  const bool ok = m.drone_id == rec->drone_id && m.msg_id == rec->msg_id;
  mt.ok[is_remote][fs] = ok ? 1 : 0;
  if (!ok) return status != OSB_OK ? status : OSB_ERR_INVALID;
  mt.meta[is_remote][fs] = m;
  if (is_remote) return status;
  const int n = mt.dev->traj_n;
  int refused = OSB_OK;
  if (n > 0 && m.stamp_ns <= mt.t_stamp[n - 1]) refused = OSB_ERR_INVALID;
  else if (n >= mt.t_cap) refused = OSB_ERR_CAPACITY;
  if (refused != OSB_OK) return status != OSB_OK ? status : refused;
  double len = 0.0;                                          // length[k] = length[k-1] + |p_k - p_(k-1)|, in sample order
  if (n > 0) {
    const double* q = mt.t_pose + (size_t)(n - 1) * 7;
    const double dx = m.pose_drone[0] - q[0], dy = m.pose_drone[1] - q[1], dz = m.pose_drone[2] - q[2];
    len = mt.t_len[n - 1] + sqrt((lc_mul(dx, dx) + lc_mul(dy, dy)) + lc_mul(dz, dz));
  }
  mt.t_stamp[n] = m.stamp_ns;
  for (int k = 0; k < 7; ++k) mt.t_pose[(size_t)n * 7 + k] = m.pose_drone[k];
  mt.t_len[n] = len;
  mt.dev->traj_n = n + 1;
  return status;
}

// add_to_database for a batch of records: phase 1 (one thread) assigns rows in record/direction order.  META: metas [n]
// beside the records go into the frame slots the records take (osb_frontend_ingest_meta); the plain ingest passes none.
template <bool META>
__global__ void fe_assign_kernel(const osb_keyframe_record* __restrict__ recs, int n_records, int skip, int self_id,
                                 long long cap, const __grid_constant__ FeStores dbs,
                                 int32_t* __restrict__ assign /*[n_records][4]: row | (remote<<30), or -1*/,
                                 CountRecord* __restrict__ fb, long long seq, long long charged,
                                 const osb_keyframe_meta* __restrict__ metas, FeMeta mt) {
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  int meta_status = OSB_OK;
  for (int r = 0; r < n_records; ++r) {
    for (int d = 0; d < OSB_MAX_DIRS; ++d) assign[r * OSB_MAX_DIRS + d] = -1;
    if (r == skip) continue;
    const osb_keyframe_record* rec = recs + r;
    const bool is_remote = rec->drone_id != self_id;
    const DbView& db = dbs.db[is_remote];
    DbDev cnt = *db.dev;                                             // this thread is the counters' only writer
    if (cnt.nframes >= cap) continue;
    const int fs = cnt.nframes++;
    db.frame_msg[fs] = rec->msg_id;
    db.frame_drone[fs] = rec->drone_id;
    if constexpr (META) meta_status = fe_store_meta(mt, is_remote ? 1 : 0, fs, rec, metas[r], meta_status);
    for (int d = 0; d < OSB_MAX_DIRS; ++d) {
      db.frame_rows[fs * OSB_MAX_DIRS + d] = -1;
      if (d >= rec->n_dirs || rec->n_kpts[d] <= 0) continue;         // landmark_num > 0 (loop_detector.cpp:153)
      if (cnt.ntotal >= cap) continue;
      const int row = (int)cnt.ntotal++;
      db.row_frame[row] = fs; db.row_dir[row] = d;
      db.frame_rows[fs * OSB_MAX_DIRS + d] = row;
      assign[r * OSB_MAX_DIRS + d] = row | (is_remote ? (1 << 30) : 0);
    }
    *db.dev = cnt;
  }
  if constexpr (META) mt.dev->status = meta_status;
  fb->publish(seq, dbs.db[0].dev->ntotal, dbs.db[1].dev->ntotal, 0, charged);
}

// phase 2: copy global + local descriptors of every assigned (record, direction) into its row
__global__ void fe_copy_rows_kernel(const osb_keyframe_record* __restrict__ recs, const int32_t* __restrict__ assign,
                                    int max_num, const __grid_constant__ FeStores dbs) {
  const int r = blockIdx.x / OSB_MAX_DIRS, d = blockIdx.x % OSB_MAX_DIRS;
  const int a = assign[blockIdx.x];
  if (a < 0) return;
  const DbView& db = dbs.db[(a >> 30) & 1];
  const int row = a & ((1 << 30) - 1);
  const osb_keyframe_record* rec = recs + r;
  const float4* g = reinterpret_cast<const float4*>(&rec->global_desc[d][0]);
  if (db.storage == OSB_DB_STORAGE_FP16) {
    __half2* __restrict__ gd = reinterpret_cast<__half2*>(static_cast<__half*>(db.rows) + (size_t)row * OSB_DEEP_DESC_SIZE);
    for (int i = threadIdx.x; i < OSB_DEEP_DESC_SIZE / 4; i += blockDim.x) {
      const float4 v = g[i];
      gd[2 * i] = __floats2half2_rn(v.x, v.y);
      gd[2 * i + 1] = __floats2half2_rn(v.z, v.w);
    }
  } else {
    float4* __restrict__ gd = reinterpret_cast<float4*>(static_cast<float*>(db.rows) + (size_t)row * OSB_DEEP_DESC_SIZE);
    for (int i = threadIdx.x; i < OSB_DEEP_DESC_SIZE / 4; i += blockDim.x) gd[i] = g[i];
  }
  const int n = min(rec->n_kpts[d], max_num);
  const float4* l = reinterpret_cast<const float4*>(&rec->local_desc[d][0][0]);
  float4* __restrict__ ld = reinterpret_cast<float4*>(db.ldesc + (size_t)row * max_num * OSB_FEATURE_DESC_SIZE);
  for (int i = threadIdx.x; i < n * OSB_FEATURE_DESC_SIZE / 4; i += blockDim.x) ld[i] = l[i];
  float* __restrict__ kp = db.kpts + (size_t)row * max_num * 2;
  int32_t* __restrict__ fl = db.lflag + (size_t)row * max_num;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    kp[2 * i] = rec->kpts[d][i][0]; kp[2 * i + 1] = rec->kpts[d][i][1];
    fl[i] = rec->landmarks_flag[d][i];
  }
  if (db.l3d) {
    const float* p = &rec->landmarks_3d[d][0][0];
    float* __restrict__ l3 = db.l3d + (size_t)row * max_num * 3;
    for (int i = threadIdx.x; i < n * 3; i += blockDim.x) l3[i] = p[i];
  }
  if (threadIdx.x == 0) db.nk[row] = n;
}

struct QueryParams {
  int self_id, n_dirs, query_dir, match_index_dist, nonkeyframe, k_remote, k_local, max_num;
  double inner_product_thres, init_mode_product_thres;
  int n;                                 // records (one thread each)
  unsigned long long init_mask;          // bit r: init_mode of record r
  const float* l_scores;                 // local top-k of record r at l_scores / l_ids + r * l_stride
  const int64_t* l_ids;
  int l_stride;
  int received, skip;                    // received: keyframes from other drones -- r == skip and own records stay unqueried
};

// literal query_from_database (loop_detector.cpp:199-242) on a top-k result held in device memory
__device__ int fe_search_rule(const float* scores, const int64_t* ids, int k, int64_t ntotal, int max_index,
                              double thres, int index_offset, double* distance) {
  int ret = -1;
  for (int i = 0; i < k; ++i) {
    const int64_t lab = ids[i];
    if (lab < 0) continue;
    // imgid2fisheye holds every row ever added (loop_detector.cpp:155), so the membership test always passes
    ret = (int)lab + index_offset;
    if (lab <= ntotal - max_index && (double)scores[i] > thres) {
      *distance = (double)scores[i];
      return ret;
    }
  }
  return ret;
}

// one thread per record (qp.n of them): the acceptance rule of query_from_database / query_fisheyeframe_from_database
// and the direction pairing of compute_correspond_features (loop_detector.cpp:455-465); fills record r's OSB_MAX_DIRS
// slots of the matcher's pair table.  The remote top-k (read for own keyframes only) is the remote store's.
// DEV_INIT: record r's init_mode is init_dev[r] (a device byte array, or null: all 0) instead of bit r of qp.init_mask.
template <bool DEV_INIT>
__global__ void fe_query_rule_kernel(QueryParams qp, const osb_keyframe_record* __restrict__ recs,
                                     const __grid_constant__ FeStores dbs, osb_loop_result* __restrict__ results,
                                     FePairView pairs, const uint8_t* __restrict__ init_dev) {
  const int rr = threadIdx.x;
  if (blockIdx.x != 0 || rr >= qp.n) return;
  const osb_keyframe_record* rec = recs + rr;
  osb_loop_result* res = results + rr;
  const int s0 = rr * OSB_MAX_DIRS;
  const DbView &L = dbs.db[0], &R = dbs.db[1];
  // a received batch queries the foreign records only (on_image_recv runs for them, :98-104); the skipped slot is not read
  const bool closed = qp.received && (rr == qp.skip || rec->drone_id == qp.self_id);
  const bool own = !closed && rec->drone_id == qp.self_id;
  bool init_mode;
  if constexpr (DEV_INIT) init_mode = init_dev != nullptr && init_dev[rr] != 0;
  else init_mode = (qp.init_mask >> rr) & 1ull;
  const float* l_scores = qp.l_scores + (size_t)rr * qp.l_stride;
  const int64_t* l_ids = qp.l_ids + (size_t)rr * qp.l_stride;
  const double thres = init_mode ? qp.init_mode_product_thres : qp.inner_product_thres;
  double distance = -1.0;                                   // loop_detector.cpp:263
  int id = -1;
  const int64_t db_size = L.dev->ntotal + R.dev->ntotal;
  // on_image_recv gate (loop_detector.cpp:93) and landmark_num > 0 of the queried direction (:262)
  const bool gate = !closed && (db_size > qp.match_index_dist || init_mode || !own) && rec->n_kpts[qp.query_dir] > 0;
  if (gate) {
    if (own) {                                              // :182-190
      const int r = fe_search_rule(R.top_scores, R.top_ids, qp.k_remote, R.dev->ntotal, 1, thres, OSB_REMOTE_MAGIN_NUMBER,
                                   &distance);
      if (!qp.nonkeyframe)
        id = fe_search_rule(l_scores, l_ids, 5 + qp.match_index_dist, L.dev->ntotal, qp.match_index_dist, thres, 0,
                            &distance);
      else if (r != -1) id = r;
    } else {                                                // :191-195
      id = fe_search_rule(l_scores, l_ids, 5 + 1, L.dev->ntotal, 1, thres, 0, &distance);
    }
  }
  const bool accepted = (id != -1) && (distance > -1.0);    // :265 (best_distance = -1)
  res->hit_id = id;
  res->hit_score = (float)distance;
  res->accepted = accepted ? 1 : 0;
  res->hit_dir = -1;
  res->swapped = 0;
  res->hit_msg_id = -1;
  res->hit_drone_id = -1;
  for (int j = 0; j < OSB_MAX_DIRS; ++j) {
    pairs.nq[s0 + j] = 0; pairs.nt[s0 + j] = 0; pairs.q[s0 + j] = nullptr; pairs.t[s0 + j] = nullptr;
    pairs.qk[s0 + j] = nullptr; pairs.tk[s0 + j] = nullptr; pairs.qflag[s0 + j] = nullptr;
    res->dir_new[j] = -1; res->dir_old[j] = -1;
  }
  if (!accepted) return;
  const bool hit_remote = id >= OSB_REMOTE_MAGIN_NUMBER;
  const int row = hit_remote ? id - OSB_REMOTE_MAGIN_NUMBER : id;
  const DbView& db = dbs.db[hit_remote];
  const int fs = db.row_frame[row];
  const int direction_old = db.row_dir[row];                // imgid2dir (:275)
  res->hit_dir = direction_old;
  // imgid2fisheye[best_image_id] -> the keyframe's msg_id, fisheyeframe_database[msg_id].drone_id (loop_detector.cpp:272-275):
  // what the host adapter needs to find the old FisheyeFrameDescriptor_t for compute_loop
  res->hit_msg_id = db.frame_msg[fs];
  res->hit_drone_id = db.frame_drone[fs];
  // compute_loop(new, old) -- or (old, new) when the hit comes from the remote database and the keyframe is ours
  // (loop_detector.cpp:113-118): the first argument plays "new_frame_desc" (the matcher's query side).
  const bool swapped = hit_remote && own;
  res->swapped = swapped ? 1 : 0;
  const int main_new = swapped ? direction_old : qp.query_dir;
  const int main_old = swapped ? qp.query_dir : direction_old;
  int slot = 0;
  for (int _dn = main_new; _dn < main_new + OSB_MAX_DIRS; ++_dn) {     // :455-465
    const int dir_new = _dn % OSB_MAX_DIRS;
    const int dir_old = ((main_old - main_new + OSB_MAX_DIRS) % OSB_MAX_DIRS + _dn) % OSB_MAX_DIRS;
    // "new" side / "old" side descriptor blocks
    const int dir_rec = swapped ? dir_old : dir_new;          // direction taken from the current keyframe record
    const int dir_db = swapped ? dir_new : dir_old;           // direction taken from the database frame
    if (dir_rec >= rec->n_dirs) continue;
    const int row_db = db.frame_rows[fs * OSB_MAX_DIRS + dir_db];
    const int n_rec = rec->n_kpts[dir_rec];
    const int n_db = row_db >= 0 ? db.nk[row_db] : 0;
    if (n_rec <= 0 || n_db <= 0) continue;                    // both landmark_num > 0 (:461)
    const float* p_rec = &rec->local_desc[dir_rec][0][0];
    const float* p_db = db.ldesc + (size_t)row_db * qp.max_num * OSB_FEATURE_DESC_SIZE;
    res->dir_new[slot] = dir_new; res->dir_old[slot] = dir_old;
    const int ps = s0 + slot;
    if (swapped) { pairs.q[ps] = p_db; pairs.nq[ps] = n_db; pairs.t[ps] = p_rec; pairs.nt[ps] = n_rec; }
    else { pairs.q[ps] = p_rec; pairs.nq[ps] = n_rec; pairs.t[ps] = p_db; pairs.nt[ps] = n_db; }
    {   // 2-D landmarks and 3-D flags of the two sides, for the geometric filter (loop_detector.cpp:569-598)
      const float* k_rec = &rec->kpts[dir_rec][0][0];
      const int32_t* f_rec = &rec->landmarks_flag[dir_rec][0];
      const float* k_db = db.kpts + (size_t)row_db * qp.max_num * 2;
      const int32_t* f_db = db.lflag + (size_t)row_db * qp.max_num;
      pairs.qk[ps] = swapped ? k_db : k_rec; pairs.tk[ps] = swapped ? k_rec : k_db;
      pairs.qflag[ps] = swapped ? f_db : f_rec;
    }
    ++slot;
  }
}

// ordered compaction in a block of 256 threads by ballot prefix: the position of this thread's element among the kept ones
// (meaningful when keep), and in *total how many the block keeps
__device__ __forceinline__ int fe_block_compact(bool keep, int* total) {
  __shared__ int warp_cnt[8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned bal = __ballot_sync(0xffffffffu, keep);
  if (lane == 0) warp_cnt[warp] = __popc(bal);
  __syncthreads();
  int base = 0, sum = 0;
  for (int w = 0; w < 8; ++w) { if (w < warp) base += warp_cnt[w]; sum += warp_cnt[w]; }
  *total = sum;
  return base + __popc(bal & ((1u << lane) - 1u));
}

// geometric filter, step 1 (loop_detector.cpp:569-586): keep, in match order, the matches whose NEW (query-side) landmark
// has a 3-D flag; gather old_2d / new_2d of the kept matches.  One CTA per direction-pair slot; slot = OSB_MAX_DIRS * r + j
// is pair j of results[r].
__global__ void __launch_bounds__(256)
fe_geo_gather_kernel(const osb_loop_result* __restrict__ results, FePairView pairs,
                     float2* __restrict__ src, float2* __restrict__ dst, int32_t* __restrict__ kept,
                     int32_t* __restrict__ n_kept) {
  const int slot = blockIdx.x, tid = threadIdx.x;
  const osb_loop_result* res = results + slot / OSB_MAX_DIRS;
  const int j = slot % OSB_MAX_DIRS;
  const int n = (res->dir_new[j] >= 0) ? res->n_matches[j] : 0;
  bool keep = false;
  int qi = 0, ti = 0;
  if (tid < n) {
    qi = res->match_new[j][tid]; ti = res->match_old[j][tid];
    keep = pairs.qflag[slot][qi] != 0;
  }
  int total;
  const int pos = fe_block_compact(keep, &total);
  if (keep) {
    const float* tk = pairs.tk[slot];
    const float* qk = pairs.qk[slot];
    src[slot * OSB_MAX_KPTS + pos] = make_float2(tk[2 * ti], tk[2 * ti + 1]);      // old_2d
    dst[slot * OSB_MAX_KPTS + pos] = make_float2(qk[2 * qi], qk[2 * qi + 1]);      // new_2d
    kept[slot * OSB_MAX_KPTS + pos] = tid;
  }
  if (tid == 0) n_kept[slot] = total;
}

// step 3 (:590-597): reduceVector by the RANSAC mask (slots as in step 1)
__global__ void __launch_bounds__(256)
fe_geo_apply_kernel(osb_loop_result* __restrict__ results, const int32_t* __restrict__ kept,
                    const int32_t* __restrict__ n_kept, const uint8_t* __restrict__ mask) {
  const int slot = blockIdx.x, tid = threadIdx.x;
  osb_loop_result* res = results + slot / OSB_MAX_DIRS;
  const int j = slot % OSB_MAX_DIRS;
  const int n = n_kept[slot];
  const bool valid = n >= 4;                                  // else the reference returns false (:598-600)
  const bool keep = valid && tid < n && mask[slot * OSB_MAX_KPTS + tid] != 0;
  int total;
  const int pos = fe_block_compact(keep, &total);
  if (keep) {
    const int m = kept[slot * OSB_MAX_KPTS + tid];
    res->geo_new[j][pos] = res->match_new[j][m];
    res->geo_old[j][pos] = res->match_old[j][m];
  }
  if (tid == 0) { res->n_geo[j] = total; res->geo_valid[j] = (res->dir_new[j] >= 0 && valid) ? 1 : 0; }
}

// what the rule, the matcher and the geometric filter of a query write besides the results: the pair table and, per
// direction-pair slot, the match distances and the filter's point lists, counts, masks and RANSAC keys
struct FeMatchScratch {
  FePairView pairs;
  float* dist = nullptr;         // [slots][max_num][max_num] distance matrices
  float* dout = nullptr;         // match distances, addressed like the results' match lists
  float *g_src = nullptr, *g_dst = nullptr;   // [slots][OSB_MAX_KPTS] float2
  int32_t *g_kept = nullptr, *g_nkept = nullptr, *g_ninl = nullptr, *g_win = nullptr;
  uint8_t* g_mask = nullptr;
  unsigned int* g_keys = nullptr;             // 2 * slots, zero between launches
};

// ---- loop edges: LoopDetector::compute_loop + the frame-level compute_correspond_features (loop_detector.cpp:431-537,
// 627-836), one CTA per candidate: assemble (gates, correspondences, PnP inputs) -> pnp_ransac_kernel -> finalise --------
constexpr int LC_MAX = FE_MAX_RECORDS;                    // candidates per call
constexpr int LC_MAXN = OSB_MAX_DIRS * OSB_MAX_KPTS;      // correspondences per candidate (:455-530: four pairs of <= 200)
constexpr int LC_PENDING = -1;                            // status between assemble and finalise: the PnP stage decides
static_assert(LC_MAXN <= PNP_MAXN, "a frame's correspondences must fit the PnP kernel");

struct LoopCams {              // the old (own) frame's camera: pinhole fx fy cx cy and the extrinsics of every direction
  double K[4];
  double ext[OSB_MAX_DIRS][7];
};
struct LoopCandBatch {         // the host's candidates, passed as kernel parameters (sm_90 takes up to 32 KB of them)
  osb_loop_candidate c[LC_MAX];
};
struct LoopCandPtr {           // candidates in device memory (osb_frontend_compute_loop_dev)
  const osb_loop_candidate* c;
};
__device__ __forceinline__ const osb_loop_candidate& lc_cand(const LoopCandBatch& b, int i) { return b.c[i]; }
__device__ __forceinline__ const osb_loop_candidate& lc_cand(const LoopCandPtr& b, int i) { return b.c[i]; }

// Swarm::Pose algebra in the evaluation order of oracle/pcm_ref.py with every product rounded on its own (__dmul_rn is never
// contracted into an FMA): the PnP prior and the rotated points are then the bits a numpy host caller computes
__device__ __forceinline__ void lc_cross(const double* a, const double* b, double* o) {
  o[0] = lc_mul(a[1], b[2]) - lc_mul(a[2], b[1]);
  o[1] = lc_mul(a[2], b[0]) - lc_mul(a[0], b[2]);
  o[2] = lc_mul(a[0], b[1]) - lc_mul(a[1], b[0]);
}
__device__ __forceinline__ void lc_q_rot(const double* q, const double* v, double* o) {    // v + 2 (w (u x v) + u x (u x v))
  double c[3], d[3];
  lc_cross(q + 1, v, c);
  lc_cross(q + 1, c, d);
  for (int k = 0; k < 3; ++k) o[k] = v[k] + lc_mul(2.0, lc_mul(q[0], c[k]) + d[k]);
}
__device__ __forceinline__ void lc_q_mul(const double* a, const double* b, double* o) {
  o[0] = lc_mul(a[0], b[0]) - lc_mul(a[1], b[1]) - lc_mul(a[2], b[2]) - lc_mul(a[3], b[3]);
  o[1] = lc_mul(a[0], b[1]) + lc_mul(a[1], b[0]) + lc_mul(a[2], b[3]) - lc_mul(a[3], b[2]);
  o[2] = lc_mul(a[0], b[2]) - lc_mul(a[1], b[3]) + lc_mul(a[2], b[0]) + lc_mul(a[3], b[1]);
  o[3] = lc_mul(a[0], b[3]) + lc_mul(a[1], b[2]) - lc_mul(a[2], b[1]) + lc_mul(a[3], b[0]);
}
__device__ __forceinline__ void lc_pose_mul(const double* a, const double* b, double* o) {     // poses x y z, qw qx qy qz
  double r[3];
  lc_q_rot(a + 3, b, r);
  for (int k = 0; k < 3; ++k) o[k] = a[k] + r[k];
  lc_q_mul(a + 3, b + 3, o + 3);
}
__device__ __forceinline__ void lc_pose_inv(const double* a, double* o) {
  const double qc[4] = {a[3], -a[4], -a[5], -a[6]};
  double r[3];
  lc_q_rot(qc, a, r);
  for (int k = 0; k < 3; ++k) o[k] = -r[k];
  for (int k = 0; k < 4; ++k) o[3 + k] = qc[k];
}
// liftProjective of the distortion-free pinhole in fp64, rounded to float (toCV), then rotate_pt_norm2d (:415-428) in fp64
// from that float, z clamped to +-1e-3, rounded to float
__device__ __forceinline__ float2 lc_lift_rotate(float kx, float ky, const double (&K)[4], const double (&dq)[4]) {
  const float u = (float)(((double)kx - K[2]) / K[0]), v = (float)(((double)ky - K[3]) / K[1]);
  const double p[3] = {(double)u, (double)v, 1.0};
  double r[3];
  lc_q_rot(dq, p, r);
  double z = r[2];
  if (z < 1e-3 && z > 0) z = 1e-3;
  if (z > -1e-3 && z < 0) z = -1e-3;
  return make_float2((float)(r[0] / z), (float)(r[1] / z));
}

// Cands: LoopCandBatch (the host's array as parameters) or LoopCandPtr (a device array, whose reserved != 0 marks a
// candidate without keyframe metadata: OSB_LOOP_NO_FRAME)
template <class Cands>
__global__ void __launch_bounds__(256)
lc_assemble_kernel(const osb_keyframe_record* __restrict__ recs, const osb_loop_result* __restrict__ results,
                   const __grid_constant__ FeStores dbs, const __grid_constant__ Cands cands,
                   const __grid_constant__ LoopCams cam, const osb_loop_params lp, int query_dir, int max_num,
                   osb_loop_edge_result* __restrict__ out, float* __restrict__ pts3d, float* __restrict__ pts2d,
                   int32_t* __restrict__ n_pts, osb_pnp_params* __restrict__ params) {
  const int c = blockIdx.x, tid = threadIdx.x;
  const osb_keyframe_record* rec = recs + c;
  const osb_loop_result* res = results + c;
  const osb_loop_candidate& cd = lc_cand(cands, c);
  osb_loop_edge_result* o = out + c;
  const DbView &L = dbs.db[0], &R = dbs.db[1];
  // roles (:113-118): swapped -> the remote hit is "new", this drone's record "old"; the old frame is always our own (:637)
  const bool swapped = res->swapped != 0, init_mode = cd.init_mode != 0;
  const int main_new = swapped ? res->hit_dir : query_dir, main_old = swapped ? query_dir : res->hit_dir;
  int status = LC_PENDING, fs = -1;
  if (!res->accepted) {
    status = OSB_LOOP_NO_HIT;
  } else {
    const bool hit_remote = res->hit_id >= OSB_REMOTE_MAGIN_NUMBER;
    const DbView& hdb = dbs.db[hit_remote];
    fs = hdb.row_frame[hit_remote ? res->hit_id - OSB_REMOTE_MAGIN_NUMBER : res->hit_id];
    // a row put in with db_load has no keyframe behind it; the new side of a swapped edge needs the remote 3-D plane
    if (res->hit_msg_id == -1 || (swapped && R.l3d == nullptr) || hit_remote != swapped) status = OSB_LOOP_NO_FRAME;
    if constexpr (std::is_same<Cands, LoopCandPtr>::value)
      if (cd.reserved != 0) status = OSB_LOOP_NO_FRAME;
  }
  if (status == LC_PENDING) {                               // new_frame_desc.landmark_num < MIN_LOOP_NUM (:632)
    int lm = 0;
    for (int d = 0; d < OSB_MAX_DIRS; ++d) {
      if (swapped) { const int row = R.frame_rows[fs * OSB_MAX_DIRS + d]; lm += row >= 0 ? R.nk[row] : 0; }
      else lm += d < rec->n_dirs ? rec->n_kpts[d] : 0;
    }
    if (lm < lp.min_loop_num) status = OSB_LOOP_FEW_LANDMARKS;
  }
  // correspondences, direction pair by direction pair in slot order (:477-530); the status is uniform over the block
  int total = 0, matched_dirs = 0;
  if (status == LC_PENDING) {
    for (int j = 0; j < OSB_MAX_DIRS; ++j) {
      const int dn = res->dir_new[j], dold = res->dir_old[j];
      if (dn < 0) continue;
      const int32_t* fl_new;                                // new side: landmarks_flag and landmarks_3d
      const float* p3_new;
      const float* k_old;                                   // old side: landmarks_2d
      if (swapped) {
        const int rn = R.frame_rows[fs * OSB_MAX_DIRS + dn];
        fl_new = R.lflag + (size_t)rn * max_num;
        p3_new = R.l3d + (size_t)rn * max_num * 3;
        k_old = &rec->kpts[dold][0][0];
      } else {
        fl_new = &rec->landmarks_flag[dn][0];
        p3_new = &rec->landmarks_3d[dn][0][0];
        k_old = L.kpts + (size_t)L.frame_rows[fs * OSB_MAX_DIRS + dold] * max_num * 2;
      }
      // geo_valid: the filtered lists.  Otherwise the 0-3 flagged matches the per-image function pushed before its
      // `return false` (:574-587, :598-600), which the frame-level caller appends all the same (:488)
      const bool geo = res->geo_valid[j] != 0;
      const int n = geo ? res->n_geo[j] : res->n_matches[j];
      bool keep = false;
      int qi = 0, ti = 0;
      if (tid < n) {
        qi = geo ? res->geo_new[j][tid] : res->match_new[j][tid];
        ti = geo ? res->geo_old[j][tid] : res->match_old[j][tid];
        keep = geo || fl_new[qi] != 0;
      }
      int cnt;
      const int pos = total + fe_block_compact(keep, &cnt);
      if (keep) {
        o->corr_dir_new[pos] = dn; o->corr_idx_new[pos] = qi;        // index2dirindex_new / _old (:521, :527)
        o->corr_dir_old[pos] = dold; o->corr_idx_old[pos] = ti;
        float* X = pts3d + ((size_t)c * LC_MAXN + pos) * 3;
        X[0] = p3_new[qi * 3]; X[1] = p3_new[qi * 3 + 1]; X[2] = p3_new[qi * 3 + 2];
        const double* qm = cam.ext[main_old] + 3;           // dq_old = main_quat_old^-1 * extrinsic_old[dir_old].att (:516)
        const double qmi[4] = {qm[0], -qm[1], -qm[2], -qm[3]};
        double dq[4];
        lc_q_mul(qmi, cam.ext[dold] + 3, dq);
        reinterpret_cast<float2*>(pts2d)[(size_t)c * LC_MAXN + pos] = lc_lift_rotate(k_old[2 * ti], k_old[2 * ti + 1], cam.K, dq);
      }
      total += cnt;
      matched_dirs += cnt >= lp.min_match_per_dir ? 1 : 0;  // _new_3d.size() >= MIN_MATCH_PRE_DIR (:503)
      __syncthreads();                                      // fe_block_compact's warp counts are reused by the next slot
    }
    if (!(total > 0 && matched_dirs >= lp.min_direction_loop)) status = OSB_LOOP_CORRESPONDENCE_FAILED;       // :532
    else if (!(total > lp.min_loop_num || (init_mode && total > lp.init_mode_min_loop_num))) status = OSB_LOOP_TOO_FEW_COMMON;
  }
  if (tid != 0) return;
  o->status = status;
  o->drone_id_a = swapped ? rec->drone_id : res->hit_drone_id;  o->drone_id_b = swapped ? res->hit_drone_id : rec->drone_id;
  o->msg_id_a = swapped ? rec->msg_id : res->hit_msg_id;        o->msg_id_b = swapped ? res->hit_msg_id : rec->msg_id;
  o->main_dir_new = main_new; o->main_dir_old = main_old;
  o->matched_dir_count = matched_dirs; o->n_corr = total; o->reserved = 0;
  // compute_relative_pose's inputs (:672-684, :376-391), exactly the osb_pnp_params of a host caller of osb_pnp_ransac
  const bool run = status == LC_PENDING;
  n_pts[c] = run ? total : 0;
  osb_pnp_params p;
  memset(&p, 0, sizeof(p));
  p.iterations = init_mode ? 1000 : 100;
  p.reproj_thresh = lp.reproj_thresh; p.seed = lp.seed; p.is_4dof = lp.is_4dof;
  p.min_loop_num = init_mode ? lp.init_mode_min_loop_num : lp.min_loop_num;
  p.same_drone = o->drone_id_a == o->drone_id_b ? 1 : 0;
  p.rperr_thres = lp.rperr_thres; p.accept_loop_yaw_rad = lp.accept_loop_yaw_rad; p.max_loop_dis = lp.max_loop_dis;
  p.odometry_consistency_threshold = lp.odometry_consistency_threshold;
  p.prior[3] = p.extrinsic[3] = p.drone_pose_now[3] = p.drone_pose_old[3] = 1.0;
  if (run) {
    const double* now = swapped ? cd.pose_hit : cd.pose_query;
    const double* old = swapped ? cd.pose_query : cd.pose_hit;
    for (int k = 0; k < 7; ++k) { p.extrinsic[k] = cam.ext[main_old][k]; p.drone_pose_now[k] = now[k]; p.drone_pose_old[k] = old[k]; }
    double a[7], b[7], e[7];                                // prior = (now^-1 old extrinsic)^-1, left to right
    lc_pose_inv(now, a);
    lc_pose_mul(a, old, b);
    lc_pose_mul(b, p.extrinsic, e);
    lc_pose_inv(e, p.prior);
    for (int k = 0; k < 7; ++k) p.odom_rel[k] = cd.odom_rel[k];
    for (int k = 0; k < 36; ++k) p.odom_edge_cov[k] = cd.odom_edge_cov[k];
  }
  params[c] = p;
}

// after the PnP stage: the status of the candidates that reached it, the PnP result, DP_old_to_new as a 7-pose, and the
// inlier mask in correspondence order
__global__ void __launch_bounds__(256)
lc_finalise_kernel(const uint8_t* __restrict__ mask, const osb_pnp_result* __restrict__ pnp,
                   const osb_pnp_params* __restrict__ params, osb_loop_edge_result* __restrict__ out) {
  const int c = blockIdx.x, tid = threadIdx.x;
  osb_loop_edge_result* o = out + c;
  const bool ran = o->status == LC_PENDING;
  for (int i = tid; i < LC_MAXN; i += blockDim.x) o->inlier[i] = ran ? mask[(size_t)c * LC_MAXN + i] : 0;
  __syncthreads();                                          // every thread has read the status before thread 0 rewrites it
  if (tid != 0) return;
  const osb_pnp_result r = pnp[c];
  for (int k = 0; k < 7; ++k) o->relative_pose[k] = 0.0;
  if (!ran) { memset(&o->pnp, 0, sizeof(o->pnp)); return; }
  o->pnp = r;
  o->status = !r.pnp_success ? OSB_LOOP_PNP_FAILED : !r.verified ? OSB_LOOP_NOT_VERIFIED
              : !r.odometry_consistent ? OSB_LOOP_ODOMETRY_INCONSISTENT : OSB_LOOP_ACCEPTED;
  if (!r.pnp_success) return;
  // DeltaPose(p_drone_old_in_new, drone_pose_now, is_4dof) (:393-400) as a pose; its x y z and yaw are r.dp_old_to_new
  const osb_pnp_params& prm = params[c];
  const PoseD P = load_pose(r.pose_cam);
  const PoseD old_in_new = pose_mul(pose_inv(P), pose_inv(load_pose(prm.extrinsic)));
  const PoseD now = load_pose(prm.drone_pose_now);
  PoseD dp;
  if (prm.is_4dof) {
    double ea[3], eb[3];
    quat2eulers(old_in_new.q, ea); quat2eulers(now.q, eb);
    const double cs = cos(ea[2]), sn = sin(ea[2]);
    const double dx = now.t[0] - old_in_new.t[0], dy = now.t[1] - old_in_new.t[1];
    dp.t[0] = cs * dx + sn * dy; dp.t[1] = -sn * dx + cs * dy; dp.t[2] = now.t[2] - old_in_new.t[2];
    double a = eb[2] - ea[2];
    a = a - 2.0 * M_PI * floor((a + M_PI) / (2.0 * M_PI));
    const double rv[3] = {0.0, 0.0, a};
    quat_from_rotvec(rv, dp.q);
  } else {
    dp = pose_mul(pose_inv(old_in_new), now);
  }
  for (int k = 0; k < 3; ++k) o->relative_pose[k] = dp.t[k];
  for (int k = 0; k < 4; ++k) o->relative_pose[3 + k] = dp.q[k];
}

// ---- loop edges -> the back-end's measurement rows: the success branch of compute_loop (loop_detector.cpp:787-829) for a
// whole round, candidate c on thread c of one 256-thread CTA ------------------------------------------------------------
constexpr long long LM_MAX_LOOP_ID = 100000000ll;        // MAX_LOOP_ID (loop_detector.cpp:9)
constexpr int LM_PAIR_DRONES = 256;                      // inter_drone_loop_count is kept for drone ids 0..255

struct LoopMeasBatch {         // the host's poses and stamps of the candidates, passed as kernel parameters (8 KB)
  double pose_query[LC_MAX][7];
  double pose_hit[LC_MAX][7];
  int64_t stamp_query[LC_MAX];
  int64_t stamp_hit[LC_MAX];
};
struct LoopMeasPtr {           // the same read from device arrays (osb_frontend_loop_measurements_dev)
  const osb_loop_candidate* cand;
  const osb_loop_stamps* stamps;
};
__device__ __forceinline__ const double* lm_pose_query(const LoopMeasBatch& b, int c) { return b.pose_query[c]; }
__device__ __forceinline__ const double* lm_pose_hit(const LoopMeasBatch& b, int c) { return b.pose_hit[c]; }
__device__ __forceinline__ int64_t lm_stamp_query(const LoopMeasBatch& b, int c) { return b.stamp_query[c]; }
__device__ __forceinline__ int64_t lm_stamp_hit(const LoopMeasBatch& b, int c) { return b.stamp_hit[c]; }
__device__ __forceinline__ const double* lm_pose_query(const LoopMeasPtr& b, int c) { return b.cand[c].pose_query; }
__device__ __forceinline__ const double* lm_pose_hit(const LoopMeasPtr& b, int c) { return b.cand[c].pose_hit; }
__device__ __forceinline__ int64_t lm_stamp_query(const LoopMeasPtr& b, int c) { return b.stamps[c].stamp_query_ns; }
__device__ __forceinline__ int64_t lm_stamp_hit(const LoopMeasPtr& b, int c) { return b.stamps[c].stamp_hit_ns; }

template <class Meas>
__global__ void __launch_bounds__(256)
lm_emit_kernel(const osb_loop_result* __restrict__ results, const osb_loop_edge_result* __restrict__ edges, int n,
               const __grid_constant__ Meas b, int self_id, double cov_pos, double cov_ang,
               osb_measurement* __restrict__ out, int32_t* __restrict__ count, long long* __restrict__ loop_count,
               int32_t* __restrict__ pair_counts) {
  const int c = threadIdx.x;
  const long long first = *loop_count;                     // read by every thread before fe_block_compact's barrier
  const bool keep = c < n && edges[c].status == OSB_LOOP_ACCEPTED;
  int total;
  const int pos = fe_block_compact(keep, &total);          // candidate order = the reference's one-keyframe-at-a-time order
  if (c == 0) { *count = total; *loop_count = first + total; }
  if (!keep) return;
  const osb_loop_edge_result& e = edges[c];
  const bool swapped = results[c].swapped != 0;            // compute_loop's roles: swapped -> old = the query record
  osb_measurement& m = out[pos];
  m.id = (long long)self_id * LM_MAX_LOOP_ID + first + pos;   // :811, in int64 (DESIGN §5)
  m.type = OSB_MEAS_LOOP;
  m.id_a = e.drone_id_a;
  m.id_b = e.drone_id_b;
  m.reserved = 0;
  m.stamp_a = swapped ? lm_stamp_query(b, c) : lm_stamp_hit(b, c);
  m.stamp_b = swapped ? lm_stamp_hit(b, c) : lm_stamp_query(b, c);
  const double* pa = swapped ? lm_pose_query(b, c) : lm_pose_hit(b, c);
  const double* pb = swapped ? lm_pose_hit(b, c) : lm_pose_query(b, c);
  for (int k = 0; k < 7; ++k) { m.relative_pose[k] = e.relative_pose[k]; m.self_pose_a[k] = pa[k]; m.self_pose_b[k] = pb[k]; }
  for (int k = 0; k < 36; ++k) m.cov[k] = (k % 7 == 0) ? (k < 21 ? cov_pos : cov_ang) : 0.0;     // pos_cov / ang_cov (:800-808)
  const int a = e.drone_id_a, nw = e.drone_id_b;           // :824-827: an intra-drone loop adds 2 to its one cell
  if (a >= 0 && a < LM_PAIR_DRONES && nw >= 0 && nw < LM_PAIR_DRONES) {
    atomicAdd(&pair_counts[nw * LM_PAIR_DRONES + a], 1);
    atomicAdd(&pair_counts[a * LM_PAIR_DRONES + nw], 1);
  }
}

// ---- a round's loop candidates from the device's keyframe metadata (osb_frontend_loop_candidates_dev) -----------------
struct CandRule {              // osb_candidate_params and the handle's self_id
  int self_id, init_frames;
  double pos_per_m, ang_per_m, loop_pos, loop_ang;
};

// on_image_recv's init_mode (loop_detector.cpp:65-72) from inter_drone_loop_count [256][256] ([new][old]); ids outside
// 0..255 count 0
__device__ __forceinline__ bool fe_init_mode(int drone, int self_id, const int32_t* __restrict__ pairs, int init_frames) {
  if (drone == self_id) return false;
  const bool in = drone >= 0 && drone < LM_PAIR_DRONES && self_id >= 0 && self_id < LM_PAIR_DRONES;
  const int cnt = in ? pairs[drone * LM_PAIR_DRONES + self_id] : 0;
  return !(cnt >= init_frames);
}

__global__ void fe_init_modes_kernel(const osb_keyframe_record* __restrict__ recs, int n, int skip, CandRule cr,
                                     const int32_t* __restrict__ pairs, uint8_t* __restrict__ out) {
  const int i = threadIdx.x;
  if (i >= n) return;
  out[i] = (i != skip && fe_init_mode(recs[i].drone_id, cr.self_id, pairs, cr.init_frames)) ? 1 : 0;
}

// osb_frontend_receive_dev: a received record as LoopNet delivers it and on_image_recv keeps it (loop_net.cpp:20-93,
// :142-166, :230-262; loop_detector.cpp:36-65).  One CTA of FE_RECV_THREADS per (record, direction).  Every CTA counts the
// flagged landmarks of all directions of its record, so it evaluates the frame gates itself; its own direction's flagged
// landmarks get their slots from a ballot prefix (stable, no atomics).  Records r == skip and own records are copied as they are.
constexpr int FE_RECV_THREADS = 256;
static_assert(FE_RECV_THREADS >= OSB_MAX_KPTS && FE_RECV_THREADS == 256, "one thread per landmark; fe_block_compact's 8 warps");
static_assert(sizeof(osb_keyframe_record) % 16 == 0 && offsetof(osb_keyframe_record, global_desc) % 16 == 0 &&
                  offsetof(osb_keyframe_record, local_desc) % 16 == 0 && offsetof(osb_keyframe_record, kpts) % 16 == 0 &&
                  offsetof(osb_keyframe_record, stereo_match) % 16 == 0 &&
                  offsetof(osb_keyframe_record, landmarks_3d) % 16 == 0 &&
                  offsetof(osb_keyframe_record, landmarks_flag) % 16 == 0,
              "the record's planes move as float4");

// n float4 from s to d (both 16-byte aligned)
__device__ __forceinline__ void fe_copy16(void* __restrict__ d, const void* __restrict__ s, int n) {
  const float4* a = static_cast<const float4*>(s);
  float4* b = static_cast<float4*>(d);
#pragma unroll 4
  for (int i = threadIdx.x; i < n; i += FE_RECV_THREADS) b[i] = a[i];
}

__device__ __forceinline__ void fe_zero16(void* __restrict__ d, int n) {
  float4* b = static_cast<float4*>(d);
  const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int i = threadIdx.x; i < n; i += FE_RECV_THREADS) b[i] = z;
}

template <class T>
constexpr int fe_f4(const T&) { return (int)(sizeof(T) / 16); }

__global__ void __launch_bounds__(FE_RECV_THREADS)
fe_receive_kernel(const osb_keyframe_record* __restrict__ in, osb_keyframe_record* __restrict__ out, int skip, int self_id,
                  int min_direction_loop, int min_loop_num, const DbDev* __restrict__ local_cnt,
                  const DbDev* __restrict__ remote_cnt) {
  const int r = blockIdx.x / OSB_MAX_DIRS, d = blockIdx.x % OSB_MAX_DIRS;
  const int tid = threadIdx.x;
  const osb_keyframe_record* src = in + r;
  osb_keyframe_record* dst = out + r;
  const int drone = src->drone_id;
  if (r == skip || drone == self_id) {                       // not received: byte for byte
    if (d == 0 && tid < 3) reinterpret_cast<float4*>(dst)[tid] = reinterpret_cast<const float4*>(src)[tid];
    fe_copy16(dst->global_desc[d], src->global_desc[d], fe_f4(src->global_desc[d]));
    fe_copy16(dst->local_desc[d], src->local_desc[d], fe_f4(src->local_desc[d]));
    fe_copy16(dst->kpts[d], src->kpts[d], fe_f4(src->kpts[d]));
    fe_copy16(dst->stereo_match[d], src->stereo_match[d], fe_f4(src->stereo_match[d]));
    fe_copy16(dst->landmarks_3d[d], src->landmarks_3d[d], fe_f4(src->landmarks_3d[d]));
    fe_copy16(dst->landmarks_flag[d], src->landmarks_flag[d], fe_f4(src->landmarks_flag[d]));
    return;
  }
  // flagged landmarks of every direction: header feature_num = landmark_num after scan_recv_packets (loop_net.cpp:43-48)
  __shared__ int cnt[OSB_MAX_DIRS];
  __shared__ int16_t from[OSB_MAX_KPTS];                     // slot -> landmark index of this CTA's direction
  const int nd = min(max(src->n_dirs, 0), OSB_MAX_DIRS);
  for (int dd = 0; dd < OSB_MAX_DIRS; ++dd) {
    const int n = dd < nd ? min(max(src->n_kpts[dd], 0), OSB_MAX_KPTS) : 0;
    const bool keep = tid < n && src->landmarks_flag[dd][tid] > 0;
    int total;
    const int pos = fe_block_compact(keep, &total);
    if (dd == d && keep) from[pos] = (int16_t)tid;
    if (tid == 0) cnt[dd] = total;
    __syncthreads();                                         // fe_block_compact's warp counts are reused next pass
  }
  int dirs = 0, sum = 0;
  for (int dd = 0; dd < OSB_MAX_DIRS; ++dd) { dirs += cnt[dd] > 0 ? 1 : 0; sum += cnt[dd]; }
  // on_image_recv's gates (loop_detector.cpp:36-38, :53-63, :65): database_size() is local + remote rows at this point
  const bool dropped = local_cnt->ntotal + remote_cnt->ntotal == 0 || dirs < min_direction_loop || sum < min_loop_num;
  const int c = dropped ? 0 : cnt[d];
  if (d == 0 && tid == 0) {
    dst->drone_id = drone; dst->msg_id = src->msg_id; dst->n_dirs = src->n_dirs;
    dst->reserved = dropped ? 0 : src->reserved;
  }
  if (tid == 0) { dst->n_kpts[d] = c; dst->n_kpts_down[d] = 0; }   // no down image travels
  if (c > 0) fe_copy16(dst->global_desc[d], src->global_desc[d], fe_f4(src->global_desc[d]));
  else fe_zero16(dst->global_desc[d], fe_f4(dst->global_desc[d]));   // a null image (generate_null_img_desc)
  // local descriptors: 16 float4 per landmark, slot s from landmark from[s]
  {
    constexpr int R4 = OSB_FEATURE_DESC_SIZE / 4;
    const float4* a = reinterpret_cast<const float4*>(src->local_desc[d]);
    float4* b = reinterpret_cast<float4*>(dst->local_desc[d]);
#pragma unroll 4
    for (int i = tid; i < OSB_MAX_KPTS * R4; i += FE_RECV_THREADS) {
      const int s = i / R4, k = i % R4;
      b[i] = s < c ? a[from[s] * R4 + k] : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
  if (tid < OSB_MAX_KPTS) {
    const int s = tid;
    const bool ok = s < c;
    const int j = ok ? from[s] : 0;
    dst->kpts[d][s][0] = ok ? src->kpts[d][j][0] : 0.f;
    dst->kpts[d][s][1] = ok ? src->kpts[d][j][1] : 0.f;
    dst->stereo_match[d][s] = ok ? src->stereo_match[d][j] : (dropped ? 0 : -1);
#pragma unroll
    for (int k = 0; k < 3; ++k) dst->landmarks_3d[d][s][k] = ok ? src->landmarks_3d[d][j][k] : 0.f;
    dst->landmarks_flag[d][s] = ok ? src->landmarks_flag[d][j] : 0;
  }
}

// candidate i on thread i: the query side from metas[i], the hit side from the meta table of the hit's store, init_mode,
// and for same-drone hits the ego-motion trajectory's relative pose and covariance (check_loop_odometry_consistency,
// loop_detector.cpp:294-303) in the order of tests/loop_candidates_ref.py
__global__ void lc_candidates_kernel(const osb_keyframe_record* __restrict__ recs, const osb_keyframe_meta* __restrict__ metas,
                                     const osb_loop_result* __restrict__ results, int n, const uint8_t* __restrict__ init_dev,
                                     const __grid_constant__ FeStores dbs, FeMeta mt, const int32_t* __restrict__ pairs,
                                     CandRule cr, osb_loop_candidate* __restrict__ cand_out,
                                     osb_loop_stamps* __restrict__ stamps_out) {
  const int i = threadIdx.x;
  if (i >= n) return;
  const osb_keyframe_record* rec = recs + i;
  const osb_loop_result* res = results + i;
  const osb_keyframe_meta& mq = metas[i];
  const bool q_ok = mq.drone_id == rec->drone_id && mq.msg_id == rec->msg_id;
  const bool accepted = res->accepted != 0;
  const osb_keyframe_meta* mh = nullptr;
  if (accepted) {
    const bool hit_remote = res->hit_id >= OSB_REMOTE_MAGIN_NUMBER;
    const int fs = dbs.db[hit_remote].row_frame[hit_remote ? res->hit_id - OSB_REMOTE_MAGIN_NUMBER : res->hit_id];
    if (mt.ok[hit_remote][fs]) mh = mt.meta[hit_remote] + fs;
  }
  osb_loop_candidate c;
  memset(&c, 0, sizeof(c));
  c.init_mode = (init_dev ? init_dev[i] != 0 : fe_init_mode(rec->drone_id, cr.self_id, pairs, cr.init_frames)) ? 1 : 0;
  const int64_t sq = q_ok ? mq.stamp_ns : 0, sh = mh ? mh->stamp_ns : 0;
  for (int k = 0; k < 7; ++k) {
    const double id = k == 3 ? 1.0 : 0.0;
    c.pose_query[k] = q_ok ? mq.pose_drone[k] : id;
    c.pose_hit[k] = mh ? mh->pose_drone[k] : id;
    c.odom_rel[k] = id;
  }
  bool mark = accepted && (!q_ok || mh == nullptr);
  if (accepted && !mark && rec->drone_id == res->hit_drone_id) {
    const int tn = mt.dev->traj_n;
    if (tn == 0) {
      mark = true;
    } else {
      const bool swapped = res->swapped != 0;                 // compute_loop's roles: a = old, b = new
      const int ka = nearest_sample(mt.t_stamp, tn, swapped ? sq : sh);
      const int kb = nearest_sample(mt.t_stamp, tn, swapped ? sh : sq);
      double inv[7];
      lc_pose_inv(mt.t_pose + (size_t)ka * 7, inv);
      lc_pose_mul(inv, mt.t_pose + (size_t)kb * 7, c.odom_rel);
      const double dl = fabs(mt.t_len[kb] - mt.t_len[ka]);
      for (int k = 0; k < 6; ++k)
        c.odom_edge_cov[k * 7] = k < 3 ? lc_mul(dl, cr.pos_per_m) + cr.loop_pos : lc_mul(dl, cr.ang_per_m) + cr.loop_ang;
    }
  }
  c.reserved = mark ? 1 : 0;
  cand_out[i] = c;
  stamps_out[i].stamp_query_ns = sq;
  stamps_out[i].stamp_hit_ns = sh;
}

}  // namespace osb

using namespace osb;

struct osb_frontend {
  osb_frontend_config cfg;
  int device = 0;
  std::mutex mu;
  cudaStream_t stream = nullptr;
  SuperPoint sp;
  NetVLAD nv;
  Resources res;                 // every buffer, stream and event of the handle (sp and nv own theirs)
  DbStore db[2];                 // 0 local, 1 remote
  uint8_t* d_img = nullptr;      // [2*n_dirs][H][W]
  // stereo matcher state
  FePairs* d_st_pairs = nullptr; // static q / t tables into sp.d_out
  int32_t *d_st_qi = nullptr, *d_st_ti = nullptr, *d_st_n = nullptr, *d_st_map = nullptr;
  float *d_st_dist = nullptr, *d_dist_scratch = nullptr;
  // query state: the direction pairs of the hit, written by fe_query_rule_kernel, and the matcher / filter scratch
  FePairs* d_q_pairs = nullptr;
  FeMatchScratch q1;
  // osb_frontend_query_received: the same for FE_MAX_RECORDS records, their query descriptors [FE_MAX_RECORDS][4096] and
  // local top-k lists [FE_MAX_RECORDS][FE_RQ_K]; acquired by the first call (rq_ready)
  bool rq_ready = false;
  FeBatchPairs* d_rq_pairs = nullptr;
  FeMatchScratch rq;
  float* d_rq_desc = nullptr;
  float* d_rq_scores = nullptr;
  int64_t* d_rq_ids = nullptr;
  // stereo triangulation (osb_frontend_set_cameras)
  bool have_cameras = false;
  double K[4] = {0, 0, 0, 0}, triangle_thres = 0.006;
  double left_ext[OSB_MAX_DIRS][7], right_ext[OSB_MAX_DIRS][7], pose_drone[7] = {0, 0, 0, 1, 0, 0, 0};
  double* d_cam_pose = nullptr;  // [2][n_dirs][7]: pose_drone * left / right extrinsics of the current keyframe
  float* d_l3d = nullptr;        // [n_dirs][max_num][3]
  uint8_t *d_lflag_up = nullptr, *d_lflag_down = nullptr;
  // osb_frontend_set_main_camera(OSB_MAIN_CAMERA_DOWN): LOWER_CAM_AS_MAIN (swarm_loop.cpp:243) -- the record is the down
  // image's, and compute_loop lifts the old frame through the right extrinsics
  bool main_down = false;
  // depth camera (osb_frontend_set_depth_camera): the PINHOLE_DEPTH keyframe of extract_depth
  bool have_depth_camera = false;
  double depth_K[4] = {0, 0, 0, 0}, depth_ext[OSB_MAX_DIRS][7], near_thres = 0.3, far_thres = 10.0;
  uint16_t* d_depth = nullptr;   // [n_dirs][H][W] mm, staging of the host-buffer depth extracts
  // loop edges (osb_frontend_set_loop_params / osb_frontend_compute_loop): the PnP stage's inputs and outputs for LC_MAX
  // candidates, acquired by the first compute_loop (lc_ready)
  bool have_loop_params = false;
  osb_loop_params loop_params{};
  bool lc_ready = false;
  float *d_lc_pts3d = nullptr, *d_lc_pts2d = nullptr;   // [LC_MAX][LC_MAXN][3] / [2]
  int32_t* d_lc_n = nullptr;
  osb_pnp_params* d_lc_params = nullptr;
  uint8_t* d_lc_mask = nullptr;                           // [LC_MAX][LC_MAXN]
  osb_pnp_result* d_lc_pnp = nullptr;
  // osb_frontend_loop_measurements: loop_count and inter_drone_loop_count [256][256] on the device, acquired by its first
  // call; ev_lm is recorded after every call so that osb_frontend_loop_counts can wait for the last one
  long long* d_lm_count = nullptr;
  int32_t* d_lm_pairs = nullptr;
  cudaEvent_t ev_lm = nullptr;
  // keyframe metadata (osb_frontend_ingest_meta): both stores' meta tables and the ego-motion trajectory, acquired by the
  // first meta ingest (meta_ready); h_meta is the pinned copy osb_frontend_meta_status reads
  bool meta_ready = false;
  FeMeta meta{};
  FeMetaDev* h_meta = nullptr;
  bool have_cand_params = false;             // osb_frontend_set_candidate_params
  osb_candidate_params cand_params{};
  int32_t* d_assign = nullptr;   // [max_records][4]
  float* d_load_stage = nullptr;   // [FE_LOAD_ROWS][4096]: osb_frontend_db_load's fp32 -> fp16 staging, acquired by the first
                                   // load into an fp16 store
  int max_records = FE_MAX_RECORDS;
  osb_keyframe_record* d_record = nullptr;   // used by process()
  osb_loop_result* d_result = nullptr;
  // stage profiling: ev[i] marks the START of stage i, ev[8] the end of the last one
  cudaStream_t stream2 = nullptr;                 // NetVLAD runs here, overlapped with the keypoint kernels
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  DbDev* h_cnt = nullptr;                         // pinned [2]: row counters read back without blocking the driver (a copy
                                                  // to pageable memory would hold other host threads' launches until it ran)
  // the stores' row counts as the ingests report them: every ingest charges the most rows it could give ONE store (a
  // record's drone_id, and so its store, is only known on the device) and publishes both ntotal
  CountFeedback fb;
  bool profiling = false;
  cudaEvent_t ev[9] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  bool ev_valid[9] = {false, false, false, false, false, false, false, false, false};
};

static inline void fe_mark(osb_frontend* h, int i, cudaStream_t st) {
  if (!h->profiling) return;
  if (!h->ev[i]) h->res.event(&h->ev[i]);
  cudaEventRecord(h->ev[i], st);
  h->ev_valid[i] = true;
}

static osb_status dbstore_alloc(Resources& m, DbStore& s, int64_t cap, int max_num) {
  s.cap = cap; s.upper = 0;
  DbView& v = s.v;
  const size_t c = (size_t)cap, cn = c * max_num;
  OSB_TRY(m.alloc(&v.dev, 1));
  OSB_CUDA(cudaMemset(v.dev, 0, sizeof(DbDev)));
  v.storage = OSB_DB_STORAGE_FP32;
  OSB_TRY(db_rows_alloc(m, &v.rows, c * OSB_DEEP_DESC_SIZE, v.storage));
  OSB_TRY(m.alloc(&v.ldesc, cn * OSB_FEATURE_DESC_SIZE));
  OSB_TRY(m.alloc(&v.kpts, cn * 2));
  OSB_TRY(m.alloc(&v.lflag, cn));
  OSB_CUDA(cudaMemset(v.kpts, 0, cn * 2 * sizeof(float)));
  OSB_CUDA(cudaMemset(v.lflag, 1, cn * sizeof(int32_t)));   // rows loaded without geometry: every landmark flagged (non-zero)
  OSB_TRY(m.alloc(&v.nk, c));
  OSB_TRY(m.alloc(&v.row_frame, c));
  OSB_TRY(m.alloc(&v.row_dir, c));
  OSB_TRY(m.alloc(&v.frame_rows, c * OSB_MAX_DIRS));
  OSB_TRY(m.alloc(&v.frame_msg, c));
  OSB_TRY(m.alloc(&v.frame_drone, c));
  int64_t chunk;
  const int gmax = db_scan_grid(cap, &chunk);
  OSB_TRY(m.alloc(&s.part_scores, (size_t)8 * gmax * FE_KMAX));
  OSB_TRY(m.alloc(&s.part_ids, (size_t)8 * gmax * FE_KMAX));
  OSB_TRY(m.alloc(&s.done, 1));
  OSB_CUDA(cudaMemset(s.done, 0, sizeof(unsigned int)));
  OSB_TRY(m.alloc(&v.top_scores, FE_KMAX));
  OSB_TRY(m.alloc(&v.top_ids, FE_KMAX));
  OSB_CUDA(cudaMemset(v.top_ids, 0xFF, FE_KMAX * sizeof(int64_t)));     // "no result" (-1) until the first scan of this store
  return OSB_OK;
}

static FeStores fe_stores(const osb_frontend* h) { return FeStores{{h->db[0].v, h->db[1].v}}; }

// the filter's buffers for `slots` direction-pair slots
static osb_status fe_geo_alloc(Resources& m, FeMatchScratch& g, int slots, cudaStream_t st) {
  const size_t sk = (size_t)slots * OSB_MAX_KPTS;
  OSB_TRY(m.alloc(&g.g_src, sk * 2));
  OSB_TRY(m.alloc(&g.g_dst, sk * 2));
  OSB_TRY(m.alloc(&g.g_kept, sk));
  OSB_TRY(m.alloc(&g.g_nkept, slots));
  OSB_TRY(m.alloc(&g.g_ninl, slots));
  OSB_TRY(m.alloc(&g.g_win, slots));
  OSB_TRY(m.alloc(&g.g_mask, sk));
  OSB_TRY(m.alloc(&g.g_keys, 2 * (size_t)slots));
  OSB_CUDA(cudaMemsetAsync(g.g_keys, 0, 2 * (size_t)slots * sizeof(unsigned int), st));   // before the first RANSAC on st
  return OSB_OK;
}

extern "C" osb_status osb_frontend_create(osb_frontend** out, const osb_frontend_config* cfg, const float* sp_weights,
                                          size_t n_sp_weights, const float* pca_comp, const float* pca_mean,
                                          const float* nv_weights, size_t n_nv_weights) {
  OSB_REQUIRE(out && cfg && sp_weights && pca_comp && pca_mean && nv_weights, "null argument");
  OSB_REQUIRE(cfg->n_dirs >= 1 && cfg->n_dirs <= OSB_MAX_DIRS, "n_dirs must be 1..4");
  OSB_REQUIRE(cfg->max_num >= 1 && cfg->max_num <= OSB_MAX_KPTS, "max_num must be 1..200");
  OSB_REQUIRE(cfg->query_dir >= 0 && cfg->query_dir < cfg->n_dirs, "query_dir out of range");
  OSB_REQUIRE(cfg->db_capacity > 0 && cfg->db_capacity < (1 << 30), "bad db_capacity");
  OSB_REQUIRE(cfg->match_index_dist >= 1 && 5 + cfg->match_index_dist <= FE_KMAX, "bad match_index_dist");
  OSB_TRY(require_device());
  std::unique_ptr<osb_frontend> h(new osb_frontend());
  h->cfg = *cfg;
  h->device = current_device();
  const int nd = cfg->n_dirs, mn = cfg->max_num;
  Resources& m = h->res;
  OSB_TRY(m.stream(&h->stream));
  OSB_TRY(m.stream(&h->stream2));
  OSB_TRY(m.event(&h->ev_fork, cudaEventDisableTiming));
  OSB_TRY(m.event(&h->ev_join, cudaEventDisableTiming));
  OSB_TRY(m.host_alloc(&h->h_cnt, 2, cudaHostAllocDefault));
  OSB_TRY(h->fb.init(m));
  OSB_TRY(h->sp.init(sp_weights, n_sp_weights, cfg->width, cfg->height, cfg->sp_thres, mn, pca_comp, pca_mean, 2 * nd));
  h->sp.ks.write_surv = false;       // the survivor plane is only a parity hook of the standalone SuperPoint handle
  if (cfg->zero_bottom_quarter) OSB_TRY(h->sp.band_init());
  OSB_TRY(h->sp.sparse_init());
  OSB_TRY(h->nv.init(nv_weights, n_nv_weights, cfg->width, cfg->height, nd));
  OSB_TRY(dbstore_alloc(m, h->db[0], cfg->db_capacity, mn));
  OSB_TRY(dbstore_alloc(m, h->db[1], cfg->db_capacity, mn));
  const size_t HW = (size_t)cfg->width * cfg->height, dk = (size_t)OSB_MAX_DIRS * OSB_MAX_KPTS, dm = (size_t)OSB_MAX_DIRS * mn;
  OSB_TRY(m.alloc(&h->d_img, 2 * nd * HW));
  OSB_TRY(m.alloc(&h->d_st_pairs, 1));
  OSB_TRY(m.alloc(&h->d_q_pairs, 1));
  OSB_TRY(m.alloc(&h->d_st_qi, dm));
  OSB_TRY(m.alloc(&h->d_st_ti, dm));
  OSB_TRY(m.alloc(&h->d_st_map, dm));
  OSB_TRY(m.alloc(&h->d_st_n, OSB_MAX_DIRS));
  OSB_TRY(m.alloc(&h->d_st_dist, dm));
  OSB_TRY(m.alloc(&h->q1.dout, dk));
  OSB_TRY(fe_geo_alloc(m, h->q1, OSB_MAX_DIRS, 0));
  OSB_TRY(m.alloc(&h->d_dist_scratch, dm * mn));
  h->q1.pairs = fe_pair_view(h->d_q_pairs);
  h->q1.dist = h->d_dist_scratch;            // shared with the stereo match of extract
  OSB_TRY(m.alloc(&h->d_assign, (size_t)h->max_records * OSB_MAX_DIRS));
  OSB_TRY(m.alloc(&h->d_cam_pose, 2 * OSB_MAX_DIRS * 7));
  OSB_TRY(m.alloc(&h->d_l3d, dm * 3));
  OSB_TRY(m.alloc(&h->d_lflag_up, dm));
  OSB_TRY(m.alloc(&h->d_lflag_down, dm));
  OSB_TRY(m.alloc(&h->d_record, 1));
  OSB_TRY(m.alloc(&h->d_result, 1));
  {
    FePairs st{};                // the stereo match pairs up[d] with down[d]; its counts are sp.d_nk
    for (int d = 0; d < nd; ++d) {
      st.q[d] = h->sp.d_out + (size_t)d * mn * OSB_FEATURE_DESC_SIZE;
      st.t[d] = h->sp.d_out + (size_t)(nd + d) * mn * OSB_FEATURE_DESC_SIZE;
    }
    OSB_CUDA(cudaMemcpy(h->d_st_pairs, &st, sizeof(st), cudaMemcpyHostToDevice));
  }
  *out = h.release();
  return OSB_OK;
}

extern "C" osb_status osb_frontend_set_precision(osb_frontend* h, int precision) {
  OSB_REQUIRE(h != nullptr, "null handle");
  std::lock_guard<std::mutex> lk(h->mu);
  OSB_TRY(h->sp.set_precision(precision));            // the same check for both networks: nv accepts what sp accepted
  return h->nv.set_precision(precision);
}

extern "C" osb_status osb_frontend_set_db_storage(osb_frontend* h, int storage) {
  OSB_REQUIRE(h != nullptr, "null handle");
  OSB_REQUIRE(storage == OSB_DB_STORAGE_FP32 || storage == OSB_DB_STORAGE_FP16,
              "storage must be OSB_DB_STORAGE_FP32 or OSB_DB_STORAGE_FP16");
  std::lock_guard<std::mutex> lk(h->mu);
  // the host bounds are charged when an ingest is enqueued, so 0 also rules out an ingest that has not run yet
  OSB_REQUIRE(h->db[0].upper == 0 && h->db[1].upper == 0,
              "the databases already hold rows: set the storage right after create or osb_frontend_db_reset");
  DeviceGuard dg(h->device);
  if (storage == h->db[0].v.storage) return OSB_OK;
  // both new planes first, so that a failed allocation leaves the handle as it was
  void* rows[2] = {nullptr, nullptr};
  for (int i = 0; i < 2; ++i) {
    const osb_status s = db_rows_alloc(h->res, &rows[i], (size_t)h->db[i].cap * OSB_DEEP_DESC_SIZE, storage);
    if (s != OSB_OK) {
      if (i == 1) h->res.release(rows[0]);
      return s;
    }
  }
  for (int i = 0; i < 2; ++i) {
    h->res.release(h->db[i].v.rows);
    h->db[i].v.rows = rows[i];
    h->db[i].v.storage = storage;
  }
  return OSB_OK;
}

extern "C" osb_status osb_frontend_destroy(osb_frontend* h) {
  delete h;
  return OSB_OK;
}

// a * b for poses (x y z, qw qx qy qz), host side
static void pose_compose_host(const double* a, const double* b, double* o) {
  const double w = a[3], x = a[4], y = a[5], z = a[6];
  const double cx = y * b[2] - z * b[1], cy = z * b[0] - x * b[2], cz = x * b[1] - y * b[0];
  const double dx = y * cz - z * cy, dy = z * cx - x * cz, dz = x * cy - y * cx;
  o[0] = a[0] + b[0] + 2.0 * (w * cx + dx);
  o[1] = a[1] + b[1] + 2.0 * (w * cy + dy);
  o[2] = a[2] + b[2] + 2.0 * (w * cz + dz);
  o[3] = w * b[3] - x * b[4] - y * b[5] - z * b[6];
  o[4] = w * b[4] + x * b[3] + y * b[6] - z * b[5];
  o[5] = w * b[5] - x * b[6] + y * b[3] + z * b[4];
  o[6] = w * b[6] + x * b[5] - y * b[4] + z * b[3];
}

// the keyframe staged in h->d_img (and h->d_depth) -> record_dev.
// depth == false: a stereo keyframe, d_img = [2*nd][H][W] up then down.
// depth == true: a PINHOLE_DEPTH keyframe (generate_gray_depth_image_descriptor, loop_cam.cpp:231-302), d_img = [nd][H][W]
// gray images and d_depth = [nd][H][W] mm: SuperPoint on the nd images, no stereo match, landmarks from the depth look-up.
// The bottom quarter is never blanked there: the reference blanks only in STEREO_FISHEYE (:536).
static osb_status fe_extract_dev(osb_frontend* h, bool depth, int32_t msg_id, osb_keyframe_record* record_dev,
                                 cudaStream_t st) {
  const osb_frontend_config& c = h->cfg;
  const int nd = c.n_dirs, mn = c.max_num;
  const int n_img = depth ? nd : 2 * nd;
  osb_status s;
  // the first blanked row, which SuperPoint's trunk is told so that it stores the band's constant tiles (-1: no blanking)
  const int zero_row = (!depth && c.zero_bottom_quarter) ? c.height * 3 / 4 : -1;
  if (zero_row >= 0) {
    OSB_LAUNCH(fe_blank_kernel, 256, 256, 0, st, h->d_img, c.height, c.width, 2 * nd, zero_row);
    OSB_CHECK_LAUNCH();
  }
  // fork: NetVLAD is independent of SuperPoint (it only reads the images).  It runs on a second stream for the whole
  // SuperPoint phase: its element-wise / depthwise kernels co-reside with the persistent convolution CTAs, its
  // tensor-core launches fill the wave tails, and while the keypoint kernels run (one CTA per image) it owns the
  // other 140 SMs.  It joins before the record is packed.
  OSB_CUDA(cudaEventRecord(h->ev_fork, st));
  OSB_CUDA(cudaStreamWaitEvent(h->stream2, h->ev_fork, 0));
  // NetVLAD writes straight into the record (image_desc, loop_cam.cpp:553-556): on the up images, or with the lower camera
  // as main on the down images (:350-351)
  const bool down_main = !depth && h->main_down;
  const uint8_t* nv_img = down_main ? h->d_img + (size_t)nd * c.width * c.height : h->d_img;
  if ((s = h->nv.infer_dev(nv_img, nd, &record_dev->global_desc[0][0], h->stream2)) != OSB_OK) return s;
  OSB_CUDA(cudaEventRecord(h->ev_join, h->stream2));
  fe_mark(h, 0, st);
  // network; the keypoint kernel is forked beside the descriptor head inside (superpoint.cu) and joined before return
  const SuperPoint::KpJob kp{h->sp.d_nk, h->sp.d_kpts, h->sp.d_conf};
  if ((s = h->sp.network(h->d_img, n_img, st, &kp, zero_row)) != OSB_OK) return s;
  h->sp.last_batch = n_img;
  fe_mark(h, 1, st);
  if ((s = h->sp.descriptors(n_img, kp, h->sp.d_out, st)) != OSB_OK) return s;
  fe_mark(h, 2, st);
  OSB_CUDA(cudaStreamWaitEvent(st, h->ev_join, 0));      // join (stage 2 = the part of NetVLAD that was not hidden)
  fe_mark(h, 3, st);
  const int32_t* stereo_map = nullptr;                    // stays null for a depth keyframe
  bool lifted = false;                                    // landmarks_3d / landmarks_flag computed on the device
  double cam[2][OSB_MAX_DIRS][7];
  if (depth) {
    // pose_cam = pose_drone * extrinsic[d] (loop_cam.cpp:273-274), then the per-keypoint depth look-up (:276-302); the gate
    // landmarks_2d.size() > ACCEPT_MIN_3D_PTS (:267) is the lift's min_pts
    for (int d = 0; d < nd; ++d) pose_compose_host(h->pose_drone, h->depth_ext[d], cam[0][d]);
    OSB_CUDA(cudaMemcpyAsync(h->d_cam_pose, cam[0], (size_t)nd * 7 * sizeof(double), cudaMemcpyHostToDevice, st));
    if ((s = depth_lift_device(h->sp.d_kpts, h->sp.d_nk, nd, mn, h->d_depth, c.height, c.width, h->depth_K, h->d_cam_pose,
                               h->near_thres, h->far_thres, c.accept_min_3d_pts, h->d_l3d, h->d_lflag_up, st)) != OSB_OK)
      return s;
    lifted = true;
  } else {
    // stereo match up[d] <-> down[d] (loop_cam.cpp:388)
    if ((s = bf_match_device(nd, mn, mn, h->d_st_pairs->q, h->sp.d_nk, h->d_st_pairs->t, h->sp.d_nk + nd, h->d_dist_scratch,
                             h->d_st_qi, h->d_st_ti, h->d_st_dist, h->d_st_n, h->d_st_map, st)) != OSB_OK) return s;
    stereo_map = h->d_st_map;
    if (h->have_cameras) {
      // pose_up / pose_down = pose_drone * extrinsics (loop_cam.cpp:394-396), then the per-keypoint triangulation (:398-432)
      for (int d = 0; d < nd; ++d) {
        pose_compose_host(h->pose_drone, h->left_ext[d], cam[0][d]);
        pose_compose_host(h->pose_drone, h->right_ext[d], cam[1][d]);
      }
      OSB_CUDA(cudaMemcpyAsync(h->d_cam_pose, cam[0], (size_t)nd * 7 * sizeof(double), cudaMemcpyHostToDevice, st));
      OSB_CUDA(cudaMemcpyAsync(h->d_cam_pose + OSB_MAX_DIRS * 7, cam[1], (size_t)nd * 7 * sizeof(double), cudaMemcpyHostToDevice, st));
      if ((s = stereo_lift_device(h->sp.d_kpts, h->sp.d_kpts + (size_t)nd * mn * 2, h->d_st_map, h->sp.d_nk, h->sp.d_nk + nd, nd,
                                  mn, h->K, h->d_cam_pose, h->d_cam_pose + OSB_MAX_DIRS * 7, h->triangle_thres,
                                  c.accept_min_3d_pts, h->d_l3d, h->d_lflag_up, h->d_lflag_down, st, down_main)) != OSB_OK)
        return s;
      lifted = true;
    }
  }
  // the record's flags: the up keypoints', or with the lower camera as main the down keypoints' (loop_cam.cpp:443-444)
  const uint8_t* lflag = lifted ? (down_main ? h->d_lflag_down : h->d_lflag_up) : nullptr;
  if (down_main)
    OSB_LAUNCH(fe_pack_kernel<true>, OSB_MAX_DIRS, 256, 0, st, record_dev, c.self_id, msg_id, nd, mn, h->sp.d_nk, h->sp.d_kpts,
               h->sp.d_out, stereo_map, c.accept_min_3d_pts, lifted ? h->d_l3d : nullptr, lflag);
  else
    OSB_LAUNCH(fe_pack_kernel<false>, OSB_MAX_DIRS, 256, 0, st, record_dev, c.self_id, msg_id, nd, mn, h->sp.d_nk, h->sp.d_kpts,
               h->sp.d_out, stereo_map, c.accept_min_3d_pts, lifted ? h->d_l3d : nullptr, lflag);
  OSB_CHECK_LAUNCH();
  fe_mark(h, 4, st);
  return OSB_OK;
}

// up and down images [n_dirs][H][W] of a stereo keyframe -> the handle's staging buffer, then extract
static osb_status fe_extract_stereo(osb_frontend* h, const uint8_t* up, const uint8_t* down, cudaMemcpyKind kind,
                                    int32_t msg_id, osb_keyframe_record* record_dev, cudaStream_t st) {
  const size_t half = (size_t)h->cfg.n_dirs * h->cfg.width * h->cfg.height;
  OSB_CUDA(cudaMemcpyAsync(h->d_img, up, half, kind, st));
  OSB_CUDA(cudaMemcpyAsync(h->d_img + half, down, half, kind, st));
  return fe_extract_dev(h, false, msg_id, record_dev, st);
}

extern "C" osb_status osb_frontend_extract_dev(osb_frontend* h, const uint8_t* images_up_dev,
                                               const uint8_t* images_down_dev, int32_t msg_id,
                                               osb_keyframe_record* record_dev, void* stream) {
  OSB_REQUIRE(h && images_up_dev && images_down_dev && record_dev, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  return fe_extract_stereo(h, images_up_dev, images_down_dev, cudaMemcpyDeviceToDevice, msg_id, record_dev,
                           (cudaStream_t)stream);
}

extern "C" osb_status osb_frontend_extract(osb_frontend* h, const uint8_t* images_up, const uint8_t* images_down,
                                           int32_t msg_id, osb_keyframe_record* record_dev, void* stream) {
  OSB_REQUIRE(h && images_up && images_down && record_dev, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  return fe_extract_stereo(h, images_up, images_down, cudaMemcpyHostToDevice, msg_id, record_dev, (cudaStream_t)stream);
}

// gray images [n_dirs][H][W] and depth [n_dirs][H][W] (mm) of a depth keyframe -> the handle's buffers, then extract
static osb_status fe_extract_depth(osb_frontend* h, const uint8_t* images, const uint16_t* depth_mm, cudaMemcpyKind kind,
                                   int32_t msg_id, osb_keyframe_record* record_dev, cudaStream_t st) {
  const size_t px = (size_t)h->cfg.n_dirs * h->cfg.width * h->cfg.height;
  OSB_CUDA(cudaMemcpyAsync(h->d_img, images, px, kind, st));
  OSB_CUDA(cudaMemcpyAsync(h->d_depth, depth_mm, px * sizeof(uint16_t), kind, st));
  return fe_extract_dev(h, true, msg_id, record_dev, st);
}

extern "C" osb_status osb_frontend_extract_depth(osb_frontend* h, const uint8_t* images, const uint16_t* depth_mm,
                                                 int32_t msg_id, osb_keyframe_record* record_dev, void* stream) {
  OSB_REQUIRE(h && images && depth_mm && record_dev, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  OSB_REQUIRE(!h->main_down, "a depth keyframe has no lower camera: the main camera must be OSB_MAIN_CAMERA_UP");
  OSB_REQUIRE(h->have_depth_camera, "no depth camera: call osb_frontend_set_depth_camera first");
  DeviceGuard dg(h->device);
  return fe_extract_depth(h, images, depth_mm, cudaMemcpyHostToDevice, msg_id, record_dev, (cudaStream_t)stream);
}

extern "C" osb_status osb_frontend_extract_depth_dev(osb_frontend* h, const uint8_t* images_dev, const uint16_t* depth_mm_dev,
                                                     int32_t msg_id, osb_keyframe_record* record_dev, void* stream) {
  OSB_REQUIRE(h && images_dev && depth_mm_dev && record_dev, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  OSB_REQUIRE(!h->main_down, "a depth keyframe has no lower camera: the main camera must be OSB_MAIN_CAMERA_UP");
  OSB_REQUIRE(h->have_depth_camera, "no depth camera: call osb_frontend_set_depth_camera first");
  DeviceGuard dg(h->device);
  return fe_extract_depth(h, images_dev, depth_mm_dev, cudaMemcpyDeviceToDevice, msg_id, record_dev, (cudaStream_t)stream);
}

static osb_status fe_refresh_counts(osb_frontend* h, cudaStream_t st);

// side: which store the host CHARGES for the batch (its bounds): 0 = unknown (both), 1 = all records are this drone's own,
// 2 = all records are foreign.  The kernel always routes by drone_id.
// metas: one osb_keyframe_meta per record (osb_frontend_ingest_meta; the tables must be acquired), or null
static osb_status fe_ingest(osb_frontend* h, const osb_keyframe_record* recs, int n_records, int skip, cudaStream_t st,
                            int side = 0, const osb_keyframe_meta* metas = nullptr) {
  OSB_REQUIRE(n_records >= 0 && n_records <= h->max_records, "too many records in one ingest (max 64)");
  if (n_records == 0) return OSB_OK;
  DbStore &L = h->db[0], &R = h->db[1];
  long long n[2], since;                        // lower the bounds with what the last ingest that has RUN reported
  if (h->fb.read(n, &since))
    for (int i = 0; i < 2; ++i) h->db[i].upper = std::min<int64_t>(h->db[i].upper, n[i] + since);
  const int64_t chg_l = side == 2 ? 0 : (int64_t)n_records * OSB_MAX_DIRS, chg_r = side == 1 ? 0 : (int64_t)n_records * OSB_MAX_DIRS;
  if (L.upper + chg_l > L.cap || R.upper + chg_r > R.cap) {
    // the upper bounds are conservative (every record charged to both databases): make them exact, and count which
    // database each record of this batch really goes to, before giving up
    osb_status rs = fe_refresh_counts(h, st);
    if (rs != OSB_OK) return rs;
    std::vector<int32_t> hdr((size_t)n_records * 4);
    OSB_CUDA(cudaMemcpy2DAsync(hdr.data(), 16, recs, sizeof(osb_keyframe_record), 16, n_records, cudaMemcpyDeviceToHost, st));
    OSB_CUDA(cudaStreamSynchronize(st));
    int64_t n_loc = 0, n_rem = 0;
    for (int r = 0; r < n_records; ++r) {
      if (r == skip) continue;
      (hdr[(size_t)r * 4] == h->cfg.self_id ? n_loc : n_rem) += OSB_MAX_DIRS;
    }
    if (L.upper + n_loc > L.cap || R.upper + n_rem > R.cap) {
      set_error("osb_frontend_ingest", "database capacity exceeded");
      return OSB_ERR_CAPACITY;
    }
  }
  fe_mark(h, 4, st);
  const FeStores dbs = fe_stores(h);
  const long long seq = h->fb.charge((long long)n_records * OSB_MAX_DIRS);
  if (metas)
    OSB_LAUNCH(fe_assign_kernel<true>, 1, 32, 0, st, recs, n_records, skip, h->cfg.self_id, (long long)L.cap, dbs, h->d_assign,
               h->fb.dev, seq, h->fb.charged, metas, h->meta);
  else
    OSB_LAUNCH(fe_assign_kernel<false>, 1, 32, 0, st, recs, n_records, skip, h->cfg.self_id, (long long)L.cap, dbs, h->d_assign,
               h->fb.dev, seq, h->fb.charged, nullptr, FeMeta{});
  OSB_CHECK_LAUNCH();
  OSB_LAUNCH(fe_copy_rows_kernel, n_records * OSB_MAX_DIRS, 256, 0, st, recs, h->d_assign, h->cfg.max_num, dbs);
  OSB_CHECK_LAUNCH();
  L.upper += chg_l;
  R.upper += chg_r;
  OSB_CUDA(h->fb.record(st));
  fe_mark(h, 5, st);
  return OSB_OK;
}

extern "C" osb_status osb_frontend_ingest_own(osb_frontend* h, const osb_keyframe_record* record_dev, void* stream) {
  OSB_REQUIRE(h && record_dev, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  return fe_ingest(h, record_dev, 1, -1, (cudaStream_t)stream, 1);
}

extern "C" osb_status osb_frontend_ingest(osb_frontend* h, const osb_keyframe_record* records_dev, int n_records,
                                          int skip, void* stream) {
  OSB_REQUIRE(h && records_dev, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  return fe_ingest(h, records_dev, n_records, skip, (cudaStream_t)stream);
}

// the fields of a query's rule parameters that come from the configuration
static QueryParams fe_query_params(const osb_frontend* h) {
  const osb_frontend_config& c = h->cfg;
  QueryParams qp{};
  qp.self_id = c.self_id; qp.n_dirs = c.n_dirs; qp.query_dir = c.query_dir; qp.match_index_dist = c.match_index_dist;
  qp.k_remote = 5 + 1; qp.k_local = 5 + c.match_index_dist;       // SEARCH_NEAREST_NUM + max_index
  qp.max_num = c.max_num;
  qp.inner_product_thres = c.inner_product_thres; qp.init_mode_product_thres = c.init_mode_product_thres;
  qp.skip = -1;
  return qp;
}

// after the scans: the acceptance rule for qp.n records, the per-direction cross-check match new vs old of every record's
// direction pairs (loop_detector.cpp:564-567; empty pairs produce n = 0) and, with the geometric filter,
// loop_detector.cpp:569-598 (3-D-flag filter, homography RANSAC mask, reduceVector) -- each one launch for all records.
// Record r's results go to res[r]; `m` holds OSB_MAX_DIRS * qp.n slots.
// dev_init: the records' init_mode flags are the device bytes init_dev (or all 0 when null), not qp.init_mask
static osb_status fe_rule_match(osb_frontend* h, const QueryParams& qp, const osb_keyframe_record* recs,
                                osb_loop_result* res, const FeMatchScratch& m, cudaStream_t st, bool dev_init = false,
                                const uint8_t* init_dev = nullptr) {
  const osb_frontend_config& c = h->cfg;
  const int slots = OSB_MAX_DIRS * qp.n;
  osb_status s;
  if (dev_init)
    OSB_LAUNCH(fe_query_rule_kernel<true>, 1, 32 * cdiv(qp.n, 32), 0, st, qp, recs, fe_stores(h), res, m.pairs, init_dev);
  else
    OSB_LAUNCH(fe_query_rule_kernel<false>, 1, 32 * cdiv(qp.n, 32), 0, st, qp, recs, fe_stores(h), res, m.pairs, nullptr);
  OSB_CHECK_LAUNCH();
  s = bf_match_device(slots, c.max_num, OSB_MAX_KPTS, m.pairs.q, m.pairs.nq, m.pairs.t, m.pairs.nt, m.dist,
                      &res->match_new[0][0], &res->match_old[0][0], m.dout, &res->n_matches[0], nullptr, st, OSB_MAX_DIRS,
                      sizeof(osb_loop_result) / sizeof(int32_t));
  if (s != OSB_OK) return s;
  if (c.geometric_filter) {
    OSB_LAUNCH(fe_geo_gather_kernel, slots, 256, 0, st, res, m.pairs, reinterpret_cast<float2*>(m.g_src),
               reinterpret_cast<float2*>(m.g_dst), m.g_kept, m.g_nkept);
    OSB_CHECK_LAUNCH();
    if ((s = homography_ransac_device(m.g_src, m.g_dst, m.g_nkept, slots, OSB_MAX_KPTS, 3.0f, (uint32_t)c.ransac_seed,
                                      m.g_mask, m.g_ninl, m.g_win, st, m.g_keys)) != OSB_OK) return s;
    OSB_LAUNCH(fe_geo_apply_kernel, slots, 256, 0, st, res, m.g_kept, m.g_nkept, m.g_mask);
    OSB_CHECK_LAUNCH();
  }
  return OSB_OK;
}

static osb_status fe_query(osb_frontend* h, const osb_keyframe_record* rec, int init_mode, int nonkeyframe,
                           osb_loop_result* res, cudaStream_t st) {
  const osb_frontend_config& c = h->cfg;
  DbStore &L = h->db[0], &R = h->db[1];
  const float* q = &rec->global_desc[c.query_dir][0];
  QueryParams qp = fe_query_params(h);
  osb_status s;
  fe_mark(h, 5, st);
  long long n[2], since;
  if (h->fb.read(n, &since))
    for (int i = 0; i < 2; ++i) h->db[i].upper = std::min<int64_t>(h->db[i].upper, n[i] + since);
  // a store that has never received a row needs no scan: its top-k list still holds the -1 labels it was created with
  // (upper is an upper bound of ntotal, so 0 is exact)
  if (R.upper > 0 &&
      (s = db_search_device(R.v.rows, R.v.storage, std::min(R.upper, R.cap), &R.v.dev->ntotal, OSB_DEEP_DESC_SIZE, q, 1, qp.k_remote,
                            R.part_scores, R.part_ids, R.done, R.v.top_scores, R.v.top_ids, st)) != OSB_OK) return s;
  if ((s = db_search_device(L.v.rows, L.v.storage, std::min(L.upper, L.cap), &L.v.dev->ntotal, OSB_DEEP_DESC_SIZE, q, 1, qp.k_local,
                            L.part_scores, L.part_ids, L.done, L.v.top_scores, L.v.top_ids, st)) != OSB_OK) return s;
  fe_mark(h, 6, st);
  qp.n = 1;
  qp.init_mask = init_mode ? 1ull : 0ull;
  qp.nonkeyframe = nonkeyframe;
  qp.l_scores = L.v.top_scores; qp.l_ids = L.v.top_ids; qp.l_stride = 0;
  if ((s = fe_rule_match(h, qp, rec, res, h->q1, st)) != OSB_OK) return s;
  fe_mark(h, 7, st);
  return OSB_OK;
}

extern "C" osb_status osb_frontend_query(osb_frontend* h, const osb_keyframe_record* record_dev, int init_mode,
                                         int nonkeyframe, osb_loop_result* result_dev, void* stream) {
  OSB_REQUIRE(h && record_dev && result_dev, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  return fe_query(h, record_dev, init_mode, nonkeyframe, result_dev, (cudaStream_t)stream);
}

// osb_frontend_query_received's scratch for FE_MAX_RECORDS records, acquired once by its first call (the matcher's distance
// matrices alone are 4 * FE_MAX_RECORDS * max_num^2 floats, 41 MB at max_num = 200: a handle that never queries received
// keyframes does not hold them)
static osb_status fe_rq_alloc(osb_frontend* h, cudaStream_t st) {
  if (h->rq_ready) return OSB_OK;
  Resources& m = h->res;
  const int slots = OSB_MAX_DIRS * FE_MAX_RECORDS, mn = h->cfg.max_num;
  OSB_TRY(m.alloc(&h->d_rq_pairs, 1));
  OSB_TRY(m.alloc(&h->rq.dist, (size_t)slots * mn * mn));
  OSB_TRY(m.alloc(&h->rq.dout, (size_t)FE_MAX_RECORDS * sizeof(osb_loop_result) / sizeof(float)));
  OSB_TRY(fe_geo_alloc(m, h->rq, slots, st));
  OSB_TRY(m.alloc(&h->d_rq_desc, (size_t)FE_MAX_RECORDS * OSB_DEEP_DESC_SIZE));
  OSB_TRY(m.alloc(&h->d_rq_scores, (size_t)FE_MAX_RECORDS * FE_RQ_K));
  OSB_TRY(m.alloc(&h->d_rq_ids, (size_t)FE_MAX_RECORDS * FE_RQ_K));
  h->rq.pairs = fe_pair_view(h->d_rq_pairs);
  h->rq_ready = true;
  return OSB_OK;
}

// query_from_database for n keyframes received from other drones (loop_detector.cpp:98-119, 191-195): such a query reads
// only the local store, which the adds of received keyframes never change, so one pass over the local store answers all of
// them as the reference's one-at-a-time add / query sequence would
static osb_status fe_query_received(osb_frontend* h, const osb_keyframe_record* recs, int n, int skip,
                                    unsigned long long init_mask, osb_loop_result* res, cudaStream_t st,
                                    bool dev_init = false, const uint8_t* init_dev = nullptr) {
  const osb_frontend_config& c = h->cfg;
  DbStore& L = h->db[0];
  osb_status s;
  if ((s = fe_rq_alloc(h, st)) != OSB_OK) return s;
  long long nr[2], since;
  if (h->fb.read(nr, &since))
    for (int i = 0; i < 2; ++i) h->db[i].upper = std::min<int64_t>(h->db[i].upper, nr[i] + since);
  // the queried direction's global descriptor of every record -> one contiguous [n][4096] slab
  OSB_CUDA(cudaMemcpy2DAsync(h->d_rq_desc, OSB_DEEP_DESC_SIZE * sizeof(float), &recs->global_desc[c.query_dir][0],
                             sizeof(osb_keyframe_record), OSB_DEEP_DESC_SIZE * sizeof(float), n, cudaMemcpyDeviceToDevice, st));
  // one scan of the local store for all n (8 queries per pass), top-k per record into the batch's own lists
  if ((s = db_search_device(L.v.rows, L.v.storage, std::min(L.upper, L.cap), &L.v.dev->ntotal, OSB_DEEP_DESC_SIZE, h->d_rq_desc, n,
                            FE_RQ_K, L.part_scores, L.part_ids, L.done, h->d_rq_scores, h->d_rq_ids, st)) != OSB_OK) return s;
  QueryParams qp = fe_query_params(h);
  qp.n = n;
  qp.init_mask = init_mask;
  qp.l_scores = h->d_rq_scores; qp.l_ids = h->d_rq_ids; qp.l_stride = FE_RQ_K;
  qp.received = 1; qp.skip = skip;
  return fe_rule_match(h, qp, recs, res, h->rq, st, dev_init, init_dev);
}

extern "C" osb_status osb_frontend_query_received(osb_frontend* h, const osb_keyframe_record* records_dev, int n_records,
                                                  int skip, const uint8_t* init_mode, osb_loop_result* results_dev,
                                                  void* stream) {
  OSB_REQUIRE(h != nullptr, "null handle");
  OSB_REQUIRE(n_records >= 0 && n_records <= FE_MAX_RECORDS, "n_records must be 0..64");
  if (n_records == 0) return OSB_OK;
  OSB_REQUIRE(records_dev && results_dev, "null argument");
  unsigned long long mask = 0;
  if (init_mode)
    for (int r = 0; r < n_records; ++r) mask |= (init_mode[r] ? 1ull : 0ull) << r;
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  return fe_query_received(h, records_dev, n_records, skip, mask, results_dev, (cudaStream_t)stream);
}

extern "C" osb_status osb_frontend_set_loop_params(osb_frontend* h, const osb_loop_params* p) {
  OSB_REQUIRE(h && p, "null argument");
  OSB_REQUIRE(p->min_loop_num >= 0 && p->init_mode_min_loop_num >= 0 && p->min_match_per_dir >= 0 &&
              p->min_direction_loop >= 0, "negative count threshold");
  OSB_REQUIRE(p->reproj_thresh > 0.f, "reproj_thresh must be positive");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  OSB_TRY(fe_refresh_counts(h, h->stream));
  // rows ingested so far carry no 3-D landmarks: the plane would hand stale points to a swapped edge
  OSB_REQUIRE(h->db[1].upper == 0, "the remote store already holds rows: set the loop parameters before the first ingest");
  DbStore& R = h->db[1];
  if (!R.v.l3d) OSB_TRY(h->res.alloc(&R.v.l3d, (size_t)R.cap * h->cfg.max_num * 3));
  h->loop_params = *p;
  h->have_loop_params = true;
  return OSB_OK;
}

// compute_loop's scratch for LC_MAX candidates (about 1 MB), acquired once by its first call
static osb_status fe_lc_alloc(osb_frontend* h) {
  if (h->lc_ready) return OSB_OK;
  Resources& m = h->res;
  OSB_TRY(m.alloc(&h->d_lc_pts3d, (size_t)LC_MAX * LC_MAXN * 3));
  OSB_TRY(m.alloc(&h->d_lc_pts2d, (size_t)LC_MAX * LC_MAXN * 2));
  OSB_TRY(m.alloc(&h->d_lc_n, LC_MAX));
  OSB_TRY(m.alloc(&h->d_lc_params, LC_MAX));
  OSB_TRY(m.alloc(&h->d_lc_mask, (size_t)LC_MAX * LC_MAXN));
  OSB_TRY(m.alloc(&h->d_lc_pnp, LC_MAX));
  h->lc_ready = true;
  return OSB_OK;
}

// the handle's state compute_loop needs (under h->mu)
static osb_status fe_compute_loop_ready(osb_frontend* h) {
  OSB_REQUIRE(h->have_loop_params, "no loop parameters: call osb_frontend_set_loop_params first");
  OSB_REQUIRE(h->cfg.geometric_filter != 0, "compute_loop needs geometric_filter = 1 (the reference's USE_FUNDMENTAL path)");
  OSB_REQUIRE(h->have_cameras != h->have_depth_camera,
              "compute_loop needs the old frame's camera: exactly one of set_cameras / set_depth_camera");
  return fe_lc_alloc(h);
}

// assemble -> PnP-RANSAC -> finalise for n candidates read from `cands` (LoopCandBatch or LoopCandPtr)
template <class Cands>
static osb_status fe_compute_loop(osb_frontend* h, const osb_keyframe_record* records_dev, const osb_loop_result* results_dev,
                                  int n, const Cands& cands, osb_loop_edge_result* out_dev, cudaStream_t st) {
  LoopCams cam{};
  const bool depth = h->have_depth_camera;
  for (int i = 0; i < 4; ++i) cam.K[i] = depth ? h->depth_K[i] : h->K[i];
  for (int d = 0; d < OSB_MAX_DIRS; ++d)
    for (int i = 0; i < 7; ++i)       // the main camera's extrinsic is the direction's camera_extrinsic (loop_cam.cpp:372)
      cam.ext[d][i] = d < h->cfg.n_dirs ? (depth ? h->depth_ext[d][i] : h->main_down ? h->right_ext[d][i] : h->left_ext[d][i])
                                        : (i == 3 ? 1.0 : 0.0);
  OSB_LAUNCH(lc_assemble_kernel<Cands>, n, 256, 0, st, records_dev, results_dev, fe_stores(h), cands, cam, h->loop_params,
             h->cfg.query_dir, h->cfg.max_num, out_dev, h->d_lc_pts3d, h->d_lc_pts2d, h->d_lc_n, h->d_lc_params);
  OSB_CHECK_LAUNCH();
  OSB_LAUNCH(pnp_ransac_kernel, n, PNP_THREADS, 0, st, h->d_lc_pts3d, h->d_lc_pts2d, h->d_lc_n, LC_MAXN, h->d_lc_params,
             h->d_lc_mask, h->d_lc_pnp);
  OSB_CHECK_LAUNCH();
  OSB_LAUNCH(lc_finalise_kernel, n, 256, 0, st, h->d_lc_mask, h->d_lc_pnp, h->d_lc_params, out_dev);
  OSB_CHECK_LAUNCH();
  return OSB_OK;
}

extern "C" osb_status osb_frontend_compute_loop(osb_frontend* h, const osb_keyframe_record* records_dev,
                                                const osb_loop_result* results_dev, int n, const osb_loop_candidate* cand,
                                                osb_loop_edge_result* out_dev, void* stream) {
  OSB_REQUIRE(h != nullptr, "null handle");
  OSB_REQUIRE(n >= 1 && n <= LC_MAX, "n must be 1..64");
  OSB_REQUIRE(records_dev && results_dev && cand && out_dev, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  OSB_TRY(fe_compute_loop_ready(h));
  DeviceGuard dg(h->device);
  LoopCandBatch cb;
  memset(&cb, 0, sizeof(cb));
  memcpy(cb.c, cand, (size_t)n * sizeof(osb_loop_candidate));
  return fe_compute_loop(h, records_dev, results_dev, n, cb, out_dev, (cudaStream_t)stream);
}

extern "C" osb_status osb_frontend_compute_loop_dev(osb_frontend* h, const osb_keyframe_record* records_dev,
                                                    const osb_loop_result* results_dev, int n,
                                                    const osb_loop_candidate* cand_dev, osb_loop_edge_result* out_dev,
                                                    void* stream) {
  OSB_REQUIRE(h != nullptr, "null handle");
  OSB_REQUIRE(n >= 1 && n <= LC_MAX, "n must be 1..64");
  OSB_REQUIRE(records_dev && results_dev && cand_dev && out_dev, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  OSB_TRY(fe_compute_loop_ready(h));
  DeviceGuard dg(h->device);
  return fe_compute_loop(h, records_dev, results_dev, n, LoopCandPtr{cand_dev}, out_dev, (cudaStream_t)stream);
}

// loop_count and inter_drone_loop_count on the device, acquired zero by the first call that needs them
static osb_status fe_lm_alloc(osb_frontend* h, cudaStream_t st) {
  if (h->d_lm_count) return OSB_OK;
  Resources& m = h->res;
  OSB_TRY(m.alloc(&h->d_lm_count, 1));
  OSB_TRY(m.alloc(&h->d_lm_pairs, (size_t)LM_PAIR_DRONES * LM_PAIR_DRONES));
  OSB_TRY(m.event(&h->ev_lm, cudaEventDisableTiming));
  OSB_CUDA(cudaMemsetAsync(h->d_lm_count, 0, sizeof(long long), st));
  OSB_CUDA(cudaMemsetAsync(h->d_lm_pairs, 0, (size_t)LM_PAIR_DRONES * LM_PAIR_DRONES * sizeof(int32_t), st));
  return OSB_OK;
}

// the rows of a round from `b` (LoopMeasBatch or LoopMeasPtr)
template <class Meas>
static osb_status fe_loop_measurements(osb_frontend* h, const osb_loop_result* results_dev, const osb_loop_edge_result* edges_dev,
                                       int n, const Meas& b, double loop_cov_pos, double loop_cov_ang, osb_measurement* out_dev,
                                       int32_t* count_dev, cudaStream_t st) {
  OSB_TRY(fe_lm_alloc(h, st));
  OSB_LAUNCH(lm_emit_kernel<Meas>, 1, 256, 0, st, results_dev, edges_dev, n, b, h->cfg.self_id, loop_cov_pos, loop_cov_ang,
             out_dev, count_dev, h->d_lm_count, h->d_lm_pairs);
  OSB_CHECK_LAUNCH();
  OSB_CUDA(record_event_capturable(h->ev_lm, st));
  return OSB_OK;
}

extern "C" osb_status osb_frontend_loop_measurements(osb_frontend* h, const osb_loop_result* results_dev,
                                                     const osb_loop_edge_result* edges_dev, int n,
                                                     const osb_loop_candidate* cand, const osb_loop_stamps* stamps,
                                                     double loop_cov_pos, double loop_cov_ang, osb_measurement* out_dev,
                                                     int32_t* count_dev, void* stream) {
  OSB_REQUIRE(h != nullptr, "null handle");
  OSB_REQUIRE(n >= 0 && n <= LC_MAX, "n must be 0..64");
  OSB_REQUIRE(out_dev && count_dev && (n == 0 || (results_dev && edges_dev && cand && stamps)), "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  LoopMeasBatch b;
  memset(&b, 0, sizeof(b));
  for (int i = 0; i < n; ++i) {
    memcpy(b.pose_query[i], cand[i].pose_query, sizeof(b.pose_query[i]));
    memcpy(b.pose_hit[i], cand[i].pose_hit, sizeof(b.pose_hit[i]));
    b.stamp_query[i] = stamps[i].stamp_query_ns;
    b.stamp_hit[i] = stamps[i].stamp_hit_ns;
  }
  return fe_loop_measurements(h, results_dev, edges_dev, n, b, loop_cov_pos, loop_cov_ang, out_dev, count_dev,
                              (cudaStream_t)stream);
}

extern "C" osb_status osb_frontend_loop_measurements_dev(osb_frontend* h, const osb_loop_result* results_dev,
                                                         const osb_loop_edge_result* edges_dev, int n,
                                                         const osb_loop_candidate* cand_dev, const osb_loop_stamps* stamps_dev,
                                                         double loop_cov_pos, double loop_cov_ang, osb_measurement* out_dev,
                                                         int32_t* count_dev, void* stream) {
  OSB_REQUIRE(h != nullptr, "null handle");
  OSB_REQUIRE(n >= 0 && n <= LC_MAX, "n must be 0..64");
  OSB_REQUIRE(out_dev && count_dev && (n == 0 || (results_dev && edges_dev && cand_dev && stamps_dev)), "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  return fe_loop_measurements(h, results_dev, edges_dev, n, LoopMeasPtr{cand_dev, stamps_dev}, loop_cov_pos, loop_cov_ang,
                              out_dev, count_dev, (cudaStream_t)stream);
}

extern "C" osb_status osb_frontend_loop_counts(osb_frontend* h, int64_t* loop_count, int32_t* pair_counts) {
  OSB_REQUIRE(h != nullptr && loop_count != nullptr, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  const size_t pair_bytes = (size_t)LM_PAIR_DRONES * LM_PAIR_DRONES * sizeof(int32_t);
  if (!h->d_lm_count) {                                    // no call yet: both counters are zero
    *loop_count = 0;
    if (pair_counts) memset(pair_counts, 0, pair_bytes);
    return OSB_OK;
  }
  DeviceGuard dg(h->device);
  cudaStream_t st = h->stream;
  OSB_CUDA(cudaStreamWaitEvent(st, h->ev_lm, 0));
  long long cnt = 0;
  OSB_CUDA(cudaMemcpyAsync(&cnt, h->d_lm_count, sizeof(long long), cudaMemcpyDeviceToHost, st));
  if (pair_counts) OSB_CUDA(cudaMemcpyAsync(pair_counts, h->d_lm_pairs, pair_bytes, cudaMemcpyDeviceToHost, st));
  OSB_CUDA(cudaStreamSynchronize(st));
  *loop_count = cnt;
  return OSB_OK;
}

// exact host-side row counts.  The counts are read on `st`, which need not be the stream that carried the last ingest
// (streams are non-blocking): wait for that ingest first, or the bound could be lowered below the true count while the
// rows are still being appended -- the scan grid is sized from it.
static osb_status fe_refresh_counts(osb_frontend* h, cudaStream_t st) {
  if (h->fb.pending) OSB_CUDA(cudaStreamWaitEvent(st, h->fb.ev, 0));
  OSB_CUDA(cudaMemcpyAsync(&h->h_cnt[0], h->db[0].v.dev, sizeof(DbDev), cudaMemcpyDeviceToHost, st));
  OSB_CUDA(cudaMemcpyAsync(&h->h_cnt[1], h->db[1].v.dev, sizeof(DbDev), cudaMemcpyDeviceToHost, st));
  OSB_CUDA(cudaStreamSynchronize(st));
  h->db[0].upper = h->h_cnt[0].ntotal; h->db[1].upper = h->h_cnt[1].ntotal;
  h->fb.pending = false;
  h->fb.exact();
  return OSB_OK;
}

// the rest of a single-drone step after extract wrote h->d_record: ingest (own), query, copies to the host, and the one
// synchronisation of the keyframe
static osb_status fe_process_tail(osb_frontend* h, osb_keyframe_record* record_host, osb_loop_result* result_host,
                                  cudaStream_t st) {
  osb_status s;
  if ((s = fe_ingest(h, h->d_record, 1, -1, st, 1)) != OSB_OK) return s;   // add_to_database (loop_detector.cpp:89): own record
  if ((s = fe_query(h, h->d_record, 0, 0, h->d_result, st)) != OSB_OK) return s;
  if (record_host) OSB_CUDA(cudaMemcpyAsync(record_host, h->d_record, sizeof(osb_keyframe_record), cudaMemcpyDeviceToHost, st));
  if (result_host) OSB_CUDA(cudaMemcpyAsync(result_host, h->d_result, sizeof(osb_loop_result), cudaMemcpyDeviceToHost, st));
  return fe_refresh_counts(h, st);
}

extern "C" osb_status osb_frontend_process(osb_frontend* h, const uint8_t* images_up, const uint8_t* images_down,
                                           int32_t msg_id, osb_keyframe_record* record_host,
                                           osb_loop_result* result_host) {
  OSB_REQUIRE(h && images_up && images_down, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  cudaStream_t st = h->stream;
  osb_status s;
  if ((s = fe_extract_stereo(h, images_up, images_down, cudaMemcpyHostToDevice, msg_id, h->d_record, st)) != OSB_OK) return s;
  return fe_process_tail(h, record_host, result_host, st);
}

extern "C" osb_status osb_frontend_process_depth(osb_frontend* h, const uint8_t* images, const uint16_t* depth_mm,
                                                 int32_t msg_id, osb_keyframe_record* record_host,
                                                 osb_loop_result* result_host) {
  OSB_REQUIRE(h && images && depth_mm, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  OSB_REQUIRE(!h->main_down, "a depth keyframe has no lower camera: the main camera must be OSB_MAIN_CAMERA_UP");
  OSB_REQUIRE(h->have_depth_camera, "no depth camera: call osb_frontend_set_depth_camera first");
  DeviceGuard dg(h->device);
  cudaStream_t st = h->stream;
  osb_status s;
  if ((s = fe_extract_depth(h, images, depth_mm, cudaMemcpyHostToDevice, msg_id, h->d_record, st)) != OSB_OK) return s;
  return fe_process_tail(h, record_host, result_host, st);
}

extern "C" osb_status osb_frontend_set_depth_camera(osb_frontend* h, const double* intrinsics, const double* extrinsics,
                                                    double near_thres, double far_thres) {
  OSB_REQUIRE(h && intrinsics && extrinsics, "null argument");
  OSB_REQUIRE(intrinsics[0] > 0 && intrinsics[1] > 0, "bad intrinsics");
  OSB_REQUIRE(near_thres < far_thres, "near_thres must be below far_thres");
  std::lock_guard<std::mutex> lk(h->mu);
  // PINHOLE_DEPTH with LOWER_CAM_AS_MAIN runs SuperPoint only and makes no global descriptor (loop_cam.cpp:241)
  OSB_REQUIRE(!h->main_down, "a depth camera cannot be set on a handle whose main camera is OSB_MAIN_CAMERA_DOWN");
  DeviceGuard dg(h->device);
  if (!h->d_depth) OSB_TRY(h->res.alloc(&h->d_depth, (size_t)h->cfg.n_dirs * h->cfg.width * h->cfg.height));
  for (int i = 0; i < 4; ++i) h->depth_K[i] = intrinsics[i];
  for (int d = 0; d < h->cfg.n_dirs; ++d)
    for (int i = 0; i < 7; ++i) h->depth_ext[d][i] = extrinsics[d * 7 + i];
  h->near_thres = near_thres; h->far_thres = far_thres;
  h->have_depth_camera = true;
  return OSB_OK;
}

extern "C" osb_status osb_frontend_set_cameras(osb_frontend* h, const double* intrinsics, const double* left_extrinsics,
                                               const double* right_extrinsics, double triangle_thres) {
  OSB_REQUIRE(h && intrinsics && left_extrinsics && right_extrinsics, "null argument");
  OSB_REQUIRE(intrinsics[0] > 0 && intrinsics[1] > 0 && triangle_thres > 0, "bad intrinsics / threshold");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  for (int i = 0; i < 4; ++i) h->K[i] = intrinsics[i];
  for (int d = 0; d < h->cfg.n_dirs; ++d)
    for (int i = 0; i < 7; ++i) { h->left_ext[d][i] = left_extrinsics[d * 7 + i]; h->right_ext[d][i] = right_extrinsics[d * 7 + i]; }
  h->triangle_thres = triangle_thres;
  h->have_cameras = true;
  return OSB_OK;
}

// LOWER_CAM_AS_MAIN (swarm_loop.cpp:243) from the next extract on; allocates nothing
extern "C" osb_status osb_frontend_set_main_camera(osb_frontend* h, int which) {
  OSB_REQUIRE(h != nullptr, "null handle");
  OSB_REQUIRE(which == OSB_MAIN_CAMERA_UP || which == OSB_MAIN_CAMERA_DOWN, "which must be OSB_MAIN_CAMERA_UP or _DOWN");
  std::lock_guard<std::mutex> lk(h->mu);
  OSB_REQUIRE(!h->have_depth_camera, "a depth-camera handle has no stereo pair to choose the main camera of");
  h->main_down = which == OSB_MAIN_CAMERA_DOWN;
  return OSB_OK;
}

extern "C" osb_status osb_frontend_set_drone_pose(osb_frontend* h, const double* pose_drone) {
  OSB_REQUIRE(h && pose_drone, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  for (int i = 0; i < 7; ++i) h->pose_drone[i] = pose_drone[i];
  return OSB_OK;
}

extern "C" osb_status osb_frontend_set_profiling(osb_frontend* h, int enable) {
  OSB_REQUIRE(h != nullptr, "null handle");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  h->profiling = enable != 0;
  for (int i = 0; i < 9; ++i) h->ev_valid[i] = false;
  return OSB_OK;
}

extern "C" osb_status osb_frontend_stage_ms(osb_frontend* h, float* ms8) {
  OSB_REQUIRE(h != nullptr && ms8 != nullptr, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  for (int i = 0; i < 8; ++i) {
    ms8[i] = 0.f;
    if (i < 7 && h->ev_valid[i] && h->ev_valid[i + 1]) {
      float t = 0.f;
      if (cudaEventElapsedTime(&t, h->ev[i], h->ev[i + 1]) == cudaSuccess) ms8[i] = t; else cudaGetLastError();
    }
  }
  return OSB_OK;
}

extern "C" osb_status osb_frontend_finish(osb_frontend* h, void* stream) {
  OSB_REQUIRE(h != nullptr, "null handle");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  return fe_refresh_counts(h, (cudaStream_t)stream);
}

extern "C" int64_t osb_frontend_db_size(osb_frontend* h, int remote) {
  if (!h) return -1;
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  if (fe_refresh_counts(h, h->stream) != OSB_OK) return -1;
  return h->db[remote ? 1 : 0].upper;
}

extern "C" osb_status osb_frontend_db_reset(osb_frontend* h) {
  OSB_REQUIRE(h != nullptr, "null handle");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  for (int i = 0; i < 2; ++i) {
    OSB_CUDA(cudaMemsetAsync(h->db[i].v.dev, 0, sizeof(DbDev), h->stream));
    OSB_CUDA(cudaMemsetAsync(h->db[i].v.top_ids, 0xFF, FE_KMAX * sizeof(int64_t), h->stream));
    h->db[i].upper = 0;
    if (h->meta_ready)                                     // the frames' metas go; the trajectory stays
      OSB_CUDA(cudaMemsetAsync(h->meta.ok[i], 0, (size_t)h->db[i].cap * sizeof(int32_t), h->stream));
  }
  h->fb.exact();
  OSB_CUDA(cudaStreamSynchronize(h->stream));
  return OSB_OK;
}

// landmarks_2d and stereo_match (>= 0 <=> landmarks_flag) of rows [first_row, first_row + n) that were put in with
// osb_frontend_db_load: the inputs of the geometric filter when such a row is the loop hit
extern "C" osb_status osb_frontend_db_set_geometry(osb_frontend* h, int remote, int64_t first_row, int64_t n,
                                                   const float* kpts, const int32_t* stereo_match) {
  OSB_REQUIRE(h && kpts && stereo_match && n >= 0 && first_row >= 0, "bad arguments");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  cudaStream_t st = h->stream;
  if (fe_refresh_counts(h, st) != OSB_OK) return OSB_ERR_CUDA;
  const DbStore& S = h->db[remote ? 1 : 0];
  OSB_REQUIRE(first_row + n <= S.upper, "rows out of range");
  const int mn = h->cfg.max_num;
  OSB_CUDA(cudaMemcpyAsync(S.v.kpts + (size_t)first_row * mn * 2, kpts, (size_t)n * mn * 2 * sizeof(float),
                           cudaMemcpyHostToDevice, st));
  std::vector<int32_t> flags((size_t)n * mn);
  for (size_t i = 0; i < flags.size(); ++i) flags[i] = stereo_match[i] >= 0 ? 1 : 0;       // landmarks_flag of the rows
  OSB_CUDA(cudaMemcpyAsync(S.v.lflag + (size_t)first_row * mn, flags.data(), flags.size() * sizeof(int32_t),
                           cudaMemcpyHostToDevice, st));
  OSB_CUDA(cudaStreamSynchronize(st));
  return OSB_OK;
}

extern "C" osb_status osb_frontend_db_load(osb_frontend* h, int remote, int64_t n, const float* global_desc,
                                           const float* local_desc, const int32_t* n_kpts) {
  OSB_REQUIRE(h && global_desc && n >= 0, "bad arguments");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  cudaStream_t st = h->stream;
  if (fe_refresh_counts(h, st) != OSB_OK) return OSB_ERR_CUDA;
  DbStore& S = h->db[remote ? 1 : 0];
  const DbView& v = S.v;
  const int64_t base = S.upper;
  if (base + n > S.cap) { set_error("osb_frontend_db_load", "database capacity exceeded"); return OSB_ERR_CAPACITY; }
  const int mn = h->cfg.max_num, qd = h->cfg.query_dir;
  DbDev hd;
  OSB_CUDA(cudaMemcpy(&hd, v.dev, sizeof(DbDev), cudaMemcpyDeviceToHost));
  // the frame tables are [cap] too, and a keyframe without keypoints adds a frame but no row (nframes may exceed ntotal)
  if ((int64_t)hd.nframes + n > S.cap) { set_error("osb_frontend_db_load", "frame table capacity exceeded"); return OSB_ERR_CAPACITY; }
  if (v.storage == OSB_DB_STORAGE_FP16) {
    if (!h->d_load_stage) OSB_TRY(h->res.alloc(&h->d_load_stage, (size_t)FE_LOAD_ROWS * OSB_DEEP_DESC_SIZE));
    for (int64_t r0 = 0; r0 < n; r0 += FE_LOAD_ROWS) {    // stream order protects the staging buffer's reuse
      const size_t e = (size_t)std::min<int64_t>(FE_LOAD_ROWS, n - r0) * OSB_DEEP_DESC_SIZE;
      OSB_CUDA(cudaMemcpyAsync(h->d_load_stage, global_desc + (size_t)r0 * OSB_DEEP_DESC_SIZE, e * sizeof(float),
                               cudaMemcpyHostToDevice, st));
      OSB_TRY(db_rows_to_half(static_cast<__half*>(v.rows) + (size_t)(base + r0) * OSB_DEEP_DESC_SIZE, h->d_load_stage, e,
                              st));
    }
  } else {
    OSB_CUDA(cudaMemcpyAsync(static_cast<float*>(v.rows) + (size_t)base * OSB_DEEP_DESC_SIZE, global_desc,
                             (size_t)n * OSB_DEEP_DESC_SIZE * sizeof(float), cudaMemcpyHostToDevice, st));
  }
  std::vector<int32_t> nk(n), rf(n), rd(n), fr((size_t)n * OSB_MAX_DIRS, -1), fm(n, -1);
  for (int64_t i = 0; i < n; ++i) {
    nk[i] = (local_desc && n_kpts) ? std::min(n_kpts[i], mn) : 0;
    rf[i] = hd.nframes + (int)i; rd[i] = qd;
    fr[(size_t)i * OSB_MAX_DIRS + qd] = (int32_t)(base + i);
  }
  if (local_desc)
    OSB_CUDA(cudaMemcpyAsync(v.ldesc + (size_t)base * mn * OSB_FEATURE_DESC_SIZE, local_desc,
                             (size_t)n * mn * OSB_FEATURE_DESC_SIZE * sizeof(float), cudaMemcpyHostToDevice, st));
  // rows loaded without geometry: landmarks at the origin, every landmark flagged (osb_frontend_db_set_geometry fills them)
  OSB_CUDA(cudaMemsetAsync(v.kpts + (size_t)base * mn * 2, 0, (size_t)n * mn * 2 * sizeof(float), st));
  OSB_CUDA(cudaMemsetAsync(v.lflag + (size_t)base * mn, 1, (size_t)n * mn * sizeof(int32_t), st));
  OSB_CUDA(cudaMemcpyAsync(v.nk + base, nk.data(), n * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  OSB_CUDA(cudaMemcpyAsync(v.row_frame + base, rf.data(), n * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  OSB_CUDA(cudaMemcpyAsync(v.row_dir + base, rd.data(), n * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  OSB_CUDA(cudaMemcpyAsync(v.frame_rows + (size_t)hd.nframes * OSB_MAX_DIRS, fr.data(), fr.size() * sizeof(int32_t),
                           cudaMemcpyHostToDevice, st));
  OSB_CUDA(cudaMemcpyAsync(v.frame_msg + hd.nframes, fm.data(), n * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  std::vector<int32_t> fd(n, remote ? -1 : h->cfg.self_id);
  OSB_CUDA(cudaMemcpyAsync(v.frame_drone + hd.nframes, fd.data(), n * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  hd.ntotal += n; hd.nframes += (int)n;
  OSB_CUDA(cudaMemcpyAsync(v.dev, &hd, sizeof(DbDev), cudaMemcpyHostToDevice, st));
  OSB_CUDA(cudaStreamSynchronize(st));
  S.upper = hd.ntotal;
  return OSB_OK;
}

// ---- keyframe metadata and a round's loop candidates on the device -----------------------------------------------------
// both stores' meta tables and the trajectory, acquired zero by the first meta ingest (db_capacity frames / samples each)
static osb_status fe_meta_alloc(osb_frontend* h, cudaStream_t st) {
  if (h->meta_ready) return OSB_OK;
  Resources& m = h->res;
  FeMeta& mt = h->meta;
  const size_t cap = (size_t)h->cfg.db_capacity;
  for (int i = 0; i < 2; ++i) {
    OSB_TRY(m.alloc(&mt.meta[i], cap));
    OSB_TRY(m.alloc(&mt.ok[i], cap));
    OSB_CUDA(cudaMemsetAsync(mt.ok[i], 0, cap * sizeof(int32_t), st));
  }
  OSB_TRY(m.alloc(&mt.t_stamp, cap));
  OSB_TRY(m.alloc(&mt.t_pose, cap * 7));
  OSB_TRY(m.alloc(&mt.t_len, cap));
  OSB_TRY(m.alloc(&mt.dev, 1));
  OSB_TRY(m.host_alloc(&h->h_meta, 1, cudaHostAllocDefault));
  OSB_CUDA(cudaMemsetAsync(mt.dev, 0, sizeof(FeMetaDev), st));
  mt.t_cap = (int)cap;
  h->meta_ready = true;
  return OSB_OK;
}

extern "C" osb_status osb_frontend_ingest_meta(osb_frontend* h, const osb_keyframe_record* records_dev,
                                               const osb_keyframe_meta* metas_dev, int n_records, int skip, void* stream) {
  OSB_REQUIRE(h && records_dev && metas_dev, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  OSB_TRY(fe_meta_alloc(h, (cudaStream_t)stream));
  return fe_ingest(h, records_dev, n_records, skip, (cudaStream_t)stream, 0, metas_dev);
}

extern "C" osb_status osb_frontend_ingest_own_meta(osb_frontend* h, const osb_keyframe_record* record_dev,
                                                   const osb_keyframe_meta* meta_dev, void* stream) {
  OSB_REQUIRE(h && record_dev && meta_dev, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  OSB_TRY(fe_meta_alloc(h, (cudaStream_t)stream));
  return fe_ingest(h, record_dev, 1, -1, (cudaStream_t)stream, 1, meta_dev);
}

extern "C" osb_status osb_frontend_meta_status(osb_frontend* h, osb_status* last) {
  OSB_REQUIRE(h && last, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  *last = OSB_OK;
  if (!h->meta_ready) return OSB_OK;
  DeviceGuard dg(h->device);
  cudaStream_t st = h->stream;
  if (h->fb.pending) OSB_CUDA(cudaStreamWaitEvent(st, h->fb.ev, 0));
  OSB_CUDA(cudaMemcpyAsync(h->h_meta, h->meta.dev, sizeof(FeMetaDev), cudaMemcpyDeviceToHost, st));
  OSB_CUDA(cudaStreamSynchronize(st));
  *last = (osb_status)h->h_meta->status;
  return *last;
}

extern "C" osb_status osb_frontend_set_candidate_params(osb_frontend* h, const osb_candidate_params* p) {
  OSB_REQUIRE(h && p, "null argument");
  OSB_REQUIRE(p->pos_covariance_per_meter >= 0 && p->yaw_covariance_per_meter >= 0 && p->loop_cov_pos >= 0 &&
              p->loop_cov_ang >= 0, "negative covariance");
  std::lock_guard<std::mutex> lk(h->mu);
  h->cand_params = *p;
  h->have_cand_params = true;
  return OSB_OK;
}

static CandRule fe_cand_rule(const osb_frontend* h) {
  const osb_candidate_params& p = h->cand_params;
  return CandRule{h->cfg.self_id, p.inter_drone_init_frames, p.pos_covariance_per_meter, p.yaw_covariance_per_meter,
                  p.loop_cov_pos, p.loop_cov_ang};
}

extern "C" osb_status osb_frontend_init_modes_dev(osb_frontend* h, const osb_keyframe_record* records_dev, int n_records,
                                                  int skip, uint8_t* init_mode_out_dev, void* stream) {
  OSB_REQUIRE(h != nullptr, "null handle");
  OSB_REQUIRE(n_records >= 0 && n_records <= FE_MAX_RECORDS, "n_records must be 0..64");
  OSB_REQUIRE(records_dev && init_mode_out_dev, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  OSB_REQUIRE(h->have_cand_params, "no candidate parameters: call osb_frontend_set_candidate_params first");
  if (n_records == 0) return OSB_OK;
  DeviceGuard dg(h->device);
  cudaStream_t st = (cudaStream_t)stream;
  OSB_TRY(fe_lm_alloc(h, st));
  OSB_LAUNCH(fe_init_modes_kernel, 1, FE_MAX_RECORDS, 0, st, records_dev, n_records, skip, fe_cand_rule(h), h->d_lm_pairs,
             init_mode_out_dev);
  OSB_CHECK_LAUNCH();
  return OSB_OK;
}

extern "C" osb_status osb_frontend_receive_dev(osb_frontend* h, const osb_keyframe_record* records_dev, int n_records,
                                               int skip, osb_keyframe_record* out_dev, void* stream) {
  OSB_REQUIRE(h != nullptr, "null handle");
  OSB_REQUIRE(n_records >= 0 && n_records <= FE_MAX_RECORDS, "n_records must be 0..64");
  std::lock_guard<std::mutex> lk(h->mu);
  OSB_REQUIRE(h->have_loop_params, "no loop parameters: call osb_frontend_set_loop_params first");
  if (n_records == 0) return OSB_OK;
  OSB_REQUIRE(records_dev && out_dev, "null argument");
  const uintptr_t a = (uintptr_t)records_dev, b = (uintptr_t)out_dev, len = (uintptr_t)n_records * sizeof(osb_keyframe_record);
  OSB_REQUIRE(a + len <= b || b + len <= a, "out_dev overlaps records_dev");
  OSB_REQUIRE(a % 16 == 0 && b % 16 == 0, "records_dev and out_dev must be 16-byte aligned");
  DeviceGuard dg(h->device);
  OSB_LAUNCH(fe_receive_kernel, n_records * OSB_MAX_DIRS, FE_RECV_THREADS, 0, (cudaStream_t)stream, records_dev, out_dev, skip,
             h->cfg.self_id, h->loop_params.min_direction_loop, h->loop_params.min_loop_num, h->db[0].v.dev, h->db[1].v.dev);
  OSB_CHECK_LAUNCH();
  return OSB_OK;
}

extern "C" osb_status osb_frontend_query_received_dev(osb_frontend* h, const osb_keyframe_record* records_dev, int n_records,
                                                      int skip, const uint8_t* init_mode_dev, osb_loop_result* results_dev,
                                                      void* stream) {
  OSB_REQUIRE(h != nullptr, "null handle");
  OSB_REQUIRE(n_records >= 0 && n_records <= FE_MAX_RECORDS, "n_records must be 0..64");
  if (n_records == 0) return OSB_OK;
  OSB_REQUIRE(records_dev && results_dev, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  return fe_query_received(h, records_dev, n_records, skip, 0ull, results_dev, (cudaStream_t)stream, true, init_mode_dev);
}

extern "C" osb_status osb_frontend_loop_candidates_dev(osb_frontend* h, const osb_keyframe_record* records_dev,
                                                       const osb_keyframe_meta* metas_dev, const osb_loop_result* results_dev,
                                                       int n, const uint8_t* init_mode_dev, osb_loop_candidate* cand_out_dev,
                                                       osb_loop_stamps* stamps_out_dev, void* stream) {
  OSB_REQUIRE(h != nullptr, "null handle");
  OSB_REQUIRE(n >= 0 && n <= LC_MAX, "n must be 0..64");
  OSB_REQUIRE(n == 0 || (records_dev && metas_dev && results_dev && cand_out_dev && stamps_out_dev), "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  OSB_REQUIRE(h->have_cand_params, "no candidate parameters: call osb_frontend_set_candidate_params first");
  if (n == 0) return OSB_OK;
  DeviceGuard dg(h->device);
  cudaStream_t st = (cudaStream_t)stream;
  OSB_TRY(fe_meta_alloc(h, st));                           // a handle without meta ingests: every hit lacks its meta
  OSB_TRY(fe_lm_alloc(h, st));
  OSB_LAUNCH(lc_candidates_kernel, 1, LC_MAX, 0, st, records_dev, metas_dev, results_dev, n, init_mode_dev, fe_stores(h),
             h->meta, h->d_lm_pairs, fe_cand_rule(h), cand_out_dev, stamps_out_dev);
  OSB_CHECK_LAUNCH();
  return OSB_OK;
}
