/* ORACLE (test infrastructure): a single-threaded C restatement of the re-anchoring walk of
 * SwarmLocalizationSolver::find_available_loops_detections (swarm_localization_solver.cpp:1594-1666), with the reference's
 * loop structure: for every measurement, frames in order and a look-up of the drone in each frame
 * (find_node_frame_for_measurement_2drones, :1429-1462), then loop_from_src_loop_connection (:1464-1553) and the factor row
 * of setup_problem_with_loops_and_detections (:1064-1100).  The definitions of the swarm_msgs arithmetic are those of
 * oracle/anchor_ref.py; the record layouts are those of osb_measurement / osb_window_entry / osb_anchor_result.
 * It is the CPU baseline of scripts/bench_anchor.py. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

enum { LOOP = 0, DET4D = 1, DET6D = 2 };
enum { OK = 0, EMPTY_WINDOW, BEFORE_WINDOW, NO_FRAME, NO_TRAJECTORY, DPOS };
#define MIN_TS_ERR_START_NS (10000ll * 1000000000ll)

typedef struct {
  int64_t id;
  int32_t type, id_a, id_b, reserved;
  int64_t stamp_a, stamp_b;
  double relative_pose[7], cov[36], self_pose_a[7], self_pose_b[7];
} meas_t;
typedef struct {
  int32_t drone_id, vo_available, block, reserved;
  int64_t stamp;
  double self_pose[7];
} entry_t;
typedef struct {
  int32_t id_a, id_b;
  double rel_pose[7], cov[36], odom_a[7], odom_b[7], len_a, len_b;
} edge_t;
typedef struct {
  int64_t id;
  int32_t type, status, frame_a, frame_b, node_a, node_b;
  int64_t stamp_a, stamp_b, dt_err_ns;
  double dpos;
  edge_t edge;
  int32_t skip, factor_type, ia, ib, huber, reserved;
  double payload[24];
} result_t;
typedef struct {
  double begin_min_loop_dt_s, det_dpos_thres, odom_pos_cov_per_m, odom_ang_cov_per_m;
  int32_t huber, reserved;
} params_t;

/* ---- Swarm::Pose algebra (oracle/pcm_ref.py, oracle/pnp_ref.py) ---- */
static void q_mul(const double* a, const double* b, double* o) {
  o[0] = a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3];
  o[1] = a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2];
  o[2] = a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1];
  o[3] = a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0];
}
static void pose_mul(const double* a, const double* b, double* o) {
  const double* q = a + 3;
  const double* v = b;
  const double cx = q[2] * v[2] - q[3] * v[1], cy = q[3] * v[0] - q[1] * v[2], cz = q[1] * v[1] - q[2] * v[0];
  const double dx = q[2] * cz - q[3] * cy, dy = q[3] * cx - q[1] * cz, dz = q[1] * cy - q[2] * cx;
  o[0] = a[0] + (v[0] + 2.0 * (q[0] * cx + dx));
  o[1] = a[1] + (v[1] + 2.0 * (q[0] * cy + dy));
  o[2] = a[2] + (v[2] + 2.0 * (q[0] * cz + dz));
  q_mul(a + 3, b + 3, o + 3);
}
static double quat_yaw(const double* q) {
  return atan2(2.0 * (q[0] * q[3] + q[1] * q[2]), 1.0 - 2.0 * (q[2] * q[2] + q[3] * q[3]));
}
static void yaw_quat(double yaw, double* q) {        /* quat_from_rotvec([0, 0, yaw]) */
  const double a = sqrt(yaw * yaw);
  if (a < 1e-12) { q[0] = 1.0; q[1] = 0.0; q[2] = 0.0; q[3] = 0.5 * yaw; }
  else { const double s = sin(0.5 * a) / a; q[0] = cos(0.5 * a); q[1] = 0.0; q[2] = 0.0; q[3] = s * yaw; }
  const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  q[0] /= n; q[1] /= n; q[2] /= n; q[3] /= n;
}
static void delta_pose4(const double* a, const double* b, double* o) {
  const double ya = quat_yaw(a + 3), yb = quat_yaw(b + 3);
  const double d0 = b[0] - a[0], d1 = b[1] - a[1], d2 = b[2] - a[2];
  const double c = cos(ya), s = sin(ya);
  const double pi = 3.141592653589793;
  const double dy = yb - ya;
  o[0] = c * d0 + s * d1;
  o[1] = -s * d0 + c * d1;
  o[2] = d2;
  yaw_quat(dy - 2.0 * pi * floor((dy + pi) / (2.0 * pi)), o + 3);
}
static void sqrt_information_4d(const double* cov, double* S) {
  double A[4][8];
  memset(A, 0, sizeof(A));
  for (int i = 0; i < 4; ++i) A[i][4 + i] = 1.0;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) A[i][j] = cov[i * 6 + j];
  A[3][3] = cov[35];
  for (int c = 0; c < 4; ++c) {
    int p = c;
    for (int r = c + 1; r < 4; ++r)
      if (fabs(A[r][c]) > fabs(A[p][c])) p = r;
    if (p != c)
      for (int j = 0; j < 8; ++j) { const double x = A[c][j]; A[c][j] = A[p][j]; A[p][j] = x; }
    const double piv = A[c][c];
    for (int j = 0; j < 8; ++j) A[c][j] /= piv;
    for (int r = 0; r < 4; ++r) {
      if (r == c) continue;
      const double f = A[r][c];
      for (int j = 0; j < 8; ++j) A[r][j] -= f * A[c][j];
    }
  }
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) S[i * 4 + j] = sqrt(fabs(A[i][4 + j]));
}

/* ---- DroneTrajectory: samples [traj_first[d], traj_first[d+1]) of the flat arrays ---- */
static int64_t nearest(const int64_t* s, int64_t n, int64_t t) {
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    const int64_t mid = (lo + hi) / 2;
    if (s[mid] < t) lo = mid + 1; else hi = mid;
  }
  if (lo == 0) return 0;
  if (lo == n) return n - 1;
  return (t - s[lo - 1]) <= (s[lo] - t) ? lo - 1 : lo;
}

static int64_t labs64(int64_t x) { return x < 0 ? -x : x; }

/* -> number of results written (n_meas), loops first */
int osb_ref_anchor(const params_t* prm, int n_drones, const int64_t* traj_first, const int64_t* traj_stamp,
                   const double* traj_pose, const double* traj_len, int n_frames, const int64_t* frame_stamps,
                   const int32_t* frame_first, const entry_t* entries, int n_meas, const meas_t* meas,
                   const uint8_t* yaw_observable, result_t* out) {
  const int64_t begin_dt = llround(prm->begin_min_loop_dt_s * 1e9);
  int k = 0;
  for (int pass = 0; pass < 2; ++pass)                     /* all_loops, then all_detections_6d (:1600-1645) */
    for (int i = 0; i < n_meas; ++i) {
      const meas_t* m = meas + i;
      if ((m->type == LOOP) != (pass == 0)) continue;
      result_t* r = out + k++;
      memset(r, 0, sizeof(*r));
      r->id = m->id;
      r->type = m->type;
      r->frame_a = r->frame_b = r->node_a = r->node_b = -1;
      r->factor_type = 1;
      r->huber = prm->huber ? 1 : 0;
      int status = OK;
      int ia = -1, ib = -1;
      const entry_t *nf_a = NULL, *nf_b = NULL;
      if (n_frames == 0) status = EMPTY_WINDOW;                                  /* :1479-1482 */
      else if (frame_stamps[0] - m->stamp_a > begin_dt) status = BEFORE_WINDOW;  /* :1484 */
      else {
        int64_t ea = MIN_TS_ERR_START_NS, eb = MIN_TS_ERR_START_NS;
        for (int f = 0; f < n_frames; ++f)                                       /* :1440-1452 */
          for (int e = frame_first[f]; e < frame_first[f + 1]; ++e) {
            const entry_t* en = entries + e;
            if (en->drone_id == m->id_a && en->vo_available && labs64(en->stamp - m->stamp_a) < ea) {
              ea = labs64(en->stamp - m->stamp_a); ia = f; nf_a = en;
            }
            if (en->drone_id == m->id_b && en->vo_available && labs64(en->stamp - m->stamp_b) < eb) {
              eb = labs64(en->stamp - m->stamp_b); ib = f; nf_b = en;
            }
          }
        r->dt_err_ns = ea + eb;
        if (nf_a) { r->frame_a = ia; r->node_a = nf_a->block; r->stamp_a = nf_a->stamp; }
        if (nf_b) { r->frame_b = ib; r->node_b = nf_b->block; r->stamp_b = nf_b->stamp; }
        if (!nf_a || !nf_b) status = NO_FRAME;
        else if (m->id_a >= n_drones || m->id_b >= n_drones || traj_first[m->id_a + 1] == traj_first[m->id_a] ||
                 traj_first[m->id_b + 1] == traj_first[m->id_b])
          status = NO_TRAJECTORY;
      }
      r->ia = r->node_a;
      r->ib = r->node_b;
      if (status == OK) {
        const int64_t a0 = traj_first[m->id_a], an = traj_first[m->id_a + 1] - a0;
        const int64_t b0 = traj_first[m->id_b], bn = traj_first[m->id_b + 1] - b0;
        const int64_t k_nfa = a0 + nearest(traj_stamp + a0, an, nf_a->stamp), k_a = a0 + nearest(traj_stamp + a0, an, m->stamp_a);
        const int64_t k_nfb = b0 + nearest(traj_stamp + b0, bn, nf_b->stamp), k_b = b0 + nearest(traj_stamp + b0, bn, m->stamp_b);
        const double da = fabs(traj_len[k_a] - traj_len[k_nfa]), db = fabs(traj_len[k_b] - traj_len[k_nfb]);
        double self_a[7], self_b[7];
        memcpy(self_a, m->self_pose_a, sizeof(self_a));
        memcpy(self_b, m->self_pose_b, sizeof(self_b));
        if (m->type != LOOP) {                                                   /* :1510-1517 */
          memcpy(self_a, traj_pose + k_a * 7, sizeof(self_a));
          memcpy(self_b, traj_pose + k_b * 7, sizeof(self_b));
          if (m->type == DET4D) {
            yaw_quat(quat_yaw(self_a + 3), self_a + 3);
            yaw_quat(quat_yaw(self_b + 3), self_b + 3);
          }
        }
        double dsa[7], dsb[7], t0[7], loop[7];
        delta_pose4(nf_a->self_pose, self_a, dsa);
        delta_pose4(self_b, nf_b->self_pose, dsb);
        pose_mul(dsa, m->relative_pose, t0);
        pose_mul(t0, dsb, loop);
        r->dpos = da + db;
        if (r->dpos > prm->det_dpos_thres) status = DPOS;
        edge_t* e = &r->edge;
        e->id_a = m->id_a;
        e->id_b = m->id_b;
        memcpy(e->rel_pose, loop, sizeof(loop));
        for (int j = 0; j < 36; ++j) {
          const double per_m = (j % 7 == 0) ? (j < 21 ? prm->odom_pos_cov_per_m : prm->odom_ang_cov_per_m) : 0.0;
          e->cov[j] = m->cov[j] + (da * per_m + db * per_m);
        }
        memcpy(e->odom_a, nf_a->self_pose, sizeof(e->odom_a));
        memcpy(e->odom_b, nf_b->self_pose, sizeof(e->odom_b));
        e->len_a = traj_len[k_nfa];
        e->len_b = traj_len[k_nfb];
        r->payload[0] = loop[0];
        r->payload[1] = loop[1];
        r->payload[2] = loop[2];
        r->payload[3] = quat_yaw(loop + 3);
        sqrt_information_4d(e->cov, r->payload + 4);
      }
      r->status = status;
      const int obs = status == OK && m->id_a < n_drones && m->id_b < n_drones && yaw_observable[m->id_a] &&
                      yaw_observable[m->id_b];
      r->skip = (obs && r->node_a != r->node_b) ? 0 : 1;                         /* :1066-1073 */
    }
  return k;
}
