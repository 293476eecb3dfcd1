// pose_algebra.cuh -- Swarm::Pose arithmetic on the device (fp64): pose = (translation, unit quaternion w x y z).
// swarm_msgs (HKUST-Swarm, not in the reference tree) defines the originals; the definitions used here are stated in
// oracle/pcm_ref.py and oracle/pnp_ref.py.
#pragma once
#include <math.h>

namespace osb {

struct PoseD { double t[3]; double q[4]; };   // translation, unit quaternion (w, x, y, z)

__device__ __forceinline__ void q_mul(const double* a, const double* b, double* o) {
  o[0] = a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3];
  o[1] = a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2];
  o[2] = a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1];
  o[3] = a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0];
}
__device__ __forceinline__ void q_rot(const double* q, const double* v, double* o) {    // v + 2 w (u x v) + 2 u x (u x v)
  const double cx = q[2] * v[2] - q[3] * v[1], cy = q[3] * v[0] - q[1] * v[2], cz = q[1] * v[1] - q[2] * v[0];
  const double dx = q[2] * cz - q[3] * cy, dy = q[3] * cx - q[1] * cz, dz = q[1] * cy - q[2] * cx;
  o[0] = v[0] + 2.0 * (q[0] * cx + dx);
  o[1] = v[1] + 2.0 * (q[0] * cy + dy);
  o[2] = v[2] + 2.0 * (q[0] * cz + dz);
}
__device__ __forceinline__ PoseD pose_mul(const PoseD& a, const PoseD& b) {
  PoseD o;
  double r[3];
  q_rot(a.q, b.t, r);
  o.t[0] = a.t[0] + r[0]; o.t[1] = a.t[1] + r[1]; o.t[2] = a.t[2] + r[2];
  q_mul(a.q, b.q, o.q);
  return o;
}
__device__ __forceinline__ PoseD pose_inv(const PoseD& a) {
  PoseD o;
  o.q[0] = a.q[0]; o.q[1] = -a.q[1]; o.q[2] = -a.q[2]; o.q[3] = -a.q[3];
  double r[3];
  q_rot(o.q, a.t, r);
  o.t[0] = -r[0]; o.t[1] = -r[1]; o.t[2] = -r[2];
  return o;
}
__device__ __forceinline__ PoseD load_pose(const double* p) {
  PoseD o;
  o.t[0] = p[0]; o.t[1] = p[1]; o.t[2] = p[2]; o.q[0] = p[3]; o.q[1] = p[4]; o.q[2] = p[5]; o.q[3] = p[6];
  return o;
}

// log map [translation ; rotation vector]
__device__ __forceinline__ void pose_log(const PoseD& p, double (&v)[6]) {
  v[0] = p.t[0]; v[1] = p.t[1]; v[2] = p.t[2];
  const double s = p.q[0] < 0 ? -1.0 : 1.0;
  const double w = s * p.q[0], x = s * p.q[1], y = s * p.q[2], z = s * p.q[3];
  const double n = sqrt(x * x + y * y + z * z);
  const double k = n < 1e-12 ? 2.0 : 2.0 * atan2(n, w) / n;
  v[3] = k * x; v[4] = k * y; v[5] = k * z;
}
// v^T C^-1 v by an unpivoted Cholesky factorisation of the symmetric 6x6 C (row-major); +inf when C is not SPD
__device__ __forceinline__ double smd6(const double (&v)[6], const double* C) {
  double L[6][6];
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    double s = C[j * 6 + j];
    for (int k = 0; k < j; ++k) s -= L[j][k] * L[j][k];
    if (!(s > 0.0)) return INFINITY;
    L[j][j] = sqrt(s);
#pragma unroll
    for (int i = j + 1; i < 6; ++i) {
      double c = C[i * 6 + j];
      for (int k = 0; k < j; ++k) c -= L[i][k] * L[j][k];
      L[i][j] = c / L[j][j];
    }
  }
  double smd = 0.0, y[6];
#pragma unroll
  for (int i = 0; i < 6; ++i) {
    double c = v[i];
    for (int k = 0; k < i; ++k) c -= L[i][k] * y[k];
    y[i] = c / L[i][i];
    smd += y[i] * y[i];
  }
  return smd;
}
__device__ __forceinline__ void quat_from_rotvec(const double* rv, double* q) {
  const double a = sqrt(rv[0] * rv[0] + rv[1] * rv[1] + rv[2] * rv[2]);
  if (a < 1e-12) { q[0] = 1.0; q[1] = 0.5 * rv[0]; q[2] = 0.5 * rv[1]; q[3] = 0.5 * rv[2]; }
  else { const double s = sin(0.5 * a) / a; q[0] = cos(0.5 * a); q[1] = s * rv[0]; q[2] = s * rv[1]; q[3] = s * rv[2]; }
  const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  q[0] /= n; q[1] /= n; q[2] /= n; q[3] /= n;
}
// ZYX (roll, pitch, yaw)
__device__ __forceinline__ void quat2eulers(const double* q, double (&e)[3]) {
  const double w = q[0], x = q[1], y = q[2], z = q[3];
  e[0] = atan2(2.0 * (w * x + y * z), 1.0 - 2.0 * (x * x + y * y));
  e[1] = asin(fmin(1.0, fmax(-1.0, 2.0 * (w * y - z * x))));
  e[2] = atan2(2.0 * (w * z + x * y), 1.0 - 2.0 * (y * y + z * z));
}
__device__ __forceinline__ double quat_yaw(const double* q) {
  return atan2(2.0 * (q[0] * q[3] + q[1] * q[2]), 1.0 - 2.0 * (q[2] * q[2] + q[3] * q[3]));
}
__device__ __forceinline__ double wrap_angle(double a) {
  const double pi = 3.141592653589793;
  return a - 2.0 * pi * floor((a + pi) / (2.0 * pi));
}
// Pose::set_yaw_only: position and yaw kept, roll and pitch zero
__device__ __forceinline__ PoseD pose_yaw_only(const PoseD& p) {
  PoseD o = p;
  const double rv[3] = {0.0, 0.0, quat_yaw(p.q)};
  quat_from_rotvec(rv, o.q);
  return o;
}
// Pose::DeltaPose(a, b, true): the 4-DoF a^-1 b (swarm_localization_factors.hpp:139-149), as oracle/pnp_ref.delta_pose
__device__ __forceinline__ PoseD delta_pose4(const PoseD& a, const PoseD& b) {
  const double ya = quat_yaw(a.q), yb = quat_yaw(b.q);
  const double d0 = b.t[0] - a.t[0], d1 = b.t[1] - a.t[1], d2 = b.t[2] - a.t[2];
  const double c = cos(ya), s = sin(ya);
  PoseD o;
  o.t[0] = c * d0 + s * d1;
  o.t[1] = -s * d0 + c * d1;
  o.t[2] = d2;
  const double rv[3] = {0.0, 0.0, wrap_angle(yb - ya)};
  quat_from_rotvec(rv, o.q);
  return o;
}

// DroneTrajectory look-up: the sample nearest to t, ties to the earlier one, clamped to the first / last sample
__device__ __forceinline__ int nearest_sample(const int64_t* __restrict__ s, int n, int64_t t) {
  int lo = 0, hi = n;                                              // first k with s[k] >= t
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (s[mid] < t) lo = mid + 1; else hi = mid;
  }
  if (lo == 0) return 0;
  if (lo == n) return n - 1;
  return (t - s[lo - 1]) <= (s[lo] - t) ? lo - 1 : lo;
}

}  // namespace osb
