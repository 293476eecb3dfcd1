// graph.cu -- osb_solver: GPU pose-graph solve replacing the body of SwarmLocalizationSolver::solve_once
// (swarm_localization/src/swarm_localization_solver.cpp:1668-1725).
//
// Factors (swarm_localization/include/swarm_localization/swarm_localization_factors.hpp):
//   DistanceMeasurementFactor :203-224, RelativePoseFactor4d :226-271 (DeltaPose :139-149, pose_error_4d :52-61),
//   DroneDetection4dFactor :273-367 (PoseMulti :165-172, DeltaPose_Naive :153-160, unit_position_error* :73-103).
// The reference evaluates them with Ceres AutoDiff jets; here residuals and ANALYTIC Jacobians are evaluated by
// one thread per factor (SURVEY.md Appendix A.6).  HuberLoss(1.0) is applied as Ceres' corrector does when
// rho'' <= 0: residual and Jacobian scaled by sqrt(rho'(s)).
//
// The solve is ONE persistent cooperative kernel: Levenberg-Marquardt outer loop (Ceres' LM step control: diagonal
// D = clip(diag(J^T J)), radius update by 1 - (2 rho - 1)^3, decrease factor doubling) and a block-Jacobi
// preconditioned conjugate gradient on the 4x4-block normal equations.  J^T J is never assembled off-diagonal:
// a factor thread computes t = Ja p_a + Jb p_b and the two 4-vectors Ja^T t, Jb^T t, and a node thread gathers the
// contributions from its own contiguous run of slots in a fixed order (no atomics: results are bit-reproducible
// run to run).  The problem (8 000 scalars, 12 000 factors for BASELINE config C5) is latency bound, not HBM bound:
// the Jacobians of a CTA's factor block stay in shared memory (SoA, conflict-free) for the whole solve, and when the
// factor list fits 16 CTAs the grid is launched as ONE thread-block cluster so that the 3 barriers per CG iteration
// are hardware cluster barriers instead of software grid barriers.
#include <cooperative_groups.h>
#include <algorithm>
#include <cmath>
#include <cstring>
#include <type_traits>
#include "common.cuh"

namespace cg = cooperative_groups;

namespace osb {

constexpr int GS_THREADS = 256;           // 255 registers per thread: the CG fast path keeps ~50 doubles live per thread
constexpr int GS_KF = 3;                  // factors per thread on the fast path (16 CTAs x 256 threads x 3 >= 12 288 factors)
constexpr int GS_MAX_CLUSTER = 16;
constexpr int GS_SMEM_J_MAX = 200 * 1024;   // bytes of shared memory a CTA may spend on its Jacobian block
constexpr int GS_SMEM_DYN_MAX = 227 * 1024 - 2048;  // opt-in limit minus the kernel's static shared memory
constexpr double kPi = 3.14159265358979323846;
constexpr double kTwoPi = 6.28318530717958647692;

__device__ __forceinline__ double normalize_angle(double a) {   // factors.hpp:34-40
  return a - kTwoPi * floor((a + kPi) / kTwoPi);
}

// residual (nr rows) and 4x4 Jacobian blocks (row-major, rows >= nr zero) of one factor, un-robustified.
// JAC = false: residual only (trial-point cost; identical arithmetic for r).
template <bool JAC>
__device__ __forceinline__ int linearize_factor_t(int type, const double* __restrict__ pa, const double* __restrict__ pb,
                                                  const double* __restrict__ pl, double r[4], double Ja[16], double Jb[16]) {
  if (JAC) {
#pragma unroll
    for (int i = 0; i < 16; ++i) { Ja[i] = 0.0; Jb[i] = 0.0; }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) r[i] = 0.0;
  if (type == OSB_FACTOR_DISTANCE) {
    const double dx = pa[0] - pb[0], dy = pa[1] - pb[1], dz = pa[2] - pb[2];
    const double nrm = sqrt(dx * dx + dy * dy + dz * dz);
    const double si = pl[1];
    r[0] = (nrm - pl[0]) * si;
    const double inv = si / nrm;
    Ja[0] = dx * inv; Ja[1] = dy * inv; Ja[2] = dz * inv;
    Jb[0] = -dx * inv; Jb[1] = -dy * inv; Jb[2] = -dz * inv;
    return 1;
  }
  if (type == OSB_FACTOR_RELPOSE) {
    double s, c;
    sincos(pa[3], &s, &c);
    const double dx = pb[0] - pa[0], dy = pb[1] - pa[1], dz = pb[2] - pa[2];
    double e[4];
    e[0] = pl[0] - (c * dx + s * dy);
    e[1] = pl[1] - (-s * dx + c * dy);
    e[2] = pl[2] - dz;
    e[3] = normalize_angle(pl[3] - normalize_angle(pb[3] - pa[3]));
    const double* S = pl + 4;
    // d est / d pose_a (columns x,y,z,yaw) and pose_b
    const double Ea[4][4] = {{-c, -s, 0.0, -s * dx + c * dy}, {s, -c, 0.0, -c * dx - s * dy}, {0.0, 0.0, -1.0, 0.0},
                             {0.0, 0.0, 0.0, -1.0}};
    const double Eb[4][4] = {{c, s, 0.0, 0.0}, {-s, c, 0.0, 0.0}, {0.0, 0.0, 1.0, 0.0}, {0.0, 0.0, 0.0, 1.0}};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      double ri = 0.0;
#pragma unroll
      for (int k = 0; k < 4; ++k) ri += S[i * 4 + k] * e[k];
      r[i] = ri;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        double a = 0.0, b = 0.0;
#pragma unroll
        for (int k = 0; k < 4; ++k) { a += S[i * 4 + k] * Ea[k][j]; b += S[i * 4 + k] * Eb[k][j]; }
        Ja[i * 4 + j] = -a; Jb[i * 4 + j] = -b;
      }
    }
    return 4;
  }
  // OSB_FACTOR_DETECTION
  const int flags = (int)pl[10];
  const double inv_dep = pl[9], ext_z = pl[11], sphere_std = pl[20], invdep_std = pl[21];
  double A[4], Bp[4];
  double Ga03 = 0.0, Ga13 = 0.0, Gb03 = 0.0, Gb13 = 0.0;   // d T' / d yaw of the raw pose (PoseMulti)
  if (flags & 2) {
    double s, c;
    sincos(pa[3], &s, &c);
    A[0] = pa[0] + c * pl[12] - s * pl[13]; A[1] = pa[1] + s * pl[12] + c * pl[13]; A[2] = pa[2] + pl[14];
    A[3] = normalize_angle(pa[3] + pl[15]);
    Ga03 = -s * pl[12] - c * pl[13]; Ga13 = c * pl[12] - s * pl[13];
    sincos(pb[3], &s, &c);
    Bp[0] = pb[0] + c * pl[16] - s * pl[17]; Bp[1] = pb[1] + s * pl[16] + c * pl[17]; Bp[2] = pb[2] + pl[18];
    Bp[3] = normalize_angle(pb[3] + pl[19]);
    Gb03 = -s * pl[16] - c * pl[17]; Gb13 = c * pl[16] - s * pl[17];
  } else {
    A[0] = pa[0]; A[1] = pa[1]; A[2] = pa[2] + ext_z; A[3] = pa[3];
    Bp[0] = pb[0]; Bp[1] = pb[1]; Bp[2] = pb[2]; Bp[3] = pb[3];
  }
  double s, c;
  sincos(A[3], &s, &c);
  const double dx = Bp[0] - A[0], dy = Bp[1] - A[1], dz = Bp[2] - A[2];
  const double rel[3] = {c * dx + s * dy, -s * dx + c * dy, dz};
  const double rho = 1.0 / sqrt(rel[0] * rel[0] + rel[1] * rel[1] + rel[2] * rel[2]);
  // d rel / d A (4 cols), d rel / d B' (4 cols)
  const double RA[3][4] = {{-c, -s, 0.0, -s * dx + c * dy}, {s, -c, 0.0, -c * dx - s * dy}, {0.0, 0.0, -1.0, 0.0}};
  const double RB[3][4] = {{c, s, 0.0, 0.0}, {-s, c, 0.0, 0.0}, {0.0, 0.0, 1.0, 0.0}};
  // chain through PoseMulti: columns 0..2 identity, column 3 gets + d rel/dT' * dT'/dyaw (yaw' = yaw + const)
  double DA[3][4], DB[3][4];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    DA[i][0] = RA[i][0]; DA[i][1] = RA[i][1]; DA[i][2] = RA[i][2];
    DA[i][3] = RA[i][3] + RA[i][0] * Ga03 + RA[i][1] * Ga13;
    DB[i][0] = RB[i][0]; DB[i][1] = RB[i][1]; DB[i][2] = RB[i][2];
    DB[i][3] = RB[i][3] + RB[i][0] * Gb03 + RB[i][1] * Gb13;
  }
  const int nr = (flags & 1) ? 3 : 2;
  double u[3], Jrel[3][3];
#pragma unroll
  for (int i = 0; i < 3; ++i) u[i] = rel[i] * rho - pl[i];
  // dU = rho (I - rel rel^T rho^2)
  double dU[3][3];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) dU[i][j] = rho * ((i == j ? 1.0 : 0.0) - rel[i] * rel[j] * rho * rho);
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const double* Bt = pl + 3 + 3 * i;
    r[i] = (Bt[0] * u[0] + Bt[1] * u[1] + Bt[2] * u[2]) / sphere_std;
#pragma unroll
    for (int j = 0; j < 3; ++j) Jrel[i][j] = (Bt[0] * dU[0][j] + Bt[1] * dU[1][j] + Bt[2] * dU[2][j]) / sphere_std;
  }
  if (nr == 3) {
    r[2] = (inv_dep - rho) / invdep_std;
    const double r3 = rho * rho * rho / invdep_std;
    Jrel[2][0] = r3 * rel[0]; Jrel[2][1] = r3 * rel[1]; Jrel[2][2] = r3 * rel[2];
  } else {
    Jrel[2][0] = Jrel[2][1] = Jrel[2][2] = 0.0;
  }
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    if (i >= nr) break;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      Ja[i * 4 + j] = Jrel[i][0] * DA[0][j] + Jrel[i][1] * DA[1][j] + Jrel[i][2] * DA[2][j];
      Jb[i * 4 + j] = Jrel[i][0] * DB[0][j] + Jrel[i][1] * DB[1][j] + Jrel[i][2] * DB[2][j];
    }
  }
  return nr;
}

__device__ __forceinline__ int linearize_factor(int type, const double* __restrict__ pa, const double* __restrict__ pb,
                                                const double* __restrict__ pl, double r[4], double Ja[16], double Jb[16]) {
  return linearize_factor_t<true>(type, pa, pb, pl, r, Ja, Jb);
}
// |r|^2 only (un-robustified): the Jacobian arithmetic of the inlined body is dead code here
__device__ __forceinline__ double factor_sqnorm(int type, const double* __restrict__ pa, const double* __restrict__ pb,
                                                const double* __restrict__ pl) {
  double r[4], Ja[16], Jb[16];
  linearize_factor_t<false>(type, pa, pb, pl, r, Ja, Jb);
  return r[0] * r[0] + r[1] * r[1] + r[2] * r[2] + r[3] * r[3];
}

// The inner (PCG) arithmetic type.  Levenberg-Marquardt only needs an INEXACT step (relative residual 1e-2), so
// everything inside the PCG -- Jacobian blocks, direction / residual / preconditioner vectors, contribution slots, the
// chain factorisation -- runs in fp32 when the requested pcg_tolerance allows (>= 1e-4); residuals, costs, the gradient
// J^T r, the diagonal, the poses and every LM decision stay fp64.  fp32 halves what bounds a CG iteration here: the
// 32-bit shuffles of the preconditioner sweeps, the bytes of every cross-thread gather through L2, the shared-memory
// footprint of the Jacobians (96 KB instead of 192 KB) and the live registers.  A numpy
// emulation of the same loop gives the same iteration counts and poses within 1e-8 of the all-fp64 solve (DESIGN.md);
// tests/test_gpu_solver.py checks it on the GPU.  T = double is kept for tight tolerances (parity tests).
struct SolverDev {
  int n, m;
  int fpc;                 // factors per CTA (contiguous block of the factor list)
  int use_cluster;         // 1: the whole grid is ONE thread-block cluster (hardware barrier); 0: cooperative grid sync
  int j_in_smem;           // 1: the CTA's Jacobians live in shared memory (SoA), 0: in `Jg`
  // graph
  const uint8_t* fixed; const int32_t* ftype; const int32_t* ia; const int32_t* ib; const uint8_t* huber;
  const double* payload;
  const int32_t* node_ptr;                 // CSR: node n owns contribution slots [node_ptr[n], node_ptr[n+1])
  const int32_t* slot_a; const int32_t* slot_b;   // slot of factor f's contribution to its node a / node b
  // state
  double* x[2];            // pose buffers (current / trial), [n][4]
  void* Jg;                // global Jacobian store, SoA [32][m] of T (used when the CTA block does not fit shared memory)
  double *g, *D, *Hnn;     // gradient, LM diagonal, diagonal Hessian blocks (fp64)
  void *Minv, *p, *z, *res, *Ap, *delta;   // PCG node vectors, element type T
  double* gs;              // gradient contribution slots [2m][4] (fp64, written at a linearisation)
  void* cs;                // PCG contribution slots [2m][4] of T
  double* hs;              // Hessian-diagonal-block slots [2m][16] (only touched at a re-linearisation)
  double* partial;         // [2][4][grid]
  osb_solve_options opt;
  osb_solve_summary* summary;
  double* poses_out;
  long long* dbg;          // [8] cycle counters of block 0 / thread 0 (profiling aid, see osb_solver_phase_cycles)
  // chain preconditioner (fast path only; see chain_apply)
  int use_chain;
  const uint8_t* link;     // [n] 1: node i-1 is node i's predecessor on a path of the cover (never set when i % 16 == 0)
  const int32_t* es_ptr;   // CSR: node i sums the coupling blocks es[es_ptr[i] .. es_ptr[i+1])
  const int32_t* es_slot;  // [m] -1, or 2 * (index into es) + (1 if the factor's node a is the later node of the pair)
  double* es;              // [<= m][16] J_i^T J_{i-1} of the chain factors (written at every linearisation)
  double* En;              // [n][16] summed coupling block of node i with node i-1
  // batched trials (osb_solver_solve_multistart): CTA b solves trial first_trial + b / ctas as CTA b % ctas of that
  // solve.  The state pointers above (x .. En) point into trial 0's block of the handle's arena (trial_layout); trial t's
  // block lies t * tstride bytes further.  The graph tables (fixed .. slot_b, link, es_ptr, es_slot) are shared, and
  // only trial 0 writes dbg.
  int ctas;                // CTAs per solve (the cluster size on the cluster path)
  int first_trial;
  long long tstride;
  // device tail (osb_solver_solve_resident_dev, graph_solve_kernel<T, false, true>): [0] status of the call's tables
  // (non-zero: refused, nothing runs), [1] m = resident factors + tail, [2] fpc = ceil(m / ctas).  m and fpc above are
  // then the bounds the launch shape was picked for.
  const int32_t* dev_word;
};

// trial t's copy of a per-trial state pointer lies t * tstride bytes past trial 0's.  It is recomputed at every use from
// the cluster id (a special register) rather than shifted once at the start: twenty shifted pointers held for the whole
// solve would not fit beside the solver's working set, which already fills the 255 registers.  A cooperative launch
// runs one trial, which the host binds at its own block of the arena.
// MULTI = false (one solve per launch) compiles this away: reading the cluster id at every use costs the latency-bound
// CG loop about 10 % (measured on C5), so a single solve runs the graph_solve_kernel<T, false> instantiation.
template <bool MULTI, typename Q>
__device__ __forceinline__ Q* tp(const SolverDev& P, Q* p) {
  if (!MULTI) return p;
  unsigned c;
  asm volatile("mov.u32 %0, %%clusterid.x;" : "=r"(c));
  return reinterpret_cast<Q*>(reinterpret_cast<char*>(p) + (long long)c * P.tstride);
}

// this CTA's index inside its solve, and the solve's trial (a cooperative launch is one solve of `ctas` = gridDim CTAs)
__device__ __forceinline__ int solve_rank(const SolverDev& P) {
  unsigned r;
  if (P.use_cluster) asm("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); else r = blockIdx.x;
  return (int)r;
}
template <bool MULTI>
__device__ __forceinline__ int solve_trial(const SolverDev& P) {
  unsigned c = 0;
  if (MULTI) asm volatile("mov.u32 %0, %%clusterid.x;" : "=r"(c));
  return P.first_trial + (int)c;
}

__device__ __forceinline__ void all_sync(const SolverDev& P, cg::grid_group& grid) {
  if (P.use_cluster) cg::this_cluster().sync(); else grid.sync();
}

__device__ __forceinline__ float warp_sum_t(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum_t(double v) { return warp_sum_d(v); }

// grid-wide sums of K values.  The warp level runs in T (cheap in fp32), the 8 warp sums, the CTA partials and the final
// sum are fp64 (a handful of instructions on warp 0 only).
template <int K, bool MT, typename T>
__device__ void grid_reduce_sum(T (&vin)[K], double (&v)[K], const SolverDev& P, int parity, double* sh, cg::grid_group& grid) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = GS_THREADS / 32, G = P.ctas;
  double* pbuf = tp<MT>(P, P.partial) + (size_t)parity * 4 * G;
  __syncwarp();
#pragma unroll
  for (int k = 0; k < K; ++k) {
    const T w = warp_sum_t(vin[k]);
    if (lane == 0) sh[k * 32 + warp] = (double)w;
  }
  __syncthreads();
  if (warp == 0) {
#pragma unroll
    for (int k = 0; k < K; ++k) {
      double xv = (lane < nw) ? sh[k * 32 + lane] : 0.0;
      xv = warp_sum_d(xv);
      if (lane == 0) __stcg(pbuf + k * G + solve_rank(P), xv);
    }
  }
  all_sync(P, grid);
  if (warp == 0) {
#pragma unroll
    for (int k = 0; k < K; ++k) {
      double xv = 0.0;
      for (int i = lane; i < G; i += 32) xv += __ldcg(pbuf + k * G + i);
      xv = warp_sum_d(xv);
      if (lane == 0) sh[k] = xv;
    }
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < K; ++k) v[k] = sh[k];
  __syncthreads();
}

template <bool MT>
__device__ double grid_reduce_max(double vmax, const SolverDev& P, int parity, double* sh, cg::grid_group& grid) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, G = P.ctas;
  __syncwarp();
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) vmax = fmax(vmax, __shfl_xor_sync(0xffffffffu, vmax, o));
  if (lane == 0) sh[warp] = vmax;
  __syncthreads();
  double* pbuf = tp<MT>(P, P.partial) + (size_t)parity * 4 * G;
  if (warp == 0) {
    double xv = (lane < GS_THREADS / 32) ? sh[lane] : 0.0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) xv = fmax(xv, __shfl_xor_sync(0xffffffffu, xv, o));
    if (lane == 0) __stcg(pbuf + solve_rank(P), xv);
  }
  all_sync(P, grid);
  if (warp == 0) {
    double xv = 0.0;
    for (int i = lane; i < G; i += 32) xv = fmax(xv, __ldcg(pbuf + i));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) xv = fmax(xv, __shfl_xor_sync(0xffffffffu, xv, o));
    if (lane == 0) sh[0] = xv;
  }
  __syncthreads();
  const double r = sh[0];
  __syncthreads();
  return r;
}

// Jacobian store accessor: element i (0..31: Ja row-major then Jb) of the factor with CTA-local index `li`
template <typename T>
struct JStore {
  T* base; int stride; int off;
  __device__ __forceinline__ T& at(int i, int li) const { return base[(size_t)i * stride + off + li]; }
};

// clock read that cannot be scheduled before `v` has been computed (phase attribution only)
__device__ __forceinline__ long long clock_after(float v) {
  long long c; asm volatile("mov.u64 %0, %%clock64;" : "=l"(c) : "f"(v) : "memory"); return c;
}
__device__ __forceinline__ long long clock_after(double v) {
  long long c; asm volatile("mov.u64 %0, %%clock64;" : "=l"(c) : "d"(v) : "memory"); return c;
}

// vector loads / stores of a node's 4-vector (one 16-byte access in fp32, two in fp64), L2-coherent
__device__ __forceinline__ void ld4(const float* p, float (&v)[4]) {
  const float4 t = __ldcg(reinterpret_cast<const float4*>(p));
  v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
}
__device__ __forceinline__ void ld4(const double* p, double (&v)[4]) {
  const double2 a = __ldcg(reinterpret_cast<const double2*>(p)), b = __ldcg(reinterpret_cast<const double2*>(p) + 1);
  v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
}
__device__ __forceinline__ void st4(float* p, const float (&v)[4]) {
  __stcg(reinterpret_cast<float4*>(p), make_float4(v[0], v[1], v[2], v[3]));
}
__device__ __forceinline__ void st4(double* p, const double (&v)[4]) {
  __stcg(reinterpret_cast<double2*>(p), make_double2(v[0], v[1]));
  __stcg(reinterpret_cast<double2*>(p) + 1, make_double2(v[2], v[3]));
}

// 4x4 SPD inverse by Gauss-Jordan (no pivoting: the LM term keeps the diagonal positive)
template <typename T>
__device__ void inv4(const T* __restrict__ M, T* __restrict__ out) {
  T a[4][8];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) { a[i][j] = M[i * 4 + j]; a[i][4 + j] = (i == j) ? T(1) : T(0); }
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const T piv = T(1) / a[c][c];
#pragma unroll
    for (int j = 0; j < 8; ++j) a[c][j] *= piv;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      if (i == c) continue;
      const T f = a[i][c];
#pragma unroll
      for (int j = 0; j < 8; ++j) a[i][j] -= f * a[c][j];
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) out[i * 4 + j] = a[i][4 + j];
}

// ---- chain preconditioner -----------------------------------------------------------------------------------------
// Block-Jacobi sees only a node's own 4x4 block, and a pose graph is dominated by long odometry chains: C5 needs 1663
// PCG iterations that way.  The host covers the graph with vertex-disjoint paths (heaviest factors first) and numbers the
// nodes along them, so a path is a run of consecutive node ids = consecutive threads.  The preconditioner is the block-
// TRIDIAGONAL part of J^T J + lam D along those paths, cut every 16 nodes so that a segment lives in one half-warp:
//   M = sum over chain factors (full 8x8 contribution) + sum over the other factors (their two diagonal blocks) + lam D,
// a sum of PSD terms plus a positive diagonal, hence SPD.  Factorisation M = (I + L) S (I + L)^T by a 16-step sweep over
// the half-warp (once per PCG solve); application z = M^-1 r = 15 forward + 15 backward steps of 4-vector shuffles.
// Same CPU emulation as the kernel (DESIGN.md): 1663 -> 385 PCG iterations on C5.
template <typename T>
__device__ __forceinline__ void mat4_mul(const T* A, const T* B, T* C) {        // C = A B
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      T a = T(0);
#pragma unroll
      for (int k = 0; k < 4; ++k) a += A[i * 4 + k] * B[k * 4 + j];
      C[i * 4 + j] = a;
    }
}

// z = M^-1 r for the segment this half-warp owns.  Si = S_i^-1, L = L_i (zero when the node has no predecessor link).
// Warp-collective: every lane of the warp must call it.
template <typename T>
__device__ __forceinline__ void chain_apply(const T (&Si)[16], const T (&L)[16], bool link, int sl, const T (&r)[4], T (&z)[4]) {
  // Branch-free on purpose (no divergent code between two shuffles): the active lane of a step is selected by a 0/1
  // multiplier; L is zero on lanes without a predecessor link.
  __syncwarp();
  T y[4] = {r[0], r[1], r[2], r[3]};
#pragma unroll
  for (int s = 1; s < 16; ++s) {                       // forward: y_i = r_i - L_i y_{i-1}
    T yp[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) yp[k] = __shfl_up_sync(0xffffffffu, y[k], 1);
    const T m = (sl == s && link) ? T(1) : T(0);
#pragma unroll
    for (int i = 0; i < 4; ++i)
      y[i] -= m * (L[i * 4] * yp[0] + L[i * 4 + 1] * yp[1] + L[i * 4 + 2] * yp[2] + L[i * 4 + 3] * yp[3]);
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) z[i] = Si[i * 4] * y[0] + Si[i * 4 + 1] * y[1] + Si[i * 4 + 2] * y[2] + Si[i * 4 + 3] * y[3];
#pragma unroll
  for (int s = 14; s >= 0; --s) {                      // backward: z_i = S_i^-1 y_i - L_{i+1}^T z_{i+1}
    const T m = (sl == s + 1 && link) ? T(1) : T(0);
    T u[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) u[j] = m * (L[j] * z[0] + L[4 + j] * z[1] + L[8 + j] * z[2] + L[12 + j] * z[3]);
#pragma unroll
    for (int k = 0; k < 4; ++k) u[k] = __shfl_down_sync(0xffffffffu, u[k], 1);
    const T mz = (sl == s) ? T(1) : T(0);              // (lane 15 receives lane 16's u, which is zero: sl = 0 there)
#pragma unroll
    for (int k = 0; k < 4; ++k) z[k] -= mz * u[k];
  }
}

// Linearise every factor of this CTA at `xp` (fp64): robustified Jacobians -> J store (as T), gradient contributions
// J^T r -> gs slots, diagonal-block contributions J^T J -> hs slots, chain couplings -> es.  Returns this thread's share
// of the cost.
template <bool MT, typename T>
__device__ double factor_linearize(const SolverDev& P, const double* __restrict__ xp, const JStore<T>& J) {
  double cost = 0.0;
  const int f0 = solve_rank(P) * P.fpc, f1 = min(P.m, f0 + P.fpc);
  for (int f = f0 + threadIdx.x; f < f1; f += GS_THREADS) {
    const int li = f - f0;
    const int a = P.ia[f], b = P.ib[f];
    double pa[4], pb[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) { pa[i] = __ldcg(xp + 4 * a + i); pb[i] = __ldcg(xp + 4 * b + i); }
    double r[4], Ja[16], Jb[16];
    linearize_factor(P.ftype[f], pa, pb, P.payload + (size_t)f * OSB_PAYLOAD_LEN, r, Ja, Jb);
    const double s = r[0] * r[0] + r[1] * r[1] + r[2] * r[2] + r[3] * r[3];
    double w = 1.0;
    if (P.huber[f] && s > 1.0) {        // ceres::HuberLoss(1.0): rho(s) = 2 sqrt(s) - 1, sqrt(rho') = s^-1/4
      cost += 0.5 * (2.0 * sqrt(s) - 1.0);
      w = 1.0 / sqrt(sqrt(s));
    } else {
      cost += 0.5 * s;
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) r[i] *= w;
#pragma unroll
    for (int i = 0; i < 16; ++i) { Ja[i] *= w; Jb[i] *= w; J.at(i, li) = (T)Ja[i]; J.at(16 + i, li) = (T)Jb[i]; }
    if (P.use_chain) {
      const int es = P.es_slot[f];
      if (es >= 0) {                      // E = J_later^T J_earlier (rows: the later node of the pair)
        const double* Jl = (es & 1) ? Ja : Jb;
        const double* Je = (es & 1) ? Jb : Ja;
        double* dst = tp<MT>(P, P.es) + 16 * (size_t)(es >> 1);
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            double t = 0.0;
#pragma unroll
            for (int i = 0; i < 4; ++i) t += Jl[i * 4 + j] * Je[i * 4 + k];
            __stcg(dst + j * 4 + k, t);
          }
      }
    }
    double* ga = tp<MT>(P, P.gs) + 4 * (size_t)P.slot_a[f];
    double* gb = tp<MT>(P, P.gs) + 4 * (size_t)P.slot_b[f];
    double* ha = tp<MT>(P, P.hs) + 16 * (size_t)P.slot_a[f];
    double* hb = tp<MT>(P, P.hs) + 16 * (size_t)P.slot_b[f];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      double sa = 0.0, sb = 0.0;
#pragma unroll
      for (int i = 0; i < 4; ++i) { sa += Ja[i * 4 + j] * r[i]; sb += Jb[i * 4 + j] * r[i]; }
      __stcg(ga + j, sa); __stcg(gb + j, sb);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        double ta = 0.0, tb = 0.0;
#pragma unroll
        for (int i = 0; i < 4; ++i) { ta += Ja[i * 4 + j] * Ja[i * 4 + k]; tb += Jb[i * 4 + j] * Jb[i * 4 + k]; }
        __stcg(ha + j * 4 + k, ta); __stcg(hb + j * 4 + k, tb);
      }
    }
  }
  return cost;
}

// cost at the trial point `xn` (fp64) and this thread's share of |J_cur delta|^2 (model decrease, in T)
template <bool MT, typename T>
__device__ void factor_trial(const SolverDev& P, const double* __restrict__ xn, const JStore<T>& J, double& cost, double& jd) {
  const int f0 = solve_rank(P) * P.fpc, f1 = min(P.m, f0 + P.fpc);
  const T* delta = static_cast<const T*>(tp<MT>(P, P.delta));
  T jdt = T(0);
  for (int f = f0 + threadIdx.x; f < f1; f += GS_THREADS) {
    const int li = f - f0;
    const int a = P.ia[f], b = P.ib[f];
    double pa[4], pb[4];
    T da[4], db[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) { pa[i] = __ldcg(xn + 4 * a + i); pb[i] = __ldcg(xn + 4 * b + i); }
    ld4(delta + 4 * a, da); ld4(delta + 4 * b, db);
    const double s = factor_sqnorm(P.ftype[f], pa, pb, P.payload + (size_t)f * OSB_PAYLOAD_LEN);
    cost += (P.huber[f] && s > 1.0) ? 0.5 * (2.0 * sqrt(s) - 1.0) : 0.5 * s;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      T t = T(0);
#pragma unroll
      for (int j = 0; j < 4; ++j) t += J.at(i * 4 + j, li) * da[j] + J.at(16 + i * 4 + j, li) * db[j];
      jdt += t * t;
    }
  }
  jd += (double)jdt;
}

// factor phase of a PCG iteration for one factor: t = Ja p_a + Jb p_b and its two contributions ca = Ja^T t, cb = Jb^T t
template <typename T>
__device__ __forceinline__ void factor_apply(const JStore<T>& J, int li, const T (&pa)[4], const T (&pb)[4], T (&ca)[4],
                                             T (&cb)[4]) {
  T t[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    T acc = T(0);
#pragma unroll
    for (int j = 0; j < 4; ++j) acc += J.at(i * 4 + j, li) * pa[j] + J.at(16 + i * 4 + j, li) * pb[j];
    t[i] = acc;
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    T sa = T(0), sb = T(0);
#pragma unroll
    for (int i = 0; i < 4; ++i) { sa += J.at(i * 4 + j, li) * t[i]; sb += J.at(16 + i * 4 + j, li) * t[i]; }
    ca[j] = sa; cb[j] = sb;
  }
}

// DT: one solve whose factor list ends in a device-side tail (osb_solver_solve_resident_dev).  The factor count and the
// CTA blocks come from P.dev_word, and a refused call leaves on every CTA before the first barrier.
template <typename T, bool MT, bool DT = false>
__global__ void __launch_bounds__(GS_THREADS, 1)
graph_solve_kernel(SolverDev P) {
  if (DT) {
    if (__ldcg(P.dev_word) != 0) return;
    P.m = __ldcg(P.dev_word + 1); P.fpc = __ldcg(P.dev_word + 2);
  }
  cg::grid_group grid = cg::this_grid();
  extern __shared__ __align__(16) unsigned char smem_raw[];
  T* smem_j = reinterpret_cast<T*>(smem_raw);
  __shared__ double sh[4 * 32];
  // from here on "the grid" is this trial's solve: `ctas` CTAs, thread ids counted inside it
  const int trial = solve_trial<MT>(P);
  const bool dbg_trial = trial == 0;
  const int T_ = P.ctas * GS_THREADS;
  const int gtid = solve_rank(P) * GS_THREADS + threadIdx.x;
  JStore<T> J;
  if (P.j_in_smem) { J.base = smem_j; J.stride = P.fpc; J.off = 0; }
  else { J.base = static_cast<T*>(tp<MT>(P, P.Jg)); J.stride = P.m; J.off = solve_rank(P) * P.fpc; }
  T* Ls = smem_j + (size_t)32 * P.fpc;          // [16][GS_THREADS]: L_i of the chain preconditioner (use_chain only)
  const auto Pp = [&] { return static_cast<T*>(tp<MT>(P, P.p)); }; const auto Pz = [&] { return static_cast<T*>(tp<MT>(P, P.z)); }; const auto Pres = [&] { return static_cast<T*>(tp<MT>(P, P.res)); };
  const auto PAp = [&] { return static_cast<T*>(tp<MT>(P, P.Ap)); }; const auto Pdelta = [&] { return static_cast<T*>(tp<MT>(P, P.delta)); }; const auto PMinv = [&] { return static_cast<T*>(tp<MT>(P, P.Minv)); };
  const auto Pcs = [&] { return static_cast<T*>(tp<MT>(P, P.cs)); };
  int parity = 0;
  unsigned long long t0 = 0;
  const long long k0 = clock64();
  if (gtid == 0) {                           // each trial's time limit counts from its own start
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t0));
    if (dbg_trial)
      for (int i = 0; i < 8 + GS_MAX_CLUSTER * (GS_THREADS / 32); ++i) P.dbg[i] = 0;
  }

  int cur = 0;
  double radius = P.opt.initial_trust_radius;
  double decrease = 2.0;
  int iters = 0, pcg_total = 0, termination = 3;

  // ---- initial linearisation ----
  double v1[1], w1[1] = {factor_linearize<MT>(P, tp<MT>(P, P.x[0]), J)};
  grid_reduce_sum<1, MT>(w1, v1, P, parity, sh, grid); parity ^= 1;
  double cost = v1[0];
  const double initial_cost = cost;
  bool need_gradient = true;
  const int f0 = solve_rank(P) * P.fpc, f1 = min(P.m, f0 + P.fpc);
  // static per-thread data of the fast CG path
  const bool fast = (P.fpc <= GS_KF * GS_THREADS) && (P.n <= T_);
  int fa[GS_KF], fb[GS_KF], fsa[GS_KF], fsb[GS_KF];
  bool fvalid[GS_KF];
#pragma unroll
  for (int k = 0; k < GS_KF; ++k) {
    fvalid[k] = false; fa[k] = fb[k] = fsa[k] = fsb[k] = 0;
    const int f = f0 + threadIdx.x + k * GS_THREADS;
    if (fast && f < f1) { fvalid[k] = true; fa[k] = P.ia[f]; fb[k] = P.ib[f]; fsa[k] = P.slot_a[f]; fsb[k] = P.slot_b[f]; }
  }
  const bool is_node = fast && gtid < P.n && !P.fixed[gtid];
  const int ns0 = is_node ? P.node_ptr[gtid] : 0, ns1 = is_node ? P.node_ptr[gtid + 1] : 0;
  const bool chain = fast && P.use_chain;
  const int sl = threadIdx.x & 15;

  while (iters < P.opt.max_iterations) {
    if (need_gradient) {
      // ---- node phase G (fp64): gather gradient and diagonal blocks from the slots, LM diagonal ----
      double vmax = 0.0;
      for (int n = gtid; n < P.n; n += T_) {
        double gn[4] = {0.0, 0.0, 0.0, 0.0};
        double Hn[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) Hn[i] = 0.0;
        if (!P.fixed[n]) {
          const int s0 = P.node_ptr[n], s1 = P.node_ptr[n + 1];
#pragma unroll 2
          for (int sidx = s0; sidx < s1; ++sidx) {
#pragma unroll
            for (int i = 0; i < 4; ++i) gn[i] += __ldcg(tp<MT>(P, P.gs) + 4 * (size_t)sidx + i);
#pragma unroll
            for (int i = 0; i < 16; ++i) Hn[i] += __ldcg(tp<MT>(P, P.hs) + 16 * (size_t)sidx + i);
          }
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          tp<MT>(P, P.g)[4 * n + i] = gn[i];
          tp<MT>(P, P.D)[4 * n + i] = fmin(fmax(Hn[i * 5], 1e-6), 1e32);
          vmax = fmax(vmax, fabs(gn[i]));
        }
#pragma unroll
        for (int i = 0; i < 16; ++i) tp<MT>(P, P.Hnn)[16 * n + i] = Hn[i];
        if (P.use_chain) {
          double En[16];
#pragma unroll
          for (int i = 0; i < 16; ++i) En[i] = 0.0;
          for (int e = P.es_ptr[n]; e < P.es_ptr[n + 1]; ++e)
#pragma unroll
            for (int i = 0; i < 16; ++i) En[i] += __ldcg(tp<MT>(P, P.es) + 16 * (size_t)e + i);
#pragma unroll
          for (int i = 0; i < 16; ++i) tp<MT>(P, P.En)[16 * n + i] = En[i];
        }
      }
      const double gmax = grid_reduce_max<MT>(vmax, P, parity, sh, grid); parity ^= 1;
      need_gradient = false;
      if (gmax <= P.opt.gradient_tolerance) { termination = 1; break; }
    }

    // ---- PCG init (node phase): preconditioner, res = -g, z = M^-1 res, p = 0, delta = 0 ----
    // Fast path (every node has its own thread, <= GS_KF factors per thread): the node's preconditioner blocks, D, res,
    // z, p, delta stay in REGISTERS for the whole CG solve and the factor's indices are preloaded, so a CG iteration
    // touches global memory only for what crosses threads: z/p gathers by the factor threads and the contribution slots.
    const double lam = 1.0 / radius;
    T v2[2] = {T(0), T(0)};
    T Mi[16], Dl[4] = {T(0), T(0), T(0), T(0)}, rn[4] = {T(0), T(0), T(0), T(0)}, zn[4] = {T(0), T(0), T(0), T(0)};
    T pn[4] = {T(0), T(0), T(0), T(0)}, dn[4] = {T(0), T(0), T(0), T(0)};     // Dl = lam * D
    bool lk = false;
    if (chain) {
      // factorise the segment's block-tridiagonal M = (I + L) S (I + L)^T: 16 steps over the half-warp, Mi := S_i^-1
      T M[16], E[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) { M[i] = (i % 5 == 0) ? T(1) : T(0); E[i] = T(0); Mi[i] = T(0); }
      if (is_node) {
        double Md[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) Md[i] = tp<MT>(P, P.Hnn)[16 * gtid + i];
#pragma unroll
        for (int i = 0; i < 4; ++i) { const double ld = lam * tp<MT>(P, P.D)[4 * gtid + i]; Dl[i] = (T)ld; Md[i * 5] += ld; }
#pragma unroll
        for (int i = 0; i < 16; ++i) M[i] = (T)Md[i];
        lk = P.link[gtid] != 0;
        if (lk) {
#pragma unroll
          for (int i = 0; i < 16; ++i) E[i] = (T)tp<MT>(P, P.En)[16 * gtid + i];
        }
      }
      T Lr[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) Lr[i] = T(0);
      for (int s = 0; s < 16; ++s) {
        T Sp[16];
        __syncwarp();                                              // converge after the previous step's divergent block
#pragma unroll
        for (int i = 0; i < 16; ++i) Sp[i] = __shfl_up_sync(0xffffffffu, Mi[i], 1);
        if (sl == s) {
          if (lk) {
            mat4_mul(E, Sp, Lr);                                   // L_i = E_i S_{i-1}^-1
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
              for (int j = 0; j < 4; ++j) {                        // S_i = M_i - L_i E_i^T
                T a = T(0);
#pragma unroll
                for (int k = 0; k < 4; ++k) a += Lr[i * 4 + k] * E[j * 4 + k];
                M[i * 4 + j] -= a;
              }
          }
          inv4(M, Mi);
        }
      }
#pragma unroll
      for (int i = 0; i < 16; ++i) Ls[i * GS_THREADS + threadIdx.x] = Lr[i];
      if (is_node) {
#pragma unroll
        for (int i = 0; i < 4; ++i) rn[i] = (T)(-tp<MT>(P, P.g)[4 * gtid + i]);
      }
      chain_apply(Mi, Lr, lk, sl, rn, zn);
      if (gtid < P.n) {
        const T zero4[4] = {T(0), T(0), T(0), T(0)};
        st4(Pres() + 4 * gtid, rn); st4(Pz() + 4 * gtid, zn); st4(Pp() + 4 * gtid, zero4); st4(Pdelta() + 4 * gtid, zero4);
      }
      if (is_node) {
#pragma unroll
        for (int i = 0; i < 4; ++i) { v2[0] += rn[i] * zn[i]; v2[1] += rn[i] * rn[i]; }
      }
    } else {
      for (int n = gtid; n < P.n; n += T_) {
        T rl[4] = {T(0), T(0), T(0), T(0)}, zl[4] = {T(0), T(0), T(0), T(0)};
        if (!P.fixed[n]) {
          double Md[16];
          T M[16];
#pragma unroll
          for (int i = 0; i < 16; ++i) Md[i] = tp<MT>(P, P.Hnn)[16 * n + i];
#pragma unroll
          for (int i = 0; i < 4; ++i) { const double ld = lam * tp<MT>(P, P.D)[4 * n + i]; Dl[i] = (T)ld; Md[i * 5] += ld; }
#pragma unroll
          for (int i = 0; i < 16; ++i) M[i] = (T)Md[i];
          inv4(M, Mi);
#pragma unroll
          for (int i = 0; i < 16; ++i) PMinv()[16 * n + i] = Mi[i];
#pragma unroll
          for (int i = 0; i < 4; ++i) rl[i] = (T)(-tp<MT>(P, P.g)[4 * n + i]);
#pragma unroll
          for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) zl[i] += Mi[i * 4 + j] * rl[j];
        }
        const T zero4[4] = {T(0), T(0), T(0), T(0)};
        st4(Pres() + 4 * n, rl); st4(Pz() + 4 * n, zl); st4(Pp() + 4 * n, zero4); st4(Pdelta() + 4 * n, zero4);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          v2[0] += rl[i] * zl[i]; v2[1] += rl[i] * rl[i];
          rn[i] = rl[i]; zn[i] = zl[i];                       // (fast path: the only iteration of this loop)
        }
      }
    }
    double r2[2];
    grid_reduce_sum<2, MT>(v2, r2, P, parity, sh, grid); parity ^= 1;
    double rz = r2[0];
    const double rr0 = r2[1];
    T beta = T(0);
    int it = 0;
    // ---- PCG iterations: 3 barriers each ----
    while (it < P.opt.max_pcg_iterations && rr0 > 0.0) {
      long long c0 = clock64();
      // factor phase: p_a = z_a + beta p_a (on the fly), t = Ja p_a + Jb p_b, contributions Ja^T t, Jb^T t
      if (fast) {
        // all gathers of this thread's (up to 3) factors are issued before any arithmetic: one L2 round trip
        T zq[GS_KF][2][4], pq[GS_KF][2][4];
#pragma unroll
        for (int k = 0; k < GS_KF; ++k) {
          ld4(Pz() + 4 * fa[k], zq[k][0]); ld4(Pz() + 4 * fb[k], zq[k][1]);
          ld4(Pp() + 4 * fa[k], pq[k][0]); ld4(Pp() + 4 * fb[k], pq[k][1]);
        }
#pragma unroll
        for (int k = 0; k < GS_KF; ++k) {
          if (!fvalid[k]) continue;
          T pa[4], pb[4], ca[4], cb[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) { pa[i] = zq[k][0][i] + beta * pq[k][0][i]; pb[i] = zq[k][1][i] + beta * pq[k][1][i]; }
          factor_apply(J, threadIdx.x + k * GS_THREADS, pa, pb, ca, cb);
          st4(Pcs() + 4 * (size_t)fsa[k], ca);
          st4(Pcs() + 4 * (size_t)fsb[k], cb);
        }
      } else {
        for (int f = f0 + threadIdx.x; f < f1; f += GS_THREADS) {
          const int a = P.ia[f], b = P.ib[f];
          T za[4], zb[4], qa[4], qb[4], pa[4], pb[4], ca[4], cb[4];
          ld4(Pz() + 4 * a, za); ld4(Pz() + 4 * b, zb); ld4(Pp() + 4 * a, qa); ld4(Pp() + 4 * b, qb);
#pragma unroll
          for (int i = 0; i < 4; ++i) { pa[i] = za[i] + beta * qa[i]; pb[i] = zb[i] + beta * qb[i]; }
          factor_apply(J, f - f0, pa, pb, ca, cb);
          st4(Pcs() + 4 * (size_t)P.slot_a[f], ca);
          st4(Pcs() + 4 * (size_t)P.slot_b[f], cb);
        }
      }
      long long c1 = clock64();
      all_sync(P, grid);
      long long c2 = clock64();
      // node phase 1: p = z + beta p, Ap = sum of the node's slots + lam D p, partial p.Ap
      T v1b[1] = {T(0)};
      T apn[4] = {T(0), T(0), T(0), T(0)};
      if (fast) {
        if (is_node) {
#pragma unroll
          for (int i = 0; i < 4; ++i) { pn[i] = zn[i] + beta * pn[i]; apn[i] = Dl[i] * pn[i]; }
          st4(Pp() + 4 * gtid, pn);
          for (int s0 = ns0; s0 < ns1; s0 += 16) {         // 16 (fp32) / 32 (fp64) independent 16-byte loads in flight
            T c[16][4];                                    // per batch: one L2 round trip covers every node of degree <= 16
#pragma unroll
            for (int k = 0; k < 16; ++k) ld4(Pcs() + 4 * (size_t)min(s0 + k, ns1 - 1), c[k]);
#pragma unroll
            for (int k = 0; k < 16; ++k)
              if (s0 + k < ns1) { apn[0] += c[k][0]; apn[1] += c[k][1]; apn[2] += c[k][2]; apn[3] += c[k][3]; }
          }
#pragma unroll
          for (int i = 0; i < 4; ++i) v1b[0] += pn[i] * apn[i];
        }
      } else {
        for (int n = gtid; n < P.n; n += T_) {
          if (P.fixed[n]) continue;
          T zl[4], ql[4], pl[4], ap[4];
          ld4(Pz() + 4 * n, zl); ld4(Pp() + 4 * n, ql);
#pragma unroll
          for (int i = 0; i < 4; ++i) { pl[i] = zl[i] + beta * ql[i]; ap[i] = (T)(lam * tp<MT>(P, P.D)[4 * n + i]) * pl[i]; }
          const int s0 = P.node_ptr[n], s1 = P.node_ptr[n + 1];
#pragma unroll 4
          for (int sidx = s0; sidx < s1; ++sidx) {
            T c[4];
            ld4(Pcs() + 4 * (size_t)sidx, c);
#pragma unroll
            for (int i = 0; i < 4; ++i) ap[i] += c[i];
          }
          st4(Pp() + 4 * n, pl); st4(PAp() + 4 * n, ap);
#pragma unroll
          for (int i = 0; i < 4; ++i) v1b[0] += pl[i] * ap[i];
        }
      }
      long long c3 = clock_after(v1b[0]);
      double r1[1];
      grid_reduce_sum<1, MT>(v1b, r1, P, parity, sh, grid); parity ^= 1;
      long long c4 = clock64();
      const double pAp = r1[0];
      if (!(pAp > 0.0)) break;
      const T alpha = (T)(rz / pAp);
      // node phase 2: delta += alpha p, res -= alpha Ap, z = M^-1 res; partial rz_new, rr
      T v22[2] = {T(0), T(0)};
      if (fast) {
        // (no is_node guard: pn / apn are zero on the other lanes, and a divergent branch here would send the warp
        //  through the slow collective-shuffle path of chain_apply)
#pragma unroll
        for (int i = 0; i < 4; ++i) { dn[i] += alpha * pn[i]; rn[i] -= alpha * apn[i]; }
        if (chain) {                                          // warp-collective: every lane takes part in the sweeps
          T Lr[16];
#pragma unroll
          for (int i = 0; i < 16; ++i) Lr[i] = Ls[i * GS_THREADS + threadIdx.x];
          const long long q0 = clock_after(rn[0] + Lr[15]);
          chain_apply(Mi, Lr, lk, sl, rn, zn);
          const long long q1 = clock_after(zn[0] + zn[3]);
          if (dbg_trial && (threadIdx.x & 31) == 0) P.dbg[8 + solve_rank(P) * (GS_THREADS / 32) + (threadIdx.x >> 5)] += q1 - q0;
        } else if (is_node) {
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            T acc = T(0);
#pragma unroll
            for (int j = 0; j < 4; ++j) acc += Mi[i * 4 + j] * rn[j];
            zn[i] = acc;
          }
        }
        if (is_node) {
          st4(Pz() + 4 * gtid, zn);
#pragma unroll
          for (int i = 0; i < 4; ++i) { v22[0] += rn[i] * zn[i]; v22[1] += rn[i] * rn[i]; }
        }
      } else {
        for (int n = gtid; n < P.n; n += T_) {
          if (P.fixed[n]) continue;
          T dl[4], pl[4], rl[4], al[4], zl[4] = {T(0), T(0), T(0), T(0)};
          ld4(Pdelta() + 4 * n, dl); ld4(Pp() + 4 * n, pl); ld4(Pres() + 4 * n, rl); ld4(PAp() + 4 * n, al);
#pragma unroll
          for (int i = 0; i < 4; ++i) { dl[i] += alpha * pl[i]; rl[i] -= alpha * al[i]; }
#pragma unroll
          for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) zl[i] += PMinv()[16 * n + i * 4 + j] * rl[j];
          st4(Pdelta() + 4 * n, dl); st4(Pres() + 4 * n, rl); st4(Pz() + 4 * n, zl);
#pragma unroll
          for (int i = 0; i < 4; ++i) { v22[0] += rl[i] * zl[i]; v22[1] += rl[i] * rl[i]; }
        }
      }
      long long c5 = clock_after(v22[0] + v22[1]);
      double r22[2];
      grid_reduce_sum<2, MT>(v22, r22, P, parity, sh, grid); parity ^= 1;
      if (dbg_trial && gtid == 0) {
        const long long c6 = clock64();
        P.dbg[0] += c1 - c0; P.dbg[1] += c2 - c1; P.dbg[2] += c3 - c2; P.dbg[3] += c4 - c3; P.dbg[4] += c5 - c4;
        P.dbg[5] += c6 - c5; P.dbg[6] += 1;
      }
      ++it;
      beta = (T)(r22[0] / rz);
      rz = r22[0];
      if (r22[1] <= P.opt.pcg_tolerance * P.opt.pcg_tolerance * rr0) break;
    }
    if (fast && is_node) st4(Pdelta() + 4 * gtid, dn);
    pcg_total += it;
    ++iters;

    // ---- trial point (fp64): x_new = x + delta; g.delta, |delta|^2, |x|^2 ----
    double* xc = tp<MT>(P, cur ? P.x[1] : P.x[0]);
    double* xn = tp<MT>(P, cur ? P.x[0] : P.x[1]);
    double v4[3] = {0.0, 0.0, 0.0}, r4[3];
    for (int n = gtid; n < P.n; n += T_) {
      T dl[4];
      ld4(Pdelta() + 4 * n, dl);
      if (fast && n == gtid && is_node) { dl[0] = dn[0]; dl[1] = dn[1]; dl[2] = dn[2]; dl[3] = dn[3]; }   // (own store)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const double d = P.fixed[n] ? 0.0 : (double)dl[i];
        const double xv = xc[4 * n + i];
        __stcg(xn + 4 * n + i, xv + d);
        v4[0] += tp<MT>(P, P.g)[4 * n + i] * d; v4[1] += d * d;
        if (!P.fixed[n]) v4[2] += xv * xv;
      }
      if (P.fixed[n]) { const T zero4[4] = {T(0), T(0), T(0), T(0)}; st4(Pdelta() + 4 * n, zero4); }
    }
    grid_reduce_sum<3, MT>(v4, r4, P, parity, sh, grid); parity ^= 1;
    // ---- evaluate trial, model decrease, elapsed time ----
    double v5[3] = {0.0, 0.0, 0.0}, r5[3];
    factor_trial<MT>(P, xn, J, v5[0], v5[1]);
    if (gtid == 0) {
      unsigned long long t1;
      asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t1));
      v5[2] = (double)(t1 - t0) * 1e-9;
    }
    grid_reduce_sum<3, MT>(v5, r5, P, parity, sh, grid); parity ^= 1;
    const double new_cost = r5[0];
    const double model = -r4[0] - 0.5 * r5[1];
    const double elapsed = r5[2];
    const double rho = (model > 0.0) ? (cost - new_cost) / model : -1.0;
    const bool finite = isfinite(new_cost);
    const bool small_step = sqrt(r4[1]) <= P.opt.parameter_tolerance * (sqrt(r4[2]) + P.opt.parameter_tolerance);
    if (finite && rho > 1e-3) {
      // accept (Ceres LevenbergMarquardtStrategy::StepAccepted)
      const double tmp = 2.0 * rho - 1.0;
      radius = fmin(radius / fmax(1.0 / 3.0, 1.0 - tmp * tmp * tmp), 1e16);
      decrease = 2.0;
      const double dcost = cost - new_cost;
      const double old_cost = cost;
      cur ^= 1;
      cost = new_cost;
      if (fabs(dcost) <= P.opt.function_tolerance * old_cost) { termination = 0; break; }
      if (small_step) { termination = 2; break; }
      if (P.opt.max_time_s > 0.0 && elapsed > P.opt.max_time_s) { termination = 4; break; }
      // re-linearise at the accepted point (the trial pass kept the old Jacobians for the model term)
      double v1c[1], w1c[1] = {factor_linearize<MT>(P, tp<MT>(P, cur ? P.x[1] : P.x[0]), J)};
      grid_reduce_sum<1, MT>(w1c, v1c, P, parity, sh, grid); parity ^= 1;
      need_gradient = true;
    } else {
      radius /= decrease;
      decrease *= 2.0;
      if (radius < 1e-32 || !isfinite(radius)) { termination = 5; break; }
      if (small_step) { termination = 2; break; }
      if (P.opt.max_time_s > 0.0 && elapsed > P.opt.max_time_s) { termination = 4; break; }
    }
  }

  // ---- write back ----
  const double* xf = tp<MT>(P, cur ? P.x[1] : P.x[0]);
  for (int i = gtid; i < 4 * P.n; i += T_) tp<MT>(P, P.poses_out)[i] = __ldcg(xf + i);
  if (gtid == 0) {
    tp<MT>(P, P.summary)->initial_cost = initial_cost;
    tp<MT>(P, P.summary)->final_cost = cost;
    tp<MT>(P, P.summary)->iterations = iters;
    tp<MT>(P, P.summary)->pcg_iterations = pcg_total;
    tp<MT>(P, P.summary)->termination = termination;
    if (dbg_trial) P.dbg[7] = clock64() - k0;
  }
}

__global__ void graph_linearize_kernel(int m, const double* __restrict__ poses, const int32_t* __restrict__ ftype,
                                       const int32_t* __restrict__ ia, const int32_t* __restrict__ ib,
                                       const double* __restrict__ payload, double* __restrict__ r,
                                       double* __restrict__ Ja, double* __restrict__ Jb) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= m) return;
  double rr[4], A[16], B[16];
  linearize_factor(ftype[f], poses + 4 * ia[f], poses + 4 * ib[f], payload + (size_t)f * OSB_PAYLOAD_LEN, rr, A, B);
  for (int i = 0; i < 4; ++i) r[(size_t)f * 4 + i] = rr[i];
  for (int i = 0; i < 16; ++i) { Ja[(size_t)f * 16 + i] = A[i]; Jb[(size_t)f * 16 + i] = B[i]; }
}

// ---- random-restart initialisation (osb_solver_solve_multistart) ----------------------------------------------------
// Counter-based draws: a value depends only on (seed, trial, caller's node id, component), not on the launch shape, the
// chain plan or the other nodes.  No FMA anywhere, so numpy restates it bit for bit (oracle/multistart_ref.py).
__device__ __forceinline__ uint64_t splitmix64(uint64_t z) {
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
__device__ __forceinline__ double multistart_draw(uint64_t seed, int trial, int node, int comp, double r) {
  const uint64_t key = ((uint64_t)trial << 34) | ((uint64_t)(uint32_t)node << 2) | (uint64_t)comp;
  const double u = (double)(splitmix64(seed ^ splitmix64(key)) >> 11) * 0x1p-53;   // [0, 1)
  return __dadd_rn(__dmul_rn(2.0 * r, u), -r);                                      // [-r, r)
}

// trial t's starting poses, internal order: random_init_pose (solver.cpp:204-216) on the masked free nodes -- x, y in
// +-rand_xy, z in +-rand_z, yaw kept -- and the caller's pose elsewhere.  The caller's poses are trial 0's x0, which
// this kernel rewrites in place.  That is race-free: in trial 0 it writes only x, y, z of the masked free nodes, and
// the other trials read only the yaw of those nodes and the whole pose of the rest.
__global__ void multistart_init_kernel(int n, int n_trials, const uint8_t* __restrict__ fixed,
                                       const int32_t* __restrict__ order, const uint8_t* __restrict__ mask, uint64_t seed,
                                       double rand_xy, double rand_z, double* x0, long long tstride) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)n * n_trials) return;
  const int t = (int)(idx / n), i = (int)(idx - (long long)t * n);
  const int node = order[i];
  double* dst = reinterpret_cast<double*>(reinterpret_cast<char*>(x0) + t * tstride) + 4 * (size_t)i;
  const double* src = x0 + 4 * (size_t)i;
  if (mask[node] && !fixed[i]) {
    dst[0] = multistart_draw(seed, t, node, 0, rand_xy);
    dst[1] = multistart_draw(seed, t, node, 1, rand_xy);
    dst[2] = multistart_draw(seed, t, node, 2, rand_z);
    if (t > 0) dst[3] = src[3];
  } else if (t > 0) {
    for (int k = 0; k < 4; ++k) dst[k] = src[k];
  }
}

// What a call brings back to the host, followed by the poses [n][4] in internal order.  The selection kernel fills one
// on the device and one copy moves it into the handle's pinned mirror; a single solve stages its poses (in and out) and
// its summary in that mirror.
constexpr int MS_MAX_TRIALS = 256;
struct SolveResults {
  int32_t chosen;
  double equv[MS_MAX_TRIALS];
  osb_solve_summary summaries[MS_MAX_TRIALS];
  __host__ __device__ double* poses() { return reinterpret_cast<double*>(this + 1); }
};

// One warp.  equv_cost of every trial (solver.cpp:1721-1725), the acceptance walk of solve_with_multiple_init
// (:783-831: best starts at acpt_cost, strictly lower wins, so the first of equal minima is kept and a NaN never is),
// then the chosen trial's poses.  summary0 / out0: trial 0's summary and output poses, trial t's lie t * tstride further.
__global__ void multistart_select_kernel(int n_trials, int n, const osb_solve_summary* __restrict__ summary0,
                                         const double* __restrict__ out0, long long tstride, int normalise, int n_res,
                                         int window, double acpt_cost, SolveResults* __restrict__ res) {
  const int lane = threadIdx.x;
  int c = -1;
  if (lane == 0) {
    double best = acpt_cost;
    for (int t = 0; t < n_trials; ++t) {
      const osb_solve_summary sm =
          *reinterpret_cast<const osb_solve_summary*>(reinterpret_cast<const char*>(summary0) + t * tstride);
      const double e = normalise ? sqrt(sm.final_cost) / (double)n_res / (double)window : sm.final_cost;
      res->equv[t] = e;
      res->summaries[t] = sm;
      if (e < best) { best = e; c = t; }
    }
    res->chosen = c;
  }
  c = __shfl_sync(0xffffffffu, c, 0);
  if (c < 0) return;
  const double* src = reinterpret_cast<const double*>(reinterpret_cast<const char*>(out0) + c * tstride);
  for (int i = lane; i < 4 * n; i += 32) res->poses()[i] = src[i];
}

// ---- device tail (osb_solver_solve_resident_dev) ---------------------------------------------------------------------
// Each call's tables are those upload_graph builds for (resident factors, then the k tail rows) under the resident plan,
// built on the device in four launches whatever k is.  A node's contribution slots are its base slots, then its tail rows
// in row order; its chain couplings likewise.  The rank of a tail row among the earlier rows that touch the same node is
// the rank inside its chunk of TL_ROWS rows (a compare over the chunk in shared memory) plus the node's count in the
// earlier chunks (a scan down each node's column of per-chunk counts): no atomics, so every table is the same on every run.
constexpr int TL_ROWS = 256;             // tail rows per CTA of tail_rank_kernel (2 slot keys each: one thread per key)

struct TailDev {
  int n, m_base, max_tail, ctas, chunks;
  const int32_t* count;                                              // the caller's k
  const int32_t *type, *ia, *ib; const double* payload; const uint8_t* huber;   // the caller's tail rows (node ids)
  // the resident plan: caller's id -> internal id and back, and the base-only tables of upload_graph
  const int32_t *inv, *order, *b_ia, *b_ib, *b_ptr, *b_slot_a, *b_slot_b, *b_es_ptr, *b_es_slot;
  const uint8_t *b_fixed, *b_link;
  // scratch
  int32_t *key_s, *rank_s;       // [2 max_tail] internal node of slot 2j (node a) / 2j+1 (node b) of row j, -1: none
  int32_t *key_e, *rank_e;       // [max_tail] the later node of a chain coupling, -1: not a coupling
  int32_t *hist_s, *hist_e;      // [chunks][n] per-chunk counts, then (tail_scan_kernel) the earlier chunks' counts
  int32_t *cnt_s, *cnt_e;        // [n] the node's tail slots / couplings, then (tail_ptr_kernel) their exclusive prefix
  int32_t* flag;                 // [chunks][2] refused row seen, tail residuals
  int32_t* word;                 // [0] status, [1] m, [2] fpc, [3] tail residuals
  // the solve's tables (the handle's one-shot buffers) and poses
  int32_t *ia_o, *ib_o, *ptr_o, *slot_a_o, *slot_b_o, *es_ptr_o, *es_slot_o, *type_o;
  double* payload_o;
  uint8_t *huber_o, *fixed_o, *link_o;
  double* poses;                 // [n][4] the resident poses, caller's order
  double *x0, *x_out;            // the solve's start and result, internal order
};

// k, or -1 when *count is outside [0, max_tail]
__device__ __forceinline__ int tail_count(const TailDev& D) {
  const int c = __ldcg(D.count);
  return (c < 0 || c > D.max_tail) ? -1 : c;
}

// one CTA per chunk of TL_ROWS rows: validate, map to internal ids, rank each key inside the chunk, per-chunk counts
__global__ void __launch_bounds__(2 * TL_ROWS) tail_rank_kernel(TailDev D) {
  __shared__ int ks[2 * TL_ROWS], ke[TL_ROWS];
  const int c = blockIdx.x, t = threadIdx.x, k = max(0, tail_count(D));
  const int j = c * TL_ROWS + (t >> 1), side = t & 1;
  int key = -1, ekey = -1, nr = 0;
  bool bad = false;
  if (j < k) {
    const int ty = D.type[j], a = D.ia[j], b = D.ib[j];
    bad = ty < 0 || ty > 2 || a < 0 || a >= D.n || b < 0 || b >= D.n || a == b;
    if (!bad) {
      const int A = D.inv[a], B = D.inv[b], hi = max(A, B);
      key = side ? B : A;
      if (side == 0) {
        if (abs(A - B) == 1 && D.b_link[hi]) ekey = hi;
        nr = ty == OSB_FACTOR_DISTANCE ? 1 : ty == OSB_FACTOR_RELPOSE ? 4
             : (((int)D.payload[(size_t)j * OSB_PAYLOAD_LEN + 10] & 1) ? 3 : 2);
      }
    }
  }
  ks[t] = key;
  if (side == 0) ke[t >> 1] = ekey;
  for (int v = t; v < D.n; v += blockDim.x) { D.hist_s[(size_t)c * D.n + v] = 0; D.hist_e[(size_t)c * D.n + v] = 0; }
  const int any_bad = __syncthreads_or(bad);
  // tail residuals of the chunk: sum of nr in 1..4 as four block counts
  const int n1 = __syncthreads_count(nr >= 1), n2 = __syncthreads_count(nr >= 2), n3 = __syncthreads_count(nr >= 3),
            n4 = __syncthreads_count(nr >= 4);
  if (t == 0) { D.flag[2 * c] = any_bad; D.flag[2 * c + 1] = n1 + n2 + n3 + n4; }
  if (key >= 0) {
    int r = 0;
    bool last = true;
    for (int u = 0; u < 2 * TL_ROWS; ++u)
      if (ks[u] == key) { if (u < t) ++r; else if (u > t) last = false; }
    D.rank_s[2 * j + side] = r;
    if (last) D.hist_s[(size_t)c * D.n + key] = r + 1;
  }
  if (side == 0 && j < D.max_tail) D.key_e[j] = ekey;
  if (ekey >= 0) {
    const int me = t >> 1;
    int r = 0;
    bool last = true;
    for (int u = 0; u < TL_ROWS; ++u)
      if (ke[u] == ekey) { if (u < me) ++r; else if (u > me) last = false; }
    D.rank_e[j] = r;
    if (last) D.hist_e[(size_t)c * D.n + ekey] = r + 1;
  }
}

// one thread per node: the exclusive scan of its per-chunk counts down the chunks, and its tail totals
__global__ void tail_scan_kernel(TailDev D) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= D.n) return;
  int rs = 0, re = 0;
  for (int c = 0; c < D.chunks; ++c) {
    int32_t* hs = D.hist_s + (size_t)c * D.n + v;
    int32_t* he = D.hist_e + (size_t)c * D.n + v;
    const int a = *hs, b = *he;
    *hs = rs; *he = re;
    rs += a; re += b;
  }
  D.cnt_s[v] = rs; D.cnt_e[v] = re;
}

// exclusive scan of v over the 1024 threads of the block; *total = the sum (sh: 32 ints)
__device__ __forceinline__ int block_excl_scan(int v, int* sh, int* total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
  if (lane == 31) sh[w] = x;
  __syncthreads();
  if (w == 0) {
    int s = sh[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, s, o); if (lane >= o) s += y; }
    sh[lane] = s;
  }
  __syncthreads();
  const int r = x - v + (w > 0 ? sh[w - 1] : 0);
  *total = sh[31];
  __syncthreads();
  return r;
}

// one CTA of 1024 threads: the call's status and m, then the CSR pointers of the slots and of the chain couplings
__global__ void __launch_bounds__(1024) tail_ptr_kernel(TailDev D) {
  __shared__ int sh[32];
  __shared__ int status;
  const int kc = tail_count(D);
  int bad = 0, nres = 0;
  for (int c = threadIdx.x; c < D.chunks; c += blockDim.x) { bad |= D.flag[2 * c]; nres += D.flag[2 * c + 1]; }
  bad = __syncthreads_or(bad);
  int nres_total = 0;
  block_excl_scan(nres, sh, &nres_total);
  if (threadIdx.x == 0) {
    const int c = __ldcg(D.count);
    status = kc < 0 ? (c < 0 ? OSB_ERR_INVALID : OSB_ERR_CAPACITY) : bad ? OSB_ERR_INVALID : OSB_OK;
    const int m = D.m_base + max(kc, 0);
    D.word[0] = status; D.word[1] = m; D.word[2] = (m + D.ctas - 1) / D.ctas; D.word[3] = nres_total;
  }
  __syncthreads();
  if (status != OSB_OK) return;
  int carry_s = 0, carry_e = 0;
  for (int v0 = 0; v0 < D.n; v0 += blockDim.x) {
    const int v = v0 + threadIdx.x;
    int ts = 0, te = 0;
    const int xs = block_excl_scan(v < D.n ? D.cnt_s[v] : 0, sh, &ts);
    const int xe = block_excl_scan(v < D.n ? D.cnt_e[v] : 0, sh, &te);
    if (v < D.n) {
      D.cnt_s[v] = carry_s + xs; D.cnt_e[v] = carry_e + xe;
      D.ptr_o[v] = D.b_ptr[v] + carry_s + xs; D.es_ptr_o[v] = D.b_es_ptr[v] + carry_e + xe;
    }
    carry_s += ts; carry_e += te;
  }
  if (threadIdx.x == 0) { D.ptr_o[D.n] = D.b_ptr[D.n] + carry_s; D.es_ptr_o[D.n] = D.b_es_ptr[D.n] + carry_e; }
}

// one thread per factor of (resident, tail) and per node: the factor tables, the tail rows behind the resident factor
// arrays, the node tables and the starting poses in internal order
__global__ void tail_tables_kernel(TailDev D) {
  if (__ldcg(D.word) != OSB_OK) return;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int m = __ldcg(D.word + 1);
  if (i < D.m_base) {
    const int a = D.b_ia[i], b = D.b_ib[i], e = D.b_es_slot[i];
    D.ia_o[i] = a; D.ib_o[i] = b;
    D.slot_a_o[i] = D.b_slot_a[i] + D.cnt_s[a];
    D.slot_b_o[i] = D.b_slot_b[i] + D.cnt_s[b];
    D.es_slot_o[i] = e < 0 ? -1 : e + 2 * D.cnt_e[max(a, b)];
  } else if (i < m) {
    const int j = i - D.m_base, c = j / TL_ROWS;
    const int A = D.inv[D.ia[j]], B = D.inv[D.ib[j]];
    D.ia_o[i] = A; D.ib_o[i] = B;
    D.slot_a_o[i] = D.ptr_o[A] + (D.b_ptr[A + 1] - D.b_ptr[A]) + D.hist_s[(size_t)c * D.n + A] + D.rank_s[2 * j];
    D.slot_b_o[i] = D.ptr_o[B] + (D.b_ptr[B + 1] - D.b_ptr[B]) + D.hist_s[(size_t)c * D.n + B] + D.rank_s[2 * j + 1];
    const int hi = D.key_e[j];
    D.es_slot_o[i] = hi < 0 ? -1
        : 2 * (D.es_ptr_o[hi] + (D.b_es_ptr[hi + 1] - D.b_es_ptr[hi]) + D.hist_e[(size_t)c * D.n + hi] + D.rank_e[j]) +
          (A == hi ? 1 : 0);
    D.type_o[i] = D.type[j]; D.huber_o[i] = D.huber[j];
    for (int q = 0; q < OSB_PAYLOAD_LEN; ++q)
      D.payload_o[(size_t)i * OSB_PAYLOAD_LEN + q] = D.payload[(size_t)j * OSB_PAYLOAD_LEN + q];
  }
  if (i < D.n) {
    D.fixed_o[i] = D.b_fixed[i]; D.link_o[i] = D.b_link[i];
    const int src = D.order[i];
#pragma unroll
    for (int q = 0; q < 4; ++q) D.x0[4 * i + q] = D.poses[4 * src + q];
  }
}

// the solution back into the resident poses (caller's order); a refused call leaves them as they were
__global__ void tail_poses_out_kernel(TailDev D) {
  if (__ldcg(D.word) != OSB_OK) return;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= D.n) return;
  const int dst = D.order[i];
#pragma unroll
  for (int q = 0; q < 4; ++q) D.poses[4 * dst + q] = __ldcg(D.x_out + 4 * i + q);
}

}  // namespace osb

using namespace osb;

// Launch shape of one solve.  It depends on the graph's size and the options only, never on how many solves run at once,
// so that a trial of osb_solver_solve_multistart runs exactly the arithmetic of osb_solver_solve.
struct SolveShape {
  bool f32;              // fp32 inner (PCG) arithmetic
  const void* kern;      // one solve per launch
  const void* kern_multi;  // several clusters per launch, one trial each (same resources, same arithmetic)
  const void* kern_dt;     // one solve whose factor count is read on the device (osb_solver_solve_resident_dev)
  int cluster;           // 1: one thread-block cluster per solve (hardware barrier); 0: one cooperative grid per launch
  int ctas, fpc, chain, jsmem;
  size_t smem;           // dynamic shared memory per CTA
};

// The state of one solve (SolverDev::x .. En) laid out from `base`: points P's state pointers into that block and returns
// its bytes (base == nullptr: only the size).  Every buffer starts on a 256-byte boundary, as its own cudaMalloc would.
static size_t trial_layout(SolverDev& P, char* base, size_t n, size_t m, const SolveShape& s) {
  const size_t d = sizeof(double), tsz = s.f32 ? sizeof(float) : sizeof(double);
  size_t at = 0;
  auto take = [&](auto*& p, size_t bytes) {
    p = reinterpret_cast<std::remove_reference_t<decltype(p)>>(reinterpret_cast<uintptr_t>(base) + at);
    at += (bytes + 255) & ~(size_t)255;
  };
  take(P.x[0], 4 * n * d); take(P.x[1], 4 * n * d); take(P.poses_out, 4 * n * d);
  take(P.g, 4 * n * d); take(P.D, 4 * n * d); take(P.Hnn, 16 * n * d); take(P.En, 16 * n * d);
  take(P.Minv, 16 * n * tsz); take(P.p, 4 * n * tsz); take(P.z, 4 * n * tsz); take(P.res, 4 * n * tsz);
  take(P.Ap, 4 * n * tsz); take(P.delta, 4 * n * tsz);
  take(P.gs, 8 * m * d); take(P.hs, 32 * m * d); take(P.es, 16 * m * d); take(P.cs, 8 * m * tsz);
  take(P.Jg, s.jsmem ? 0 : 32 * m * tsz);
  take(P.partial, 2 * 4 * (size_t)s.ctas * d);
  take(P.summary, sizeof(osb_solve_summary));
  return at;
}

struct osb_solver {
  Resources res;
  int max_nodes = 0, max_factors = 0;
  bool cluster_ok = false;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  std::mutex mu;
  // device: the graph tables
  uint8_t *d_fixed = nullptr, *d_huber = nullptr;
  int32_t *d_type = nullptr, *d_ia = nullptr, *d_ib = nullptr, *d_ptr = nullptr, *d_slot_a = nullptr, *d_slot_b = nullptr;
  double* d_payload = nullptr;
  uint8_t* d_link = nullptr;
  int32_t *d_es_ptr = nullptr, *d_es_slot = nullptr;
  // the state of the solves: trial blocks of trial_layout, one after another.  osb_solver_create sizes it for one trial
  // at the handle's capacity, so a single solve never allocates; osb_solver_solve_multistart grows it to K blocks.
  char* d_arena = nullptr;
  size_t arena_bytes = 0;
  // osb_solver_solve_multistart's inputs (internal -> caller's node id, init mask) and results
  int32_t* d_order = nullptr;
  uint8_t* d_mask = nullptr;
  SolveResults* d_res = nullptr;
  double* d_lin = nullptr;        // osb_solver_linearize: poses [n][4], r [m][4], Ja, Jb [m][16]
  long long* d_dbg = nullptr;
  // pinned staging for what crosses PCIe on EVERY solve (poses in, poses + summary out): a copy to / from pageable memory
  // blocks inside the driver until the stream reaches it -- for the results that is the whole solve, and other host threads
  // (the keyframe front-end of the same process) could not launch meanwhile (measured: 640 -> 57 keyframes/s beside a
  // back-to-back solver thread).  Pinned copies are asynchronous; the one wait is a cudaStreamSynchronize.
  SolveResults* h_res = nullptr;
  int device = 0;
  SolveShape last_shape = {};
  // resident graph (osb_solver_graph_*): host mirrors of what is already in device memory
  std::vector<double> g_poses, g_payload;
  std::vector<uint8_t> g_fixed, g_huber;
  std::vector<int32_t> g_type, g_ia, g_ib;
  size_t g_uploaded = 0;            // factors whose type / huber / payload are already on the device
  bool g_static_valid = false;      // false after a one-shot osb_solver_solve overwrote the device factor arrays
  // topology cache of the resident graph: the path cover, the internal numbering and the CSR / slot tables depend only on
  // (fixed, type, ia, ib, payload weights), not on the poses -- a window that is re-solved without new frames (or after
  // set_poses) re-uses them on the host AND on the device (0.5 ms of host work per solve otherwise)
  unsigned long long g_topo_version = 1, cached_topo = 0;
  std::vector<int32_t> cached_order;
  int cached_nres = 0;
  // device tail (osb_solver_solve_resident_dev).  The resident plan's base-only tables live in d_tail (acquired by the
  // first device call, carved by tail_layout) beside the call's scratch, so a one-shot solve never overwrites them.
  char* d_tail = nullptr;
  TailDev tail = {};                // d_tail's pointers
  double* d_rposes = nullptr;       // the resident poses on the device, caller's order
  osb_solve_summary* d_tsummary = nullptr;
  cudaEvent_t ev_done = nullptr;
  unsigned long long tail_topo = 0; // topology the base tables were built for
  std::vector<int32_t> tail_order;
  int tail_nres = 0;                // residuals of the resident factors
  bool rposes_current = false;      // d_rposes holds g_poses (false: the next device call uploads them)
  long long tail_shape_key = -1;    // (n, m + max_tail, precision, preconditioner) of tail_shape
  SolveShape tail_shape = {};
  // the last device call: pending until a host-side call synchronises with it and refreshes g_poses from d_rposes
  bool dev_pending = false, dev_captured = false, dev_called = false;
  osb_status dev_status = OSB_OK;
  osb_solve_summary dev_summary = {};
};

static osb_status finish_device_call(osb_solver* h);

extern "C" void osb_solve_default_options(osb_solve_options* o) {
  if (!o) return;
  o->max_iterations = 1000;         // swarm_localization_solver.cpp:1697
  o->max_pcg_iterations = 500;
  o->max_time_s = 0.0;
  o->function_tolerance = 1e-6;     // Ceres defaults
  o->gradient_tolerance = 1e-10;
  o->parameter_tolerance = 1e-8;
  o->pcg_tolerance = 1e-2;
  o->preconditioner = OSB_PRECOND_AUTO;
  o->inner_precision = OSB_INNER_AUTO;
  o->initial_trust_radius = 1e4;
}

extern "C" osb_status osb_solver_create(osb_solver** out, int max_nodes, int max_factors) {
  OSB_REQUIRE(out != nullptr && max_nodes > 0 && max_factors > 0, "bad sizes");
  OSB_TRY(require_device());
  std::unique_ptr<osb_solver> h(new osb_solver());
  h->max_nodes = max_nodes; h->max_factors = max_factors;
  const size_t n = max_nodes, m = max_factors;
  OSB_TRY(h->res.stream(&h->stream));
  OSB_TRY(h->res.event(&h->ev0));
  OSB_TRY(h->res.event(&h->ev1));
  h->cluster_ok = true;
  for (const void* k : {(const void*)graph_solve_kernel<float, false>, (const void*)graph_solve_kernel<double, false>,
                        (const void*)graph_solve_kernel<float, true>, (const void*)graph_solve_kernel<double, true>,
                        (const void*)graph_solve_kernel<float, false, true>,
                        (const void*)graph_solve_kernel<double, false, true>}) {
    OSB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, GS_SMEM_DYN_MAX));
    h->cluster_ok = h->cluster_ok && cudaFuncSetAttribute(k, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) == cudaSuccess;
  }
  cudaGetLastError();
  OSB_TRY(h->res.alloc(&h->d_fixed, n));
  OSB_TRY(h->res.alloc(&h->d_huber, m));
  OSB_TRY(h->res.alloc(&h->d_type, m));
  OSB_TRY(h->res.alloc(&h->d_ia, m));
  OSB_TRY(h->res.alloc(&h->d_ib, m));
  OSB_TRY(h->res.alloc(&h->d_slot_a, m));
  OSB_TRY(h->res.alloc(&h->d_slot_b, m));
  OSB_TRY(h->res.alloc(&h->d_ptr, n + 1));
  OSB_TRY(h->res.alloc(&h->d_payload, m * OSB_PAYLOAD_LEN));
  OSB_TRY(h->res.alloc(&h->d_link, n));
  OSB_TRY(h->res.alloc(&h->d_es_ptr, n + 1));
  OSB_TRY(h->res.alloc(&h->d_es_slot, m));
  // one trial of the worst shape: fp64 Jacobians in global memory, partials for a cooperative grid of every SM
  SolveShape worst = {};
  worst.ctas = num_sms();
  SolverDev unbound = {};
  h->arena_bytes = trial_layout(unbound, nullptr, n, m, worst);
  OSB_TRY(h->res.alloc(&h->d_arena, h->arena_bytes));
  OSB_TRY(h->res.alloc(&h->d_order, n));
  OSB_TRY(h->res.alloc(&h->d_mask, n));
  OSB_TRY(h->res.alloc((char**)&h->d_res, sizeof(SolveResults) + 4 * n * sizeof(double)));
  OSB_TRY(h->res.host_alloc((char**)&h->h_res, sizeof(SolveResults) + 4 * n * sizeof(double), cudaHostAllocDefault));
  OSB_TRY(h->res.alloc(&h->d_lin, 4 * n + 36 * m));
  OSB_TRY(h->res.alloc(&h->d_dbg, 8 + 128));
  OSB_CUDA(cudaMemset(h->d_dbg, 0, (8 + 128) * sizeof(long long)));
  h->device = current_device();
  *out = h.release();
  return OSB_OK;
}

extern "C" osb_status osb_solver_destroy(osb_solver* h) {
  delete h;
  return OSB_OK;
}


// ---- host: path cover + node numbering for the chain preconditioner ------------------------------------------------
// Greedy maximum-weight path cover: factors sorted by information weight (descending, ties by index), a factor joins two
// free nodes when both still have degree < 2 and lie in different components (union-find: no cycles).  On a swarm graph
// this recovers every drone's odometry chain (ego-motion edges carry ~100x the information of loops / UWB).  Nodes are
// then numbered path by path (fixed nodes last); link[i] = 1 iff node i-1 precedes i on its path and i % 16 != 0.
struct ChainPlan {
  std::vector<int32_t> order;   // new id -> caller's id
  std::vector<int32_t> inv;     // caller's id -> new id
  std::vector<uint8_t> link;    // by new id
};

static double factor_weight(int type, const double* pl) {
  if (type == OSB_FACTOR_DISTANCE) return pl[1] * pl[1];
  if (type == OSB_FACTOR_RELPOSE) { double w = 0.0; for (int i = 4; i < 20; ++i) w += pl[i] * pl[i]; return w; }
  return pl[20] > 0.0 ? 1.0 / (pl[20] * pl[20]) : 0.0;
}

static void build_chain_plan(int n, const uint8_t* fixed, int m, const int32_t* type, const int32_t* ia, const int32_t* ib,
                             const double* payload, ChainPlan& pl) {
  // sort key: (inverted bits of the weight as a non-negative float) : factor index -> ascending u64 order is weight
  // descending, ties by index (weights only need float resolution here)
  std::vector<uint64_t> keys(m);
  for (int f = 0; f < m; ++f) {
    const float wf = (float)factor_weight(type[f], payload + (size_t)f * OSB_PAYLOAD_LEN);
    uint32_t bits;
    std::memcpy(&bits, &wf, sizeof(bits));
    keys[f] = ((uint64_t)(~bits) << 32) | (uint32_t)f;
  }
  std::sort(keys.begin(), keys.end());
  std::vector<int32_t> parent(n), nb0(n, -1), nb1(n, -1);
  for (int i = 0; i < n; ++i) parent[i] = i;
  auto find = [&](int x) { while (parent[x] != x) { parent[x] = parent[parent[x]]; x = parent[x]; } return x; };
  for (uint64_t key : keys) {
    const int32_t f = (int32_t)(key & 0xffffffffu);
    const int a = ia[f], b = ib[f];
    if (fixed[a] || fixed[b] || nb1[a] >= 0 || nb1[b] >= 0) continue;
    const int ra = find(a), rb = find(b);
    if (ra == rb) continue;
    parent[ra] = rb;
    (nb0[a] < 0 ? nb0[a] : nb1[a]) = b;
    (nb0[b] < 0 ? nb0[b] : nb1[b]) = a;
  }
  pl.order.clear(); pl.order.reserve(n);
  pl.inv.assign(n, -1); pl.link.assign(n, 0);
  for (int s0 = 0; s0 < n; ++s0) {
    if (fixed[s0] || pl.inv[s0] >= 0 || nb1[s0] >= 0) continue;      // start at path ends (degree <= 1)
    int prev = -1, cur = s0;
    while (cur >= 0) {
      const int id = (int)pl.order.size();
      pl.inv[cur] = id; pl.order.push_back(cur);
      if (prev >= 0 && (id % 16) != 0) pl.link[id] = 1;
      const int nxt = (nb0[cur] >= 0 && nb0[cur] != prev) ? nb0[cur] : (nb1[cur] >= 0 && nb1[cur] != prev) ? nb1[cur] : -1;
      prev = cur; cur = nxt;
    }
  }
  for (int i = 0; i < n; ++i)
    if (pl.inv[i] < 0) { pl.inv[i] = (int)pl.order.size(); pl.order.push_back(i); }   // fixed nodes last
}

// host-only view of the plan (tests): order_out[new] = caller's node id, link_out[new]
extern "C" osb_status osb_solver_chain_plan(int n_nodes, const uint8_t* fixed, int n_factors, const int32_t* type,
                                            const int32_t* ia, const int32_t* ib, const double* payload,
                                            int32_t* order_out, uint8_t* link_out) {
  OSB_REQUIRE(fixed && type && ia && ib && payload && order_out && link_out && n_nodes > 0 && n_factors > 0, "bad argument");
  for (int f = 0; f < n_factors; ++f)
    OSB_REQUIRE(ia[f] >= 0 && ia[f] < n_nodes && ib[f] >= 0 && ib[f] < n_nodes && ia[f] != ib[f], "bad factor indices");
  ChainPlan pl;
  build_chain_plan(n_nodes, fixed, n_factors, type, ia, ib, payload, pl);
  for (int i = 0; i < n_nodes; ++i) { order_out[i] = pl.order[i]; link_out[i] = pl.link[i]; }
  return OSB_OK;
}

static osb_status validate_graph(int n_nodes, int n_factors, const int32_t* type, const int32_t* ia, const int32_t* ib) {
  for (int f = 0; f < n_factors; ++f) {
    OSB_REQUIRE(type[f] >= 0 && type[f] <= 2, "unknown factor type");
    OSB_REQUIRE(ia[f] >= 0 && ia[f] < n_nodes && ib[f] >= 0 && ib[f] < n_nodes, "factor node index out of range");
    // the reference skips factors whose two parameter blocks coincide (solver.cpp:1071-1073,1176)
    OSB_REQUIRE(ia[f] != ib[f], "factor connects a pose block to itself (the adapter must skip it)");
  }
  return OSB_OK;
}

// The index tables of one factor list under a chain plan: internal ids, the CSR of contribution slots, the chain
// couplings, the fixed flags in internal order and the residual count.
struct GraphTables {
  std::vector<int32_t> ia, ib, ptr, slot_a, slot_b, es_ptr, es_slot;
  std::vector<uint8_t> fixed;
  int n_res = 0;
};

static void build_tables(int n_nodes, const uint8_t* fixed, int n_factors, const int32_t* type, const int32_t* ia,
                         const int32_t* ib, const double* payload, const ChainPlan& plan, GraphTables& t) {
  const size_t n = n_nodes, m = n_factors;
  std::vector<int32_t>& ia_p = t.ia; std::vector<int32_t>& ib_p = t.ib;
  ia_p.resize(m); ib_p.resize(m);
  std::vector<uint8_t>& fixed_p = t.fixed;
  fixed_p.resize(n);
  for (size_t f = 0; f < m; ++f) { ia_p[f] = plan.inv[ia[f]]; ib_p[f] = plan.inv[ib[f]]; }
  for (size_t i = 0; i < n; ++i) fixed_p[i] = fixed[plan.order[i]];
  // chain couplings: factor f couples node hi with hi-1 when its two nodes are consecutive and linked
  std::vector<int32_t>& es_ptr = t.es_ptr; std::vector<int32_t>& es_slot = t.es_slot;
  es_ptr.assign(n + 1, 0); es_slot.assign(m, -1);
  for (size_t f = 0; f < m; ++f) {
    const int a = ia_p[f], b = ib_p[f], hi = std::max(a, b);
    if (std::abs(a - b) == 1 && plan.link[hi]) es_ptr[hi + 1]++;
  }
  for (size_t i = 0; i < n; ++i) es_ptr[i + 1] += es_ptr[i];
  {
    std::vector<int32_t> fill(es_ptr.begin(), es_ptr.end() - 1);
    for (size_t f = 0; f < m; ++f) {
      const int a = ia_p[f], b = ib_p[f], hi = std::max(a, b);
      if (std::abs(a - b) == 1 && plan.link[hi]) es_slot[f] = 2 * (fill[hi]++) + (a == hi ? 1 : 0);
    }
  }
  // CSR of contribution slots: node n owns slots [ptr[n], ptr[n+1]); factors in index order within a node, so the
  // gather order -- and therefore every floating-point sum -- is fixed.
  std::vector<int32_t>& ptr = t.ptr; std::vector<int32_t>& slot_a = t.slot_a; std::vector<int32_t>& slot_b = t.slot_b;
  ptr.assign(n + 1, 0); slot_a.resize(m); slot_b.resize(m);
  for (size_t f = 0; f < m; ++f) { ptr[ia_p[f] + 1]++; ptr[ib_p[f] + 1]++; }
  for (size_t i = 0; i < n; ++i) ptr[i + 1] += ptr[i];
  {
    std::vector<int32_t> fill(ptr.begin(), ptr.end() - 1);
    for (size_t f = 0; f < m; ++f) { slot_a[f] = fill[ia_p[f]]++; slot_b[f] = fill[ib_p[f]]++; }
  }
  int& n_res = t.n_res;
  n_res = 0;
  for (size_t f = 0; f < m; ++f)
    n_res += type[f] == OSB_FACTOR_DISTANCE ? 1 : type[f] == OSB_FACTOR_RELPOSE ? 4
             : (((int)payload[f * OSB_PAYLOAD_LEN + 10] & 1) ? 3 : 2);
}

// Upload the graph of one solve and the caller's poses: the chain plan, the internal numbering and the index tables
// (unless the resident graph's topology is unchanged), the factor arrays when upload_static (the resident entry point has
// already appended them), then the poses in internal order into x0 through the pinned staging.  The caller holds h->mu.
static osb_status upload_graph(osb_solver* h, int n_nodes, const double* poses, const uint8_t* fixed, int n_factors,
                               const int32_t* type, const int32_t* ia, const int32_t* ib, const double* payload,
                               const uint8_t* huber, bool upload_static, unsigned long long topo_key, double* x0) {
  // Internal node numbering: the paths of the chain plan are runs of consecutive ids (fixed nodes last).  Everything on
  // the device uses the internal ids; poses are permuted on the way in and out.
  const size_t n = n_nodes, m = n_factors;
  cudaStream_t st = h->stream;
  // resident graph with unchanged topology: plan, numbering and every index table are already on the device
  const bool reuse = topo_key != 0 && topo_key == h->cached_topo && h->cached_order.size() == n;
  if (!reuse) {
    ChainPlan plan;
    build_chain_plan(n_nodes, fixed, n_factors, type, ia, ib, payload, plan);
    GraphTables t;
    build_tables(n_nodes, fixed, n_factors, type, ia, ib, payload, plan, t);
    const std::vector<int32_t> &ia_p = t.ia, &ib_p = t.ib, &ptr = t.ptr, &slot_a = t.slot_a, &slot_b = t.slot_b;
    const std::vector<int32_t> &es_ptr = t.es_ptr, &es_slot = t.es_slot;
    const std::vector<uint8_t>& fixed_p = t.fixed;
    const int n_res = t.n_res;
    OSB_CUDA(cudaMemcpyAsync(h->d_fixed, fixed_p.data(), n, cudaMemcpyHostToDevice, st));
    if (upload_static) {
      OSB_CUDA(cudaMemcpyAsync(h->d_huber, huber, m, cudaMemcpyHostToDevice, st));
      OSB_CUDA(cudaMemcpyAsync(h->d_type, type, m * sizeof(int32_t), cudaMemcpyHostToDevice, st));
      OSB_CUDA(cudaMemcpyAsync(h->d_payload, payload, m * OSB_PAYLOAD_LEN * sizeof(double), cudaMemcpyHostToDevice, st));
    }
    OSB_CUDA(cudaMemcpyAsync(h->d_ia, ia_p.data(), m * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    OSB_CUDA(cudaMemcpyAsync(h->d_ib, ib_p.data(), m * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    OSB_CUDA(cudaMemcpyAsync(h->d_ptr, ptr.data(), (n + 1) * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    OSB_CUDA(cudaMemcpyAsync(h->d_slot_a, slot_a.data(), m * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    OSB_CUDA(cudaMemcpyAsync(h->d_slot_b, slot_b.data(), m * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    OSB_CUDA(cudaMemcpyAsync(h->d_link, plan.link.data(), n, cudaMemcpyHostToDevice, st));
    OSB_CUDA(cudaMemcpyAsync(h->d_es_ptr, es_ptr.data(), (n + 1) * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    OSB_CUDA(cudaMemcpyAsync(h->d_es_slot, es_slot.data(), m * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    // the staging vectors above die at the end of this block: the copies must have left them
    OSB_CUDA(cudaStreamSynchronize(st));
    h->cached_order = plan.order;
    h->cached_nres = n_res;
    h->cached_topo = topo_key;               // 0 (one-shot solve) never matches
  }
  double* xs = h->h_res->poses();
  for (size_t i = 0; i < n; ++i)
    for (int k = 0; k < 4; ++k) xs[4 * i + k] = poses[4 * (size_t)h->cached_order[i] + k];
  OSB_CUDA(cudaMemcpyAsync(x0, xs, 4 * n * sizeof(double), cudaMemcpyHostToDevice, st));
  return OSB_OK;
}

static osb_status solve_shape(const osb_solver* h, int n_nodes, int n_factors, const osb_solve_options& o, SolveShape& s) {
  // inner precision: fp32 PCG unless the caller asks for a tighter inner solve than fp32 can deliver
  s.f32 = o.inner_precision == OSB_INNER_FP32 || (o.inner_precision == OSB_INNER_AUTO && o.pcg_tolerance >= 1e-4);
  const size_t tsz = s.f32 ? sizeof(float) : sizeof(double);
  s.kern = s.f32 ? (const void*)graph_solve_kernel<float, false> : (const void*)graph_solve_kernel<double, false>;
  s.kern_multi = s.f32 ? (const void*)graph_solve_kernel<float, true> : (const void*)graph_solve_kernel<double, true>;
  s.kern_dt = s.f32 ? (const void*)graph_solve_kernel<float, false, true> : (const void*)graph_solve_kernel<double, false, true>;
  s.chain = 0;
  // ONE thread-block cluster (hardware barrier, ~0.2 us) when the factor list fits 16 CTAs with their Jacobians in
  // shared memory; otherwise a cooperative grid (software grid barrier).
  {
    const int G = std::max(1, std::min(GS_MAX_CLUSTER, cdiv(std::max(n_nodes, n_factors), GS_THREADS)));
    const int fpc = cdiv(n_factors, G);
    const size_t jbytes = (size_t)fpc * 32 * tsz, cbytes = (size_t)16 * GS_THREADS * tsz;
    if (h->cluster_ok && jbytes <= (size_t)GS_SMEM_J_MAX && cdiv(n_nodes, GS_THREADS) <= 4 * G) {
      // chain preconditioner: needs the fast path (one thread per node, <= GS_KF factors per thread) and room for L
      const bool chain = o.preconditioner != OSB_PRECOND_BLOCK_JACOBI && fpc <= GS_KF * GS_THREADS &&
                         n_nodes <= G * GS_THREADS && jbytes + cbytes <= (size_t)GS_SMEM_DYN_MAX;
      cudaLaunchConfig_t cfg = {};
      cudaLaunchAttribute attr[1];
      cfg.blockDim = dim3(GS_THREADS); cfg.gridDim = dim3(G); cfg.stream = h->stream; cfg.attrs = attr; cfg.numAttrs = 1;
      cfg.dynamicSmemBytes = jbytes + (chain ? cbytes : 0);
      attr[0].id = cudaLaunchAttributeClusterDimension;
      attr[0].val.clusterDim.x = G; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
      int nclusters = 0;
      if (cudaOccupancyMaxActiveClusters(&nclusters, s.kern, &cfg) == cudaSuccess && nclusters >= 1) {
        s.cluster = 1; s.ctas = G; s.fpc = fpc; s.chain = chain ? 1 : 0; s.jsmem = 1; s.smem = cfg.dynamicSmemBytes;
        return OSB_OK;
      }
      cudaGetLastError();
    }
  }
  int per_sm = 0;
  const int G0 = std::max(1, std::min(num_sms(), cdiv(std::max(n_nodes, n_factors), GS_THREADS)));
  const int fpc = cdiv(n_factors, G0);
  const size_t jbytes = (size_t)fpc * 32 * tsz;
  s.jsmem = (jbytes <= (size_t)GS_SMEM_J_MAX) ? 1 : 0;
  s.smem = s.jsmem ? jbytes : 0;
  OSB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, s.kern, GS_THREADS, s.smem));
  if (per_sm < 1) { set_error("osb_solver_solve", "solve kernel cannot be made resident"); return OSB_ERR_CUDA; }
  s.cluster = 0; s.ctas = G0; s.fpc = fpc;
  return OSB_OK;
}

// the graph tables on the device (shared by every trial) and the solve's options
static SolverDev graph_dev(const osb_solver* h, int n_nodes, int n_factors, const osb_solve_options& o) {
  SolverDev P = {};
  P.n = n_nodes; P.m = n_factors;
  P.fixed = h->d_fixed; P.ftype = h->d_type; P.ia = h->d_ia; P.ib = h->d_ib; P.huber = h->d_huber;
  P.payload = h->d_payload; P.node_ptr = h->d_ptr; P.slot_a = h->d_slot_a; P.slot_b = h->d_slot_b;
  P.link = h->d_link; P.es_ptr = h->d_es_ptr; P.es_slot = h->d_es_slot;
  P.opt = o; P.dbg = h->d_dbg;
  return P;
}

// n_trials solves of one shape, P bound at trial 0 = the start of the arena, trial t's block tstride bytes further.
// Cluster path: ONE launch of n_trials clusters (clusters do not wait for each other, so the grid may exceed what is
// resident).  Cooperative path: one grid per trial, in order on the stream.  dt: the one solve of
// osb_solver_solve_resident_dev, on the caller's stream `st`.
static osb_status launch_solves(osb_solver* h, SolverDev P, const SolveShape& s, int n_trials, long long tstride,
                                cudaStream_t st, bool dt = false) {
  P.fpc = s.fpc; P.use_cluster = s.cluster; P.j_in_smem = s.jsmem; P.use_chain = s.chain;
  P.ctas = s.ctas; P.first_trial = 0; P.tstride = tstride;
  h->last_shape = s;
  cudaLaunchConfig_t cfg = {};
  cudaLaunchAttribute attr[1];
  cfg.blockDim = dim3(GS_THREADS); cfg.stream = st; cfg.attrs = attr; cfg.numAttrs = 1;
  cfg.dynamicSmemBytes = s.smem;
  const void* single = dt ? s.kern_dt : s.kern;
  if (s.cluster) {
    cfg.gridDim = dim3(n_trials * s.ctas);
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = s.ctas; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    void* kargs[1] = {&P};
    OSB_CUDA(cudaLaunchKernelExC(&cfg, n_trials > 1 ? s.kern_multi : single, kargs));
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return OSB_OK;
  }
  cfg.gridDim = dim3(s.ctas);
  attr[0].id = cudaLaunchAttributeCooperative;
  attr[0].val.cooperative = 1;
  for (int t = 0; t < n_trials; ++t) {
    SolverDev Q = P;
    Q.first_trial = t;
    trial_layout(Q, h->d_arena + t * tstride, P.n, P.m, s);
    if (dt) Q.summary = P.summary;
    void* kargs[1] = {&Q};
    OSB_CUDA(cudaLaunchKernelExC(&cfg, single, kargs));
    g_launches.fetch_add(1, std::memory_order_relaxed);
  }
  return OSB_OK;
}

// One call of the solver, shared by every entry point: pick the shape, lay the trials out in the arena, upload the graph
// and the caller's poses into trial 0's x0, launch, copy back, and return the poses in the caller's numbering.
// ms == nullptr: one solve from the caller's poses, its summary in summaries[0].  Otherwise ms->n_trials random
// restarts of the init_mask nodes, ranked on the device: summaries and equv [K], chosen, and the chosen trial's poses
// (the caller's stay as they were when no trial is accepted).  upload_static: see upload_graph.  The caller holds h->mu.
static osb_status solver_run(osb_solver* h, int n_nodes, double* poses, const uint8_t* fixed, int n_factors,
                             const int32_t* type, const int32_t* ia, const int32_t* ib, const double* payload,
                             const uint8_t* huber, bool upload_static, unsigned long long topo_key,
                             const osb_solve_options* opt, const osb_multistart_options* ms, const uint8_t* init_mask,
                             osb_solve_summary* summaries, double* equv = nullptr, int32_t* chosen = nullptr) {
  osb_solve_options o;
  if (opt) o = *opt; else osb_solve_default_options(&o);
  const int K = ms ? ms->n_trials : 1;
  const size_t n = n_nodes;
  cudaStream_t st = h->stream;
  SolveShape shape;
  osb_status s = solve_shape(h, n_nodes, n_factors, o, shape);
  if (s != OSB_OK) return s;
  SolverDev P = graph_dev(h, n_nodes, n_factors, o);
  const size_t tstride = trial_layout(P, nullptr, n, n_factors, shape);
  if (K * tstride > h->arena_bytes) {     // multistart only; a failed allocation leaves the old arena in place
    char* grown = nullptr;
    OSB_TRY(h->res.alloc(&grown, K * tstride));
    h->res.release(h->d_arena);
    h->d_arena = grown;
    h->arena_bytes = K * tstride;
  }
  trial_layout(P, h->d_arena, n, n_factors, shape);
  s = upload_graph(h, n_nodes, poses, fixed, n_factors, type, ia, ib, payload, huber, upload_static, topo_key, P.x[0]);
  if (s != OSB_OK) return s;
  if (ms) {
    OSB_CUDA(cudaMemcpyAsync(h->d_order, h->cached_order.data(), n * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    OSB_CUDA(cudaMemcpyAsync(h->d_mask, init_mask, n, cudaMemcpyHostToDevice, st));
    const long long kn = (long long)K * n_nodes;
    OSB_LAUNCH(multistart_init_kernel, (unsigned)((kn + 255) / 256), 256, 0, st, n_nodes, K, h->d_fixed, h->d_order,
               h->d_mask, ms->seed, ms->rand_xy, ms->rand_z, P.x[0], (long long)tstride);
    OSB_CHECK_LAUNCH();
  }
  OSB_CUDA(cudaEventRecord(h->ev0, st));
  s = launch_solves(h, P, shape, K, (long long)tstride, st);
  if (s != OSB_OK) return s;
  OSB_CUDA(cudaEventRecord(h->ev1, st));
  SolveResults* r = h->h_res;
  if (ms) {
    OSB_LAUNCH(multistart_select_kernel, 1, 32, 0, st, K, n_nodes, P.summary, P.poses_out, (long long)tstride,
               ms->normalise ? 1 : 0, h->cached_nres, ms->window_size, ms->acpt_cost, h->d_res);
    OSB_CHECK_LAUNCH();
    OSB_CUDA(cudaMemcpyAsync(r, h->d_res, sizeof(SolveResults) + 4 * n * sizeof(double), cudaMemcpyDeviceToHost, st));
  } else {
    OSB_CUDA(cudaMemcpyAsync(r->poses(), P.poses_out, 4 * n * sizeof(double), cudaMemcpyDeviceToHost, st));
    OSB_CUDA(cudaMemcpyAsync(&r->summaries[0], P.summary, sizeof(osb_solve_summary), cudaMemcpyDeviceToHost, st));
  }
  OSB_CUDA(cudaStreamSynchronize(st));
  float msec = 0.f;
  OSB_CUDA(cudaEventElapsedTime(&msec, h->ev0, h->ev1));
  for (int t = 0; t < K; ++t) {
    summaries[t] = r->summaries[t];
    summaries[t].solve_ms = msec;
    summaries[t].n_residuals = h->cached_nres;
  }
  if (ms) {
    std::memcpy(equv, r->equv, K * sizeof(double));
    *chosen = r->chosen;
  }
  if (!ms || r->chosen >= 0)
    for (size_t i = 0; i < n; ++i)
      for (int k = 0; k < 4; ++k) poses[4 * (size_t)h->cached_order[i] + k] = r->poses()[4 * i + k];
  return OSB_OK;
}

extern "C" osb_status osb_solver_solve(osb_solver* h, int n_nodes, double* poses, const uint8_t* fixed, int n_factors,
                                       const int32_t* type, const int32_t* ia, const int32_t* ib,
                                       const double* payload, const uint8_t* huber, const osb_solve_options* opt,
                                       osb_solve_summary* summary) {
  OSB_REQUIRE(h && poses && fixed && type && ia && ib && payload && huber && summary, "null argument");
  OSB_REQUIRE(n_nodes > 0 && n_nodes <= h->max_nodes && n_factors > 0 && n_factors <= h->max_factors,
              "graph larger than the solver capacity");
  osb_status s = validate_graph(n_nodes, n_factors, type, ia, ib);
  if (s != OSB_OK) return s;
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  OSB_TRY(finish_device_call(h));
  h->g_static_valid = false;              // the device factor arrays now hold this graph, not the resident one
  h->cached_topo = 0;                     // ... and so do the index tables
  return solver_run(h, n_nodes, poses, fixed, n_factors, type, ia, ib, payload, huber, true, 0, opt, nullptr, nullptr,
                    summary);
}

// ---- random-restart initialisation: solve_with_multiple_init (swarm_localization_solver.cpp:781-845) ----------------
// Trials start from the caller's poses with the masked free nodes scattered (multistart_init_kernel), run as one launch
// of n_trials solves of the osb_solver_solve shape, and are ranked on the device (multistart_select_kernel).
extern "C" osb_status osb_solver_solve_multistart(osb_solver* h, int n_nodes, double* poses, const uint8_t* fixed,
                                                  const uint8_t* init_mask, int n_factors, const int32_t* type,
                                                  const int32_t* ia, const int32_t* ib, const double* payload,
                                                  const uint8_t* huber, const osb_solve_options* opt,
                                                  const osb_multistart_options* ms, osb_solve_summary* trial_summaries,
                                                  double* equv_costs, int32_t* chosen) {
  OSB_REQUIRE(h && poses && fixed && init_mask && type && ia && ib && payload && huber && ms && trial_summaries &&
              equv_costs && chosen, "null argument");
  OSB_REQUIRE(ms->n_trials >= 1 && ms->n_trials <= MS_MAX_TRIALS, "n_trials must be 1 ... 256");
  OSB_REQUIRE(!ms->normalise || ms->window_size >= 1, "window_size must be >= 1 when normalise is set");
  OSB_REQUIRE(std::isfinite(ms->rand_xy) && ms->rand_xy >= 0.0 && std::isfinite(ms->rand_z) && ms->rand_z >= 0.0,
              "rand_xy and rand_z must be finite and >= 0");
  OSB_REQUIRE(!std::isnan(ms->acpt_cost), "acpt_cost is NaN");
  OSB_REQUIRE(n_nodes > 0 && n_nodes <= h->max_nodes && n_factors > 0 && n_factors <= h->max_factors,
              "graph larger than the solver capacity");
  osb_status s = validate_graph(n_nodes, n_factors, type, ia, ib);
  if (s != OSB_OK) return s;
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  OSB_TRY(finish_device_call(h));
  h->g_static_valid = false;              // as osb_solver_solve: the device factor arrays and tables now hold this graph
  h->cached_topo = 0;
  return solver_run(h, n_nodes, poses, fixed, n_factors, type, ia, ib, payload, huber, true, 0, opt, ms, init_mask,
                    trial_summaries, equv_costs, chosen);
}

// -------------------------------------------------------------------------------------------------------------
// Resident graph (SURVEY.md section 8f-4).  The reference re-flattens its whole window into a ceres::Problem on every
// solve (setup_problem_with_sferror / _loops_and_detections / _ego_motion, swarm_localization_solver.cpp:1064-1214).
// Here the factor list lives in device memory between solves: add_new_swarm_frame / add_new_loop_connection
// (swarm_localization_solver.hpp:197-214) append what a frame adds, only the new factors cross PCIe, and the poses
// stay where the last solve left them (the reference's est_poses persist the same way).
// -------------------------------------------------------------------------------------------------------------
extern "C" osb_status osb_solver_graph_clear(osb_solver* h) {
  OSB_REQUIRE(h != nullptr, "null handle");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  OSB_TRY(finish_device_call(h));
  h->g_poses.clear(); h->g_payload.clear(); h->g_fixed.clear(); h->g_huber.clear();
  h->g_type.clear(); h->g_ia.clear(); h->g_ib.clear();
  h->g_uploaded = 0; h->g_static_valid = true;
  ++h->g_topo_version;
  h->rposes_current = false; h->dev_pending = false;
  return OSB_OK;
}

extern "C" osb_status osb_solver_graph_add_nodes(osb_solver* h, int n, const double* poses, const uint8_t* fixed,
                                                 int32_t* first_id) {
  OSB_REQUIRE(h != nullptr && n > 0 && poses != nullptr, "bad argument");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  OSB_TRY(finish_device_call(h));
  const size_t have = h->g_fixed.size();
  if (have + (size_t)n > (size_t)h->max_nodes) { set_error("osb_solver_graph_add_nodes", "node capacity exceeded"); return OSB_ERR_CAPACITY; }
  if (first_id) *first_id = (int32_t)have;
  h->g_poses.insert(h->g_poses.end(), poses, poses + 4 * (size_t)n);
  for (int i = 0; i < n; ++i) h->g_fixed.push_back(fixed ? fixed[i] : 0);
  ++h->g_topo_version;
  h->rposes_current = false; h->dev_pending = false;
  return OSB_OK;
}

extern "C" osb_status osb_solver_graph_add_factors(osb_solver* h, int m, const int32_t* type, const int32_t* ia,
                                                   const int32_t* ib, const double* payload, const uint8_t* huber) {
  OSB_REQUIRE(h != nullptr && m > 0 && type && ia && ib && payload && huber, "bad argument");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  OSB_TRY(finish_device_call(h));
  const size_t have = h->g_type.size();
  if (have + (size_t)m > (size_t)h->max_factors) { set_error("osb_solver_graph_add_factors", "factor capacity exceeded"); return OSB_ERR_CAPACITY; }
  osb_status s = validate_graph((int)h->g_fixed.size(), m, type, ia, ib);
  if (s != OSB_OK) return s;
  h->g_type.insert(h->g_type.end(), type, type + m);
  h->g_ia.insert(h->g_ia.end(), ia, ia + m);
  h->g_ib.insert(h->g_ib.end(), ib, ib + m);
  h->g_huber.insert(h->g_huber.end(), huber, huber + m);
  h->g_payload.insert(h->g_payload.end(), payload, payload + (size_t)m * OSB_PAYLOAD_LEN);
  ++h->g_topo_version;
  return OSB_OK;
}

extern "C" osb_status osb_solver_graph_set_fixed(osb_solver* h, int node, int fixed) {
  OSB_REQUIRE(h != nullptr, "null handle");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  OSB_TRY(finish_device_call(h));
  OSB_REQUIRE(node >= 0 && (size_t)node < h->g_fixed.size(), "node out of range");
  h->g_fixed[node] = fixed ? 1 : 0;
  ++h->g_topo_version;
  return OSB_OK;
}

extern "C" osb_status osb_solver_graph_set_poses(osb_solver* h, int first, int n, const double* poses) {
  OSB_REQUIRE(h != nullptr && poses != nullptr, "bad argument");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  OSB_TRY(finish_device_call(h));
  OSB_REQUIRE(first >= 0 && n >= 0 && (size_t)(first + n) <= h->g_fixed.size(), "node range out of bounds");
  std::copy(poses, poses + 4 * (size_t)n, h->g_poses.begin() + 4 * (size_t)first);
  h->rposes_current = false; h->dev_pending = false;
  return OSB_OK;
}

extern "C" osb_status osb_solver_graph_get_poses(osb_solver* h, int first, int n, double* poses) {
  OSB_REQUIRE(h != nullptr && poses != nullptr, "bad argument");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  OSB_TRY(finish_device_call(h));          // a device call's poses reach g_poses first
  OSB_REQUIRE(first >= 0 && n >= 0 && (size_t)(first + n) <= h->g_fixed.size(), "node range out of bounds");
  std::copy(h->g_poses.begin() + 4 * (size_t)first, h->g_poses.begin() + 4 * (size_t)(first + n), poses);
  return OSB_OK;
}

extern "C" osb_status osb_solver_graph_size(osb_solver* h, int32_t* n_nodes, int32_t* n_factors) {
  OSB_REQUIRE(h != nullptr, "null handle");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  OSB_TRY(finish_device_call(h));
  if (n_nodes) *n_nodes = (int32_t)h->g_fixed.size();
  if (n_factors) *n_factors = (int32_t)h->g_type.size();
  return OSB_OK;
}

// sliding window (solver.cpp:186-202 trims old keyframes): drop the first `n_nodes` nodes and every factor touching them;
// the remaining nodes are renumbered (id - n_nodes).  A rare operation: the device factor arrays are rebuilt.
extern "C" osb_status osb_solver_graph_drop_oldest(osb_solver* h, int n_nodes) {
  OSB_REQUIRE(h != nullptr && n_nodes >= 0, "bad argument");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  OSB_TRY(finish_device_call(h));
  OSB_REQUIRE((size_t)n_nodes <= h->g_fixed.size(), "cannot drop more nodes than the graph holds");
  if (n_nodes == 0) return OSB_OK;
  h->g_poses.erase(h->g_poses.begin(), h->g_poses.begin() + 4 * (size_t)n_nodes);
  h->g_fixed.erase(h->g_fixed.begin(), h->g_fixed.begin() + n_nodes);
  size_t w = 0;
  for (size_t f = 0; f < h->g_type.size(); ++f) {
    if (h->g_ia[f] < n_nodes || h->g_ib[f] < n_nodes) continue;
    h->g_type[w] = h->g_type[f]; h->g_ia[w] = h->g_ia[f] - n_nodes; h->g_ib[w] = h->g_ib[f] - n_nodes;
    h->g_huber[w] = h->g_huber[f];
    if (w != f) std::copy(h->g_payload.begin() + f * OSB_PAYLOAD_LEN, h->g_payload.begin() + (f + 1) * OSB_PAYLOAD_LEN,
                          h->g_payload.begin() + w * OSB_PAYLOAD_LEN);
    ++w;
  }
  h->g_type.resize(w); h->g_ia.resize(w); h->g_ib.resize(w); h->g_huber.resize(w); h->g_payload.resize(w * OSB_PAYLOAD_LEN);
  h->g_uploaded = 0;                       // factor positions moved: re-send on the next solve
  ++h->g_topo_version;
  h->rposes_current = false; h->dev_pending = false;
  return OSB_OK;
}

static osb_status flush_resident_factors(osb_solver* h);

extern "C" osb_status osb_solver_solve_resident(osb_solver* h, const osb_solve_options* opt, osb_solve_summary* summary) {
  OSB_REQUIRE(h != nullptr && summary != nullptr, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  OSB_TRY(finish_device_call(h));
  const size_t n = h->g_fixed.size(), m = h->g_type.size();
  OSB_REQUIRE(n > 0 && m > 0, "the resident graph is empty");
  OSB_TRY(flush_resident_factors(h));
  h->rposes_current = false;               // this solve writes g_poses
  h->dev_pending = false;
  return solver_run(h, (int)n, h->g_poses.data(), h->g_fixed.data(), (int)m, h->g_type.data(), h->g_ia.data(),
                    h->g_ib.data(), h->g_payload.data(), h->g_huber.data(), false, h->g_topo_version, opt, nullptr,
                    nullptr, summary);
}

// ---- device tail (osb_solver_solve_resident_dev) -----------------------------------------------------------------
// Carve the device-tail buffers from `base` (nullptr: size only) for a handle of n nodes and m factors.
static size_t tail_layout(TailDev& D, char* base, size_t n, size_t m) {
  const size_t chunks = std::max<size_t>(1, (m + TL_ROWS - 1) / TL_ROWS);
  size_t at = 0;
  auto take = [&](auto*& p, size_t count) {
    using Q = std::remove_const_t<std::remove_pointer_t<std::remove_reference_t<decltype(p)>>>;
    p = reinterpret_cast<Q*>(reinterpret_cast<uintptr_t>(base) + at);
    at += (count * sizeof(Q) + 255) & ~(size_t)255;
  };
  take(D.inv, n); take(D.order, n); take(D.b_ia, m); take(D.b_ib, m); take(D.b_ptr, n + 1); take(D.b_slot_a, m);
  take(D.b_slot_b, m); take(D.b_es_ptr, n + 1); take(D.b_es_slot, m); take(D.b_fixed, n); take(D.b_link, n);
  take(D.key_s, 2 * m); take(D.rank_s, 2 * m); take(D.key_e, m); take(D.rank_e, m);
  take(D.hist_s, chunks * n); take(D.hist_e, chunks * n); take(D.cnt_s, n); take(D.cnt_e, n);
  take(D.flag, 2 * chunks); take(D.word, 4);
  return at;
}

// The first host-side call after a device call waits for it and refreshes the host mirror of the poses, the call's status
// and its summary.  A captured call stays pending: every host-side call re-reads what the last replay left (the caller
// has synchronised it), until a host-side change of the poses or the graph takes over.  The caller holds h->mu.
static osb_status finish_device_call(osb_solver* h) {
  if (!h->dev_pending) return OSB_OK;
  if (!h->dev_captured) h->dev_pending = false;
  if (!h->dev_captured) OSB_CUDA(cudaEventSynchronize(h->ev_done));
  int32_t word[4];
  osb_solve_summary sm;
  cudaStream_t st = h->stream;
  OSB_CUDA(cudaMemcpyAsync(word, h->tail.word, sizeof(word), cudaMemcpyDeviceToHost, st));
  OSB_CUDA(cudaMemcpyAsync(&sm, h->d_tsummary, sizeof(sm), cudaMemcpyDeviceToHost, st));
  OSB_CUDA(cudaMemcpyAsync(h->g_poses.data(), h->d_rposes, h->g_poses.size() * sizeof(double), cudaMemcpyDeviceToHost, st));
  OSB_CUDA(cudaStreamSynchronize(st));
  h->dev_status = (osb_status)word[0];
  if (h->dev_status == OSB_OK) {
    float msec = 0.f;
    if (!h->dev_captured) OSB_CUDA(cudaEventElapsedTime(&msec, h->ev0, h->ev1));
    sm.solve_ms = msec;
    sm.n_residuals = h->tail_nres + word[3];
    h->dev_summary = sm;
  }
  return OSB_OK;
}

// the resident factors added since the last solve -> device (all of them after a one-shot call overwrote the arrays)
static osb_status flush_resident_factors(osb_solver* h) {
  const size_t m = h->g_type.size();
  if (!h->g_static_valid) { h->g_uploaded = 0; h->g_static_valid = true; h->cached_topo = 0; }
  if (h->g_uploaded < m) {                 // only the factors added since the last solve cross PCIe
    const size_t f0 = h->g_uploaded, k = m - f0;
    cudaStream_t st = h->stream;
    OSB_CUDA(cudaMemcpyAsync(h->d_huber + f0, h->g_huber.data() + f0, k, cudaMemcpyHostToDevice, st));
    OSB_CUDA(cudaMemcpyAsync(h->d_type + f0, h->g_type.data() + f0, k * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    OSB_CUDA(cudaMemcpyAsync(h->d_payload + f0 * OSB_PAYLOAD_LEN, h->g_payload.data() + f0 * OSB_PAYLOAD_LEN,
                             k * OSB_PAYLOAD_LEN * sizeof(double), cudaMemcpyHostToDevice, st));
    h->g_uploaded = m;
  }
  return OSB_OK;
}

extern "C" osb_status osb_solver_solve_resident_dev(osb_solver* h, int max_tail, const int32_t* type_dev,
                                                    const int32_t* ia_dev, const int32_t* ib_dev, const double* payload_dev,
                                                    const uint8_t* huber_dev, const int32_t* count_dev,
                                                    const osb_solve_options* opt, void* stream) {
  OSB_REQUIRE(h && type_dev && ia_dev && ib_dev && payload_dev && huber_dev && count_dev, "null argument");
  OSB_REQUIRE(max_tail >= 0, "max_tail must be >= 0");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  cudaStream_t st = (cudaStream_t)stream;
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  OSB_CUDA(cudaStreamIsCapturing(st, &cap));
  const bool capturing = cap != cudaStreamCaptureStatusNone;
  const size_t n = h->g_fixed.size(), m_base = h->g_type.size();
  OSB_REQUIRE(n > 0 && m_base > 0, "the resident graph is empty");
  if (m_base + (size_t)max_tail > (size_t)h->max_factors) {
    set_error("osb_solver_solve_resident_dev", "resident factors + max_tail exceed the solver capacity");
    return OSB_ERR_CAPACITY;
  }
  osb_solve_options o;
  if (opt) o = *opt; else osb_solve_default_options(&o);
  const int m_bound = (int)m_base + max_tail;
  // the launch shape is solve_shape's for (n, m + max_tail); cached so that a captured call makes no occupancy query
  const bool f32 = o.inner_precision == OSB_INNER_FP32 || (o.inner_precision == OSB_INNER_AUTO && o.pcg_tolerance >= 1e-4);
  const long long shape_key = (((long long)n * (h->max_factors + 1LL) + m_bound) * 2 + (f32 ? 1 : 0)) * 2 +
                              (o.preconditioner == OSB_PRECOND_BLOCK_JACOBI ? 1 : 0);
  const bool host_work = h->d_tail == nullptr || h->tail_topo != h->g_topo_version || !h->g_static_valid ||
                         h->g_uploaded < m_base || !h->rposes_current || shape_key != h->tail_shape_key;
  if (capturing && (host_work || !h->tail_shape.cluster)) {
    set_error("osb_solver_solve_resident_dev", capturing && !host_work
              ? "the cooperative path cannot be captured"
              : "a captured call cannot do host work: run the call once outside the capture after the graph changed");
    return OSB_ERR_INVALID;
  }
  if (host_work) {
    if (h->d_tail == nullptr) {                // everything a device call needs, once per handle
      TailDev D = {};
      OSB_TRY(h->res.alloc(&h->d_tail, tail_layout(D, nullptr, h->max_nodes, h->max_factors)));
      OSB_TRY(h->res.alloc(&h->d_rposes, 4 * (size_t)h->max_nodes));
      OSB_TRY(h->res.alloc(&h->d_tsummary, 1));
      OSB_TRY(h->res.event(&h->ev_done));
      tail_layout(h->tail, h->d_tail, h->max_nodes, h->max_factors);
    }
    OSB_TRY(flush_resident_factors(h));
    cudaStream_t hs = h->stream;
    GraphTables t;
    ChainPlan plan;
    if (h->tail_topo != h->g_topo_version) {   // the resident plan and its base-only tables
      build_chain_plan((int)n, h->g_fixed.data(), (int)m_base, h->g_type.data(), h->g_ia.data(), h->g_ib.data(),
                       h->g_payload.data(), plan);
      build_tables((int)n, h->g_fixed.data(), (int)m_base, h->g_type.data(), h->g_ia.data(), h->g_ib.data(),
                   h->g_payload.data(), plan, t);
      const TailDev& D = h->tail;
      const size_t i4 = sizeof(int32_t);
      OSB_CUDA(cudaMemcpyAsync((void*)D.inv, plan.inv.data(), n * i4, cudaMemcpyHostToDevice, hs));
      OSB_CUDA(cudaMemcpyAsync((void*)D.order, plan.order.data(), n * i4, cudaMemcpyHostToDevice, hs));
      OSB_CUDA(cudaMemcpyAsync((void*)D.b_ia, t.ia.data(), m_base * i4, cudaMemcpyHostToDevice, hs));
      OSB_CUDA(cudaMemcpyAsync((void*)D.b_ib, t.ib.data(), m_base * i4, cudaMemcpyHostToDevice, hs));
      OSB_CUDA(cudaMemcpyAsync((void*)D.b_ptr, t.ptr.data(), (n + 1) * i4, cudaMemcpyHostToDevice, hs));
      OSB_CUDA(cudaMemcpyAsync((void*)D.b_slot_a, t.slot_a.data(), m_base * i4, cudaMemcpyHostToDevice, hs));
      OSB_CUDA(cudaMemcpyAsync((void*)D.b_slot_b, t.slot_b.data(), m_base * i4, cudaMemcpyHostToDevice, hs));
      OSB_CUDA(cudaMemcpyAsync((void*)D.b_es_ptr, t.es_ptr.data(), (n + 1) * i4, cudaMemcpyHostToDevice, hs));
      OSB_CUDA(cudaMemcpyAsync((void*)D.b_es_slot, t.es_slot.data(), m_base * i4, cudaMemcpyHostToDevice, hs));
      OSB_CUDA(cudaMemcpyAsync((void*)D.b_fixed, t.fixed.data(), n, cudaMemcpyHostToDevice, hs));
      OSB_CUDA(cudaMemcpyAsync((void*)D.b_link, plan.link.data(), n, cudaMemcpyHostToDevice, hs));
      h->tail_order = plan.order;
      h->tail_nres = t.n_res;
      h->tail_topo = h->g_topo_version;
    }
    if (!h->rposes_current) {
      OSB_CUDA(cudaMemcpyAsync(h->d_rposes, h->g_poses.data(), 4 * n * sizeof(double), cudaMemcpyHostToDevice, hs));
      h->rposes_current = true;
    }
    if (shape_key != h->tail_shape_key) {
      OSB_TRY(solve_shape(h, (int)n, m_bound, o, h->tail_shape));
      h->tail_shape_key = shape_key;
    }
    OSB_CUDA(cudaStreamSynchronize(hs));       // the staging vectors above die here; the caller's stream comes after
  }
  const SolveShape& shape = h->tail_shape;
  SolverDev P = graph_dev(h, (int)n, m_bound, o);
  trial_layout(P, h->d_arena, n, m_bound, shape);
  P.summary = h->d_tsummary;
  P.dev_word = h->tail.word;
  TailDev D = h->tail;
  D.n = (int)n; D.m_base = (int)m_base; D.max_tail = max_tail; D.ctas = shape.ctas;
  D.chunks = std::max(1, cdiv(max_tail, TL_ROWS));
  D.count = count_dev; D.type = type_dev; D.ia = ia_dev; D.ib = ib_dev; D.payload = payload_dev; D.huber = huber_dev;
  D.ia_o = h->d_ia; D.ib_o = h->d_ib; D.ptr_o = h->d_ptr; D.slot_a_o = h->d_slot_a; D.slot_b_o = h->d_slot_b;
  D.es_ptr_o = h->d_es_ptr; D.es_slot_o = h->d_es_slot; D.type_o = h->d_type; D.payload_o = h->d_payload;
  D.huber_o = h->d_huber; D.fixed_o = h->d_fixed; D.link_o = h->d_link;
  D.poses = h->d_rposes; D.x0 = P.x[0]; D.x_out = P.poses_out;
  h->cached_topo = 0;                          // the one-shot index tables now hold this call's list
  OSB_LAUNCH(tail_rank_kernel, D.chunks, 2 * TL_ROWS, 0, st, D);
  OSB_CHECK_LAUNCH();
  OSB_LAUNCH(tail_scan_kernel, cdiv((int)n, 256), 256, 0, st, D);
  OSB_CHECK_LAUNCH();
  OSB_LAUNCH(tail_ptr_kernel, 1, 1024, 0, st, D);
  OSB_CHECK_LAUNCH();
  OSB_LAUNCH(tail_tables_kernel, cdiv(std::max(m_bound, (int)n), 256), 256, 0, st, D);
  OSB_CHECK_LAUNCH();
  if (!capturing) OSB_CUDA(cudaEventRecord(h->ev0, st));
  OSB_TRY(launch_solves(h, P, shape, 1, 0, st, true));
  if (!capturing) OSB_CUDA(cudaEventRecord(h->ev1, st));
  OSB_LAUNCH(tail_poses_out_kernel, cdiv((int)n, 256), 256, 0, st, D);
  OSB_CHECK_LAUNCH();
  if (!capturing) OSB_CUDA(cudaEventRecord(h->ev_done, st));
  h->dev_pending = true; h->dev_captured = capturing; h->dev_called = true;
  return OSB_OK;
}

extern "C" osb_status osb_solver_last_summary(osb_solver* h, osb_solve_summary* summary) {
  OSB_REQUIRE(h != nullptr && summary != nullptr, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  OSB_TRY(finish_device_call(h));
  OSB_REQUIRE(h->dev_called, "no osb_solver_solve_resident_dev call on this handle");
  if (h->dev_status != OSB_OK) {
    set_error("osb_solver_last_summary", h->dev_status == OSB_ERR_CAPACITY
              ? "the device call was refused: *count_dev > max_tail"
              : "the device call was refused: a tail row has an unknown type or a bad node id, or *count_dev < 0");
    return h->dev_status;
  }
  *summary = h->dev_summary;
  return OSB_OK;
}

extern "C" osb_status osb_solver_phase_cycles(osb_solver* h, double* out12) {
  OSB_REQUIRE(h != nullptr && out12 != nullptr, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  OSB_TRY(finish_device_call(h));
  long long c[8];
  OSB_CUDA(cudaMemcpy(c, h->d_dbg, sizeof(c), cudaMemcpyDeviceToHost));
  for (int i = 0; i < 8; ++i) out12[i] = (double)c[i];
  const SolveShape& s = h->last_shape;
  out12[8] = s.ctas; out12[9] = s.cluster; out12[10] = s.jsmem + 2 * s.chain + 4 * (s.f32 ? 1 : 0); out12[11] = GS_THREADS;
  return OSB_OK;
}

// profiling aid: per-warp cycles spent in the chain preconditioner sweeps of the last solve, [16 CTAs][8 warps]
extern "C" osb_status osb_solver_chain_cycles(osb_solver* h, double* out128) {
  OSB_REQUIRE(h != nullptr && out128 != nullptr, "null argument");
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  OSB_TRY(finish_device_call(h));
  long long c[128];
  OSB_CUDA(cudaMemcpy(c, h->d_dbg + 8, sizeof(c), cudaMemcpyDeviceToHost));
  for (int i = 0; i < 128; ++i) out128[i] = (double)c[i];
  return OSB_OK;
}

extern "C" osb_status osb_solver_linearize(osb_solver* h, int n_nodes, const double* poses, int n_factors,
                                           const int32_t* type, const int32_t* ia, const int32_t* ib,
                                           const double* payload, double* r, double* Ja, double* Jb) {
  OSB_REQUIRE(h && poses && type && ia && ib && payload && r && Ja && Jb, "null argument");
  OSB_REQUIRE(n_nodes > 0 && n_nodes <= h->max_nodes && n_factors > 0 && n_factors <= h->max_factors,
              "graph larger than the solver capacity");
  osb_status s = validate_graph(n_nodes, n_factors, type, ia, ib);
  if (s != OSB_OK) return s;
  std::lock_guard<std::mutex> lk(h->mu);
  DeviceGuard dg(h->device);
  OSB_TRY(finish_device_call(h));
  h->g_static_valid = false;              // as osb_solver_solve: the device factor arrays and tables now hold this graph
  h->cached_topo = 0;
  const size_t n = n_nodes, m = n_factors;
  cudaStream_t st = h->stream;
  double* d_x = h->d_lin;             // [n][4]
  double* d_r = d_x + 4 * n;          // [m][4]
  double* d_ja = d_r + 4 * m;         // [m][16]
  double* d_jb = d_ja + 16 * m;       // [m][16]
  OSB_CUDA(cudaMemcpyAsync(h->d_type, type, m * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  OSB_CUDA(cudaMemcpyAsync(h->d_ia, ia, m * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  OSB_CUDA(cudaMemcpyAsync(h->d_ib, ib, m * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  OSB_CUDA(cudaMemcpyAsync(h->d_payload, payload, m * OSB_PAYLOAD_LEN * sizeof(double), cudaMemcpyHostToDevice, st));
  OSB_CUDA(cudaMemcpyAsync(d_x, poses, 4 * n * sizeof(double), cudaMemcpyHostToDevice, st));
  OSB_LAUNCH(graph_linearize_kernel, cdiv(n_factors, 128), 128, 0, st, n_factors, d_x, h->d_type, h->d_ia, h->d_ib,
             h->d_payload, d_r, d_ja, d_jb);
  OSB_CHECK_LAUNCH();
  OSB_CUDA(cudaMemcpyAsync(r, d_r, 4 * m * sizeof(double), cudaMemcpyDeviceToHost, st));
  OSB_CUDA(cudaMemcpyAsync(Ja, d_ja, 16 * m * sizeof(double), cudaMemcpyDeviceToHost, st));
  OSB_CUDA(cudaMemcpyAsync(Jb, d_jb, 16 * m * sizeof(double), cudaMemcpyDeviceToHost, st));
  OSB_CUDA(cudaStreamSynchronize(st));
  return OSB_OK;
}
