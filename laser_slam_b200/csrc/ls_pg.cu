// Pose-graph solve on the device (K5 linearise, K6 Gauss-Newton update), C ABI ls_pg_* of include/ls_b200.h.
//
// Replaces what IncrementalEstimator asks of gtsam::ISAM2 (reference laser_slam/src/incremental_estimator.cpp:
// 151-163 estimate, 165-266 estimateAndRemove, 268-291 registerPrior): factors are the ExpressionFactor<SE3>s built
// by LaserTrack::makeMeasurementFactor / makeRelativeMeasurementFactor (reference laser_slam/src/laser_track.cpp:
// 431-458) with Diagonal or Robust(Cauchy(1)) noise (laser_track.cpp:37-64).  Conventions are those of
// oracle/posegraph_oracle.py ([translation; rotation-vector] tangent, decoupled Local, t += dt, R <- R Exp(dr)).
//
// Structure exploited: a laser_slam graph is, per track, a CHAIN (prior on the first pose, odometry + ICP factors
// between consecutive poses) plus a few loop closures.  Poses are ordered track by track, so
//   H = H_c + U^T U,   H_c block-tridiagonal (chain + priors),   U = whitened Jacobians of the "extra" factors
// and the update solves H d = -g exactly through the Woodbury identity:
//   y = H_c^-1 (-g),  Z = H_c^-1 U^T,  (I + U Z) w = U y,  d = y - Z w,
// with H_c^-1 applied to all 6 #LC + 1 right-hand sides at once by block cyclic reduction (log2 P parallel levels).
// All arithmetic is float64; every sum that enters the solve has a fixed order (deterministic); only the reported cost
// statistic is an atomic sum.  Not HBM-bound (a few MB per iteration,
// SURVEY.md §8d): the cost is latency -- kernel launches and dependent levels -- not bandwidth.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <map>
#include <string>
#include <unordered_map>
#include <vector>

#include <cuda_runtime.h>

#include "../../include/ls_b200.h"
#include "ls_buffer.cuh"

using ls::Buffer;

namespace {

struct FactorDev {
  int type, robust, fix_a, extra;  // extra: index among border factors or -1
  int ia, ib;                      // pose indices (ia = -1: factor does not depend on node a)
  int chain;                       // 1: couples consecutive poses ia+1 == ib of one track
  int pad;
  double meas[7], sigma[6], fixed_a[7];
};

// ---------------------------------------------------------------- small dense helpers (row-major 3x3 / 6x6)
__device__ __forceinline__ void quat_to_R(const double* q, double* R) {
  const double n = 1.0 / sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  const double w = q[0] * n, x = q[1] * n, y = q[2] * n, z = q[3] * n;
  R[0] = 1 - 2 * (y * y + z * z); R[1] = 2 * (x * y - w * z); R[2] = 2 * (x * z + w * y);
  R[3] = 2 * (x * y + w * z); R[4] = 1 - 2 * (x * x + z * z); R[5] = 2 * (y * z - w * x);
  R[6] = 2 * (x * z - w * y); R[7] = 2 * (y * z + w * x); R[8] = 1 - 2 * (x * x + y * y);
}
__device__ __forceinline__ void mat3_mul(const double* A, const double* B, double* C) {
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) C[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
}
__device__ __forceinline__ void mat3_tmul(const double* A, const double* B, double* C) {  // A^T B
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) C[3 * i + j] = A[i] * B[j] + A[3 + i] * B[3 + j] + A[6 + i] * B[6 + j];
}
__device__ __forceinline__ void so3_log(const double* R, double* w) {
  const double vx = 0.5 * (R[7] - R[5]), vy = 0.5 * (R[2] - R[6]), vz = 0.5 * (R[3] - R[1]);
  const double s = sqrt(vx * vx + vy * vy + vz * vz);
  const double c = 0.5 * (R[0] + R[4] + R[8] - 1.0);
  const double th = atan2(s, c);
  const double scale = s < 1e-8 ? 1.0 + th * th / 6.0 : th / s;
  w[0] = vx * scale; w[1] = vy * scale; w[2] = vz * scale;
}
__device__ __forceinline__ void jr_inv(const double* p, double* J) {
  const double th2 = p[0] * p[0] + p[1] * p[1] + p[2] * p[2];
  const double th = sqrt(th2);
  const double c = th < 1e-6 ? 1.0 / 12.0 : 1.0 / th2 - (1.0 + cos(th)) / (2.0 * th * sin(th));
  const double K[9] = {0, -p[2], p[1], p[2], 0, -p[0], -p[1], p[0], 0};
  double K2[9];
  mat3_mul(K, K, K2);
  for (int i = 0; i < 9; ++i) J[i] = 0.5 * K[i] + c * K2[i];
  J[0] += 1.0; J[4] += 1.0; J[8] += 1.0;
}

// ---------------------------------------------------------------- K5: linearise every factor
__global__ void pg_linearize_kernel(int F, const FactorDev* __restrict__ fac, const double* __restrict__ poses,
                                    double* __restrict__ Ja, double* __restrict__ Jb, double* __restrict__ r,
                                    double* cost) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  const FactorDev& fc = fac[f];
  double ja[36], jb[36], res[6];
  for (int i = 0; i < 36; ++i) { ja[i] = 0.0; jb[i] = 0.0; }
  double Rm[9];
  quat_to_R(fc.meas, Rm);
  const double* tm = fc.meas + 4;
  if (fc.type == 0) {  // prior on node b
    const double* X = poses + 7 * (size_t)fc.ib;
    double R[9], RE[9], w[3], Ji[9];
    quat_to_R(X, R);
    const double d[3] = {X[4] - tm[0], X[5] - tm[1], X[6] - tm[2]};
    for (int i = 0; i < 3; ++i) res[i] = Rm[i] * d[0] + Rm[3 + i] * d[1] + Rm[6 + i] * d[2];
    mat3_tmul(Rm, R, RE);
    so3_log(RE, w);
    jr_inv(w, Ji);
    for (int i = 0; i < 3; ++i) {
      res[3 + i] = w[i];
      for (int j = 0; j < 3; ++j) {
        jb[6 * i + j] = Rm[3 * j + i];
        jb[6 * (3 + i) + 3 + j] = Ji[3 * i + j];
      }
    }
  } else {
    const double* A = fc.fix_a ? fc.fixed_a : poses + 7 * (size_t)fc.ia;
    const double* B = poses + 7 * (size_t)fc.ib;
    double Ra[9], Rb[9], RmtRat[9], RE[9], w[3], Ji[9], tmp[9];
    quat_to_R(A, Ra);
    quat_to_R(B, Rb);
    const double d[3] = {B[4] - A[4], B[5] - A[5], B[6] - A[6]};
    double v[3];
    for (int i = 0; i < 3; ++i) v[i] = Ra[i] * d[0] + Ra[3 + i] * d[1] + Ra[6 + i] * d[2];
    const double u[3] = {v[0] - tm[0], v[1] - tm[1], v[2] - tm[2]};
    for (int i = 0; i < 3; ++i) res[i] = Rm[i] * u[0] + Rm[3 + i] * u[1] + Rm[6 + i] * u[2];
    // RmtRat = Rm^T Ra^T
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) RmtRat[3 * i + j] = Rm[i] * Ra[3 * j] + Rm[3 + i] * Ra[3 * j + 1] + Rm[6 + i] * Ra[3 * j + 2];
    mat3_mul(RmtRat, Rb, RE);
    so3_log(RE, w);
    jr_inv(w, Ji);
    const double Kv[9] = {0, -v[2], v[1], v[2], 0, -v[0], -v[1], v[0], 0};
    double RmtKv[9], RbtRa[9], JiRbtRa[9];
    mat3_tmul(Rm, Kv, RmtKv);
    mat3_tmul(Rb, Ra, RbtRa);
    mat3_mul(Ji, RbtRa, JiRbtRa);
    (void)tmp;
    for (int i = 0; i < 3; ++i) {
      res[3 + i] = w[i];
      for (int j = 0; j < 3; ++j) {
        jb[6 * i + j] = RmtRat[3 * i + j];
        jb[6 * (3 + i) + 3 + j] = Ji[3 * i + j];
        if (!fc.fix_a) {
          ja[6 * i + j] = -RmtRat[3 * i + j];
          ja[6 * i + 3 + j] = RmtKv[3 * i + j];
          ja[6 * (3 + i) + 3 + j] = -JiRbtRa[3 * i + j];
        }
      }
    }
  }
  double e2 = 0.0;
  for (int i = 0; i < 6; ++i) {
    const double inv = 1.0 / fc.sigma[i];
    res[i] *= inv;
    e2 += res[i] * res[i];
    for (int j = 0; j < 6; ++j) { ja[6 * i + j] *= inv; jb[6 * i + j] *= inv; }
  }
  double c = 0.5 * e2;
  if (fc.robust) {
    const double sw = sqrt(1.0 / (1.0 + e2));
    c = 0.5 * log1p(e2);
    for (int i = 0; i < 6; ++i) res[i] *= sw;
    for (int i = 0; i < 36; ++i) { ja[i] *= sw; jb[i] *= sw; }
  }
  for (int i = 0; i < 36; ++i) { Ja[36 * (size_t)f + i] = ja[i]; Jb[36 * (size_t)f + i] = jb[i]; }
  for (int i = 0; i < 6; ++i) r[6 * (size_t)f + i] = res[i];
  atomicAdd(cost, c);
}

// ---------------------------------------------------------------- K5b: block-tridiagonal H_c and gradient
// thread per pose; incident factors through a CSR list (fixed order => deterministic sums)
__global__ void pg_assemble_kernel(int P, const int* __restrict__ inc_ptr, const int* __restrict__ inc_fac,
                                   const FactorDev* __restrict__ fac, const double* __restrict__ Ja,
                                   const double* __restrict__ Jb, const double* __restrict__ r,
                                   const int* __restrict__ damp, double* __restrict__ D, double* __restrict__ Bsub,
                                   double* __restrict__ g) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= P) return;
  double d[36], b[36], gg[6];
  for (int i = 0; i < 36; ++i) { d[i] = 0.0; b[i] = 0.0; }
  for (int i = 0; i < 6; ++i) gg[i] = 0.0;
  for (int e = inc_ptr[k]; e < inc_ptr[k + 1]; ++e) {
    const int f = inc_fac[e];
    const FactorDev& fc = fac[f];
    const bool self_is_b = (fc.ib == k);
    const double* Js = (self_is_b ? Jb : Ja) + 36 * (size_t)f;
    const double* Jo = (self_is_b ? Ja : Jb) + 36 * (size_t)f;
    const double* rf = r + 6 * (size_t)f;
    for (int i = 0; i < 6; ++i) {
      double s = 0.0;
      for (int m = 0; m < 6; ++m) s += Js[6 * m + i] * rf[m];
      gg[i] += s;
    }
    if (fc.extra >= 0) continue;  // border factors live in U, not in H_c
    for (int i = 0; i < 6; ++i)
      for (int j = 0; j < 6; ++j) {
        double s = 0.0;
        for (int m = 0; m < 6; ++m) s += Js[6 * m + i] * Js[6 * m + j];
        d[6 * i + j] += s;
      }
    if (fc.chain && self_is_b) {  // H[k][k-1] = Jb^T Ja
      for (int i = 0; i < 6; ++i)
        for (int j = 0; j < 6; ++j) {
          double s = 0.0;
          for (int m = 0; m < 6; ++m) s += Js[6 * m + i] * Jo[6 * m + j];
          b[6 * i + j] += s;
        }
    }
  }
  if (damp[k]) {
    // Gauge damping on the first pose of a chain segment that has no prior / fixed-node factor of its own (a track
    // whose prior was removed when it got linked, incremental_estimator.cpp:212-237): added to H only, never to g,
    // so the Gauss-Newton fixed point is unchanged while the chain block becomes positive definite.
    for (int i = 0; i < 3; ++i) { d[7 * i] += 1.0; d[7 * (3 + i)] += 4.0; }  // sigma 1 m / 0.5 rad: << any real factor
  }
  for (int i = 0; i < 36; ++i) { D[36 * (size_t)k + i] = d[i]; Bsub[36 * (size_t)k + i] = b[i]; }
  for (int i = 0; i < 6; ++i) g[6 * (size_t)k + i] = gg[i];
}

// ---------------------------------------------------------------- K6a': block cyclic reduction of H_c
// The sequential block sweeps above cost 2 x P dependent steps per right-hand side (a serial chain of 10000 steps per
// Gauss-Newton iteration at 5000 poses).  Odd-even (cyclic) reduction solves the same block-tridiagonal SPD system in
// log2(P) levels, every level fully parallel over nodes and right-hand sides: level l (stride s = 2^l, nodes numbered
// m = 1..P) eliminates the nodes m = s (mod 2s) into their neighbours m +- s, which keep a Schur complement and a coupling
// of stride 2s; the back-substitution walks the levels down again.  Tracks are just zero couplings.
//   Dc[m]      current diagonal block of node m (final once the node is eliminated)
//   Di[m]      its inverse, formed at the node's elimination level
//   Ll[l][j]   coupling H^(l)[m][m - s] of node m = j << l at level l  (the right coupling is the transpose of the right
//              neighbour's left one: the matrix stays symmetric)
__device__ __forceinline__ bool inv6_spd(const double* A, double* X) {  // X = A^-1 through Cholesky; false: not positive definite
  double L[36];
  for (int i = 0; i < 36; ++i) L[i] = 0.0;
  for (int j = 0; j < 6; ++j) {
    double s = A[6 * j + j];
    for (int m = 0; m < j; ++m) s -= L[6 * j + m] * L[6 * j + m];
    if (!(s > 0.0)) return false;
    const double d = sqrt(s), id = 1.0 / d;
    L[6 * j + j] = d;
    for (int i = j + 1; i < 6; ++i) {
      double v = A[6 * i + j];
      for (int m = 0; m < j; ++m) v -= L[6 * i + m] * L[6 * j + m];
      L[6 * i + j] = v * id;
    }
  }
  for (int c = 0; c < 6; ++c) {  // solve L L^T x = e_c
    double y[6];
    for (int i = 0; i < 6; ++i) {
      double v = (i == c) ? 1.0 : 0.0;
      for (int m = 0; m < i; ++m) v -= L[6 * i + m] * y[m];
      y[i] = v / L[6 * i + i];
    }
    for (int i = 5; i >= 0; --i) {
      double v = y[i];
      for (int m = i + 1; m < 6; ++m) v -= L[6 * m + i] * X[6 * m + c];
      X[6 * i + c] = v / L[6 * i + i];
    }
  }
  return true;
}
__device__ __forceinline__ void mm6(const double* A, const double* B, double* C) {  // C = A B
  for (int i = 0; i < 6; ++i)
    for (int j = 0; j < 6; ++j) {
      double s = 0.0;
      for (int m = 0; m < 6; ++m) s += A[6 * i + m] * B[6 * m + j];
      C[6 * i + j] = s;
    }
}
__device__ __forceinline__ void mmt6(const double* A, const double* B, double* C) {  // C = A B^T
  for (int i = 0; i < 6; ++i)
    for (int j = 0; j < 6; ++j) {
      double s = 0.0;
      for (int m = 0; m < 6; ++m) s += A[6 * i + m] * B[6 * j + m];
      C[6 * i + j] = s;
    }
}
__device__ __forceinline__ void mtm6(const double* A, const double* B, double* C) {  // C = A^T B
  for (int i = 0; i < 6; ++i)
    for (int j = 0; j < 6; ++j) {
      double s = 0.0;
      for (int m = 0; m < 6; ++m) s += A[6 * m + i] * B[6 * m + j];
      C[6 * i + j] = s;
    }
}

__global__ void cr_init_kernel(int P, const double* __restrict__ D, const double* __restrict__ Bsub, double* __restrict__ Dc,
                               double* __restrict__ L0) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= P) return;
  for (int i = 0; i < 36; ++i) { Dc[36 * (size_t)k + i] = D[36 * (size_t)k + i]; L0[36 * (size_t)(k + 1) + i] = Bsub[36 * (size_t)k + i]; }
}
// nodes eliminated at this level: invert their (final) diagonal
__global__ void cr_invert_kernel(int P, int s, const double* __restrict__ Dc, double* __restrict__ Di, int* fail) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  const long long m = (long long)s + (long long)t * 2 * s;  // m = s (mod 2s)
  if (m > P) return;
  double X[36];
  if (!inv6_spd(Dc + 36 * (size_t)(m - 1), X)) {
    *fail = 1;
    for (int i = 0; i < 36; ++i) X[i] = (i % 7 == 0) ? 1.0 : 0.0;
  }
  for (int i = 0; i < 36; ++i) Di[36 * (size_t)(m - 1) + i] = X[i];
}
// nodes kept at this level: Schur complement and the coupling of stride 2s
__global__ void cr_reduce_kernel(int P, int s, int lshift, double* __restrict__ Dc, const double* __restrict__ Di,
                                 const double* __restrict__ Lcur, double* __restrict__ Lnext) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  const long long m = (long long)(t + 1) * 2 * s;  // m = 0 (mod 2s)
  if (m > P) return;
  double A[36], W[36], T[36];
  for (int i = 0; i < 36; ++i) A[i] = Dc[36 * (size_t)(m - 1) + i];
  const double* Lm = Lcur + 36 * (size_t)(m >> lshift);             // H[m][m-s]
  mm6(Lm, Di + 36 * (size_t)(m - s - 1), W);                        // W = Lm Dinv[m-s]   (m - s >= s >= 1 always)
  mmt6(W, Lm, T);
  for (int i = 0; i < 36; ++i) A[i] -= T[i];
  double* Ln = Lnext + 36 * (size_t)(m >> (lshift + 1));
  if (m - 2 * s >= 1) {
    mm6(W, Lcur + 36 * (size_t)((m - s) >> lshift), T);             // - W H[m-s][m-2s]
    for (int i = 0; i < 36; ++i) Ln[i] = -T[i];
  } else {
    for (int i = 0; i < 36; ++i) Ln[i] = 0.0;
  }
  if (m + s <= P) {
    const double* Lp = Lcur + 36 * (size_t)((m + s) >> lshift);     // H[m+s][m]
    mtm6(Lp, Di + 36 * (size_t)(m + s - 1), W);                     // V = Lp^T Dinv[m+s]
    mm6(W, Lp, T);
    for (int i = 0; i < 36; ++i) A[i] -= T[i];
  }
  for (int i = 0; i < 36; ++i) Dc[36 * (size_t)(m - 1) + i] = A[i];
}

// right-hand sides: Z[(k*6+i)*ncol + c] = -g (c == 0) or the c-th column of U^T
__global__ void cr_rhs_kernel(int P, int ncol, const FactorDev* __restrict__ fac, const int* __restrict__ extra_fac,
                              const double* __restrict__ Ja, const double* __restrict__ Jb, const double* __restrict__ g,
                              double* __restrict__ Z) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= ncol) return;
  if (c == 0) {
    for (int r = blockIdx.y; r < 6 * P; r += gridDim.y) Z[(size_t)r * ncol] = -g[r];
    return;
  }
  if (blockIdx.y != 0) return;
  const int f = extra_fac[(c - 1) / 6], row = (c - 1) % 6;
  const int ia = fac[f].ia, ib = fac[f].ib;
  for (int i = 0; i < 6; ++i) {
    if (ia >= 0) Z[((size_t)ia * 6 + i) * ncol + c] = Ja[36 * (size_t)f + 6 * row + i];
    Z[((size_t)ib * 6 + i) * ncol + c] = Jb[36 * (size_t)f + 6 * row + i];
  }
}
// unit right-hand sides of the marginals: column c = e_(pose[c / 6], c % 6)
__global__ void cr_unit_rhs_kernel(int ncol, const int* __restrict__ qpos, double* __restrict__ X) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < ncol) X[((size_t)qpos[c / 6] * 6 + c % 6) * ncol + c] = 1.0;
}
// The three kernels below run over (right-hand side column = x, node = y).  gridDim.y is capped at kMaxGridY (the CUDA
// limit); a level with more nodes than that (level 0 of a graph of more than 131070 poses) is launched with kStride and
// walks its nodes with a grid stride.  Every (node, column) is computed by the same arithmetic whatever the grid, and a
// level that fits one grid runs the single-node code.
constexpr int kMaxGridY = 65535;
// forward, eliminated nodes: t = Dinv b (in place)
template <bool kStride>
__global__ void cr_fwd_elim_kernel(int P, int s, int ncol, const double* __restrict__ Di, double* __restrict__ Z) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= ncol) return;
  for (long long m = (long long)s + (long long)blockIdx.y * 2 * s; m <= P; m += (long long)gridDim.y * 2 * s) {
    const double* X = Di + 36 * (size_t)(m - 1);
    double b[6], t[6];
    for (int i = 0; i < 6; ++i) b[i] = Z[((size_t)(m - 1) * 6 + i) * ncol + c];
    for (int i = 0; i < 6; ++i) {
      double v = 0.0;
      for (int j = 0; j < 6; ++j) v += X[6 * i + j] * b[j];
      t[i] = v;
    }
    for (int i = 0; i < 6; ++i) Z[((size_t)(m - 1) * 6 + i) * ncol + c] = t[i];
    if (!kStride) break;
  }
}
// forward, kept nodes: b -= H[m][m-s] t[m-s] + H[m][m+s] t[m+s]
template <bool kStride>
__global__ void cr_fwd_keep_kernel(int P, int s, int lshift, int ncol, const double* __restrict__ Lcur, double* __restrict__ Z) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= ncol) return;
  for (long long m = (long long)(blockIdx.y + 1) * 2 * s; m <= P; m += (long long)gridDim.y * 2 * s) {
    double b[6];
    for (int i = 0; i < 6; ++i) b[i] = Z[((size_t)(m - 1) * 6 + i) * ncol + c];
    {
      const double* Lm = Lcur + 36 * (size_t)(m >> lshift);
      double t[6];
      for (int i = 0; i < 6; ++i) t[i] = Z[((size_t)(m - s - 1) * 6 + i) * ncol + c];
      for (int i = 0; i < 6; ++i) {
        double v = 0.0;
        for (int j = 0; j < 6; ++j) v += Lm[6 * i + j] * t[j];
        b[i] -= v;
      }
    }
    if (m + s <= P) {
      const double* Lp = Lcur + 36 * (size_t)((m + s) >> lshift);
      double t[6];
      for (int i = 0; i < 6; ++i) t[i] = Z[((size_t)(m + s - 1) * 6 + i) * ncol + c];
      for (int i = 0; i < 6; ++i) {
        double v = 0.0;
        for (int j = 0; j < 6; ++j) v += Lp[6 * j + i] * t[j];
        b[i] -= v;
      }
    }
    for (int i = 0; i < 6; ++i) Z[((size_t)(m - 1) * 6 + i) * ncol + c] = b[i];
    if (!kStride) break;
  }
}
// backward, nodes eliminated at this level: x = t - Dinv (H[m][m-s] x[m-s] + H[m][m+s] x[m+s])
template <bool kStride>
__global__ void cr_bwd_kernel(int P, int s, int lshift, int ncol, const double* __restrict__ Di, const double* __restrict__ Lcur,
                              double* __restrict__ Z) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= ncol) return;
  for (long long m = (long long)s + (long long)blockIdx.y * 2 * s; m <= P; m += (long long)gridDim.y * 2 * s) {
    double r[6] = {0, 0, 0, 0, 0, 0};
    if (m - s >= 1) {
      const double* Lm = Lcur + 36 * (size_t)(m >> lshift);
      double x[6];
      for (int i = 0; i < 6; ++i) x[i] = Z[((size_t)(m - s - 1) * 6 + i) * ncol + c];
      for (int i = 0; i < 6; ++i)
        for (int j = 0; j < 6; ++j) r[i] += Lm[6 * i + j] * x[j];
    }
    if (m + s <= P) {
      const double* Lp = Lcur + 36 * (size_t)((m + s) >> lshift);
      double x[6];
      for (int i = 0; i < 6; ++i) x[i] = Z[((size_t)(m + s - 1) * 6 + i) * ncol + c];
      for (int i = 0; i < 6; ++i)
        for (int j = 0; j < 6; ++j) r[i] += Lp[6 * j + i] * x[j];
    }
    const double* X = Di + 36 * (size_t)(m - 1);
    for (int i = 0; i < 6; ++i) {
      double v = 0.0;
      for (int j = 0; j < 6; ++j) v += X[6 * i + j] * r[j];
      Z[((size_t)(m - 1) * 6 + i) * ncol + c] -= v;
    }
    if (!kStride) break;
  }
}

// ---------------------------------------------------------------- K6c: S = I + U Z (padded to n16), rhs = U y
__global__ void pg_border_kernel(int n, int n16, int ncol, const FactorDev* __restrict__ fac,
                                 const int* __restrict__ extra_fac, const double* __restrict__ Ja,
                                 const double* __restrict__ Jb, const double* __restrict__ Z, double* __restrict__ S,
                                 double* __restrict__ rhs) {
  const int col = blockIdx.x * blockDim.x + threadIdx.x;  // 0..n16 (col n16 => rhs)
  const int rowi = blockIdx.y;
  if (col > n16 || rowi >= n16) return;
  double v = 0.0;
  if (rowi < n && (col < n || col == n16)) {
    const int f = extra_fac[rowi / 6], rr = rowi % 6;
    const int zc = (col == n16) ? 0 : col + 1;
    const double* ja = Ja + 36 * (size_t)f + 6 * rr;
    const double* jb = Jb + 36 * (size_t)f + 6 * rr;
    const int ia = fac[f].ia, ib = fac[f].ib;
    if (ia >= 0)
      for (int i = 0; i < 6; ++i) v += ja[i] * Z[((size_t)ia * 6 + i) * ncol + zc];
    for (int i = 0; i < 6; ++i) v += jb[i] * Z[((size_t)ib * 6 + i) * ncol + zc];
  }
  if (col == n16) {
    rhs[rowi] = v;
  } else {
    if (rowi == col) v += 1.0;  // identity (also on the padding so the padded matrix stays SPD)
    S[(size_t)rowi * n16 + col] = v;
  }
}

// ---------------------------------------------------------------- K6d: dense SPD solve (right-looking, 16-wide panels)
constexpr int NB = 16;
__global__ void dense_panel_kernel(int n16, int p, double* __restrict__ A) {
  __shared__ double Lpp[NB][NB + 1];
  const int tid = threadIdx.x;
  for (int e = tid; e < NB * NB; e += blockDim.x) Lpp[e / NB][e % NB] = A[(size_t)(p + e / NB) * n16 + p + e % NB];
  __syncthreads();
  if (tid == 0) {
    for (int j = 0; j < NB; ++j) {
      double s = Lpp[j][j];
      for (int m = 0; m < j; ++m) s -= Lpp[j][m] * Lpp[j][m];
      const double dd = sqrt(s > 0.0 ? s : 1.0);
      Lpp[j][j] = dd;
      for (int i = j + 1; i < NB; ++i) {
        double v = Lpp[i][j];
        for (int m = 0; m < j; ++m) v -= Lpp[i][m] * Lpp[j][m];
        Lpp[i][j] = v / dd;
      }
    }
  }
  __syncthreads();
  for (int e = tid; e < NB * NB; e += blockDim.x) {
    const int i = e / NB, j = e % NB;
    A[(size_t)(p + i) * n16 + p + j] = (j <= i) ? Lpp[i][j] : 0.0;
  }
  // rows below the diagonal block: L[i, p:p+NB] = A[i, p:p+NB] * Lpp^-T
  for (int i = p + NB + tid; i < n16; i += blockDim.x) {
    double row[NB];
    for (int j = 0; j < NB; ++j) {
      double v = A[(size_t)i * n16 + p + j];
      for (int m = 0; m < j; ++m) v -= row[m] * Lpp[j][m];
      row[j] = v / Lpp[j][j];
    }
    for (int j = 0; j < NB; ++j) A[(size_t)i * n16 + p + j] = row[j];
  }
}

__global__ void dense_update_kernel(int n16, int p, double* __restrict__ A) {
  // trailing update of the lower triangle: A[i][j] -= sum_k L[i][p+k] L[j][p+k], tiles of 16x16
  const int bi = blockIdx.y + (p / NB) + 1, bj = blockIdx.x + (p / NB) + 1;
  if (bj > bi || bi * NB >= n16) return;
  __shared__ double Li[NB][NB + 1], Lj[NB][NB + 1];
  const int ty = threadIdx.y, tx = threadIdx.x;
  Li[ty][tx] = A[(size_t)(bi * NB + ty) * n16 + p + tx];
  Lj[ty][tx] = A[(size_t)(bj * NB + ty) * n16 + p + tx];
  __syncthreads();
  double s = 0.0;
  for (int k = 0; k < NB; ++k) s += Li[ty][k] * Lj[tx][k];
  A[(size_t)(bi * NB + ty) * n16 + bj * NB + tx] -= s;
}

// single CTA: forward then backward substitution with the factor in A's lower triangle
__global__ void dense_solve_kernel(int n16, const double* __restrict__ A, double* __restrict__ x) {
  __shared__ double xj;
  for (int j = 0; j < n16; ++j) {
    if (threadIdx.x == 0) { x[j] = x[j] / A[(size_t)j * n16 + j]; xj = x[j]; }
    __syncthreads();
    for (int i = j + 1 + threadIdx.x; i < n16; i += blockDim.x) x[i] -= A[(size_t)i * n16 + j] * xj;
    __syncthreads();
  }
  for (int j = n16 - 1; j >= 0; --j) {
    if (threadIdx.x == 0) { x[j] = x[j] / A[(size_t)j * n16 + j]; xj = x[j]; }
    __syncthreads();
    for (int i = threadIdx.x; i < j; i += blockDim.x) x[i] -= A[(size_t)j * n16 + i] * xj;
    __syncthreads();
  }
}

// ---------------------------------------------------------------- K6e: d = y - Z w, retract (warp per pose)
__global__ void pg_update_kernel(int P, int ncol, const double* __restrict__ Z, const double* __restrict__ w,
                                 double* __restrict__ poses, unsigned long long* dmax_bits) {
  const int k = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (k >= P) return;
  double d[6];
  for (int i = 0; i < 6; ++i) {
    const double* zr = Z + ((size_t)k * 6 + i) * ncol;
    double s = 0.0;
    for (int c = 1 + lane; c < ncol; c += 32) s += zr[c] * w[c - 1];
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    d[i] = zr[0] - s;
  }
  if (lane != 0) return;
  double* X = poses + 7 * (size_t)k;
  double m = 0.0;
  for (int i = 0; i < 6; ++i) m = fmax(m, fabs(d[i]));
  atomicMax(dmax_bits, (unsigned long long)__double_as_longlong(m));
  X[4] += d[0]; X[5] += d[1]; X[6] += d[2];
  const double th = sqrt(d[3] * d[3] + d[4] * d[4] + d[5] * d[5]);
  const double half = 0.5 * th;
  const double sc = th < 1e-8 ? 0.5 - th * th / 48.0 : sin(half) / th;
  const double dq[4] = {cos(half), sc * d[3], sc * d[4], sc * d[5]};
  const double q[4] = {X[0], X[1], X[2], X[3]};
  double o[4] = {q[0] * dq[0] - q[1] * dq[1] - q[2] * dq[2] - q[3] * dq[3],
                 q[0] * dq[1] + q[1] * dq[0] + q[2] * dq[3] - q[3] * dq[2],
                 q[0] * dq[2] - q[1] * dq[3] + q[2] * dq[0] + q[3] * dq[1],
                 q[0] * dq[3] + q[1] * dq[2] - q[2] * dq[1] + q[3] * dq[0]};
  const double n = 1.0 / sqrt(o[0] * o[0] + o[1] * o[1] + o[2] * o[2] + o[3] * o[3]);
  for (int i = 0; i < 4; ++i) X[i] = o[i] * n;
}

// ---------------------------------------------------------------- marginal covariances (gtsam::Marginals)
// Sigma_kk = (H^-1)_kk at the current estimate, for a chunk of requested poses.  Column c = 6*q + j is the unit vector
// e_(pose[q], j): X = H_c^-1 E through the cyclic-reduction levels (cr_unit_rhs_kernel + cr_solve), then the border correction
// through the same Woodbury identity as the update: Sigma = X - Z S^-1 (U X), of which only the 6x6 block of rows
// pose[q] is wanted.  X layout as Z: X[(k*6+i)*ncol + c].
// T = U X for the border rows (n of them, padded to n16 with zeros): T[row*ncol + c].  X is zero outside the column's track.
__global__ void pg_border_rhs_kernel(int n, int n16, int ncol, const FactorDev* __restrict__ fac, const int* __restrict__ extra_fac,
                                     const double* __restrict__ Ja, const double* __restrict__ Jb, const int* __restrict__ tb,
                                     const int* __restrict__ te, const double* __restrict__ X, double* __restrict__ T) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  const int rowi = blockIdx.y;
  if (c >= ncol || rowi >= n16) return;
  double v = 0.0;
  if (rowi < n) {
    const int f = extra_fac[rowi / 6], rr = rowi % 6;
    const int ia = fac[f].ia, ib = fac[f].ib;
    const int k0 = tb[c / 6], k1 = te[c / 6];
    const double* ja = Ja + 36 * (size_t)f + 6 * rr;
    const double* jb = Jb + 36 * (size_t)f + 6 * rr;
    if (ia >= k0 && ia < k1)
      for (int i = 0; i < 6; ++i) v += ja[i] * X[((size_t)ia * 6 + i) * ncol + c];
    if (ib >= k0 && ib < k1)
      for (int i = 0; i < 6; ++i) v += jb[i] * X[((size_t)ib * 6 + i) * ncol + c];
  }
  T[(size_t)rowi * ncol + c] = v;
}

// many right-hand sides against the dense factor (thread per column; W[row*ncol + c], coalesced across the threads)
__global__ void dense_solve_multi_kernel(int n16, int ncol, const double* __restrict__ A, double* __restrict__ W) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= ncol) return;
  for (int j = 0; j < n16; ++j) {
    double v = W[(size_t)j * ncol + c];
    for (int m = 0; m < j; ++m) v -= A[(size_t)j * n16 + m] * W[(size_t)m * ncol + c];
    W[(size_t)j * ncol + c] = v / A[(size_t)j * n16 + j];
  }
  for (int j = n16 - 1; j >= 0; --j) {
    double v = W[(size_t)j * ncol + c];
    for (int m = j + 1; m < n16; ++m) v -= A[(size_t)m * n16 + j] * W[(size_t)m * ncol + c];
    W[(size_t)j * ncol + c] = v / A[(size_t)j * n16 + j];
  }
}

// cov[q][i][j] = X[(pose q, i)][6q + j] - sum_r Z[(pose q, i)][1 + r] * W[r][6q + j]
__global__ void pg_marginal_block_kernel(int nq, int ncol, int n, int ncolZ, const int* __restrict__ qpos,
                                         const double* __restrict__ X, const double* __restrict__ Z, const double* __restrict__ W,
                                         double* __restrict__ cov) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= nq * 36) return;
  const int q = e / 36, i = (e % 36) / 6, j = e % 6;
  const int kp = qpos[q], c = 6 * q + j;
  double v = X[((size_t)kp * 6 + i) * ncol + c];
  const double* zr = Z + ((size_t)kp * 6 + i) * ncolZ + 1;
  for (int r = 0; r < n; ++r) v -= zr[r] * W[(size_t)r * ncol + c];
  cov[e] = v;
}

struct HostFactor {
  ls_factor f;
  bool active;
};

}  // namespace

struct ls_pg {
  int device = 0;
  cudaStream_t stream = nullptr;
  std::string err;
  // graph (host)
  std::vector<uint64_t> keys;        // insertion order
  std::vector<uint32_t> tracks;
  std::vector<double> poses;         // 7 per pose, insertion order
  std::unordered_map<uint64_t, int> key_index;
  std::vector<HostFactor> factors;
  uint64_t launches = 0;
  // device buffers, grown on demand in groups (solve); the first array of a group tells its capacity
  Buffer<FactorDev> d_fac;  // per factor
  Buffer<double> d_Ja, d_Jb, d_r;
  Buffer<double> d_poses, d_D, d_B, d_g;  // per pose
  Buffer<int> d_inc_ptr, d_track_begin, d_damp;
  Buffer<double> d_Dc, d_Di, d_Ll;  // cyclic reduction: current diagonals, inverses, per-level couplings
  Buffer<int> d_inc_fac, d_extra;
  Buffer<double> d_Z, d_S, d_rhs;
  Buffer<double> d_cost;
  Buffer<int> d_fail;
  Buffer<unsigned long long> d_dmax;
  // marginals scratch
  Buffer<double> d_X, d_W;
  Buffer<int> d_qpos, d_qtb, d_qte;  // per marginal, with d_cov
  Buffer<double> d_cov;
  cudaEvent_t e0 = nullptr, e1 = nullptr;
};

namespace {

int pg_fail(ls_pg* pg, int code, const char* msg) {
  if (pg) pg->err = msg;
  return code;
}

#define PGCU(call)                                                               \
  do {                                                                           \
    cudaError_t e_ = (call);                                                     \
    if (e_ != cudaSuccess) return pg_fail(pg, LS_ERR_CUDA, cudaGetErrorString(e_)); \
  } while (0)

}  // namespace

extern "C" {

int ls_pg_create(int device, ls_pg** out) {
  if (!out) return LS_ERR_ARG;
  *out = nullptr;
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || count <= 0) return LS_ERR_CUDA;  // no CPU fallback
  if (device < 0 || device >= count) return LS_ERR_ARG;
  ls_pg* pg = new ls_pg();
  pg->device = device;
  cudaSetDevice(device);
  if (cudaStreamCreateWithFlags(&pg->stream, cudaStreamNonBlocking) != cudaSuccess) { delete pg; return LS_ERR_CUDA; }
  if (pg->d_cost.reserve(1, 1) != cudaSuccess || pg->d_fail.reserve(1, 1) != cudaSuccess ||
      pg->d_dmax.reserve(1, 1) != cudaSuccess || cudaEventCreate(&pg->e0) != cudaSuccess ||
      cudaEventCreate(&pg->e1) != cudaSuccess) {
    ls_pg_destroy(pg);
    return LS_ERR_NOMEM;
  }
  *out = pg;
  return LS_OK;
}

void ls_pg_destroy(ls_pg* pg) {
  if (!pg) return;
  cudaSetDevice(pg->device);
  if (pg->stream) cudaStreamSynchronize(pg->stream);
  if (pg->e0) cudaEventDestroy(pg->e0);
  if (pg->e1) cudaEventDestroy(pg->e1);
  if (pg->stream) cudaStreamDestroy(pg->stream);
  delete pg;
}

const char* ls_pg_last_error(const ls_pg* pg) { return pg ? pg->err.c_str() : "null graph"; }
uint64_t ls_pg_launch_count(const ls_pg* pg) { return pg ? pg->launches : 0; }
int ls_pg_num_poses(const ls_pg* pg) { return pg ? (int)pg->keys.size() : LS_ERR_ARG; }
int ls_pg_num_factors(const ls_pg* pg) {
  if (!pg) return LS_ERR_ARG;
  int n = 0;
  for (const auto& f : pg->factors) n += f.active ? 1 : 0;
  return n;
}

int ls_pg_add_poses(ls_pg* pg, const uint64_t* keys, const uint32_t* track_ids, const double* poses7, int n) {
  if (!pg || !keys || !poses7 || n < 0) return pg_fail(pg, LS_ERR_ARG, "bad argument");
  for (int i = 0; i < n; ++i) {
    if (pg->key_index.count(keys[i])) return pg_fail(pg, LS_ERR_ARG, "duplicate pose key");
    pg->key_index[keys[i]] = (int)pg->keys.size();
    pg->keys.push_back(keys[i]);
    pg->tracks.push_back(track_ids ? track_ids[i] : 0u);
    pg->poses.insert(pg->poses.end(), poses7 + 7 * (size_t)i, poses7 + 7 * (size_t)i + 7);
  }
  return LS_OK;
}

int ls_pg_set_poses(ls_pg* pg, const uint64_t* keys, const double* poses7, int n) {
  if (!pg || !keys || !poses7 || n < 0) return pg_fail(pg, LS_ERR_ARG, "bad argument");
  for (int i = 0; i < n; ++i) {
    auto it = pg->key_index.find(keys[i]);
    if (it == pg->key_index.end()) return pg_fail(pg, LS_ERR_ARG, "unknown pose key");
    std::memcpy(&pg->poses[7 * (size_t)it->second], poses7 + 7 * (size_t)i, 7 * sizeof(double));
  }
  return LS_OK;
}

int ls_pg_add_factors(ls_pg* pg, const ls_factor* f, int n, uint64_t* out_indices) {
  if (!pg || !f || n < 0) return pg_fail(pg, LS_ERR_ARG, "bad argument");
  for (int i = 0; i < n; ++i) {
    if (f[i].type != LS_FACTOR_PRIOR && f[i].type != LS_FACTOR_BETWEEN) return pg_fail(pg, LS_ERR_ARG, "bad factor type");
    for (int s = 0; s < 6; ++s)
      if (!(f[i].sigma[s] > 0.0)) return pg_fail(pg, LS_ERR_ARG, "sigma must be positive");
    if (out_indices) out_indices[i] = pg->factors.size();
    pg->factors.push_back(HostFactor{f[i], true});
  }
  return LS_OK;
}

int ls_pg_remove_factors(ls_pg* pg, const uint64_t* idx, int n) {
  if (!pg || !idx || n < 0) return pg_fail(pg, LS_ERR_ARG, "bad argument");
  for (int i = 0; i < n; ++i) {
    if (idx[i] >= pg->factors.size() || !pg->factors[idx[i]].active) return pg_fail(pg, LS_ERR_ARG, "bad factor index");
    pg->factors[idx[i]].active = false;
  }
  return LS_OK;
}

int ls_pg_get_poses(const ls_pg* pg, uint64_t* out_keys, double* out_poses7, int* n) {
  if (!pg || !n) return LS_ERR_ARG;
  *n = (int)pg->keys.size();
  if (out_keys) std::memcpy(out_keys, pg->keys.data(), pg->keys.size() * sizeof(uint64_t));
  if (out_poses7) std::memcpy(out_poses7, pg->poses.data(), pg->poses.size() * sizeof(double));
  return LS_OK;
}

}  // extern "C"

namespace {
// gn_iters Gauss-Newton iterations, then -- when n_mk > 0 -- the marginal covariances of the poses mkeys[0..n_mk) at
// the resulting estimate (one more linearisation, no update).
int pg_run(ls_pg* pg, int gn_iters, ls_pg_stats* stats, const uint64_t* mkeys, int n_mk, double* cov_out) {
  if (stats) std::memset(stats, 0, sizeof(*stats));
  const int P = (int)pg->keys.size();
  if (P == 0 || (gn_iters == 0 && n_mk == 0)) return LS_OK;
  PGCU(cudaSetDevice(pg->device));
  // ---- ordering: track by track, insertion order inside a track (= time order in laser_slam)
  std::map<uint32_t, std::vector<int>> by_track;
  for (int i = 0; i < P; ++i) by_track[pg->tracks[i]].push_back(i);
  std::vector<int> order, pos_of(P), track_begin;
  for (auto& kv : by_track) {
    track_begin.push_back((int)order.size());
    for (int i : kv.second) { pos_of[i] = (int)order.size(); order.push_back(i); }
  }
  track_begin.push_back(P);
  const int n_tracks = (int)track_begin.size() - 1;
  std::vector<int> track_of_pos(P);
  for (int t = 0; t < n_tracks; ++t)
    for (int k = track_begin[t]; k < track_begin[t + 1]; ++k) track_of_pos[k] = t;
  // ---- factor table
  std::vector<FactorDev> fd;
  std::vector<int> extra_fac;
  for (const auto& hf : pg->factors) {
    if (!hf.active) continue;
    const ls_factor& f = hf.f;
    FactorDev d;
    std::memset(&d, 0, sizeof(d));
    d.type = f.type;
    d.robust = f.robust;
    d.fix_a = (f.type == LS_FACTOR_BETWEEN) ? f.fix_a : 0;
    d.extra = -1;
    auto ita = pg->key_index.find(f.key_a), itb = pg->key_index.find(f.key_b);
    if (f.type == LS_FACTOR_PRIOR) {
      if (ita == pg->key_index.end()) return pg_fail(pg, LS_ERR_ARG, "prior on unknown key");
      d.ia = -1;
      d.ib = pos_of[ita->second];
    } else {
      if (itb == pg->key_index.end() || (!d.fix_a && ita == pg->key_index.end()))
        return pg_fail(pg, LS_ERR_ARG, "between factor on unknown key");
      d.ib = pos_of[itb->second];
      d.ia = d.fix_a ? -1 : pos_of[ita->second];
      if (!d.fix_a && d.ib == d.ia + 1 && track_of_pos[d.ia] == track_of_pos[d.ib]) {
        d.chain = 1;  // consecutive poses of one track: part of the block-tridiagonal H_c
      }
      if (!d.fix_a && !d.chain) {  // everything else (loop closures, reversed pairs) goes to the border
        if (d.ia == d.ib) return pg_fail(pg, LS_ERR_ARG, "between factor with identical nodes");
        d.extra = (int)extra_fac.size();
        extra_fac.push_back((int)fd.size());
      }
    }
    std::memcpy(d.meas, f.meas, sizeof(d.meas));
    std::memcpy(d.sigma, f.sigma, sizeof(d.sigma));
    std::memcpy(d.fixed_a, f.fixed_a, sizeof(d.fixed_a));
    fd.push_back(d);
  }
  const int F = (int)fd.size();
  if (F == 0) return LS_OK;
  // the dense border system is n16 x n16 (n16 = 6 E padded to the panel width) and its kernels launch n16 rows on
  // gridDim.y: at most 65520 rows, i.e. 10920 border factors (a 34 GB matrix)
  constexpr int kMaxBorder = (kMaxGridY / NB) * NB / 6;
  if ((int)extra_fac.size() > kMaxBorder)
    return pg_fail(pg, LS_ERR_ARG, ("more than " + std::to_string(kMaxBorder) + " border factors (loop closures, skip and "
                                    "reversed factors): the dense border solve supports at most " +
                                    std::to_string(kMaxBorder)).c_str());
  // ---- gauge, per chain segment: a maximal run of positions joined by chain factors is one independent block of H_c.
  // A segment without prior / fixed-node factor must at least be tied to the rest by a border factor; its first pose is
  // then damped.  For a track without gaps the segment is the whole track; a gap (a removed odometry factor, a pose with
  // only border factors) starts a new segment that needs its own anchor or damping.
  std::vector<int> damp(P, 0);
  {
    std::vector<char> joined(P, 0);  // joined[k]: a chain factor couples positions k - 1 and k
    for (const auto& d : fd)
      if (d.chain) joined[d.ib] = 1;
    std::vector<int> seg_of(P), seg_begin;
    for (int k = 0; k < P; ++k) {
      if (!joined[k]) seg_begin.push_back(k);
      seg_of[k] = (int)seg_begin.size() - 1;
    }
    const int n_seg = (int)seg_begin.size();
    std::vector<char> anchored(n_seg, 0), linked(n_seg, 0);
    for (const auto& d : fd)
      if (d.type == LS_FACTOR_PRIOR || d.fix_a) anchored[seg_of[d.ib]] = 1;
    for (int fi : extra_fac) {
      if (fd[fi].ia >= 0) linked[seg_of[fd[fi].ia]] = 1;
      linked[seg_of[fd[fi].ib]] = 1;
    }
    for (int sg = 0; sg < n_seg; ++sg)
      if (!anchored[sg]) {
        if (!linked[sg])
          return pg_fail(pg, LS_ERR_STATE, ("pose " + std::to_string(pg->keys[order[seg_begin[sg]]]) +
                                            " starts a chain segment with no prior, no fixed-node factor and no link to "
                                            "the rest of the graph: the graph has a free gauge").c_str());
        damp[seg_begin[sg]] = 1;
      }
  }
  const int E = (int)extra_fac.size();
  const int n = 6 * E, n16 = ((n + NB - 1) / NB) * NB, ncol = n + 1;
  // incidence lists
  std::vector<int> inc_ptr(P + 1, 0), inc_fac;
  for (const auto& d : fd) { if (d.ia >= 0) ++inc_ptr[d.ia + 1]; ++inc_ptr[d.ib + 1]; }
  for (int k = 0; k < P; ++k) inc_ptr[k + 1] += inc_ptr[k];
  inc_fac.resize(inc_ptr[P]);
  {
    std::vector<int> cur(inc_ptr.begin(), inc_ptr.end() - 1);
    for (int f = 0; f < F; ++f) {
      if (fd[f].ia >= 0) inc_fac[cur[fd[f].ia]++] = f;
      inc_fac[cur[fd[f].ib]++] = f;
    }
  }
  std::vector<double> hp(7 * (size_t)P);
  for (int k = 0; k < P; ++k) std::memcpy(&hp[7 * (size_t)k], &pg->poses[7 * (size_t)order[k]], 7 * sizeof(double));
  // ---- device buffers
  // each group grows all or nothing: when one array fails the group is emptied, so a later call regrows all of it
  cudaError_t e;
  if ((size_t)F > pg->d_fac.capacity()) {
    const size_t cap = (size_t)F + F / 4 + 64;
    if ((e = pg->d_fac.reserve(cap, cap)) || (e = pg->d_Ja.reserve(cap * 36, cap * 36)) ||
        (e = pg->d_Jb.reserve(cap * 36, cap * 36)) || (e = pg->d_r.reserve(cap * 6, cap * 6))) {
      pg->d_fac.reset(), pg->d_Ja.reset(), pg->d_Jb.reset(), pg->d_r.reset();
      PGCU(e);
    }
  }
  if ((size_t)P > pg->d_poses.capacity() / 7) {
    const size_t cap = (size_t)P + P / 4 + 64;
    if ((e = pg->d_poses.reserve(cap * 7, cap * 7)) || (e = pg->d_D.reserve(cap * 36, cap * 36)) ||
        (e = pg->d_B.reserve(cap * 36, cap * 36)) || (e = pg->d_g.reserve(cap * 6, cap * 6)) ||
        (e = pg->d_inc_ptr.reserve(cap + 1, cap + 1)) || (e = pg->d_track_begin.reserve(cap + 1, cap + 1)) ||
        (e = pg->d_damp.reserve(cap + 1, cap + 1))) {
      pg->d_poses.reset(), pg->d_D.reset(), pg->d_B.reset(), pg->d_g.reset(), pg->d_inc_ptr.reset(), pg->d_track_begin.reset();
      pg->d_damp.reset();
      PGCU(e);
    }
  }
  // cyclic-reduction levels: level l holds one coupling per node m = j << l, j = 1 .. P >> l
  std::vector<size_t> lvl_off;
  size_t lvl_total = 0;
  int n_levels = 0;
  for (int l = 0; (1ll << l) <= (long long)P; ++l) {
    lvl_off.push_back(lvl_total);
    lvl_total += ((size_t)P >> l) + 1;
    ++n_levels;
  }
  lvl_off.push_back(lvl_total);
  lvl_total += 2;  // the "next level" slot the top level's (empty) reduction would write
  const size_t capCR = pg->d_Dc.capacity() / 36;
  if (lvl_total > capCR || (size_t)P > capCR) {
    const size_t cap = (lvl_total + lvl_total / 4 + 64) * 36;
    if ((e = pg->d_Dc.reserve(cap, cap)) || (e = pg->d_Di.reserve(cap, cap)) || (e = pg->d_Ll.reserve(cap, cap))) {
      pg->d_Dc.reset(), pg->d_Di.reset(), pg->d_Ll.reset();
      PGCU(e);
    }
  }
  PGCU(pg->d_inc_fac.reserve(inc_fac.size(), inc_fac.size() * 2 + 64));
  PGCU(pg->d_extra.reserve((size_t)E + 1, (size_t)E * 2 + 64));
  const size_t needZ = (size_t)P * 6 * ncol;
  PGCU(pg->d_Z.reserve(needZ, needZ + needZ / 4));
  const size_t needS = (size_t)n16 * n16 + n16 + 16;
  if (needS > pg->d_S.capacity()) {
    const size_t capR = (size_t)n16 * 2 + 64;
    if ((e = pg->d_S.reserve(needS * 2, needS * 2)) || (e = pg->d_rhs.reserve(capR, capR))) {
      pg->d_S.reset(), pg->d_rhs.reset();
      PGCU(e);
    }
  }
  cudaStream_t st = pg->stream;
  PGCU(cudaMemcpyAsync(pg->d_fac.get(), fd.data(), (size_t)F * sizeof(FactorDev), cudaMemcpyHostToDevice, st));
  PGCU(cudaMemcpyAsync(pg->d_poses.get(), hp.data(), hp.size() * sizeof(double), cudaMemcpyHostToDevice, st));
  PGCU(cudaMemcpyAsync(pg->d_inc_ptr.get(), inc_ptr.data(), inc_ptr.size() * sizeof(int), cudaMemcpyHostToDevice, st));
  PGCU(cudaMemcpyAsync(pg->d_inc_fac.get(), inc_fac.data(), inc_fac.size() * sizeof(int), cudaMemcpyHostToDevice, st));
  if (E) PGCU(cudaMemcpyAsync(pg->d_extra.get(), extra_fac.data(), (size_t)E * sizeof(int), cudaMemcpyHostToDevice, st));
  PGCU(cudaMemcpyAsync(pg->d_track_begin.get(), track_begin.data(), track_begin.size() * sizeof(int), cudaMemcpyHostToDevice,
                       st));
  PGCU(cudaMemcpyAsync(pg->d_damp.get(), damp.data(), (size_t)P * sizeof(int), cudaMemcpyHostToDevice, st));
  PGCU(cudaMemsetAsync(pg->d_fail.get(), 0, sizeof(int), st));
  cudaEvent_t e0 = pg->e0, e1 = pg->e1;
  cudaEventRecord(e0, st);
  double cost_first = 0.0, cost_last = 0.0, dmax_last = 0.0;
  // every right-hand side of `buf` (6P x ncols, column index fastest) through the factored levels, in place
  auto cr_solve = [&](double* buf, int ncols) {
    for (int l = 0; l < n_levels; ++l) {
      const long long sl = 1ll << l;
      const int n_elim = (int)((P - sl) / (2 * sl)) + 1, n_keep = (int)(P / (2 * sl));
      if (n_elim > kMaxGridY)
        cr_fwd_elim_kernel<true><<<dim3((ncols + 127) / 128, kMaxGridY), 128, 0, st>>>(P, (int)sl, ncols, pg->d_Di.get(), buf);
      else
        cr_fwd_elim_kernel<false><<<dim3((ncols + 127) / 128, n_elim), 128, 0, st>>>(P, (int)sl, ncols, pg->d_Di.get(), buf);
      if (n_keep > kMaxGridY)
        cr_fwd_keep_kernel<true><<<dim3((ncols + 127) / 128, kMaxGridY), 128, 0, st>>>(P, (int)sl, l, ncols,
                                                                                       pg->d_Ll.get() + 36 * lvl_off[l], buf);
      else if (n_keep > 0)
        cr_fwd_keep_kernel<false><<<dim3((ncols + 127) / 128, n_keep), 128, 0, st>>>(P, (int)sl, l, ncols,
                                                                                     pg->d_Ll.get() + 36 * lvl_off[l], buf);
      pg->launches += n_keep > 0 ? 2 : 1;
    }
    for (int l = n_levels - 1; l >= 0; --l) {
      const long long sl = 1ll << l;
      const int n_elim = (int)((P - sl) / (2 * sl)) + 1;
      if (n_elim > kMaxGridY)
        cr_bwd_kernel<true><<<dim3((ncols + 127) / 128, kMaxGridY), 128, 0, st>>>(P, (int)sl, l, ncols, pg->d_Di.get(),
                                                                                  pg->d_Ll.get() + 36 * lvl_off[l], buf);
      else
        cr_bwd_kernel<false><<<dim3((ncols + 127) / 128, n_elim), 128, 0, st>>>(P, (int)sl, l, ncols, pg->d_Di.get(),
                                                                                pg->d_Ll.get() + 36 * lvl_off[l], buf);
      ++pg->launches;
    }
  };
  const int n_pass = gn_iters + (n_mk > 0 ? 1 : 0);  // the last pass of a marginals request only linearises and factors
  for (int it = 0; it < n_pass; ++it) {
    const bool update = it < gn_iters;
    PGCU(cudaMemsetAsync(pg->d_cost.get(), 0, sizeof(double), st));
    PGCU(cudaMemsetAsync(pg->d_dmax.get(), 0, sizeof(unsigned long long), st));
    pg_linearize_kernel<<<(F + 127) / 128, 128, 0, st>>>(F, pg->d_fac.get(), pg->d_poses.get(), pg->d_Ja.get(), pg->d_Jb.get(),
                                                         pg->d_r.get(), pg->d_cost.get());
    pg_assemble_kernel<<<(P + 127) / 128, 128, 0, st>>>(P, pg->d_inc_ptr.get(), pg->d_inc_fac.get(), pg->d_fac.get(),
                                                        pg->d_Ja.get(), pg->d_Jb.get(), pg->d_r.get(),
                                                        pg->d_damp.get(), pg->d_D.get(), pg->d_B.get(), pg->d_g.get());
    // H_c^-1 [ -g | U^T ] by block cyclic reduction (K6a'): factor the levels, then every right-hand side through them
    cr_init_kernel<<<(P + 127) / 128, 128, 0, st>>>(P, pg->d_D.get(), pg->d_B.get(), pg->d_Dc.get(),
                                                    pg->d_Ll.get() + 36 * lvl_off[0]);
    for (int l = 0; l < n_levels; ++l) {
      const long long sl = 1ll << l;
      const int n_elim = (int)((P - sl) / (2 * sl)) + 1, n_keep = (int)(P / (2 * sl));
      cr_invert_kernel<<<(n_elim + 63) / 64, 64, 0, st>>>(P, (int)sl, pg->d_Dc.get(), pg->d_Di.get(), pg->d_fail.get());
      if (n_keep > 0)
        cr_reduce_kernel<<<(n_keep + 63) / 64, 64, 0, st>>>(P, (int)sl, l, pg->d_Dc.get(), pg->d_Di.get(),
                                                            pg->d_Ll.get() + 36 * lvl_off[l],
                                                            pg->d_Ll.get() + 36 * lvl_off[l + 1]);
      pg->launches += n_keep > 0 ? 2 : 1;
    }
    PGCU(cudaMemsetAsync(pg->d_Z.get(), 0, (size_t)P * 6 * ncol * sizeof(double), st));
    cr_rhs_kernel<<<dim3((ncol + 127) / 128, 256), 128, 0, st>>>(P, ncol, pg->d_fac.get(), pg->d_extra.get(), pg->d_Ja.get(),
                                                                 pg->d_Jb.get(), pg->d_g.get(), pg->d_Z.get());
    cr_solve(pg->d_Z.get(), ncol);
    pg->launches += 4;
    if (E) {
      pg_border_kernel<<<dim3((n16 + 1 + 127) / 128, n16), 128, 0, st>>>(n, n16, ncol, pg->d_fac.get(), pg->d_extra.get(),
                                                                         pg->d_Ja.get(), pg->d_Jb.get(),
                                                                        pg->d_Z.get(), pg->d_S.get(), pg->d_rhs.get());
      ++pg->launches;
      for (int p = 0; p < n16; p += NB) {
        dense_panel_kernel<<<1, 256, 0, st>>>(n16, p, pg->d_S.get());
        const int rem = (n16 - p - NB) / NB;
        if (rem > 0) dense_update_kernel<<<dim3(rem, rem), dim3(NB, NB), 0, st>>>(n16, p, pg->d_S.get());
        pg->launches += rem > 0 ? 2 : 1;
      }
      if (update) {
        dense_solve_kernel<<<1, 1024, 0, st>>>(n16, pg->d_S.get(), pg->d_rhs.get());
        ++pg->launches;
      }
    }
    if (!update) break;
    pg_update_kernel<<<(P * 32 + 255) / 256, 256, 0, st>>>(P, ncol, pg->d_Z.get(), pg->d_rhs.get(), pg->d_poses.get(),
                                                           pg->d_dmax.get());
    ++pg->launches;
    if (it == 0 || it == gn_iters - 1) {
      double c;
      unsigned long long dm;
      PGCU(cudaMemcpyAsync(&c, pg->d_cost.get(), sizeof(double), cudaMemcpyDeviceToHost, st));
      PGCU(cudaMemcpyAsync(&dm, pg->d_dmax.get(), sizeof(dm), cudaMemcpyDeviceToHost, st));
      PGCU(cudaStreamSynchronize(st));
      if (it == 0) cost_first = c;
      cost_last = c;
      std::memcpy(&dmax_last, &dm, sizeof(double));
    }
  }
  // ---- marginal covariances at the estimate just linearised: chunks of requested poses
  if (n_mk > 0) {
    constexpr int kChunk = 64;
    std::vector<int> qpos(n_mk), qtb(n_mk), qte(n_mk);
    for (int q = 0; q < n_mk; ++q) {
      auto it = pg->key_index.find(mkeys[q]);
      if (it == pg->key_index.end()) return pg_fail(pg, LS_ERR_ARG, "marginal of an unknown key");
      qpos[q] = pos_of[it->second];
      qtb[q] = track_begin[track_of_pos[qpos[q]]];
      qte[q] = track_begin[track_of_pos[qpos[q]] + 1];
    }
    const int ncm = 6 * kChunk;
    const size_t needX = (size_t)P * 6 * ncm, needW = (size_t)(n16 > 0 ? n16 : 1) * ncm;
    PGCU(pg->d_X.reserve(needX, needX));
    PGCU(pg->d_W.reserve(needW, needW));
    if ((size_t)n_mk > pg->d_qpos.capacity()) {
      const size_t cap = (size_t)n_mk + 64;
      if ((e = pg->d_qpos.reserve(cap, cap)) || (e = pg->d_qtb.reserve(cap, cap)) || (e = pg->d_qte.reserve(cap, cap)) ||
          (e = pg->d_cov.reserve(cap * 36, cap * 36))) {
        pg->d_qpos.reset(), pg->d_qtb.reset(), pg->d_qte.reset(), pg->d_cov.reset();
        PGCU(e);
      }
    }
    PGCU(cudaMemcpyAsync(pg->d_qpos.get(), qpos.data(), (size_t)n_mk * sizeof(int), cudaMemcpyHostToDevice, st));
    PGCU(cudaMemcpyAsync(pg->d_qtb.get(), qtb.data(), (size_t)n_mk * sizeof(int), cudaMemcpyHostToDevice, st));
    PGCU(cudaMemcpyAsync(pg->d_qte.get(), qte.data(), (size_t)n_mk * sizeof(int), cudaMemcpyHostToDevice, st));
    for (int q0 = 0; q0 < n_mk; q0 += kChunk) {
      const int nq = n_mk - q0 < kChunk ? n_mk - q0 : kChunk, nc = 6 * nq;
      PGCU(cudaMemsetAsync(pg->d_X.get(), 0, (size_t)P * 6 * nc * sizeof(double), st));
      cr_unit_rhs_kernel<<<(nc + 127) / 128, 128, 0, st>>>(nc, pg->d_qpos.get() + q0, pg->d_X.get());
      ++pg->launches;
      cr_solve(pg->d_X.get(), nc);
      if (E) {
        pg_border_rhs_kernel<<<dim3((nc + 127) / 128, n16), 128, 0, st>>>(n, n16, nc, pg->d_fac.get(), pg->d_extra.get(),
                                                                          pg->d_Ja.get(), pg->d_Jb.get(), pg->d_qtb.get() + q0,
                                                                          pg->d_qte.get() + q0, pg->d_X.get(), pg->d_W.get());
        dense_solve_multi_kernel<<<(nc + 63) / 64, 64, 0, st>>>(n16, nc, pg->d_S.get(), pg->d_W.get());
        pg->launches += 2;
      }
      pg_marginal_block_kernel<<<(nq * 36 + 127) / 128, 128, 0, st>>>(nq, nc, E ? n : 0, ncol, pg->d_qpos.get() + q0,
                                                                      pg->d_X.get(), pg->d_Z.get(),
                                                                      pg->d_W.get(), pg->d_cov.get() + 36 * (size_t)q0);
      ++pg->launches;
    }
    PGCU(cudaMemcpyAsync(cov_out, pg->d_cov.get(), (size_t)n_mk * 36 * sizeof(double), cudaMemcpyDeviceToHost, st));
  }
  cudaEventRecord(e1, st);
  int fail = 0;
  PGCU(cudaMemcpyAsync(&fail, pg->d_fail.get(), sizeof(int), cudaMemcpyDeviceToHost, st));
  PGCU(cudaMemcpyAsync(hp.data(), pg->d_poses.get(), hp.size() * sizeof(double), cudaMemcpyDeviceToHost, st));
  PGCU(cudaStreamSynchronize(st));
  PGCU(cudaGetLastError());
  float ms = 0.f;
  cudaEventElapsedTime(&ms, e0, e1);
  if (fail) return pg_fail(pg, LS_ERR_CONVERGENCE, "chain block not positive definite (under-constrained graph)");
  for (int k = 0; k < P; ++k)
    for (int i = 0; i < 7; ++i)
      if (!std::isfinite(hp[7 * (size_t)k + i])) return pg_fail(pg, LS_ERR_CONVERGENCE, "non-finite pose after update");
  for (int k = 0; k < P; ++k) std::memcpy(&pg->poses[7 * (size_t)order[k]], &hp[7 * (size_t)k], 7 * sizeof(double));
  if (stats) {
    stats->iterations = gn_iters;
    stats->n_poses = P;
    stats->n_factors = F;
    stats->n_border = E;
    stats->cost_first = cost_first;
    stats->cost_last = cost_last;
    stats->last_step_max = dmax_last;
    stats->device_ms = ms;
  }
  return LS_OK;
}
}  // namespace

extern "C" {

int ls_pg_optimize(ls_pg* pg, int gn_iters, ls_pg_stats* stats) {
  if (!pg || gn_iters < 0) return pg_fail(pg, LS_ERR_ARG, "bad argument");
  return pg_run(pg, gn_iters, stats, nullptr, 0, nullptr);
}

int ls_pg_marginals(ls_pg* pg, const uint64_t* keys, int n, double* out_cov36) {
  if (!pg || !keys || !out_cov36 || n < 0) return pg_fail(pg, LS_ERR_ARG, "bad argument");
  if (n == 0) return LS_OK;
  return pg_run(pg, 0, nullptr, keys, n, out_cov36);
}

}  // extern "C"
