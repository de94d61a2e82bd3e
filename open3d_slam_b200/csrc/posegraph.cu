// posegraph.cu -- G1: the submap pose-graph optimisation, [O3D] GlobalOptimization with GlobalOptimizationLevenbergMarquardt as
// OptimizationProblem::solve (core/src/OptimizationProblem.cpp:25-44) calls it.  The semantics restated here (DESIGN.md row G1, and
// tests/oracle_pose_graph.py, which holds the same list):
//   1. validation: ids in [0, N) (checked by the C entry point); connected from node 0 over all edges and over the certain edges
//      alone (BFS), else the poses stay and valid = 0
//   2. lpw = preference_loop_closure * max_correspondence_distance^2 * mean_e information_e(5,5), 0 without edges
//   3. zeta_e = lin(X^-1 Tt^-1 Ts), lin(M) = ((M21-M12)/2, (M02-M20)/2, (M10-M01)/2, M03, M13, M23), Js[:,i] = lin(X^-1 Tt^-1 G_i Ts),
//      Jt = -Js (bit for bit: -G_i Ts = -(G_i Ts)).  Inverses are the rigid ones (R', -R't) where [O3D] calls Eigen's general inverse
//   4. uncertain edges: conf = (lpw / (lpw + zeta' Info zeta))^2, certain edges keep theirs (1); residual = sum_e conf q_e +
//      lpw (sqrt(conf) - 1)^2; H and b get the four blocks of every edge, which are +-conf Js' Info Js and -+conf (zeta' Info Js)'
//   5. the LM loop of GlobalOptimizationLevenbergMarquardt::OptimizePoseGraph, on the host (op_global_optimization below)
//   6. two passes (all edges; the certain ones and the uncertain ones with conf > edge_prune_threshold), then the reference node
//   7. delta = (H + lambda I)^-1 b by an UNPIVOTED LDL' with Eigen's zero-pivot rule (|d| <= 1/DBL_MAX: the component is 0)
//
// Kernels of one LM try, captured once as a CUDA graph per (padded size, node count, edge capacity) and replayed per try:
//   K-pg-form      F = lower(H) + lambda I, padded to whole 64 x 64 tiles with an identity block; rhs = b
//   per tile column K:  K-pg-diag (one CTA: the tile's LDL' in shared memory), K-pg-panel (one CTA per tile row: L = A L_KK^-T D^-1,
//                  W = L D kept for the update), K-pg-trailing (one CTA per lower tile: A_IJ -= W_I L_J' on mma.sync m8n8k4 f64)
//   per tile:      K-pg-fwd (L y = rhs, z = D^-1 y), then K-pg-bwd (L' delta = z): every CTA re-solves the diagonal tile and updates
//                  its own tile of the right-hand side
//   K-pg-update    trial poses V2M(delta_i) T_i; K-pg-edge (trial zeta and residual terms); K-pg-reduce-try (one record)
// An accepted try adds K-pg-edge (linearise: confidences, per-edge blocks), K-pg-assemble (one CTA per nonzero node block: its
// incident edges summed in edge order from host-built lists) and K-pg-reduce-lin.  Every sum has a fixed order and there are no
// atomics: a repeated call is bit-identical.  The test hooks b2s_debug_pose_graph_solve / _linearize run the same launch functions
// (pg_factor_solve; pg_load, pg_eval and pg_linearize) on host-given inputs.
#include "common.cuh"

#include <algorithm>
#include <cfloat>
#include <cmath>

namespace b2s {

constexpr int PG_NB = 64;                 // tile of the blocked factorisation
constexpr double PG_TINY = 1.0 / DBL_MAX;   // Eigen's LDLT::solve: a pivot with |d| <= this zeroes its component
constexpr int PG_RED = 256;
enum { PG_C_SOURCE = 0, PG_C_TARGET = 1, PG_C_CROSS = 2 };   // contribution codes: +Hss and b -= g / +Hss and b += g / -Hss
enum { PG_S_LAMBDA = 0, PG_S_LPW = 1 };                        // device scalars
enum { PG_R_RES = 0, PG_R_DD = 1, PG_R_DLB = 2, PG_R_MAXB = 3, PG_R_MAXDIAG = 4, PG_R_XX = 5, PG_R_WORDS = 8 };

struct PgTask { int32_t row, col, begin, end; };   // node block (row >= col) and its contribution list [begin, end)

__device__ __forceinline__ void pg_mul4(const double* A, const double* B, double* C) {
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < 4; j++) {
      double s = 0.0;
#pragma unroll
      for (int k = 0; k < 4; k++) s += A[4 * i + k] * B[4 * k + j];
      C[4 * i + j] = s;
    }
}

__device__ __forceinline__ void pg_inv_rigid(const double* T, double* R) {
#pragma unroll
  for (int i = 0; i < 3; i++)
#pragma unroll
    for (int j = 0; j < 3; j++) R[4 * i + j] = T[4 * j + i];
#pragma unroll
  for (int i = 0; i < 3; i++) R[4 * i + 3] = -((R[4 * i] * T[3] + R[4 * i + 1] * T[7]) + R[4 * i + 2] * T[11]);
  R[12] = 0.0; R[13] = 0.0; R[14] = 0.0; R[15] = 1.0;
}

__device__ __forceinline__ void pg_lin(const double* M, double* v) {   // GetLinearized6DVector
  v[0] = (M[9] - M[6]) / 2.0; v[1] = (M[2] - M[8]) / 2.0; v[2] = (M[4] - M[1]) / 2.0;
  v[3] = M[3]; v[4] = M[7]; v[5] = M[11];
}

// K-pg-edge, one thread per edge.  linearize = 0: the residual term of the poses P with the current confidences.  linearize = 1:
// the confidence update, then Hss = conf Js' Info Js and g = conf (zeta' Info Js)' of the edge
__global__ void __launch_bounds__(128) pg_edge_kernel(const b2s_pose_graph_edge* __restrict__ E, const int32_t* __restrict__ ne_dev,
                                                      const double* __restrict__ P, double* __restrict__ conf, const double* __restrict__ scal,
                                                      int linearize, double* __restrict__ term, double* __restrict__ hss, double* __restrict__ gv) {
  pdl_wait();
  const int ne = *ne_dev;
  const double lpw = scal[PG_S_LPW];
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < ne; e += gridDim.x * blockDim.x) {
    const b2s_pose_graph_edge& ed = E[e];
    const double* Ts = P + 16 * (size_t)ed.source;
    double Xi[16], Tti[16], Q[16], M[16], z[6], eI[6];
    pg_inv_rigid(ed.T, Xi);
    pg_inv_rigid(P + 16 * (size_t)ed.target, Tti);
    pg_mul4(Xi, Tti, Q);
    pg_mul4(Q, Ts, M);
    pg_lin(M, z);
    double q = 0.0;
    for (int k = 0; k < 6; k++) {
      double s = 0.0;
      for (int m = 0; m < 6; m++) s += z[m] * ed.information[6 * m + k];
      eI[k] = s;
    }
    for (int k = 0; k < 6; k++) q += eI[k] * z[k];
    const double c_in = conf[e];
    if (!linearize) {
      const double sc = sqrt(c_in) - 1.0;
      term[e] = c_in * q + lpw * (sc * sc);
      continue;
    }
    double c = c_in;
    if (ed.uncertain) {
      const double t = lpw / (lpw + q);
      c = t * t;
      conf[e] = c;
    }
    double Js[36];   // Js[6 * m + i]: component m of lin(Q G_i Ts)
    for (int i = 0; i < 6; i++) {
      double GT[16];
      for (int k = 0; k < 16; k++) GT[k] = 0.0;
      for (int j = 0; j < 4; j++) {
        const double r0 = Ts[j], r1 = Ts[4 + j], r2 = Ts[8 + j], r3 = Ts[12 + j];
        switch (i) {   // rows of G_i Ts, G_i the generators of [O3D]'s jacobian_operator
          case 0: GT[4 + j] = -r2; GT[8 + j] = r1; break;
          case 1: GT[j] = r2; GT[8 + j] = -r0; break;
          case 2: GT[j] = -r1; GT[4 + j] = r0; break;
          default: GT[4 * (i - 3) + j] = r3; break;
        }
      }
      double QG[16], v[6];
      pg_mul4(Q, GT, QG);
      pg_lin(QG, v);
      for (int m = 0; m < 6; m++) Js[6 * m + i] = v[m];
    }
    double JI[36];   // Js' Info
    for (int a = 0; a < 6; a++)
      for (int k = 0; k < 6; k++) {
        double s = 0.0;
        for (int m = 0; m < 6; m++) s += Js[6 * m + a] * ed.information[6 * m + k];
        JI[6 * a + k] = s;
      }
    double* H = hss + 36 * (size_t)e;
    for (int a = 0; a < 6; a++)
      for (int col = 0; col < 6; col++) {
        double s = 0.0;
        for (int k = 0; k < 6; k++) s += JI[6 * a + k] * Js[6 * k + col];
        H[6 * a + col] = c * s;
      }
    for (int col = 0; col < 6; col++) {
      double s = 0.0;
      for (int k = 0; k < 6; k++) s += eI[k] * Js[6 * k + col];
      gv[6 * (size_t)e + col] = c * s;
    }
  }
}

// K-pg-assemble: one CTA per nonzero node block of the lower triangle; thread t < 36 sums entry t of the block over the block's
// contributions in edge order, threads 36..41 the block's right-hand side (diagonal blocks)
__global__ void pg_assemble_kernel(const PgTask* __restrict__ tasks, const int32_t* __restrict__ contrib, const double* __restrict__ hss,
                                   const double* __restrict__ gv, double* __restrict__ A, double* __restrict__ b, int M) {
  pdl_wait();
  const PgTask t = tasks[blockIdx.x];
  const int tid = threadIdx.x;
  if (tid < 36) {
    double s = 0.0;
    for (int k = t.begin; k < t.end; k++) {
      const int v = contrib[k];
      const double x = hss[36 * (size_t)(v >> 2) + tid];
      s = ((v & 3) == PG_C_CROSS) ? s - x : s + x;
    }
    A[(size_t)(6 * t.row + tid / 6) * M + 6 * t.col + tid % 6] = s;
  } else if (tid < 42 && t.row == t.col) {
    double s = 0.0;
    for (int k = t.begin; k < t.end; k++) {
      const int v = contrib[k];
      const double x = gv[6 * (size_t)(v >> 2) + tid - 36];
      if ((v & 3) == PG_C_SOURCE) s -= x;
      else if ((v & 3) == PG_C_TARGET) s += x;
    }
    b[6 * t.row + tid - 36] = s;
  }
}

// fixed-order block sum (per-thread partials, warp tree, warps in rank order); the total is valid in thread 0
__device__ double pg_block_sum(double v, double* sh) {
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
  if (threadIdx.x == 0)
    for (int w = 0; w < PG_RED / 32; w++) s += sh[w];
  __syncthreads();
  return s;
}

// K-pg-reduce-try: residual of the trial, |delta|^2, delta . (lambda delta + b)
__global__ void __launch_bounds__(PG_RED) pg_reduce_try_kernel(const double* __restrict__ term, const int32_t* __restrict__ ne_dev,
                                                               const double* __restrict__ delta, const double* __restrict__ b,
                                                               const double* __restrict__ scal, int n6, double* __restrict__ rec) {
  pdl_wait();
  __shared__ double sh[PG_RED / 32];
  const int ne = *ne_dev;
  const double lam = scal[PG_S_LAMBDA];
  double r = 0.0, dd = 0.0, dl = 0.0;
  for (int e = threadIdx.x; e < ne; e += PG_RED) r += term[e];
  for (int i = threadIdx.x; i < n6; i += PG_RED) {
    const double d = delta[i];
    dd += d * d;
    dl += d * (lam * d + b[i]);
  }
  r = pg_block_sum(r, sh); dd = pg_block_sum(dd, sh); dl = pg_block_sum(dl, sh);
  if (threadIdx.x == 0) { rec[PG_R_RES] = r; rec[PG_R_DD] = dd; rec[PG_R_DLB] = dl; }
}

// K-pg-reduce-lin: max b (signed), max diag H, |x|^2 with x the TransformMatrix4dToVector6d of every pose
__global__ void __launch_bounds__(PG_RED) pg_reduce_lin_kernel(const double* __restrict__ A, const double* __restrict__ b,
                                                               const double* __restrict__ P, int N, int M, double* __restrict__ rec) {
  pdl_wait();
  __shared__ double sh[PG_RED / 32];
  const int n6 = 6 * N;
  double mb = -INFINITY, md = -INFINITY, xx = 0.0;
  for (int i = threadIdx.x; i < n6; i += PG_RED) { mb = fmax(mb, b[i]); md = fmax(md, A[(size_t)i * M + i]); }
  for (int i = threadIdx.x; i < N; i += PG_RED) {
    const double* T = P + 16 * (size_t)i;
    const double sy = sqrt(T[0] * T[0] + T[4] * T[4]);
    double a0, a1, a2;
    if (!(sy < 1e-6)) { a0 = atan2(T[9], T[10]); a1 = atan2(-T[8], sy); a2 = atan2(T[4], T[0]); }
    else { a0 = atan2(-T[6], T[5]); a1 = atan2(-T[8], sy); a2 = 0.0; }
    xx += a0 * a0 + a1 * a1 + a2 * a2 + T[3] * T[3] + T[7] * T[7] + T[11] * T[11];
  }
  mb = warp_max(mb); md = warp_max(md);
  __shared__ double smb[PG_RED / 32], smd[PG_RED / 32];
  if ((threadIdx.x & 31) == 0) { smb[threadIdx.x >> 5] = mb; smd[threadIdx.x >> 5] = md; }
  xx = pg_block_sum(xx, sh);   // its barriers also publish smb / smd
  if (threadIdx.x == 0) {
    for (int w = 0; w < PG_RED / 32; w++) { mb = fmax(mb, smb[w]); md = fmax(md, smd[w]); }
    rec[PG_R_MAXB] = mb; rec[PG_R_MAXDIAG] = md; rec[PG_R_XX] = xx;
  }
}

// K-pg-form: the lower triangle of F = H + lambda I on the first n6 rows / columns, the identity on the padding; rhs = b (0 padded)
__global__ void pg_form_kernel(const double* __restrict__ A, const double* __restrict__ b, const double* __restrict__ scal, int n6, int M,
                               double* __restrict__ F, double* __restrict__ rhs) {
  pdl_wait();
  const double lam = scal[PG_S_LAMBDA];
  const size_t total = (size_t)M * M;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int r = (int)(idx / M), c = (int)(idx % M);
    if (c > r) continue;
    double v;
    if (r < n6) v = (r == c) ? A[idx] + lam : A[idx];
    else v = (r == c) ? 1.0 : 0.0;
    F[idx] = v;
    if (c == 0) rhs[r] = r < n6 ? b[r] : 0.0;
  }
}

// K-pg-diag: LDL' of the diagonal tile (K, K) in shared memory, right-looking column by column (A_ik -= l_i col_k); the strict
// lower part becomes L, the pivots go to D
__global__ void __launch_bounds__(256) pg_diag_kernel(double* __restrict__ F, double* __restrict__ D, int K, int M) {
  pdl_wait();
  __shared__ double S[PG_NB][PG_NB + 1];
  __shared__ double col[PG_NB], lv[PG_NB];
  const int tid = threadIdx.x;
  double* T = F + (size_t)(PG_NB * K) * M + PG_NB * K;
  for (int idx = tid; idx < PG_NB * PG_NB; idx += 256) {
    const int r = idx / PG_NB, c = idx % PG_NB;
    if (c <= r) S[r][c] = T[(size_t)r * M + c];
  }
  __syncthreads();
  for (int j = 0; j < PG_NB; j++) {
    const double d = S[j][j];
    if (tid > j && tid < PG_NB) {
      const double v = S[tid][j];
      col[tid] = v;
      lv[tid] = fabs(d) > PG_TINY ? v / d : 0.0;
    }
    __syncthreads();
    const int m = PG_NB - 1 - j;
    for (int idx = tid; idx < m * m; idx += 256) {
      const int i = j + 1 + idx / m, k = j + 1 + idx % m;
      if (k <= i) S[i][k] -= lv[i] * col[k];
    }
    if (tid > j && tid < PG_NB) S[tid][j] = lv[tid];
    __syncthreads();
  }
  for (int idx = tid; idx < PG_NB * PG_NB; idx += 256) {
    const int r = idx / PG_NB, c = idx % PG_NB;
    if (c <= r) T[(size_t)r * M + c] = S[r][c];
  }
  if (tid < PG_NB) D[PG_NB * K + tid] = S[tid][tid];
}

// K-pg-panel: tile row I = K + 1 + blockIdx.x of the panel.  W = A_IK L_KK^-T (forward substitution, column by column),
// L_IK = W D_K^-1 (0 where the pivot is zeroed)
constexpr size_t PG_PANEL_SMEM = 2 * sizeof(double) * PG_NB * (PG_NB + 1);
__global__ void __launch_bounds__(256) pg_panel_kernel(double* __restrict__ F, const double* __restrict__ D, double* __restrict__ W, int K, int M) {
  pdl_wait();
  extern __shared__ double pg_smem[];
  double (*Lk)[PG_NB + 1] = reinterpret_cast<double (*)[PG_NB + 1]>(pg_smem);
  double (*S)[PG_NB + 1] = reinterpret_cast<double (*)[PG_NB + 1]>(pg_smem + PG_NB * (PG_NB + 1));
  const int tid = threadIdx.x, I = K + 1 + blockIdx.x;
  const double* Tk = F + (size_t)(PG_NB * K) * M + PG_NB * K;
  double* Ti = F + (size_t)(PG_NB * I) * M + PG_NB * K;
  for (int idx = tid; idx < PG_NB * PG_NB; idx += 256) {
    const int r = idx / PG_NB, c = idx % PG_NB;
    Lk[r][c] = c < r ? Tk[(size_t)r * M + c] : 0.0;
    S[r][c] = Ti[(size_t)r * M + c];
  }
  __syncthreads();
  for (int j = 0; j < PG_NB - 1; j++) {
    for (int idx = tid; idx < PG_NB * PG_NB; idx += 256) {
      const int r = idx / PG_NB, m = idx % PG_NB;
      if (m > j) S[r][m] -= S[r][j] * Lk[m][j];
    }
    __syncthreads();
  }
  for (int idx = tid; idx < PG_NB * PG_NB; idx += 256) {
    const int r = idx / PG_NB, c = idx % PG_NB;
    const double w = S[r][c], d = D[PG_NB * K + c];
    W[(size_t)(PG_NB * I + r) * PG_NB + c] = w;
    Ti[(size_t)r * M + c] = fabs(d) > PG_TINY ? w / d : 0.0;
  }
}

__device__ __forceinline__ void pg_dmma(double (&c)[2], double a, double b) {   // c += A(8x4) B(4x8), one fragment each
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n" : "+d"(c[0]), "+d"(c[1]) : "d"(a), "d"(b));
}

// K-pg-trailing: tile (I, J), K < J <= I, of the trailing matrix: A_IJ -= W_I L_JK'.  4 warps, each a 32 x 32 quarter as 4 x 4
// m8n8k4 fragments; k in chunks of 16 through shared memory
__global__ void __launch_bounds__(128) pg_trailing_kernel(double* __restrict__ F, const double* __restrict__ W, int K, int M) {
  pdl_wait();
  __shared__ double Ws[PG_NB][17], Ls[PG_NB][17];
  const int t = blockIdx.x;
  int i = (int)((sqrt(8.0 * t + 1.0) - 1.0) * 0.5);
  while ((i + 1) * (i + 2) / 2 <= t) i++;
  while (i * (i + 1) / 2 > t) i--;
  const int I = K + 1 + i, J = K + 1 + (t - i * (i + 1) / 2);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, tg = lane & 3;
  const int wm = warp >> 1, wn = warp & 1;
  double acc[4][4][2];
#pragma unroll
  for (int a = 0; a < 4; a++)
#pragma unroll
    for (int c = 0; c < 4; c++) { acc[a][c][0] = 0.0; acc[a][c][1] = 0.0; }
  const double* Wt = W + (size_t)(PG_NB * I) * PG_NB;
  const double* Lt = F + (size_t)(PG_NB * J) * M + PG_NB * K;
  for (int kc = 0; kc < PG_NB; kc += 16) {
    for (int idx = tid; idx < PG_NB * 16; idx += 128) {
      const int r = idx >> 4, c = idx & 15;
      Ws[r][c] = Wt[(size_t)r * PG_NB + kc + c];
      Ls[r][c] = Lt[(size_t)r * M + kc + c];
    }
    __syncthreads();
#pragma unroll
    for (int k0 = 0; k0 < 16; k0 += 4) {
      double a[4], bb[4];
#pragma unroll
      for (int m = 0; m < 4; m++) a[m] = Ws[wm * 32 + m * 8 + g][k0 + tg];
#pragma unroll
      for (int n = 0; n < 4; n++) bb[n] = Ls[wn * 32 + n * 8 + g][k0 + tg];   // B[k][n] = L[n][k]
#pragma unroll
      for (int m = 0; m < 4; m++)
#pragma unroll
        for (int n = 0; n < 4; n++) pg_dmma(acc[m][n], a[m], bb[n]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int m = 0; m < 4; m++)
#pragma unroll
    for (int n = 0; n < 4; n++) {
      double* o = F + (size_t)(PG_NB * I + wm * 32 + m * 8 + g) * M + PG_NB * J + wn * 32 + n * 8 + 2 * tg;
      o[0] -= acc[m][n][0];
      o[1] -= acc[m][n][1];
    }
}

// the unit lower diagonal tile (K, K) of the factor, strict part, into shared memory
__device__ void pg_load_lkk(const double* F, int K, int M, double (*Lk)[PG_NB + 1]) {
  const double* T = F + (size_t)(PG_NB * K) * M + PG_NB * K;
  for (int idx = threadIdx.x; idx < PG_NB * PG_NB; idx += blockDim.x) {
    const int r = idx / PG_NB, c = idx % PG_NB;
    Lk[r][c] = c < r ? T[(size_t)r * M + c] : 0.0;
  }
}

// K-pg-fwd, tile K of L y = rhs: every CTA solves the diagonal tile; CTA 0 writes z_K = D^-1 y_K, CTA c > 0 updates
// rhs_{K+c} -= L_{K+c,K} y_K
__global__ void __launch_bounds__(256) pg_fwd_kernel(const double* __restrict__ F, const double* __restrict__ D, double* __restrict__ rhs,
                                                     double* __restrict__ z, int K, int M) {
  pdl_wait();
  __shared__ double Lk[PG_NB][PG_NB + 1];
  __shared__ double y[PG_NB], part[4][PG_NB];
  const int tid = threadIdx.x;
  pg_load_lkk(F, K, M, Lk);
  if (tid < PG_NB) y[tid] = rhs[PG_NB * K + tid];
  __syncthreads();
  for (int j = 0; j < PG_NB - 1; j++) {
    if (tid > j && tid < PG_NB) y[tid] -= y[j] * Lk[tid][j];
    __syncthreads();
  }
  if (blockIdx.x == 0) {
    if (tid < PG_NB) {
      const double d = D[PG_NB * K + tid];
      z[PG_NB * K + tid] = fabs(d) > PG_TINY ? y[tid] / d : 0.0;
    }
    return;
  }
  const int I = K + blockIdx.x, r = tid >> 2, q = tid & 3;
  const double* row = F + (size_t)(PG_NB * I + r) * M + PG_NB * K + 16 * q;
  double s = 0.0;
  for (int j = 0; j < 16; j++) s += row[j] * y[16 * q + j];
  part[q][r] = s;
  __syncthreads();
  if (tid < PG_NB) rhs[PG_NB * I + tid] -= ((part[0][tid] + part[1][tid]) + part[2][tid]) + part[3][tid];
}

// K-pg-bwd, tile K of L' delta = z: every CTA solves the diagonal tile; CTA 0 writes delta_K, CTA c > 0 updates
// z_{c-1} -= L_{K,c-1}' delta_K
__global__ void __launch_bounds__(256) pg_bwd_kernel(const double* __restrict__ F, double* __restrict__ z, double* __restrict__ delta, int K, int M) {
  pdl_wait();
  __shared__ double Lk[PG_NB][PG_NB + 1];
  __shared__ double x[PG_NB], part[4][PG_NB];
  const int tid = threadIdx.x;
  pg_load_lkk(F, K, M, Lk);
  if (tid < PG_NB) x[tid] = z[PG_NB * K + tid];
  __syncthreads();
  for (int j = PG_NB - 1; j > 0; j--) {
    if (tid < j) x[tid] -= Lk[j][tid] * x[j];
    __syncthreads();
  }
  if (blockIdx.x == 0) {
    if (tid < PG_NB) delta[PG_NB * K + tid] = x[tid];
    return;
  }
  const int J = blockIdx.x - 1, c = tid & (PG_NB - 1), q = tid >> 6;
  double s = 0.0;
  for (int i = 16 * q; i < 16 * q + 16; i++) s += F[(size_t)(PG_NB * K + i) * M + PG_NB * J + c] * x[i];
  part[q][c] = s;
  __syncthreads();
  if (tid < PG_NB) z[PG_NB * J + tid] -= ((part[0][tid] + part[1][tid]) + part[2][tid]) + part[3][tid];
}

// K-pg-update: trial pose i = V2M(delta_i) T_i (UpdatePoseGraph)
__global__ void pg_update_kernel(const double* __restrict__ P, const double* __restrict__ delta, double* __restrict__ Pt, int N) {
  pdl_wait();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  double x[6], V[16];
  for (int k = 0; k < 6; k++) x[k] = delta[6 * i + k];
  vec6_to_mat4_dev(x, V);
  pg_mul4(V, P + 16 * (size_t)i, Pt + 16 * (size_t)i);
}

// ---------------------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------------------
namespace {

struct PgLayout {   // pointers into the handle's pose-graph buffers
  int N, n6, M, nt, ecap;
  double *A, *F, *W;
  double *b, *rhs, *z, *delta, *D, *rec, *scal;
  double *P, *Pt;
  b2s_pose_graph_edge* E;
  double *conf, *hss, *gv, *term;
  int32_t* ne;
  PgTask* tasks;
  int32_t* contrib;
};

// BFS from node 0 (ValidatePoseGraphConnectivity); certain_only: uncertain edges are ignored
bool pg_connected(int N, const std::vector<b2s_pose_graph_edge>& E, bool certain_only) {
  std::vector<std::vector<int>> adj((size_t)N);
  for (const b2s_pose_graph_edge& e : E) {
    if (certain_only && e.uncertain) continue;
    adj[e.source].push_back(e.target);
    adj[e.target].push_back(e.source);
  }
  std::vector<char> seen((size_t)N, 0);
  std::vector<int> q{0};
  seen[0] = 1;
  for (size_t k = 0; k < q.size(); k++)
    for (int v : adj[q[k]])
      if (!seen[v]) { seen[v] = 1; q.push_back(v); }
  return q.size() == (size_t)N;
}

int32_t pg_prepare(b2s_handle* h, int N, int ne, int ntasks, int ncontrib, PgLayout* L) {
  L->N = N; L->n6 = 6 * N; L->nt = (6 * N + PG_NB - 1) / PG_NB; L->M = L->nt * PG_NB;
  const size_t MM = (size_t)L->M * L->M;
  if (h->pg_edge_cap < ne) { int c = 64; while (c < ne) c *= 2; h->pg_edge_cap = c; }
  L->ecap = h->pg_edge_cap;
  B2S_TRY(h->pg_A.ensure(MM * 8, h->stream));
  B2S_TRY(h->pg_F.ensure(MM * 8, h->stream));
  B2S_TRY(h->pg_W.ensure((size_t)L->M * PG_NB * 8, h->stream));
  B2S_TRY(h->pg_vec.ensure((5 * (size_t)L->M + PG_R_WORDS + 8) * 8, h->stream));
  B2S_TRY(h->pg_nodes.ensure(2 * 16 * 8 * (size_t)N, h->stream));
  const size_t ec = (size_t)L->ecap;
  B2S_TRY(carve(h->pg_edges, h->stream, [&](Layout& E) {
    L->E = E.take<b2s_pose_graph_edge>(ec);
    L->conf = E.take<double>(ec); L->hss = E.take<double>(ec * 36); L->gv = E.take<double>(ec * 6); L->term = E.take<double>(ec);
    L->ne = E.take<int32_t>(1); L->tasks = E.take<PgTask>(ntasks); L->contrib = E.take<int32_t>((size_t)ncontrib + 1);
  }));
  // K-pg-panel holds two 64 x 65 tiles, above the default 48 KB of shared memory; the attribute is per device, set on every pass
  // (a host call, cheap next to a pass) rather than cached behind an unsynchronised flag
  B2S_CUDA(cudaFuncSetAttribute(pg_panel_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)PG_PANEL_SMEM));
  L->A = h->pg_A.as<double>(); L->F = h->pg_F.as<double>(); L->W = h->pg_W.as<double>();
  double* v = h->pg_vec.as<double>();
  L->b = v; L->rhs = v + L->M; L->z = v + 2 * L->M; L->delta = v + 3 * L->M; L->D = v + 4 * L->M; L->rec = v + 5 * L->M;
  L->scal = L->rec + PG_R_WORDS;
  L->P = h->pg_nodes.as<double>(); L->Pt = L->P + 16 * (size_t)N;
  return B2S_OK;
}

int edge_grid(int ecap) { return (ecap + 127) / 128; }

struct PgCtx { PgLayout L; b2s_handle* h; };

// H + lambda I -> blocked LDL' -> delta: K-pg-form, per tile column K-pg-diag, K-pg-panel and K-pg-trailing, then K-pg-fwd and
// K-pg-bwd per tile.  Returns the number of launches
int64_t pg_factor_solve(b2s_handle* h, const PgLayout& L) {
  const int M = L.M, nt = L.nt;
  int64_t n = 0;
  launch_pdl(pg_form_kernel, grid_for((size_t)M * M, 256, 4 * device_sms()), 256, 0, h->stream, (const double*)L.A, (const double*)L.b,
             (const double*)L.scal, L.n6, M, L.F, L.rhs);
  n++;
  for (int K = 0; K < nt; K++) {
    launch_pdl(pg_diag_kernel, 1, 256, 0, h->stream, L.F, L.D, K, M);
    n++;
    const int m = nt - 1 - K;
    if (m == 0) continue;
    launch_pdl(pg_panel_kernel, m, 256, PG_PANEL_SMEM, h->stream, L.F, (const double*)L.D, L.W, K, M);
    launch_pdl(pg_trailing_kernel, m * (m + 1) / 2, 128, 0, h->stream, L.F, (const double*)L.W, K, M);
    n += 2;
  }
  for (int K = 0; K < nt; K++) { launch_pdl(pg_fwd_kernel, nt - K, 256, 0, h->stream, (const double*)L.F, (const double*)L.D, L.rhs, L.z, K, M); n++; }
  for (int K = nt - 1; K >= 0; K--) { launch_pdl(pg_bwd_kernel, K + 1, 256, 0, h->stream, (const double*)L.F, L.z, L.delta, K, M); n++; }
  return n;
}

// one LM try: H + lambda I -> LDL' -> delta -> trial poses -> trial residual; the record lands in L->rec
int32_t pg_try_chain(void* ctx) {
  const PgLayout& L = static_cast<const PgCtx*>(ctx)->L;
  b2s_handle* h = static_cast<const PgCtx*>(ctx)->h;
  int64_t n = pg_factor_solve(h, L);
  launch_pdl(pg_update_kernel, (L.N + 127) / 128, 128, 0, h->stream, (const double*)L.P, (const double*)L.delta, L.Pt, L.N);
  launch_pdl(pg_edge_kernel, edge_grid(L.ecap), 128, 0, h->stream, (const b2s_pose_graph_edge*)L.E, (const int32_t*)L.ne, (const double*)L.Pt,
             L.conf, (const double*)L.scal, 0, L.term, L.hss, L.gv);
  launch_pdl(pg_reduce_try_kernel, 1, PG_RED, 0, h->stream, (const double*)L.term, (const int32_t*)L.ne, (const double*)L.delta,
             (const double*)L.b, (const double*)L.scal, L.n6, L.rec);
  n += 3;
  h->launches += n;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

// residual terms of the poses P with the current confidences, reduced into rec[PG_R_RES]
int32_t pg_eval(b2s_handle* h, const PgLayout& L, const double* P) {
  launch_pdl(pg_edge_kernel, edge_grid(L.ecap), 128, 0, h->stream, (const b2s_pose_graph_edge*)L.E, (const int32_t*)L.ne, P, L.conf,
             (const double*)L.scal, 0, L.term, L.hss, L.gv);
  launch_pdl(pg_reduce_try_kernel, 1, PG_RED, 0, h->stream, (const double*)L.term, (const int32_t*)L.ne, (const double*)L.delta,
             (const double*)L.b, (const double*)L.scal, L.n6, L.rec);
  h->launches += 2;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

// UpdateConfidence + ComputeLinearSystem at the current poses, then the record of max b, max diag H and |x|^2
int32_t pg_linearize(b2s_handle* h, const PgLayout& L, int ntasks) {
  launch_pdl(pg_edge_kernel, edge_grid(L.ecap), 128, 0, h->stream, (const b2s_pose_graph_edge*)L.E, (const int32_t*)L.ne, (const double*)L.P,
             L.conf, (const double*)L.scal, 1, L.term, L.hss, L.gv);
  launch_pdl(pg_assemble_kernel, ntasks, 64, 0, h->stream, (const PgTask*)L.tasks, (const int32_t*)L.contrib, (const double*)L.hss,
             (const double*)L.gv, L.A, L.b, L.M);
  launch_pdl(pg_reduce_lin_kernel, 1, PG_RED, 0, h->stream, (const double*)L.A, (const double*)L.b, (const double*)L.P, L.N, L.M, L.rec);
  h->launches += 3;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

// the assembly lists: diagonal block of every node, then the off-diagonal blocks in (row, col) order; contributions in edge order
void pg_assembly_lists(int N, const std::vector<b2s_pose_graph_edge>& E, std::vector<PgTask>& tasks, std::vector<int32_t>& contrib) {
  const int ne = (int)E.size();
  std::vector<std::vector<int32_t>> diag((size_t)N);
  std::vector<std::pair<std::pair<int, int>, int32_t>> off;
  for (int e = 0; e < ne; e++) {
    const int s = E[e].source, t = E[e].target;
    if (s == t) {   // the four blocks of [O3D]'s loop all land on the diagonal: ss, st, ts, tt
      for (int c : {PG_C_SOURCE, PG_C_CROSS, PG_C_CROSS, PG_C_TARGET}) diag[s].push_back(4 * e + c);
      continue;
    }
    diag[s].push_back(4 * e + PG_C_SOURCE);
    diag[t].push_back(4 * e + PG_C_TARGET);
    off.push_back({{std::max(s, t), std::min(s, t)}, 4 * e + PG_C_CROSS});
  }
  std::stable_sort(off.begin(), off.end(), [](const auto& a, const auto& b) { return a.first < b.first; });
  for (int i = 0; i < N; i++) {
    tasks.push_back({i, i, (int32_t)contrib.size(), 0});
    contrib.insert(contrib.end(), diag[i].begin(), diag[i].end());
    tasks.back().end = (int32_t)contrib.size();
  }
  for (size_t k = 0; k < off.size(); k++) {
    if (k == 0 || off[k].first != off[k - 1].first) tasks.push_back({off[k].first.first, off[k].first.second, (int32_t)contrib.size(), 0});
    contrib.push_back(off[k].second);
    tasks.back().end = (int32_t)contrib.size();
  }
}

// a pass's device state: the buffers (pg_prepare), the edges, their confidences, the assembly lists (built into tasks / contrib),
// lambda = 0 and the line-process weight, a zeroed H and delta.  The node poses are the caller's
int32_t pg_load(b2s_handle* h, int N, const std::vector<b2s_pose_graph_edge>& E, const std::vector<double>& conf, const b2s_global_optimization_params& p,
                std::vector<PgTask>& tasks, std::vector<int32_t>& contrib, PgLayout* Lo) {
  const int ne = (int)E.size();
  pg_assembly_lists(N, E, tasks, contrib);
  B2S_TRY(pg_prepare(h, N, ne, (int)tasks.size(), (int)contrib.size(), Lo));
  const PgLayout& L = *Lo;
  double lpw = 0.0;   // ComputeLineProcessWeight
  for (const b2s_pose_graph_edge& e : E) lpw += e.information[35];
  if (ne > 0) lpw /= (double)ne;
  lpw = p.preference_loop_closure * (p.max_correspondence_distance * p.max_correspondence_distance) * lpw;
  const int32_t ne32 = ne;
  if (ne > 0) {
    B2S_CUDA(cudaMemcpyAsync(L.E, E.data(), sizeof(b2s_pose_graph_edge) * (size_t)ne, cudaMemcpyHostToDevice, h->stream));
    B2S_CUDA(cudaMemcpyAsync(L.conf, conf.data(), 8 * (size_t)ne, cudaMemcpyHostToDevice, h->stream));
  }
  B2S_CUDA(cudaMemcpyAsync(L.ne, &ne32, 4, cudaMemcpyHostToDevice, h->stream));
  B2S_CUDA(cudaMemcpyAsync(L.tasks, tasks.data(), sizeof(PgTask) * tasks.size(), cudaMemcpyHostToDevice, h->stream));
  if (!contrib.empty()) B2S_CUDA(cudaMemcpyAsync(L.contrib, contrib.data(), 4 * contrib.size(), cudaMemcpyHostToDevice, h->stream));
  const double scal[2] = {0.0, lpw};
  B2S_CUDA(cudaMemcpyAsync(L.scal, scal, sizeof(scal), cudaMemcpyHostToDevice, h->stream));
  B2S_CUDA(cudaMemsetAsync(L.A, 0, (size_t)L.M * L.M * 8, h->stream));
  B2S_CUDA(cudaMemsetAsync(L.delta, 0, (size_t)L.M * 8, h->stream));   // read (unused) by the first residual's reduction
  return B2S_OK;
}

// GlobalOptimizationLevenbergMarquardt::OptimizePoseGraph over the edges E (the node poses are resident in L->P).  conf: the
// edges' confidences, in and out
int32_t pg_pass(b2s_handle* h, int N, const std::vector<b2s_pose_graph_edge>& E, std::vector<double>& conf, const b2s_global_optimization_params& p,
                b2s_global_optimization_stats* st) {
  const int ne = (int)E.size();
  std::vector<PgTask> tasks;
  std::vector<int32_t> contrib;
  PgLayout L;
  B2S_TRY(pg_load(h, N, E, conf, p, tasks, contrib, &L));

  double rec[PG_R_WORDS];
  auto fetch = [&]() { return read_back(h, {{rec, L.rec, sizeof(rec)}}); };
  // initial residual (the confidences as they come in), then UpdateConfidence and the linear system
  B2S_TRY(pg_eval(h, L, L.P));
  B2S_TRY(fetch());
  double cur = rec[PG_R_RES], nres = cur;
  B2S_TRY(pg_linearize(h, L, (int)tasks.size()));
  B2S_TRY(fetch());
  double maxb = rec[PG_R_MAXB], xx = rec[PG_R_XX];
  double lambda = 1e-5 * rec[PG_R_MAXDIAG], nu = 2.0, rho = 0.0;
  st->valid = 1; st->n_edges = ne; st->initial_residual = cur;
  bool stop = false;
  int reason = B2S_LM_STOP_NONE;
  auto stop_on = [&](bool cond, int why) { if (!stop && cond) { stop = true; reason = why; } };
  stop_on(maxb < p.min_right_term, B2S_LM_STOP_RIGHT_TERM);
  PgCtx ctx{L, h};
  const unsigned long long key = ((unsigned long long)L.M << 40) ^ ((unsigned long long)N << 20) ^ (unsigned long long)L.ecap;
  for (int iter = 0; !stop && iter < p.max_iteration; iter++) {
    st->outer_iterations++;
    int lm_count = 0;
    do {
      B2S_CUDA(cudaMemcpyAsync(L.scal + PG_S_LAMBDA, &lambda, 8, cudaMemcpyHostToDevice, h->stream));
      B2S_TRY(graph_step(h, &h->pg_graph, key, pg_try_chain, &ctx));
      B2S_TRY(fetch());
      st->lm_tries++;
      stop_on(sqrt(rec[PG_R_DD]) < p.min_relative_increment * (sqrt(xx) + p.min_relative_increment), B2S_LM_STOP_RELATIVE_INCREMENT);
      if (!stop) {
        nres = rec[PG_R_RES];
        rho = (cur - nres) / (rec[PG_R_DLB] + 1e-3);
        if (rho > 0) {
          stop_on(cur - nres < p.min_relative_residual_increment * cur, B2S_LM_STOP_RELATIVE_RESIDUAL_INCREMENT);
          const double alpha = std::min(1.0 - std::pow(2.0 * rho - 1.0, 3.0), p.upper_scale_factor);
          lambda *= std::max(p.lower_scale_factor, alpha);
          nu = 2.0;
          cur = nres;
          st->accepted_steps++;
          B2S_CUDA(cudaMemcpyAsync(L.P, L.Pt, 16 * 8 * (size_t)N, cudaMemcpyDeviceToDevice, h->stream));
          B2S_TRY(pg_linearize(h, L, (int)tasks.size()));
          B2S_TRY(fetch());
          maxb = rec[PG_R_MAXB]; xx = rec[PG_R_XX];
          stop_on(maxb < p.min_right_term, B2S_LM_STOP_RIGHT_TERM);
          if (stop) break;
        } else {
          lambda *= nu;
          nu *= 2.0;
        }
      }
      lm_count++;
      stop_on(lm_count >= p.max_iteration_lm, B2S_LM_STOP_MAX_ITERATION_LM);
    } while (!(rho > 0 || stop));
    stop_on(nres < p.min_residual, B2S_LM_STOP_RESIDUAL);
  }
  if (!stop) reason = B2S_LM_STOP_MAX_ITERATION;
  st->stop_reason = reason; st->final_residual = cur; st->final_lambda = lambda;
  if (ne > 0) B2S_CUDA(cudaMemcpyAsync(conf.data(), L.conf, 8 * (size_t)ne, cudaMemcpyDeviceToHost, h->stream));
  return check_status(h);
}

void host_inv_rigid(const double* T, double* R) {
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) R[4 * i + j] = T[4 * j + i];
  for (int i = 0; i < 3; i++) R[4 * i + 3] = -((R[4 * i] * T[3] + R[4 * i + 1] * T[7]) + R[4 * i + 2] * T[11]);
  R[12] = 0.0; R[13] = 0.0; R[14] = 0.0; R[15] = 1.0;
}

void host_mul4(const double* A, const double* B, double* C) {
  for (int i = 0; i < 4; i++)
    for (int j = 0; j < 4; j++) {
      double s = 0.0;
      for (int k = 0; k < 4; k++) s += A[4 * i + k] * B[4 * k + j];
      C[4 * i + j] = s;
    }
}

}  // namespace

int32_t op_global_optimization(b2s_handle* h, int N, double* poses, int ne, const b2s_pose_graph_edge* edges,
                               const b2s_global_optimization_params& p, int32_t* kept_out, double* conf_out, b2s_global_optimization_stats* stats) {
  b2s_global_optimization_stats st[2];
  memset(st, 0, sizeof(st));
  std::vector<b2s_pose_graph_edge> E(edges, edges + ne);
  std::vector<double> conf((size_t)ne, 1.0);   // PoseGraphEdge's confidence_ starts at 1
  std::vector<int32_t> kept((size_t)ne, 1);
  auto finish = [&]() {
    if (stats) memcpy(stats, st, sizeof(st));
    if (kept_out) memcpy(kept_out, kept.data(), 4 * (size_t)ne);
    if (conf_out) memcpy(conf_out, conf.data(), 8 * (size_t)ne);
    return B2S_OK;
  };
  if (!pg_connected(N, E, false) || !pg_connected(N, E, true)) return finish();   // ValidatePoseGraph: poses unchanged
  if (ne == 0) { st[0].valid = st[1].valid = 1; return finish(); }
  B2S_TRY(h->pg_nodes.ensure(2 * 16 * 8 * (size_t)N, h->stream));
  B2S_CUDA(cudaMemcpyAsync(h->pg_nodes.p, poses, 16 * 8 * (size_t)N, cudaMemcpyHostToDevice, h->stream));
  B2S_TRY(pg_pass(h, N, E, conf, p, &st[0]));
  // CreatePoseGraphWithoutInvalidEdges: certain edges, and uncertain ones with conf > edge_prune_threshold (the confidence travels)
  std::vector<b2s_pose_graph_edge> E2;
  std::vector<double> conf2;
  std::vector<int> idx2;
  for (int e = 0; e < ne; e++) {
    kept[e] = (!E[e].uncertain || conf[e] > p.edge_prune_threshold) ? 1 : 0;
    if (kept[e]) { E2.push_back(E[e]); conf2.push_back(conf[e]); idx2.push_back(e); }
  }
  B2S_TRY(pg_pass(h, N, E2, conf2, p, &st[1]));
  for (size_t k = 0; k < idx2.size(); k++) conf[idx2[k]] = conf2[k];
  std::vector<double> out((size_t)N * 16);
  B2S_CUDA(cudaMemcpyAsync(out.data(), h->pg_nodes.p, 16 * 8 * (size_t)N, cudaMemcpyDeviceToHost, h->stream));
  B2S_TRY(check_status(h));
  if (p.reference_node >= 0 && p.reference_node < N) {   // CompensateReferencePoseGraphNode
    double inv[16], C[16], T[16];
    host_inv_rigid(&out[16 * (size_t)p.reference_node], inv);
    host_mul4(poses + 16 * (size_t)p.reference_node, inv, C);
    for (int i = 0; i < N; i++) {
      host_mul4(C, &out[16 * (size_t)i], T);
      memcpy(&out[16 * (size_t)i], T, sizeof(T));
    }
  }
  memcpy(poses, out.data(), out.size() * 8);
  return finish();
}

int32_t op_debug_pose_graph_solve(b2s_handle* h, int N, const double* A, const double* b, double lambda, double* delta_out, double* d_out,
                                  double* L_out) {
  PgLayout L;
  B2S_TRY(pg_prepare(h, N, 0, 0, 0, &L));
  const size_t n6 = (size_t)L.n6, M = (size_t)L.M;
  B2S_CUDA(cudaMemcpy2DAsync(L.A, M * 8, A, n6 * 8, n6 * 8, n6, cudaMemcpyHostToDevice, h->stream));
  B2S_CUDA(cudaMemcpyAsync(L.b, b, n6 * 8, cudaMemcpyHostToDevice, h->stream));
  B2S_CUDA(cudaMemcpyAsync(L.scal + PG_S_LAMBDA, &lambda, 8, cudaMemcpyHostToDevice, h->stream));
  h->launches += pg_factor_solve(h, L);
  B2S_CUDA(cudaGetLastError());
  B2S_CUDA(cudaMemcpyAsync(delta_out, L.delta, n6 * 8, cudaMemcpyDeviceToHost, h->stream));
  if (d_out) B2S_CUDA(cudaMemcpyAsync(d_out, L.D, n6 * 8, cudaMemcpyDeviceToHost, h->stream));
  if (L_out) B2S_CUDA(cudaMemcpy2DAsync(L_out, n6 * 8, L.F, M * 8, n6 * 8, n6, cudaMemcpyDeviceToHost, h->stream));
  B2S_TRY(check_status(h));
  if (L_out)   // F holds the pivots on its diagonal and stale values above it
    for (size_t r = 0; r < n6; r++) {
      L_out[r * n6 + r] = 1.0;
      for (size_t c = r + 1; c < n6; c++) L_out[r * n6 + c] = 0.0;
    }
  return B2S_OK;
}

int32_t op_debug_pose_graph_linearize(b2s_handle* h, int N, const double* poses, int ne, const b2s_pose_graph_edge* edges,
                                      const b2s_global_optimization_params& p, const double* conf_in, double* conf_out, double* H_out,
                                      double* b_out, double* rec_out) {
  const std::vector<b2s_pose_graph_edge> E(edges, edges + ne);
  const std::vector<double> conf(conf_in, conf_in + ne);
  std::vector<PgTask> tasks;
  std::vector<int32_t> contrib;
  PgLayout L;
  B2S_TRY(pg_load(h, N, E, conf, p, tasks, contrib, &L));
  B2S_CUDA(cudaMemcpyAsync(L.P, poses, 16 * 8 * (size_t)N, cudaMemcpyHostToDevice, h->stream));
  double rec[PG_R_WORDS];
  B2S_TRY(pg_eval(h, L, L.P));   // as pg_pass: the residual with the incoming confidences, then the linear system
  B2S_TRY(read_back(h, {{rec, L.rec, sizeof(rec)}}));
  rec_out[0] = rec[PG_R_RES];
  B2S_TRY(pg_linearize(h, L, (int)tasks.size()));
  const size_t n6 = (size_t)L.n6, M = (size_t)L.M;
  if (ne > 0) B2S_CUDA(cudaMemcpyAsync(conf_out, L.conf, 8 * (size_t)ne, cudaMemcpyDeviceToHost, h->stream));
  B2S_CUDA(cudaMemcpy2DAsync(H_out, n6 * 8, L.A, M * 8, n6 * 8, n6, cudaMemcpyDeviceToHost, h->stream));
  B2S_CUDA(cudaMemcpyAsync(b_out, L.b, n6 * 8, cudaMemcpyDeviceToHost, h->stream));
  B2S_TRY(read_back(h, {{rec, L.rec, sizeof(rec)}}));
  for (size_t r = 0; r < n6; r++)   // the factorisation reads the lower triangle; above it lie the diagonal blocks' upper halves
    for (size_t c = r + 1; c < n6; c++) H_out[r * n6 + c] = 0.0;
  rec_out[1] = rec[PG_R_MAXB]; rec_out[2] = rec[PG_R_MAXDIAG]; rec_out[3] = rec[PG_R_XX];
  return B2S_OK;
}

}  // namespace b2s
