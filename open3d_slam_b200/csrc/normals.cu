// normals.cu -- K-normals (P3): RegistrationIcpPointToPlane::estimateNormalsOrCovariancesIfNeeded
// (core/src/CloudRegistration.cpp:49-56) = [O3D] EstimateNormals(KDTreeSearchParamHybrid(radius, knn)) +
// NormalizeNormals + OrientNormalsTowardsCameraLocation(0,0,0).
//
// One WARP per query point, three kernels:
//   normals_select2_kernel  gathers the (2R+1)^3 block of grid cells (grid_index.cu) around the query into a per-warp shared-memory
//                           buffer, R grown until the k-th neighbour provably lies inside the block (ball-within-bounds, like a
//                           KD-tree), selects the k nearest by counting (32-bin histogram of d2 + exact ranking of the boundary
//                           bin; ties -> lower index) and sums the nine cumulants with a transposed warp butterfly;
//   normals_finish_kernel   one thread per query: analytic 3x3 eigen-solver ([O3D] FastEigen3x3, geometrictools
//                           RobustEigenSymmetric3x3), normalise, orient;
//   normals_phase2_kernel   the few queries the block gather cannot certify (more than NS2_CAP candidates, or a search radius the
//                           row table cannot cover): the warp ring walk grid_knn_walk (common.cuh), one list entry per lane.
// The neighbour SET is the oracle's exactly; the cumulants are summed in butterfly order instead of ascending-distance order, which
// moves the normal by < 1e-9.
#include "common.cuh"

namespace b2s {

constexpr int NK_THREADS = 128;

__device__ __forceinline__ void cross3d(const double* a, const double* b, double* o) {
  o[0] = a[1] * b[2] - a[2] * b[1]; o[1] = a[2] * b[0] - a[0] * b[2]; o[2] = a[0] * b[1] - a[1] * b[0];
}
__device__ __forceinline__ double dot3d(const double* a, const double* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

__device__ void eigvec0_dev(const double* A, double eval0, double* out) {
  double row0[3] = {A[0] - eval0, A[1], A[2]}, row1[3] = {A[1], A[4] - eval0, A[5]}, row2[3] = {A[2], A[5], A[8] - eval0};
  double r01[3], r02[3], r12[3];
  cross3d(row0, row1, r01); cross3d(row0, row2, r02); cross3d(row1, row2, r12);
  const double d0 = dot3d(r01, r01), d1 = dot3d(r02, r02), d2 = dot3d(r12, r12);
  double dmax = d0; int imax = 0;
  if (d1 > dmax) { dmax = d1; imax = 1; }
  if (d2 > dmax) { imax = 2; }
  const double* v = imax == 0 ? r01 : (imax == 1 ? r02 : r12);
  const double s = sqrt(imax == 0 ? d0 : (imax == 1 ? d1 : d2));
  out[0] = v[0] / s; out[1] = v[1] / s; out[2] = v[2] / s;
}

__device__ void eigvec1_dev(const double* A, const double* e0, double eval1, double* out) {
  double U[3], V[3];
  if (fabs(e0[0]) > fabs(e0[1])) {
    const double inv = 1 / sqrt(e0[0] * e0[0] + e0[2] * e0[2]);
    U[0] = -e0[2] * inv; U[1] = 0; U[2] = e0[0] * inv;
  } else {
    const double inv = 1 / sqrt(e0[1] * e0[1] + e0[2] * e0[2]);
    U[0] = 0; U[1] = e0[2] * inv; U[2] = -e0[1] * inv;
  }
  cross3d(e0, U, V);
  const double AU[3] = {A[0] * U[0] + A[1] * U[1] + A[2] * U[2], A[1] * U[0] + A[4] * U[1] + A[5] * U[2], A[2] * U[0] + A[5] * U[1] + A[8] * U[2]};
  const double AV[3] = {A[0] * V[0] + A[1] * V[1] + A[2] * V[2], A[1] * V[0] + A[4] * V[1] + A[5] * V[2], A[2] * V[0] + A[5] * V[1] + A[8] * V[2]};
  double m00 = dot3d(U, AU) - eval1, m01 = dot3d(U, AV), m11 = dot3d(V, AV) - eval1;
  const double a00 = fabs(m00), a01 = fabs(m01), a11 = fabs(m11);
  if (a00 >= a11) {
    const double mx = a00 > a01 ? a00 : a01;
    if (mx > 0) {
      if (a00 >= a01) { m01 /= m00; m00 = 1 / sqrt(1 + m01 * m01); m01 *= m00; }
      else { m00 /= m01; m01 = 1 / sqrt(1 + m00 * m00); m00 *= m01; }
      for (int d = 0; d < 3; d++) out[d] = m01 * U[d] - m00 * V[d];
    } else { out[0] = U[0]; out[1] = U[1]; out[2] = U[2]; }
  } else {
    const double mx = a11 > a01 ? a11 : a01;
    if (mx > 0) {
      if (a11 >= a01) { m01 /= m11; m11 = 1 / sqrt(1 + m01 * m01); m01 *= m11; }
      else { m11 /= m01; m01 = 1 / sqrt(1 + m11 * m11); m11 *= m01; }
      for (int d = 0; d < 3; d++) out[d] = m11 * U[d] - m01 * V[d];
    } else { out[0] = U[0]; out[1] = U[1]; out[2] = U[2]; }
  }
}

// eigenvector of the smallest eigenvalue of a symmetric 3x3 (row-major, full)
__device__ void fast_eigen3x3_dev(const double* cov, double* out) {
  double A[9];
  for (int i = 0; i < 9; i++) A[i] = cov[i];
  double mc = A[0];
  for (int i = 1; i < 9; i++) if (A[i] > mc) mc = A[i];
  if (mc == 0) { out[0] = out[1] = out[2] = 0; return; }
  for (int i = 0; i < 9; i++) A[i] /= mc;
  const double norm = A[1] * A[1] + A[2] * A[2] + A[5] * A[5];
  if (norm > 0) {
    double eval[3], e0[3], e1[3], e2[3];
    const double q = (A[0] + A[4] + A[8]) / 3;
    const double b00 = A[0] - q, b11 = A[4] - q, b22 = A[8] - q;
    const double p = sqrt((b00 * b00 + b11 * b11 + b22 * b22 + norm * 2) / 6);
    const double c00 = b11 * b22 - A[5] * A[5];
    const double c01 = A[1] * b22 - A[5] * A[2];
    const double c02 = A[1] * A[5] - b11 * A[2];
    const double det = (b00 * c00 - A[1] * c01 + A[2] * c02) / (p * p * p);
    double half_det = det * 0.5;
    half_det = fmin(fmax(half_det, -1.0), 1.0);
    const double angle = acos(half_det) / 3.0;
    const double two_thirds_pi = 2.09439510239319549;
    const double beta2 = cos(angle) * 2;
    const double beta0 = cos(angle + two_thirds_pi) * 2;
    const double beta1 = -(beta0 + beta2);
    eval[0] = q + p * beta0; eval[1] = q + p * beta1; eval[2] = q + p * beta2;
    if (half_det >= 0) {
      eigvec0_dev(A, eval[2], e2);
      if (eval[2] < eval[0] && eval[2] < eval[1]) { out[0] = e2[0]; out[1] = e2[1]; out[2] = e2[2]; return; }
      eigvec1_dev(A, e2, eval[1], e1);
      if (eval[1] < eval[0] && eval[1] < eval[2]) { out[0] = e1[0]; out[1] = e1[1]; out[2] = e1[2]; return; }
      cross3d(e1, e2, e0);
      out[0] = e0[0]; out[1] = e0[1]; out[2] = e0[2];
    } else {
      eigvec0_dev(A, eval[0], e0);
      if (eval[0] < eval[1] && eval[0] < eval[2]) { out[0] = e0[0]; out[1] = e0[1]; out[2] = e0[2]; return; }
      eigvec1_dev(A, e0, eval[1], e1);
      if (eval[1] < eval[0] && eval[1] < eval[2]) { out[0] = e1[0]; out[1] = e1[1]; out[2] = e1[2]; return; }
      cross3d(e0, e1, e2);
      out[0] = e2[0]; out[1] = e2[1]; out[2] = e2[2];
    }
  } else {
    const double a0 = A[0] * mc, a1 = A[4] * mc, a2 = A[8] * mc;
    if (a0 < a1 && a0 < a2) { out[0] = 1; out[1] = 0; out[2] = 0; }
    else if (a1 < a0 && a1 < a2) { out[0] = 0; out[1] = 1; out[2] = 0; }
    else { out[0] = 0; out[1] = 0; out[2] = 1; }
  }
}


// Post-search part shared by the finish and phase-2 kernels: covariance in the reference's neighbour order (ascending (d2, index)) with
// the reference's single-pass cumulant formula in explicitly rounded fp64, analytic eigen-solver, normalise, orient.
// prior (optional): the query's normal before the estimation -- [O3D] EstimateNormals on a cloud that already has normals keeps
// the prior where the solver returns a zero vector and otherwise flips the new normal when it points against the prior.  The
// caller reads it from the very slot nr is stored to afterwards (see op_estimate_normals).
__device__ __forceinline__ void finish_normal(const double c_in[9], int kk, double qx, double qy, double qz, const double* prior, double* nr) {
  double cov[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};  // [O3D] fewer than 3 neighbours -> identity covariance
  if (kk >= 3) {
    double c[9];
    const double kf = (double)kk;
#pragma unroll
    for (int t = 0; t < 9; t++) c[t] = __ddiv_rn(c_in[t], kf);
    cov[0] = __dsub_rn(c[3], __dmul_rn(c[0], c[0]));
    cov[4] = __dsub_rn(c[6], __dmul_rn(c[1], c[1]));
    cov[8] = __dsub_rn(c[8], __dmul_rn(c[2], c[2]));
    cov[1] = cov[3] = __dsub_rn(c[4], __dmul_rn(c[0], c[1]));
    cov[2] = cov[6] = __dsub_rn(c[5], __dmul_rn(c[0], c[2]));
    cov[5] = cov[7] = __dsub_rn(c[7], __dmul_rn(c[1], c[2]));
  }
  fast_eigen3x3_dev(cov, nr);
  if (prior) {
    const double pv[3] = {prior[0], prior[1], prior[2]};
    if (sqrt(dot3d(nr, nr)) == 0.0) { nr[0] = pv[0]; nr[1] = pv[1]; nr[2] = pv[2]; }
    else if (__dadd_rn(__dadd_rn(__dmul_rn(nr[0], pv[0]), __dmul_rn(nr[1], pv[1])), __dmul_rn(nr[2], pv[2])) < 0.0) {
      nr[0] *= -1.0; nr[1] *= -1.0; nr[2] *= -1.0;
    }
  } else if (sqrt(dot3d(nr, nr)) == 0.0) { nr[0] = 0; nr[1] = 0; nr[2] = 1; }
  const double zz = dot3d(nr, nr);  // NormalizeNormals
  if (zz > 0) { const double sn = sqrt(zz); nr[0] /= sn; nr[1] /= sn; nr[2] /= sn; }
  if (nr[0] != nr[0]) { nr[0] = 0; nr[1] = 0; nr[2] = 1; }
  const double ref[3] = {-qx, -qy, -qz};  // OrientNormalsTowardsCameraLocation(0,0,0)
  if (sqrt(dot3d(nr, nr)) == 0.0) {
    const double rn = sqrt(dot3d(ref, ref));
    if (rn == 0.0) { nr[0] = 0; nr[1] = 0; nr[2] = 1; }
    else { nr[0] = ref[0] / rn; nr[1] = ref[1] / rn; nr[2] = ref[2] / rn; }
  } else if (dot3d(nr, ref) < 0.0) { nr[0] *= -1.0; nr[1] *= -1.0; nr[2] *= -1.0; }
}

// Phase 2: one WARP per queued query, the ring walk of grid_knn_walk (common.cuh) with one list entry per lane (k <= 32).
template <bool kDebug>
__global__ void __launch_bounds__(NK_THREADS) normals_phase2_kernel(const GridHeader* __restrict__ hdr, const int32_t* __restrict__ cs,
                                                                    const double4* __restrict__ pts, int knn, double radius,
                                                                    const int32_t* __restrict__ queue, const int32_t* __restrict__ queue_n,
                                                                    const double* prior_nrm, double* out_nrm, double* __restrict__ dbg_rec) {
  pdl_wait();
  __shared__ GridHeader g;
  if (threadIdx.x == 0) g = *hdr;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int warps_total = gridDim.x * (NK_THREADS / 32);
  const int nq = *queue_n;
  const double r2 = radius * radius;
  for (int w = blockIdx.x * (NK_THREADS / 32) + (threadIdx.x >> 5); w < nq; w += warps_total) {
    const int s = queue[w];
    const double4 qp = pts[s];
    const double qx = qp.x, qy = qp.y, qz = qp.z;
    const int qi = (int)__double_as_longlong(qp.w);
    double ed[1]; int ei[1], es[1];   // this lane's entry of the sorted k-best list
    grid_knn_walk<1, true>(g, cs, pts, qx, qy, qz, knn, r2, ed, ei, es);
    // cumulants in ascending (d2, index) order: lane t holds the t-th neighbour, broadcast by shuffles
    const int kk = __popc(__ballot_sync(0xffffffffu, lane < knn && es[0] >= 0));
    double4 np = make_double4(0, 0, 0, 0);
    if (lane < kk) np = pts[es[0]];
    double c[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (int t = 0; t < kk; ++t) {
      const double x = __shfl_sync(0xffffffffu, np.x, t), y = __shfl_sync(0xffffffffu, np.y, t), z = __shfl_sync(0xffffffffu, np.z, t);
      c[0] = __dadd_rn(c[0], x); c[1] = __dadd_rn(c[1], y); c[2] = __dadd_rn(c[2], z);
      c[3] = __dadd_rn(c[3], __dmul_rn(x, x)); c[4] = __dadd_rn(c[4], __dmul_rn(x, y)); c[5] = __dadd_rn(c[5], __dmul_rn(x, z));
      c[6] = __dadd_rn(c[6], __dmul_rn(y, y)); c[7] = __dadd_rn(c[7], __dmul_rn(y, z)); c[8] = __dadd_rn(c[8], __dmul_rn(z, z));
    }
    if (lane == 0) {
      if (kDebug) {   // debug record (b2s_debug_estimate_normals): what finish_normal receives
        for (int t = 0; t < 9; t++) dbg_rec[10 * (size_t)qi + t] = c[t];
        dbg_rec[10 * (size_t)qi + 9] = (double)kk;
      }
      double nr[3];
      finish_normal(c, kk, qx, qy, qz, prior_nrm ? prior_nrm + 3 * (size_t)qi : nullptr, nr);
      out_nrm[3 * (size_t)qi] = nr[0]; out_nrm[3 * (size_t)qi + 1] = nr[1]; out_nrm[3 * (size_t)qi + 2] = nr[2];
    }
  }
}

// Butterfly sum of 9 values over the warp with the exchanges TRANSPOSED: at distance 16 the two halves of the warp split the values
// between them (each lane keeps the half it will finish and receives the partner's copy of it), at distance 8 the quarters do, and so
// on -- 8 + 4 + 2 + 1 + 1 = 16 exchanges instead of 9 x 5.  Every partial sum is the same pair of operands the plain xor butterfly
// adds at that distance (fp addition commutes), so the totals are bit-identical to it.  On return lane l holds the total of value
// l >> 1 in v[0] (values 9..15 are padding).
__device__ __forceinline__ void warp_sum9_transposed(double (&v)[9], int lane) {
  const unsigned FULL = 0xffffffffu;
  double a[8];
  {  // distance 16: lower half keeps 0..7, upper half keeps 8..15 (only 8 is real)
    const bool up = (lane & 16) != 0;
#pragma unroll
    for (int k = 0; k < 8; k++) {
      const double hi = k == 0 ? v[8] : 0.0;                 // value 8 + k
      const double send = up ? v[k] : hi;
      const double recv = __shfl_xor_sync(FULL, send, 16);
      a[k] = (up ? hi : v[k]) + recv;
    }
  }
  double b[4];
  {
    const bool up = (lane & 8) != 0;
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const double send = up ? a[k] : a[k + 4];
      const double recv = __shfl_xor_sync(FULL, send, 8);
      b[k] = (up ? a[k + 4] : a[k]) + recv;
    }
  }
  double c[2];
  {
    const bool up = (lane & 4) != 0;
#pragma unroll
    for (int k = 0; k < 2; k++) {
      const double send = up ? b[k] : b[k + 2];
      const double recv = __shfl_xor_sync(FULL, send, 4);
      c[k] = (up ? b[k + 2] : b[k]) + recv;
    }
  }
  double d;
  {
    const bool up = (lane & 2) != 0;
    const double send = up ? c[0] : c[1];
    const double recv = __shfl_xor_sync(FULL, send, 2);
    d = (up ? c[1] : c[0]) + recv;
  }
  d += __shfl_xor_sync(FULL, d, 1);
  v[0] = d;
}

// Block gather: one warp per query GATHERs the candidates of a cell block into a per-warp shared-memory buffer, SELECTs the k
// nearest by counting and sums their cumulants with a BUTTERFLY of shuffles.  The buffer lets the block radius R grow (1, 2, 3 cells)
// until the k-th neighbour provably lies inside the block: dense areas finish at R = 1, sparse far-range areas at
// R = 2 or 3, and only what is still unresolved (or holds more than NS2_CAP candidates) goes to normals_phase2_kernel.
constexpr int NS2_MIN_BLOCKS = 8;   // resident CTAs per SM the select kernel is compiled for (8 -> 64 registers)
constexpr int NS2_CAP = 256;
constexpr int NS2_CHUNKS = NS2_CAP / 32;
constexpr int NS2_RMAX = 3;
constexpr int NS2_ROWS = 320;   // row-table entries per warp: (2 R + 1)^2 rows of the largest block, rounded up to 32 (R = 8 -> 289)
// path codes of the debug record (b2s_debug_estimate_normals, include/b2s.h): 1..NS2_RMAX = select2 resolved the query at that block
// radius, then the block that covers the whole radius, then the two ways a query goes to normals_phase2_kernel
enum : int32_t { NPATH_FULL_BLOCK = NS2_RMAX + 1, NPATH_OVER_CAPACITY, NPATH_NOT_CERTIFIED };

// kDebug (b2s_debug_estimate_normals only): per grid slot, the path code (dbg_path) and the selection at the last block tried (dbg_sel,
// 4 doubles: candidates inside the certified ball nc, the histogram bin of the k-th key or -1 without a histogram, that bin's member count,
// lim2).  The production instantiation (kDebug = false) compiles none of it.
template <bool kDebug>
__global__ void __launch_bounds__(NK_THREADS, NS2_MIN_BLOCKS) normals_select2_kernel(const GridHeader* __restrict__ hdr, const int32_t* __restrict__ cs,
                                                                     const double4* __restrict__ pts, int knn, double radius,
                                                                     const int32_t* __restrict__ qlist, const int32_t* __restrict__ qcount,
                                                                     int32_t* __restrict__ queue, int32_t* queue_n,
                                                                     double* __restrict__ cum, int32_t* __restrict__ dbg_path,
                                                                     double* __restrict__ dbg_sel) {
  pdl_wait();
  __shared__ GridHeader g;
  __shared__ double s_d[NK_THREADS / 32][NS2_CAP];
  __shared__ int s_i[NK_THREADS / 32][NS2_CAP];
  __shared__ int s_s[NK_THREADS / 32][NS2_CAP];
  __shared__ int s_hist[NK_THREADS / 32][32];
  __shared__ int s_ra[NK_THREADS / 32][NS2_ROWS];       // first slot of every (y, z) row of the current block
  __shared__ int s_rp[NK_THREADS / 32][NS2_ROWS + 1];   // exclusive prefix of the row sizes
  if (threadIdx.x == 0) g = *hdr;
  __syncthreads();
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const unsigned lt_mask = (1u << lane) - 1u;
  const int n = g.n;
  const int nq = qlist ? *qcount : n;
  const double r2 = radius * radius;
  const double eps = 1e-9 * g.cell;
  const int nx = g.dims[0], ny = g.dims[1], nz = g.dims[2];
  const int warps_total = gridDim.x * (NK_THREADS / 32);
  for (int tq = blockIdx.x * (NK_THREADS / 32) + wib; tq < nq; tq += warps_total) {
    const int s = qlist ? qlist[tq] : tq;
    const double4 qp = pts[s];
    const double qx = qp.x, qy = qp.y, qz = qp.z;
    const double q[3] = {qx, qy, qz};
    const int c[3] = {grid_axis_cell(qx, g.origin[0], g.inv_cell, nx), grid_axis_cell(qy, g.origin[1], g.inv_cell, ny),
                      grid_axis_cell(qz, g.origin[2], g.inv_cell, nz)};
    const int cx = c[0], cy = c[1], cz = c[2];
    bool resolved = false;
    int need = 0;
    double c9[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    // starting radius from the local density: 25 lanes read the run boundaries of the 5x5 rows once; a 3x3x3 block with
    // fewer than ~3k points will almost never contain the k-th neighbour provably, so sparse queries start at R = 2
    int Rstart = 1;
    {
      int c1 = 0, c2 = 0;
      if (lane < 25) {
        const int dy = lane % 5 - 2, dz = lane / 5 - 2;
        const int y = cy + dy, z = cz + dz;
        if (y >= 0 && y < ny && z >= 0 && z < nz) {
          const int row = (z * ny + y) * nx;
          c2 = cs[row + min(cx + 2, nx - 1) + 1] - cs[row + max(cx - 2, 0)];
          if (dy >= -1 && dy <= 1 && dz >= -1 && dz <= 1) c1 = cs[row + min(cx + 1, nx - 1) + 1] - cs[row + max(cx - 1, 0)];
        }
      }
      const int n1 = warp_sum_i(c1), n2 = warp_sum_i(c2);
      const int n1b = __shfl_sync(0xffffffffu, n1, 0), n2b = __shfl_sync(0xffffffffu, n2, 0);
      if (n1b < 3 * knn && n2b <= NS2_CAP) Rstart = 2;
    }
    // Block radii tried: Rstart .. NS2_RMAX, then -- for the sparse queries that are still open (isolated far-range points, whose k
    // neighbours lie further apart than any certified ball of a small block) -- ONE block that covers the whole search radius, if its
    // rows fit the table: everything within the radius is then in the buffer and the answer is final even with fewer than k members.
    const int Rfull = (int)ceil(radius * g.inv_cell);
    const bool full_fits = Rfull > NS2_RMAX && (2 * Rfull + 1) * (2 * Rfull + 1) <= NS2_ROWS;
    constexpr int R_NONE = 1 << 20;
    for (int R = Rstart; !resolved && R != R_NONE; R = (R < NS2_RMAX ? R + 1 : (full_fits && R == NS2_RMAX ? Rfull : R_NONE))) {
      const bool last_try = R > NS2_RMAX || (R == NS2_RMAX && !full_fits);
      // ---- gather the (2R+1)^3 block into shared memory (valid = inside the radius), rows resolved by the lanes ----
      const int side = 2 * R + 1;
      const int x0 = max(cx - R, 0), x1 = min(cx + R, nx - 1);
      const double bound = ring_bound(g, q, c, R, eps);
      const double b2 = bound == INFINITY ? INFINITY : bound * bound;
      const double lim2 = fmin(r2, b2);   // candidates beyond the guaranteed ball cannot be certified at this R: drop them
      int nc = 0;
      // rows of the block -> (first slot, exclusive prefix of the row sizes) in shared memory; the candidates are then
      // walked as ONE flat sequence, 32 per step, so that short rows (a handful of points each) do not leave lanes idle
      int total = 0;
      const int nrows = (side * side + 31) & ~31;
      for (int t0 = 0; t0 < nrows; t0 += 32) {
        int a = 0, b = 0;
        const int t = t0 + lane;
        if (t < side * side) {
          const int z = cz - R + t / side, y = cy - R + t % side;
          if (z >= 0 && z < nz && y >= 0 && y < ny) { const int row = (z * ny + y) * nx; a = cs[row + x0]; b = cs[row + x1 + 1]; }
        }
        const int cnt = b - a;
        int inc = cnt;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += v; }
        s_ra[wib][t] = a;
        s_rp[wib][t] = total + inc - cnt;
        total += __shfl_sync(0xffffffffu, inc, 31);
      }
      if (lane == 0) s_rp[wib][nrows] = total;
      __syncwarp();
      for (int t0 = 0; t0 < total; t0 += 32) {
        const int t = t0 + lane;
        double dd = INFINITY; int ii = 0x7fffffff, j = -1;
        if (t < total) {
          int lo = 0, hi = side * side;   // first index whose prefix exceeds t; s_rp[side * side] = total > t (the padding rows are empty)
          while (lo < hi) { const int mid = (lo + hi) >> 1; if (s_rp[wib][mid] > t) hi = mid; else lo = mid + 1; }
          const int r = lo - 1;
          j = s_ra[wib][r] + (t - s_rp[wib][r]);
          const double4 p = pts[j];
          dd = dist2_exact(qx, qy, qz, p.x, p.y, p.z);
          ii = (int)__double_as_longlong(p.w);
        }
        const bool ok = j >= 0 && dd < lim2;
        const unsigned m = __ballot_sync(0xffffffffu, ok);
        const int pos = nc + __popc(m & lt_mask);
        if (ok && pos < NS2_CAP) { s_d[wib][pos] = dd; s_i[wib][pos] = ii; s_s[wib][pos] = j; }
        nc += __popc(m);
      }
      __syncwarp();
      if (nc > NS2_CAP) {   // too dense for the buffer: general kernel
        if (kDebug && lane == 0) { dbg_path[s] = NPATH_OVER_CAPACITY; dbg_sel[4 * (size_t)s] = nc; dbg_sel[4 * (size_t)s + 1] = -1; dbg_sel[4 * (size_t)s + 2] = 0; dbg_sel[4 * (size_t)s + 3] = lim2; }
        break;
      }
      // ---- candidates -> registers (round-robin), statistics ----
      // nc is uniform over the warp, so is the number of 32-candidate chunks in use: every chunk loop below stops there
      // (the loops stay fully unrolled -- the register arrays need static indices -- but the unused tail is branched over)
      const int nch = (nc + 31) >> 5;
      // only the keys live in registers; a candidate's slot stays in the shared buffer until the cumulants need it, and its
      // histogram bin is recomputed where it is used (one multiply) -- registers, i.e. resident warps, are what this kernel is short of
      double d[NS2_CHUNKS]; int idx[NS2_CHUNKS];
#pragma unroll
      for (int c = 0; c < NS2_CHUNKS; c++) {
        if (c >= nch) break;
        const int t = c * 32 + lane;
        d[c] = INFINITY; idx[c] = 0x7fffffff;
        if (t < nc) { d[c] = s_d[wib][t]; idx[c] = s_i[wib][t]; }
      }
      __syncwarp();
      need = min(knn, nc);
      double td = INFINITY; int ti = 0x7fffffff;
      int dbg_bin = -1, dbg_nb = 0;   // debug record only
      if (nc > knn) {   // k-th smallest (d2, index) by counting: 32-bin histogram over d2, then arg-min rounds in one bin
        // every candidate kept lies below lim2 (finite: lim2 <= radius^2), so that is the histogram's range -- no maximum to reduce
        const double scale = lim2 > 0.0 ? 32.0 / lim2 : 0.0;
        s_hist[wib][lane] = 0;
        __syncwarp();
#pragma unroll
        for (int c = 0; c < NS2_CHUNKS; c++) {
          if (c >= nch) break;
          if (c * 32 + lane < nc) atomicAdd(&s_hist[wib][min(31, (int)(d[c] * scale))], 1);
        }
        __syncwarp();
        int cumh = s_hist[wib][lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, cumh, o); if (lane >= o) cumh += t; }
        const int B = __ffs(__ballot_sync(0xffffffffu, cumh >= need)) - 1;
        const int below = B > 0 ? __shfl_sync(0xffffffffu, cumh, B - 1) : 0;
        const int m = need - below;
        // the m-th smallest (d2, index) of bin B by counting: its members go back to the (now free) candidate buffer, every lane ranks
        // one of them against all the others -- the keys are distinct, so exactly one member has rank m - 1
        int nb = 0;
#pragma unroll
        for (int c = 0; c < NS2_CHUNKS; c++) {
          if (c >= nch) break;
          const bool in_bin = c * 32 + lane < nc && min(31, (int)(d[c] * scale)) == B;
          const unsigned bm = __ballot_sync(0xffffffffu, in_bin);
          if (in_bin) { const int pos = nb + __popc(bm & lt_mask); s_d[wib][pos] = d[c]; s_i[wib][pos] = idx[c]; }
          nb += __popc(bm);
        }
        __syncwarp();
        if (kDebug) { dbg_bin = B; dbg_nb = nb; }
        for (int base = 0; base < nb; base += 32) {
          const int t = base + lane;
          double md = INFINITY; int mi = 0x7fffffff, rank = -1;
          if (t < nb) {
            md = s_d[wib][t]; mi = s_i[wib][t]; rank = 0;
            for (int u = 0; u < nb; u++) { const double od = s_d[wib][u]; const int oi = s_i[wib][u]; rank += (od < md || (od == md && oi < mi)) ? 1 : 0; }
          }
          const unsigned hit = __ballot_sync(0xffffffffu, rank == m - 1);
          if (hit) { const int src = __ffs(hit) - 1; td = __shfl_sync(0xffffffffu, md, src); ti = __shfl_sync(0xffffffffu, mi, src); break; }
        }
        __syncwarp();   // the buffer is written again by the next block radius
      }
      // (td, ti) = the k-th smallest key (inf when there are at most k candidates): the selected set is every key up to it
      // ---- exact?  every candidate kept lies strictly inside the guaranteed ball (radius sqrt(lim2) <= distance to the
      // nearest block face), so k kept candidates contain the true k nearest; fewer than k is final only when the
      // block covers the whole search radius ----
      if (!(nc >= knn || b2 > r2)) {   // grow the block
        if (last_try) {
          if (kDebug && lane == 0) { dbg_path[s] = NPATH_NOT_CERTIFIED; dbg_sel[4 * (size_t)s] = nc; dbg_sel[4 * (size_t)s + 1] = dbg_bin; dbg_sel[4 * (size_t)s + 2] = dbg_nb; dbg_sel[4 * (size_t)s + 3] = lim2; }
          break;
        }
        continue;
      }
      // ---- cumulants of the selected candidates, butterfly sum over the warp ----
#pragma unroll
      for (int c = 0; c < NS2_CHUNKS; c++) {
        if (c >= nch) break;
        const int t = c * 32 + lane;
        if (t < nc && (d[c] < td || (d[c] == td && idx[c] <= ti))) {
          const double4 p = pts[s_s[wib][t]];
          c9[0] += p.x; c9[1] += p.y; c9[2] += p.z;
          c9[3] += p.x * p.x; c9[4] += p.x * p.y; c9[5] += p.x * p.z;
          c9[6] += p.y * p.y; c9[7] += p.y * p.z; c9[8] += p.z * p.z;
        }
      }
      warp_sum9_transposed(c9, lane);   // lane l now holds the warp total of cumulant l >> 1 in c9[0] (l < 18)
      resolved = true;
      if (kDebug && lane == 0) { dbg_path[s] = R <= NS2_RMAX ? R : NPATH_FULL_BLOCK; dbg_sel[4 * (size_t)s] = nc; dbg_sel[4 * (size_t)s + 1] = dbg_bin; dbg_sel[4 * (size_t)s + 2] = dbg_nb; dbg_sel[4 * (size_t)s + 3] = lim2; }
    }
    if (!resolved) {
      if (lane == 0) { queue[atomicAdd(queue_n, 1)] = s; cum[10 * (size_t)tq + 9] = -1.0; }
      continue;
    }
    {
      // lanes 0, 2, .., 16 hold one cumulant each (see warp_sum9_transposed), lane 18 writes the neighbour count
      const int slot = lane >> 1;
      if (!(lane & 1) && slot < 10) cum[10 * (size_t)tq + slot] = slot < 9 ? c9[0] : (double)need;
    }
  }
}

// eigen-solver + normalise + orient for the queries the select kernel resolved: one THREAD per query
template <bool kDebug>
__global__ void __launch_bounds__(NK_THREADS) normals_finish_kernel(const GridHeader* __restrict__ hdr, const double4* __restrict__ pts,
                                                                    const int32_t* __restrict__ qlist, const int32_t* __restrict__ qcount,
                                                                    const double* __restrict__ cum, const double* prior_nrm, double* out_nrm,
                                                                    double* __restrict__ dbg_rec) {
  pdl_wait();
  const int nq = qlist ? *qcount : hdr->n;
  for (int tq = blockIdx.x * blockDim.x + threadIdx.x; tq < nq; tq += gridDim.x * blockDim.x) {
    const double kkd = cum[10 * (size_t)tq + 9];
    if (kkd < 0.0) continue;   // left to normals_phase2_kernel
    double c9[9];
#pragma unroll
    for (int t = 0; t < 9; t++) c9[t] = cum[10 * (size_t)tq + t];
    const double4 qp = pts[qlist ? qlist[tq] : tq];
    const size_t qi = (size_t)(int)__double_as_longlong(qp.w);
    if (kDebug) {   // debug record (b2s_debug_estimate_normals): what finish_normal receives
#pragma unroll
      for (int t = 0; t < 9; t++) dbg_rec[10 * qi + t] = c9[t];
      dbg_rec[10 * qi + 9] = kkd;
    }
    double nr[3];
    finish_normal(c9, (int)kkd, qp.x, qp.y, qp.z, prior_nrm ? prior_nrm + 3 * qi : nullptr, nr);
    out_nrm[3 * qi] = nr[0]; out_nrm[3 * qi + 1] = nr[1]; out_nrm[3 * qi + 2] = nr[2];
  }
}


__global__ void zero_i32_kernel(int32_t* p) {
  pdl_wait(); p[0] = 0; p[1] = 0; }

// query list = grid slots whose original point is flagged; warp-aggregated append keeps neighbouring slots together
__global__ void __launch_bounds__(NK_THREADS) normals_qlist_kernel(const GridHeader* __restrict__ hdr, const double4* __restrict__ pts,
                                                                   const int32_t* __restrict__ flags, int32_t* __restrict__ qlist,
                                                                   int32_t* qcount) {
  pdl_wait();
  const int n = hdr->n;
  const int lane = threadIdx.x & 31;
  const int n_round = (n + 31) & ~31;
  for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < n_round; s += gridDim.x * blockDim.x) {
    bool take = false;
    if (s < n) take = flags[(int)__double_as_longlong(pts[s].w)] != 0;
    const unsigned m = __ballot_sync(0xffffffffu, take);
    int base = 0;
    if (lane == 0 && m) base = atomicAdd(qcount, __popc(m));
    base = __shfl_sync(0xffffffffu, base, 0);
    if (take) qlist[base + __popc(m & ((1u << lane) - 1u))] = s;
  }
}

int32_t op_estimate_normals(b2s_handle* h, b2s_cloud* c, int knn, double radius, double cell_hint, const int32_t* flags, bool with_prior,
                            const NormalsDebug* dbg) {
  B2S_REQUIRE(radius > 0.0, B2S_E_INVALID, "maxRadiusNormalEstimation_ must be > 0");  // CloudRegistration.cpp:50
  B2S_REQUIRE(knn > 0, B2S_E_INVALID, "knnNormalEstimation_ must be > 0");            // CloudRegistration.cpp:51
  B2S_REQUIRE(knn <= 32, B2S_E_UNSUPPORTED, "knn > 32 is not supported by the register-resident k-best list yet");
  B2S_REQUIRE(!with_prior || c->has_normals, B2S_E_NO_NORMALS, "prior normals requested for a cloud without normals");
  double cell = cell_hint > 0.0 ? cell_hint : radius / 4.0;
  if (cell < radius / 16.0) cell = radius / 16.0;  // bound the ring count of the worst case
  B2S_TRY(grid_build(h, &h->grid_b, c, cell, nullptr));
  const size_t n_max = c->n_max > 0 ? c->n_max : 1;
  B2S_TRY(c->nrm.ensure(n_max * 24, h->stream, with_prior));
  int blocks = (int)((n_max + NK_THREADS - 1) / NK_THREADS);
  if (blocks > 16 * device_sms()) blocks = 16 * device_sms();
  if (blocks < 1) blocks = 1;
  // phase-2 queue: counter + one slot per point
  B2S_TRY(h->tmp_i32.ensure((2 * n_max + 64) * 4, h->stream));
  int32_t* qn = h->tmp_i32.as<int32_t>() + 8;        // [0] phase-2 queue length, [1] query-list length
  int32_t* queue = h->tmp_i32.as<int32_t>() + 16;
  int32_t* qlist = flags ? queue + n_max : nullptr;
  const int32_t* qcount = flags ? qn + 1 : nullptr;
  ProfScope prof(h, PK_NORMALS);
  const GridHeader* hdr = h->grid_b.hdr.as<GridHeader>();
  const int32_t* cs = grid_starts(&h->grid_b);
  const double4* pts = h->grid_b.pts.as<double4>();
  double* out = c->nrm.as<double>();
  // The prior normals are the output array itself.  That is safe because every kernel below reads only the POSITIONS of other
  // points, and each point's normal slot is read (its prior) and then written by exactly one thread: the finish kernel or the
  // phase-2 kernel, whichever resolves the query.  Keep it so: a kernel that read another point's normal, or two kernels writing
  // the same slot, would see overwritten priors.
  const double* prior = with_prior ? out : nullptr;
  launch_pdl(zero_i32_kernel, 1, 1, 0, h->stream, qn);
  if (flags) {
    launch_pdl(normals_qlist_kernel, blocks, NK_THREADS, 0, h->stream, hdr, pts, flags, qlist, qn + 1);
    h->launches++;
  }
  // gather + select (one warp per query, grid-stride; B2S_NS2_GRID: A/B knob of the grid size), stragglers to the phase-2 kernel
  static const int ns2_grid_env = getenv("B2S_NS2_GRID") ? atoi(getenv("B2S_NS2_GRID")) : 0;
  const int ns2_cap = ns2_grid_env > 0 ? ns2_grid_env : 16 * device_sms();
  int wblocks = (int)((n_max + (NK_THREADS / 32) - 1) / (NK_THREADS / 32));
  if (wblocks > ns2_cap) wblocks = ns2_cap;
  if (wblocks < 1) wblocks = 1;
  B2S_TRY(h->tmp_f64.ensure((n_max + 1) * 80, h->stream));
  double* cum = h->tmp_f64.as<double>();
  if (dbg) launch_pdl(normals_select2_kernel<true>, wblocks, NK_THREADS, 0, h->stream, hdr, cs, pts, knn, radius, qlist, qcount, queue, qn,
                      cum, dbg->path, dbg->sel);
  else launch_pdl(normals_select2_kernel<false>, wblocks, NK_THREADS, 0, h->stream, hdr, cs, pts, knn, radius, qlist, qcount, queue, qn, cum,
                  nullptr, nullptr);
  if (dbg) launch_pdl(normals_finish_kernel<true>, blocks, NK_THREADS, 0, h->stream, hdr, pts, qlist, qcount, cum, prior, out, dbg->rec);
  else launch_pdl(normals_finish_kernel<false>, blocks, NK_THREADS, 0, h->stream, hdr, pts, qlist, qcount, cum, prior, out, nullptr);
  if (dbg) launch_pdl(normals_phase2_kernel<true>, 4 * device_sms(), NK_THREADS, 0, h->stream, hdr, cs, pts, knn, radius, queue, qn, prior, out,
                      dbg->rec);
  else launch_pdl(normals_phase2_kernel<false>, 4 * device_sms(), NK_THREADS, 0, h->stream, hdr, cs, pts, knn, radius, queue, qn, prior, out,
                  nullptr);
  h->launches += 4;
  c->has_normals = true;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

}  // namespace b2s
