// icp.cu -- K-icp-iter: the whole ICP loop of one registration inside ONE persistent kernel.
//
// Replaces [O3D] RegistrationICP as called by the reference's three CloudRegistration classes
// (core/src/CloudRegistration.cpp:15-20 generalized, :44-48 point-to-plane, :69-75 point-to-point), i.e. SURVEY.md 8a rows
// R3 (correspondence search), R4 (per-estimator sums), R5 (solve, SE(3) update, convergence test), plus one-evaluation
// mode for [O3D] GetInformationMatrixFromPointClouds.  Three instantiations (icp_kernel<MODE>): 0 point-to-plane only
// (the headline path carries no code of the others), 1 point-to-point + information matrix, 2 generalized ICP.
//
// Mapping to the machine:
//   * one thread-block CLUSTER (1..8 CTAs, one per SM; 16 on request) per registration, blockIdx.y = registration in the batch;
//   * the working copy of the source cloud lives in shared memory for the whole loop and is advanced by the per-iteration update
//     like [O3D] pcd.Transform(update); the cloud is dealt out in tiles of 64 points, tile t to CTA t % cluster size, every full
//     tile staged by one bulk-async copy (cp.async.bulk + mbarrier);
//   * exact nearest neighbour with the strict d2 < r2 cut through the dense grid of grid_index.cu.  Per evaluation:
//       sweep A, every point: apply the update; CERTIFICATES decide whether the previous answer provably still stands (one distance
//                evaluation instead of a search); the points that need a search are compacted into a list;
//       sweep B, one thread per listed point: BOX QUERY -- the cells overlapping [q - d, q + d], one contiguous slot range per
//                (y, z) row, with d = distance to the previous evaluation's neighbour; without a neighbour to start from (first
//                evaluation) a half-cell box, then a one-cell box; four rows / four candidates in flight per thread;
//       phase 2, one WARP per unresolved point (outliers / empty neighbourhoods, queued in shared memory): the rows of the box
//                around the search sphere are spread over the 32 lanes, then a warp lexicographic-min; the queues of all CTAs
//                are drained by all warps of the cluster through distributed shared memory.
//     Ties -> lower target index.  Gathers hit the L2-resident target.
//   * the 29 sums (plane / GICP: 21 JtJ + 6 Jtr; point-to-point: means + cross moments; information: target moments; + sum d2 +
//     count) are never per-thread state: each warp reduces the terms of 32 points at once (transposed butterfly, lane k ends up
//     with term k) into its row of a shared-memory accumulator; rows -> CTA partial -> DSMEM exchange: every CTA reads all cluster
//     partials in rank order and redundantly computes the update (6x6 LDLT with diagonal pivoting, or umeyama with a one-thread
//     Jacobi SVD), so no host round trip ever happens;
//   * all arithmetic fp64; distances and the point transform use explicitly rounded ops (no FMA contraction) so that
//     correspondences are bit-identical to the CPU oracle.
#include <cooperative_groups.h>

#include "common.cuh"

namespace cg = cooperative_groups;

namespace b2s {

constexpr int NACC = 29;  // 21 upper-triangular JtJ + 6 Jtr + sum d2 + count
// threads per CTA by instantiation: the point-to-plane / point-to-point / information kernels keep NO per-thread accumulators
// (every contribution is warp-reduced at once into a per-warp accumulator in shared memory) and run 768 threads = 24 warps per SM
// at 80 registers; the generalized-ICP kernel carries 3x3 covariance algebra per correspondence and stays at 512 threads
#ifndef B2S_ICP_PLANE_THREADS
#define B2S_ICP_PLANE_THREADS 768   // 768 threads: 80 registers each still fit one CTA per SM (make alt ALT_THREADS=... builds libb2s_alt<N>.so for A/B runs)
#endif
constexpr int icp_threads(int mode) { return mode == 2 ? 512 : B2S_ICP_PLANE_THREADS; }
constexpr int ICP_TILE = 64;   // points per tile of the source cloud (tile t belongs to CTA t % cluster size)
constexpr int ICP_R1 = -1;  // phase 1 is a box query, not a ring walk: phase 2 starts its ring walk at ring 0
constexpr int ICP_MAX_CLUSTER = 16;   // 8 is the portable limit; 16 needs cudaFuncAttributeNonPortableClusterSizeAllowed

// ---- bulk-async (TMA engine) staging of the source chunk: global -> shared, completion on an mbarrier --------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(unsigned long long* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// cp.async.bulk: 16-byte aligned source / destination, size a multiple of 16 (SASS: UBLKCP)
__device__ __forceinline__ void bulk_copy_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)), "l"(src_gmem),
               "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void mbar_wait_parity(unsigned long long* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "LAB_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
      "@P1 bra DONE;\n"
      "bra LAB_WAIT;\n"
      "DONE:\n"
      "}" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}

struct GridView {
  double ox, oy, oz, cell, inv, eps;
  int nx, ny, nz;
  const int32_t* __restrict__ cs;
  const double4* __restrict__ pts;
  const double* __restrict__ nrm;   // the target cloud's normals in cloud order: point pts[slot] has nrm[3 * bits(pts[slot].w)]
};

__device__ __forceinline__ double4 target_normal(const GridView& g, const double4& q) {
  const double* n = g.nrm + 3 * (size_t)__double_as_longlong(q.w);
  return make_double4(n[0], n[1], n[2], 0.0);
}

struct NNState {
  double best;     // d2 of the best candidate so far (or the search limit while bslot < 0)
  double second;   // d2 of the best OTHER candidate seen (inf: none) -- with `gb` the raw material of the gap certificate
  double gb;       // every target that was NOT looked at lies further than this from the query (distance, not squared)
  int bidx, bslot;
  int scanned;   // candidates looked at (only read by the counting instantiation, icp_kernel<3>)
};

__device__ __forceinline__ double slab_gap(double q, double o, double cell, int i, int n, double eps) {
  double g = 0.0;
  if (i > 0) { double lo = o + (double)i * cell; if (q < lo) g = lo - q; }
  if (i < n - 1) { double hi = o + (double)(i + 1) * cell; if (q > hi) g = q - hi; }
  g -= eps;  // slack: cell membership was decided with floor((p-o)*inv), which can disagree with o+i*cell by an ulp
  return g > 0.0 ? g : 0.0;
}

__device__ __forceinline__ void nn_scan_range(const double4* __restrict__ pts, int s, int e, double qx, double qy, double qz, NNState& st) {
  st.scanned += e > s ? e - s : 0;   // statistics (dead code unless the counting instantiation reads it)
#pragma unroll 4
  for (int j = s; j < e; ++j) {
    const double4 p = pts[j];
    const double d = dist2_exact(qx, qy, qz, p.x, p.y, p.z);
    const int idx = (int)__double_as_longlong(p.w);
    if (d < st.best || (d == st.best && st.bslot >= 0 && idx < st.bidx)) {
      if (st.bslot >= 0) st.second = st.best;
      st.best = d; st.bidx = idx; st.bslot = j;
    } else if (j != st.bslot && d < st.second) {
      st.second = d;
    }
  }
}

// one (y, z) row of ring R around cell (cx, cy, cz): the whole (clipped) x-run on the shell, else the two end cells
__device__ __forceinline__ void nn_scan_row(const GridView& g, double qx, double qy, double qz, int cx, int cy, int cz, int R, int y, int z,
                                            NNState& st) {
  const double gz = slab_gap(qz, g.oz, g.cell, z, g.nz, g.eps);
  const double gy = slab_gap(qy, g.oy, g.cell, y, g.ny, g.eps);
  const double g2 = gz * gz + gy * gy;
  if (g2 > st.best) return;
  const int row = (z * g.ny + y) * g.nx;
  if (z == cz - R || z == cz + R || y == cy - R || y == cy + R) {
    const int x0 = max(cx - R, 0), x1 = min(cx + R, g.nx - 1);
    // clip the run to the cells the current best sphere can reach along x
    const double xr = sqrt(fmax(st.best - g2, 0.0)) + g.eps;
    const int xa = max(x0, (int)fmin(fmax(floor((qx - xr - g.ox) * g.inv), 0.0), (double)(g.nx - 1)));
    const int xb = min(x1, (int)fmin(fmax(floor((qx + xr - g.ox) * g.inv), 0.0), (double)(g.nx - 1)));
    if (xa <= xb) nn_scan_range(g.pts, g.cs[row + xa], g.cs[row + xb + 1], qx, qy, qz, st);
  } else {
    if (cx - R >= 0) nn_scan_range(g.pts, g.cs[row + cx - R], g.cs[row + cx - R + 1], qx, qy, qz, st);
    if (cx + R <= g.nx - 1) nn_scan_range(g.pts, g.cs[row + cx + R], g.cs[row + cx + R + 1], qx, qy, qz, st);
  }
}

// distance below which every unvisited point must lie after the (2R+1)^3 block has been scanned (inf: grid exhausted)
__device__ __forceinline__ double ring_bound(const GridView& g, double qx, double qy, double qz, int cx, int cy, int cz, int R) {
  double bound = INFINITY;
  if (cx - R > 0) bound = fmin(bound, qx - (g.ox + (double)(cx - R) * g.cell));
  if (cx + R < g.nx - 1) bound = fmin(bound, (g.ox + (double)(cx + R + 1) * g.cell) - qx);
  if (cy - R > 0) bound = fmin(bound, qy - (g.oy + (double)(cy - R) * g.cell));
  if (cy + R < g.ny - 1) bound = fmin(bound, (g.oy + (double)(cy + R + 1) * g.cell) - qy);
  if (cz - R > 0) bound = fmin(bound, qz - (g.oz + (double)(cz - R) * g.cell));
  if (cz + R < g.nz - 1) bound = fmin(bound, (g.oz + (double)(cz + R + 1) * g.cell) - qz);
  if (bound == INFINITY) return bound;
  bound -= g.eps;
  return bound > 0.0 ? bound : 0.0;
}

__device__ __forceinline__ void cell_of(const GridView& g, double qx, double qy, double qz, int& cx, int& cy, int& cz) {
  cx = (int)fmin(fmax(floor((qx - g.ox) * g.inv), 0.0), (double)(g.nx - 1));
  cy = (int)fmin(fmax(floor((qy - g.oy) * g.inv), 0.0), (double)(g.ny - 1));
  cz = (int)fmin(fmax(floor((qz - g.oz) * g.inv), 0.0), (double)(g.nz - 1));
}

// every cell overlapping the box [q - rad, q + rad]: one contiguous slot range per (y, z) row.
// The walk is software-pipelined, because one thread's search is nothing but a chain of L2 round trips: the slot ranges of FOUR
// rows are fetched at once (8 independent loads), their candidates are then addressed as one flat sequence and fetched four at a
// time (x, y, z only: 24 bytes) before any of them is looked at.  The original index of a candidate (the tie-breaker of equal
// distances) is only read when two distances are exactly equal; st.bidx is NOT maintained here (phase 1 never needs it).
__device__ __forceinline__ void nn_scan_box(const GridView& g, double qx, double qy, double qz, double rad, NNState& st) {
  const int ix0 = (int)fmin(fmax(floor((qx - rad - g.ox) * g.inv), 0.0), (double)(g.nx - 1));
  const int ix1 = (int)fmin(fmax(floor((qx + rad - g.ox) * g.inv), 0.0), (double)(g.nx - 1));
  const int iy0 = (int)fmin(fmax(floor((qy - rad - g.oy) * g.inv), 0.0), (double)(g.ny - 1));
  const int iy1 = (int)fmin(fmax(floor((qy + rad - g.oy) * g.inv), 0.0), (double)(g.ny - 1));
  const int iz0 = (int)fmin(fmax(floor((qz - rad - g.oz) * g.inv), 0.0), (double)(g.nz - 1));
  const int iz1 = (int)fmin(fmax(floor((qz + rad - g.oz) * g.inv), 0.0), (double)(g.nz - 1));
  int y = iy0, z = iz0;
  while (z <= iz1) {
    int rs[4], rn[4];   // first slot of each of the next four rows, inclusive prefix of their sizes
#pragma unroll
    for (int u = 0; u < 4; u++) {
      int a = 0, b = 0;
      if (z <= iz1) {
        const int row = (z * g.ny + y) * g.nx;
        a = g.cs[row + ix0]; b = g.cs[row + ix1 + 1];
        if (++y > iy1) { y = iy0; ++z; }
      }
      rs[u] = a; rn[u] = b - a;
    }
    rn[1] += rn[0]; rn[2] += rn[1]; rn[3] += rn[2];
    const int total = rn[3];
    st.scanned += total;
    for (int c0 = 0; c0 < total; c0 += 4) {
      int j[4]; double cx[4], cy[4], cz[4];
#pragma unroll
      for (int v = 0; v < 4; v++) {
        const int c = min(c0 + v, total - 1);
        j[v] = c < rn[0] ? rs[0] + c : (c < rn[1] ? rs[1] + (c - rn[0]) : (c < rn[2] ? rs[2] + (c - rn[1]) : rs[3] + (c - rn[2])));
        const double2 xy = *reinterpret_cast<const double2*>(&g.pts[j[v]]);
        cx[v] = xy.x; cy[v] = xy.y; cz[v] = g.pts[j[v]].z;
      }
#pragma unroll
      for (int v = 0; v < 4; v++) {
        if (c0 + v < total) {
          const double d = dist2_exact(qx, qy, qz, cx[v], cy[v], cz[v]);
          if (d < st.best) {
            if (st.bslot >= 0) st.second = st.best;
            st.best = d; st.bslot = j[v];
          } else if (j[v] != st.bslot) {
            if (d < st.second) st.second = d;
            if (d == st.best && st.bslot >= 0) {   // exact tie: the lower original index wins
              const int ia = (int)__double_as_longlong(g.pts[j[v]].w), ib = (int)__double_as_longlong(g.pts[st.bslot].w);
              if (ia < ib) st.bslot = j[v];
            }
          }
        }
      }
    }
  }
  // the block of cells just walked: whatever was not looked at lies beyond its faces (faces on the grid border have nothing behind
  // them: outside points were clamped INTO the border cells)
  double gb = INFINITY;
  if (ix0 > 0) gb = fmin(gb, qx - (g.ox + (double)ix0 * g.cell));
  if (ix1 < g.nx - 1) gb = fmin(gb, (g.ox + (double)(ix1 + 1) * g.cell) - qx);
  if (iy0 > 0) gb = fmin(gb, qy - (g.oy + (double)iy0 * g.cell));
  if (iy1 < g.ny - 1) gb = fmin(gb, (g.oy + (double)(iy1 + 1) * g.cell) - qy);
  if (iz0 > 0) gb = fmin(gb, qz - (g.oz + (double)iz0 * g.cell));
  if (iz1 < g.nz - 1) gb = fmin(gb, (g.oz + (double)(iz1 + 1) * g.cell) - qz);
  if (gb != INFINITY) gb = fmax(gb - g.eps, 0.0);
  st.gb = gb;
}

// phase 1 (one thread): BOX QUERY.  The previous iteration's neighbour (`hint`, -1 = none) is almost always still the
// nearest or next to it, so the exact answer lies within its distance d_h of the query: scan exactly the cells that
// overlap the box [q - d_h, q + d_h] (one contiguous slot range per (y, z) row) -- a handful of candidates, no ring
// walk, no per-row bounds.  Without a usable hint the box half-width is one cell edge; a hit inside that radius is
// exact as well.  Anything else (no point within the box radius, or a box wider than 2 cells) is left to phase 2.
// Cell indices use the same floor((v - o) * inv) expression as the index build, which is monotone in v, so no point
// inside the box can sit in a cell outside the index range.  Returns true when st holds the exact answer.
__device__ __forceinline__ bool nn_phase1(const GridView& g, double qx, double qy, double qz, double r2, int hint, NNState& st) {
  st.best = r2; st.second = INFINITY; st.gb = 0.0; st.bidx = 0x7fffffff; st.bslot = -1; st.scanned = 0;
  if (!(qx == qx && qy == qy && qz == qz)) return true;
  double rad2 = fmin(r2, g.cell * g.cell);
  bool seeded = false;
  if (hint >= 0) {
    const double4 p = g.pts[hint];
    const double d = dist2_exact(qx, qy, qz, p.x, p.y, p.z);
    if (d < r2) { st.best = d; st.bidx = (int)__double_as_longlong(p.w); st.bslot = hint; rad2 = d; seeded = true; }
  }
  const double radm = sqrt(rad2) * (1.0 + 1e-12) + 1e-300;
  if (radm > 2.0 * g.cell) return false;
  if (!seeded) {
    // stage A: a half-cell box first (at most 2 x 2 x 2 cells instead of 3 x 3 x 3).  Every point within half a cell edge of
    // the query lies inside it, so a hit at that distance is already exact -- which is the case for almost every inlier
    // of the first evaluation, the one that has no neighbours to start from.
    const double ra = 0.5 * g.cell;
    if (ra * ra < rad2) {
      nn_scan_box(g, qx, qy, qz, ra, st);
      if (st.bslot >= 0 && st.best <= ra * ra) return true;
    }
  }
  nn_scan_box(g, qx, qy, qz, radm, st);   // cells seen in stage A are seen again: an equal candidate never replaces the best
  // seeded: every point at distance <= d_h was scanned.  unseeded: exact iff the best lies within the box radius.
  return seeded || (st.bslot >= 0 && st.best <= rad2);
}

// phase 2 (one warp, all lanes with the same query): continues from ring ICP_R1 + 1 with the rows of each ring spread
// over the lanes.  st must hold the phase-1 state; on return every lane holds the exact answer.
__device__ __forceinline__ void nn_phase2_warp(const GridView& g, double qx, double qy, double qz, double clip2, NNState& st) {
  // One pass over the box that encloses the sphere of the seed distance (or of the correspondence radius when there is
  // no seed): the (y, z) rows of the box are independent, so they are spread over the lanes and every lane clips its
  // row's x-run to the sphere.  No ring-by-ring termination tests, one warp reduction at the end.
  const int lane = threadIdx.x & 31;
  // clip2: FIXED square radius of the ball that is searched completely (it does not shrink with the best candidate, so that on
  // return every target within sqrt(clip2) has been looked at: the guarantee behind the gap certificate)
  const double radm = sqrt(clip2) * (1.0 + 1e-12) + 1e-300;
  const int iy0 = (int)fmin(fmax(floor((qy - radm - g.oy) * g.inv), 0.0), (double)(g.ny - 1));
  const int iy1 = (int)fmin(fmax(floor((qy + radm - g.oy) * g.inv), 0.0), (double)(g.ny - 1));
  const int iz0 = (int)fmin(fmax(floor((qz - radm - g.oz) * g.inv), 0.0), (double)(g.nz - 1));
  const int iz1 = (int)fmin(fmax(floor((qz + radm - g.oz) * g.inv), 0.0), (double)(g.nz - 1));
  const int ny_ = iy1 - iy0 + 1, nrows = ny_ * (iz1 - iz0 + 1);
  for (int t0 = lane; t0 < nrows; t0 += 128) {   // four rows per lane and trip: their slot ranges are fetched together (8 independent loads)
    int ra[4], rb[4];
#pragma unroll
    for (int u = 0; u < 4; u++) {
      const int t = t0 + 32 * u;
      ra[u] = 0; rb[u] = 0;
      if (t < nrows) {
        const int y = iy0 + t % ny_, z = iz0 + t / ny_;
        const double gz = slab_gap(qz, g.oz, g.cell, z, g.nz, g.eps);
        const double gy = slab_gap(qy, g.oy, g.cell, y, g.ny, g.eps);
        const double g2 = gz * gz + gy * gy;
        if (!(g2 > clip2)) {
          const double xr = sqrt(fmax(clip2 - g2, 0.0)) * (1.0 + 1e-12) + g.eps;
          const int xa = (int)fmin(fmax(floor((qx - xr - g.ox) * g.inv), 0.0), (double)(g.nx - 1));
          const int xb = (int)fmin(fmax(floor((qx + xr - g.ox) * g.inv), 0.0), (double)(g.nx - 1));
          const int row = (z * g.ny + y) * g.nx;
          ra[u] = g.cs[row + xa]; rb[u] = g.cs[row + xb + 1];
        }
      }
    }
#pragma unroll
    for (int u = 0; u < 4; u++) nn_scan_range(g.pts, ra[u], rb[u], qx, qy, qz, st);
  }
  // lexicographic (d2, index) minimum over the lanes; a lane without a hit carries slot -1
  const double my_best = st.best, my_second = st.second;
  const int my_slot = st.bslot;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double od = __shfl_xor_sync(0xffffffffu, st.best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, st.bidx, o);
    const int os = __shfl_xor_sync(0xffffffffu, st.bslot, o);
    const bool take = os >= 0 && (st.bslot < 0 || od < st.best || (od == st.best && oi < st.bidx));
    if (take) { st.best = od; st.bidx = oi; st.bslot = os; }
  }
  // the best OTHER candidate: every lane's runner-up, and every lane's own best unless that is the winner itself
  double sec = my_second;
  if (my_slot >= 0 && my_slot != st.bslot) sec = fmin(sec, my_best);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sec = fmin(sec, __shfl_xor_sync(0xffffffffu, sec, o));
  st.second = sec;
}

// ---- small fp64 linear algebra on one thread, registers only -----------------------------------------------------

// A x = b, A symmetric 6x6.  LDL^T with symmetric pivoting on the largest |diagonal|, the scheme Eigen's LDLT uses for [O3D]
// SolveLinearSystemPSD (no determinant / PSD check on this call path).  ONE thread, the matrix in shared memory with dynamic
// indices: a pivot swap is a real (and rare) exchange of one row and one column.  (The round-1 version kept everything in
// registers with select-based swaps so that nothing went to local memory -- and spent most of its ~2000 instructions on the
// selects: 4 us per evaluation with every other thread of the cluster waiting.)
// a: 36 doubles (row-major, full storage), b: 6 doubles; the solution is left in b.
__device__ __forceinline__ void ldlt6_solve_smem(double* a, double* b) {
  int piv[6];
#pragma unroll
  for (int k = 0; k < 6; k++) {
    int p = k;
    double best = fabs(a[7 * k]);
#pragma unroll
    for (int i = k + 1; i < 6; i++) { const double v = fabs(a[7 * i]); if (v > best) { best = v; p = i; } }
    piv[k] = p;
    if (p != k) {
      for (int j = 0; j < 6; j++) { const double u = a[6 * k + j]; a[6 * k + j] = a[6 * p + j]; a[6 * p + j] = u; }
      for (int j = 0; j < 6; j++) { const double u = a[6 * j + k]; a[6 * j + k] = a[6 * j + p]; a[6 * j + p] = u; }
      { const double u = b[k]; b[k] = b[p]; b[p] = u; }
    }
    const double d = a[7 * k];
    if (d != 0.0) {
#pragma unroll
      for (int i = k + 1; i < 6; i++) a[6 * i + k] /= d;
#pragma unroll
      for (int i = k + 1; i < 6; i++)
#pragma unroll
        for (int j = k + 1; j <= i; j++) {
          const double v = a[6 * i + j] - a[6 * i + k] * d * a[6 * j + k];
          a[6 * i + j] = v;
          a[6 * j + i] = v;
        }
    }
  }
#pragma unroll
  for (int i = 0; i < 6; i++)
#pragma unroll
    for (int j = 0; j < i; j++) b[i] -= a[6 * i + j] * b[j];
#pragma unroll
  for (int i = 0; i < 6; i++) { const double d = a[7 * i]; b[i] = (fabs(d) > 2.2250738585072014e-308) ? b[i] / d : 0.0; }
#pragma unroll
  for (int i = 5; i >= 0; i--)
#pragma unroll
    for (int j = i + 1; j < 6; j++) b[i] -= a[6 * j + i] * b[j];
  // undo the permutation: apply the recorded transpositions in reverse order
#pragma unroll
  for (int k = 5; k >= 0; k--) {
    const int p = piv[k];
    if (p != k) { const double u = b[k]; b[k] = b[p]; b[p] = u; }
  }
}

// [O3D] TransformVector6dToMatrix4d: R = Rz(x2) Ry(x1) Rx(x0), t = x[3..5]
__device__ __forceinline__ void vec6_to_mat4_dev(const double (&x)[6], double* T) {
  double sa, ca, sb, cb, sg, cgm;
  sincos(x[0], &sa, &ca); sincos(x[1], &sb, &cb); sincos(x[2], &sg, &cgm);
  T[0] = cgm * cb; T[1] = cgm * sb * sa - sg * ca; T[2] = cgm * sb * ca + sg * sa; T[3] = x[3];
  T[4] = sg * cb;  T[5] = sg * sb * sa + cgm * ca; T[6] = sg * sb * ca - cgm * sa; T[7] = x[4];
  T[8] = -sb;      T[9] = cb * sa;                 T[10] = cb * ca;                T[11] = x[5];
  T[12] = 0; T[13] = 0; T[14] = 0; T[15] = 1;
}

__device__ bool mat4_is_identity_dev(const double* T) {  // Eigen isIdentity(1e-12)
  const double prec = 1e-12;
  for (int i = 0; i < 4; i++)
    for (int j = 0; j < 4; j++) {
      const double v = T[4 * i + j];
      if (i == j) { if (!(fabs(v - 1.0) <= prec * fmin(fabs(v), 1.0))) return false; }
      else if (!(fabs(v) <= prec)) return false;
    }
  return true;
}

constexpr int icp_fixed_smem_doubles(int threads) { return ((threads / 32) * NACC + 2 * NACC + NACC + 16 + 16 + 8 + 42 + 1) & ~1; }   // even: what follows stays 16-byte aligned
constexpr int icp_fixed_smem_bytes(int threads) { return icp_fixed_smem_doubles(threads) * 8 + (int)sizeof(GridHeader) + 16 + 16; }   // + header + queue length + mbarrier
constexpr int ICP_BYTES_PER_POINT = 24 + 4 + 4 + 4 + 4;  // working point, neighbour slot / search state, phase-2 queue entry, certificate slack, search-list entry

// ---- contributions of one correspondence to the per-estimator sums ---------------------------------------------------------
// Every 32 points (one per lane; slot < 0 = no correspondence, contributes zeros) are reduced by a warp butterfly at once and lane 0
// adds the warp's sum to ITS warp's accumulator in shared memory (wacc, [NACC]).  LANE0 = true: called by lane 0 alone (phase 2,
// one point per warp), added directly.  No thread keeps accumulators in registers, and the summation order is fixed.
template <bool LANE0>
__device__ __forceinline__ void wadd(double* wacc, int k, double v, int lane) {
  if (LANE0) { wacc[k] += v; return; }
  v = warp_sum(v);
  if (lane == 0) wacc[k] += v;
}

// Warp sums of 32 values at once with the butterfly exchanges TRANSPOSED: at distance 16 the two halves of the warp split the values
// between them (a lane keeps the half it will finish and receives its partner's copy of that half), at distance 8 the quarters do,
// ... -- 16 + 8 + 4 + 2 + 1 = 31 exchanges instead of 32 x 5, and lane l ends up with the total of value l.  Every partial sum adds
// the same two operands as the plain butterfly at that distance (fp addition commutes), so each total is bit-identical to warp_sum.
// val(k): value k of the calling lane, evaluated on demand (keeps the live set at the 16 partial sums of the first stage).
template <class F>
__device__ __forceinline__ double warp_sum32_transposed(F val, int lane) {
  const unsigned FULL = 0xffffffffu;
  double a[16];
  {
    const bool up = (lane & 16) != 0;
#pragma unroll
    for (int k = 0; k < 16; k++) {
      const double lo = val(k), hi = val(k + 16);
      a[k] = (up ? hi : lo) + __shfl_xor_sync(FULL, up ? lo : hi, 16);
    }
  }
  double b[8];
  {
    const bool up = (lane & 8) != 0;
#pragma unroll
    for (int k = 0; k < 8; k++) b[k] = (up ? a[k + 8] : a[k]) + __shfl_xor_sync(FULL, up ? a[k] : a[k + 8], 8);
  }
  double c[4];
  {
    const bool up = (lane & 4) != 0;
#pragma unroll
    for (int k = 0; k < 4; k++) c[k] = (up ? b[k + 4] : b[k]) + __shfl_xor_sync(FULL, up ? b[k] : b[k + 4], 4);
  }
  double d[2];
  {
    const bool up = (lane & 2) != 0;
#pragma unroll
    for (int k = 0; k < 2; k++) d[k] = (up ? c[k + 2] : c[k]) + __shfl_xor_sync(FULL, up ? c[k] : c[k + 2], 2);
  }
  const bool up = (lane & 1) != 0;
  return (up ? d[1] : d[0]) + __shfl_xor_sync(FULL, up ? d[0] : d[1], 1);
}

// point-to-point ([O3D] TransformationEstimationPointToPoint = Eigen::umeyama): sums for the means and the cross moments, every
// coordinate taken relative to a reference point c known before the pass (the centre of the target grid's box, in shared memory).
// Raw moments E[t s^T] - mt ms^T cancel catastrophically far from the origin (a cloud 1e4 m out loses ~8 digits of the covariance);
// moments about a point inside the target's box cancel only at the scale of the clouds' spread.
//   acc[0..2] = sum (source - c), acc[3..5] = sum (target - c), acc[6 + 3a + b] = sum (target - c)_a * (source - c)_b
template <bool LANE0>
__device__ __forceinline__ void icp_contribute_p2p(double* wacc, const GridView& g, const double* c, int slot, double px, double py, double pz,
                                                   int lane) {
  const bool ok = slot >= 0;
  double4 q = make_double4(0, 0, 0, 0);
  if (ok) q = g.pts[slot];
  const double d2 = ok ? dist2_exact(px, py, pz, q.x, q.y, q.z) : 0.0;
  if (!ok) { px = 0; py = 0; pz = 0; }
  else { q.x -= c[0]; q.y -= c[1]; q.z -= c[2]; px -= c[0]; py -= c[1]; pz -= c[2]; }
  wadd<LANE0>(wacc, 0, px, lane); wadd<LANE0>(wacc, 1, py, lane); wadd<LANE0>(wacc, 2, pz, lane);
  wadd<LANE0>(wacc, 3, q.x, lane); wadd<LANE0>(wacc, 4, q.y, lane); wadd<LANE0>(wacc, 5, q.z, lane);
  wadd<LANE0>(wacc, 6, q.x * px, lane); wadd<LANE0>(wacc, 7, q.x * py, lane); wadd<LANE0>(wacc, 8, q.x * pz, lane);
  wadd<LANE0>(wacc, 9, q.y * px, lane); wadd<LANE0>(wacc, 10, q.y * py, lane); wadd<LANE0>(wacc, 11, q.y * pz, lane);
  wadd<LANE0>(wacc, 12, q.z * px, lane); wadd<LANE0>(wacc, 13, q.z * py, lane); wadd<LANE0>(wacc, 14, q.z * pz, lane);
  wadd<LANE0>(wacc, 27, d2, lane);
  wadd<LANE0>(wacc, 28, ok ? 1.0 : 0.0, lane);
}

// information matrix ([O3D] GetInformationMatrixFromPointClouds): first and second moments of the matched TARGET points
//   acc[0..2] = sum (x, y, z), acc[3..5] = sum (x2, y2, z2), acc[6..8] = sum (xy, xz, yz)
template <bool LANE0>
__device__ __forceinline__ void icp_contribute_info(double* wacc, const GridView& g, int slot, double px, double py, double pz, int lane) {
  const bool ok = slot >= 0;
  double4 q = make_double4(0, 0, 0, 0);
  if (ok) q = g.pts[slot];
  const double d2 = ok ? dist2_exact(px, py, pz, q.x, q.y, q.z) : 0.0;
  wadd<LANE0>(wacc, 0, q.x, lane); wadd<LANE0>(wacc, 1, q.y, lane); wadd<LANE0>(wacc, 2, q.z, lane);
  wadd<LANE0>(wacc, 3, q.x * q.x, lane); wadd<LANE0>(wacc, 4, q.y * q.y, lane); wadd<LANE0>(wacc, 5, q.z * q.z, lane);
  wadd<LANE0>(wacc, 6, q.x * q.y, lane); wadd<LANE0>(wacc, 7, q.x * q.z, lane); wadd<LANE0>(wacc, 8, q.y * q.z, lane);
  wadd<LANE0>(wacc, 27, d2, lane);
  wadd<LANE0>(wacc, 28, ok ? 1.0 : 0.0, lane);
}

// GTG = sum over matched target points of the three rank-one terms of [O3D]: rows (0,z,-y,1,0,0), (-z,0,x,0,1,0), (y,-x,0,0,0,1)
__device__ void info_from_moments(const double* t, double* G) {
  const double sx = t[0], sy = t[1], sz = t[2], xx = t[3], yy = t[4], zz = t[5], xy = t[6], xz = t[7], yz = t[8], n = t[28];
  const double M[6][6] = {{zz + yy, -xy, -xz, 0.0, -sz, sy}, {-xy, zz + xx, -yz, sz, 0.0, -sx}, {-xz, -yz, yy + xx, -sy, sx, 0.0},
                          {0.0, sz, -sy, n, 0.0, 0.0},       {-sz, 0.0, sx, 0.0, n, 0.0},       {sy, -sx, 0.0, 0.0, 0.0, n}};
  for (int a = 0; a < 6; a++)
    for (int b = 0; b < 6; b++) G[6 * a + b] = M[a][b];
}

// Eigen::umeyama without scaling from the accumulated moments (tot as filled by icp_contribute_p2p about the reference point c,
// tot[28] = n, c the reference point of the sums): sigma = E[(t - c)(s - c)^T] - (mt - c)(ms - c)^T, the means are c + E[. - c].
// Not inlined: one thread runs it once per evaluation, and inlined its SVD crowds the registers of the kernel's point loops.
__device__ __noinline__ void umeyama_from_moments(const double* tot, const double* c, double* Upd) {
  const double one_over_n = 1.0 / tot[28];
  double ms[3], mt[3], sigma[9];
  for (int a = 0; a < 3; a++) { ms[a] = tot[a] * one_over_n; mt[a] = tot[3 + a] * one_over_n; }
  for (int a = 0; a < 3; a++)
    for (int b = 0; b < 3; b++) sigma[3 * a + b] = tot[6 + 3 * a + b] * one_over_n - mt[a] * ms[b];
  for (int a = 0; a < 3; a++) { ms[a] += c[a]; mt[a] += c[a]; }
  double U[9], S[3], V[9];
  svd3_dev(sigma, U, S, V);
  const double sgn = det3_dev(U) * det3_dev(V) < 0 ? -1.0 : 1.0;
  for (int i = 0; i < 16; i++) Upd[i] = (i % 5 == 0) ? 1.0 : 0.0;
  for (int a = 0; a < 3; a++) {
    for (int b = 0; b < 3; b++) Upd[4 * a + b] = U[3 * a] * V[3 * b] + U[3 * a + 1] * V[3 * b + 1] + sgn * U[3 * a + 2] * V[3 * b + 2];
    Upd[4 * a + 3] = mt[a] - (Upd[4 * a] * ms[0] + Upd[4 * a + 1] * ms[1] + Upd[4 * a + 2] * ms[2]);
  }
}

// point-to-plane ([O3D] TransformationEstimationPointToPlane::ComputeTransformation -> ComputeJTJandJTr): r = (p - q) . n,
// J = [p x n ; n]
template <bool LANE0>
__device__ __forceinline__ void icp_contribute_plane(double* wacc, const GridView& g, int slot, double px, double py, double pz, int lane) {
  const bool ok = slot >= 0;
  double4 q = make_double4(0, 0, 0, 0), nn = make_double4(0, 0, 0, 0);
  if (ok) { q = g.pts[slot]; nn = target_normal(g, q); }
  const double d2 = ok ? dist2_exact(px, py, pz, q.x, q.y, q.z) : 0.0;
  const double r = (px - q.x) * nn.x + (py - q.y) * nn.y + (pz - q.z) * nn.z;   // zero normal for a lane without correspondence: all terms vanish
  double J[6];
  J[0] = py * nn.z - pz * nn.y; J[1] = pz * nn.x - px * nn.z; J[2] = px * nn.y - py * nn.x;
  J[3] = nn.x; J[4] = nn.y; J[5] = nn.z;
  const double cnt1 = ok ? 1.0 : 0.0;
  auto val = [&](int k) -> double {   // k is a compile-time constant at every call site (fully unrolled)
    // upper triangle of J^T J row by row: row a starts at 6a - a(a-1)/2
    if (k < 6) return J[0] * J[k];
    if (k < 11) return J[1] * J[k - 5];
    if (k < 15) return J[2] * J[k - 9];
    if (k < 18) return J[3] * J[k - 12];
    if (k < 20) return J[4] * J[k - 14];
    if (k < 21) return J[5] * J[5];
    if (k < 27) return J[k - 21] * r;
    if (k == 27) return d2;
    if (k == 28) return cnt1;
    return 0.0;
  };
  if (LANE0) {
#pragma unroll
    for (int k = 0; k < NACC; k++) wacc[k] += val(k);
  } else {
    const double tot = warp_sum32_transposed(val, lane);
    if (lane < NACC) wacc[lane] += tot;
  }
}

// ---- Generalized ICP ([O3D] pipelines/registration/GeneralizedICP.cpp) --------------------------------------------
// covariance of a point from its normal: Rx diag(eps, 1, 1) Rx^T with Rx = GetRotationFromE1ToX(n) (identity when
// e1 . n < -0.99), every product written out like the reference does
__device__ __forceinline__ void gicp_cov_from_normal(double nx, double ny, double nz, double eps, double (&C)[9]) {
  double Rx[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  if (!(nx < -0.99)) {
    const double v1 = -nz, v2 = ny;                       // v = e1 x n = (0, -nz, ny)
    const double sv[9] = {0, -v2, v1, v2, 0, -0.0, -v1, 0.0, 0};
    const double f = 1 / (1 + nx);
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
      for (int j = 0; j < 3; j++) {
        const double sv2 = sv[3 * i] * sv[j] + sv[3 * i + 1] * sv[3 + j] + sv[3 * i + 2] * sv[6 + j];
        Rx[3 * i + j] = (i == j ? 1.0 : 0.0) + sv[3 * i + j] + sv2 * f;
      }
  }
  double t[9];   // Rx * D
#pragma unroll
  for (int i = 0; i < 3; i++) { t[3 * i] = Rx[3 * i] * eps; t[3 * i + 1] = Rx[3 * i + 1]; t[3 * i + 2] = Rx[3 * i + 2]; }
#pragma unroll
  for (int i = 0; i < 3; i++)
#pragma unroll
    for (int j = 0; j < 3; j++) C[3 * i + j] = t[3 * i] * Rx[3 * j] + t[3 * i + 1] * Rx[3 * j + 1] + t[3 * i + 2] * Rx[3 * j + 2];
}

// one correspondence of TransformationEstimationForGeneralizedICP: M = Ct + R Cs0 R^T, J = M^-1/2 [-skew(p) | I],
// r = M^-1/2 (p - q); accumulated as J^T J = A^T M^-1 A and J^T r = A^T M^-1 d (the square root only appears squared)
template <bool LANE0>
__device__ __forceinline__ void icp_contribute_gicp(double* wacc, const GridView& g, int slot, double px, double py, double pz,
                                                    const double* __restrict__ R, const double* __restrict__ sn_ptr, double eps, int lane) {
  const bool ok = slot >= 0;
  // a lane without correspondence runs the algebra on a harmless stand-in (unit normals) and contributes with weight zero
  double4 q = make_double4(px, py, pz, 0), nt = make_double4(1, 0, 0, 0);
  double sn[3] = {1.0, 0.0, 0.0};
  if (ok) { q = g.pts[slot]; nt = target_normal(g, q); sn[0] = sn_ptr[0]; sn[1] = sn_ptr[1]; sn[2] = sn_ptr[2]; }
  const double wgt = ok ? 1.0 : 0.0;
  const double d2 = ok ? dist2_exact(px, py, pz, q.x, q.y, q.z) : 0.0;
  double Ct[9], Cs0[9], M[9];
  gicp_cov_from_normal(nt.x, nt.y, nt.z, eps, Ct);
  gicp_cov_from_normal(sn[0], sn[1], sn[2], eps, Cs0);
  {
    double t[9];   // R * Cs0, then (R Cs0) R^T   ([O3D] TransformCovariances)
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
      for (int j = 0; j < 3; j++) t[3 * i + j] = R[3 * i] * Cs0[j] + R[3 * i + 1] * Cs0[3 + j] + R[3 * i + 2] * Cs0[6 + j];
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
      for (int j = 0; j < 3; j++) M[3 * i + j] = Ct[3 * i + j] + (t[3 * i] * R[3 * j] + t[3 * i + 1] * R[3 * j + 1] + t[3 * i + 2] * R[3 * j + 2]);
  }
  double Mi[9];
  {
    const double a = M[0], b = M[1], c = M[2], d = M[3], e = M[4], f = M[5], gg = M[6], h = M[7], i = M[8];
    const double det = a * (e * i - f * h) - b * (d * i - f * gg) + c * (d * h - e * gg);
    const double id = 1.0 / det;
    Mi[0] = (e * i - f * h) * id; Mi[1] = (c * h - b * i) * id; Mi[2] = (b * f - c * e) * id;
    Mi[3] = (f * gg - d * i) * id; Mi[4] = (a * i - c * gg) * id; Mi[5] = (c * d - a * f) * id;
    Mi[6] = (d * h - e * gg) * id; Mi[7] = (b * gg - a * h) * id; Mi[8] = (a * e - b * d) * id;
  }
  const double dd[3] = {px - q.x, py - q.y, pz - q.z};
  const double A[18] = {0, pz, -py, 1, 0, 0, -pz, 0, px, 0, 1, 0, py, -px, 0, 0, 0, 1};
  double MA[18], Md[3];
#pragma unroll
  for (int r = 0; r < 3; r++) {
#pragma unroll
    for (int c = 0; c < 6; c++) MA[6 * r + c] = Mi[3 * r] * A[c] + Mi[3 * r + 1] * A[6 + c] + Mi[3 * r + 2] * A[12 + c];
    Md[r] = Mi[3 * r] * dd[0] + Mi[3 * r + 1] * dd[1] + Mi[3 * r + 2] * dd[2];
  }
  double v[NACC];
  {
    int k = 0;
#pragma unroll
    for (int a = 0; a < 6; a++)
#pragma unroll
      for (int b = a; b < 6; b++) v[k++] = wgt * (A[a] * MA[b] + A[6 + a] * MA[6 + b] + A[12 + a] * MA[12 + b]);
#pragma unroll
    for (int a = 0; a < 6; a++) v[21 + a] = wgt * (A[a] * Md[0] + A[6 + a] * Md[1] + A[12 + a] * Md[2]);
    v[27] = d2; v[28] = wgt;
  }
  if (LANE0) {
#pragma unroll
    for (int k = 0; k < NACC; k++) wacc[k] += v[k];
  } else {
    const double tot = warp_sum32_transposed([&](int k) -> double { return k < NACC ? v[k] : 0.0; }, lane);
    if (lane < NACC) wacc[lane] += tot;
  }
}

// `single` carries the problem by value (kernel parameter space) for the one-registration calls, so that no
// host->device copy -- and no implicit stream synchronisation of a pageable copy -- sits in front of the launch;
// batches pass an array.  dbg (optional): clock64 stamps of problem 0 / CTA 0 per evaluation {start, search, reduce, solve}.
// MODE selects what is compiled in, so that the headline point-to-plane path carries no code (registers, stack) of the others:
//   0 = point-to-plane only, 1 = point-to-point + information matrix (+ plane), 2 = generalized ICP,
//   3 = point-to-plane with search statistics (b2s_debug_icp_clocks): dbg[512 + 8 e + {0,1,2,3}] = candidates scanned in phase 1,
//       point evaluations, points queued for phase 2, candidates scanned in phase 2 -- per evaluation e < 32, whole cluster
template <int MODE>
__global__ void __launch_bounds__(icp_threads(MODE), 1) icp_kernel(const __grid_constant__ IcpProblem single,
                                                                   const IcpProblem* __restrict__ problems, int smem_pts_cap,
                                                                   long long* dbg) {
  pdl_wait();
  constexpr int THREADS = icp_threads(MODE);
  constexpr int WARPS = THREADS / 32;
  cg::cluster_group cluster = cg::this_cluster();
  const unsigned crank = cluster.block_rank();
  const unsigned csize = cluster.num_blocks();
  const IcpProblem& P = problems ? problems[blockIdx.y] : single;
  const bool dbg_on = dbg != nullptr && blockIdx.y == 0 && crank == 0 && threadIdx.x == 0;

  extern __shared__ __align__(16) unsigned char smem_raw[];
  double* s_wacc = reinterpret_cast<double*>(smem_raw); // [WARPS][NACC]  per-warp accumulators (lane 0 of the warp owns its row)
  double* s_part = s_wacc + WARPS * NACC;               // [2][NACC]  (read by the other CTAs through DSMEM)
  double* s_tot = s_part + 2 * NACC;                    // [NACC]
  double* s_U = s_tot + NACC;                           // [16] update of the current iteration
  double* s_T = s_U + 16;                               // [16] accumulated transformation
  double* s_misc = s_T + 16;                            // [0] prev fitness [1] prev rmse [2] done [3] apply [4..6] point-to-point reference point
  double* s_A = s_misc + 8;                             // [36 + 6] the 6x6 system of the solve
  GridHeader* s_g = reinterpret_cast<GridHeader*>(smem_raw + icp_fixed_smem_doubles(THREADS) * 8);
  int* s_qn = reinterpret_cast<int*>(s_g + 1);          // phase-2 queue length (16 bytes reserved)
  unsigned long long* s_bar = reinterpret_cast<unsigned long long*>(s_qn + 4);   // mbarrier of the bulk-async staging (16 bytes reserved)
  double* s_pts = reinterpret_cast<double*>(smem_raw + icp_fixed_smem_bytes(THREADS));    // 16-byte aligned
  int* s_prev = reinterpret_cast<int*>(s_pts + 3 * (size_t)smem_pts_cap);  // neighbour slot per point (state between the phases, warm start)
  int* s_queue = s_prev + smem_pts_cap;                                    // local indices of points left to phase 2
  // CERTIFICATES (slack[i], a distance).  Every evaluation moves point i by m_i = |U p - p|; a search result stays valid while the
  // accumulated motion is provably too small to change it:
  //   * no correspondence (state -1): slack = (distance to the nearest target) - r.  While the motion stays below it no target can
  //     have come within r (outliers at the map frontier would otherwise repeat the most expensive search of all, every evaluation);
  //   * a correspondence (state >= 0): slack = (lower bound of the distance to every other target) - (distance to the neighbour).
  //     While TWICE the motion stays below it the neighbour is still the unique nearest target: the evaluation costs one distance.
  // ICP converges geometrically, so after the first two or three evaluations almost every point is certified and the correspondence
  // search all but disappears.  Both tests are conservative (rounded against the certificate), never approximate.
  float* s_slack = reinterpret_cast<float*>(s_queue + smem_pts_cap);
  int* s_list = reinterpret_cast<int*>(s_slack + smem_pts_cap);   // points that need a search in this evaluation (s_qn[1] = how many)

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int n = *P.src_n;
  // The source cloud is dealt out in TILES of ICP_TILE consecutive points, tile t to CTA t % csize: the cloud is Morton-ordered, so
  // a contiguous split would hand whole regions (the sparse far range, the map frontier) to single CTAs and the cluster would wait
  // for the unluckiest one at every barrier; tiles keep the locality inside a warp and spread the regions over all CTAs.
  const int ntiles = (n + ICP_TILE - 1) / ICP_TILE;
  const int chunk = ((ntiles + (int)csize - 1) / (int)csize) * ICP_TILE;   // capacity, uniform over the cluster
  const int my_tiles = (int)crank < ntiles ? (ntiles - (int)crank + (int)csize - 1) / (int)csize : 0;
  const bool has_last = my_tiles > 0 && ((ntiles - 1) % (int)csize) == (int)crank;   // the (possibly partial) last tile is mine
  const int cnt = my_tiles * ICP_TILE - (has_last ? ntiles * ICP_TILE - n : 0);
  const bool in_smem = chunk <= smem_pts_cap;   // uniform over the cluster (phase 2 shares work across CTAs)
  // local index -> index in the source cloud (of CTA `r`), and -> index in the working arrays (local in shared memory, global otherwise)
  auto gidx_of = [csize](int i, int r) { return ((i / ICP_TILE) * (int)csize + r) * ICP_TILE + (i % ICP_TILE); };
  auto widx = [&](int i) { return in_smem ? i : gidx_of(i, (int)crank); };
  double* work = in_smem ? s_pts : P.work_xyz;
  // per-point state: >= -1 = slot of the correspondence (-1: none); <= -2 = queued for phase 2, -(slot + 3) = best seen so far
  int* prev = in_smem ? s_prev : P.work_prev;

  if (tid == 0) {
    *s_g = *P.ghdr;
    const double* init = P.init_dev ? P.init_dev : P.init;
    for (int i = 0; i < 16; i++) { s_T[i] = init[i]; s_U[i] = init[i]; }
    s_misc[0] = 0.0; s_misc[1] = 0.0; s_misc[2] = 0.0;
    s_misc[3] = mat4_is_identity_dev(init) ? 0.0 : 1.0;  // [O3D]: if (!init.isIdentity()) pcd.Transform(init)
    for (int a = 0; a < 3; a++) s_misc[4 + a] = s_g->origin[a] + 0.5 * (double)s_g->dims[a] * s_g->cell;   // centre of the target's box
    s_qn[0] = 0; s_qn[1] = 0;
    if (in_smem) { mbar_init(s_bar, 1); mbar_fence_init(); }
  }
  for (int i = tid; i < WARPS * NACC; i += THREADS) s_wacc[i] = 0.0;
  __syncthreads();
  {  // stage this CTA's tiles of the source cloud
    if (in_smem) {
      // one elected thread hands every full tile to the bulk-async copy engine (cp.async.bulk global -> shared, 24 * ICP_TILE bytes
      // each: a multiple of 16 at a 16-byte aligned offset); completion is counted in bytes on the mbarrier
      const int full_tiles = my_tiles - ((has_last && (n % ICP_TILE) != 0) ? 1 : 0);
      const uint32_t total = (uint32_t)full_tiles * (24u * ICP_TILE);
      if (tid == 0 && total > 0) {
        mbar_arrive_expect_tx(s_bar, total);
        for (int t = 0; t < full_tiles; t++)
          bulk_copy_g2s(reinterpret_cast<char*>(s_pts) + (size_t)t * (24 * ICP_TILE),
                        reinterpret_cast<const char*>(P.src_xyz) + (size_t)(t * (int)csize + (int)crank) * (24 * ICP_TILE), 24u * ICP_TILE, s_bar);
      }
      for (int i = full_tiles * ICP_TILE + tid; i < cnt; i += THREADS) {   // the partial last tile
        const size_t gi = (size_t)gidx_of(i, (int)crank);
        s_pts[3 * i] = P.src_xyz[3 * gi]; s_pts[3 * i + 1] = P.src_xyz[3 * gi + 1]; s_pts[3 * i + 2] = P.src_xyz[3 * gi + 2];
      }
      if (total > 0) mbar_wait_parity(s_bar, 0);
    } else {
      for (int i = tid; i < cnt; i += THREADS) {
        const size_t gi = (size_t)gidx_of(i, (int)crank);
        work[3 * gi] = P.src_xyz[3 * gi]; work[3 * gi + 1] = P.src_xyz[3 * gi + 1]; work[3 * gi + 2] = P.src_xyz[3 * gi + 2];
      }
    }
    for (int i = tid; i < cnt; i += THREADS) { prev[widx(i)] = -1; if (in_smem) s_slack[i] = 0.0f; }
  }
  __syncthreads();

  GridView g;
  g.ox = s_g->origin[0]; g.oy = s_g->origin[1]; g.oz = s_g->origin[2];
  g.cell = s_g->cell; g.inv = s_g->inv_cell; g.eps = 1e-9 * s_g->cell;
  g.nx = s_g->dims[0]; g.ny = s_g->dims[1]; g.nz = s_g->dims[2];
  g.cs = P.cell_start;
  g.pts = reinterpret_cast<const double4*>(P.tgt_pts);
  g.nrm = P.tgt_nrm;
  const double r2 = P.max_corr * P.max_corr;
  const int max_iter = P.max_iter;
  constexpr bool GICP = MODE == 2;
  constexpr bool COUNT = MODE == 3;
  int n_scanned1 = 0, n_evals1 = 0, n_queued = 0, n_scanned2 = 0;
  const bool p2p = MODE == 1 && P.estimator == B2S_REG_POINT_TO_POINT;
  const bool corr_only = MODE == 1 && P.estimator == EST_CORRESPONDENCES;
  const bool info = MODE == 1 && (P.estimator == EST_INFORMATION || corr_only);   // one evaluation, output = 6x6 information matrix
  double* wacc = s_wacc + warp * NACC;

  for (int e = 0;; ++e) {
    if (dbg_on && e < 64) dbg[4 * e] = clock64();
    const bool bal_on = dbg != nullptr && blockIdx.y == 0 && tid == 0 && e < 8;
    long long t_start = 0;
    if (bal_on) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_start));
    const bool apply = s_misc[3] != 0.0;

    // ---- phase 1a: move the points, settle what the certificates settle, search the rest ----
    // Sweep A touches every point: apply the update, then (certificates) decide whether the previous answer still stands.  Points
    // that need a search are COMPACTED into a list (warp-aggregated append), so that sweep B runs the search with full warps: in the
    // later evaluations a few percent of the points search, and scattered over all warps they would make every warp walk the whole
    // search path (and wait for its L2 round trips) for one or two live lanes.
    const unsigned lt_mask = (1u << lane) - 1u;
    for (int base = warp * 32; base < cnt; base += THREADS) {
      const int i = base + lane;
      bool need = false;
      if (i < cnt) {
        const int wi = widx(i);
        double px = work[3 * wi], py = work[3 * wi + 1], pz = work[3 * wi + 2];
        double moved = 0.0;
        if (apply) {  // [O3D] TransformPoints with w == 1 exactly for a rigid update; same association as Eigen's product
          const double x = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(s_U[0], px), __dmul_rn(s_U[1], py)), __dmul_rn(s_U[2], pz)), s_U[3]);
          const double y = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(s_U[4], px), __dmul_rn(s_U[5], py)), __dmul_rn(s_U[6], pz)), s_U[7]);
          const double z = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(s_U[8], px), __dmul_rn(s_U[9], py)), __dmul_rn(s_U[10], pz)), s_U[11]);
          moved = sqrt((x - px) * (x - px) + (y - py) * (y - py) + (z - pz) * (z - pz));
          px = x; py = y; pz = z;
          work[3 * wi] = px; work[3 * wi + 1] = py; work[3 * wi + 2] = pz;
        }
        need = true;
        if (in_smem) {
          const int hint = prev[wi];
          if (hint == -1) {   // no correspondence last time: still provably none?
            const float left = s_slack[i] - (float)(moved * (1.0 + 1e-6)) - 1e-7f;   // float rounding only ever shortens the slack
            s_slack[i] = left > 0.0f ? left : 0.0f;
            if (left > 0.0f) need = false;   // prev[i] stays -1
          } else if (hint >= 0) {   // a correspondence last time: still provably the same target?
            // slack = (lower bound of the distance to every OTHER target) - (distance to the neighbour) when it was last searched.  A
            // move by m brings the neighbour at most m further and every other target at most m closer: while 2 m stays below the
            // slack the neighbour is still the unique nearest target, and the search is replaced by one distance evaluation.
            const float left = s_slack[i] - (float)(2.0 * moved * (1.0 + 1e-6)) - 1e-7f;
            if (left > 0.0f) {
              const double4 q = g.pts[hint];
              const double d = dist2_exact(px, py, pz, q.x, q.y, q.z);
              if (d < r2) {
                s_slack[i] = left;
              } else {   // the nearest target has left the correspondence radius: nothing is within it (and stays so for sqrt(d) - r)
                prev[wi] = -1;
                s_slack[i] = (float)fmax((sqrt(d) - P.max_corr) * (1.0 - 1e-6) - 1e-7, 0.0);
              }
              need = false;
            }
          }
          if (COUNT && !need) n_evals1++;
        }
      }
      if (in_smem) {
        const unsigned m = __ballot_sync(0xffffffffu, need);
        if (m) {
          int pos = 0;
          if (lane == 0) pos = atomicAdd(&s_qn[1], __popc(m));
          pos = __shfl_sync(0xffffffffu, pos, 0);
          if (need) s_list[pos + __popc(m & lt_mask)] = i;
        }
      }
    }
    __syncthreads();
    // Sweep B: one thread per listed point (without shared-memory residency there is no list: every point, no certificates)
    const int n_search = in_smem ? s_qn[1] : cnt;
    for (int t = tid; t < n_search; t += THREADS) {
      const int i = in_smem ? s_list[t] : t;
      const int wi = widx(i);
      const double px = work[3 * wi], py = work[3 * wi + 1], pz = work[3 * wi + 2];
      const int hint = prev[wi];
      NNState st;
      bool done = nn_phase1(g, px, py, pz, r2, hint >= 0 ? hint : -1, st);
      if (!done && !in_smem) {  // no queue for clouds that overflow shared memory: finish serially
        if (st.bslot >= 0) st.bidx = (int)__double_as_longlong(g.pts[st.bslot].w);   // the box walk does not track it
        int cx, cy, cz;
        cell_of(g, px, py, pz, cx, cy, cz);
        for (int R = ICP_R1 + 1;; ++R) {
          const int z0 = max(cz - R, 0), z1 = min(cz + R, g.nz - 1), y0 = max(cy - R, 0), y1 = min(cy + R, g.ny - 1);
          for (int z = z0; z <= z1; ++z)
            for (int y = y0; y <= y1; ++y) nn_scan_row(g, px, py, pz, cx, cy, cz, R, y, z, st);
          const double bound = ring_bound(g, px, py, pz, cx, cy, cz, R);
          if (bound == INFINITY || bound * bound > st.best) break;
        }
        done = true;
      }
      prev[wi] = done ? st.bslot : -(st.bslot + 3);
      if (in_smem) {   // gap certificate of the answer: runner-up among the cells walked, or the walked block's nearest face
        float sl = 0.0f;
        if (done && st.bslot >= 0) sl = (float)fmax((fmin(sqrt(st.second), st.gb) - sqrt(st.best)) * (1.0 - 1e-6) - 1e-7, 0.0);
        s_slack[i] = sl;
      }
      if (COUNT) { n_scanned1 += st.scanned; n_evals1++; n_queued += done ? 0 : 1; }
      if (!done) s_queue[atomicAdd(s_qn, 1)] = i;
    }
    __syncthreads();
    // ---- phase 1b: the sums, 32 points per warp step, every term warp-reduced into the warp's shared-memory accumulator ----
    double RT[9];   // GICP: rotation of the accumulated transformation = what [O3D] has applied to the source covariances so far
    if (GICP) {
      const bool moved = e > 0 || apply;   // identity init is not applied at all (isIdentity), like the covariance transform
#pragma unroll
      for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++) RT[3 * i + j] = moved ? s_T[4 * i + j] : (i == j ? 1.0 : 0.0);
    }
    {
      for (int base = warp * 32; base < cnt; base += THREADS) {
        const int i = base + lane;
        int slot = -1;
        double px = 0.0, py = 0.0, pz = 0.0;
        if (i < cnt) { const int wi = widx(i); slot = prev[wi]; px = work[3 * wi]; py = work[3 * wi + 1]; pz = work[3 * wi + 2]; }   // queued points (<= -2) are phase 2's
        if (GICP) icp_contribute_gicp<false>(wacc, g, slot, px, py, pz, RT, P.src_nrm + 3 * (size_t)gidx_of(i < cnt ? i : 0, (int)crank), P.gicp_eps, lane);
        else if (p2p) icp_contribute_p2p<false>(wacc, g, s_misc + 4, slot, px, py, pz, lane);
        else if (info) icp_contribute_info<false>(wacc, g, slot, px, py, pz, lane);
        else icp_contribute_plane<false>(wacc, g, slot, px, py, pz, lane);
      }
    }
    long long t_p1 = 0;
    if (bal_on) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_p1));
    // ---- phase 2: one warp per point that needs more than phase 1's box ----
    // The unresolved points cluster spatially (map frontier), i.e. in one or two CTAs of the Morton-ordered source:
    // the queues of ALL CTAs are therefore drained by ALL warps of the cluster, through distributed shared memory.
    // The sums are cluster totals anyway, so a point may be accumulated by any CTA.
    if (in_smem) {
      cluster.sync();  // every queue is complete
      // queue lengths of the cluster's CTAs: lane r reads CTA r's counter, the warp scans them (no per-thread offset table)
      int qinc = lane < (int)csize ? *cluster.map_shared_rank(s_qn, lane) : 0;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, qinc, o); if (lane >= o) qinc += v; }
      const int qtotal = __shfl_sync(0xffffffffu, qinc, 31);
      for (int gi = (int)crank * WARPS + warp; gi < qtotal; gi += (int)csize * WARPS) {
        const unsigned before = __ballot_sync(0xffffffffu, qinc <= gi);   // CTAs whose queues end at or before entry gi (a prefix of the lanes)
        const int r = __popc(before);
        const int li = gi - (r > 0 ? __shfl_sync(0xffffffffu, qinc, r - 1) : 0);
        const int i = cluster.map_shared_rank(s_queue, r)[li];
        const double* rw = cluster.map_shared_rank(s_pts, r);
        int* rp = cluster.map_shared_rank(s_prev, r);
        const double px = rw[3 * i], py = rw[3 * i + 1], pz = rw[3 * i + 2];
        NNState st;
        st.best = r2; st.second = INFINITY; st.gb = 0.0; st.bidx = 0x7fffffff; st.bslot = -1; st.scanned = 0;
        const int hs = -rp[i] - 3;  // best of the box query (or the seed), -1 when nothing was in range
        if (hs >= 0) {
          const double4 p = g.pts[hs];
          st.best = dist2_exact(px, py, pz, p.x, p.y, p.z); st.bidx = (int)__double_as_longlong(p.w); st.bslot = hs;
          if (!(st.best < r2)) { st.best = r2; st.bidx = 0x7fffffff; st.bslot = -1; }
        }
        // The ball searched completely reaches a margin beyond the seed distance (beyond r without a seed).  What lies in the margin
        // is never the answer, but it is what the certificates are made of: the runner-up bounds how far the point may move before
        // the neighbour can change, the nearest target beyond r how far before a point without correspondence can get one.
        const double margin = 0.25 * g.cell;
        const bool unseeded = st.bslot < 0;
        const double rc = (unseeded ? P.max_corr : sqrt(st.best)) + margin;
        if (unseeded) st.best = rc * rc;
        nn_phase2_warp(g, px, py, pz, rc * rc, st);
        if (COUNT) n_scanned2 += st.scanned;
        float sl;
        if (unseeded && st.bslot >= 0 && !(st.best < r2)) {   // nearest target lies in the margin shell: none within r, slack = distance - r
          sl = (float)fmax((sqrt(st.best) - P.max_corr) * (1.0 - 1e-6) - 1e-7, 0.0);
          st.bslot = -1;
        } else if (unseeded && st.bslot < 0) {
          sl = (float)(margin * (1.0 - 1e-6));
        } else {   // a correspondence: gap to the runner-up, or to the edge of the searched ball
          sl = (float)fmax((fmin(sqrt(st.second), rc) - sqrt(st.best)) * (1.0 - 1e-6) - 1e-7, 0.0);
        }
        if (lane == 0) cluster.map_shared_rank(s_slack, r)[i] = sl;
        if (lane == 0) {
          rp[i] = st.bslot;
          if (st.bslot >= 0) {
            if (GICP) icp_contribute_gicp<true>(wacc, g, st.bslot, px, py, pz, RT, P.src_nrm + 3 * (size_t)gidx_of(i, r), P.gicp_eps, 0);
            else if (p2p) icp_contribute_p2p<true>(wacc, g, s_misc + 4, st.bslot, px, py, pz, 0);
            else if (info) icp_contribute_info<true>(wacc, g, st.bslot, px, py, pz, 0);
            else icp_contribute_plane<true>(wacc, g, st.bslot, px, py, pz, 0);
          }
        }
      }
    }
    if (COUNT && dbg != nullptr && blockIdx.y == 0 && e < 32) {
      const int a = warp_sum_i(n_scanned1), b = warp_sum_i(n_evals1), c = warp_sum_i(n_queued), d = warp_sum_i(n_scanned2);
      if (lane == 0) {
        atomicAdd(reinterpret_cast<unsigned long long*>(dbg) + 512 + 8 * e + 0, (unsigned long long)a);
        atomicAdd(reinterpret_cast<unsigned long long*>(dbg) + 512 + 8 * e + 1, (unsigned long long)b);
        atomicAdd(reinterpret_cast<unsigned long long*>(dbg) + 512 + 8 * e + 2, (unsigned long long)c);
        atomicAdd(reinterpret_cast<unsigned long long*>(dbg) + 512 + 8 * e + 3, (unsigned long long)d);
      }
      n_scanned1 = n_evals1 = n_queued = n_scanned2 = 0;
    }
    if (dbg_on && e < 64) dbg[4 * e + 1] = clock64();
    if (dbg != nullptr && blockIdx.y == 0 && e < 8 && crank < 8) {   // per-CTA balance: {phase-1 end, phase-2 end (all warps), queue length, points}
      __syncthreads();
      if (tid == 0) {
        long long t_p2;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_p2));
        long long* d = dbg + 256 + (e * 8 + (int)crank) * 4;
        d[0] = t_p1 - t_start; d[1] = t_p2 - t_p1; d[2] = *s_qn; d[3] = cnt;   // ns, ns, queue length, points
      }
    }
    // per-warp accumulators -> CTA partial (fixed order => run-to-run deterministic up to who drained which phase-2 entry)
    __syncthreads();
    const int buf = e & 1;
    if (tid < NACC) {
      double v = 0.0;
      for (int w = 0; w < WARPS; w++) { v += s_wacc[w * NACC + tid]; s_wacc[w * NACC + tid] = 0.0; }
      s_part[buf * NACC + tid] = v;
    }
    cluster.sync();
    if (tid == 0) { s_qn[0] = 0; s_qn[1] = 0; }   // only after the barrier: peers read this queue during their phase 2
    if (tid < NACC) {
      double v = 0.0;
      for (unsigned r = 0; r < csize; r++) {
        const double* rp = cluster.map_shared_rank(s_part, r);
        v += rp[buf * NACC + tid];
      }
      s_tot[tid] = v;
    }
    __syncthreads();
    if (dbg_on && e < 64) dbg[4 * e + 2] = clock64();
    if (tid == 0) {
      const double c = s_tot[28];
      const double fit = (c > 0.0 && n > 0) ? c / (double)n : 0.0;
      const double rmse = c > 0.0 ? sqrt(s_tot[27] / c) : 0.0;
      bool done = false;
      if (e > 0 && fabs(s_misc[0] - fit) < P.rel_fitness && fabs(s_misc[1] - rmse) < P.rel_rmse) done = true;
      if (e >= max_iter) done = true;
      if (info) {
        done = true;
        if (crank == 0 && P.info_out) info_from_moments(s_tot, P.info_out);
      }
      if (!done) {
        double Upd[16];
        if (c > 0.0 && p2p) {
          umeyama_from_moments(s_tot, s_misc + 4, Upd);
        } else if (c > 0.0) {
          double x[6];
          {
            int k = 0;
#pragma unroll
            for (int a = 0; a < 6; a++)
#pragma unroll
              for (int bb = a; bb < 6; bb++) { s_A[6 * a + bb] = s_tot[k]; s_A[6 * bb + a] = s_tot[k]; k++; }
          }
#pragma unroll
          for (int a = 0; a < 6; a++) s_A[36 + a] = -s_tot[21 + a];
          ldlt6_solve_smem(s_A, s_A + 36);
#pragma unroll
          for (int a = 0; a < 6; a++) x[a] = s_A[36 + a];
          vec6_to_mat4_dev(x, Upd);
        } else {  // [O3D] ComputeTransformation: corres.empty() -> Identity
#pragma unroll
          for (int i = 0; i < 16; i++) Upd[i] = (i % 5 == 0) ? 1.0 : 0.0;
        }
        double Tn[16];
#pragma unroll
        for (int i = 0; i < 4; i++)
#pragma unroll
          for (int j = 0; j < 4; j++) {
            double s = 0;
#pragma unroll
            for (int k = 0; k < 4; k++) s += Upd[4 * i + k] * s_T[4 * k + j];
            Tn[4 * i + j] = s;
          }
#pragma unroll
        for (int i = 0; i < 16; i++) { s_T[i] = Tn[i]; s_U[i] = Upd[i]; }
        s_misc[0] = fit; s_misc[1] = rmse; s_misc[3] = 1.0;
      } else {
        s_misc[2] = 1.0;
        if (crank == 0) {
          b2s_result* out = P.out;
          for (int i = 0; i < 16; i++) out->T[i] = s_T[i];
          out->fitness = fit; out->inlier_rmse = rmse; out->n_corr = (int32_t)c; out->iters = e;
        }
      }
    }
    if (dbg_on && e < 64) dbg[4 * e + 3] = clock64();
    __syncthreads();
    if (s_misc[2] != 0.0) {
      // correspondence_set_ of the final evaluation: every CTA reports its own chunk (phase 2 wrote its results into the owners'
      // per-point state before the cluster barrier above)
      if (MODE == 1 && P.corr_index != nullptr) {
        for (int i = tid; i < cnt; i += THREADS) {
          const int wi = widx(i);
          const int sl = prev[wi];
          int oi = -1; double d2 = -1.0;
          if (sl >= 0) {
            const double4 q = g.pts[sl];
            oi = (int)__double_as_longlong(q.w);
            d2 = dist2_exact(work[3 * wi], work[3 * wi + 1], work[3 * wi + 2], q.x, q.y, q.z);
          }
          const int gi = gidx_of(i, (int)crank);
          P.corr_index[gi] = oi;
          if (P.corr_d2) P.corr_d2[gi] = d2;
        }
      }
      break;
    }
  }
  cluster.sync();  // no CTA may exit while a peer can still read its shared memory
}

constexpr int ICP_DYN_SMEM = 200 * 1024;

static size_t icp_chunk_points(size_t n, int csize) {   // per-CTA capacity in points, as icp_kernel computes it
  const size_t ntiles = (n + ICP_TILE - 1) / ICP_TILE;
  return ((ntiles + (size_t)csize - 1) / (size_t)csize) * ICP_TILE;
}

// the opt-in attributes are per DEVICE (a process may hold handles on several GPUs): one flag per device, set under a lock
static std::mutex g_icp_attr_mu;
static bool g_icp_attr_set[64] = {false};

static int icp_max_cluster(const b2s_handle* h) {   // 16 spreads one registration over 16 SMs (non-portable cluster size)
  static const int env = getenv("B2S_ICP_MAX_CLUSTER") ? atoi(getenv("B2S_ICP_MAX_CLUSTER")) : 0;
  const int v = h->cfg.icp_cluster_ctas > 0 ? h->cfg.icp_cluster_ctas : (env > 0 ? env : 8);
  return v >= 16 ? 16 : (v >= 8 ? 8 : (v >= 4 ? 4 : (v >= 2 ? 2 : 1)));
}

template <int MODE>
static cudaError_t icp_set_attrs() {
  cudaError_t e = cudaFuncSetAttribute(icp_kernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, ICP_DYN_SMEM);
  if (e != cudaSuccess) return e;
  return cudaFuncSetAttribute(icp_kernel<MODE>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
}

int32_t icp_launch(b2s_handle* h, const IcpProblem* single_host, const IcpProblem* problems_dev, int n_problems, size_t max_src_points,
                   int batch_estimator) {
  if (n_problems <= 0) return B2S_OK;
  IcpProblem single;
  memset(&single, 0, sizeof(single));
  if (single_host) { single = *single_host; problems_dev = nullptr; n_problems = 1; }
  {
    std::lock_guard<std::mutex> lk(g_icp_attr_mu);
    const int d = h->device >= 0 && h->device < 64 ? h->device : 0;
    if (!g_icp_attr_set[d]) {
      B2S_CUDA(icp_set_attrs<0>());
      B2S_CUDA(icp_set_attrs<1>());
      B2S_CUDA(icp_set_attrs<2>());
      B2S_CUDA(icp_set_attrs<3>());
      g_icp_attr_set[d] = true;
    }
  }
  const int estimator = single_host ? single_host->estimator : (batch_estimator >= 0 ? batch_estimator : h->cfg.icp.reg_type);   // uniform over a batch
  int csize = 1;
  const int cmax = icp_max_cluster(h);
  long long* const dbg = h->icp_dbg.as<long long>();
  const int mode = estimator == B2S_REG_GENERALIZED ? 2 : (estimator == B2S_REG_POINT_TO_PLANE ? (dbg ? 3 : 0) : 1);
  const int threads = icp_threads(mode);
  while (csize < cmax && (size_t)csize * threads < max_src_points) csize *= 2;
  const int fixed = icp_fixed_smem_bytes(threads);
  {
    // a batch that already fills the GPU is served better by small clusters (one CTA per SM is resident either way, and
    // every evaluation pays its barriers and reduction once per cluster): shrink while the chunk still fits shared memory
    const size_t smem_pts = (size_t)((ICP_DYN_SMEM - fixed) / ICP_BYTES_PER_POINT) - 64;
    static const int forced = getenv("B2S_ICP_BATCH_CSIZE") ? atoi(getenv("B2S_ICP_BATCH_CSIZE")) : 0;
    if (n_problems > 1 && forced > 0) csize = forced;
    else while (csize > 1 && (size_t)n_problems * (size_t)csize > 2 * (size_t)device_sms() && icp_chunk_points(max_src_points, csize / 2) <= smem_pts) csize /= 2;
  }
  // shared memory is sized for THIS launch's chunk only: whatever is not claimed stays L1, and the candidate gathers of
  // neighbouring queries hit the same lines (4 target points per 128-byte line)
  int pts_cap = (ICP_DYN_SMEM - fixed) / ICP_BYTES_PER_POINT;
  {
    const size_t want = icp_chunk_points(max_src_points, csize) + 64;   // the kernel's capacity per CTA
    if (want < (size_t)pts_cap) pts_cap = (int)want;
  }
  const int dyn_smem = fixed + pts_cap * ICP_BYTES_PER_POINT;
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(csize, n_problems, 1);
  cfg.blockDim = dim3(threads, 1, 1);
  cfg.dynamicSmemBytes = (size_t)dyn_smem;
  cfg.stream = h->stream;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = csize; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
  attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;   // see pdl_wait (common.cuh)
  attr[1].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 2 : 1;
  ProfScope prof(h, PK_ICP);
  if (estimator == B2S_REG_GENERALIZED) B2S_CUDA(cudaLaunchKernelEx(&cfg, icp_kernel<2>, single, problems_dev, pts_cap, dbg));
  else if (estimator == B2S_REG_POINT_TO_PLANE && dbg) B2S_CUDA(cudaLaunchKernelEx(&cfg, icp_kernel<3>, single, problems_dev, pts_cap, dbg));
  else if (estimator == B2S_REG_POINT_TO_PLANE) B2S_CUDA(cudaLaunchKernelEx(&cfg, icp_kernel<0>, single, problems_dev, pts_cap, dbg));
  else B2S_CUDA(cudaLaunchKernelEx(&cfg, icp_kernel<1>, single, problems_dev, pts_cap, dbg));
  h->launches++;
  return B2S_OK;
}

}  // namespace b2s
