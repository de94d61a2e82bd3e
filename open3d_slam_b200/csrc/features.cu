// features.cu -- K-fpfh: the feature half of Submap::computeFeatures (core/src/Submap.cpp:244) =
// [O3D] ComputeFPFHFeature(cloud, KDTreeSearchParamHybrid(radius, knn)) (pipelines/registration/Feature.cpp).
//
// Three kernels over a K-index grid of the cloud (grid_index.cu):
//   fpfh_knn_kernel   one WARP per query: the exact hybrid search (k nearest with d2 < r2, ties -> lower index, ascending
//                     (d2, index)) by the warp ring walk grid_knn_walk (common.cuh), the k best kept as a sorted list of up to
//                     B2S_FEATURE_MAX_KNN entries, FK_PER_LANE per lane.  Each neighbour list (index + d2) is written once and
//                     read by both passes.
//   fpfh_spfh_kernel  one thread per point: SPFH.  The first list entry is skipped as "self" (kept literally, also when a
//                     coincident lower-index point takes that place); bins are counted, then every bin is the count-fold sum
//                     of hist_incr -- the reference's sequential `+= hist_incr`, whose value depends on the count only.
//   fpfh_kernel       one thread per (point, 11-bin block): sums spfh[nb] / d2 in neighbour order (d2 == 0 skipped),
//                     normalises the block to 100 and adds the point's own SPFH.
// The library builds with -fmad=false, so every expression is evaluated as written, like the fp64 CPU restatement; a row can
// differ only where the device's atan2 / acos and the host libm put a pair feature on different sides of a bin boundary.
#include <algorithm>

#include "common.cuh"

namespace b2s {

constexpr int FK_THREADS = 128;
constexpr int FK_PER_LANE = B2S_FEATURE_MAX_KNN / 32;
static_assert(B2S_FEATURE_MAX_KNN % 32 == 0, "the k-best list is FK_PER_LANE entries per lane");

// one WARP per query: the ring walk grid_knn_walk (common.cuh) with FK_PER_LANE list entries per lane
__global__ void __launch_bounds__(FK_THREADS) fpfh_knn_kernel(const GridHeader* __restrict__ hdr, const int32_t* __restrict__ cs,
                                                              const double4* __restrict__ pts, int knn, double radius,
                                                              int32_t* __restrict__ nb_idx, double* __restrict__ nb_d2,
                                                              int32_t* __restrict__ nb_cnt) {
  pdl_wait();
  __shared__ GridHeader g;
  if (threadIdx.x == 0) g = *hdr;
  __syncthreads();
  const unsigned FULL = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const int warps_total = gridDim.x * (FK_THREADS / 32);
  const double r2 = radius * radius;
  for (int w = blockIdx.x * (FK_THREADS / 32) + (threadIdx.x >> 5); w < g.n; w += warps_total) {
    const double4 qp = pts[w];
    const int qi = (int)__double_as_longlong(qp.w);
    double ed[FK_PER_LANE]; int ei[FK_PER_LANE], es[FK_PER_LANE];   // es: unused, the lists hold original indices
    grid_knn_walk<FK_PER_LANE, false>(g, cs, pts, qp.x, qp.y, qp.z, knn, r2, ed, ei, es);
    int kk = 0;
#pragma unroll
    for (int m = 0; m < FK_PER_LANE; ++m) {
      const int p = m * 32 + lane;
      const bool valid = p < knn && ei[m] != 0x7fffffff;
      kk += __popc(__ballot_sync(FULL, valid));
      if (valid) { nb_idx[(size_t)qi * knn + p] = ei[m]; nb_d2[(size_t)qi * knn + p] = ed[m]; }
    }
    if (lane == 0) nb_cnt[qi] = kk;
  }
}

// [O3D] ComputePairFeatures, only the three angular features the histogram uses
__device__ __forceinline__ void pair_features(const double* p1, const double* n1, const double* p2, const double* n2, double f[3]) {
  double dp[3] = {p2[0] - p1[0], p2[1] - p1[1], p2[2] - p1[2]};
  const double len = sqrt(dp[0] * dp[0] + dp[1] * dp[1] + dp[2] * dp[2]);
  f[0] = f[1] = f[2] = 0.0;
  if (len == 0.0) return;
  const double* a = n1; const double* b = n2;
  const double angle1 = (n1[0] * dp[0] + n1[1] * dp[1] + n1[2] * dp[2]) / len;
  const double angle2 = (n2[0] * dp[0] + n2[1] * dp[1] + n2[2] * dp[2]) / len;
  double f2;
  if (acos(fabs(angle1)) > acos(fabs(angle2))) {
    a = n2; b = n1;
    dp[0] *= -1.0; dp[1] *= -1.0; dp[2] *= -1.0;
    f2 = -angle2;
  } else {
    f2 = angle1;
  }
  double v[3] = {dp[1] * a[2] - dp[2] * a[1], dp[2] * a[0] - dp[0] * a[2], dp[0] * a[1] - dp[1] * a[0]};
  const double vn = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
  if (vn == 0.0) return;
  v[0] /= vn; v[1] /= vn; v[2] /= vn;
  const double w[3] = {a[1] * v[2] - a[2] * v[1], a[2] * v[0] - a[0] * v[2], a[0] * v[1] - a[1] * v[0]};
  f[2] = f2;
  f[1] = v[0] * b[0] + v[1] * b[1] + v[2] * b[2];
  f[0] = atan2(w[0] * b[0] + w[1] * b[1] + w[2] * b[2], a[0] * b[0] + a[1] * b[1] + a[2] * b[2]);
}

__device__ __forceinline__ int fpfh_bin(double t) {
  int h = (int)floor(t);
  if (h < 0) h = 0;
  if (h >= 11) h = 10;
  return h;
}

__global__ void __launch_bounds__(FK_THREADS) fpfh_spfh_kernel(const double* __restrict__ xyz, const double* __restrict__ nrm,
                                                               const int32_t* __restrict__ d_n, int knn, const int32_t* __restrict__ nb_idx,
                                                               const int32_t* __restrict__ nb_cnt, double* __restrict__ spfh) {
  pdl_wait();
  __shared__ unsigned char hist[FK_THREADS][33];   // per-thread bin counts (at most B2S_FEATURE_MAX_KNN - 1 each)
  unsigned char* hc = hist[threadIdx.x];
  const int n = *d_n;
  const double pi = 3.14159265358979323846;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    for (int b = 0; b < 33; ++b) hc[b] = 0;
    const int cnt = nb_cnt[i];
    double hist_incr = 0.0;
    if (cnt > 1) {
      const double p1[3] = {xyz[3 * (size_t)i], xyz[3 * (size_t)i + 1], xyz[3 * (size_t)i + 2]};
      const double n1[3] = {nrm[3 * (size_t)i], nrm[3 * (size_t)i + 1], nrm[3 * (size_t)i + 2]};
      hist_incr = 100.0 / (double)(cnt - 1);
      for (int k = 1; k < cnt; ++k) {
        const size_t j = (size_t)nb_idx[(size_t)i * knn + k];
        const double p2[3] = {xyz[3 * j], xyz[3 * j + 1], xyz[3 * j + 2]};
        const double n2[3] = {nrm[3 * j], nrm[3 * j + 1], nrm[3 * j + 2]};
        double f[3];
        pair_features(p1, n1, p2, n2, f);
        hc[fpfh_bin(11 * (f[0] + pi) / (2.0 * pi))]++;
        hc[11 + fpfh_bin(11 * (f[1] + 1.0) * 0.5)]++;
        hc[22 + fpfh_bin(11 * (f[2] + 1.0) * 0.5)]++;
      }
    }
    for (int b = 0; b < 33; ++b) {
      double v = 0.0;
      for (int t = 0; t < hc[b]; ++t) v += hist_incr;
      spfh[(size_t)i * 33 + b] = v;
    }
  }
}

__global__ void __launch_bounds__(FK_THREADS) fpfh_kernel(const int32_t* __restrict__ d_n, int knn, const int32_t* __restrict__ nb_idx,
                                                          const double* __restrict__ nb_d2, const int32_t* __restrict__ nb_cnt,
                                                          const double* __restrict__ spfh, double* __restrict__ out) {
  pdl_wait();
  const int n = *d_n;
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < 3 * n; t += gridDim.x * blockDim.x) {
    const int i = t / 3, blk = 11 * (t % 3);
    const int cnt = nb_cnt[i];
    double* o = out + (size_t)i * 33 + blk;
    if (cnt <= 1) {
      for (int j = 0; j < 11; ++j) o[j] = 0.0;
      continue;
    }
    double acc[11];
#pragma unroll
    for (int j = 0; j < 11; ++j) acc[j] = 0.0;
    double sum = 0.0;
    for (int k = 1; k < cnt; ++k) {
      const double d = nb_d2[(size_t)i * knn + k];
      if (d == 0.0) continue;
      const double* s = spfh + (size_t)nb_idx[(size_t)i * knn + k] * 33 + blk;
#pragma unroll
      for (int j = 0; j < 11; ++j) {
        const double val = s[j] / d;
        sum += val;
        acc[j] += val;
      }
    }
    if (sum != 0.0) sum = 100.0 / sum;
    const double* own = spfh + (size_t)i * 33 + blk;
#pragma unroll
    for (int j = 0; j < 11; ++j) o[j] = acc[j] * sum + own[j];
  }
}

int32_t op_compute_fpfh(b2s_handle* h, const b2s_cloud* c, size_t n, double radius, int knn, b2s_feature* f) {
  B2S_REQUIRE(n < (size_t)0x7fffffff / B2S_FEATURE_MAX_KNN, B2S_E_INVALID, "cloud too large for the neighbour lists");
  f->n = 0;
  if (n == 0) return B2S_OK;
  // cell edge as for the normals (radius / 4): a hybrid search ends within about four rings
  B2S_TRY(grid_build(h, &h->grid_b, c, radius / 4.0, nullptr));
  B2S_TRY(f->data.ensure(n * 33 * 8, h->stream));
  B2S_TRY(f->spfh.ensure(n * 33 * 8, h->stream));
  B2S_TRY(f->nb_idx.ensure(n * (size_t)knn * 4, h->stream));
  B2S_TRY(f->nb_d2.ensure(n * (size_t)knn * 8, h->stream));
  B2S_TRY(f->nb_cnt.ensure(n * 4, h->stream));
  // points the grid leaves out (a NaN coordinate) have no neighbour list: zero rows
  B2S_CUDA(cudaMemsetAsync(f->nb_cnt.p, 0, n * 4, h->stream));
  const GridHeader* hdr = h->grid_b.hdr.as<GridHeader>();
  const int32_t* d_n = c->dn.as<int32_t>();
  const int cap = 16 * device_sms();
  const int wblocks = (int)std::min<size_t>((n + FK_THREADS / 32 - 1) / (FK_THREADS / 32), (size_t)cap);
  launch_pdl(fpfh_knn_kernel, wblocks, FK_THREADS, 0, h->stream, hdr, grid_starts(&h->grid_b), h->grid_b.pts.as<double4>(), knn, radius,
             f->nb_idx.as<int32_t>(), f->nb_d2.as<double>(), f->nb_cnt.as<int32_t>());
  launch_pdl(fpfh_spfh_kernel, grid_for(n, FK_THREADS, cap), FK_THREADS, 0, h->stream, c->xyz.as<double>(), c->nrm.as<double>(), d_n, knn,
             f->nb_idx.as<int32_t>(), f->nb_cnt.as<int32_t>(), f->spfh.as<double>());
  launch_pdl(fpfh_kernel, grid_for(3 * n, FK_THREADS, cap), FK_THREADS, 0, h->stream, d_n, knn, f->nb_idx.as<int32_t>(), f->nb_d2.as<double>(),
             f->nb_cnt.as<int32_t>(), f->spfh.as<double>(), f->data.as<double>());
  h->launches += 3;
  B2S_CUDA(cudaGetLastError());
  f->n = n;
  return B2S_OK;
}

}  // namespace b2s
