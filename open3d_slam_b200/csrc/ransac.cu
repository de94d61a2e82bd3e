// ransac.cu -- K-ransac: [O3D] RegistrationRANSACBasedOnFeatureMatching as PlaceRecognition::buildLoopClosureConstraints calls it
// (core/src/PlaceRecognition.cpp:81-86), one source against n candidate targets per call.  Semantics: DESIGN.md row K-ransac.
//
//   fm_tile_kernel     (source tile of 64 rows, pair): the exact fp64 d2 of the 64 rows against every target row, 64 x 64 tiles
//                      staged in shared memory, each thread a 4 x 4 block.  One d2 feeds both argmins: the rows' running best
//                      stays in registers, the columns' best of this source tile is written as a partial.
//   fm_merge_kernel    (target row, pair): the column partials merged over the source tiles -> tgt_to_src.
//   mutual flags -> batched look-back scan (runtime.cu) -> rs_set_kernel: the mutual set in ascending i, or the one-way set when
//                      it has fewer than 3 ransac_n pairs.
// Then, per batch of B hypotheses h0 .. h0 + B - 1 (B2S_RANSAC_BATCH):
//   rs_hyp_kernel      (hypothesis, pair): draw, edge-length checker, umeyama, distance checker -> survivor flag + T
//   scan + rs_compact_kernel: the survivors and their T per pair, in h order
//   rs_validate_kernel (survivor, pair), one CTA each: inliers and sum d2 of the moved source sparse cloud against the target's grid
//                      (1-NN with d2 < r2, ties to the lower index), reduced in a fixed order
//   rs_replay_kernel   (pair), one warp: walks the survivors in h order and applies the sequential best / stop rule, so the result
//                      cannot depend on B, on the other pairs of the call or on scheduling.
// Every comparison is lexicographic on (d2, index), which is associative: the reduction order never changes an argmin.
#include <math.h>
#include <stdlib.h>

#include <algorithm>
#include <vector>

#include "common.cuh"

namespace b2s {

constexpr int FM_TILE = 64, FM_THREADS = 256, FM_DIM = B2S_FEATURE_DIM;
constexpr int RS_THREADS = 128, RV_THREADS = 256;
constexpr int NONE = 0x7fffffff;


struct MatchJob {
  const double* tgt; int nt;
  int32_t* s2t; int32_t* t2s;
  double* part_d; int32_t* part_i;   // [source tiles][nt] column partials
};

__global__ void __launch_bounds__(FM_THREADS) fm_tile_kernel(const double* __restrict__ src, int ns, const MatchJob* __restrict__ jobs) {
  pdl_wait();
  const MatchJob J = jobs[blockIdx.y];
  const int s0 = blockIdx.x * FM_TILE;
  __shared__ double ss[FM_TILE][FM_DIM], st[FM_TILE][FM_DIM];
  __shared__ double cd[FM_THREADS / 32][FM_TILE];
  __shared__ int ci[FM_THREADS / 32][FM_TILE];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4, warp = tid >> 5;
  const unsigned FULL = 0xffffffffu;
  for (int e = tid; e < FM_TILE * FM_DIM; e += FM_THREADS) {
    const int r = e / FM_DIM, k = e % FM_DIM;
    ss[r][k] = s0 + r < ns ? src[(size_t)(s0 + r) * FM_DIM + k] : 0.0;
  }
  double rb[4]; int ri[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) { rb[r] = INFINITY; ri[r] = NONE; }
  for (int t0 = 0; t0 < J.nt; t0 += FM_TILE) {
    __syncthreads();   // the previous tile's reads of st / cd are done
    for (int e = tid; e < FM_TILE * FM_DIM; e += FM_THREADS) {
      const int r = e / FM_DIM, k = e % FM_DIM;
      st[r][k] = t0 + r < J.nt ? J.tgt[(size_t)(t0 + r) * FM_DIM + k] : 0.0;
    }
    __syncthreads();
    double acc[4][4];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[r][c] = 0.0;
    for (int k = 0; k < FM_DIM; ++k) {   // ascending k: the order of the restatement (the library builds with -fmad=false)
      double a[4], b[4];
#pragma unroll
      for (int r = 0; r < 4; ++r) a[r] = ss[ty + 16 * r][k];
#pragma unroll
      for (int c = 0; c < 4; ++c) b[c] = st[tx + 16 * c][k];
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) { const double d = a[r] - b[c]; acc[r][c] = acc[r][c] + d * d; }
    }
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int j = t0 + tx + 16 * c;
      double bd = INFINITY; int bi = NONE;
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int i = s0 + ty + 16 * r;
        if (j < J.nt && nn_key_less(acc[r][c], j, rb[r], ri[r])) { rb[r] = acc[r][c]; ri[r] = j; }
        if (i < ns && nn_key_less(acc[r][c], i, bd, bi)) { bd = acc[r][c]; bi = i; }
      }
      const double od = __shfl_xor_sync(FULL, bd, 16);   // the other row group (ty ^ 1) of this warp
      const int oi = __shfl_xor_sync(FULL, bi, 16);
      if (nn_key_less(od, oi, bd, bi)) { bd = od; bi = oi; }
      if ((tid & 16) == 0) { cd[warp][tx + 16 * c] = bd; ci[warp][tx + 16 * c] = bi; }
    }
    __syncthreads();
    if (tid < FM_TILE && t0 + tid < J.nt) {
      double bd = INFINITY; int bi = NONE;
      for (int w = 0; w < FM_THREADS / 32; ++w) if (nn_key_less(cd[w][tid], ci[w][tid], bd, bi)) { bd = cd[w][tid]; bi = ci[w][tid]; }
      J.part_d[(size_t)blockIdx.x * J.nt + t0 + tid] = bd;
      J.part_i[(size_t)blockIdx.x * J.nt + t0 + tid] = bi;
    }
  }
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    double bd = rb[r]; int bi = ri[r];
#pragma unroll
    for (int o = 1; o < 16; o <<= 1) {
      const double od = __shfl_xor_sync(FULL, bd, o);
      const int oi = __shfl_xor_sync(FULL, bi, o);
      if (nn_key_less(od, oi, bd, bi)) { bd = od; bi = oi; }
    }
    const int i = s0 + ty + 16 * r;
    if (tx == 0 && i < ns) J.s2t[i] = bi == NONE ? -1 : bi;
  }
}

__global__ void fm_merge_kernel(int n_stiles, const MatchJob* __restrict__ jobs) {
  pdl_wait();
  const MatchJob J = jobs[blockIdx.y];
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < J.nt; j += gridDim.x * blockDim.x) {
    double bd = INFINITY; int bi = NONE;
    for (int t = 0; t < n_stiles; ++t) {
      const double d = J.part_d[(size_t)t * J.nt + j];
      const int i = J.part_i[(size_t)t * J.nt + j];
      if (nn_key_less(d, i, bd, bi)) { bd = d; bi = i; }
    }
    J.t2s[j] = bi == NONE ? -1 : bi;
  }
}

// ---- RANSAC -----------------------------------------------------------------------------------------------------------
struct RansacPair {        // device state of one (source, target) pair, read back once per batch
  double best_T[16];
  double best_sum;         // sum d2 of best's inliers
  long long est_k;         // the loop runs while h < est_k
  long long stop_h;        // the h the loop stopped at (valid once done)
  long long best_h;        // -1 = the empty result
  long long last_update;   // h of the last hypothesis that replaced best
  long long validations;
  int best_inl;
  int set_size;
  int used_mutual;
  int done;
};

struct RansacJob {
  const double* txyz; int nt;
  const int32_t* s2t; const int32_t* t2s;
  int32_t* mflag; int32_t* moff;       // mutual flags / their exclusive scan (ns + 1)
  int32_t* set_s; int32_t* set_t;      // the correspondence set
  const GridHeader* ghdr; const int32_t* gcs; const double4* gpts;
  int32_t* hflag; int32_t* hoff;       // per batch: survivor flags / their scan (B + 1)
  long long* surv_h; double* hyp_T; double* surv_T; int32_t* surv_inl; double* surv_sum;
  RansacPair* st;
};

struct RansacConst {
  const double* sxyz; int ns;
  int n; int mutual;
  double max_corr, checker_dist, checker_edge, confidence;
  unsigned long long seed;
  int B;
};

__global__ void rs_mutual_kernel(int ns, const RansacJob* __restrict__ jobs) {
  pdl_wait();
  const RansacJob& J = jobs[blockIdx.y];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < ns; i += gridDim.x * blockDim.x) {
    const int j = J.s2t[i];
    J.mflag[i] = j >= 0 && J.t2s[j] == i ? 1 : 0;
  }
}

__global__ void rs_set_kernel(RansacConst c, const RansacJob* __restrict__ jobs) {
  pdl_wait();
  const RansacJob& J = jobs[blockIdx.y];
  const int n_mutual = J.moff[c.ns];
  const bool mutual = c.mutual && n_mutual >= 3 * c.n;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < c.ns; i += gridDim.x * blockDim.x) {
    if (!mutual) { J.set_s[i] = i; J.set_t[i] = J.s2t[i]; }
    else if (J.mflag[i]) { J.set_s[J.moff[i]] = i; J.set_t[J.moff[i]] = J.s2t[i]; }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) { J.st->set_size = mutual ? n_mutual : c.ns; J.st->used_mutual = mutual ? 1 : 0; }
}

__device__ __forceinline__ unsigned long long splitmix64(unsigned long long z) {
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

__device__ __forceinline__ double norm3(double x, double y, double z) { return sqrt(x * x + y * y + z * z); }

// T . [p; 1], row sums left to right
__device__ __forceinline__ void xform(const double* T, double x, double y, double z, double* o) {
  o[0] = ((T[0] * x + T[1] * y) + T[2] * z) + T[3];
  o[1] = ((T[4] * x + T[5] * y) + T[6] * z) + T[7];
  o[2] = ((T[8] * x + T[9] * y) + T[10] * z) + T[11];
}

__global__ void __launch_bounds__(RS_THREADS) rs_hyp_kernel(RansacConst c, long long h0, const RansacJob* __restrict__ jobs) {
  pdl_wait();
  const RansacJob& J = jobs[blockIdx.y];
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= c.B) return;
  const long long h = h0 + b;
  int ok = 0;
  if (!J.st->done && h < J.st->est_k) {
    const unsigned long long size = (unsigned long long)J.st->set_size;
    double S[B2S_RANSAC_MAX_N][3], Q[B2S_RANSAC_MAX_N][3];
#pragma unroll
    for (int j = 0; j < B2S_RANSAC_MAX_N; ++j) {
      if (j < c.n) {
        const unsigned long long u = splitmix64(c.seed + (unsigned long long)(h * c.n + j + 1) * 0x9E3779B97F4A7C15ull);
        const int k = (int)__umul64hi(u, size);
        const size_t si = (size_t)J.set_s[k], ti = (size_t)J.set_t[k];
        S[j][0] = c.sxyz[3 * si]; S[j][1] = c.sxyz[3 * si + 1]; S[j][2] = c.sxyz[3 * si + 2];
        Q[j][0] = J.txyz[3 * ti]; Q[j][1] = J.txyz[3 * ti + 1]; Q[j][2] = J.txyz[3 * ti + 2];
      }
    }
    ok = 1;
    // CorrespondenceCheckerBasedOnEdgeLength: every sample pair i < j, in sample order
#pragma unroll
    for (int i = 0; i < B2S_RANSAC_MAX_N; ++i)
#pragma unroll
      for (int j = i + 1; j < B2S_RANSAC_MAX_N; ++j)
        if (j < c.n && ok) {
          const double ds = norm3(S[i][0] - S[j][0], S[i][1] - S[j][1], S[i][2] - S[j][2]);
          const double dt = norm3(Q[i][0] - Q[j][0], Q[i][1] - Q[j][1], Q[i][2] - Q[j][2]);
          if (ds < dt * c.checker_edge || dt < ds * c.checker_edge) ok = 0;
        }
    double T[16];
    if (ok) {   // Eigen::umeyama without scaling, two passes: means, then the demeaned covariance times 1/n
      const double one_over_n = 1.0 / (double)c.n;
      double ms[3] = {0, 0, 0}, mt[3] = {0, 0, 0}, sigma[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
      for (int j = 0; j < B2S_RANSAC_MAX_N; ++j)
        if (j < c.n)
#pragma unroll
          for (int a = 0; a < 3; ++a) { ms[a] += S[j][a]; mt[a] += Q[j][a]; }
#pragma unroll
      for (int a = 0; a < 3; ++a) { ms[a] *= one_over_n; mt[a] *= one_over_n; }
#pragma unroll
      for (int j = 0; j < B2S_RANSAC_MAX_N; ++j)
        if (j < c.n)
#pragma unroll
          for (int a = 0; a < 3; ++a)
#pragma unroll
            for (int bb = 0; bb < 3; ++bb) sigma[3 * a + bb] += (Q[j][a] - mt[a]) * (S[j][bb] - ms[bb]);
#pragma unroll
      for (int a = 0; a < 9; ++a) sigma[a] *= one_over_n;
      double U[9], Sv[3], V[9], R[9];
      svd3_dev(sigma, U, Sv, V);
      const double sgn = det3_dev(U) * det3_dev(V) < 0 ? -1.0 : 1.0;
#pragma unroll
      for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int bb = 0; bb < 3; ++bb) R[3 * a + bb] = U[3 * a] * V[3 * bb] + U[3 * a + 1] * V[3 * bb + 1] + sgn * U[3 * a + 2] * V[3 * bb + 2];
#pragma unroll
      for (int i = 0; i < 16; ++i) T[i] = (i % 5 == 0) ? 1.0 : 0.0;
#pragma unroll
      for (int a = 0; a < 3; ++a) {
#pragma unroll
        for (int bb = 0; bb < 3; ++bb) T[4 * a + bb] = R[3 * a + bb];
        T[4 * a + 3] = mt[a] - (R[3 * a] * ms[0] + R[3 * a + 1] * ms[1] + R[3 * a + 2] * ms[2]);
      }
      // CorrespondenceCheckerBasedOnDistance: ||t - T s|| <= threshold for every sample
#pragma unroll
      for (int j = 0; j < B2S_RANSAC_MAX_N; ++j)
        if (j < c.n && ok) {
          double p[3];
          xform(T, S[j][0], S[j][1], S[j][2], p);
          if (norm3(Q[j][0] - p[0], Q[j][1] - p[1], Q[j][2] - p[2]) > c.checker_dist) ok = 0;
        }
      if (ok) {
        double* o = J.hyp_T + (size_t)b * 16;
#pragma unroll
        for (int i = 0; i < 16; ++i) o[i] = T[i];
      }
    }
  }
  J.hflag[b] = ok;
}

__global__ void rs_compact_kernel(RansacConst c, long long h0, const RansacJob* __restrict__ jobs) {
  pdl_wait();
  const RansacJob& J = jobs[blockIdx.y];
  for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < c.B; b += gridDim.x * blockDim.x) {
    if (!J.hflag[b]) continue;
    const int s = J.hoff[b];
    J.surv_h[s] = h0 + b;
    for (int i = 0; i < 16; ++i) J.surv_T[(size_t)s * 16 + i] = J.hyp_T[(size_t)b * 16 + i];
  }
}

// GetRegistrationResultAndCorrespondences of the source sparse cloud moved by T: 1-NN in the target grid with d2 < r2
__global__ void __launch_bounds__(RV_THREADS, 1) rs_validate_kernel(RansacConst c, const RansacJob* __restrict__ jobs) {
  pdl_wait();
  const RansacJob& J = jobs[blockIdx.y];
  const int s = blockIdx.x;
  if (s >= J.hoff[c.B] || J.surv_h[s] >= J.st->est_k) return;   // not a survivor / past the stop the previous batches set
  __shared__ GridHeader g;
  __shared__ double T[16];
  __shared__ double rsum[RV_THREADS];
  __shared__ int rinl[RV_THREADS];
  if (threadIdx.x == 0) g = *J.ghdr;
  if (threadIdx.x < 16) T[threadIdx.x] = J.surv_T[(size_t)s * 16 + threadIdx.x];
  __syncthreads();
  const double r = c.max_corr;
  double sum = 0.0; int inl = 0;
  for (int i = threadIdx.x; i < c.ns; i += RV_THREADS) {
    double q[3];
    xform(T, c.sxyz[3 * (size_t)i], c.sxyz[3 * (size_t)i + 1], c.sxyz[3 * (size_t)i + 2], q);
    double d2;
    if (grid_nearest(g, J.gcs, J.gpts, q[0], q[1], q[2], r, &d2) >= 0) { ++inl; sum += d2; }
  }
  rsum[threadIdx.x] = sum; rinl[threadIdx.x] = inl;
  for (int o = RV_THREADS / 2; o > 0; o >>= 1) {   // fixed tree: a run is bit-reproducible
    __syncthreads();
    if (threadIdx.x < o) { rsum[threadIdx.x] += rsum[threadIdx.x + o]; rinl[threadIdx.x] += rinl[threadIdx.x + o]; }
  }
  if (threadIdx.x == 0) { J.surv_inl[s] = rinl[0]; J.surv_sum[s] = rsum[0]; }
}

// the sequential loop of DESIGN.md K-ransac rule 7 over this batch's survivors
__global__ void rs_replay_kernel(RansacConst c, long long h0, const RansacJob* __restrict__ jobs) {
  pdl_wait();
  const RansacJob& J = jobs[blockIdx.x];
  if (threadIdx.x != 0) return;
  RansacPair& P = *J.st;
  if (P.done) return;
  const int cnt = J.hoff[c.B];
  for (int s = 0; s < cnt; ++s) {
    const long long h = J.surv_h[s];
    if (h >= P.est_k) break;
    P.validations++;
    const int inl = J.surv_inl[s];
    const double sum = J.surv_sum[s];
    if (inl > 0 && (inl > P.best_inl || (inl == P.best_inl && sum < P.best_sum))) {
      P.best_inl = inl; P.best_sum = sum; P.best_h = h; P.last_update = h;
      for (int i = 0; i < 16; ++i) P.best_T[i] = J.surv_T[(size_t)s * 16 + i];
      const double fitness = (double)inl / (double)c.ns;
      const double k_d = log(1.0 - c.confidence) / log(1.0 - pow(fitness, (double)c.n));
      if (k_d < (double)P.est_k) P.est_k = (long long)ceil(k_d);
    }
  }
  if (P.est_k <= h0 + c.B) {
    P.done = 1;
    P.stop_h = P.est_k > P.last_update + 1 ? P.est_k : P.last_update + 1;
  }
}

static int ransac_batch() {   // B2S_RANSAC_BATCH: hypotheses per batch (tuning knob, read once; default not tuned)
  static const int v = getenv("B2S_RANSAC_BATCH") ? atoi(getenv("B2S_RANSAC_BATCH")) : 0;
  return v > 0 ? v : 1024;
}

// Carves the per-pair partial arrays of the feature matching from L into jobs
static void fm_carve(Layout& L, const b2s_feature* src, int n, const b2s_feature* const* tgts, MatchJob* jobs) {
  const size_t n_stiles = (src->n + FM_TILE - 1) / FM_TILE;
  for (int k = 0; k < n; ++k) {
    jobs[k].part_d = L.take<double>(n_stiles * tgts[k]->n);
    jobs[k].part_i = L.take<int32_t>(n_stiles * tgts[k]->n);
  }
}

// Uploads the feature matching's jobs (their partial arrays carved by fm_carve) to jobs_dev and launches it
static int32_t feature_match(b2s_handle* h, const b2s_feature* src, int n, const b2s_feature* const* tgts, int32_t* const* s2t, int32_t* const* t2s,
                             MatchJob* jobs_dev, std::vector<MatchJob>& jobs) {
  const int ns = (int)src->n;
  const int n_stiles = (ns + FM_TILE - 1) / FM_TILE;
  int max_nt = 1;
  for (int k = 0; k < n; ++k) {
    const int nt = (int)tgts[k]->n;
    max_nt = std::max(max_nt, nt);
    jobs[k].tgt = tgts[k]->data.as<double>(); jobs[k].nt = nt;
    jobs[k].s2t = s2t[k]; jobs[k].t2s = t2s[k];
  }
  B2S_CUDA(cudaMemcpyAsync(jobs_dev, jobs.data(), sizeof(MatchJob) * n, cudaMemcpyHostToDevice, h->stream));
  if (ns > 0) launch_pdl(fm_tile_kernel, dim3(n_stiles, n), FM_THREADS, 0, h->stream, src->data.as<double>(), ns, (const MatchJob*)jobs_dev);
  launch_pdl(fm_merge_kernel, dim3(std::max(1, std::min((max_nt + 255) / 256, 4 * device_sms())), n), 256, 0, h->stream, n_stiles,
             (const MatchJob*)jobs_dev);
  h->launches += ns > 0 ? 2 : 1;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

int32_t op_feature_correspondences(b2s_handle* h, const b2s_feature* src, int n, const b2s_feature* const* tgts, int32_t* const* s2t,
                                   int32_t* const* t2s) {
  if (n <= 0) return B2S_OK;
  std::vector<MatchJob> jobs(n);
  MatchJob* jobs_dev = nullptr;
  B2S_TRY(carve(h->lc, h->stream, [&](Layout& L) {
    jobs_dev = L.take<MatchJob>(n);
    fm_carve(L, src, n, tgts, jobs.data());
  }));
  return feature_match(h, src, n, tgts, s2t, t2s, jobs_dev, jobs);
}

int32_t op_ransac(b2s_handle* h, const b2s_cloud* src, size_t ns_, const b2s_feature* src_f, int n, const b2s_cloud* const* tgts, const size_t* nts,
                  const b2s_feature* const* tgt_fs, const b2s_ransac_params& p, b2s_ransac_result* out) {
  const double I[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  for (int k = 0; k < n; ++k) {   // rule 2: the empty result
    memset(&out[k], 0, sizeof(out[k]));
    memcpy(out[k].result.T, I, sizeof(I));
    out[k].best_hypothesis = -1;
  }
  if (p.ransac_n < 3 || !(p.max_correspondence_distance > 0.0) || ns_ < (size_t)p.ransac_n) return B2S_OK;
  std::vector<int> live;   // pairs that run
  for (int k = 0; k < n; ++k) if (nts[k] > 0) live.push_back(k);
  const int m = (int)live.size();
  if (m == 0) return B2S_OK;
  const int ns = (int)ns_, B = ransac_batch();
  std::vector<const b2s_feature*> lf(m);
  std::vector<const b2s_cloud*> lc(m);
  for (int q = 0; q < m; ++q) { lf[q] = tgt_fs[live[q]]; lc[q] = tgts[live[q]]; }
  // scratch: MatchJob[m] | RansacJob[m] | ScanJob[2m] | RansacPair[m] | {ns, B} | scan states (every mutual scan's, then every survivor
  // scan's) | per pair: s2t, t2s, mutual flags / offsets, the set, survivor flags / offsets, survivors, hypothesis T | feature matching
  std::vector<RansacJob> rj(m);
  std::vector<ScanJob> sj(2 * m);
  std::vector<MatchJob> mj(m);
  std::vector<int32_t*> s2t(m), t2s(m);
  MatchJob* mj_dev = nullptr; RansacJob* rj_dev = nullptr; ScanJob* sj_dev = nullptr; RansacPair* st_dev = nullptr;
  int32_t* d_consts = nullptr;
  size_t states = 0, surv_states = 0, states_end = 0;
  B2S_TRY(carve(h->lc, h->stream, [&](Layout& L) {
    mj_dev = L.take<MatchJob>(m);
    rj_dev = L.take<RansacJob>(m);
    sj_dev = L.take<ScanJob>(2 * m);
    st_dev = L.take<RansacPair>(m);
    d_consts = L.take<int32_t>(2);
    states = L.size;
    for (int q = 0; q < m; ++q) scan_bind_state(L, sj[q], (size_t)ns);
    surv_states = L.size;
    for (int q = 0; q < m; ++q) scan_bind_state(L, sj[m + q], (size_t)B);
    states_end = L.size;
    for (int q = 0; q < m; ++q) {
      RansacJob& J = rj[q];
      J.txyz = lc[q]->xyz.as<double>(); J.nt = (int)nts[live[q]];
      s2t[q] = L.take<int32_t>(ns); J.s2t = s2t[q];
      t2s[q] = L.take<int32_t>(J.nt); J.t2s = t2s[q];
      J.mflag = L.take<int32_t>(ns); J.moff = L.take<int32_t>(ns + 1);
      J.set_s = L.take<int32_t>(ns); J.set_t = L.take<int32_t>(ns);
      J.hflag = L.take<int32_t>(B); J.hoff = L.take<int32_t>(B + 1);
      J.surv_h = L.take<long long>(B);
      J.hyp_T = L.take<double>((size_t)B * 16); J.surv_T = L.take<double>((size_t)B * 16);
      J.surv_inl = L.take<int32_t>(B); J.surv_sum = L.take<double>(B);
      J.st = st_dev + q;
    }
    fm_carve(L, src_f, m, lf.data(), mj.data());
  }));
  unsigned char* base = h->lc.as<unsigned char>();
  // target grids, built once per call (cell = the validation radius: a 3 x 3 x 3 box of cells holds every candidate)
  while (h->batch_grids.size() < (size_t)m) h->batch_grids.emplace_back(new GridIndex());
  std::vector<GridIndex*> grids(m);
  for (int q = 0; q < m; ++q) grids[q] = h->batch_grids[q].get();
  B2S_TRY(grid_build_batch(h, grids.data(), lc.data(), m, p.max_correspondence_distance));
  for (int q = 0; q < m; ++q) {
    rj[q].ghdr = grids[q]->hdr.as<GridHeader>(); rj[q].gcs = grid_starts(grids[q]); rj[q].gpts = grids[q]->pts.as<double4>();
  }
  B2S_TRY(feature_match(h, src_f, m, lf.data(), s2t.data(), t2s.data(), mj_dev, mj));
  // device tables and the initial state
  std::vector<RansacPair> st(m);
  for (int q = 0; q < m; ++q) {
    sj[q].in = rj[q].mflag; sj[q].out = rj[q].moff; sj[q].d_n = d_consts;
    sj[m + q].in = rj[q].hflag; sj[m + q].out = rj[q].hoff; sj[m + q].d_n = d_consts + 1;
    memset(&st[q], 0, sizeof(st[q]));
    memcpy(st[q].best_T, I, sizeof(I));
    st[q].est_k = p.max_iteration; st[q].best_h = -1; st[q].last_update = -1;
    st[q].done = p.max_iteration == 0;
  }
  B2S_CUDA(cudaMemsetAsync(base + states, 0, states_end - states, h->stream));
  const int32_t consts[2] = {ns, B};
  B2S_CUDA(cudaMemcpyAsync(d_consts, consts, 8, cudaMemcpyHostToDevice, h->stream));
  B2S_CUDA(cudaMemcpyAsync(rj_dev, rj.data(), sizeof(RansacJob) * m, cudaMemcpyHostToDevice, h->stream));
  B2S_CUDA(cudaMemcpyAsync(sj_dev, sj.data(), sizeof(ScanJob) * 2 * m, cudaMemcpyHostToDevice, h->stream));
  B2S_CUDA(cudaMemcpyAsync(st_dev, st.data(), sizeof(RansacPair) * m, cudaMemcpyHostToDevice, h->stream));
  RansacConst c;
  c.sxyz = src->xyz.as<double>(); c.ns = ns; c.n = p.ransac_n; c.mutual = p.mutual_filter ? 1 : 0;
  c.max_corr = p.max_correspondence_distance; c.checker_dist = p.checker_distance; c.checker_edge = p.checker_edge_length;
  c.confidence = p.confidence; c.seed = (unsigned long long)p.seed; c.B = B;
  const int gx = std::max(1, std::min((ns + 255) / 256, 4 * device_sms()));
  launch_pdl(rs_mutual_kernel, dim3(gx, m), 256, 0, h->stream, ns, (const RansacJob*)rj_dev);
  h->launches++;
  B2S_TRY(scan_exclusive_i32_batch(h, sj_dev, m, (size_t)ns));
  launch_pdl(rs_set_kernel, dim3(gx, m), 256, 0, h->stream, c, (const RansacJob*)rj_dev);
  h->launches++;
  for (long long h0 = 0;; h0 += B) {
    bool all_done = true;
    for (int q = 0; q < m; ++q) all_done = all_done && st[q].done;
    if (all_done) break;
    // the scan states of the survivor scan are single-use: zero them for this batch
    B2S_CUDA(cudaMemsetAsync(base + surv_states, 0, states_end - surv_states, h->stream));
    launch_pdl(rs_hyp_kernel, dim3((B + RS_THREADS - 1) / RS_THREADS, m), RS_THREADS, 0, h->stream, c, h0, (const RansacJob*)rj_dev);
    h->launches++;
    B2S_TRY(scan_exclusive_i32_batch(h, sj_dev + m, m, (size_t)B));
    launch_pdl(rs_compact_kernel, dim3((B + 255) / 256, m), 256, 0, h->stream, c, h0, (const RansacJob*)rj_dev);
    launch_pdl(rs_validate_kernel, dim3(B, m), RV_THREADS, 0, h->stream, c, (const RansacJob*)rj_dev);
    launch_pdl(rs_replay_kernel, m, 32, 0, h->stream, c, h0, (const RansacJob*)rj_dev);
    h->launches += 3;
    B2S_CUDA(cudaGetLastError());
    B2S_TRY(read_back(h, {{st.data(), st_dev, sizeof(RansacPair) * m}}));
  }
  for (int q = 0; q < m; ++q) {
    const RansacPair& P = st[q];
    b2s_ransac_result& o = out[live[q]];
    memcpy(o.result.T, P.best_T, sizeof(P.best_T));
    o.result.n_corr = P.best_inl;
    o.result.fitness = P.best_inl > 0 ? (double)P.best_inl / (double)ns : 0.0;
    o.result.inlier_rmse = P.best_inl > 0 ? sqrt(P.best_sum / (double)P.best_inl) : 0.0;
    o.result.iters = 0;
    o.hypotheses = P.done ? P.stop_h : p.max_iteration;
    o.validations = P.validations;
    o.best_hypothesis = P.best_h;
    o.n_feature_corr = P.set_size;
    o.used_mutual = P.used_mutual;
  }
  return B2S_OK;
}

}  // namespace b2s
