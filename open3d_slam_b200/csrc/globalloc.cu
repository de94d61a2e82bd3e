// globalloc.cu -- global localisation in a prior map (DESIGN.md row M3): an exhaustive (x, y, yaw[, z]) search scored by the share of
// query points that land in an occupied voxel of the map, the best distinct hypotheses refined by the scan-to-map ICP.  The rules are
// stated in include/b2s.h (b2s_submap_global_localization) and restated by tests/oracle_global_localization.{c,py}.
//
// Kernels, in launch order:
//   gl_occ_kernel       one bit per voxel (score_voxel) of the map's live-point box, set by atomicOr for every live map slot
//   gl_score_kernel     one CTA per (z level, yaw, tile of GL_THREADS translations): the yaw's rotated query R_j q is staged in shared
//                       memory (fp64, GL_CHUNK points per pass), every thread owns one translation and counts the probes that hit a set
//                       bit.  One int32 per hypothesis, written directly (no atomics, no reordering)
//   gl_hist_kernel      histogram of the hits (warp-aggregated atomics); gl_threshold_kernel finds the M-th largest value T
//   gl_eq_kernel + scan, gl_sel_kernel + scan, gl_scatter_kernel: order-preserving compaction of the hypotheses with hits > T and of the
//                       first ones (by index) with hits == T, M entries in all, as (hits, h) sort keys
//   gl_nms_kernel       one CTA: bitonic sort of the M keys in shared memory, greedy suppression, the candidates' poses
// Refinement: every candidate's patch is built as b2s_register_to_submap builds it; the registrations run 16 per batched ICP launch.
//
// Over a set of submaps (b2s_submaps_global_localization, DESIGN.md row M4) two kernels take gl_occ_kernel's place, each over a device
// job table of one {slot array, slot count, bbox} per submap (blockIdx.y = submap):
//   gl_union_box_kernel  the live-point box of the union and the union of the submaps' b2s_submap::bbox, one pass
//   gl_union_occ_kernel  gl_occ_kernel's bit for every live slot of every submap, into one grid spanning the union of the bboxes
// The score, selection and suppression kernels are the same launches; each candidate is refined in the submap whose centre is nearest.
#include "common.cuh"

#include <math.h>

using namespace b2s;

namespace b2s {

constexpr int GL_THREADS = 256;
constexpr int GL_CHUNK = 1024;             // query points staged per pass (24 KB of shared memory)
constexpr int GL_NMS_THREADS = 1024;
constexpr int GL_MAX_CANDIDATES = 256;
constexpr int GL_POOL_PER_CANDIDATE = 64;  // M = 64 n_candidates hypotheses enter the suppression
constexpr size_t GL_MAX_BYTES = (size_t)1 << 30;   // byte cap of the occupancy grid and of the score array (B2S_E_CAPACITY above it)
constexpr double GL_TWO_PI = 6.283185307179586;    // 2 pi rounded to double
constexpr int GL_BATCH = 16;               // registrations per batched ICP launch (the handle keeps GL_BATCH indices)

struct GlBox {              // the hypothesis grid
  double x_min, y_min, step, z0, z_step, inv;
  int32_t nx, ny, n_yaw, n_z;
};
struct GlOcc {              // the occupancy bit grid: voxel keys k in [kmin, kmin + dims) per axis
  const uint32_t* bits;
  int32_t kmin[3];
  int32_t dims[3];
};

__device__ __forceinline__ bool gl_probe(const GlOcc& o, double x, double y, double z, double inv) {
  const double fx = floor(__dmul_rn(x, inv)), fy = floor(__dmul_rn(y, inv)), fz = floor(__dmul_rn(z, inv));
  if (!(fabs(fx) < 1048575.0 && fabs(fy) < 1048575.0 && fabs(fz) < 1048575.0)) return false;   // voxel_key_of's limit; also NaN
  const unsigned kx = (unsigned)((int)fx - o.kmin[0]), ky = (unsigned)((int)fy - o.kmin[1]), kz = (unsigned)((int)fz - o.kmin[2]);
  if (kx >= (unsigned)o.dims[0] || ky >= (unsigned)o.dims[1] || kz >= (unsigned)o.dims[2]) return false;
  const size_t bit = ((size_t)kz * (size_t)o.dims[1] + ky) * (size_t)o.dims[0] + kx;
  return (__ldg(&o.bits[bit >> 5]) >> (bit & 31)) & 1u;
}

// sets the bit of map point i (rule 3: tombstones and keys beyond the limit set nothing)
__device__ __forceinline__ void gl_occ_set(const GlOcc& o, const double* __restrict__ xyz, int i, double inv, uint32_t* bits) {
  const double x = xyz[3 * i], y = xyz[3 * i + 1], z = xyz[3 * i + 2];
  if (!(x == x && y == y && z == z)) return;   // tombstone
  const double fx = floor(__dmul_rn(x, inv)), fy = floor(__dmul_rn(y, inv)), fz = floor(__dmul_rn(z, inv));
  if (!(fabs(fx) < 1048575.0 && fabs(fy) < 1048575.0 && fabs(fz) < 1048575.0)) return;
  const unsigned kx = (unsigned)((int)fx - o.kmin[0]), ky = (unsigned)((int)fy - o.kmin[1]), kz = (unsigned)((int)fz - o.kmin[2]);
  if (kx >= (unsigned)o.dims[0] || ky >= (unsigned)o.dims[1] || kz >= (unsigned)o.dims[2]) return;
  const size_t bit = ((size_t)kz * (size_t)o.dims[1] + ky) * (size_t)o.dims[0] + kx;
  atomicOr(&bits[bit >> 5], 1u << (bit & 31));
}

__global__ void __launch_bounds__(GL_THREADS) gl_occ_kernel(const double* __restrict__ xyz, const int32_t* __restrict__ d_n, double inv,
                                                            GlOcc o, uint32_t* bits) {
  pdl_wait();
  const int n = *d_n;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) gl_occ_set(o, xyz, i, inv, bits);
}

struct GlJob {              // one submap of the union: its map slots, their device count and its b2s_submap::bbox words
  const double* xyz;
  const int32_t* d_n;
  const unsigned long long* bbox;
};

// grid (blocks, n_jobs).  box[0..5]: the live points' box (ord_encode'd min xyz, max xyz), box[6..11]: the union of the bboxes; both
// reset to the empty box by the caller
__global__ void __launch_bounds__(GL_THREADS) gl_union_box_kernel(const GlJob* __restrict__ jobs, unsigned long long* box) {
  pdl_wait();
  const GlJob job = jobs[blockIdx.y];
  const int n = *job.d_n;
  double mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const double p[3] = {job.xyz[3 * i], job.xyz[3 * i + 1], job.xyz[3 * i + 2]};
    if (!(p[0] == p[0] && p[1] == p[1] && p[2] == p[2])) continue;   // tombstone
#pragma unroll
    for (int d = 0; d < 3; d++) { mn[d] = fmin(mn[d], p[d]); mx[d] = fmax(mx[d], p[d]); }
  }
  box_fold_block<GL_THREADS>(mn, mx, box);
  if (blockIdx.x == 0 && threadIdx.x < 6) {   // the empty bbox (+inf / -inf) leaves the union as it is
    if (threadIdx.x < 3) atomicMin(&box[6 + threadIdx.x], job.bbox[threadIdx.x]);
    else atomicMax(&box[6 + threadIdx.x], job.bbox[threadIdx.x]);
  }
}

// grid (blocks, n_jobs): gl_occ_kernel over every submap of the job table into one grid
__global__ void __launch_bounds__(GL_THREADS) gl_union_occ_kernel(const GlJob* __restrict__ jobs, double inv, GlOcc o, uint32_t* bits) {
  pdl_wait();
  const GlJob job = jobs[blockIdx.y];
  const int n = *job.d_n;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) gl_occ_set(o, job.xyz, i, inv, bits);
}

// grid (ceil(nx ny / GL_THREADS), n_yaw, n_z).  rot: 9 doubles per yaw, row-major
__global__ void __launch_bounds__(GL_THREADS) gl_score_kernel(const double* __restrict__ q, const int32_t* __restrict__ d_nq,
                                                              const double* __restrict__ rot, GlBox b, GlOcc o, int32_t* __restrict__ hits) {
  __shared__ double s_q[3 * GL_CHUNK];
  pdl_wait();
  const int nq = *d_nq;
  const int j = blockIdx.y, iz = blockIdx.z;
  const long long t = (long long)blockIdx.x * GL_THREADS + threadIdx.x;
  const bool valid = t < (long long)b.nx * b.ny;
  const int ix = valid ? (int)(t % b.nx) : 0, iy = valid ? (int)(t / b.nx) : 0;
  const double tx = __dadd_rn(b.x_min, __dmul_rn((double)ix, b.step));
  const double ty = __dadd_rn(b.y_min, __dmul_rn((double)iy, b.step));
  const double tz = __dadd_rn(b.z0, __dmul_rn((double)iz, b.z_step));
  double R[9];
#pragma unroll
  for (int k = 0; k < 9; k++) R[k] = rot[9 * j + k];
  int cnt = 0;
  for (int base = 0; base < nq; base += GL_CHUNK) {
    const int m = min(GL_CHUNK, nq - base);
    __syncthreads();
    for (int i = threadIdx.x; i < m; i += GL_THREADS) {
      const double x = q[3 * (base + i)], y = q[3 * (base + i) + 1], z = q[3 * (base + i) + 2];
      s_q[3 * i] = __dadd_rn(__dadd_rn(__dmul_rn(R[0], x), __dmul_rn(R[1], y)), __dmul_rn(R[2], z));
      s_q[3 * i + 1] = __dadd_rn(__dadd_rn(__dmul_rn(R[3], x), __dmul_rn(R[4], y)), __dmul_rn(R[5], z));
      s_q[3 * i + 2] = __dadd_rn(__dadd_rn(__dmul_rn(R[6], x), __dmul_rn(R[7], y)), __dmul_rn(R[8], z));
    }
    __syncthreads();
    if (valid) {
#pragma unroll 4
      for (int i = 0; i < m; i++)
        cnt += gl_probe(o, __dadd_rn(s_q[3 * i], tx), __dadd_rn(s_q[3 * i + 1], ty), __dadd_rn(s_q[3 * i + 2], tz), b.inv) ? 1 : 0;
    }
  }
  if (valid) hits[(((size_t)iz * b.n_yaw + j) * b.ny + iy) * b.nx + ix] = cnt;
}

__global__ void gl_set_n_kernel(int32_t* d_n, int32_t n) { pdl_wait(); *d_n = n; }

__global__ void __launch_bounds__(GL_THREADS) gl_hist_kernel(const int32_t* __restrict__ hits, long long n, int32_t* hist) {
  pdl_wait();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int v = hits[i];
    const unsigned peers = __match_any_sync(__activemask(), v);
    if ((threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&hist[v], __popc(peers));
  }
}

// sel[0] = T, the M-th largest hit count (M = min(pool, n)); sel[1] = how many hypotheses with hits == T enter the pool; sel[2] = M
__global__ void gl_threshold_kernel(const int32_t* __restrict__ hist, int nq, long long n, int pool, int32_t* sel) {
  pdl_wait();
  const int M = (long long)pool < n ? pool : (int)n;
  long long acc = 0;
  int T = 0, need = M;
  for (int v = nq; v >= 0; v--) {
    if (acc + hist[v] >= M) { T = v; need = (int)(M - acc); break; }
    acc += hist[v];
  }
  sel[0] = T; sel[1] = need; sel[2] = M;
}

__global__ void __launch_bounds__(GL_THREADS) gl_eq_kernel(const int32_t* __restrict__ hits, long long n, const int32_t* __restrict__ sel,
                                                           int32_t* __restrict__ eq) {
  pdl_wait();
  const int T = sel[0];
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) eq[i] = hits[i] == T;
}
__global__ void __launch_bounds__(GL_THREADS) gl_sel_kernel(const int32_t* __restrict__ hits, long long n, const int32_t* __restrict__ sel,
                                                            const int32_t* __restrict__ eq_rank, int32_t* __restrict__ flag) {
  pdl_wait();
  const int T = sel[0], need = sel[1];
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int v = hits[i];
    flag[i] = v > T || (v == T && eq_rank[i] < need);
  }
}
__global__ void __launch_bounds__(GL_THREADS) gl_scatter_kernel(const int32_t* __restrict__ hits, long long n, const int32_t* __restrict__ flag,
                                                                const int32_t* __restrict__ pos, int nq, unsigned long long* __restrict__ keys) {
  pdl_wait();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    if (flag[i]) keys[pos[i]] = ((unsigned long long)(unsigned)(nq - hits[i]) << 32) | (unsigned long long)i;   // (hits desc, h asc)
}

struct GlNms {
  double nms_distance, nms_yaw, yaw0, yaw_step;
  int32_t n_candidates;
};

__device__ __forceinline__ void gl_decode(const GlBox& b, const GlNms& p, unsigned h, double* t, double* yaw, int* j) {
  const int ix = (int)(h % (unsigned)b.nx);
  unsigned r = h / (unsigned)b.nx;
  const int iy = (int)(r % (unsigned)b.ny);
  r /= (unsigned)b.ny;
  *j = (int)(r % (unsigned)b.n_yaw);
  const int iz = (int)(r / (unsigned)b.n_yaw);
  t[0] = __dadd_rn(b.x_min, __dmul_rn((double)ix, b.step));
  t[1] = __dadd_rn(b.y_min, __dmul_rn((double)iy, b.step));
  t[2] = __dadd_rn(b.z0, __dmul_rn((double)iz, b.z_step));
  *yaw = __dadd_rn(p.yaw0, __dmul_rn((double)*j, p.yaw_step));
}

// out_i32: [0] candidate count, then per candidate {h, hits}; out_T: 16 doubles per candidate
__global__ void __launch_bounds__(GL_NMS_THREADS) gl_nms_kernel(const unsigned long long* __restrict__ keys_in, const int32_t* __restrict__ sel,
                                                                int P, GlBox b, GlNms p, const double* __restrict__ rot, int nq,
                                                                int32_t* __restrict__ out_i32, double* __restrict__ out_T) {
  extern __shared__ unsigned long long s_keys[];
  __shared__ double s_t[GL_MAX_CANDIDATES][3];
  __shared__ double s_yaw[GL_MAX_CANDIDATES];
  __shared__ int s_nk;
  pdl_wait();
  const int M = sel[2];
  for (int i = threadIdx.x; i < P; i += GL_NMS_THREADS) s_keys[i] = i < M ? keys_in[i] : ~0ull;
  __syncthreads();
  for (int k = 2; k <= P; k <<= 1)
    for (int jj = k >> 1; jj > 0; jj >>= 1) {
      for (int i = threadIdx.x; i < P; i += GL_NMS_THREADS) {
        const int l = i ^ jj;
        if (l > i) {
          const unsigned long long a = s_keys[i], c = s_keys[l];
          if (((i & k) == 0) == (a > c)) { s_keys[i] = c; s_keys[l] = a; }
        }
      }
      __syncthreads();
    }
  if (threadIdx.x == 0) s_nk = 0;
  __syncthreads();
  for (int i = 0; i < M; i++) {
    const int nk = s_nk;
    if (nk >= p.n_candidates) break;
    const unsigned h = (unsigned)(s_keys[i] & 0xFFFFFFFFull);
    double t[3], yaw;
    int j;
    gl_decode(b, p, h, t, &yaw, &j);
    bool close = false;
    if (threadIdx.x < nk) {
      const double dx = __dsub_rn(t[0], s_t[threadIdx.x][0]), dy = __dsub_rn(t[1], s_t[threadIdx.x][1]), dz = __dsub_rn(t[2], s_t[threadIdx.x][2]);
      const double d = sqrt(__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)));
      const double dyaw = fabs(remainder(__dsub_rn(yaw, s_yaw[threadIdx.x]), GL_TWO_PI));
      close = d <= p.nms_distance && dyaw <= p.nms_yaw;
    }
    const int suppressed = __syncthreads_or(close);
    if (!suppressed && threadIdx.x == 0) {
      s_t[nk][0] = t[0]; s_t[nk][1] = t[1]; s_t[nk][2] = t[2]; s_yaw[nk] = yaw;
      out_i32[1 + 2 * nk] = (int32_t)h;
      out_i32[2 + 2 * nk] = nq - (int32_t)(s_keys[i] >> 32);
      double* T = out_T + 16 * nk;
      for (int r = 0; r < 3; r++) { T[4 * r] = rot[9 * j + 3 * r]; T[4 * r + 1] = rot[9 * j + 3 * r + 1]; T[4 * r + 2] = rot[9 * j + 3 * r + 2]; T[4 * r + 3] = t[r]; }
      T[12] = 0.0; T[13] = 0.0; T[14] = 0.0; T[15] = 1.0;
      s_nk = nk + 1;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) out_i32[0] = s_nk;
}

// the call's own scratch, freed on return: the search runs once per (re)localisation, and none of it may count as a re-allocation of the
// buffers a captured mapper chain holds
struct GlScratch {
  DevBuf box, jobs, rot, occ, hits, eq, rank, flag, pos, hist, keys, sel, cand_i32, cand_T, scan_state, problems, work, results, hdrs;
  b2s_cloud cropped, query, merge, match;   // merge / match: S1 of the raw scan, kept apart from the mapper's last processed scan
  GlScratch() {
    for (DevBuf* d : {&box, &jobs, &rot, &occ, &hits, &eq, &rank, &flag, &pos, &hist, &keys, &sel, &cand_i32, &cand_T, &scan_state, &problems,
                      &work, &results, &hdrs})
      d->tracked = false;
    for (b2s_cloud* c : {&cropped, &query, &merge, &match}) c->xyz.tracked = c->nrm.tracked = c->dn.tracked = false;
  }
};

static bool finite(double v) { return v == v && v - v == 0.0; }

static int32_t gl_check_params(const b2s_global_localization_params& p) {
  B2S_REQUIRE(p.step > 0.0 && finite(p.step) && p.score_voxel > 0.0 && finite(p.score_voxel), B2S_E_INVALID,
              "global localisation: step and score_voxel must be finite and > 0");
  B2S_REQUIRE(p.n_yaw >= 1 && p.n_z >= 1 && p.n_candidates >= 1, B2S_E_INVALID, "global localisation: n_yaw, n_z and n_candidates must be >= 1");
  B2S_REQUIRE(p.n_candidates <= GL_MAX_CANDIDATES, B2S_E_INVALID, "global localisation: n_candidates must be <= %d", GL_MAX_CANDIDATES);
  B2S_REQUIRE(finite(p.x_min) && finite(p.x_max) && finite(p.y_min) && finite(p.y_max), B2S_E_INVALID, "global localisation: non-finite box bound");
  B2S_REQUIRE(finite(p.z0) && finite(p.z_step) && finite(p.yaw0) && finite(p.yaw_step) && finite(p.roll) && finite(p.pitch) &&
                  finite(p.nms_distance) && finite(p.nms_yaw),
              B2S_E_INVALID, "global localisation: non-finite parameter");
  return B2S_OK;
}

// R_j = Rz(yaw_j) Ry(pitch) Rx(roll), yaw_j = yaw0 + j yaw_step; (Rz Ry) first, then times Rx, every entry summed left to right
static void gl_rotations(const b2s_global_localization_params& p, std::vector<double>& rot) {
  rot.assign(9 * (size_t)p.n_yaw, 0.0);
  const double cp = cos(p.pitch), sp = sin(p.pitch), cr = cos(p.roll), sr = sin(p.roll);
  const double Ry[9] = {cp, 0.0, sp, 0.0, 1.0, 0.0, -sp, 0.0, cp};
  const double Rx[9] = {1.0, 0.0, 0.0, 0.0, cr, -sr, 0.0, sr, cr};
  for (int j = 0; j < p.n_yaw; j++) {
    volatile double m = (double)j * p.yaw_step;   // one rounded multiply, one rounded add
    const double yaw = p.yaw0 + m;
    const double cy = cos(yaw), sy = sin(yaw);
    const double Rz[9] = {cy, -sy, 0.0, sy, cy, 0.0, 0.0, 0.0, 1.0};
    double A[9];
    for (int r = 0; r < 3; r++)
      for (int c = 0; c < 3; c++) {
        volatile double a0 = Rz[3 * r] * Ry[c], a1 = Rz[3 * r + 1] * Ry[3 + c], a2 = Rz[3 * r + 2] * Ry[6 + c];
        volatile double s = a0 + a1;
        A[3 * r + c] = s + a2;
      }
    for (int r = 0; r < 3; r++)
      for (int c = 0; c < 3; c++) {
        volatile double a0 = A[3 * r] * Rx[c], a1 = A[3 * r + 1] * Rx[3 + c], a2 = A[3 * r + 2] * Rx[6 + c];
        volatile double s = a0 + a1;
        rot[9 * (size_t)j + 3 * r + c] = s + a2;
      }
  }
}

static double gl_yaw_of(const double* T) { return atan2(T[4], T[0]); }

// what the score and the candidate stages share: the query, the box and the occupancy grid, set up by gl_prepare
struct GlSetup {
  GlBox box;
  GlOcc occ;
  long long n_hyp = 0;
  int32_t nq = 0;
  std::vector<double> rot;
};

// S1 of the raw scan into match (when given), the query cloud, the live box of the map, the hypothesis grid and the occupancy grid.
// union_grid false (one submap, b2s_submap_global_localization): the occupancy grid spans the live box, set by gl_occ_kernel.
// union_grid true (b2s_submaps_global_localization): it spans the union of the submaps' bboxes, set by gl_union_occ_kernel from every
// submap.  Both set the same bits: every live slot lies inside either box.  Synchronises once (query size and boxes).
static int32_t gl_prepare(b2s_handle* h, const b2s_submap* const* sms, int n_sm, bool union_grid, const b2s_cloud* raw,
                          const b2s_global_localization_params& p, b2s_cloud* match, GlScratch& S, GlSetup& G) {
  B2S_TRY(gl_check_params(p));
  size_t n_max = 0;
  for (int s = 0; s < n_sm; s++) n_max = std::max(n_max, sms[s]->cloud[0]->n_max);
  B2S_REQUIRE(n_max > 0, B2S_E_EMPTY, "global localisation: the map is empty");
  if (match) B2S_TRY(process_scan_impl(h, raw, &S.merge, match));
  b2s_cropper c1 = h->cfg.scan.scan_matcher_cropper;
  c1.center[0] = c1.center[1] = c1.center[2] = 0.0;   // the crop S1 applies to match_, at identity
  {
    WideGridScope wide(raw->n_max);
    B2S_TRY(op_crop(h, raw, make_crop(&c1), &S.cropped));
    B2S_TRY(op_voxel_down_sample(h, &S.cropped, nullptr, p.score_voxel, &S.query));
  }
  B2S_TRY(S.box.ensure(96, h->stream));
  unsigned long long* box = S.box.as<unsigned long long>();
  if (union_grid) {
    std::vector<GlJob> jobs((size_t)n_sm);
    for (int s = 0; s < n_sm; s++) {
      const b2s_cloud* map = sms[s]->cloud[0].get();
      jobs[s] = GlJob{map->xyz.as<double>(), map->dn.as<int32_t>(), sms[s]->bbox.as<unsigned long long>()};
    }
    B2S_TRY(S.jobs.ensure(sizeof(GlJob) * jobs.size(), h->stream));
    B2S_CUDA(cudaMemcpyAsync(S.jobs.p, jobs.data(), sizeof(GlJob) * jobs.size(), cudaMemcpyHostToDevice, h->stream));
    B2S_TRY(box_reset(h, box));
    B2S_TRY(box_reset(h, box + 6));
    launch_pdl(gl_union_box_kernel, dim3((unsigned)grid_for(n_max, GL_THREADS), (unsigned)n_sm), GL_THREADS, 0, h->stream,
               static_cast<const GlJob*>(S.jobs.as<GlJob>()), box);
    h->launches++;
  } else {
    const b2s_cloud* map = sms[0]->cloud[0].get();
    B2S_TRY(bbox_reduce(h, map->xyz.as<double>(), map->dn.as<int32_t>(), map->n_max, nullptr, box));
  }
  unsigned long long box_enc[12];
  int32_t nq = 0;
  B2S_TRY(read_back(h, {{&nq, S.query.dn.p, 4}, {box_enc, S.box.p, union_grid ? 96u : 48u}}));
  if (!union_grid) memcpy(box_enc + 6, box_enc, 48);   // the occupancy grid spans the live box
  double bmin[3], bmax[3], omin[3], omax[3];
  for (int d = 0; d < 3; d++) {
    bmin[d] = ord_decode(box_enc[d]); bmax[d] = ord_decode(box_enc[3 + d]);
    omin[d] = fmin(ord_decode(box_enc[6 + d]), bmin[d]); omax[d] = fmax(ord_decode(box_enc[9 + d]), bmax[d]);
  }
  B2S_REQUIRE(bmin[0] <= bmax[0], B2S_E_EMPTY, "global localisation: the map has no live point");
  B2S_REQUIRE(nq > 0, B2S_E_EMPTY, "global localisation: the query cloud is empty");
  G.nq = nq;
  double x_min = p.x_min, x_max = p.x_max, y_min = p.y_min, y_max = p.y_max;
  if (x_min > x_max) { x_min = bmin[0]; x_max = bmax[0]; y_min = bmin[1]; y_max = bmax[1]; }
  B2S_REQUIRE(y_min <= y_max, B2S_E_INVALID, "global localisation: y_min > y_max");
  const double fx = floor((x_max - x_min) / p.step) + 1.0, fy = floor((y_max - y_min) / p.step) + 1.0;
  const double total = fx * fy * (double)p.n_yaw * (double)p.n_z;
  B2S_REQUIRE(fx >= 1.0 && fy >= 1.0 && total <= 2147483647.0, B2S_E_INVALID, "global localisation: %.0f hypotheses, at most 2^31 - 1", total);
  G.box = GlBox{x_min, y_min, p.step, p.z0, p.z_step, 1.0 / p.score_voxel, (int32_t)fx, (int32_t)fy, p.n_yaw, p.n_z};
  G.n_hyp = (long long)total;
  // the occupancy grid spans the voxel keys of its box, cut to the key limit
  size_t nbits = 1;
  for (int d = 0; d < 3; d++) {
    double k0 = floor(omin[d] * G.box.inv), k1 = floor(omax[d] * G.box.inv);
    k0 = fmax(k0, -1048574.0); k1 = fmin(k1, 1048574.0);
    if (k1 < k0) k1 = k0;
    G.occ.kmin[d] = (int32_t)k0;
    G.occ.dims[d] = (int32_t)(k1 - k0) + 1;
    nbits *= (size_t)G.occ.dims[d];
  }
  const size_t occ_bytes = ((nbits + 31) / 32) * 4;
  B2S_REQUIRE(occ_bytes <= GL_MAX_BYTES, B2S_E_CAPACITY, "global localisation: occupancy grid of %zu bytes, cap %zu", occ_bytes, GL_MAX_BYTES);
  B2S_REQUIRE((size_t)G.n_hyp * 4 <= GL_MAX_BYTES, B2S_E_CAPACITY, "global localisation: score array of %zu bytes, cap %zu", (size_t)G.n_hyp * 4,
              GL_MAX_BYTES);
  B2S_TRY(S.occ.ensure(occ_bytes, h->stream));
  B2S_CUDA(cudaMemsetAsync(S.occ.p, 0, occ_bytes, h->stream));
  G.occ.bits = S.occ.as<uint32_t>();
  if (union_grid) {
    launch_pdl(gl_union_occ_kernel, dim3((unsigned)grid_for(n_max, GL_THREADS), (unsigned)n_sm), GL_THREADS, 0, h->stream,
               static_cast<const GlJob*>(S.jobs.as<GlJob>()), G.box.inv, G.occ, S.occ.as<uint32_t>());
  } else {
    const b2s_cloud* map = sms[0]->cloud[0].get();
    launch_pdl(gl_occ_kernel, grid_for(map->n_max, GL_THREADS), GL_THREADS, 0, h->stream, static_cast<const double*>(map->xyz.as<double>()),
               static_cast<const int32_t*>(map->dn.as<int32_t>()), G.box.inv, G.occ, S.occ.as<uint32_t>());
  }
  h->launches++;
  gl_rotations(p, G.rot);
  B2S_TRY(S.rot.ensure(G.rot.size() * 8, h->stream));
  B2S_CUDA(cudaMemcpyAsync(S.rot.p, G.rot.data(), G.rot.size() * 8, cudaMemcpyHostToDevice, h->stream));
  B2S_TRY(S.hits.ensure((size_t)G.n_hyp * 4, h->stream));
  const long long nxy = (long long)G.box.nx * G.box.ny;
  const dim3 grid((unsigned)((nxy + GL_THREADS - 1) / GL_THREADS), (unsigned)p.n_yaw, (unsigned)p.n_z);
  B2S_REQUIRE(grid.y <= 65535 && grid.z <= 65535, B2S_E_INVALID, "global localisation: n_yaw and n_z must be <= 65535");
  launch_pdl(gl_score_kernel, grid, GL_THREADS, 0, h->stream, static_cast<const double*>(S.query.xyz.as<double>()),
             static_cast<const int32_t*>(S.query.dn.as<int32_t>()), static_cast<const double*>(S.rot.as<double>()), G.box, G.occ,
             S.hits.as<int32_t>());
  h->launches++;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

// the candidates of the scored hypotheses (selection and suppression); synchronises once
static int32_t gl_candidates(b2s_handle* h, const b2s_global_localization_params& p, GlScratch& S, const GlSetup& G, int32_t* n_cand,
                             std::vector<int32_t>& hyp, std::vector<int32_t>& hits, std::vector<double>& T) {
  const long long n = G.n_hyp;
  const int pool = GL_POOL_PER_CANDIDATE * p.n_candidates;
  const int blocks = grid_for((size_t)n, GL_THREADS, 4 * device_sms());
  B2S_TRY(S.hist.ensure(((size_t)G.nq + 1) * 4, h->stream));
  B2S_CUDA(cudaMemsetAsync(S.hist.p, 0, ((size_t)G.nq + 1) * 4, h->stream));
  B2S_TRY(S.sel.ensure(64, h->stream));
  for (DevBuf* d : {&S.eq, &S.rank, &S.flag, &S.pos}) B2S_TRY(d->ensure(((size_t)n + 1) * 4, h->stream));
  B2S_TRY(S.keys.ensure((size_t)pool * 8, h->stream));
  int32_t* sel = S.sel.as<int32_t>();
  int32_t* d_n = sel + 8;   // the hypothesis count the scans read
  launch_pdl(gl_set_n_kernel, 1, 1, 0, h->stream, d_n, (int32_t)n);
  launch_pdl(gl_hist_kernel, blocks, GL_THREADS, 0, h->stream, static_cast<const int32_t*>(S.hits.as<int32_t>()), n, S.hist.as<int32_t>());
  launch_pdl(gl_threshold_kernel, 1, 1, 0, h->stream, static_cast<const int32_t*>(S.hist.as<int32_t>()), G.nq, n, pool, sel);
  launch_pdl(gl_eq_kernel, blocks, GL_THREADS, 0, h->stream, static_cast<const int32_t*>(S.hits.as<int32_t>()), n,
             static_cast<const int32_t*>(sel), S.eq.as<int32_t>());
  h->launches += 4;
  B2S_TRY(scan_exclusive_i32(h, S.eq.as<int32_t>(), S.rank.as<int32_t>(), d_n, (size_t)n, nullptr, &S.scan_state));
  launch_pdl(gl_sel_kernel, blocks, GL_THREADS, 0, h->stream, static_cast<const int32_t*>(S.hits.as<int32_t>()), n,
             static_cast<const int32_t*>(sel), static_cast<const int32_t*>(S.rank.as<int32_t>()), S.flag.as<int32_t>());
  h->launches++;
  B2S_TRY(scan_exclusive_i32(h, S.flag.as<int32_t>(), S.pos.as<int32_t>(), d_n, (size_t)n, nullptr, &S.scan_state));
  launch_pdl(gl_scatter_kernel, blocks, GL_THREADS, 0, h->stream, static_cast<const int32_t*>(S.hits.as<int32_t>()), n,
             static_cast<const int32_t*>(S.flag.as<int32_t>()), static_cast<const int32_t*>(S.pos.as<int32_t>()), G.nq,
             S.keys.as<unsigned long long>());
  h->launches++;
  int P = 1;
  while (P < pool) P <<= 1;
  const size_t smem = (size_t)P * 8;
  B2S_CUDA(cudaFuncSetAttribute(gl_nms_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  B2S_TRY(S.cand_i32.ensure((1 + 2 * (size_t)GL_MAX_CANDIDATES) * 4, h->stream));
  B2S_TRY(S.cand_T.ensure(16 * (size_t)GL_MAX_CANDIDATES * 8, h->stream));
  const GlNms nm{p.nms_distance, p.nms_yaw, p.yaw0, p.yaw_step, p.n_candidates};
  launch_pdl(gl_nms_kernel, 1, GL_NMS_THREADS, smem, h->stream, static_cast<const unsigned long long*>(S.keys.as<unsigned long long>()),
             static_cast<const int32_t*>(sel), P, G.box, nm, static_cast<const double*>(S.rot.as<double>()), G.nq, S.cand_i32.as<int32_t>(),
             S.cand_T.as<double>());
  h->launches++;
  B2S_CUDA(cudaGetLastError());
  std::vector<int32_t> ci(1 + 2 * (size_t)GL_MAX_CANDIDATES);
  T.assign(16 * (size_t)GL_MAX_CANDIDATES, 0.0);
  B2S_TRY(read_back(h, {{ci.data(), S.cand_i32.p, ci.size() * 4}, {T.data(), S.cand_T.p, T.size() * 8}}));
  *n_cand = ci[0];
  hyp.resize((size_t)ci[0]); hits.resize((size_t)ci[0]);
  for (int k = 0; k < ci[0]; k++) { hyp[k] = ci[1 + 2 * k]; hits[k] = ci[2 + 2 * k]; }
  return B2S_OK;
}

// one registration per candidate, each what b2s_register_to_submap(match, sm_of[c], T_c, T_c) computes: the patch around T_c's translation
// in the candidate's submap, built by the same path into the candidate's own index, the same problem, GL_BATCH problems per ICP launch
// (the candidates of one launch may read different submaps).  The ICP kernel's cluster-wide sums are not reproducible to the last bit from
// one launch to the next (two b2s_register_to_submap calls on the same inputs differ there as well), so batching costs nothing in
// exactness.  Synchronises once.
static int32_t gl_refine(b2s_handle* h, const b2s_submap* const* sm_of, const b2s_cloud* match, int n, const double* Ts, GlScratch& S,
                         b2s_result* out) {
  if (n == 0) return B2S_OK;
  B2S_TRY(check_icp_params(h->cfg.icp));
  B2S_REQUIRE(match->has_normals || h->cfg.icp.reg_type != B2S_REG_GENERALIZED, B2S_E_NO_NORMALS, "GeneralizedIcp: the scan has no normals");
  const double cell = nn_cell(h, h->cfg.icp.max_corr_dist);
  const size_t work_each = (icp_work_bytes(match->n_max) + 7) / 8;
  B2S_TRY(S.problems.ensure(sizeof(IcpProblem) * (size_t)n, h->stream));
  B2S_TRY(S.work.ensure(work_each * 8 * (size_t)n, h->stream));
  B2S_TRY(S.results.ensure(sizeof(b2s_result) * (size_t)n, h->stream));
  B2S_TRY(S.hdrs.ensure(sizeof(GridHeader) * (size_t)n, h->stream));
  while ((int)h->batch_grids.size() < GL_BATCH) h->batch_grids.push_back(std::make_unique<GridIndex>());
  std::vector<IcpProblem> probs((size_t)n);
  for (int b0 = 0; b0 < n; b0 += GL_BATCH) {
    const int nb = n - b0 < GL_BATCH ? n - b0 : GL_BATCH;
    for (int i = 0; i < nb; i++) {
      const b2s_submap* sm = sm_of[b0 + i];
      const b2s_cloud* map = sm->cloud[0].get();
      const double* T = Ts + 16 * (size_t)(b0 + i);
      GridIndex* g = h->batch_grids[i].get();   // stream order keeps each build after the previous batch's ICP
      b2s_cropper c = h->cfg.scan.scan_matcher_cropper;   // ScanToMapRegistration.cpp:58 setPose(mapToRangeSensor)
      c.center[0] = T[3]; c.center[1] = T[7]; c.center[2] = T[11];
      CropDev patch = make_crop(&c);
      if (tile_patch_usable(sm, patch)) B2S_TRY(tile_patch_build(h, const_cast<b2s_submap*>(sm), patch, cell, g));
      else B2S_TRY(grid_build(h, g, map, cell, &patch, nullptr, sm->bbox.as<unsigned long long>(), &patch));
      B2S_CUDA(cudaMemcpyAsync(S.hdrs.as<GridHeader>() + b0 + i, g->hdr.p, sizeof(GridHeader), cudaMemcpyDeviceToDevice, h->stream));
      fill_problem(&probs[b0 + i], h->cfg.icp, match, g, map, T, nullptr, S.work.as<double>() + work_each * (b0 + i),
                   S.results.as<b2s_result>() + b0 + i);
    }
    IcpProblem* dst = S.problems.as<IcpProblem>() + b0;
    B2S_CUDA(cudaMemcpyAsync(dst, probs.data() + b0, sizeof(IcpProblem) * nb, cudaMemcpyHostToDevice, h->stream));
    B2S_TRY(icp_launch(h, nullptr, dst, nb, match->n_max));
  }
  std::vector<GridHeader> gh((size_t)n);
  B2S_CUDA(cudaMemcpyAsync(out, S.results.p, sizeof(b2s_result) * (size_t)n, cudaMemcpyDeviceToHost, h->stream));
  B2S_CUDA(cudaMemcpyAsync(gh.data(), S.hdrs.p, sizeof(GridHeader) * (size_t)n, cudaMemcpyDeviceToHost, h->stream));
  B2S_TRY(check_status(h));
  for (int i = 0; i < n; i++)
    if (gh[i].n <= 0) {   // an empty patch: b2s_register_to_submap reports B2S_E_EMPTY; here the candidate scores nothing
      memcpy(out[i].T, Ts + 16 * (size_t)i, 16 * sizeof(double));
      out[i].fitness = 0.0; out[i].inlier_rmse = 0.0; out[i].n_corr = 0; out[i].iters = 0;
    }
  return B2S_OK;
}

// SubmapCollection::findClosestSubmap (src/SubmapCollection.cpp:147-158) for the translation t: the first submap whose centre is
// nearest, the distance sqrt((dx^2 + dy^2) + dz^2) as Eigen's norm() of a 3-vector sums it
static int gl_closest(const double* t, const double* centers, int n_sm) {
  int best = 0;
  double best_d = 0.0;
  for (int s = 0; s < n_sm; s++) {
    const double dx = t[0] - centers[3 * s], dy = t[1] - centers[3 * s + 1], dz = t[2] - centers[3 * s + 2];
    volatile double sx = dx * dx, sy = dy * dy, sz = dz * dz;
    volatile double s2 = sx + sy;
    const double d = sqrt(s2 + sz);
    if (s == 0 || d < best_d) { best = s; best_d = d; }
  }
  return best;
}

// rules 1-6 over n_sm submaps.  centers (n_sm x 3, or nullptr: every candidate in sms[0]) assign each candidate its submap; union_grid as
// in gl_prepare.  out is cleared first; cand_submaps / winner_submap (optional) receive the submap of each listed candidate / the winner.
static int32_t gl_run(b2s_handle* h, const b2s_submap* const* sms, int n_sm, const double* centers, bool union_grid, const b2s_cloud* raw,
                      const b2s_global_localization_params& p, double min_refinement_fitness, b2s_global_localization_candidate* cands,
                      int32_t capacity, int32_t* cand_submaps, b2s_global_localization_result* out, int32_t* winner_submap) {
  memset(out, 0, sizeof(*out));
  out->winner_rank = -1; out->runner_up_fitness = -1.0;
  if (winner_submap) *winner_submap = -1;
  GlScratch S;
  GlSetup G;
  b2s_cloud* match = &S.match;
  B2S_TRY(gl_prepare(h, sms, n_sm, union_grid, raw, p, match, S, G));
  int32_t nc = 0;
  std::vector<int32_t> hyp, hits;
  std::vector<double> Ts;
  B2S_TRY(gl_candidates(h, p, S, G, &nc, hyp, hits, Ts));
  std::vector<int32_t> owner((size_t)nc, 0);
  std::vector<const b2s_submap*> sm_of((size_t)nc);
  for (int k = 0; k < nc; k++) {
    const double* T = Ts.data() + 16 * (size_t)k;
    const double t[3] = {T[3], T[7], T[11]};
    if (centers) owner[k] = gl_closest(t, centers, n_sm);
    sm_of[k] = sms[owner[k]];
  }
  std::vector<b2s_result> res((size_t)nc);
  B2S_TRY(gl_refine(h, sm_of.data(), match, nc, Ts.data(), S, res.data()));
  out->n_hypotheses = G.n_hyp; out->n_query = G.nq; out->n_candidates = nc;
  int w = -1;
  for (int k = 0; k < nc; k++) if (w < 0 || res[k].fitness > res[w].fitness) w = k;
  if (w >= 0) {
    memcpy(out->T, res[w].T, sizeof(out->T));
    out->fitness = res[w].fitness; out->inlier_rmse = res[w].inlier_rmse; out->winner_rank = w;
    out->found = res[w].fitness >= min_refinement_fitness ? 1 : 0;
    if (winner_submap) *winner_submap = owner[w];
    const double yw = gl_yaw_of(res[w].T);
    for (int k = 0; k < nc; k++) {
      const double dx = res[k].T[3] - res[w].T[3], dy = res[k].T[7] - res[w].T[7], dz = res[k].T[11] - res[w].T[11];
      volatile double sx = dx * dx, sy = dy * dy, sz = dz * dz;
      volatile double s2 = sx + sy;
      const double d = sqrt(s2 + sz);
      const double dyaw = fabs(remainder(gl_yaw_of(res[k].T) - yw, GL_TWO_PI));
      if ((d > p.nms_distance || dyaw > p.nms_yaw) && res[k].fitness > out->runner_up_fitness) out->runner_up_fitness = res[k].fitness;
    }
  }
  for (int k = 0; k < nc && k < capacity; k++) {
    if (cands) {
      b2s_global_localization_candidate& c = cands[k];
      memcpy(c.T_hypothesis, Ts.data() + 16 * (size_t)k, sizeof(c.T_hypothesis));
      c.hypothesis = hyp[k]; c.hits = hits[k]; c.icp = res[k];
    }
    if (cand_submaps) cand_submaps[k] = owner[k];
  }
  return B2S_OK;
}

// rules 1-3 only (the debug aids): the hits of every hypothesis and, optionally, the query cloud
static int32_t gl_debug_scores(b2s_handle* h, const b2s_submap* const* sms, int n_sm, bool union_grid, const b2s_cloud* raw,
                               const b2s_global_localization_params& p, int32_t* hits_out, size_t capacity, size_t* n_hypotheses,
                               double* query_out_or_null, size_t query_capacity, size_t* n_query) {
  GlScratch S;
  GlSetup G;
  B2S_TRY(gl_prepare(h, sms, n_sm, union_grid, raw, p, nullptr, S, G));
  *n_hypotheses = (size_t)G.n_hyp; *n_query = (size_t)G.nq;
  B2S_REQUIRE(capacity >= (size_t)G.n_hyp, B2S_E_CAPACITY, "hits_out holds %zu entries, %lld needed", capacity, G.n_hyp);
  B2S_REQUIRE(!query_out_or_null || query_capacity >= (size_t)G.nq, B2S_E_CAPACITY, "query_out holds %zu points, %d needed", query_capacity, G.nq);
  B2S_CUDA(cudaMemcpyAsync(hits_out, S.hits.p, (size_t)G.n_hyp * 4, cudaMemcpyDeviceToHost, h->stream));
  if (query_out_or_null) B2S_CUDA(cudaMemcpyAsync(query_out_or_null, S.query.xyz.p, (size_t)G.nq * 24, cudaMemcpyDeviceToHost, h->stream));
  return check_status(h);
}

// the argument rules of the submap-set calls (rule 7 of M4)
static int32_t gl_check_submaps(b2s_handle* h, const b2s_submap* const* sms, int32_t n_submaps, const double* centers) {
  B2S_REQUIRE(n_submaps >= 1, B2S_E_INVALID, "global localisation: n_submaps must be >= 1");
  B2S_REQUIRE(n_submaps <= B2S_ASSEMBLY_MAX_SUBMAPS, B2S_E_UNSUPPORTED, "global localisation: %d submaps, at most %d", n_submaps,
              B2S_ASSEMBLY_MAX_SUBMAPS);
  for (int32_t s = 0; s < n_submaps; s++) {
    B2S_REQUIRE(sms[s], B2S_E_INVALID, "global localisation: null submap %d", s);
    B2S_REQUIRE(sms[s]->h == h, B2S_E_INVALID, "global localisation: submap %d belongs to another handle", s);
    if (centers)
      B2S_REQUIRE(finite(centers[3 * s]) && finite(centers[3 * s + 1]) && finite(centers[3 * s + 2]), B2S_E_INVALID,
                  "global localisation: the centre of submap %d is not finite", s);
  }
  return B2S_OK;
}

}  // namespace b2s

extern "C" {

void b2s_default_global_localization_params(b2s_global_localization_params* p) {
  memset(p, 0, sizeof(*p));
  p->x_min = 1.0; p->x_max = -1.0; p->y_min = 1.0; p->y_max = -1.0;   // x_min > x_max: the map's live extent
  p->step = 0.25;
  p->z0 = 0.0; p->z_step = 0.25; p->n_z = 1;
  p->n_yaw = 144; p->yaw0 = -3.141592653589793; p->yaw_step = GL_TWO_PI / 144.0;
  p->roll = 0.0; p->pitch = 0.0;
  p->score_voxel = 1.0;
  p->n_candidates = 16;
  p->nms_distance = 1.0; p->nms_yaw = 10.0 * 3.141592653589793 / 180.0;
}

int32_t b2s_submap_global_localization(b2s_handle* h, const b2s_submap* sm, const b2s_cloud* raw_scan, const b2s_global_localization_params* p,
                                       double min_refinement_fitness, b2s_global_localization_candidate* candidates_or_null, int32_t capacity,
                                       b2s_global_localization_result* out) {
  B2S_REQUIRE(h && sm && raw_scan && p && out, B2S_E_INVALID, "null argument");
  B2S_REQUIRE(sm->h == h && raw_scan->h == h, B2S_E_INVALID, "the submap or the scan belongs to another handle");
  B2S_REQUIRE(!candidates_or_null || capacity >= 0, B2S_E_INVALID, "negative capacity");
  LOCK(h);
  return gl_run(h, &sm, 1, nullptr, false, raw_scan, *p, min_refinement_fitness, candidates_or_null, candidates_or_null ? capacity : 0, nullptr,
                out, nullptr);
}

int32_t b2s_submaps_global_localization(b2s_handle* h, const b2s_submap* const* sms, int32_t n_submaps, const double* centers,
                                        const b2s_cloud* raw_scan, const b2s_global_localization_params* p, double min_refinement_fitness,
                                        b2s_global_localization_candidate* candidates_or_null, int32_t capacity,
                                        int32_t* candidate_submaps_or_null, b2s_global_localization_result* out, int32_t* winner_submap) {
  B2S_REQUIRE(h && sms && centers && raw_scan && p && out && winner_submap, B2S_E_INVALID, "null argument");
  B2S_REQUIRE(raw_scan->h == h, B2S_E_INVALID, "the scan belongs to another handle");
  B2S_REQUIRE((!candidates_or_null && !candidate_submaps_or_null) || capacity >= 0, B2S_E_INVALID, "negative capacity");
  B2S_TRY(gl_check_submaps(h, sms, n_submaps, centers));
  LOCK(h);
  const bool listed = candidates_or_null || candidate_submaps_or_null;
  return gl_run(h, sms, n_submaps, centers, true, raw_scan, *p, min_refinement_fitness, candidates_or_null, listed ? capacity : 0,
                candidate_submaps_or_null, out, winner_submap);
}

int32_t b2s_debug_global_localization_scores(b2s_handle* h, const b2s_submap* sm, const b2s_cloud* raw_scan, const b2s_global_localization_params* p,
                                             int32_t* hits_out, size_t capacity, size_t* n_hypotheses, double* query_out_or_null,
                                             size_t query_capacity, size_t* n_query) {
  B2S_REQUIRE(h && sm && raw_scan && p && hits_out && n_hypotheses && n_query, B2S_E_INVALID, "null argument");
  B2S_REQUIRE(sm->h == h && raw_scan->h == h, B2S_E_INVALID, "the submap or the scan belongs to another handle");
  LOCK(h);
  return gl_debug_scores(h, &sm, 1, false, raw_scan, *p, hits_out, capacity, n_hypotheses, query_out_or_null, query_capacity, n_query);
}

int32_t b2s_debug_submaps_global_localization_scores(b2s_handle* h, const b2s_submap* const* sms, int32_t n_submaps, const b2s_cloud* raw_scan,
                                                     const b2s_global_localization_params* p, int32_t* hits_out, size_t capacity,
                                                     size_t* n_hypotheses, double* query_out_or_null, size_t query_capacity, size_t* n_query) {
  B2S_REQUIRE(h && sms && raw_scan && p && hits_out && n_hypotheses && n_query, B2S_E_INVALID, "null argument");
  B2S_REQUIRE(raw_scan->h == h, B2S_E_INVALID, "the scan belongs to another handle");
  B2S_TRY(gl_check_submaps(h, sms, n_submaps, nullptr));
  LOCK(h);
  return gl_debug_scores(h, sms, n_submaps, true, raw_scan, *p, hits_out, capacity, n_hypotheses, query_out_or_null, query_capacity, n_query);
}

}  // extern "C"
