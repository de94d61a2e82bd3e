// constraints.cu -- the constraints between two resident submaps, batched over pairs and read from the map slots:
//   L2  the odometry constraints between consecutive submaps (buildOdometryConstraint, core/src/constraint_builders.cpp:33-90)
//   L3  the refinement of loop closures (PlaceRecognition::buildLoopClosureConstraints, src/PlaceRecognition.cpp:96-149)
// Both run through one driver (op_submap_constraints below); they differ in the overlap's sourceToTarget (the identity / the RANSAC
// proposal), in whether and from where the ICP runs, in the radii and in the record they fill.
//
//   overlap                    op_overlap_batch (overlap.cu): one set of launches for every pair, straight from the map slots
//   target-overlap indexes     grid_build_batch (grid_index.cu): one build for all pairs, shared by the ICP and K-info-wide
//   refinement                 the batched K-icp-iter launch with the job's estimator (icp.cu): L2 point-to-plane, L3 the caller's
//   information matrix         K-info-wide (below): [O3D] GetInformationMatrixFromPointClouds over ALL SMs
//
// K-info-wide.  b2s_information_matrix evaluates on K-icp-iter, one registration per 8-CTA cluster: sized for scans of ~10^4 points,
// while a submap overlap holds ~10^5.  Here the source points of every pair are dealt out in tiles of WI_TILE points
// (pair k owns tiles [tile0_k, tile0_k + ntiles_k), sized by the host-side bound of its overlap), and a grid-stride loop of CTAs
// walks the tiles of the whole batch.  Per point: the transform of [O3D]'s branch (none at the identity), the exact 1-NN of the
// project (strict d2 < r2, ties to the lower original index) against the target overlap's GridIndex, and the moment terms
// EST_INFORMATION accumulates.  Every tile writes its own partial sums (fixed order within the tile: per thread, warp tree, warps
// in rank order); a second kernel adds a pair's tile partials in tile order.  No atomics touch the sums, and the result does not
// depend on the grid size: it repeats bit for bit from run to run and equals one call per pair.
#include "common.cuh"

namespace b2s {

constexpr int WI_THREADS = 256;
constexpr int WI_TILE = 1024;   // points per tile: 4 per thread
constexpr int WI_MOM = 10;      // sum x, y, z, xx, yy, zz, xy, xz, yz, count

struct InfoPair {
  const double* src_xyz; const int32_t* src_n; const int32_t* tgt_n;   // the two overlap clouds
  const GridHeader* ghdr; const int32_t* cell_start; const double4* pts;   // the child overlap's index
  const b2s_result* icp;   // refined: the ICP result (T is read from it); nullptr: identity, no refinement
  int32_t tile0, ntiles;
};

// [O3D] TransformationEstimation... isIdentity(1e-12), as K-icp-iter decides whether GetInformationMatrixFromPointClouds transforms
__device__ bool wi_is_identity(const double* T) {
  for (int i = 0; i < 4; i++)
    for (int j = 0; j < 4; j++) {
      const double v = T[4 * i + j];
      if (i == j) { if (!(fabs(v - 1.0) <= 1e-12 * fmin(fabs(v), 1.0))) return false; }
      else if (!(fabs(v) <= 1e-12)) return false;
    }
  return true;
}

__global__ void __launch_bounds__(WI_THREADS) info_wide_kernel(const InfoPair* __restrict__ pairs, int npairs, int total_tiles, double r,
                                                               double* __restrict__ partials) {
  pdl_wait();
  __shared__ GridHeader sg;
  __shared__ double sT[16];
  __shared__ int s_apply;
  __shared__ double sred[WI_THREADS / 32][WI_MOM];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    int lo = 0, hi = npairs - 1;   // the pair whose tile range holds `tile` (tile0 ascending)
    while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (pairs[mid].tile0 <= tile) lo = mid; else hi = mid - 1; }
    const InfoPair P = pairs[lo];
    if (tid == 0) {
      sg = *P.ghdr;
      for (int i = 0; i < 16; i++) sT[i] = P.icp ? P.icp->T[i] : ((i % 5 == 0) ? 1.0 : 0.0);
      s_apply = wi_is_identity(sT) ? 0 : 1;   // [O3D]: if (!transformation.isIdentity()) pcd.Transform(transformation)
    }
    __syncthreads();
    const int n = *P.src_n;
    const int base = (tile - P.tile0) * WI_TILE;
    double acc[WI_MOM];
#pragma unroll
    for (int m = 0; m < WI_MOM; m++) acc[m] = 0.0;
    if (base < n) {
      for (int u = 0; u < WI_TILE / WI_THREADS; u++) {
        const int i = base + u * WI_THREADS + tid;
        if (i >= n) break;
        double px = P.src_xyz[3 * (size_t)i], py = P.src_xyz[3 * (size_t)i + 1], pz = P.src_xyz[3 * (size_t)i + 2];
        if (s_apply) {   // [O3D] TransformPoints with w == 1 for a rigid T; the association of K-icp-iter
          const double x = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(sT[0], px), __dmul_rn(sT[1], py)), __dmul_rn(sT[2], pz)), sT[3]);
          const double y = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(sT[4], px), __dmul_rn(sT[5], py)), __dmul_rn(sT[6], pz)), sT[7]);
          const double z = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(sT[8], px), __dmul_rn(sT[9], py)), __dmul_rn(sT[10], pz)), sT[11]);
          px = x; py = y; pz = z;
        }
        if (!(px == px && py == py && pz == pz) || sg.n == 0) continue;
        double d2;
        const int slot = grid_nearest(sg, P.cell_start, P.pts, px, py, pz, r, &d2);
        if (slot < 0) continue;
        const double4 q = P.pts[slot];   // the moments of the matched TARGET point (EST_INFORMATION)
        acc[0] += q.x; acc[1] += q.y; acc[2] += q.z;
        acc[3] += q.x * q.x; acc[4] += q.y * q.y; acc[5] += q.z * q.z;
        acc[6] += q.x * q.y; acc[7] += q.x * q.z; acc[8] += q.y * q.z;
        acc[9] += 1.0;
      }
    }
#pragma unroll
    for (int m = 0; m < WI_MOM; m++) {
      const double v = warp_sum(acc[m]);
      if (lane == 0) sred[warp][m] = v;
    }
    __syncthreads();
    if (tid < WI_MOM) {
      double v = 0.0;
      for (int w = 0; w < WI_THREADS / 32; w++) v += sred[w][tid];
      partials[(size_t)tile * WI_MOM + tid] = v;
    }
    __syncthreads();   // sg / sT / sred are rewritten by the next tile
  }
}

// the record of one pair from its information matrix M (row-major): L2's constraint ...
__device__ __forceinline__ void finish_record(b2s_odometry_constraint& o, const InfoPair& P, const double* M, double) {
  for (int i = 0; i < 36; i++) o.information[i] = M[i];
  if (P.icp) {
    o.icp = *P.icp;
    for (int i = 0; i < 16; i++) o.T[i] = P.icp->T[i];
  } else {
    memset(&o.icp, 0, sizeof(o.icp));
    for (int i = 0; i < 16; i++) o.T[i] = (i % 5 == 0) ? 1.0 : 0.0;
  }
  o.n_source_overlap = *P.src_n;
  o.n_target_overlap = *P.tgt_n;
  o.refined = P.icp ? 1 : 0;
}
// ... and L3's refinement: the ICP always ran; the fitness gate of PlaceRecognition.cpp:118, NaN passing as the reference's `<` lets it
__device__ __forceinline__ void finish_record(b2s_loop_closure_refinement& o, const InfoPair& P, const double* M, double min_fitness) {
  for (int i = 0; i < 36; i++) o.information[i] = M[i];
  o.icp = *P.icp;
  o.n_source_overlap = *P.src_n;
  o.n_target_overlap = *P.tgt_n;
  o.accepted = !(P.icp->fitness < min_fitness) ? 1 : 0;
}

// one CTA per pair: the tile partials in tile order, the 6x6 of [O3D] (rows (0,z,-y,1,0,0), (-z,0,x,0,1,0), (y,-x,0,0,0,1) summed over
// the matched target points, as K-icp-iter's info_from_moments), and the whole record
template <class Rec>
__global__ void info_finish_kernel(const InfoPair* __restrict__ pairs, const double* __restrict__ partials, double min_fitness, Rec* __restrict__ out) {
  pdl_wait();
  __shared__ double t[WI_MOM];
  const InfoPair P = pairs[blockIdx.x];
  if (threadIdx.x < WI_MOM) {
    double v = 0.0;
    for (int k = 0; k < P.ntiles; k++) v += partials[(size_t)(P.tile0 + k) * WI_MOM + threadIdx.x];
    t[threadIdx.x] = v;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  const double sx = t[0], sy = t[1], sz = t[2], xx = t[3], yy = t[4], zz = t[5], xy = t[6], xz = t[7], yz = t[8], n = t[9];
  const double M[36] = {zz + yy, -xy, -xz, 0.0, -sz, sy,  -xy, zz + xx, -yz, sz, 0.0, -sx,  -xz, -yz, yy + xx, -sy, sx, 0.0,
                        0.0, sz, -sy, n, 0.0, 0.0,        -sz, 0.0, sx, 0.0, n, 0.0,        sy, -sx, 0.0, 0.0, 0.0, n};
  finish_record(out[blockIdx.x], P, M, min_fitness);
}

namespace {
// what one batch of pair constraints runs; the two kinds differ only here
struct PairJob {
  const double* inits;       // n row-major 4x4 (host): the overlap's sourceToTarget and the ICP's start; nullptr = the identity
  double overlap_voxel;      // edge of the overlap's voxels
  int32_t min_pts;           // minNumPointsPerVoxel
  bool refine;               // run the ICP
  int32_t estimator;         // B2S_REG_*: its estimator, one for the whole batch
  int32_t max_iter;
  double rel_fitness, rel_rmse;
  double radius;             // max_correspondence_distance of the ICP and of GetInformationMatrixFromPointClouds (equal in both kinds)
  double grid_cell;          // cell edge of the target-overlap indexes
  double min_fitness;        // L3's gate (the L2 record has none)
};

// overlap -> target-overlap indexes -> [ICP] -> K-info-wide -> records, for n (sources[k], targets[k]) pairs.  so_out / to_out: the
// caller's overlap clouds or nullptr (the handle's own); out: host records.  One set of launches, synchronises once at the end.
template <class Rec>
int32_t op_submap_constraints(b2s_handle* h, int n, const b2s_submap* const* sources, const b2s_submap* const* targets, const PairJob& J,
                              b2s_cloud* const* so_out, b2s_cloud* const* to_out, Rec* out) {
  // the overlap clouds: the caller's, or the handle's own
  while (h->odo_clouds.size() < (size_t)(2 * n)) {
    std::unique_ptr<b2s_cloud> c;
    B2S_TRY(make_cloud(h, 1, true, false, &c));
    h->odo_clouds.push_back(std::move(c));
  }
  std::vector<const b2s_submap*> maps((size_t)(2 * n));
  std::vector<b2s_cloud*> outs((size_t)(2 * n));
  for (int k = 0; k < n; k++) {
    maps[2 * k] = sources[k]; maps[2 * k + 1] = targets[k];
    outs[2 * k] = so_out ? so_out[k] : h->odo_clouds[2 * k].get();
    outs[2 * k + 1] = to_out ? to_out[k] : h->odo_clouds[2 * k + 1].get();
  }
  // page-locked staging of every table this call uploads (nothing waits for the device before the final read-back)
  Layout S;
  const OverlapTables ov = overlap_tables(S, n);
  const size_t st_icp = S.off((size_t)n * sizeof(IcpProblem)), st_info = S.off((size_t)n * sizeof(InfoPair));
  if (h->odo_stage.cap < S.size) B2S_TRY(h->odo_stage.alloc(2 * S.size));   // the last call synchronised
  unsigned char* stage = h->odo_stage.as<unsigned char>();
  B2S_TRY(op_overlap_batch(h, n, maps.data(), J.inits, J.overlap_voxel, J.min_pts, outs.data(), stage, ov));

  // the index of every target overlap, one batched build
  std::vector<GridIndex*> grids((size_t)n);
  std::vector<const b2s_cloud*> tclouds((size_t)n);
  while (h->batch_grids.size() < (size_t)n) h->batch_grids.push_back(std::make_unique<GridIndex>());
  for (int k = 0; k < n; k++) { grids[k] = h->batch_grids[k].get(); tclouds[k] = outs[2 * k + 1]; }
  B2S_TRY(grid_build_batch(h, grids.data(), tclouds.data(), n, J.grid_cell));

  // refinement: RegistrationICP / RegistrationGeneralizedICP(sourceOverlap, targetOverlap, r, T0, estimator, criteria) for every pair in one launch
  if (J.refine) {
    b2s_icp_params icp;
    memset(&icp, 0, sizeof(icp));
    icp.reg_type = J.estimator; icp.max_iter = J.max_iter; icp.max_corr_dist = J.radius; icp.rel_fitness = J.rel_fitness;
    icp.rel_rmse = J.rel_rmse;
    size_t work_total = 0, max_src = 1;
    for (int k = 0; k < n; k++) {
      work_total += (icp_work_bytes(outs[2 * k]->n_max) + 7) / 8;
      if (outs[2 * k]->n_max > max_src) max_src = outs[2 * k]->n_max;
    }
    B2S_TRY(h->work_xyz.ensure(work_total * 8, h->stream));
    B2S_TRY(h->problems.ensure(sizeof(IcpProblem) * (size_t)n, h->stream));
    B2S_TRY(h->results.ensure(sizeof(b2s_result) * (size_t)n, h->stream));
    IcpProblem* probs = reinterpret_cast<IcpProblem*>(stage + st_icp);
    const double I[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    size_t woff = 0;
    for (int k = 0; k < n; k++) {
      fill_problem(&probs[k], icp, outs[2 * k], grids[k], outs[2 * k + 1], J.inits ? J.inits + 16 * (size_t)k : I, nullptr,
                   h->work_xyz.as<double>() + woff, h->results.as<b2s_result>() + k);
      woff += (icp_work_bytes(outs[2 * k]->n_max) + 7) / 8;
    }
    B2S_CUDA(cudaMemcpyAsync(h->problems.p, probs, sizeof(IcpProblem) * (size_t)n, cudaMemcpyHostToDevice, h->stream));
    B2S_TRY(icp_launch(h, nullptr, h->problems.as<IcpProblem>(), n, max_src, J.estimator));
  }

  // the information matrices: K-info-wide over the tiles of every pair, then one CTA per pair
  InfoPair* ip = reinterpret_cast<InfoPair*>(stage + st_info);
  int tiles = 0;
  for (int k = 0; k < n; k++) {
    const b2s_cloud* s = outs[2 * k];
    InfoPair& P = ip[k];
    P.src_xyz = s->xyz.as<double>(); P.src_n = s->dn.as<int32_t>(); P.tgt_n = outs[2 * k + 1]->dn.as<int32_t>();
    P.ghdr = grids[k]->hdr.as<GridHeader>(); P.cell_start = grid_starts(grids[k]); P.pts = grids[k]->pts.as<double4>();
    P.icp = J.refine ? h->results.as<b2s_result>() + k : nullptr;
    const size_t nt = (s->n_max + WI_TILE - 1) / WI_TILE;
    P.tile0 = tiles; P.ntiles = (int32_t)(nt > 0 ? nt : 1);
    tiles += P.ntiles;
  }
  InfoPair* dpairs = nullptr;
  double* partials = nullptr;
  Rec* dout = nullptr;
  B2S_TRY(carve(h->odo_info, h->stream, [&](Layout& D) {
    dpairs = D.take<InfoPair>(n); partials = D.take<double>((size_t)tiles * WI_MOM); dout = D.take<Rec>(n);
  }));
  B2S_CUDA(cudaMemcpyAsync(dpairs, ip, (size_t)n * sizeof(InfoPair), cudaMemcpyHostToDevice, h->stream));
  {
    ProfScope prof(h, PK_ICP);
    launch_pdl(info_wide_kernel, grid_for((size_t)tiles, 1, 4 * device_sms()), WI_THREADS, 0, h->stream, dpairs, n, tiles, J.radius, partials);
    launch_pdl(info_finish_kernel<Rec>, n, 32, 0, h->stream, dpairs, (const double*)partials, J.min_fitness, dout);
    h->launches += 2;
  }
  B2S_CUDA(cudaGetLastError());
  B2S_CUDA(cudaMemcpyAsync(out, dout, (size_t)n * sizeof(Rec), cudaMemcpyDeviceToHost, h->stream));
  return check_status(h);
}
}  // namespace

int32_t op_odometry_constraints(b2s_handle* h, int n, const b2s_submap* const* sources, const b2s_submap* const* targets,
                                const b2s_odometry_constraint_params& p, double voxel, b2s_cloud* const* so_out, b2s_cloud* const* to_out,
                                b2s_odometry_constraint* out) {
  PairJob J;
  J.inits = nullptr;                                   // the overlap and the ICP at the identity (:51-58, :62-68)
  J.overlap_voxel = p.overlap_factor * voxel;
  J.min_pts = p.min_points_per_voxel;
  J.refine = p.refine != 0;
  J.estimator = B2S_REG_POINT_TO_PLANE;               // raw RegistrationICP with TransformationEstimationPointToPlane (:62-68)
  J.max_iter = p.max_iter; J.rel_fitness = p.rel_fitness; J.rel_rmse = p.rel_rmse;
  J.radius = p.icp_factor * voxel;                     // icpMaxCorrespondenceDistance, also the information matrix's radius (:36, :71)
  J.grid_cell = 0.5 * J.radius;
  J.min_fitness = 0.0;
  return op_submap_constraints(h, n, sources, targets, J, so_out, to_out, out);
}

int32_t op_loop_closure_refinement(b2s_handle* h, const b2s_submap* source, int n, const b2s_submap* const* targets, const double* inits,
                                   const b2s_loop_closure_refinement_params& p, double voxel, b2s_cloud* const* so_out, b2s_cloud* const* to_out,
                                   b2s_loop_closure_refinement* out) {
  const std::vector<const b2s_submap*> sources((size_t)n, source);
  PairJob J;
  J.inits = inits;                                     // the RANSAC proposal: the overlap's sourceToTarget and the ICP's start (:103, :110)
  J.overlap_voxel = p.overlap_factor * voxel;          // :100
  J.min_pts = p.min_points_per_voxel;
  J.refine = true;
  J.estimator = p.reg_type;                            // cloudRegistrationFactory(toCloudRegistrationType(scanMatcher_)) (:47)
  J.max_iter = p.max_iter; J.rel_fitness = p.rel_fitness; J.rel_rmse = p.rel_rmse;
  J.radius = p.max_corr_dist;                          // maxIcpCorrespondenceDistance_: the ICP's (:46) and the information's (:149)
  J.grid_cell = nn_cell(h, p.max_corr_dist);           // the cell b2s_register_batch indexes its targets at
  J.min_fitness = p.min_refinement_fitness;
  return op_submap_constraints(h, n, sources.data(), targets, J, so_out, to_out, out);
}

}  // namespace b2s
