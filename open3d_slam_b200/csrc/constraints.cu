// constraints.cu -- L2: the odometry constraints between consecutive submaps (buildOdometryConstraint, core/src/constraint_builders.cpp:33-90),
// batched over (parent, child) pairs and read from the resident submaps.
//
//   overlap at the identity    op_overlap_batch (overlap.cu): one set of launches for every pair, straight from the map slots
//   child-overlap indexes      grid_build_batch (grid_index.cu): one build for all pairs
//   refinement (opt-in)        the batched K-icp-iter launch with the point-to-plane estimator forced (icp.cu)
//   information matrix         K-info-wide (below): [O3D] GetInformationMatrixFromPointClouds over ALL SMs
//
// K-info-wide.  b2s_information_matrix evaluates on K-icp-iter, one registration per 8-CTA cluster: sized for scans of ~10^4 points,
// while an odometry-constraint overlap holds ~10^5.  Here the source points of every pair are dealt out in tiles of WI_TILE points
// (pair k owns tiles [tile0_k, tile0_k + ntiles_k), sized by the host-side bound of its overlap), and a grid-stride loop of CTAs
// walks the tiles of the whole batch.  Per point: the transform of [O3D]'s branch (none at the identity), the exact 1-NN of the
// project (strict d2 < r2, ties to the lower original index) against the child overlap's GridIndex, and the moment terms
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

// exact 1-NN within r: every cell that overlaps the box [q - r, q + r] (cell indices by the build's floor((v - o) * inv), which is
// monotone, clamped like the build clamps), strict d2 < r2 with dist2_exact, equal distances to the lower original index.
// Returns the slot in g's point array, -1 = none.
__device__ __forceinline__ int wi_nearest(const GridHeader& g, const int32_t* __restrict__ cs, const double4* __restrict__ pts, double qx, double qy,
                                          double qz, double rad, double r2) {
  const double ox = g.origin[0], oy = g.origin[1], oz = g.origin[2], inv = g.inv_cell;
  const int nx = g.dims[0], ny = g.dims[1], nz = g.dims[2];
  const int ix0 = (int)fmin(fmax(floor((qx - rad - ox) * inv), 0.0), (double)(nx - 1));
  const int ix1 = (int)fmin(fmax(floor((qx + rad - ox) * inv), 0.0), (double)(nx - 1));
  const int iy0 = (int)fmin(fmax(floor((qy - rad - oy) * inv), 0.0), (double)(ny - 1));
  const int iy1 = (int)fmin(fmax(floor((qy + rad - oy) * inv), 0.0), (double)(ny - 1));
  const int iz0 = (int)fmin(fmax(floor((qz - rad - oz) * inv), 0.0), (double)(nz - 1));
  const int iz1 = (int)fmin(fmax(floor((qz + rad - oz) * inv), 0.0), (double)(nz - 1));
  double best = r2;
  int bidx = 0x7fffffff, bslot = -1;
  for (int z = iz0; z <= iz1; z++)
    for (int y = iy0; y <= iy1; y++) {
      const int row = (z * ny + y) * nx;
      const int s = cs[row + ix0], e = cs[row + ix1 + 1];
      for (int j = s; j < e; j++) {
        const double4 p = pts[j];
        const double d = dist2_exact(qx, qy, qz, p.x, p.y, p.z);
        const int idx = (int)__double_as_longlong(p.w);
        if (d < best || (d == best && bslot >= 0 && idx < bidx)) { best = d; bidx = idx; bslot = j; }
      }
    }
  return bslot;
}

__global__ void __launch_bounds__(WI_THREADS) info_wide_kernel(const InfoPair* __restrict__ pairs, int npairs, int total_tiles, double r,
                                                               double* __restrict__ partials) {
  pdl_wait();
  __shared__ GridHeader sg;
  __shared__ double sT[16];
  __shared__ int s_apply;
  __shared__ double sred[WI_THREADS / 32][WI_MOM];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const double r2 = r * r;
  const double rad = r * (1.0 + 1e-12) + 1e-300;
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
        const int slot = wi_nearest(sg, P.cell_start, P.pts, px, py, pz, rad, r2);
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

// one CTA per pair: the tile partials in tile order, the 6x6 of [O3D] (rows (0,z,-y,1,0,0), (-z,0,x,0,1,0), (y,-x,0,0,0,1) summed over
// the matched target points, as K-icp-iter's info_from_moments), and the whole constraint record
__global__ void info_finish_kernel(const InfoPair* __restrict__ pairs, const double* __restrict__ partials, b2s_odometry_constraint* __restrict__ out) {
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
  b2s_odometry_constraint& o = out[blockIdx.x];
  const double sx = t[0], sy = t[1], sz = t[2], xx = t[3], yy = t[4], zz = t[5], xy = t[6], xz = t[7], yz = t[8], n = t[9];
  const double M[36] = {zz + yy, -xy, -xz, 0.0, -sz, sy,  -xy, zz + xx, -yz, sz, 0.0, -sx,  -xz, -yz, yy + xx, -sy, sx, 0.0,
                        0.0, sz, -sy, n, 0.0, 0.0,        -sz, 0.0, sx, 0.0, n, 0.0,        sy, -sx, 0.0, 0.0, 0.0, n};
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

size_t op_overlap_batch_stage_bytes(int n);
int32_t op_overlap_batch(b2s_handle* h, int n, const b2s_submap* const* maps, double voxel, int min_pts, b2s_cloud* const* outs,
                         unsigned char* host_stage);

int32_t op_odometry_constraints(b2s_handle* h, int n, const b2s_submap* const* sources, const b2s_submap* const* targets,
                                const b2s_odometry_constraint_params& p, double voxel, b2s_cloud* const* so_out, b2s_cloud* const* to_out,
                                b2s_odometry_constraint* out) {
  auto al = [](size_t b) { return (b + 255) & ~(size_t)255; };
  const double r = p.icp_factor * voxel;   // icpMaxCorrespondenceDistance, also the information matrix's radius (:36, :71)
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
  const size_t st_ov = al(op_overlap_batch_stage_bytes(n)), st_icp = al((size_t)n * sizeof(IcpProblem)), st_info = (size_t)n * sizeof(InfoPair);
  if (h->odo_stage.cap < st_ov + st_icp + st_info) B2S_TRY(h->odo_stage.alloc(2 * (st_ov + st_icp + st_info)));   // the last call synchronised
  unsigned char* stage = h->odo_stage.as<unsigned char>();
  B2S_TRY(op_overlap_batch(h, n, maps.data(), p.overlap_factor * voxel, p.min_points_per_voxel, outs.data(), stage));

  // the index of every child overlap, one batched build
  std::vector<GridIndex*> grids((size_t)n);
  std::vector<const b2s_cloud*> tclouds((size_t)n);
  while (h->batch_grids.size() < (size_t)n) h->batch_grids.push_back(std::make_unique<GridIndex>());
  for (int k = 0; k < n; k++) { grids[k] = h->batch_grids[k].get(); tclouds[k] = outs[2 * k + 1]; }
  B2S_TRY(grid_build_batch(h, grids.data(), tclouds.data(), n, 0.5 * r));

  // refinement: RegistrationICP(source, target, r, Identity, PointToPlane, criteria) for every pair in one launch (:62-68)
  if (p.refine) {
    b2s_icp_params icp;
    memset(&icp, 0, sizeof(icp));
    icp.reg_type = B2S_REG_POINT_TO_PLANE; icp.max_iter = p.max_iter; icp.max_corr_dist = r; icp.rel_fitness = p.rel_fitness; icp.rel_rmse = p.rel_rmse;
    size_t work_total = 0, max_src = 1;
    for (int k = 0; k < n; k++) {
      work_total += (icp_work_bytes(outs[2 * k]->n_max) + 7) / 8;
      if (outs[2 * k]->n_max > max_src) max_src = outs[2 * k]->n_max;
    }
    B2S_TRY(h->work_xyz.ensure(work_total * 8, h->stream));
    B2S_TRY(h->problems.ensure(sizeof(IcpProblem) * (size_t)n, h->stream));
    B2S_TRY(h->results.ensure(sizeof(b2s_result) * (size_t)n, h->stream));
    IcpProblem* probs = reinterpret_cast<IcpProblem*>(stage + st_ov);
    const double I[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    size_t woff = 0;
    for (int k = 0; k < n; k++) {
      fill_problem(&probs[k], icp, outs[2 * k], grids[k], outs[2 * k + 1], I, nullptr, h->work_xyz.as<double>() + woff, h->results.as<b2s_result>() + k);
      woff += (icp_work_bytes(outs[2 * k]->n_max) + 7) / 8;
    }
    B2S_CUDA(cudaMemcpyAsync(h->problems.p, probs, sizeof(IcpProblem) * (size_t)n, cudaMemcpyHostToDevice, h->stream));
    B2S_TRY(icp_launch(h, nullptr, h->problems.as<IcpProblem>(), n, max_src, B2S_REG_POINT_TO_PLANE));
  }

  // the information matrices: K-info-wide over the tiles of every pair, then one CTA per pair
  InfoPair* ip = reinterpret_cast<InfoPair*>(stage + st_ov + st_icp);
  int tiles = 0;
  for (int k = 0; k < n; k++) {
    const b2s_cloud* s = outs[2 * k];
    InfoPair& P = ip[k];
    P.src_xyz = s->xyz.as<double>(); P.src_n = s->dn.as<int32_t>(); P.tgt_n = outs[2 * k + 1]->dn.as<int32_t>();
    P.ghdr = grids[k]->hdr.as<GridHeader>(); P.cell_start = grid_starts(grids[k]); P.pts = grids[k]->pts.as<double4>();
    P.icp = p.refine ? h->results.as<b2s_result>() + k : nullptr;
    const size_t nt = (s->n_max + WI_TILE - 1) / WI_TILE;
    P.tile0 = tiles; P.ntiles = (int32_t)(nt > 0 ? nt : 1);
    tiles += P.ntiles;
  }
  const size_t b_pairs = al((size_t)n * sizeof(InfoPair)), b_part = al((size_t)tiles * WI_MOM * 8);
  B2S_TRY(h->odo_info.ensure(b_pairs + b_part + (size_t)n * sizeof(b2s_odometry_constraint), h->stream));
  unsigned char* dev = h->odo_info.as<unsigned char>();
  const InfoPair* dpairs = reinterpret_cast<const InfoPair*>(dev);
  double* partials = reinterpret_cast<double*>(dev + b_pairs);
  b2s_odometry_constraint* dout = reinterpret_cast<b2s_odometry_constraint*>(dev + b_pairs + b_part);
  B2S_CUDA(cudaMemcpyAsync(dev, ip, (size_t)n * sizeof(InfoPair), cudaMemcpyHostToDevice, h->stream));
  {
    ProfScope prof(h, PK_ICP);
    launch_pdl(info_wide_kernel, grid_for((size_t)tiles, 1, 4 * device_sms()), WI_THREADS, 0, h->stream, dpairs, n, tiles, r, partials);
    launch_pdl(info_finish_kernel, n, 32, 0, h->stream, dpairs, (const double*)partials, dout);
    h->launches += 2;
  }
  B2S_CUDA(cudaGetLastError());
  B2S_CUDA(cudaMemcpyAsync(out, dout, (size_t)n * sizeof(b2s_odometry_constraint), cudaMemcpyDeviceToHost, h->stream));
  return check_status(h);
}

}  // namespace b2s
