// grid_index.cu -- K-index: the spatial index that replaces the KD-tree the reference rebuilds inside every
// [O3D] RegistrationICP / EstimateNormals call (KDTreeFlann::SetGeometry; SURVEY.md section 8a row R2).
//
// Layout (HBM): a dense grid of cells over the (optionally cropped) point set; points are counting-sorted by
// linear cell id (x fastest) into a packed double4 array {x,y,z,bits(original index)}.  Normals are not copied: a
// search needs them only for its final correspondences, and reads them from the cloud through the original index
// (copying them was half of the scatter's bytes, for every indexed point of every build).
// cell_start[c] .. cell_start[c+1] is the slot range of cell c.  Because x is the fastest axis, a run of
// neighbouring cells along x is ONE contiguous slot range, so a 3x3x3 neighbourhood is 9 ranges.
// Points outside the grid box are clamped into the border cells, which the search treats as semi-infinite.
//
// Build = bbox reduce -> header (1 thread) -> count (atomics, keeps the rank) -> look-back scan -> scatter.  The map index of a
// registration against a submap has no bbox reduce: its header comes from the submap's box (grid_header_box_kernel).
#include <stdlib.h>

#include "common.cuh"

namespace b2s {

constexpr int GB_THREADS = 256;

__global__ void grid_bbox_init_kernel(unsigned long long* bbox) {
  pdl_wait();
  int t = threadIdx.x;
  if (t < 3) bbox[t] = ord_encode(INFINITY);
  else if (t < 6) bbox[t] = ord_encode(-INFINITY);
}

__device__ __forceinline__ void grid_bbox_body(const double* __restrict__ xyz, const int32_t* __restrict__ d_n, const CropDev& crop,
                                               int use_crop, unsigned long long* bbox) {
  const int n = *d_n;
  double mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    double x = xyz[3 * i], y = xyz[3 * i + 1], z = xyz[3 * i + 2];
    if (use_crop && !crop_within(crop, x, y, z)) continue;
    if (!(x == x && y == y && z == z)) continue;
    mn[0] = fmin(mn[0], x); mn[1] = fmin(mn[1], y); mn[2] = fmin(mn[2], z);
    mx[0] = fmax(mx[0], x); mx[1] = fmax(mx[1], y); mx[2] = fmax(mx[2], z);
  }
  box_fold_block<GB_THREADS>(mn, mx, bbox);
}

__global__ void __launch_bounds__(GB_THREADS) grid_bbox_kernel(const double* __restrict__ xyz, const int32_t* __restrict__ d_n,
                                                               CropDev crop, int use_crop, unsigned long long* bbox) {
  pdl_wait();
  grid_bbox_body(xyz, d_n, crop, use_crop, bbox);
}

// the header of a grid over the box [mn, mx] (an empty box on any axis, or NaN: the empty set)
__device__ void grid_header_of(double (&mn)[3], double (&mx)[3], double cell, int cap_cells, GridHeader* hdr) {
  if (!(mn[0] <= mx[0] && mn[1] <= mx[1] && mn[2] <= mx[2])) { for (int d = 0; d < 3; d++) { mn[d] = 0.0; mx[d] = 0.0; } }  // empty set
  int dims[3];
  for (;;) {
    double total = 1.0;
    for (int d = 0; d < 3; d++) {
      double e = floor((mx[d] - mn[d]) / cell) + 1.0;
      if (e > 2.0e9) e = 2.0e9;
      dims[d] = (int)e;
      total *= e;
    }
    if (total <= (double)cap_cells) break;
    cell *= 2.0;  // coarser cells only cost speed, never exactness
  }
  for (int d = 0; d < 3; d++) { hdr->origin[d] = mn[d]; hdr->dims[d] = dims[d]; }
  hdr->cell = cell;
  hdr->inv_cell = 1.0 / cell;
  hdr->ncell = dims[0] * dims[1] * dims[2];
  hdr->n = 0;
}

__device__ void grid_header_body(const unsigned long long* bbox, double cell, int cap_cells, GridHeader* hdr) {
  double mn[3], mx[3];
  for (int d = 0; d < 3; d++) { mn[d] = ord_decode(bbox[d]); mx[d] = ord_decode(bbox[3 + d]); }
  grid_header_of(mn, mx, cell, cap_cells, hdr);
}

__global__ void grid_header_kernel(const unsigned long long* bbox, double cell, int cap_cells, GridHeader* hdr) {
  pdl_wait();
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  grid_header_body(bbox, cell, cap_cells, hdr);
}

// The axis-aligned box [lo, hi] that holds what crop_within can accept, up to the rounding of crop_within itself (a point a few ulps
// outside may pass); false when the cropper is not bounded (no box).  The cylinder compares the absolute z.
__device__ __forceinline__ bool crop_aabb(const CropDev& crop, double* lo, double* hi) {
  double c[3] = {crop.cx, crop.cy, crop.cz};
  if (crop.pose_dev) { c[0] = crop.pose_dev[3]; c[1] = crop.pose_dev[7]; c[2] = crop.pose_dev[11]; }
  for (int d = 0; d < 3; d++) { lo[d] = c[d] - crop.rmax; hi[d] = c[d] + crop.rmax; }
  if (crop.kind == B2S_CROP_CYLINDER) { lo[2] = crop.zmin; hi[2] = crop.zmax; }
  return !crop.invert && (crop.kind == B2S_CROP_MAX_RADIUS || crop.kind == B2S_CROP_MINMAX_RADIUS || crop.kind == B2S_CROP_CYLINDER);
}

__device__ __forceinline__ int grid_cell_of(const GridHeader& g, double x, double y, double z) {
  return (grid_axis_cell(z, g.origin[2], g.inv_cell, g.dims[2]) * g.dims[1] + grid_axis_cell(y, g.origin[1], g.inv_cell, g.dims[1])) * g.dims[0] +
         grid_axis_cell(x, g.origin[0], g.inv_cell, g.dims[0]);
}

__global__ void grid_zero_kernel(const GridHeader* hdr, int32_t* counts) {
  pdl_wait();
  const int nc = hdr->ncell + 1;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nc; i += gridDim.x * blockDim.x) counts[i] = 0;
}

__device__ __forceinline__ void grid_count_body(const double* __restrict__ xyz, const int32_t* __restrict__ d_n, const CropDev& crop,
                                                int use_crop, const GridHeader* __restrict__ hdr, int32_t* counts,
                                                int32_t* __restrict__ rank) {
  const int n = *d_n;
  __shared__ GridHeader g;
  if (threadIdx.x == 0) g = *hdr;
  __syncthreads();
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    double x = xyz[3 * i], y = xyz[3 * i + 1], z = xyz[3 * i + 2];
    int r = -1;
    if ((x == x && y == y && z == z) && (!use_crop || crop_within(crop, x, y, z))) r = atomicAdd(&counts[grid_cell_of(g, x, y, z)], 1);
    rank[i] = r;
  }
}

__global__ void __launch_bounds__(GB_THREADS) grid_count_kernel(const double* __restrict__ xyz, const int32_t* __restrict__ d_n,
                                                                CropDev crop, int use_crop, const GridHeader* __restrict__ hdr,
                                                                int32_t* counts, int32_t* __restrict__ rank) {
  pdl_wait();
  grid_count_body(xyz, d_n, crop, use_crop, hdr, counts, rank);
}

__device__ __forceinline__ void grid_scatter_body(const double* __restrict__ xyz, const int32_t* __restrict__ d_n, GridHeader* hdr,
                                                  const int32_t* __restrict__ cell_start, const int32_t* __restrict__ rank,
                                                  double4* __restrict__ pts, const int32_t* __restrict__ orig) {
  const int n = *d_n;
  __shared__ GridHeader g;
  if (threadIdx.x == 0) g = *hdr;
  __syncthreads();
  if (blockIdx.x == 0 && threadIdx.x == 0) hdr->n = cell_start[g.ncell];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    int r = rank[i];
    if (r < 0) continue;
    double x = xyz[3 * i], y = xyz[3 * i + 1], z = xyz[3 * i + 2];
    int slot = cell_start[grid_cell_of(g, x, y, z)] + r;
    pts[slot] = make_double4(x, y, z, __longlong_as_double((long long)(orig ? orig[i] : i)));
  }
}

__global__ void __launch_bounds__(GB_THREADS) grid_scatter_kernel(const double* __restrict__ xyz, const int32_t* __restrict__ d_n,
                                                                  GridHeader* hdr, const int32_t* __restrict__ cell_start,
                                                                  const int32_t* __restrict__ rank, double4* __restrict__ pts,
                                                                  const int32_t* __restrict__ orig) {
  pdl_wait();
  grid_scatter_body(xyz, d_n, hdr, cell_start, rank, pts, orig);
}

// ---- map index: the grid box from the submap's box -----------------------------------------------------------------------------
// The grid box is the submap's box (it holds every live slot) cut to the cropper's box: a superset of the patch, so only the cell
// geometry differs from the measured box, never the indexed set (a point outside the grid box lands in a border cell, which the search
// treats as semi-infinite).  No pass over the map: the header comes from twelve words.
__global__ void grid_header_box_kernel(const unsigned long long* __restrict__ map_box, CropDev crop, double cell, int cap_cells, GridHeader* hdr) {
  pdl_wait();
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  double mn[3], mx[3], lo[3], hi[3];
  for (int d = 0; d < 3; d++) { mn[d] = ord_decode(map_box[d]); mx[d] = ord_decode(map_box[3 + d]); }
  if (crop_aabb(crop, lo, hi))
    for (int d = 0; d < 3; d++) { mn[d] = fmax(mn[d], lo[d]); mx[d] = fmin(mx[d], hi[d]); }   // a NaN bound keeps the map's
  grid_header_of(mn, mx, cell, cap_cells, hdr);
}

// ---- batched build: blockIdx.y = job -------------------------------------------------------------------------------
struct GridJob {
  const double* xyz; const int32_t* d_n;
  unsigned long long* bbox; GridHeader* hdr; int32_t* counts; int32_t* starts; int32_t* rank; double4* pts;
  int32_t cap_cells; int32_t pad;
};

__global__ void gridb_init_kernel(const GridJob* __restrict__ jobs, int njobs) {
  pdl_wait();
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= njobs * 6) return;
  const int t = j % 6;
  jobs[j / 6].bbox[t] = t < 3 ? ord_encode(INFINITY) : ord_encode(-INFINITY);
}
__global__ void __launch_bounds__(GB_THREADS) gridb_bbox_kernel(const GridJob* __restrict__ jobs) {
  pdl_wait();
  const GridJob j = jobs[blockIdx.y];
  CropDev none; none.kind = 0; none.invert = 0; none.pose_dev = nullptr;
  grid_bbox_body(j.xyz, j.d_n, none, 0, j.bbox);
}
__global__ void gridb_header_kernel(const GridJob* __restrict__ jobs, int njobs, double cell) {
  pdl_wait();
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < njobs) grid_header_body(jobs[j].bbox, cell, jobs[j].cap_cells, jobs[j].hdr);
}
__global__ void gridb_zero_kernel(const GridJob* __restrict__ jobs) {
  pdl_wait();
  const GridJob j = jobs[blockIdx.y];
  const int nc = j.hdr->ncell + 1;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nc; i += gridDim.x * blockDim.x) j.counts[i] = 0;
}
__global__ void __launch_bounds__(GB_THREADS) gridb_count_kernel(const GridJob* __restrict__ jobs) {
  pdl_wait();
  const GridJob j = jobs[blockIdx.y];
  CropDev none; none.kind = 0; none.invert = 0; none.pose_dev = nullptr;
  grid_count_body(j.xyz, j.d_n, none, 0, j.hdr, j.counts, j.rank);
}
__global__ void __launch_bounds__(GB_THREADS) gridb_scatter_kernel(const GridJob* __restrict__ jobs) {
  pdl_wait();
  const GridJob j = jobs[blockIdx.y];
  grid_scatter_body(j.xyz, j.d_n, j.hdr, j.starts, j.rank, j.pts, nullptr);
}

int32_t box_reset(b2s_handle* h, unsigned long long* box) {
  launch_pdl(grid_bbox_init_kernel, 1, 32, 0, h->stream, box);
  h->launches++;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

CropDev make_crop(const b2s_cropper* c, const double* pose_dev) {
  CropDev d;
  memset(&d, 0, sizeof(d));
  if (c) {
    d.kind = c->kind; d.invert = c->invert; d.rmin = c->rmin; d.rmax = c->rmax; d.zmin = c->zmin; d.zmax = c->zmax;
    d.cx = c->center[0]; d.cy = c->center[1]; d.cz = c->center[2];
  }
  d.pose_dev = pose_dev;
  return d;
}

int32_t grid_build(b2s_handle* h, GridIndex* g, const b2s_cloud* cloud, double cell, const CropDev* patch, const int32_t* orig,
                   const unsigned long long* map_box, const CropDev* map_crop) {
  B2S_REQUIRE(cell > 0.0, B2S_E_INVALID, "grid_build: cell size must be > 0");
  // B2S_GRID_BBOX_PASS=1: the map index measures its grid box with a pass over the map, as every other index build does (A/B switch
  // and test reference; read once per process)
  static const bool bbox_pass = getenv("B2S_GRID_BBOX_PASS") && atoi(getenv("B2S_GRID_BBOX_PASS")) != 0;
  const bool from_box = map_box && map_crop && !bbox_pass;
  const size_t n_max = cloud->n_max > 0 ? cloud->n_max : 1;
  // buffers follow the ALLOCATION of the cloud, not its current size: a growing map never re-allocates its index
  // (a cudaMalloc/cudaFree pair is a device-wide synchronisation)
  size_t n_alloc = cloud->xyz.cap / 24;
  if (n_alloc < n_max) n_alloc = n_max;
  // cell budget: 8 cells per point, at most 2^21 (a 128 m x 128 m x 32 m box at 0.5 m); when the box needs more the
  // header kernel doubles the cell edge, which only costs speed
  size_t want = n_alloc * 8 + 4096;
  if (want > (size_t)1 << 21) want = (size_t)1 << 21;
  if (want < (size_t)1 << 16) want = (size_t)1 << 16;
  if ((size_t)g->cap_cells < want) {
    B2S_TRY(g->cell_start.ensure((want + 8) * 4 * 2, h->stream));  // counts + starts
    g->cap_cells = (int32_t)want;
  }
  B2S_TRY(g->hdr.ensure(sizeof(GridHeader), h->stream));
  B2S_TRY(g->bbox.ensure(64, h->stream));
  B2S_TRY(g->rank.ensure(n_alloc * 4, h->stream));
  B2S_TRY(g->pts.ensure(n_alloc * 32, h->stream));
  CropDev cd = patch ? *patch : make_crop(nullptr);
  const int use_crop = patch ? 1 : 0;
  const int blocks = grid_for(n_max, GB_THREADS);
  int32_t* counts = g->cell_start.as<int32_t>();
  int32_t* starts = counts + g->cap_cells + 4;
  const int32_t* d_n = cloud->dn.as<int32_t>();
  GridHeader* hdr = g->hdr.as<GridHeader>();
  ProfScope prof(h, PK_GRID);
  if (from_box) {
    launch_pdl(grid_header_box_kernel, 1, 32, 0, h->stream, map_box, *map_crop, cell, g->cap_cells, hdr);
    h->launches++;
  } else {
    launch_pdl(grid_bbox_init_kernel, 1, 32, 0, h->stream, g->bbox.as<unsigned long long>());
    launch_pdl(grid_bbox_kernel, blocks, GB_THREADS, 0, h->stream, cloud->xyz.as<double>(), d_n, cd, use_crop, g->bbox.as<unsigned long long>());
    launch_pdl(grid_header_kernel, 1, 32, 0, h->stream, g->bbox.as<unsigned long long>(), cell, g->cap_cells, hdr);
    h->launches += 3;
  }
  launch_pdl(grid_zero_kernel, 4 * device_sms(), 256, 0, h->stream, hdr, counts);
  launch_pdl(grid_count_kernel, blocks, GB_THREADS, 0, h->stream, cloud->xyz.as<double>(), d_n, cd, use_crop, hdr, counts, g->rank.as<int32_t>());
  h->launches += 2;
  // scan over ncell (device-known) counts; launch sized for the capacity
  B2S_TRY(scan_exclusive_i32(h, counts, starts, &hdr->ncell, (size_t)g->cap_cells, nullptr));
  launch_pdl(grid_scatter_kernel, blocks, GB_THREADS, 0, h->stream, cloud->xyz.as<double>(), d_n, hdr, starts, g->rank.as<int32_t>(),
             g->pts.as<double4>(), orig);
  h->launches++;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}


static int32_t grid_reserve(b2s_handle* h, GridIndex* g, const b2s_cloud* cloud, size_t* n_alloc_out) {
  const size_t n_max = cloud->n_max > 0 ? cloud->n_max : 1;
  size_t n_alloc = cloud->xyz.cap / 24;
  if (n_alloc < n_max) n_alloc = n_max;
  size_t want = n_alloc * 8 + 4096;
  if (want > (size_t)1 << 21) want = (size_t)1 << 21;
  if (want < (size_t)1 << 16) want = (size_t)1 << 16;
  if ((size_t)g->cap_cells < want) {
    B2S_TRY(g->cell_start.ensure((want + 8) * 4 * 2, h->stream));  // counts + starts
    g->cap_cells = (int32_t)want;
  }
  B2S_TRY(g->hdr.ensure(sizeof(GridHeader), h->stream));
  B2S_TRY(g->bbox.ensure(64, h->stream));
  B2S_TRY(g->rank.ensure(n_alloc * 4, h->stream));
  B2S_TRY(g->pts.ensure(n_alloc * 32, h->stream));
  *n_alloc_out = n_alloc;
  return B2S_OK;
}

int32_t grid_build_batch(b2s_handle* h, GridIndex* const* g, const b2s_cloud* const* clouds, int n, double cell) {
  B2S_REQUIRE(cell > 0.0, B2S_E_INVALID, "grid_build: cell size must be > 0");
  if (n <= 0) return B2S_OK;
  size_t max_pts = 1, max_cells = 1;
  for (int i = 0; i < n; i++) {
    size_t n_alloc;
    B2S_TRY(grid_reserve(h, g[i], clouds[i], &n_alloc));
    if (clouds[i]->n_max > max_pts) max_pts = clouds[i]->n_max;
    if ((size_t)g[i]->cap_cells > max_cells) max_cells = (size_t)g[i]->cap_cells;
  }
  // device tables: GridJob[n] | ScanJob[n], uploaded from batch_jobs_host at the same offsets, then the scan tile states (zeroed)
  Layout T;
  const size_t o_jobs = T.off((size_t)n * sizeof(GridJob)), o_scan = T.off((size_t)n * sizeof(ScanJob)), staged = T.size;
  h->batch_jobs_host.assign(staged, 0);
  GridJob* gj = reinterpret_cast<GridJob*>(h->batch_jobs_host.data() + o_jobs);
  ScanJob* sj = reinterpret_cast<ScanJob*>(h->batch_jobs_host.data() + o_scan);
  size_t state_end = 0;
  B2S_TRY(carve(h->batch_jobs, h->stream, [&](Layout& D) {
    D.off(staged);
    for (int i = 0; i < n; i++) scan_bind_state(D, sj[i], max_cells);
    state_end = D.size;
  }));
  unsigned char* dev = h->batch_jobs.as<unsigned char>();
  for (int i = 0; i < n; i++) {
    int32_t* counts = g[i]->cell_start.as<int32_t>();
    int32_t* starts = counts + g[i]->cap_cells + 4;
    GridHeader* hdr = g[i]->hdr.as<GridHeader>();
    gj[i].xyz = clouds[i]->xyz.as<double>();
    gj[i].d_n = clouds[i]->dn.as<int32_t>();
    gj[i].bbox = g[i]->bbox.as<unsigned long long>();
    gj[i].hdr = hdr; gj[i].counts = counts; gj[i].starts = starts; gj[i].rank = g[i]->rank.as<int32_t>();
    gj[i].pts = g[i]->pts.as<double4>();
    gj[i].cap_cells = g[i]->cap_cells;
    sj[i].in = counts; sj[i].out = starts; sj[i].d_n = &hdr->ncell;
  }
  B2S_CUDA(cudaMemcpyAsync(dev, h->batch_jobs_host.data(), staged, cudaMemcpyHostToDevice, h->stream));
  B2S_CUDA(cudaMemsetAsync(dev + staged, 0, state_end - staged, h->stream));
  const GridJob* dj = reinterpret_cast<const GridJob*>(dev + o_jobs);
  const ScanJob* ds = reinterpret_cast<const ScanJob*>(dev + o_scan);
  int bx = grid_for(max_pts, GB_THREADS, 2 * device_sms());   // x blocks per job; y = job
  const dim3 gpts((unsigned)bx, (unsigned)n);
  ProfScope prof(h, PK_GRID);
  launch_pdl(gridb_init_kernel, (n * 6 + 127) / 128, 128, 0, h->stream, dj, n);
  launch_pdl(gridb_bbox_kernel, gpts, GB_THREADS, 0, h->stream, dj);
  launch_pdl(gridb_header_kernel, (n + 127) / 128, 128, 0, h->stream, dj, n, cell);
  launch_pdl(gridb_zero_kernel, dim3((unsigned)device_sms(), (unsigned)n), 256, 0, h->stream, dj);
  launch_pdl(gridb_count_kernel, gpts, GB_THREADS, 0, h->stream, dj);
  h->launches += 5;
  B2S_TRY(scan_exclusive_i32_batch(h, ds, n, max_cells));
  launch_pdl(gridb_scatter_kernel, gpts, GB_THREADS, 0, h->stream, dj);
  h->launches++;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

// ---- K-patch: the static map patch of a submap whose map cannot change (merge off, pure localisation) -------------------------------
// Tile table: the submap's GridIndex `tile`, built once over the map slots with cell = TILE_EDGE and no cropper (the K-index build:
// bbox -> header -> count -> scan -> scatter), so the slots are counting-sorted by tile, x fastest, and a run of tiles along x is one
// contiguous slot range.  The header doubles the edge when the map's box needs more than the cell budget, like every K-index build.
// Per registration: tile_gather_kernel reads the sensor position from the device pose (or the host-given centre), takes the tiles the
// cropper's box overlaps, grown by TILE_MARGIN tiles on every side (the box is computed in rounded arithmetic, and crop_within accepts a
// point up to a few ulps outside it), and appends the points of those tiles that pass the unchanged crop_within, each with its map slot.
// The NN grid is then built over exactly those points with the slot as original index: the same set, header (both paths take it from
// the submap's box and the cropper) and original indices as the full path's crop inside the build, at O(points in the touched tiles) instead of O(map).  Why 2 m: a few map voxels, fine enough
// that the cube of tiles around a 20-30 m cropper holds little beyond the sphere's own box, coarse enough that a site-sized map's table
// stays within the cell budget.  Launches are sized from the map's bound (grid-stride over the device count): graph-capturable.
__global__ void tile_zero_kernel(int32_t* n) {
  pdl_wait();
  if (threadIdx.x == 0) *n = 0;
}

// the tile box of the cropper: [lo, hi] per axis, clamped to the table; empty when lo > hi on an axis
__device__ __forceinline__ void tile_box(const GridHeader& g, const CropDev& crop, int* box) {
  double lo[3], hi[3];
  crop_aabb(crop, lo, hi);   // bounded: tile_patch_usable
  for (int d = 0; d < 3; d++) {
    const double a = fmax(floor((lo[d] - g.origin[d]) * g.inv_cell) - TILE_MARGIN, 0.0);
    const double b = fmin(floor((hi[d] - g.origin[d]) * g.inv_cell) + TILE_MARGIN, (double)(g.dims[d] - 1));
    const bool ok = a <= b;   // false for NaN as well
    box[d] = ok ? (int)a : 1;
    box[3 + d] = ok ? (int)b : 0;
  }
}

__global__ void __launch_bounds__(GB_THREADS) tile_gather_kernel(const GridHeader* __restrict__ thdr, const int32_t* __restrict__ tstart,
                                                                 const double4* __restrict__ tpts, CropDev crop, double* __restrict__ out_xyz,
                                                                 int32_t* __restrict__ out_idx, int32_t* __restrict__ out_n) {
  pdl_wait();
  __shared__ GridHeader g;
  __shared__ int box[6];
  if (threadIdx.x == 0) { g = *thdr; tile_box(g, crop, box); }
  __syncthreads();
  if (box[0] > box[3] || box[1] > box[4] || box[2] > box[5]) return;
  const int ny = box[4] - box[1] + 1, nz = box[5] - box[2] + 1;
  const int lane = threadIdx.x & 31;
  for (int r = blockIdx.x; r < ny * nz; r += gridDim.x) {   // one (y, z) row of tiles per CTA
    const int row = ((box[2] + r / ny) * g.dims[1] + (box[1] + r % ny)) * g.dims[0];
    const int s0 = tstart[row + box[0]], s1 = tstart[row + box[3] + 1];
    for (int j0 = s0; j0 < s1; j0 += blockDim.x) {   // uniform trip count over the CTA: every lane reaches the ballot
      const int j = j0 + threadIdx.x;
      double4 q = make_double4(0.0, 0.0, 0.0, 0.0);
      bool pass = false;
      if (j < s1) { q = tpts[j]; pass = crop_within(crop, q.x, q.y, q.z); }
      const unsigned m = __ballot_sync(0xffffffffu, pass);
      int base = 0;
      if (lane == 0 && m) base = atomicAdd(out_n, __popc(m));
      base = __shfl_sync(0xffffffffu, base, 0);
      if (pass) {
        const int o = base + __popc(m & ((1u << lane) - 1u));
        out_xyz[3 * o] = q.x; out_xyz[3 * o + 1] = q.y; out_xyz[3 * o + 2] = q.z;
        out_idx[o] = (int32_t)__double_as_longlong(q.w);
      }
    }
  }
}

bool tile_patch_usable(const b2s_submap* sm, const CropDev& crop) {
  // B2S_PATCH_FULL=1: every registration builds its patch from the whole map (A/B switch and test reference; read once per process)
  static const bool full = getenv("B2S_PATCH_FULL") && atoi(getenv("B2S_PATCH_FULL")) != 0;
  const bool bounded = !crop.invert && (crop.kind == B2S_CROP_MAX_RADIUS || crop.kind == B2S_CROP_MINMAX_RADIUS || crop.kind == B2S_CROP_CYLINDER);
  return !full && !sm->merge_scans && bounded;
}

int32_t tile_drop(b2s_handle* h, b2s_submap* sm) {
  if (!sm->tile_valid) return B2S_OK;
  sm->tile_valid = false;
  sm->opts_gen++;                      // the combined chain's graphs compare it
  return graph_drop(h, &sm->graph);    // a captured chain reads the table: never replay it over a dropped one
}

int32_t tile_patch_build(b2s_handle* h, b2s_submap* sm, const CropDev& crop, double cell, GridIndex* g) {
  const b2s_cloud* map = sm->cloud[0].get();
  const size_t map_alloc = map->xyz.cap / 24;
  if (!sm->patch) B2S_TRY(make_cloud(h, map_alloc, false, false, &sm->patch));
  b2s_cloud* pc = sm->patch.get();
  B2S_TRY(cloud_reserve(h, pc, map_alloc, false));   // the map's allocation: the NN grid's cell budget follows it
  B2S_TRY(sm->patch_idx.ensure(map_alloc * 4 + 16, h->stream));
  if (!sm->tile_valid) {
    B2S_TRY(grid_build(h, &sm->tile, map, TILE_EDGE, nullptr));
    sm->tile_valid = true;
  }
  pc->n_max = map->n_max; pc->n_known = -1; pc->has_normals = false;
  {
    launch_pdl(tile_zero_kernel, 1, 32, 0, h->stream, pc->dn.as<int32_t>());
    launch_pdl(tile_gather_kernel, 2 * device_sms(), GB_THREADS, 0, h->stream, static_cast<const GridHeader*>(sm->tile.hdr.as<GridHeader>()),
               grid_starts(&sm->tile), static_cast<const double4*>(sm->tile.pts.as<double4>()), crop, pc->xyz.as<double>(),
               sm->patch_idx.as<int32_t>(), pc->dn.as<int32_t>());
    h->launches += 2;
  }
  return grid_build(h, g, pc, cell, nullptr, sm->patch_idx.as<int32_t>(), sm->bbox.as<unsigned long long>(), &crop);   // the full path's header
}

}  // namespace b2s
