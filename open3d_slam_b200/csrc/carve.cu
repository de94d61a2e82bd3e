// carve.cu -- K-carve: space carving of the sparse map (SURVEY.md section 8f rank 1).
//
// Reference: Submap::carve (core/src/Submap.cpp:109-123) -> getIdxsOfCarvedPoints (core/src/helpers.cpp:235-271) over a
// VoxelMap (core/src/Voxel.cpp:123-149) keyed by floor(p * (1/voxel)) (VoxelHashMap.hpp:47-50,124).  Every ray sensor ->
// scan point is marched in steps of one carving voxel up to max(voxel, min(length - truncation, maxRaytracingLength)); a
// map point (inside the map-builder cropper) lying in a visited voxel is removed unless the ray is nearly parallel to
// its surface (|dir . n| <= minDotProductWithNormal).  The reference does this with OpenMP over the rays and an
// `omp critical` insert into an unordered_set per hit.
//
// Device: (1) open-addressing hash of the carving voxels that hold in-cropper map points, each voxel the head of a chain
// of point indices (atomicCAS on the packed key, atomicExch on the chain head); (2) one thread per ray, same fp64
// expressions as the reference (library built with -fmad=false), hits clear keep[id] (idempotent store, no atomics);
// (3) order-preserving compaction of the map (removeByIds = SelectByIndex(invert) keeps the order).
#include "common.cuh"

namespace b2s {

constexpr int CV_THREADS = 256;

// enable (optional): device-side schedule of the mapper chain -- every kernel of the carving sequence returns at once unless
// *enable != 0; n_eff (optional) receives the point count the compaction works on (0 when skipped)
__global__ void __launch_bounds__(CV_THREADS) carve_init_kernel(unsigned long long* __restrict__ keys, int32_t* __restrict__ head, size_t cap,
                                                                int32_t* __restrict__ keep, int n_max, const int32_t* __restrict__ enable,
                                                                const int32_t* __restrict__ d_nmap, int32_t* n_eff) {
  pdl_wait();
  const bool on = enable == nullptr || *enable != 0;
  if (n_eff && blockIdx.x == 0 && threadIdx.x == 0) *n_eff = on ? *d_nmap : 0;
  if (!on) return;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < cap; i += (size_t)gridDim.x * blockDim.x) { keys[i] = VOXEL_KEY_EMPTY; head[i] = -1; }
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_max; i += gridDim.x * blockDim.x) keep[i] = 1;
}

__global__ void __launch_bounds__(CV_THREADS) carve_insert_kernel(const double* __restrict__ xyz, const int32_t* __restrict__ d_n, CropDev crop,
                                                                  double inv, unsigned long long* keys, int32_t* head,
                                                                  int32_t* __restrict__ next, size_t mask, uint32_t* status,
                                                                  const int32_t* __restrict__ enable, int32_t* __restrict__ keep) {
  pdl_wait();
  if (enable != nullptr && *enable == 0) return;
  const int n = *d_n;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const double x = xyz[3 * i], y = xyz[3 * i + 1], z = xyz[3 * i + 2];
    next[i] = -1;
    if (!(x == x)) { keep[i] = 0; continue; }      // tombstone of the fusion (fuse.cu): dropped by the compaction below
    if (!crop_within(crop, x, y, z)) continue;     // getIndicesWithinVolume(*map): only these are candidates
    unsigned long long key;
    if (!voxel_key_of(x, y, z, inv, inv, inv, &key)) { atomicOr(status, ST_KEY_OVERFLOW); continue; }
    bool fresh;
    const long long s = voxel_key_claim(keys, mask, key, &fresh);
    if (s >= 0) next[i] = atomicExch(&head[s], i);
  }
}

// one thread per scan point: transform into the map frame exactly like o3d_slam::transform (helpers.cpp:293-296), then march
__global__ void __launch_bounds__(CV_THREADS) carve_march_kernel(const double* __restrict__ scan, const int32_t* __restrict__ d_nscan,
                                                                 const double* __restrict__ Tdev, const double* __restrict__ map_nrm,
                                                                 const unsigned long long* __restrict__ keys, const int32_t* __restrict__ head,
                                                                 const int32_t* __restrict__ next, size_t mask, double voxel, double inv,
                                                                 double max_len, double trunc, double min_dot, int32_t* keep,
                                                                 const int32_t* __restrict__ enable) {
  pdl_wait();
  if (enable != nullptr && *enable == 0) return;
  const int n = *d_nscan;
  double T[16];
#pragma unroll
  for (int i = 0; i < 16; i++) T[i] = Tdev[i];
  const double sx = T[3], sy = T[7], sz = T[11];   // mapToRangeSensor.translation()
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    double qx, qy, qz;
    transform_point(T, scan[3 * i], scan[3 * i + 1], scan[3 * i + 2], &qx, &qy, &qz);
    const double dx = qx - sx, dy = qy - sy, dz = qz - sz;
    const double length = sqrt(dx * dx + dy * dy + dz * dz);
    const double ux = dx / length, uy = dy / length, uz = dz / length;
    double mp = length - trunc;
    if (max_len < mp) mp = max_len;   // std::min(length - truncation, maxRaytracingLength)
    if (voxel > mp) mp = voxel;       // std::max(voxelSize, ...)
    if (!(mp == mp)) continue;
    double distance = 0.0;
    while (distance < mp) {
      const double cx = distance * ux + sx, cy = distance * uy + sy, cz = distance * uz + sz;
      unsigned long long key;
      const long long s = voxel_key_of(cx, cy, cz, inv, inv, inv, &key) ? voxel_key_find(keys, mask, key) : -1;
      for (int id = s >= 0 ? head[s] : -1; id >= 0; id = next[id]) {
        bool rm = true;
        if (map_nrm) {
          double nx = map_nrm[3 * (size_t)id], ny = map_nrm[3 * (size_t)id + 1], nz = map_nrm[3 * (size_t)id + 2];
          const double nn = sqrt(nx * nx + ny * ny + nz * nz);
          if (nn > 0.0) { nx /= nn; ny /= nn; nz /= nn; }   // Eigen normalized()
          rm = fabs(ux * nx + uy * ny + uz * nz) > min_dot;
        }
        if (rm) keep[id] = 0;
      }
      distance += voxel;
    }
  }
}

// commit of the compacted map back into the map's own buffers (captured graphs and indices hold their addresses), the
// removed count, and the chain's carving counters
__global__ void __launch_bounds__(CV_THREADS) carve_commit_kernel(const double* __restrict__ txyz, const double* __restrict__ tnrm,
                                                                  const int32_t* __restrict__ d_after, double* __restrict__ mxyz,
                                                                  double* __restrict__ mnrm, int32_t* d_nmap, int32_t* removed,
                                                                  const int32_t* __restrict__ enable, int32_t* mstate) {
  pdl_wait();
  if (enable != nullptr && *enable == 0) { if (removed && blockIdx.x == 0 && threadIdx.x == 0) *removed = 0; return; }
  const int before = *d_nmap, n = *d_after;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < 3 * n; i += gridDim.x * blockDim.x) { mxyz[i] = txyz[i]; if (mnrm) mnrm[i] = tnrm[i]; }
  // d_nmap is read by every block before any block can reach this point of a LATER kernel; within this kernel only block 0
  // writes it, after its own copy loop -- other blocks may still read `before`, so the write goes through a grid-wide
  // ticket: the last block to finish publishes the new count
  __shared__ int s_last;
  __syncthreads();
  if (threadIdx.x == 0) s_last = (atomicAdd(&mstate[MS_TMP], 1) == (int)gridDim.x - 1);
  __syncthreads();
  if (s_last && threadIdx.x == 0) {
    const int dead = mstate[MS_NDEAD];   // tombstones went with the compaction: they are not carved points
    mstate[MS_TMP] = 0;
    mstate[MS_NDEAD] = 0;
    *d_nmap = n;
    if (removed) *removed = before - dead - n;
    mstate[MS_NCARVE] += 1;
    mstate[MS_CARVED] += before - dead - n;
  }
}

int32_t compact_cloud(b2s_handle* h, const b2s_cloud* in, const int32_t* flags, b2s_cloud* out, const int32_t* d_n_override = nullptr);   // voxel.cu

int32_t op_submap_carve(b2s_handle* h, b2s_submap* sm, const b2s_cloud* raw_scan, const double* T_dev, const CropDev& crop,
                        const b2s_carving_params& prm, int32_t* removed_dev, const int32_t* enable_dev) {
  b2s_cloud* map = sm->cloud[0].get();
  b2s_cloud* tmp = sm->cloud[1].get();
  // graph replay: constant launch dimensions (the map's host-side bound moves from scan to scan)
  const size_t n_max = sm->fixed_launch ? sm->capacity : (map->n_max > 0 ? map->n_max : 1);
  size_t cap = 1024;
  while (cap < 2 * n_max) cap <<= 1;
  B2S_TRY(h->keys.ensure(cap * 8, h->stream));                    // packed voxel keys
  B2S_TRY(h->vals.ensure(cap * 4, h->stream));                    // chain heads
  B2S_TRY(h->tmp_i32.ensure((n_max + 64) * 4, h->stream));        // chain links
  B2S_TRY(h->flags.ensure((n_max + 1) * 4, h->stream));           // keep flags
  unsigned long long* keys = h->keys.as<unsigned long long>();
  int32_t* head = h->vals.as<int32_t>();
  int32_t* next = h->tmp_i32.as<int32_t>();
  int32_t* keep = h->flags.as<int32_t>();
  int32_t* ms = sm->mstate.as<int32_t>();
  int32_t* n_eff = ms + MS_CARVE_N;
  const double inv = 1.0 / prm.voxel_size;   // fromVoxelSize (VoxelHashMap.hpp:43-45)
  ProfScope prof(h, PK_FUSE);
  launch_pdl(carve_init_kernel, grid_for(cap, CV_THREADS), CV_THREADS, 0, h->stream, keys, head, cap, keep, (int)n_max, enable_dev, map->dn.as<int32_t>(),
                                                                             n_eff);
  launch_pdl(carve_insert_kernel, grid_for(n_max, CV_THREADS), CV_THREADS, 0, h->stream, map->xyz.as<double>(), map->dn.as<int32_t>(), crop, inv, keys,
                                                                                head, next, cap - 1, h->status.as<uint32_t>(), enable_dev, keep);
  launch_pdl(carve_march_kernel, grid_for(raw_scan->n_max > 0 ? raw_scan->n_max : 1, CV_THREADS), CV_THREADS, 0, h->stream, 
      raw_scan->xyz.as<double>(), raw_scan->dn.as<int32_t>(), T_dev, map->has_normals ? map->nrm.as<double>() : nullptr, keys, head, next,
      cap - 1, prm.voxel_size, inv, prm.max_raytracing_length, prm.truncation_distance, prm.min_dot_product_with_normal, keep, enable_dev);
  h->launches += 3;
  const size_t keep_n_max = map->n_max;
  if (sm->fixed_launch) map->n_max = n_max;
  const int32_t rc = compact_cloud(h, map, keep, tmp, n_eff);   // order-preserving (removeByIds = SelectByIndex(invert))
  map->n_max = keep_n_max;
  B2S_TRY(rc);
  launch_pdl(carve_commit_kernel, grid_for(n_max, CV_THREADS), CV_THREADS, 0, h->stream, tmp->xyz.as<double>(), tmp->nrm.as<double>(),
                                                                               tmp->dn.as<int32_t>(), map->xyz.as<double>(),
                                                                               map->has_normals ? map->nrm.as<double>() : nullptr,
                                                                               map->dn.as<int32_t>(), removed_dev, enable_dev, ms);
  h->launches++;
  map->n_known = -1;
  B2S_CUDA(cudaGetLastError());
  return fuse_rehash(h, sm, enable_dev);   // the points moved: the fusion's voxel hash follows
}

}  // namespace b2s
