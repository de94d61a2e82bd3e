// overlap.cu -- K-overlap: the overlap selection in front of the loop-closure ICP (SURVEY.md section 8f rank 2).
//
// Reference: computeIndicesOfOverlappingPoints (core/src/helpers.cpp:307-332), called from
// PlaceRecognition::buildLoopClosureConstraints (core/src/PlaceRecognition.cpp:103-106): both clouds are binned into a
// VoxelMap (key = floor(p * (1/voxel)), the source after sourceToTarget), and a point survives when its voxel holds at least
// minNumPointsPerVoxel points of BOTH clouds.  The reference walks an unordered_map with string-keyed layers and returns
// index lists in hash order; the callers only feed them to SelectByIndex, so the selected SETS are the contract.
//
// Device: one open-addressing hash of packed voxel keys with a (source, target) counter pair per slot; every point
// remembers its slot, a second pass turns the counters into keep-flags, and the two clouds are compacted in their
// original order.  Three kernels + two compactions, all bandwidth-trivial (the clouds are a few MB).
#include "common.cuh"

namespace b2s {

constexpr int OV_THREADS = 256;

__global__ void __launch_bounds__(OV_THREADS) ov_init_kernel(unsigned long long* __restrict__ keys, int32_t* __restrict__ cnt, size_t cap) {
  pdl_wait();
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < cap; i += (size_t)gridDim.x * blockDim.x) {
    keys[i] = VOXEL_KEY_EMPTY; cnt[2 * i] = 0; cnt[2 * i + 1] = 0;
  }
}

// which = 0: source (transformed by T like [O3D] PointCloud::Transform), which = 1: target
__global__ void __launch_bounds__(OV_THREADS) ov_insert_kernel(const double* __restrict__ xyz, const int32_t* __restrict__ d_n,
                                                               const double* __restrict__ Tdev, int which, double inv, unsigned long long* keys,
                                                               int32_t* cnt, size_t mask, int32_t* __restrict__ slot_of, uint32_t* status) {
  pdl_wait();
  const int n = *d_n;
  double T[16];
#pragma unroll
  for (int i = 0; i < 16; i++) T[i] = Tdev ? Tdev[i] : ((i % 5 == 0) ? 1.0 : 0.0);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    double x = xyz[3 * i], y = xyz[3 * i + 1], z = xyz[3 * i + 2];
    if (which == 0) transform_point(T, x, y, z, &x, &y, &z);
    slot_of[i] = -1;
    unsigned long long key;
    if (!voxel_key_of(x, y, z, inv, inv, inv, &key)) { atomicOr(status, ST_KEY_OVERFLOW); continue; }
    bool fresh;
    const long long s = voxel_key_claim(keys, mask, key, &fresh);
    if (s >= 0) { atomicAdd(&cnt[2 * s + which], 1); slot_of[i] = (int32_t)s; }
  }
}

__global__ void __launch_bounds__(OV_THREADS) ov_flags_kernel(const int32_t* __restrict__ d_n, const int32_t* __restrict__ slot_of,
                                                              const int32_t* __restrict__ cnt, int min_pts, int32_t* __restrict__ keep) {
  pdl_wait();
  const int n = *d_n;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int s = slot_of[i];
    keep[i] = (s >= 0 && cnt[2 * s] >= min_pts && cnt[2 * s + 1] >= min_pts) ? 1 : 0;
  }
}

int32_t compact_cloud(b2s_handle* h, const b2s_cloud* in, const int32_t* flags, b2s_cloud* out, const int32_t* d_n_override = nullptr);   // voxel.cu

int32_t op_overlap(b2s_handle* h, const b2s_cloud* source, const b2s_cloud* target, const double* T_dev, double voxel, int min_pts,
                   b2s_cloud* source_overlap, b2s_cloud* target_overlap) {
  const size_t ns = source->n_max > 0 ? source->n_max : 1, nt = target->n_max > 0 ? target->n_max : 1;
  size_t cap = 1024;
  while (cap < 2 * (ns + nt)) cap <<= 1;
  B2S_TRY(h->keys.ensure(cap * 8, h->stream));
  B2S_TRY(h->vals.ensure(cap * 8, h->stream));                       // (source, target) counters
  B2S_TRY(h->tmp_i32.ensure((ns + nt + 64) * 4, h->stream));         // slot of every point
  B2S_TRY(h->flags.ensure((ns + nt + 2) * 4, h->stream));
  unsigned long long* keys = h->keys.as<unsigned long long>();
  int32_t* cnt = h->vals.as<int32_t>();
  int32_t* slot_s = h->tmp_i32.as<int32_t>();
  int32_t* slot_t = slot_s + ns;
  int32_t* keep_s = h->flags.as<int32_t>();
  int32_t* keep_t = keep_s + ns + 1;
  const double inv = 1.0 / voxel;   // VoxelMap(Eigen::Vector3d::Constant(voxelSize)) -> fromVoxelSize
  ProfScope prof(h, PK_FUSE);
  launch_pdl(ov_init_kernel, grid_for(cap, OV_THREADS), OV_THREADS, 0, h->stream, keys, cnt, cap);
  launch_pdl(ov_insert_kernel, grid_for(nt, OV_THREADS), OV_THREADS, 0, h->stream, target->xyz.as<double>(), target->dn.as<int32_t>(), nullptr, 1, inv, keys,
                                                                          cnt, cap - 1, slot_t, h->status.as<uint32_t>());
  launch_pdl(ov_insert_kernel, grid_for(ns, OV_THREADS), OV_THREADS, 0, h->stream, source->xyz.as<double>(), source->dn.as<int32_t>(), T_dev, 0, inv, keys,
                                                                          cnt, cap - 1, slot_s, h->status.as<uint32_t>());
  launch_pdl(ov_flags_kernel, grid_for(ns, OV_THREADS), OV_THREADS, 0, h->stream, source->dn.as<int32_t>(), slot_s, cnt, min_pts, keep_s);
  launch_pdl(ov_flags_kernel, grid_for(nt, OV_THREADS), OV_THREADS, 0, h->stream, target->dn.as<int32_t>(), slot_t, cnt, min_pts, keep_t);
  h->launches += 5;
  B2S_TRY(compact_cloud(h, source, keep_s, source_overlap));   // SelectByIndex on the ORIGINAL (untransformed) source
  B2S_TRY(compact_cloud(h, target, keep_t, target_overlap));
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

// ---- batched, in place on the submaps: the overlap of n (source, target) map pairs (odometry constraints, loop-closure refinement) ----
// Every pair owns a segment of one hash (sized like op_overlap's table for the pair's two maps); job 2k reads pair k's source map,
// job 2k + 1 its target map, straight from the map slots: a tombstone (NaN, left by fusion) is skipped, so the compacted result is the
// one b2s_submap_to_cloud + op_overlap give, cloud by cloud and in order.  Each kernel takes its job from blockIdx.y.
// T: the source job's sourceToTarget (device, row-major), applied to the keys like ov_insert_kernel does ([O3D] PointCloud::Transform);
// nullptr = the identity, the points as they are.  The compacted points are the untransformed ones either way (SelectByIndex on the
// original source, PlaceRecognition.cpp:105).
struct OvJob {
  const double* xyz; const double* nrm; const int32_t* d_n;   // map slots
  unsigned long long* keys; int32_t* cnt; size_t mask;          // the pair's hash segment
  int32_t* slot_of; int32_t* keep; int32_t* offs;               // per map slot
  double* oxyz; double* onrm; int32_t* out_n;                   // the overlap cloud
  const double* T;                                              // source jobs: sourceToTarget or nullptr; target jobs: nullptr
  int32_t which, pad;                                           // 0 = source (parent), 1 = target (child)
};

__global__ void __launch_bounds__(OV_THREADS) ovb_init_kernel(const OvJob* __restrict__ jobs) {
  pdl_wait();
  const OvJob j = jobs[2 * blockIdx.y];
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i <= j.mask; i += (size_t)gridDim.x * blockDim.x) {
    j.keys[i] = VOXEL_KEY_EMPTY; j.cnt[2 * i] = 0; j.cnt[2 * i + 1] = 0;
  }
}

__global__ void __launch_bounds__(OV_THREADS) ovb_insert_kernel(const OvJob* __restrict__ jobs, double inv, uint32_t* status) {
  pdl_wait();
  const OvJob j = jobs[blockIdx.y];
  const int n = *j.d_n;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    double x = j.xyz[3 * (size_t)i], y = j.xyz[3 * (size_t)i + 1], z = j.xyz[3 * (size_t)i + 2];
    j.slot_of[i] = -1;
    if (!(x == x)) continue;   // tombstone
    if (j.T) transform_point(j.T, x, y, z, &x, &y, &z);
    unsigned long long key;
    if (!voxel_key_of(x, y, z, inv, inv, inv, &key)) { atomicOr(status, ST_KEY_OVERFLOW); continue; }
    bool fresh;
    const long long s = voxel_key_claim(j.keys, j.mask, key, &fresh);
    if (s >= 0) { atomicAdd(&j.cnt[2 * s + j.which], 1); j.slot_of[i] = (int32_t)s; }
  }
}

__global__ void __launch_bounds__(OV_THREADS) ovb_flags_kernel(const OvJob* __restrict__ jobs, int min_pts) {
  pdl_wait();
  const OvJob j = jobs[blockIdx.y];
  const int n = *j.d_n;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int s = j.slot_of[i];
    j.keep[i] = (s >= 0 && j.cnt[2 * s] >= min_pts && j.cnt[2 * s + 1] >= min_pts) ? 1 : 0;
  }
}

__global__ void __launch_bounds__(OV_THREADS) ovb_compact_kernel(const OvJob* __restrict__ jobs) {
  pdl_wait();
  const OvJob j = jobs[blockIdx.y];
  const int n = *j.d_n;
  if (blockIdx.x == 0 && threadIdx.x == 0) *j.out_n = j.offs[n];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (!j.keep[i]) continue;
    const size_t o = (size_t)j.offs[i];
    j.oxyz[3 * o] = j.xyz[3 * (size_t)i]; j.oxyz[3 * o + 1] = j.xyz[3 * (size_t)i + 1]; j.oxyz[3 * o + 2] = j.xyz[3 * (size_t)i + 2];
    j.onrm[3 * o] = j.nrm[3 * (size_t)i]; j.onrm[3 * o + 1] = j.nrm[3 * (size_t)i + 1]; j.onrm[3 * o + 2] = j.nrm[3 * (size_t)i + 2];
  }
}

OverlapTables overlap_tables(Layout& stage, int n) {
  OverlapTables t;
  t.jobs = stage.off((size_t)2 * n * sizeof(OvJob));
  t.scan = stage.off((size_t)2 * n * sizeof(ScanJob));
  t.T = stage.off((size_t)n * 16 * sizeof(double));
  t.end = stage.size;
  return t;
}

// maps[2k], maps[2k + 1]: pair k's source and target; outs[2k], outs[2k + 1]: their overlap clouds (reserved here).  inits: n row-major
// 4x4 sourceToTarget (host), or nullptr for the identity.  The job tables, the transforms and the per-slot arrays live in h->odo; the
// tables and transforms are staged through stage (page-locked, at the offsets tb) so that nothing here waits for the device.
int32_t op_overlap_batch(b2s_handle* h, int n, const b2s_submap* const* maps, const double* inits, double voxel, int min_pts,
                         b2s_cloud* const* outs, unsigned char* stage, const OverlapTables& tb) {
  const int nj = 2 * n;
  auto slots_of = [&](int j) { const size_t m = maps[j]->cloud[0]->n_max; return m > 0 ? m : 1; };
  size_t max_n = 1;
  std::vector<size_t> caps((size_t)n);
  for (int k = 0; k < n; k++) {
    const size_t ns = slots_of(2 * k), nt = slots_of(2 * k + 1);
    size_t cap = 1024;
    while (cap < 2 * (ns + nt)) cap <<= 1;
    caps[(size_t)k] = cap;
    for (size_t m : {ns, nt}) if (m > max_n) max_n = m;
  }
  for (int j = 0; j < nj; j++) {
    const b2s_cloud* map = maps[j]->cloud[0].get();
    B2S_TRY(cloud_reserve(h, outs[j], map->n_max, true));
    outs[j]->has_normals = true;
    outs[j]->n_max = map->n_max;
    outs[j]->n_known = -1;
  }
  OvJob* oj = reinterpret_cast<OvJob*>(stage + tb.jobs);
  ScanJob* sj = reinterpret_cast<ScanJob*>(stage + tb.scan);
  if (inits) memcpy(stage + tb.T, inits, (size_t)n * 16 * sizeof(double));
  // h->odo: the tables at their stage offsets, then every job's tile state (the region zeroed below), then per pair its hash segment
  // and per job its slot, flag and offset arrays
  size_t state_begin = 0, state_end = 0;
  B2S_TRY(carve(h->odo, h->stream, [&](Layout& D) {
    D.off(tb.end);
    state_begin = D.size;
    for (int j = 0; j < nj; j++) scan_bind_state(D, sj[j], slots_of(j));
    state_end = D.size;
    for (int k = 0; k < n; k++) {
      unsigned long long* keys = D.take<unsigned long long>(caps[(size_t)k]);
      int32_t* cnt = D.take<int32_t>(2 * caps[(size_t)k]);
      for (int j = 2 * k; j < 2 * k + 2; j++) {
        oj[j].keys = keys; oj[j].cnt = cnt;
        oj[j].slot_of = D.take<int32_t>(slots_of(j) + 2);
        oj[j].keep = D.take<int32_t>(slots_of(j) + 2);
        oj[j].offs = D.take<int32_t>(slots_of(j) + 2);
      }
    }
  }));
  unsigned char* dev = h->odo.as<unsigned char>();
  for (int j = 0; j < nj; j++) {
    const b2s_cloud* map = maps[j]->cloud[0].get();
    const int k = j / 2, w = j % 2;
    OvJob& J = oj[j];
    J.xyz = map->xyz.as<double>(); J.nrm = map->nrm.as<double>(); J.d_n = map->dn.as<int32_t>();
    J.mask = caps[(size_t)k] - 1;
    J.oxyz = outs[j]->xyz.as<double>(); J.onrm = outs[j]->nrm.as<double>(); J.out_n = outs[j]->dn.as<int32_t>();
    J.T = (inits && w == 0) ? reinterpret_cast<const double*>(dev + tb.T) + 16 * (size_t)k : nullptr;
    J.which = w; J.pad = 0;
    sj[j].in = J.keep; sj[j].out = J.offs; sj[j].d_n = J.d_n;
  }
  B2S_CUDA(cudaMemcpyAsync(dev + tb.jobs, stage + tb.jobs, (inits ? tb.end : tb.T) - tb.jobs, cudaMemcpyHostToDevice, h->stream));
  B2S_CUDA(cudaMemsetAsync(dev + state_begin, 0, state_end - state_begin, h->stream));
  const OvJob* dj = reinterpret_cast<const OvJob*>(dev + tb.jobs);
  const ScanJob* ds = reinterpret_cast<const ScanJob*>(dev + tb.scan);
  size_t max_cap = 1;
  for (size_t c : caps) if (c > max_cap) max_cap = c;
  const int bx = grid_for(max_n, OV_THREADS, 2 * device_sms());   // x blocks per job (grid-stride); y = job
  ProfScope prof(h, PK_FUSE);
  launch_pdl(ovb_init_kernel, dim3((unsigned)grid_for(max_cap, OV_THREADS, 2 * device_sms()), (unsigned)n), OV_THREADS, 0, h->stream, dj);
  launch_pdl(ovb_insert_kernel, dim3((unsigned)bx, (unsigned)nj), OV_THREADS, 0, h->stream, dj, 1.0 / voxel, h->status.as<uint32_t>());
  launch_pdl(ovb_flags_kernel, dim3((unsigned)bx, (unsigned)nj), OV_THREADS, 0, h->stream, dj, min_pts);
  h->launches += 3;
  B2S_TRY(scan_exclusive_i32_batch(h, ds, nj, max_n));
  launch_pdl(ovb_compact_kernel, dim3((unsigned)bx, (unsigned)nj), OV_THREADS, 0, h->stream, dj);
  h->launches++;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

}  // namespace b2s
