// assemble.cu -- A1: the global map assembled on the device, for saving and publishing it; A2: every submap's dense map exported.
//
//   Mapper::getAssembledMapPointCloud                      core/src/Mapper.cpp:183-208 (SlamWrapper::saveMap, SlamWrapperRos::publishMaps)
//   assembleColoredPointCloud                              ros/open3d_slam_ros/src/helpers_ros.cpp:51-70
//   o3d_slam::voxelize -> [O3D] VoxelDownSample             core/src/helpers.cpp:107-113 (assembledMapVoxelSize_, submapVoxelSize_)
//   VoxelizedPointCloud::toPointCloud of every submap       core/src/Voxel.cpp:90-115 (SubmapCollection::dumpToFile(.., true), publishDenseMap)
//
// K-assemble is one set of launches over every submap, whatever their number: a job table holds each submap's map slots, device count
// and list position; a live flag per slot (fusion's tombstones are NaN) with blockIdx.y = job, the batched scan of the flags gives each
// live point its offset within its submap, one CTA scans the per-submap totals into each submap's base, and a scatter writes points,
// normals and, for the coloured map, the point's palette entry.  The voxel path is op_voxel_down_sample on the assembled cloud, with
// the palette entries averaged beside the points.  Every buffer here is the assembly's own and untracked (AssemblyScratch).
#include "assemble.cuh"

namespace b2s {

// Color::getColor(j % 11 + 2) (ros/open3d_slam_ros/include/open3d_slam_ros/Color.hpp:22-32): Gray, Red, Green, Blue, Yellow, Orange,
// Purple, Chartreuse, Teal, Pink, Magenta.  std_msgs/ColorRGBA holds float32: the values are the float32 ones promoted to double.
static const double kPalette[33] = {
    (double)0.5f, (double)0.5f, (double)0.5f, 1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0, 1.0, 1.0, 0.0, 1.0, (double)0.5f, 0.0,
    (double)0.5f, 0.0, 1.0, (double)0.5f, 1.0, 0.0, 0.0, 1.0, 1.0, 1.0, 0.0, (double)0.5f, (double)0.78f, 0.0, (double)0.9f};

struct AsmJob {
  const double* xyz; const double* nrm; const int32_t* d_n;   // the submap's map slots
  int32_t* flags; int32_t* offs;                                 // per slot: live, offset of the live point within the submap
  int32_t label;                                                 // palette entry: list position % 11
  int32_t no_normals;                                            // the map has no normals (b2s_submap::no_normals)
  __device__ long long live() const { return offs[*d_n]; }       // the job's contribution (after the batched scan)
  __device__ bool lacks_normals() const { return no_normals != 0; }
};

__global__ void __launch_bounds__(AS_THREADS) asm_flags_kernel(const AsmJob* __restrict__ jobs) {
  pdl_wait();
  const AsmJob j = jobs[blockIdx.y];
  const int n = *j.d_n;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const double x = j.xyz[3 * (size_t)i];
    j.flags[i] = (x == x) ? 1 : 0;
  }
}

// onrm / olabel / orgb optional: normals, the palette entry (voxel path), the colour itself (unvoxelized coloured map)
__global__ void __launch_bounds__(AS_THREADS) asm_scatter_kernel(const AsmJob* __restrict__ jobs, const long long* __restrict__ base,
                                                                 const int32_t* __restrict__ words, const double* __restrict__ palette,
                                                                 double* __restrict__ oxyz, double* __restrict__ onrm, int32_t* __restrict__ olabel,
                                                                 double* __restrict__ orgb) {
  pdl_wait();
  if (words[0] == 0) return;   // nothing to write, or more than AS_MAX_POINTS
  const AsmJob j = jobs[blockIdx.y];
  const int n = *j.d_n;
  const long long b = base[blockIdx.y];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (!j.flags[i]) continue;
    const size_t o = (size_t)(b + j.offs[i]), s = (size_t)i;
    oxyz[3 * o] = j.xyz[3 * s]; oxyz[3 * o + 1] = j.xyz[3 * s + 1]; oxyz[3 * o + 2] = j.xyz[3 * s + 2];
    if (onrm) { onrm[3 * o] = j.nrm[3 * s]; onrm[3 * o + 1] = j.nrm[3 * s + 1]; onrm[3 * o + 2] = j.nrm[3 * s + 2]; }
    if (olabel) olabel[o] = j.label;
    if (orgb) { const double* c = palette + 3 * j.label; orgb[3 * o] = c[0]; orgb[3 * o + 1] = c[1]; orgb[3 * o + 2] = c[2]; }
  }
}

int32_t op_assemble_map(b2s_handle* h, int n, const b2s_submap* const* submaps, double voxel, b2s_cloud* out, bool colored, double* rgb,
                        size_t capacity, size_t* n_out) {
  if (n == 0) {   // an empty cloud; [O3D] HasNormals() is false for it
    B2S_TRY(cloud_reserve(h, out, 0, false));
    B2S_TRY(cloud_set_count(h, out, 0));
    out->has_normals = false;
    if (n_out) *n_out = 0;
    return B2S_OK;
  }
  AssemblyScratch& A = h->assembly;
  A.cloud.h = h; A.cloud.device = h->device;
  const bool vox = voxel > 0.0;   // helpers.cpp:108-110: voxelize() is a no-op for voxelSize <= 0
  size_t bound = 0, max_n = 1;
  for (int k = 0; k < n; k++) {
    bound += submaps[k]->cloud[0]->n_max;
    if (submaps[k]->cloud[0]->n_max > max_n) max_n = submaps[k]->cloud[0]->n_max;
  }
  // a larger live total is refused on the device before anything is written, so the assembled cloud never needs more
  if (bound > (size_t)AS_MAX_POINTS) bound = (size_t)AS_MAX_POINTS;
  WideGridScope wide(bound);
  b2s_cloud* dst = vox ? &A.cloud : out;
  B2S_TRY(cloud_reserve(h, dst, bound, !colored));
  if (colored && vox) B2S_TRY(A.labels.ensure((bound > 0 ? bound : 1) * 4, h->stream));
  if (colored) B2S_TRY(A.rgb.ensure((bound > 0 ? bound : 1) * 24, h->stream));

  // tables: [AsmJob x n][ScanJob x n][palette] staged from the host, then [base x (n + 1)][words] written on the device
  Layout T;
  const size_t t_jobs = T.off((size_t)n * sizeof(AsmJob)), t_scan = T.off((size_t)n * sizeof(ScanJob)), t_pal = T.off(sizeof(kPalette));
  const size_t staged = T.size, t_base = T.off(((size_t)n + 1) * 8), t_words = T.off(8);
  B2S_TRY(A.tables.ensure(T.size, h->stream));
  if (A.stage.cap < staged) B2S_TRY(A.stage.alloc(2 * staged));   // every call ends with a synchronisation: the stage is free
  unsigned char* st = A.stage.as<unsigned char>();
  unsigned char* tab = A.tables.as<unsigned char>();
  AsmJob* hj = reinterpret_cast<AsmJob*>(st + t_jobs);
  ScanJob* hs = reinterpret_cast<ScanJob*>(st + t_scan);
  memcpy(st + t_pal, kPalette, sizeof(kPalette));
  // slots: every submap's tile state (the region zeroed below), then its flags and offsets
  auto slots_of = [&](int k) { const size_t m = submaps[k]->cloud[0]->n_max; return m > 0 ? m : 1; };
  size_t state_bytes = 0;
  B2S_TRY(carve(A.slots, h->stream, [&](Layout& L) {
    for (int k = 0; k < n; k++) scan_bind_state(L, hs[k], slots_of(k));
    state_bytes = L.size;
    for (int k = 0; k < n; k++) { hj[k].flags = L.take<int32_t>(slots_of(k) + 2); hj[k].offs = L.take<int32_t>(slots_of(k) + 2); }
  }));
  for (int k = 0; k < n; k++) {
    const b2s_submap* sm = submaps[k];
    const b2s_cloud* map = sm->cloud[0].get();
    AsmJob& J = hj[k];
    J.xyz = map->xyz.as<double>(); J.nrm = map->nrm.as<double>(); J.d_n = map->dn.as<int32_t>();
    J.label = k % 11;
    J.no_normals = sm->no_normals ? 1 : 0;
    hs[k].in = J.flags; hs[k].out = J.offs; hs[k].d_n = J.d_n;
  }
  B2S_CUDA(cudaMemcpyAsync(tab, st, staged, cudaMemcpyHostToDevice, h->stream));
  B2S_CUDA(cudaMemsetAsync(A.slots.p, 0, state_bytes, h->stream));
  const AsmJob* dj = reinterpret_cast<const AsmJob*>(tab + t_jobs);
  const ScanJob* ds = reinterpret_cast<const ScanJob*>(tab + t_scan);
  const double* palette = reinterpret_cast<const double*>(tab + t_pal);
  long long* base = reinterpret_cast<long long*>(tab + t_base);
  int32_t* words = reinterpret_cast<int32_t*>(tab + t_words);

  const int bx = grid_for(max_n, AS_THREADS, 2 * device_sms());   // x blocks per job (grid-stride); y = job
  launch_pdl(asm_flags_kernel, dim3((unsigned)bx, (unsigned)n), AS_THREADS, 0, h->stream, dj);
  h->launches++;
  B2S_TRY(scan_exclusive_i32_batch(h, ds, n, max_n));
  launch_pdl(asm_base_kernel<AsmJob>, 1, AS_BASE_THREADS, 0, h->stream, dj, n, base, dst->dn.as<int32_t>(), words, h->status.as<uint32_t>());
  launch_pdl(asm_scatter_kernel, dim3((unsigned)bx, (unsigned)n), AS_THREADS, 0, h->stream, dj, base, words, palette, dst->xyz.as<double>(),
             colored ? nullptr : dst->nrm.as<double>(), colored && vox ? A.labels.as<int32_t>() : nullptr,
             colored && !vox ? A.rgb.as<double>() : nullptr);
  h->launches += 2;
  B2S_CUDA(cudaGetLastError());

  // synchronisation 1: the assembled count, the normals rule and (voxel path) the extent that sizes the voxel key
  unsigned long long hb[6] = {0, 0, 0, 0, 0, 0};
  int32_t hw[2] = {0, 0};
  if (vox) {
    B2S_TRY(h->misc.ensure(256, h->stream));
    B2S_TRY(bbox_reduce(h, dst->xyz.as<double>(), dst->dn.as<int32_t>(), bound > 0 ? bound : 1, nullptr, h->misc.as<unsigned long long>()));
    B2S_TRY(read_back(h, {{hw, words, 8}, {hb, h->misc.p, 48}}));
  } else {
    B2S_TRY(read_back(h, {{hw, words, 8}}));
  }
  size_t cnt = (size_t)hw[0];
  const bool normals = !colored && cnt > 0 && hw[1] == 0;   // Mapper.cpp:201-203: a submap without normals pushes none
  dst->has_normals = normals; dst->n_max = cnt; dst->n_known = (long long)cnt;
  if (vox) {
    if (cnt == 0) {
      B2S_TRY(cloud_reserve(h, out, 0, false));
      B2S_TRY(cloud_set_count(h, out, 0));
      out->has_normals = false;
    } else {
      double ext = 0.0;
      for (int d = 0; d < 3; d++) { const double e = ord_decode(hb[3 + d]) - ord_decode(hb[d]); if (e > ext) ext = e; }
      const int bits = voxel_key_bits(ext, voxel);
      B2S_REQUIRE(bits <= 21, B2S_E_INVALID, "[VoxelDownSample] voxel_size is too small for the extent of the assembled map");
      B2S_TRY(op_voxel_down_sample(h, dst, nullptr, voxel, out, bits, &A.vox, colored ? A.labels.as<int32_t>() : nullptr, palette,
                                   colored ? A.rgb.as<double>() : nullptr));
      // synchronisation 2: the voxel count
      int32_t nv = 0;
      B2S_TRY(read_back(h, {{&nv, out->dn.p, 4}}));
      cnt = (size_t)nv;
      out->n_max = cnt; out->n_known = (long long)cnt;
    }
  }
  if (n_out) *n_out = cnt;
  if (!colored) return B2S_OK;
  B2S_REQUIRE(cnt <= capacity, B2S_E_CAPACITY, "colour buffer too small: %zu points, capacity %zu", cnt, capacity);
  if (cnt && rgb) {
    B2S_CUDA(cudaMemcpyAsync(rgb, A.rgb.p, cnt * 24, cudaMemcpyDeviceToHost, h->stream));
    B2S_CUDA(cudaStreamSynchronize(h->stream));
  }
  return B2S_OK;
}

// ---- A2: the dense maps ---------------------------------------------------------------------------------------------------------------
// K-dense-export is one set of launches over every listed dense table.  The tables are mostly empty (2^22 slots, at most 7/8 usable), so
// nothing is kept per slot: a count pass writes the live slots of every 2048-slot tile (blockIdx.y = table), the batched scan turns them
// into tile offsets, asm_base_kernel scans the per-entry totals into int64 bases and checks the capacity, and after the one
// synchronisation (the total sizes the output) a gather recomputes each live slot's rank within its tile and writes sum / count.
struct DenseTable {                  // one listed entry that has a dense map
  const int32_t* cnt; const double* sum;         // the table: count and 6 running sums per slot
  int32_t* tiles; int32_t* toffs;                // per tile: live slots; their exclusive scan (toffs[ntiles] = the table's live voxels)
  long long cap;                                 // slots
  int32_t ntiles;                                // tiles of DX_TILE slots (the batched scan reads its length here)
  int32_t entry;                                 // list position: where its points go
  __device__ unsigned live_mask(long long s0) const;
};
struct DenseJob {                    // one listed entry, for asm_base_kernel
  const int32_t* total;                          // its table's toffs[ntiles], or a zero word without a dense map
  __device__ long long live() const { return *total; }
  __device__ bool lacks_normals() const { return true; }   // the dense export has no normals
};

// the counts of slots s0 .. s0 + DX_ITEMS - 1 (0 past the table) into c; returns how many are live (count > 0)
__device__ __forceinline__ int dx_load(const int32_t* __restrict__ cnt, long long cap, long long s0, int32_t c[DX_ITEMS]) {
  if (s0 + DX_ITEMS <= cap) {
    const int4 a = *reinterpret_cast<const int4*>(cnt + s0), b = *reinterpret_cast<const int4*>(cnt + s0 + 4);
    c[0] = a.x; c[1] = a.y; c[2] = a.z; c[3] = a.w; c[4] = b.x; c[5] = b.y; c[6] = b.z; c[7] = b.w;
  } else {
#pragma unroll
    for (int k = 0; k < DX_ITEMS; k++) c[k] = s0 + k < cap ? cnt[s0 + k] : 0;
  }
  int live = 0;
#pragma unroll
  for (int k = 0; k < DX_ITEMS; k++) live += c[k] > 0;
  return live;
}

__device__ unsigned DenseTable::live_mask(long long s0) const {
  int32_t c[DX_ITEMS];
  dx_load(cnt, cap, s0, c);
  unsigned m = 0;
#pragma unroll
  for (int k = 0; k < DX_ITEMS; k++) m |= (c[k] > 0 ? 1u : 0u) << k;
  return m;
}

// Voxel.cpp:90-115 per live slot, in slot order: the same division as dense_gather_kernel (b2s_submap_dense_download)
__global__ void __launch_bounds__(AS_THREADS) dx_gather_kernel(const DenseTable* __restrict__ tabs, const long long* __restrict__ base,
                                                               double* __restrict__ oxyz) {
  pdl_wait();
  const DenseTable t = tabs[blockIdx.y];
  if ((int)blockIdx.x >= t.ntiles) return;
  const long long s0 = (long long)blockIdx.x * DX_TILE + threadIdx.x * DX_ITEMS;
  int32_t c[DX_ITEMS];
  const int live = dx_load(t.cnt, t.cap, s0, c);
  const int rank = tile_rank(live);
  if (live == 0) return;
  size_t o = (size_t)(base[t.entry] + t.toffs[blockIdx.x] + rank);
#pragma unroll
  for (int k = 0; k < DX_ITEMS; k++) {
    if (c[k] <= 0) continue;
    const double* s = t.sum + 6 * (size_t)(s0 + k);
    const double n = (double)c[k];
    oxyz[3 * o] = s[0] / n; oxyz[3 * o + 1] = s[1] / n; oxyz[3 * o + 2] = s[2] / n;
    o++;
  }
}

int32_t op_assemble_dense_maps(b2s_handle* h, int n, const b2s_submap* const* submaps, b2s_cloud* out, int64_t* offsets) {
  auto tiles_of = [&](int k) { return (submaps[k]->dense_cap + DX_TILE - 1) / DX_TILE; };
  int m = 0;   // entries with a dense map
  size_t max_tiles = 1;
  for (int k = 0; k < n; k++) {
    if (submaps[k]->dense_cap == 0) continue;
    if (tiles_of(k) > max_tiles) max_tiles = tiles_of(k);
    m++;
  }
  if (m == 0) {   // nothing to read: every range is empty
    if (offsets) for (int k = 0; k <= n; k++) offsets[k] = 0;
    B2S_TRY(cloud_reserve(h, out, 0, false));
    B2S_TRY(cloud_set_count(h, out, 0));
    out->has_normals = false;
    return B2S_OK;
  }
  AssemblyScratch& A = h->assembly;
  // tables: [DenseTable x m][ScanJob x m][DenseJob x n][zero word] staged from the host, then [base x (n + 1)][out_n, words x 2] written
  // on the device.  The stage also receives the bases.
  Layout L;
  const size_t t_tab = L.off((size_t)m * sizeof(DenseTable)), t_scan = L.off((size_t)m * sizeof(ScanJob));
  const size_t t_jobs = L.off((size_t)n * sizeof(DenseJob)), t_zero = L.off(4), staged = L.size;
  const size_t t_base = L.off(((size_t)n + 1) * 8), t_words = L.off(12);   // words: [0] the count, [1..2] asm_base_kernel's words
  B2S_TRY(A.tables.ensure(L.size, h->stream));
  if (A.stage.cap < t_words) B2S_TRY(A.stage.alloc(2 * t_words));   // with the bases; every earlier call synchronised after its upload
  unsigned char* st = A.stage.as<unsigned char>();
  unsigned char* tab = A.tables.as<unsigned char>();
  DenseTable* ht = reinterpret_cast<DenseTable*>(st + t_tab);
  ScanJob* hs = reinterpret_cast<ScanJob*>(st + t_scan);
  DenseJob* hj = reinterpret_cast<DenseJob*>(st + t_jobs);
  memset(st + t_zero, 0, 4);
  const int32_t* zero = reinterpret_cast<const int32_t*>(tab + t_zero);
  // slots: every table's tile state (the region zeroed below), then its tile counts and offsets
  size_t state_bytes = 0;
  B2S_TRY(carve(A.slots, h->stream, [&](Layout& S) {
    for (int k = 0, t = 0; k < n; k++) if (submaps[k]->dense_cap) scan_bind_state(S, hs[t++], tiles_of(k));
    state_bytes = S.size;
    for (int k = 0, t = 0; k < n; k++)
      if (submaps[k]->dense_cap) { ht[t].tiles = S.take<int32_t>(tiles_of(k)); ht[t].toffs = S.take<int32_t>(tiles_of(k) + 2); t++; }
  }));
  for (int k = 0, t = 0; k < n; k++) {
    const b2s_submap* sm = submaps[k];
    if (sm->dense_cap == 0) { hj[k].total = zero; continue; }
    const size_t nt = tiles_of(k);
    DenseTable& T = ht[t];
    T.cnt = sm->dense_cnt.as<int32_t>(); T.sum = sm->dense_sum.as<double>();
    T.cap = (long long)sm->dense_cap; T.ntiles = (int32_t)nt; T.entry = k;
    hs[t].in = T.tiles; hs[t].out = T.toffs;
    hs[t].d_n = reinterpret_cast<const int32_t*>(tab + t_tab + (size_t)t * sizeof(DenseTable) + offsetof(DenseTable, ntiles));
    hj[k].total = T.toffs + nt;
    t++;
  }
  B2S_CUDA(cudaMemcpyAsync(tab, st, staged, cudaMemcpyHostToDevice, h->stream));
  B2S_CUDA(cudaMemsetAsync(A.slots.p, 0, state_bytes, h->stream));
  const DenseTable* dt = reinterpret_cast<const DenseTable*>(tab + t_tab);
  const ScanJob* ds = reinterpret_cast<const ScanJob*>(tab + t_scan);
  const DenseJob* dj = reinterpret_cast<const DenseJob*>(tab + t_jobs);
  long long* base = reinterpret_cast<long long*>(tab + t_base);
  int32_t* words = reinterpret_cast<int32_t*>(tab + t_words);

  launch_pdl(tile_count_kernel<DenseTable>, dim3((unsigned)max_tiles, (unsigned)m), AS_THREADS, 0, h->stream, dt);
  h->launches++;
  B2S_TRY(scan_exclusive_i32_batch(h, ds, m, max_tiles));
  launch_pdl(asm_base_kernel<DenseJob>, 1, AS_BASE_THREADS, 0, h->stream, dj, n, base, words, words + 1, h->status.as<uint32_t>());
  h->launches++;
  B2S_CUDA(cudaGetLastError());

  // the one synchronisation: the bases are the offsets, the last one the total; above AS_MAX_POINTS the status reports ST_CAPACITY
  // and nothing has been written
  long long* hb = reinterpret_cast<long long*>(st + t_base);
  B2S_CUDA(cudaMemcpyAsync(hb, base, ((size_t)n + 1) * 8, cudaMemcpyDeviceToHost, h->stream));
  B2S_TRY(check_status(h));
  const size_t total = (size_t)hb[n];
  if (offsets) for (int k = 0; k <= n; k++) offsets[k] = hb[k];
  B2S_TRY(cloud_reserve(h, out, total, false));
  if (total > 0) {
    launch_pdl(dx_gather_kernel, dim3((unsigned)max_tiles, (unsigned)m), AS_THREADS, 0, h->stream, dt, base, out->xyz.as<double>());
    h->launches++;
  }
  B2S_TRY(cloud_set_count(h, out, total));
  out->has_normals = false;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

}  // namespace b2s
