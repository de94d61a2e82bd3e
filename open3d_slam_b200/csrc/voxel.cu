// voxel.cu -- K-crop+voxel (P1+P2), K-select (P4), F0 transform and the order-preserving compaction they share.
//
//   P1  CroppingVolume::crop                       core/src/croppers.cpp:76-106,121-165
//   P2  o3d_slam::voxelize -> [O3D] VoxelDownSample core/src/helpers.cpp:107-113
//   P4  [O3D] RandomDownSample (seeded stand-in)    core/src/ScanToMapRegistration.cpp:39, core/src/Odometry.cpp:29
//   F0  o3d_slam::transform                         core/src/helpers.cpp:273-305
//
// Voxel down-sample = Morton-keyed radix bucketing: the crop predicate is folded into the key kernel (cropped-out
// points get the sentinel key and sort to the tail), keys are the Morton interleave of
// floor((p - (minBound - v/2)) / v) computed with the reference's fp64 operations, a stable LSD radix sort groups the
// members of each voxel in input order, and one thread per segment head accumulates them in that order in fp64 --
// the voxel means are therefore bit-identical to the CPU reference; only the output ORDER differs (Morton order
// instead of std::unordered_map iteration order, which the reference leaves unspecified).
#include "common.cuh"

namespace b2s {

constexpr int VX_THREADS = 256;

// ---- bbox of the points that pass the cropper (shared with grid_index.cu) ------------------------------------------
__global__ void bbox_init_kernel(unsigned long long* bbox, int32_t* kept) {
  pdl_wait();
  int t = threadIdx.x;
  if (t < 3) bbox[t] = ord_encode(INFINITY);
  else if (t < 6) bbox[t] = ord_encode(-INFINITY);
  if (t == 6 && kept) *kept = 0;
}

__global__ void __launch_bounds__(VX_THREADS) bbox_kernel(const double* __restrict__ xyz, const int32_t* __restrict__ d_n, CropDev crop,
                                                          int use_crop, unsigned long long* bbox) {
  pdl_wait();
  const int n = *d_n;
  double mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    double x = xyz[3 * i], y = xyz[3 * i + 1], z = xyz[3 * i + 2];
    if (!(x == x && y == y && z == z)) continue;
    if (use_crop && !crop_within(crop, x, y, z)) continue;
    mn[0] = fmin(mn[0], x); mn[1] = fmin(mn[1], y); mn[2] = fmin(mn[2], z);
    mx[0] = fmax(mx[0], x); mx[1] = fmax(mx[1], y); mx[2] = fmax(mx[2], z);
  }
  __shared__ double s[6][VX_THREADS / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int d = 0; d < 3; d++) { mn[d] = warp_min(mn[d]); mx[d] = warp_max(mx[d]); }
  if (lane == 0) { for (int d = 0; d < 3; d++) { s[d][warp] = mn[d]; s[3 + d][warp] = mx[d]; } }
  __syncthreads();
  if (threadIdx.x < 6) {
    int d = threadIdx.x;
    double v = s[d][0];
    for (int w = 1; w < VX_THREADS / 32; w++) v = d < 3 ? fmin(v, s[d][w]) : fmax(v, s[d][w]);
    if (d < 3) atomicMin(&bbox[d], ord_encode(v)); else atomicMax(&bbox[d], ord_encode(v));
  }
}

int32_t bbox_reduce(b2s_handle* h, const double* xyz, const int32_t* d_n, size_t n_max, const CropDev* crop, unsigned long long* bbox) {
  CropDev cd = crop ? *crop : make_crop(nullptr);
  launch_pdl(bbox_init_kernel, 1, 32, 0, h->stream, bbox, nullptr);
  launch_pdl(bbox_kernel, grid_for(n_max, VX_THREADS), VX_THREADS, 0, h->stream, xyz, d_n, cd, crop ? 1 : 0, bbox);
  h->launches += 2;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

// ---- cloud helpers ----------------------------------------------------------------------------------------------------
__global__ void set_count_kernel(int32_t* dn, int32_t n) {
  pdl_wait(); *dn = n; }

int32_t cloud_reserve(b2s_handle* h, b2s_cloud* c, size_t n, bool normals) {
  size_t m = n > 0 ? n : 1;
  B2S_TRY(c->xyz.ensure(m * 24, h->stream, true));
  if (normals) B2S_TRY(c->nrm.ensure(m * 24, h->stream, true));
  B2S_TRY(c->dn.ensure(4, h->stream, true));
  return B2S_OK;
}
int32_t cloud_set_count(b2s_handle* h, b2s_cloud* c, size_t n) {
  B2S_TRY(c->dn.ensure(4, h->stream, true));
  launch_pdl(set_count_kernel, 1, 1, 0, h->stream, c->dn.as<int32_t>(), (int32_t)n);
  h->launches++;
  c->n_known = (long long)n;
  c->n_max = c->fixed_cap ? c->fixed_cap : n;
  return B2S_OK;
}

// ---- P1: order-preserving crop (flags -> scan -> scatter) -----------------------------------------------------------
__global__ void __launch_bounds__(VX_THREADS) crop_flags_kernel(const double* __restrict__ xyz, const int32_t* __restrict__ d_n,
                                                                CropDev crop, int32_t* __restrict__ flags) {
  pdl_wait();
  const int n = *d_n;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    flags[i] = crop_within(crop, xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]) ? 1 : 0;
}

__global__ void __launch_bounds__(VX_THREADS) compact_kernel(const double* __restrict__ xyz, const double* __restrict__ nrm,
                                                             const int32_t* __restrict__ d_n, const int32_t* __restrict__ flags,
                                                             const int32_t* __restrict__ offs, double* __restrict__ oxyz,
                                                             double* __restrict__ onrm, int32_t* out_n) {
  pdl_wait();
  const int n = *d_n;
  if (blockIdx.x == 0 && threadIdx.x == 0) *out_n = offs[n];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (!flags[i]) continue;
    const int o = offs[i];
    oxyz[3 * o] = xyz[3 * i]; oxyz[3 * o + 1] = xyz[3 * i + 1]; oxyz[3 * o + 2] = xyz[3 * i + 2];
    if (nrm) { onrm[3 * o] = nrm[3 * i]; onrm[3 * o + 1] = nrm[3 * i + 1]; onrm[3 * o + 2] = nrm[3 * i + 2]; }
  }
}

int32_t compact_cloud(b2s_handle* h, const b2s_cloud* in, const int32_t* flags, b2s_cloud* out, const int32_t* d_n_override = nullptr);
int32_t compact_cloud(b2s_handle* h, const b2s_cloud* in, const int32_t* flags, b2s_cloud* out, const int32_t* d_n_override) {
  const size_t n_max = in->n_max;
  const int32_t* d_n = d_n_override ? d_n_override : in->dn.as<int32_t>();
  B2S_TRY(h->offs.ensure((n_max + 2) * 4, h->stream));
  B2S_TRY(cloud_reserve(h, out, n_max, in->has_normals));
  B2S_TRY(scan_exclusive_i32(h, flags, h->offs.as<int32_t>(), d_n, n_max, nullptr));
  launch_pdl(compact_kernel, grid_for(n_max, VX_THREADS), VX_THREADS, 0, h->stream, 
      in->xyz.as<double>(), in->has_normals ? in->nrm.as<double>() : nullptr, d_n, flags, h->offs.as<int32_t>(),
      out->xyz.as<double>(), in->has_normals ? out->nrm.as<double>() : nullptr, out->dn.as<int32_t>());
  h->launches++;
  out->has_normals = in->has_normals;
  out->n_max = n_max;
  out->n_known = -1;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

int32_t op_crop(b2s_handle* h, const b2s_cloud* in, const CropDev& crop, b2s_cloud* out) {
  const size_t n_max = in->n_max;
  B2S_TRY(h->flags.ensure((n_max + 1) * 4, h->stream));
  launch_pdl(crop_flags_kernel, grid_for(n_max, VX_THREADS), VX_THREADS, 0, h->stream, in->xyz.as<double>(), in->dn.as<int32_t>(), crop,
                                                                               h->flags.as<int32_t>());
  h->launches++;
  return compact_cloud(h, in, h->flags.as<int32_t>(), out);
}

// ---- P2: voxel down-sample ------------------------------------------------------------------------------------------
template <typename K>
__device__ __forceinline__ K morton3(uint32_t x, uint32_t y, uint32_t z);
template <>
__device__ __forceinline__ uint32_t morton3<uint32_t>(uint32_t x, uint32_t y, uint32_t z) {
  return morton_part10(x) | (morton_part10(y) << 1) | (morton_part10(z) << 2);
}
template <>
__device__ __forceinline__ uint64_t morton3<uint64_t>(uint32_t x, uint32_t y, uint32_t z) {
  return morton_part21(x) | (morton_part21(y) << 1) | (morton_part21(z) << 2);
}

template <typename K>
__global__ void __launch_bounds__(VX_THREADS) voxel_keys_kernel(const double* __restrict__ xyz, const int32_t* __restrict__ d_n,
                                                                CropDev crop, int use_crop, const unsigned long long* __restrict__ bbox,
                                                                double voxel, int bits, K* __restrict__ keys, uint32_t* __restrict__ vals,
                                                                uint32_t* status) {
  pdl_wait();
  const int n = *d_n;
  const K invalid = (K)1 << (3 * bits);
  // [O3D] voxel_min_bound = GetMinBound() - voxel_size * 0.5
  const double half = __dmul_rn(voxel, 0.5);
  const double vmx = __dsub_rn(ord_decode(bbox[0]), half), vmy = __dsub_rn(ord_decode(bbox[1]), half), vmz = __dsub_rn(ord_decode(bbox[2]), half);
  const double lim = (double)(1u << bits);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const double x = xyz[3 * i], y = xyz[3 * i + 1], z = xyz[3 * i + 2];
    K key = invalid;
    if ((x == x && y == y && z == z) && (!use_crop || crop_within(crop, x, y, z))) {
      // ref_coord = (p - voxel_min_bound) / voxel_size ; voxel_index = int(floor(ref_coord))
      const double fx = floor(__ddiv_rn(__dsub_rn(x, vmx), voxel)), fy = floor(__ddiv_rn(__dsub_rn(y, vmy), voxel)),
                   fz = floor(__ddiv_rn(__dsub_rn(z, vmz), voxel));
      if (fx >= 0.0 && fy >= 0.0 && fz >= 0.0 && fx < lim && fy < lim && fz < lim) key = morton3<K>((uint32_t)fx, (uint32_t)fy, (uint32_t)fz);
      else atomicOr(status, ST_KEY_OVERFLOW);
    }
    keys[i] = key;
    vals[i] = (uint32_t)i;
  }
}

// head[j] = 1 where a new voxel segment starts in the sorted key array (sentinel keys never start one)
template <typename K>
__global__ void __launch_bounds__(VX_THREADS) seg_head_kernel(const K* __restrict__ keys, const int32_t* __restrict__ d_n, int bits,
                                                              int singletons_for_invalid, int32_t* __restrict__ head) {
  pdl_wait();
  const int n = *d_n;
  const K invalid = (K)1 << (3 * bits);
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
    const K k = keys[j];
    int hd;
    if (k >= invalid) hd = singletons_for_invalid;
    else hd = (j == 0 || keys[j - 1] != k) ? 1 : 0;
    head[j] = hd;
  }
}

// one thread per segment head: accumulate the members in input order (the sort is stable), AccumulatedPoint semantics
template <typename K>
__global__ void __launch_bounds__(VX_THREADS) voxel_mean_kernel(const K* __restrict__ keys, const uint32_t* __restrict__ vals,
                                                                const int32_t* __restrict__ d_n, const int32_t* __restrict__ head,
                                                                const int32_t* __restrict__ offs, const double* __restrict__ xyz,
                                                                const double* __restrict__ nrm, double* __restrict__ oxyz,
                                                                double* __restrict__ onrm, int32_t* out_n) {
  pdl_wait();
  const int n = *d_n;
  if (blockIdx.x == 0 && threadIdx.x == 0) *out_n = offs[n];
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
    if (!head[j]) continue;
    const K k = keys[j];
    double sx = 0, sy = 0, sz = 0, nx = 0, ny = 0, nz = 0;
    int cnt = 0;
    for (int t = j; t < n && keys[t] == k; ++t) {
      const uint32_t i = vals[t];
      sx = __dadd_rn(sx, xyz[3 * i]); sy = __dadd_rn(sy, xyz[3 * i + 1]); sz = __dadd_rn(sz, xyz[3 * i + 2]);
      if (nrm) {
        const double a = nrm[3 * i], b = nrm[3 * i + 1], c = nrm[3 * i + 2];
        if (a == a && b == b && c == c) { nx = __dadd_rn(nx, a); ny = __dadd_rn(ny, b); nz = __dadd_rn(nz, c); }
      }
      cnt++;
    }
    const int o = offs[j];
    const double c = (double)cnt;
    oxyz[3 * o] = __ddiv_rn(sx, c); oxyz[3 * o + 1] = __ddiv_rn(sy, c); oxyz[3 * o + 2] = __ddiv_rn(sz, c);
    if (nrm) { onrm[3 * o] = __ddiv_rn(nx, c); onrm[3 * o + 1] = __ddiv_rn(ny, c); onrm[3 * o + 2] = __ddiv_rn(nz, c); }
  }
}

static int bits_for(double extent, double voxel) {
  double cells = floor(extent / voxel) + 3.0;
  int b = 1;
  while ((double)(1u << b) < cells && b < 22) b++;
  return b;
}

template <typename K>
static int32_t voxel_impl(b2s_handle* h, const b2s_cloud* in, const CropDev* crop, double voxel, int bits, b2s_cloud* out) {
  const size_t n_max = in->n_max > 0 ? in->n_max : 1;
  B2S_TRY(h->keys.ensure(n_max * sizeof(K) * 2, h->stream));
  B2S_TRY(h->vals.ensure(n_max * 4 * 2, h->stream));
  B2S_TRY(h->flags.ensure((n_max + 1) * 4, h->stream));
  B2S_TRY(h->offs.ensure((n_max + 2) * 4, h->stream));
  B2S_TRY(cloud_reserve(h, out, n_max, in->has_normals));
  K* keys = h->keys.as<K>(); K* keys_alt = keys + n_max;
  uint32_t* vals = h->vals.as<uint32_t>(); uint32_t* vals_alt = vals + n_max;
  const int32_t* d_n = in->dn.as<int32_t>();
  const int blocks = grid_for(n_max, VX_THREADS);
  CropDev cd = crop ? *crop : make_crop(nullptr);
  { ProfScope prof(h, PK_VOXEL);
  launch_pdl(voxel_keys_kernel<K>, blocks, VX_THREADS, 0, h->stream, in->xyz.as<double>(), d_n, cd, crop ? 1 : 0, h->misc.as<unsigned long long>(),
                                                             voxel, bits, keys, vals, h->status.as<uint32_t>());
  h->launches++; }
  if constexpr (sizeof(K) == 4) {
    B2S_TRY(radix_sort_pairs_u32(h, keys, vals, keys_alt, vals_alt, d_n, n_max, 3 * bits + 1));
  } else {
    B2S_TRY(radix_sort_pairs_u64(h, keys, vals, keys_alt, vals_alt, d_n, n_max, 3 * bits + 1));
  }
  ProfScope prof2(h, PK_VOXEL);
  launch_pdl(seg_head_kernel<K>, blocks, VX_THREADS, 0, h->stream, keys, d_n, bits, 0, h->flags.as<int32_t>());
  h->launches++;
  B2S_TRY(scan_exclusive_i32(h, h->flags.as<int32_t>(), h->offs.as<int32_t>(), d_n, n_max, nullptr));
  launch_pdl(voxel_mean_kernel<K>, blocks, VX_THREADS, 0, h->stream, keys, vals, d_n, h->flags.as<int32_t>(), h->offs.as<int32_t>(),
                                                             in->xyz.as<double>(), in->has_normals ? in->nrm.as<double>() : nullptr,
                                                             out->xyz.as<double>(), in->has_normals ? out->nrm.as<double>() : nullptr,
                                                             out->dn.as<int32_t>());
  h->launches++;
  out->has_normals = in->has_normals;
  out->n_max = in->n_max;
  out->n_known = -1;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

int32_t op_voxel_down_sample(b2s_handle* h, const b2s_cloud* in, const CropDev* crop, double voxel, b2s_cloud* out, int fixed_key_bits) {
  if (voxel <= 0.0) {  // helpers.cpp:108-110: voxelize() is a no-op for voxelSize <= 0 (the crop still applies)
    if (crop) return op_crop(h, in, *crop, out);
    B2S_TRY(cloud_reserve(h, out, in->n_max, in->has_normals));
    B2S_CUDA(cudaMemcpyAsync(out->xyz.p, in->xyz.p, in->n_max * 24, cudaMemcpyDeviceToDevice, h->stream));
    if (in->has_normals) B2S_CUDA(cudaMemcpyAsync(out->nrm.p, in->nrm.p, in->n_max * 24, cudaMemcpyDeviceToDevice, h->stream));
    B2S_CUDA(cudaMemcpyAsync(out->dn.p, in->dn.p, 4, cudaMemcpyDeviceToDevice, h->stream));
    out->has_normals = in->has_normals; out->n_max = in->n_max; out->n_known = in->n_known;
    return B2S_OK;
  }
  B2S_TRY(h->misc.ensure(256, h->stream));
  unsigned long long* bbox = h->misc.as<unsigned long long>();
  B2S_TRY(bbox_reduce(h, in->xyz.as<double>(), in->dn.as<int32_t>(), in->n_max > 0 ? in->n_max : 1, crop, bbox));
  // key width: from the cropper when it bounds the extent, otherwise from the measured bounding box (one sync)
  int bits;
  const bool bounded = crop && !crop->invert && !crop->pose_dev &&
                       (crop->kind == B2S_CROP_MAX_RADIUS || crop->kind == B2S_CROP_MINMAX_RADIUS);
  if (fixed_key_bits > 0) bits = fixed_key_bits;
  else if (bounded) bits = bits_for(2.0 * crop->rmax, voxel);
  else {
    unsigned long long hb[6];
    B2S_CUDA(cudaMemcpyAsync(hb, bbox, 48, cudaMemcpyDeviceToHost, h->stream));
    B2S_CUDA(cudaStreamSynchronize(h->stream));
    double ext = 0.0;
    for (int d = 0; d < 3; d++) { double e = ord_decode(hb[3 + d]) - ord_decode(hb[d]); if (e > ext) ext = e; }
    if (!(ext >= 0.0)) ext = 0.0;  // empty set
    bits = bits_for(ext, voxel);
  }
  B2S_REQUIRE(bits <= 21, B2S_E_INVALID, "[VoxelDownSample] voxel_size is too small for the extent of the cloud");
  if (bits <= 10) return voxel_impl<uint32_t>(h, in, crop, voxel, bits, out);
  return voxel_impl<uint64_t>(h, in, crop, voxel, bits, out);
}

// ---- P4: seeded random down-sample ------------------------------------------------------------------------------------
// hash of the point's bit pattern (not of its index): the selected subset is independent of the order in which the
// voxel down-sample emitted the points, so the Morton-ordered device cloud and any other ordering select the same set
__device__ __forceinline__ uint32_t select_hash(uint32_t seed, double x, double y, double z) {
  const uint64_t a = (uint64_t)__double_as_longlong(x), b = (uint64_t)__double_as_longlong(y), c = (uint64_t)__double_as_longlong(z);
  uint64_t v = a * 0x9E3779B97F4A7C15ull;
  v ^= (b + 0x7F4A7C15F39CC060ull) * 0xC2B2AE3D27D4EB4Full;
  v ^= (c + 0x165667B19E3779F9ull) * 0xD6E8FEB86659FD93ull;
  v += (uint64_t)seed * 0x85EBCA77C2B2AE63ull;
  v ^= v >> 29; v *= 0xBF58476D1CE4E5B9ull; v ^= v >> 32; v *= 0x94D049BB133111EBull; v ^= v >> 29;
  return (uint32_t)(v >> 32);
}
__global__ void __launch_bounds__(VX_THREADS) select_keys_kernel(const double* __restrict__ xyz, const int32_t* __restrict__ d_n, uint32_t seed,
                                                                 uint32_t* __restrict__ keys, uint32_t* __restrict__ vals,
                                                                 int32_t* __restrict__ flags) {
  pdl_wait();
  const int n = *d_n;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    keys[i] = select_hash(seed, xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]);
    vals[i] = (uint32_t)i;
    flags[i] = 0;
  }
}
__global__ void __launch_bounds__(VX_THREADS) select_mark_kernel(const int32_t* __restrict__ d_n, double ratio, const uint32_t* __restrict__ vals,
                                                                 int32_t* __restrict__ flags) {
  pdl_wait();
  const int n = *d_n;
  size_t k = (size_t)((double)n * ratio);  // [O3D]: size_t(points_.size() * sampling_ratio)
  if (k > (size_t)n) k = (size_t)n;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < (int)k; j += gridDim.x * blockDim.x) flags[vals[j]] = 1;
}

// k-th smallest hash by radix SELECT (no sort): one CTA walks the four digits from the top, each pass histograms the
// keys that match the prefix found so far.  sel[0] = the k-th smallest key, sel[1] = how many of the keys EQUAL to it
// belong to the k smallest (ties go to the lower index, like the stable sort / the oracle's (hash, index) order),
// sel[2] = how many keys equal it, sel[3] = k.
constexpr int SK_THREADS = 1024;
__global__ void __launch_bounds__(SK_THREADS) select_kth_kernel(const uint32_t* __restrict__ keys, const int32_t* __restrict__ d_n,
                                                                double ratio, uint32_t* __restrict__ sel) {
  pdl_wait();
  __shared__ int s_hist[256];
  __shared__ int s_scan[8];
  __shared__ uint32_t s_prefix;
  __shared__ int s_rem, s_cnt;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int n = *d_n;
  size_t k = (size_t)((double)n * ratio);  // [O3D]: size_t(points_.size() * sampling_ratio)
  if (k > (size_t)n) k = (size_t)n;
  if (k == 0) { if (tid < 4) sel[tid] = 0; return; }
  uint32_t prefix = 0;
  int rem = (int)k;
  for (int pass = 3; pass >= 0; --pass) {
    const int shift = 8 * pass;
    const uint32_t hi_mask = pass == 3 ? 0u : (0xFFFFFFFFu << (shift + 8));
    if (tid < 256) s_hist[tid] = 0;
    __syncthreads();
    for (int i = tid; i < n; i += SK_THREADS) {
      const uint32_t key = keys[i];
      if ((key & hi_mask) == prefix) atomicAdd(&s_hist[(key >> shift) & 0xFF], 1);
    }
    __syncthreads();
    int h = 0, inc = 0;
    if (tid < 256) {
      h = s_hist[tid];
      inc = h;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
      if (lane == 31) s_scan[warp] = inc;
    }
    __syncthreads();
    if (tid < 256) {
      for (int w = 0; w < warp; ++w) inc += s_scan[w];
      const int exc = inc - h;
      if (exc < rem && rem <= inc) { s_prefix = prefix | ((uint32_t)tid << shift); s_rem = rem - exc; s_cnt = h; }
    }
    __syncthreads();
    prefix = s_prefix; rem = s_rem;
    __syncthreads();
  }
  if (tid == 0) { sel[0] = prefix; sel[1] = (uint32_t)rem; sel[2] = (uint32_t)s_cnt; sel[3] = (uint32_t)k; }
}

__global__ void __launch_bounds__(VX_THREADS) select_mark_kth_kernel(const int32_t* __restrict__ d_n, const uint32_t* __restrict__ keys,
                                                                     const uint32_t* __restrict__ sel, int32_t* __restrict__ flags) {
  pdl_wait();
  const int n = *d_n;
  const uint32_t kth = sel[0], need = sel[1], cnt_eq = sel[2], k = sel[3];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const uint32_t key = keys[i];
    int f = 0;
    if (k > 0) {
      if (key < kth) f = 1;
      else if (key == kth) {
        if (need == cnt_eq) f = 1;
        else {   // several points share the threshold hash and only some belong: lowest indices first (vanishingly rare)
          uint32_t before = 0;
          for (int j = 0; j < i; ++j) before += keys[j] == kth;
          f = before < need;
        }
      }
    }
    flags[i] = f;
  }
}

// Selection flags of the seeded down-sample, one int per point of `in`, left in h->flags (ratio < 1 only).
// The hash depends on the point POSITION only, so the flags can be computed before the normals exist: the fused
// pre-processing chain estimates normals for the selected points only (their neighbours still come from the full
// voxelised cloud, so the result is identical to the reference's normals-then-select order).
int32_t select_flags(b2s_handle* h, const b2s_cloud* in, double ratio, uint32_t seed) {
  B2S_REQUIRE(ratio >= 0.0 && ratio < 1.0, B2S_E_INVALID, "[RandomDownSample] sampling_ratio must be in [0, 1]");
  const size_t n_max = in->n_max > 0 ? in->n_max : 1;
  B2S_TRY(h->keys.ensure(n_max * 4 * 2, h->stream));
  B2S_TRY(h->vals.ensure(n_max * 4 * 2, h->stream));
  B2S_TRY(h->flags.ensure((n_max + 1) * 4, h->stream));
  uint32_t* keys = h->keys.as<uint32_t>(); uint32_t* keys_alt = keys + n_max;
  uint32_t* vals = h->vals.as<uint32_t>(); uint32_t* vals_alt = vals + n_max;
  const int blocks = grid_for(n_max, VX_THREADS);
  launch_pdl(select_keys_kernel, blocks, VX_THREADS, 0, h->stream, in->xyz.as<double>(), in->dn.as<int32_t>(), seed, keys, vals,
                                                           h->flags.as<int32_t>());
  h->launches++;
  static const bool sort_select = getenv("B2S_SELECT_SORT") != nullptr;   // A/B knob: the full sort this replaced
  if (!sort_select && n_max <= ((size_t)1 << 18)) {
    ProfScope prof(h, PK_SELECT);
    B2S_TRY(h->misc.ensure(256, h->stream));
    uint32_t* sel = h->misc.as<uint32_t>() + 32;   // words 0..11 of misc hold the voxel bounding box
    launch_pdl(select_kth_kernel, 1, SK_THREADS, 0, h->stream, keys, in->dn.as<int32_t>(), ratio, sel);
    launch_pdl(select_mark_kth_kernel, blocks, VX_THREADS, 0, h->stream, in->dn.as<int32_t>(), keys, sel, h->flags.as<int32_t>());
    h->launches += 2;
    B2S_CUDA(cudaGetLastError());
    return B2S_OK;
  }
  B2S_TRY(radix_sort_pairs_u32(h, keys, vals, keys_alt, vals_alt, in->dn.as<int32_t>(), n_max, 32));
  launch_pdl(select_mark_kernel, blocks, VX_THREADS, 0, h->stream, in->dn.as<int32_t>(), ratio, vals, h->flags.as<int32_t>());
  h->launches++;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

// compaction of `in` by h->flags (as left by select_flags) into `out`
int32_t select_compact(b2s_handle* h, const b2s_cloud* in, double ratio, b2s_cloud* out) {
  B2S_TRY(compact_cloud(h, in, h->flags.as<int32_t>(), out));
  // floor(ratio * n) <= ratio * n_max: keeps the launch bounds of everything downstream (ICP shared memory!) tight
  const size_t bound = (size_t)((double)in->n_max * ratio) + 1;
  if (bound < out->n_max) out->n_max = bound;
  return B2S_OK;
}

int32_t op_random_down_sample(b2s_handle* h, const b2s_cloud* in, double ratio, uint32_t seed, b2s_cloud* out) {
  B2S_REQUIRE(ratio >= 0.0, B2S_E_INVALID, "[RandomDownSample] sampling_ratio must be in [0, 1]");
  const size_t n_max = in->n_max > 0 ? in->n_max : 1;
  if (ratio >= 1.0) {  // the reference only shuffles in this case; the order carries no meaning downstream
    B2S_TRY(cloud_reserve(h, out, n_max, in->has_normals));
    B2S_CUDA(cudaMemcpyAsync(out->xyz.p, in->xyz.p, n_max * 24, cudaMemcpyDeviceToDevice, h->stream));
    if (in->has_normals) B2S_CUDA(cudaMemcpyAsync(out->nrm.p, in->nrm.p, n_max * 24, cudaMemcpyDeviceToDevice, h->stream));
    B2S_CUDA(cudaMemcpyAsync(out->dn.p, in->dn.p, 4, cudaMemcpyDeviceToDevice, h->stream));
    out->has_normals = in->has_normals; out->n_max = in->n_max; out->n_known = in->n_known;
    return B2S_OK;
  }
  B2S_TRY(select_flags(h, in, ratio, seed));
  return select_compact(h, in, ratio, out);
}

// ---- F0: transform (with the reference's near-identity duplication quirk) --------------------------------------------
__global__ void __launch_bounds__(VX_THREADS) transform_kernel(const double* __restrict__ xyz, const double* __restrict__ nrm,
                                                               const int32_t* __restrict__ d_n, const double* __restrict__ Tdev,
                                                               double* __restrict__ oxyz, double* __restrict__ onrm, int32_t* out_n) {
  pdl_wait();
  const int n = *d_n;
  double T[16];
#pragma unroll
  for (int i = 0; i < 16; i++) T[i] = Tdev[i];
  double mx = 0.0;
#pragma unroll
  for (int i = 0; i < 16; i++) mx = fmax(mx, fabs(T[i] - ((i % 5 == 0) ? 1.0 : 0.0)));
  const bool ident = mx < 1e-4;
  const int base = ident ? n : 0;
  if (blockIdx.x == 0 && threadIdx.x == 0) *out_n = base + n;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const double px = xyz[3 * i], py = xyz[3 * i + 1], pz = xyz[3 * i + 2];
    if (ident) { oxyz[3 * i] = px; oxyz[3 * i + 1] = py; oxyz[3 * i + 2] = pz; }
    const double x = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[0], px), __dmul_rn(T[1], py)), __dmul_rn(T[2], pz)), T[3]);
    const double y = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[4], px), __dmul_rn(T[5], py)), __dmul_rn(T[6], pz)), T[7]);
    const double z = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[8], px), __dmul_rn(T[9], py)), __dmul_rn(T[10], pz)), T[11]);
    const double w = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[12], px), __dmul_rn(T[13], py)), __dmul_rn(T[14], pz)), T[15]);
    const int o = base + i;
    oxyz[3 * o] = __ddiv_rn(x, w); oxyz[3 * o + 1] = __ddiv_rn(y, w); oxyz[3 * o + 2] = __ddiv_rn(z, w);
    if (nrm) {
      const double a = nrm[3 * i], b = nrm[3 * i + 1], c = nrm[3 * i + 2];
      if (ident) { onrm[3 * i] = a; onrm[3 * i + 1] = b; onrm[3 * i + 2] = c; }
      onrm[3 * o] = __dadd_rn(__dadd_rn(__dmul_rn(T[0], a), __dmul_rn(T[1], b)), __dmul_rn(T[2], c));
      onrm[3 * o + 1] = __dadd_rn(__dadd_rn(__dmul_rn(T[4], a), __dmul_rn(T[5], b)), __dmul_rn(T[6], c));
      onrm[3 * o + 2] = __dadd_rn(__dadd_rn(__dmul_rn(T[8], a), __dmul_rn(T[9], b)), __dmul_rn(T[10], c));
    }
  }
}

__global__ void write_pose_kernel(double* dst, double t0, double t1, double t2, double t3, double t4, double t5, double t6, double t7,
                                  double t8, double t9, double t10, double t11, double t12, double t13, double t14, double t15) {
  pdl_wait();
  dst[0] = t0; dst[1] = t1; dst[2] = t2; dst[3] = t3; dst[4] = t4; dst[5] = t5; dst[6] = t6; dst[7] = t7;
  dst[8] = t8; dst[9] = t9; dst[10] = t10; dst[11] = t11; dst[12] = t12; dst[13] = t13; dst[14] = t14; dst[15] = t15;
}

// copies a host 4x4 into a device slot without a staging buffer (the values travel as kernel arguments)
int32_t pose_to_device(b2s_handle* h, const double* T, double* dst) {
  launch_pdl(write_pose_kernel, 1, 1, 0, h->stream, dst, T[0], T[1], T[2], T[3], T[4], T[5], T[6], T[7], T[8], T[9], T[10], T[11], T[12], T[13],
                                            T[14], T[15]);
  h->launches++;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

int32_t op_transform(b2s_handle* h, const b2s_cloud* in, const double* T_host, b2s_cloud* out) {
  const size_t n_max = in->n_max > 0 ? in->n_max : 1;
  B2S_TRY(cloud_reserve(h, out, 2 * n_max, in->has_normals));
  double* Td = h->poses.as<double>() + 16 * PS_TRANSFORM;
  B2S_TRY(pose_to_device(h, T_host, Td));
  launch_pdl(transform_kernel, grid_for(n_max, VX_THREADS), VX_THREADS, 0, h->stream, in->xyz.as<double>(),
                                                                              in->has_normals ? in->nrm.as<double>() : nullptr,
                                                                              in->dn.as<int32_t>(), Td, out->xyz.as<double>(),
                                                                              in->has_normals ? out->nrm.as<double>() : nullptr,
                                                                              out->dn.as<int32_t>());
  h->launches++;
  out->has_normals = in->has_normals;
  out->n_max = 2 * in->n_max;
  out->n_known = -1;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

// ---- D1: constant-velocity de-skew (SURVEY.md 8f rank 4) ------------------------------------------------------------
// ConstantVelocityMotionCompensation::undistortInputPointCloud (core/src/MotionCompensation.cpp:64-139): every point is moved by the
// sensor motion accumulated up to its azimuth phase (undistort_point, common.cuh).  The velocities come from the host's pose buffer.
__global__ void __launch_bounds__(VX_THREADS) undistort_kernel(const double* __restrict__ xyz, const int32_t* __restrict__ d_n, double vx, double vy,
                                                               double vz, double wr, double wp, double wy, double duration, int clockwise,
                                                               double* __restrict__ out, int32_t* out_n) {
  pdl_wait();
  const int n = *d_n;
  if (blockIdx.x == 0 && threadIdx.x == 0) *out_n = n;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    undistort_point(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], vx, vy, vz, wr, wp, wy, duration, clockwise, out + 3 * i);
}

int32_t op_undistort(b2s_handle* h, const b2s_cloud* in, const double* lin_vel, const double* ang_vel_rpy, double scan_duration, int clockwise,
                     b2s_cloud* out) {
  const size_t n_max = in->n_max > 0 ? in->n_max : 1;
  B2S_TRY(cloud_reserve(h, out, n_max, false));
  ProfScope prof(h, PK_CROP);
  launch_pdl(undistort_kernel, grid_for(n_max, VX_THREADS), VX_THREADS, 0, h->stream, in->xyz.as<double>(), in->dn.as<int32_t>(), lin_vel[0], lin_vel[1],
                                                                              lin_vel[2], ang_vel_rpy[0], ang_vel_rpy[1], ang_vel_rpy[2],
                                                                              scan_duration, clockwise, out->xyz.as<double>(), out->dn.as<int32_t>());
  h->launches++;
  out->has_normals = false;   // the reference copies the input cloud and rewrites points_ only; raw scans carry no normals
  out->n_max = in->n_max;
  out->n_known = in->n_known;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

// ---- Submap::transform (core/src/Submap.cpp:94-107): [O3D] PointCloud::Transform of the map cloud IN PLACE ----------------
// TransformPoints: (T p).head3 / w ; TransformNormals: R n.  No near-identity duplication here (that quirk belongs to
// o3d_slam::transform, helpers.cpp:273-305).  The pose state follows: mapToRangeSensor_ = mapToRangeSensor_ * T.
struct Mat4 { double m[16]; };
__global__ void __launch_bounds__(VX_THREADS) o3d_transform_inplace_kernel(double* __restrict__ xyz, double* __restrict__ nrm,
                                                                           const int32_t* __restrict__ d_n, Mat4 M) {
  pdl_wait();
  const int n = *d_n;
  const double* T = M.m;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const double px = xyz[3 * i], py = xyz[3 * i + 1], pz = xyz[3 * i + 2];
    const double x = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[0], px), __dmul_rn(T[1], py)), __dmul_rn(T[2], pz)), T[3]);
    const double y = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[4], px), __dmul_rn(T[5], py)), __dmul_rn(T[6], pz)), T[7]);
    const double z = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[8], px), __dmul_rn(T[9], py)), __dmul_rn(T[10], pz)), T[11]);
    const double w = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[12], px), __dmul_rn(T[13], py)), __dmul_rn(T[14], pz)), T[15]);
    xyz[3 * i] = __ddiv_rn(x, w); xyz[3 * i + 1] = __ddiv_rn(y, w); xyz[3 * i + 2] = __ddiv_rn(z, w);
    if (nrm) {
      const double a = nrm[3 * i], b = nrm[3 * i + 1], c = nrm[3 * i + 2];
      nrm[3 * i] = __dadd_rn(__dadd_rn(__dmul_rn(T[0], a), __dmul_rn(T[1], b)), __dmul_rn(T[2], c));
      nrm[3 * i + 1] = __dadd_rn(__dadd_rn(__dmul_rn(T[4], a), __dmul_rn(T[5], b)), __dmul_rn(T[6], c));
      nrm[3 * i + 2] = __dadd_rn(__dadd_rn(__dmul_rn(T[8], a), __dmul_rn(T[9], b)), __dmul_rn(T[10], c));
    }
  }
}
__global__ void pose_right_multiply_kernel(double* pose, Mat4 M) {
  pdl_wait();   // pose = pose * T (row-major), one thread
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  double P[16], R[16];
  for (int i = 0; i < 16; i++) P[i] = pose[i];
  for (int i = 0; i < 4; i++)
    for (int j = 0; j < 4; j++) {
      double s = 0.0;
      for (int k = 0; k < 4; k++) s += P[4 * i + k] * M.m[4 * k + j];
      R[4 * i + j] = s;
    }
  for (int i = 0; i < 16; i++) pose[i] = R[i];
}
// VoxelizedPointCloud::transform (core/src/Voxel.cpp:49-64): the transform is applied to the position SUM, keys stay
__global__ void dense_transform_kernel(double* __restrict__ sums, const int32_t* __restrict__ cnts, size_t cap, Mat4 M) {
  pdl_wait();
  const double* T = M.m;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < cap; i += (size_t)gridDim.x * blockDim.x) {
    if (cnts[i] <= 0) continue;
    const double a = sums[6 * i], b = sums[6 * i + 1], c = sums[6 * i + 2];
    sums[6 * i] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[0], a), __dmul_rn(T[1], b)), __dmul_rn(T[2], c)), T[3]);
    sums[6 * i + 1] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[4], a), __dmul_rn(T[5], b)), __dmul_rn(T[6], c)), T[7]);
    sums[6 * i + 2] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[8], a), __dmul_rn(T[9], b)), __dmul_rn(T[10], c)), T[11]);
  }
}

int32_t op_submap_transform(b2s_handle* h, b2s_submap* sm, const double* T_host) {
  Mat4 M;
  for (int i = 0; i < 16; i++) M.m[i] = T_host[i];
  b2s_cloud* map = sm->cloud[0].get();
  const size_t n_max = map->n_max > 0 ? map->n_max : 1;
  launch_pdl(o3d_transform_inplace_kernel, grid_for(n_max, VX_THREADS), VX_THREADS, 0, h->stream, map->xyz.as<double>(),
                                                                                          map->has_normals ? map->nrm.as<double>() : nullptr,
                                                                                          map->dn.as<int32_t>(), M);
  launch_pdl(pose_right_multiply_kernel, 1, 32, 0, h->stream, sm->pose.as<double>(), M);
  h->launches += 2;
  if (sm->dense_cap > 0) {
    launch_pdl(dense_transform_kernel, 4 * device_sms(), 256, 0, h->stream, sm->dense_sum.as<double>(), sm->dense_cnt.as<int32_t>(), sm->dense_cap, M);
    h->launches++;
  }
  B2S_CUDA(cudaGetLastError());
  return fuse_rehash(h, sm);   // the points moved into other voxels: the fusion's voxel hash follows
}

}  // namespace b2s
