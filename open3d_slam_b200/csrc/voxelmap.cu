// voxelmap.cu -- F4: o3d_slam::VoxelMap as a device container (SURVEY.md section 8a row F4).
//
// Reference: VoxelMap : VoxelHashMap<VoxelWithIdxs>  (core/include/open3d_slam/Voxel.hpp:19-36, core/src/Voxel.cpp:123-160):
// an unordered_map from the voxel key floor(p * (1 / voxelSize)) (VoxelHashMap.hpp:43-50) to, per named layer, the list
// of point indices that fell into the voxel.  Its users on this path: the revisit check of SubmapCollection
// (isSwitchingSubmapsConsistant, core/src/SubmapCollection.cpp:352-364: the share of scan points that hit an occupied
// voxel of the candidate submap's map), space carving and the overlap selection (which have kernels of their own).
//
// Device layout: open-addressing table of packed 3 x 21-bit keys; per (layer, slot) a chain of entries {point index,
// next} built with atomicExch, plus a per-(layer, slot) entry count.  Layers are small integers (the shim maps the
// reference's layer names, e.g. Submap::voxelMapLayer = "map", to 0..B2S_VOXEL_MAP_LAYERS-1).
// getIndicesInVoxel answers come back sorted ascending, which is the reference's order whenever a layer was filled by
// insertCloud(layer, cloud) (iota indices, appended in order).
#include "common.cuh"

using namespace b2s;

struct b2s_voxel_map {
  b2s_handle* h = nullptr;
  int device = 0;
  double voxel[3] = {0, 0, 0};
  double inv[3] = {0, 0, 0};
  size_t cap = 0;              // slots (power of two)
  DevBuf keys;                 // uint64 packed key, EMPTY = ~0
  DevBuf head;                 // int32 [LAYERS][cap]: first entry of the chain, -1 = none
  DevBuf cnt;                  // int32 [LAYERS][cap]: entries of that layer in the voxel
  DevBuf next, eidx;           // per entry
  DevBuf used;                 // int32 [0] occupied voxels, [1] entries
  size_t entries_bound = 0;    // host-side upper bound of the entries in use
};

namespace b2s {

constexpr int VM_THREADS = 256;
constexpr int VM_LAYERS = 4;

struct VmView {
  double ix, iy, iz;
  size_t mask;
  const unsigned long long* keys;
};

__global__ void __launch_bounds__(VM_THREADS) vm_clear_kernel(unsigned long long* keys, int32_t* head, int32_t* cnt, size_t cap, int32_t* used) {
  pdl_wait();
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < cap; i += (size_t)gridDim.x * blockDim.x) {
    keys[i] = VOXEL_KEY_EMPTY;
    for (int l = 0; l < VM_LAYERS; l++) { head[(size_t)l * cap + i] = -1; cnt[(size_t)l * cap + i] = 0; }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) { used[0] = 0; used[1] = 0; }
}

// VoxelMap::insertCloud(layer, cloud): voxels_[getKey(p_i)].idxs_[layer].emplace_back(i)      Voxel.cpp:123-135
__global__ void __launch_bounds__(VM_THREADS) vm_insert_kernel(const double* __restrict__ xyz, const int32_t* __restrict__ d_n, double ix, double iy,
                                                               double iz, int layer, unsigned long long* keys, int32_t* head, int32_t* cnt,
                                                               int32_t* __restrict__ next, int32_t* __restrict__ eidx, size_t cap, size_t entries_cap,
                                                               int32_t* used, uint32_t* status) {
  pdl_wait();
  const int n = *d_n;
  const size_t mask = cap - 1;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    unsigned long long key;
    if (!voxel_key_of(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], ix, iy, iz, &key)) { atomicOr(status, ST_KEY_OVERFLOW); continue; }
    bool fresh;
    const long long s = voxel_key_claim(keys, mask, key, &fresh);
    if (fresh) { if ((size_t)atomicAdd(&used[0], 1) + 1 > cap - cap / 8) atomicOr(status, ST_HASH_FULL); }
    if (s < 0) continue;
    const int e = atomicAdd(&used[1], 1);
    if ((size_t)e >= entries_cap) { atomicOr(status, ST_CAPACITY); continue; }
    eidx[e] = i;
    next[e] = atomicExch(&head[(size_t)layer * cap + s], e);
    atomicAdd(&cnt[(size_t)layer * cap + s], 1);
  }
}

// VoxelHashMap::hasVoxelContainingPoint (VoxelHashMap.hpp:112-118) for every point, optionally moved by T first
// (isSwitchingSubmapsConsistant: p = mapToRangeSensor * scan.points_[i], an isometry applied as R p + t)
__global__ void __launch_bounds__(VM_THREADS) vm_has_kernel(const double* __restrict__ xyz, const int32_t* __restrict__ d_n,
                                                            const double* __restrict__ Tdev, VmView v, int32_t* __restrict__ flags, int32_t* hits) {
  pdl_wait();
  const int n = *d_n;
  double T[12];
  if (Tdev) {
#pragma unroll
    for (int i = 0; i < 12; i++) T[i] = Tdev[i];
  }
  int local = 0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    double x = xyz[3 * i], y = xyz[3 * i + 1], z = xyz[3 * i + 2];
    if (Tdev) affine_point(T, x, y, z, &x, &y, &z);
    unsigned long long key;
    const bool has = voxel_key_of(x, y, z, v.ix, v.iy, v.iz, &key) && voxel_key_find(v.keys, v.mask, key) >= 0;
    if (flags) flags[i] = has ? 1 : 0;
    local += has ? 1 : 0;
  }
  local = warp_sum_i(local);
  if ((threadIdx.x & 31) == 0 && local) atomicAdd(hits, local);
}

// getIndicesInVoxel(layer, p), batched: first the list lengths ...
__global__ void __launch_bounds__(VM_THREADS) vm_count_kernel(const double* __restrict__ xyz, const int32_t* __restrict__ d_n, VmView v, int layer,
                                                              const int32_t* __restrict__ cnt, size_t cap, int32_t* __restrict__ out) {
  pdl_wait();
  const int n = *d_n;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    unsigned long long key;
    int c = 0;
    if (voxel_key_of(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], v.ix, v.iy, v.iz, &key)) {
      const long long s = voxel_key_find(v.keys, v.mask, key);
      if (s >= 0) c = cnt[(size_t)layer * cap + (size_t)s];
    }
    out[i] = c;
  }
}
// ... then the lists themselves (chain order is arbitrary: each list is sorted ascending in place)
__global__ void __launch_bounds__(VM_THREADS) vm_fill_kernel(const double* __restrict__ xyz, const int32_t* __restrict__ d_n, VmView v, int layer,
                                                             const int32_t* __restrict__ head, const int32_t* __restrict__ next,
                                                             const int32_t* __restrict__ eidx, size_t cap, const int32_t* __restrict__ offs,
                                                             int32_t* __restrict__ out) {
  pdl_wait();
  const int n = *d_n;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    unsigned long long key;
    if (!voxel_key_of(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], v.ix, v.iy, v.iz, &key)) continue;
    const long long s = voxel_key_find(v.keys, v.mask, key);
    if (s < 0) continue;
    int32_t* dst = out + offs[i];
    int m = 0;
    for (int e = head[(size_t)layer * cap + (size_t)s]; e >= 0; e = next[e]) {
      const int val = eidx[e];
      int j = m++;
      while (j > 0 && dst[j - 1] > val) { dst[j] = dst[j - 1]; --j; }   // insertion sort: lists are a handful of entries
      dst[j] = val;
    }
  }
}

}  // namespace b2s

extern "C" {

int32_t b2s_voxel_map_create(b2s_handle* h, const double voxel_size[3], size_t capacity_voxels, b2s_voxel_map** out) {
  B2S_REQUIRE(h && voxel_size && out && capacity_voxels > 0, B2S_E_INVALID, "bad argument");
  B2S_REQUIRE(voxel_size[0] > 0.0 && voxel_size[1] > 0.0 && voxel_size[2] > 0.0, B2S_E_INVALID, "voxel size must be > 0");
  LOCK(h);
  return create_object(out, [&](b2s_voxel_map* vm) -> int32_t {
    vm->h = h; vm->device = h->device;
    for (int d = 0; d < 3; d++) { vm->voxel[d] = voxel_size[d]; vm->inv[d] = 1.0 / voxel_size[d]; }   // fromVoxelSize, VoxelHashMap.hpp:43-45
    size_t cap = 1024;
    while (cap < 2 * capacity_voxels) cap <<= 1;
    vm->cap = cap;
    B2S_TRY(vm->keys.ensure(cap * 8, h->stream));
    B2S_TRY(vm->head.ensure(cap * 4 * VM_LAYERS, h->stream));
    B2S_TRY(vm->cnt.ensure(cap * 4 * VM_LAYERS, h->stream));
    B2S_TRY(vm->used.ensure(64, h->stream));
    return b2s_voxel_map_clear(h, vm);
  });
}

void b2s_voxel_map_destroy(b2s_voxel_map* vm) { destroy_object(vm); }

int32_t b2s_voxel_map_clear(b2s_handle* h, b2s_voxel_map* vm) {
  B2S_REQUIRE(h && vm, B2S_E_INVALID, "null argument");
  LOCK(h);
  launch_pdl(vm_clear_kernel, 4 * device_sms(), VM_THREADS, 0, h->stream, vm->keys.as<unsigned long long>(), vm->head.as<int32_t>(), vm->cnt.as<int32_t>(), vm->cap,
                                                         vm->used.as<int32_t>());
  h->launches++;
  vm->entries_bound = 0;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

int32_t b2s_voxel_map_insert_cloud(b2s_handle* h, b2s_voxel_map* vm, int32_t layer, const b2s_cloud* cloud) {
  B2S_REQUIRE(h && vm && cloud, B2S_E_INVALID, "null argument");
  B2S_REQUIRE(layer >= 0 && layer < VM_LAYERS, B2S_E_INVALID, "layer must be in [0, %d)", VM_LAYERS);
  LOCK(h);
  const size_t n_max = cloud->n_max;
  if (n_max == 0) return B2S_OK;
  const size_t want = vm->entries_bound + n_max;
  B2S_TRY(vm->next.ensure(want * 4, h->stream, true));
  B2S_TRY(vm->eidx.ensure(want * 4, h->stream, true));
  const size_t ecap = (vm->next.cap < vm->eidx.cap ? vm->next.cap : vm->eidx.cap) / 4;
  launch_pdl(vm_insert_kernel, grid_for(n_max, VM_THREADS), VM_THREADS, 0, h->stream, 
      cloud->xyz.as<double>(), cloud->dn.as<int32_t>(), vm->inv[0], vm->inv[1], vm->inv[2], layer, vm->keys.as<unsigned long long>(),
      vm->head.as<int32_t>(), vm->cnt.as<int32_t>(), vm->next.as<int32_t>(), vm->eidx.as<int32_t>(), vm->cap, ecap, vm->used.as<int32_t>(),
      h->status.as<uint32_t>());
  h->launches++;
  vm->entries_bound = want;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

int32_t b2s_voxel_map_size(b2s_handle* h, const b2s_voxel_map* vm, size_t* n_voxels) {
  B2S_REQUIRE(h && vm && n_voxels, B2S_E_INVALID, "null argument");
  LOCK(h);
  int32_t used = 0;
  const int32_t rc = read_back(h, {{&used, vm->used.p, 4}});
  *n_voxels = (size_t)used;
  return rc;
}

int32_t b2s_voxel_map_has_voxel(b2s_handle* h, const b2s_voxel_map* vm, const b2s_cloud* points, const double T_or_null[16], int32_t* flags_or_null,
                                size_t capacity, size_t* n_hits) {
  B2S_REQUIRE(h && vm && points, B2S_E_INVALID, "null argument");
  LOCK(h);
  const size_t n_max = points->n_max > 0 ? points->n_max : 1;
  B2S_REQUIRE(!flags_or_null || capacity >= points->n_max, B2S_E_CAPACITY, "flag array holds %zu entries, the cloud has up to %zu points", capacity,
              points->n_max);
  B2S_TRY(h->tmp_i32.ensure((n_max + 64) * 4, h->stream));
  int32_t* d_hits = h->tmp_i32.as<int32_t>();
  int32_t* d_flags = d_hits + 16;
  B2S_CUDA(cudaMemsetAsync(d_hits, 0, 4, h->stream));
  const double* Td = nullptr;
  if (T_or_null) {
    double* slot = h->poses.as<double>() + 16 * PS_VOXEL_MAP;
    B2S_TRY(pose_to_device(h, T_or_null, slot));
    Td = slot;
  }
  VmView v{vm->inv[0], vm->inv[1], vm->inv[2], vm->cap - 1, vm->keys.as<unsigned long long>()};
  launch_pdl(vm_has_kernel, grid_for(n_max, VM_THREADS), VM_THREADS, 0, h->stream, points->xyz.as<double>(), points->dn.as<int32_t>(), Td, v,
                                                                          flags_or_null ? d_flags : nullptr, d_hits);
  h->launches++;
  if (flags_or_null && points->n_max) B2S_CUDA(cudaMemcpyAsync(flags_or_null, d_flags, points->n_max * 4, cudaMemcpyDeviceToHost, h->stream));
  int32_t hits = 0;
  const int32_t rc = read_back(h, {{&hits, d_hits, 4}});
  if (n_hits) *n_hits = (size_t)hits;
  return rc;
}

int32_t b2s_voxel_map_indices_in_voxel(b2s_handle* h, const b2s_voxel_map* vm, int32_t layer, const b2s_cloud* points, int32_t* offsets,
                                       size_t offsets_capacity, int32_t* indices, size_t indices_capacity, size_t* n_indices) {
  B2S_REQUIRE(h && vm && points && offsets, B2S_E_INVALID, "null argument");
  B2S_REQUIRE(layer >= 0 && layer < VM_LAYERS, B2S_E_INVALID, "layer must be in [0, %d)", VM_LAYERS);
  LOCK(h);
  const size_t n_max = points->n_max;
  B2S_REQUIRE(offsets_capacity >= n_max + 1, B2S_E_CAPACITY, "offsets must hold n + 1 = %zu entries", n_max + 1);
  const size_t nm = n_max > 0 ? n_max : 1;
  B2S_TRY(h->flags.ensure((nm + 1) * 4, h->stream));
  B2S_TRY(h->offs.ensure((nm + 2) * 4, h->stream));
  VmView v{vm->inv[0], vm->inv[1], vm->inv[2], vm->cap - 1, vm->keys.as<unsigned long long>()};
  launch_pdl(vm_count_kernel, grid_for(nm, VM_THREADS), VM_THREADS, 0, h->stream, points->xyz.as<double>(), points->dn.as<int32_t>(), v, layer,
                                                                         vm->cnt.as<int32_t>(), vm->cap, h->flags.as<int32_t>());
  h->launches++;
  B2S_TRY(scan_exclusive_i32(h, h->flags.as<int32_t>(), h->offs.as<int32_t>(), points->dn.as<int32_t>(), nm, nullptr));
  // the total decides how much scratch the lists need: one small synchronising read
  int32_t n = 0;
  B2S_CUDA(cudaMemcpyAsync(&n, points->dn.p, 4, cudaMemcpyDeviceToHost, h->stream));
  B2S_CUDA(cudaStreamSynchronize(h->stream));
  int32_t total = 0;
  B2S_CUDA(cudaMemcpyAsync(&total, h->offs.as<int32_t>() + n, 4, cudaMemcpyDeviceToHost, h->stream));
  B2S_CUDA(cudaStreamSynchronize(h->stream));
  if (n_indices) *n_indices = (size_t)total;
  B2S_REQUIRE(!indices || (size_t)total <= indices_capacity, B2S_E_CAPACITY, "index array holds %zu entries, %d needed", indices_capacity, total);
  B2S_CUDA(cudaMemcpyAsync(offsets, h->offs.p, ((size_t)n + 1) * 4, cudaMemcpyDeviceToHost, h->stream));
  if (indices && total > 0) {
    B2S_TRY(h->tmp_i32.ensure(((size_t)total + 64) * 4, h->stream));
    launch_pdl(vm_fill_kernel, grid_for(nm, VM_THREADS), VM_THREADS, 0, h->stream, points->xyz.as<double>(), points->dn.as<int32_t>(), v, layer,
                                                                          vm->head.as<int32_t>(), vm->next.as<int32_t>(), vm->eidx.as<int32_t>(),
                                                                          vm->cap, h->offs.as<int32_t>(), h->tmp_i32.as<int32_t>());
    h->launches++;
    B2S_CUDA(cudaMemcpyAsync(indices, h->tmp_i32.p, (size_t)total * 4, cudaMemcpyDeviceToHost, h->stream));
  }
  return check_status(h);
}

}  // extern "C"
