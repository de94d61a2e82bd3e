// fuse.cu -- K-fuse (F0+F1) and K-dense (F3): the map side of the hot path.
//
//   F1  Submap::insertScan (no carving)        core/src/Submap.cpp:39-75
//         transform(T, scan)                   core/src/helpers.cpp:273-305   (duplication quirk when T ~ identity)
//         mapCloud_ += scan
//         voxelizeWithinCroppingVolume(...)    core/src/helpers.cpp:115-183   (+ AccumulatedPoint :30-70)
//   F3  Submap::insertScanDenseMap -> VoxelizedPointCloud::insert   core/src/Submap.cpp:77-92, core/src/Voxel.cpp:66-88
//
// F1 on the device keeps the reference's semantics exactly (every in-cropper point of the map is bucketed by
// floor(p * (1/v)) on the GLOBAL-origin grid, an old map point counts as ONE member, members are summed in map order, normals:
// mean of non-NaN then normalized(), points outside the cropper pass through untouched) but does the work of one SCAN, not of
// the whole map: see "K-fuse" below.  Nothing happens unless the (device-resident) gate is open, which is how the gates of
// Mapper::addRangeMeasurement (core/src/Mapper.cpp:151,170-176) run without a host sync.  Map order: stable slots; new voxels
// are appended (the reference: pass-through first, then std::unordered_map order -- unspecified, nothing depends on it).
#include "common.cuh"

namespace b2s {

constexpr int FZ_THREADS = 256;

int32_t pose_to_device(b2s_handle* h, const double* T, double* dst);  // voxel.cu

// ---------------------------------------------------------------------------------------------------------------------
// K-fuse.  The reference re-buckets EVERY in-cropper point of the whole map on every insertion (helpers.cpp:152-167); here the
// map keeps a persistent voxel hash (key = floor(p * (1/v)) on the global-origin grid, VoxelHashMap.hpp:47-50; value = the
// chain of map points inside that voxel), and an insertion only does work proportional to the SCAN:
//   K1 stage+link   every scan point: transform (o3d_slam::transform, duplication quirk kept), stage, key, find-or-insert the
//                   voxel, link the staged point into its chain, first toucher of a voxel queues it;
//   K2 merge        one thread per touched voxel (+ per voxel of the short list of voxels that hold more than one map
//                   point): AccumulatedPoint over the in-cropper members in map order -- old map points first (each counts as
//                   ONE member, helpers.cpp:30-70), then the scan points in scan order -- mean, normalized mean normal; the result
//                   takes the slot of the oldest member (or a fresh slot), merged-away map points become tombstones (NaN),
//                   out-of-cropper members pass through (a staged one gets a slot of its own), the chain is rebuilt.  The
//                   mean of three or more members can round across a face of the voxel: such a result is left out of the
//                   chain and marked (pstamp = -stamp) for K3;
//   K3 renormalize  the reference's pass also rewrites the normal of every UNTOUCHED in-cropper point as normalized(n / 1)
//                   (helpers.cpp:172), which is not idempotent in floating point.  Most normals reach a fixed point of that
//                   operation after one or two applications, and skipping a point whose normal already is one is exact.  So the
//                   submap keeps a worklist of the slots whose normal may not be a fixed point yet: every slot after a rehash,
//                   every slot K2 writes a normal to.  K3 applies the operation to the worklist entries K2 did not rewrite and
//                   that are inside the cropper, and drops an entry once its normal is a fixed point (or it is a tombstone):
//                   O(worklist), not O(map), and the normals stay bit-faithful.  K3 also links every marked mean (all of
//                   them are on the worklist) into the chain of the voxel its position now keys to (the reference re-buckets
//                   it there at the next insertion), and queues that voxel as a duplicate when it already held a point; + commit
//                   of the counters and the pose.  No chain is walked in K3, so relinking cannot race with a reader.
//                   B2S_RENORM_FULL=1 visits every map slot instead of the worklist (A/B switch and test reference).
// Positions of untouched voxels are unchanged by the reference's pass (mean of one member = p / 1), so the map is identical
// as a keyed set.  Tombstones are skipped by every reader (NaN never passes a cropper or enters an index) and dropped whenever
// the map is compacted (carving) or leaves the device.
// ---------------------------------------------------------------------------------------------------------------------
// slot of `key`, inserting it when absent (-1: table full); the table counts as full past 3/4 of its slots.  The fusion table keeps
// this probe of its own instead of voxel_key_claim: counting the claimed slot inside the loop measured faster in the per-scan chain.
__device__ __forceinline__ long long fv_find_or_insert(unsigned long long* keys, size_t mask, unsigned long long key, int32_t* ms, uint32_t* status) {
  size_t s = (size_t)voxel_key_hash(key) & mask;
  for (size_t probe = 0; probe <= mask; ++probe, s = (s + 1) & mask) {
    const unsigned long long old = atomicCAS(&keys[s], VOXEL_KEY_EMPTY, key);
    if (old == VOXEL_KEY_EMPTY) {
      if ((size_t)atomicAdd(&ms[MS_VUSED], 1) + 1 > mask - mask / 4) atomicOr(status, ST_HASH_FULL);
      return (long long)s;
    }
    if (old == key) return (long long)s;
  }
  atomicOr(status, ST_HASH_FULL);
  return -1;
}

// K2 writes a position into a map slot: the submap's box takes it.  An atomic only when the box grows, which it stops doing once the
// map covers the place (a mean can still leave its members' box by the rounding of the sum and the division); a stale read of the
// box only costs an atomic that changes nothing.
__device__ __forceinline__ void box_fold_point(unsigned long long* box, const double* p) {
  for (int d = 0; d < 3; d++) {
    const unsigned long long e = ord_encode(p[d]);
    if (e < box[d]) atomicMin(&box[d], e);
    if (e > box[3 + d]) atomicMax(&box[3 + d], e);
  }
}

struct FuseView {
  double* mxyz; double* mnrm; int32_t* vnext; int32_t* pstamp;
  const double* sxyz; const double* snrm; int32_t* snext; const int32_t* sin;
};
__device__ __forceinline__ int fv_next(const FuseView& v, int idx) { return idx >= FUSE_STAGE_BASE ? v.snext[idx - FUSE_STAGE_BASE] : v.vnext[idx]; }

// K3's renormalisation worklist (wflag == nullptr: B2S_RENORM_FULL, K3 visits every slot and no list is kept)
struct Worklist { int32_t* wflag; int32_t* wlist; size_t stride; };
// K2 wrote the normal of `slot`: it joins the current half once
__device__ __forceinline__ void fv_worklist_join(const Worklist& w, int32_t* ms, int slot) {
  if (w.wflag == nullptr || atomicExch(&w.wflag[slot], 1) != 0) return;
  const int sel = ms[MS_WSEL] & 1;
  w.wlist[(size_t)sel * w.stride + atomicAdd(&ms[MS_NW + sel], 1)] = slot;
}

// K1
__global__ void __launch_bounds__(FZ_THREADS) fuse_stage_kernel(const double* __restrict__ sxyz_in, const double* __restrict__ snrm_in,
                                                                const int32_t* __restrict__ d_nscan, const double* __restrict__ Tdev,
                                                                const int32_t* __restrict__ gate, CropDev crop, double inv, size_t stage_cap,
                                                                double* __restrict__ stage_xyz, double* __restrict__ stage_nrm,
                                                                int32_t* __restrict__ stage_next, int32_t* __restrict__ stage_in,
                                                                unsigned long long* vkeys, int32_t* vhead, int32_t* vstamp, size_t vmask,
                                                                int32_t* __restrict__ touched, int32_t* ms, uint32_t* status) {
  pdl_wait();
  const int ns = *d_nscan;
  const bool open = (gate == nullptr || *gate != 0) && ns > 0;  // Submap.cpp:41-43: empty scan -> nothing happens
  if (!open) return;
  double T[16];
#pragma unroll
  for (int i = 0; i < 16; i++) T[i] = Tdev[i];
  const bool ident = near_identity(T);
  const size_t m = (size_t)(ident ? 2 : 1) * (size_t)ns;
  if (m > stage_cap) { if (blockIdx.x == 0 && threadIdx.x == 0) atomicOr(status, ST_CAPACITY); return; }
  const int cur = ms[MS_STAMP] + 1;
  for (size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x; j < m; j += (size_t)gridDim.x * blockDim.x) {
    const bool copy = ident && j < (size_t)ns;
    const size_t i = copy || !ident ? j : j - (size_t)ns;
    const double px = sxyz_in[3 * i], py = sxyz_in[3 * i + 1], pz = sxyz_in[3 * i + 2];
    // a scan without normals (point-to-point pipelines: estimateNormalsOrCovariancesIfNeeded is a no-op there) fuses with "no
    // normal" = NaN, which AccumulatedPoint skips
    const double qnan = __longlong_as_double(0x7ff8000000000000ll);
    const double a = snrm_in ? snrm_in[3 * i] : qnan, b = snrm_in ? snrm_in[3 * i + 1] : qnan, c = snrm_in ? snrm_in[3 * i + 2] : qnan;
    double x = px, y = py, z = pz, nx = a, ny = b, nz = c;
    if (!copy) {
      transform_point(T, px, py, pz, &x, &y, &z);
      rotate_vector(T, a, b, c, &nx, &ny, &nz);
    }
    stage_xyz[3 * j] = x; stage_xyz[3 * j + 1] = y; stage_xyz[3 * j + 2] = z;
    stage_nrm[3 * j] = nx; stage_nrm[3 * j + 1] = ny; stage_nrm[3 * j + 2] = nz;
    stage_in[j] = crop_within(crop, x, y, z) ? 1 : 0;
    stage_next[j] = -1;
    unsigned long long key;
    if (!(x == x && y == y && z == z)) { stage_in[j] = -1; continue; }   // NaN never survives S1's croppers; dropped here (-1: not linked anywhere)
    if (!voxel_key_of(x, y, z, inv, inv, inv, &key)) { atomicOr(status, ST_KEY_OVERFLOW); stage_in[j] = -1; continue; }
    const long long s = fv_find_or_insert(vkeys, vmask, key, ms, status);
    if (s < 0) { stage_in[j] = -1; continue; }
    stage_next[j] = atomicExch(&vhead[s], FUSE_STAGE_BASE + (int)j);
    if (atomicExch(&vstamp[s], cur) != cur) touched[atomicAdd(&ms[MS_NTOUCHED], 1)] = (int32_t)s;
  }
}

// K2
__global__ void __launch_bounds__(128) fuse_merge_kernel(const int32_t* __restrict__ gate, const int32_t* __restrict__ d_nscan, CropDev crop,
                                                         FuseView v, const unsigned long long* __restrict__ vkeys, double inv, int32_t* vhead,
                                                         int32_t* vstamp, const int32_t* __restrict__ touched, int32_t* dups, int32_t* d_nmap,
                                                         size_t capacity, Worklist wl, int32_t* ms, uint32_t* status, unsigned long long* box) {
  pdl_wait();
  if (!((gate == nullptr || *gate != 0) && *d_nscan > 0)) return;
  const int cur = ms[MS_STAMP] + 1;
  const int ntouched = ms[MS_NTOUCHED];
  const int sel = ms[MS_DUPSEL] & 1;
  const int ndup = min(ms[MS_NDUP + sel], FUSE_DUP_CAP);
  const int32_t* dup_cur = dups + (size_t)sel * FUSE_DUP_CAP;
  int32_t* dup_nxt = dups + (size_t)(sel ^ 1) * FUSE_DUP_CAP;
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < ntouched + ndup; t += gridDim.x * blockDim.x) {
    int slot;
    if (t < ntouched) slot = touched[t];
    else {
      slot = dup_cur[t - ntouched];
      // touched by this insertion as well, or listed twice (K3 may queue a voxel K2 queued already): one thread deals with it
      if (atomicExch(&vstamp[slot], cur) == cur) continue;
    }
    // pass 1: who is in the bucket?  (a map point counts when it is alive and inside the cropper; a staged one by its flag)
    int nin = 0, dest = 0x7fffffff;
    for (int idx = vhead[slot]; idx >= 0; idx = fv_next(v, idx)) {
      bool in;
      if (idx >= FUSE_STAGE_BASE) in = v.sin[idx - FUSE_STAGE_BASE] > 0;
      else {
        const double x = v.mxyz[3 * (size_t)idx], y = v.mxyz[3 * (size_t)idx + 1], z = v.mxyz[3 * (size_t)idx + 2];
        in = (x == x) && crop_within(crop, x, y, z);
        if (in && idx < dest) dest = idx;
      }
      nin += in ? 1 : 0;
    }
    double sx = 0, sy = 0, sz = 0, nx = 0, ny = 0, nz = 0;
    if (nin > 0) {
      // pass 2: AccumulatedPoint in map order: ascending index, map points (< FUSE_STAGE_BASE) before the staged scan points
      int last = -1;
      for (int c = 0; c < nin; ++c) {
        int best = 0x7fffffff;
        for (int idx = vhead[slot]; idx >= 0; idx = fv_next(v, idx)) {
          if (idx <= last || idx >= best) continue;
          bool in;
          if (idx >= FUSE_STAGE_BASE) in = v.sin[idx - FUSE_STAGE_BASE] > 0;
          else {
            const double x = v.mxyz[3 * (size_t)idx], y = v.mxyz[3 * (size_t)idx + 1], z = v.mxyz[3 * (size_t)idx + 2];
            in = (x == x) && crop_within(crop, x, y, z);
          }
          if (in) best = idx;
        }
        last = best;
        const double* px = best >= FUSE_STAGE_BASE ? v.sxyz + 3 * (size_t)(best - FUSE_STAGE_BASE) : v.mxyz + 3 * (size_t)best;
        const double* pn = best >= FUSE_STAGE_BASE ? v.snrm + 3 * (size_t)(best - FUSE_STAGE_BASE) : v.mnrm + 3 * (size_t)best;
        sx = __dadd_rn(sx, px[0]); sy = __dadd_rn(sy, px[1]); sz = __dadd_rn(sz, px[2]);
        const double a = pn[0], b = pn[1], c2 = pn[2];
        if (a == a && b == b && c2 == c2) { nx = __dadd_rn(nx, a); ny = __dadd_rn(ny, b); nz = __dadd_rn(nz, c2); }
      }
      if (dest == 0x7fffffff) {   // a voxel the map did not hold yet: fresh slot
        dest = atomicAdd(d_nmap, 1);
        if ((size_t)dest >= capacity) { atomicOr(status, ST_CAPACITY); atomicSub(d_nmap, 1); dest = -1; }
      }
    }
    // pass 3: rebuild the chain; merged-away map points die, out-of-cropper members pass through
    int newhead = -1, survivors = 0;
    for (int idx = vhead[slot]; idx >= 0;) {
      const int nxt = fv_next(v, idx);
      if (idx >= FUSE_STAGE_BASE) {
        const int j = idx - FUSE_STAGE_BASE;
        if (v.sin[j] == 0) {   // staged point outside the cropper: copied through unchanged (helpers.cpp:156-166)
          const int sl = atomicAdd(d_nmap, 1);
          if ((size_t)sl >= capacity) { atomicOr(status, ST_CAPACITY); atomicSub(d_nmap, 1); }
          else {
            for (int k = 0; k < 3; k++) { v.mxyz[3 * (size_t)sl + k] = v.sxyz[3 * (size_t)j + k]; v.mnrm[3 * (size_t)sl + k] = v.snrm[3 * (size_t)j + k]; }
            box_fold_point(box, v.sxyz + 3 * (size_t)j);
            v.pstamp[sl] = cur;
            v.vnext[sl] = newhead; newhead = sl; survivors++;
            fv_worklist_join(wl, ms, sl);
          }
        }
      } else {
        const double x = v.mxyz[3 * (size_t)idx], y = v.mxyz[3 * (size_t)idx + 1], z = v.mxyz[3 * (size_t)idx + 2];
        const bool alive = x == x;
        const bool in = alive && crop_within(crop, x, y, z);
        if (in) {
          if (idx != dest) {   // merged into `dest`: tombstone
            const double nan = __longlong_as_double(0x7ff8000000000000ll);
            for (int k = 0; k < 3; k++) { v.mxyz[3 * (size_t)idx + k] = nan; v.mnrm[3 * (size_t)idx + k] = nan; }
            atomicAdd(&ms[MS_NDEAD], 1);
          }
        } else if (alive) { v.vnext[idx] = newhead; newhead = idx; survivors++; }
      }
      idx = nxt;
    }
    if (nin > 0 && dest >= 0) {
      const double c = (double)nin;
      v.mxyz[3 * (size_t)dest] = __ddiv_rn(sx, c); v.mxyz[3 * (size_t)dest + 1] = __ddiv_rn(sy, c); v.mxyz[3 * (size_t)dest + 2] = __ddiv_rn(sz, c);
      double a0 = __ddiv_rn(nx, c), a1 = __ddiv_rn(ny, c), a2 = __ddiv_rn(nz, c);
      const double zz = __dadd_rn(__dadd_rn(__dmul_rn(a0, a0), __dmul_rn(a1, a1)), __dmul_rn(a2, a2));
      if (zz > 0.0) { const double sn = sqrt(zz); a0 = __ddiv_rn(a0, sn); a1 = __ddiv_rn(a1, sn); a2 = __ddiv_rn(a2, sn); }  // .normalized()
      v.mnrm[3 * (size_t)dest] = a0; v.mnrm[3 * (size_t)dest + 1] = a1; v.mnrm[3 * (size_t)dest + 2] = a2;
      fv_worklist_join(wl, ms, dest);   // also how K3 finds a mean marked below
      unsigned long long key;
      const double* m = v.mxyz + 3 * (size_t)dest;
      box_fold_point(box, m);
      if (voxel_key_of(m[0], m[1], m[2], inv, inv, inv, &key) && key == vkeys[slot]) {
        v.pstamp[dest] = cur;
        v.vnext[dest] = newhead; newhead = dest; survivors++;
      } else {
        v.pstamp[dest] = -cur;   // the mean left the voxel: K3 links it where it now belongs
        v.vnext[dest] = -1;
      }
    }
    vhead[slot] = newhead;
    if (survivors >= 2) {   // more than one map point in this voxel: they merge as soon as both are inside the cropper
      const int k = atomicAdd(&ms[MS_NDUP + (sel ^ 1)], 1);
      if (k < FUSE_DUP_CAP) dup_nxt[k] = slot; else atomicOr(status, ST_CAPACITY);
    }
  }
}

// the reference's normalized(n / 1) of an untouched in-cropper point (a NaN normal sums to zero in AccumulatedPoint)
__device__ __forceinline__ void fv_renormalized(double& a0, double& a1, double& a2) {
  if (!(a0 == a0 && a1 == a1 && a2 == a2)) { a0 = 0.0; a1 = 0.0; a2 = 0.0; }
  const double zz = __dadd_rn(__dadd_rn(__dmul_rn(a0, a0), __dmul_rn(a1, a1)), __dmul_rn(a2, a2));
  if (zz > 0.0) { const double sn = sqrt(zz); a0 = __ddiv_rn(a0, sn); a1 = __ddiv_rn(a1, sn); a2 = __ddiv_rn(a2, sn); }
}
__device__ __forceinline__ bool fv_same_bits(double a0, double a1, double a2, double b0, double b1, double b2) {
  return __double_as_longlong(a0) == __double_as_longlong(b0) && __double_as_longlong(a1) == __double_as_longlong(b1) &&
         __double_as_longlong(a2) == __double_as_longlong(b2);
}

// K3: normalized(n / 1) for the in-cropper points this insertion did not rewrite, relinking of the means that left their voxel;
// the last block commits the insertion
__global__ void __launch_bounds__(FZ_THREADS) fuse_renorm_commit_kernel(const int32_t* __restrict__ gate, const int32_t* __restrict__ d_nscan,
                                                                        CropDev crop, const double* __restrict__ mxyz, double* __restrict__ mnrm,
                                                                        int32_t* __restrict__ pstamp, const int32_t* __restrict__ d_nmap, double inv,
                                                                        unsigned long long* vkeys, int32_t* vhead, size_t vmask, int32_t* __restrict__ vnext,
                                                                        int32_t* dups, Worklist wl, int32_t* ms, uint32_t* status, double* last_pose,
                                                                        const double* __restrict__ Tdev) {
  pdl_wait();
  if (!((gate == nullptr || *gate != 0) && *d_nscan > 0)) return;
  const int cur = ms[MS_STAMP] + 1;
  const int nxt = (ms[MS_DUPSEL] & 1) ^ 1;   // the list K2 filled for the next insertion
  int32_t* dup_nxt = dups + (size_t)nxt * FUSE_DUP_CAP;
  const bool full = wl.wflag == nullptr;
  const int wsel = ms[MS_WSEL] & 1;
  const int nw = full ? *d_nmap : ms[MS_NW + wsel];
  const int32_t* wcur = wl.wlist + (size_t)wsel * wl.stride;
  int32_t* wnxt = wl.wlist + (size_t)(wsel ^ 1) * wl.stride;
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < nw; t += gridDim.x * blockDim.x) {
    const int i = full ? t : wcur[t];
    const int ps = pstamp[i];
    bool keep = true;   // K2 rewrote the normal in this insertion: it stays on the list untouched
    if (ps == -cur) {   // a mean K2 left out of its chain: find-or-insert the voxel it keys to now (a far key stays unlinked, like a rehash)
      pstamp[i] = cur;
      unsigned long long key;
      const long long s = voxel_key_of(mxyz[3 * (size_t)i], mxyz[3 * (size_t)i + 1], mxyz[3 * (size_t)i + 2], inv, inv, inv, &key)
                              ? fv_find_or_insert(vkeys, vmask, key, ms, status) : -1;
      if (s >= 0) {
        const int prev = atomicExch(&vhead[s], i);
        vnext[i] = prev;
        if (prev >= 0) {   // the voxel holds another map point now: they merge once both are inside the cropper (K2 skips a repeat)
          const int k = atomicAdd(&ms[MS_NDUP + nxt], 1);
          if (k < FUSE_DUP_CAP) dup_nxt[k] = (int32_t)s; else atomicOr(status, ST_CAPACITY);
        }
      }
    } else if (ps != cur) {
      const double x = mxyz[3 * (size_t)i], y = mxyz[3 * (size_t)i + 1], z = mxyz[3 * (size_t)i + 2];
      if (!(x == x)) keep = false;   // a tombstone never changes again
      else {
        const double n0 = mnrm[3 * (size_t)i], n1 = mnrm[3 * (size_t)i + 1], n2 = mnrm[3 * (size_t)i + 2];
        double a0 = n0, a1 = n1, a2 = n2;
        fv_renormalized(a0, a1, a2);
        if (fv_same_bits(a0, a1, a2, n0, n1, n2)) keep = false;   // a fixed point: the operation is the identity from now on
        else if (crop_within(crop, x, y, z)) {
          mnrm[3 * (size_t)i] = a0; mnrm[3 * (size_t)i + 1] = a1; mnrm[3 * (size_t)i + 2] = a2;
          double b0 = a0, b1 = a1, b2 = a2;
          fv_renormalized(b0, b1, b2);
          keep = !fv_same_bits(b0, b1, b2, a0, a1, a2);
        }   // outside the cropper: unchanged, and it stays on the list until it enters the cropper -- a point that never does
            // (a NaN normal of a point-to-point map, a loaded normal of non-unit length) is looked at again on every insertion
      }
    }
    if (!full) {   // survivors go to the other half, warp-aggregated; a dropped slot may join again when K2 rewrites it
      const unsigned act = __activemask();
      const unsigned km = __ballot_sync(act, keep);
      const int lane = threadIdx.x & 31, leader = __ffs(act) - 1;
      int base = 0;
      if (lane == leader && km) base = atomicAdd(&ms[MS_NW + (wsel ^ 1)], __popc(km));
      base = __shfl_sync(act, base, leader);
      if (keep) wnxt[base + __popc(km & ((1u << lane) - 1u))] = i;
      else wl.wflag[i] = 0;
    }
  }
  __shared__ int s_last;
  __syncthreads();
  if (threadIdx.x == 0) s_last = (atomicAdd(&ms[MS_TICKET2], 1) == (int)gridDim.x - 1);
  __syncthreads();
  if (s_last && threadIdx.x == 0) {   // every block has read the stamp and the worklist: commit
    const int sel = ms[MS_DUPSEL] & 1;
    ms[MS_TICKET2] = 0;
    ms[MS_STAMP] = cur;
    ms[MS_NTOUCHED] = 0;
    ms[MS_NDUP + sel] = 0;
    ms[MS_DUPSEL] = sel ^ 1;
    ms[MS_NW + wsel] = 0;
    ms[MS_WSEL] = wsel ^ 1;
    ms[MS_NINS] += 1;                                      // Submap::nScansInsertedMap_
    if (last_pose) for (int i = 0; i < 16; i++) last_pose[i] = Tdev[i];   // mapBuilderCropper_ pose / mapToRangeSensorLastScanInsertion_
  }
}

// ---- (re)build of the voxel hash from the map cloud --------------------------------------------------------------------------
__global__ void fuse_table_clear_kernel(unsigned long long* vkeys, int32_t* vhead, int32_t* vstamp, size_t vcap, int32_t* __restrict__ wflag,
                                        size_t wcap, int32_t* ms, const int32_t* __restrict__ enable, unsigned long long* box) {
  pdl_wait();
  if (enable != nullptr && *enable == 0) return;
  if (blockIdx.x == 0 && threadIdx.x < 6) box[threadIdx.x] = threadIdx.x < 3 ? ord_encode(INFINITY) : ord_encode(-INFINITY);   // the link pass refills it
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < vcap; i += (size_t)gridDim.x * blockDim.x) { vkeys[i] = VOXEL_KEY_EMPTY; vhead[i] = -1; vstamp[i] = 0; }
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < wcap; i += (size_t)gridDim.x * blockDim.x) wflag[i] = 0;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    ms[MS_VUSED] = 0; ms[MS_NTOUCHED] = 0; ms[MS_NDUP] = 0; ms[MS_NDUP + 1] = 0; ms[MS_DUPSEL] = 0; ms[MS_STAMP] = 0;
    ms[MS_WSEL] = 0; ms[MS_NW] = 0; ms[MS_NW + 1] = 0;
  }
}
// relinks every map point, puts every slot on the renormalisation worklist (the normals may have been rewritten) and measures the
// submap's box
__global__ void __launch_bounds__(FZ_THREADS) fuse_table_link_kernel(const double* __restrict__ mxyz, const int32_t* __restrict__ d_nmap, double inv,
                                                                     unsigned long long* vkeys, int32_t* vhead, size_t vmask, int32_t* __restrict__ vnext,
                                                                     int32_t* __restrict__ pstamp, int32_t* __restrict__ wflag, int32_t* __restrict__ wlist,
                                                                     int32_t* ms, uint32_t* status, const int32_t* __restrict__ enable,
                                                                     unsigned long long* box) {
  pdl_wait();
  if (enable != nullptr && *enable == 0) return;
  const int n = *d_nmap;
  if (blockIdx.x == 0 && threadIdx.x == 0) ms[MS_NW] = n;   // half 0 (the clear kernel selected it)
  double mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    vnext[i] = -1; pstamp[i] = 0;
    wflag[i] = 1; wlist[i] = i;
    const double x = mxyz[3 * (size_t)i], y = mxyz[3 * (size_t)i + 1], z = mxyz[3 * (size_t)i + 2];
    if (x == x && y == y && z == z) {   // every live slot, the far ones too
      mn[0] = fmin(mn[0], x); mn[1] = fmin(mn[1], y); mn[2] = fmin(mn[2], z);
      mx[0] = fmax(mx[0], x); mx[1] = fmax(mx[1], y); mx[2] = fmax(mx[2], z);
    }
    unsigned long long key;
    if (!voxel_key_of(x, y, z, inv, inv, inv, &key)) continue;   // tombstones / far points stay unlinked
    const long long s = fv_find_or_insert(vkeys, vmask, key, ms, status);
    if (s >= 0) vnext[i] = atomicExch(&vhead[s], i);
  }
  box_fold_block<FZ_THREADS>(mn, mx, box);
}
// voxels whose chain holds more than one point, reported once (by the chain head)
__global__ void __launch_bounds__(FZ_THREADS) fuse_table_dups_kernel(const unsigned long long* __restrict__ vkeys, const int32_t* __restrict__ vhead,
                                                                     size_t vcap, const int32_t* __restrict__ vnext, int32_t* dups, int32_t* ms,
                                                                     uint32_t* status, const int32_t* __restrict__ enable) {
  pdl_wait();
  if (enable != nullptr && *enable == 0) return;
  for (size_t s = (size_t)blockIdx.x * blockDim.x + threadIdx.x; s < vcap; s += (size_t)gridDim.x * blockDim.x) {
    const int hd = vhead[s];
    if (hd < 0 || vnext[hd] < 0) continue;
    const int k = atomicAdd(&ms[MS_NDUP], 1);
    if (k < FUSE_DUP_CAP) dups[k] = (int32_t)s; else atomicOr(status, ST_CAPACITY);
  }
  (void)vkeys;
}

size_t fuse_table_slots(const b2s_submap* sm) {
  size_t vcap = 4096;
  while (vcap < 2 * sm->capacity) vcap <<= 1;
  return vcap;
}

int32_t fuse_reserve(b2s_handle* h, b2s_submap* sm) {
  if (sm->vcap) return B2S_OK;
  const size_t vcap = fuse_table_slots(sm);
  B2S_TRY(sm->vkeys.ensure(vcap * 8, h->stream));
  B2S_TRY(sm->vhead.ensure(vcap * 4, h->stream));
  B2S_TRY(sm->vstamp.ensure(vcap * 4, h->stream));
  B2S_TRY(sm->vnext.ensure((sm->capacity + 1) * 4, h->stream));
  B2S_TRY(sm->pstamp.ensure((sm->capacity + 1) * 4, h->stream));
  B2S_TRY(sm->dups.ensure((size_t)2 * FUSE_DUP_CAP * 4, h->stream));
  B2S_TRY(sm->wflag.ensure((sm->capacity + 1) * 4, h->stream));
  B2S_TRY(sm->wlist.ensure(2 * (sm->capacity + 1) * 4, h->stream));
  sm->vcap = vcap;
  launch_pdl(fuse_table_clear_kernel, 4 * device_sms(), 256, 0, h->stream, sm->vkeys.as<unsigned long long>(), sm->vhead.as<int32_t>(), sm->vstamp.as<int32_t>(), vcap,
                                                         sm->wflag.as<int32_t>(), sm->capacity + 1, sm->mstate.as<int32_t>(), nullptr,
                                                         sm->bbox.as<unsigned long long>());
  h->launches++;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

int32_t fuse_rehash(b2s_handle* h, b2s_submap* sm, const int32_t* enable_dev) {
  B2S_TRY(fuse_reserve(h, sm));
  b2s_cloud* map = sm->cloud[0].get();
  const size_t n_max = sm->fixed_launch ? sm->capacity : (map->n_max > 0 ? map->n_max : 1);
  int32_t* ms = sm->mstate.as<int32_t>();
  ProfScope prof(h, PK_FUSE);
  launch_pdl(fuse_table_clear_kernel, 4 * device_sms(), 256, 0, h->stream, sm->vkeys.as<unsigned long long>(), sm->vhead.as<int32_t>(), sm->vstamp.as<int32_t>(), sm->vcap,
                                                         sm->wflag.as<int32_t>(), sm->capacity + 1, ms, enable_dev, sm->bbox.as<unsigned long long>());
  launch_pdl(fuse_table_link_kernel, grid_for(n_max, FZ_THREADS), FZ_THREADS, 0, h->stream, map->xyz.as<double>(), map->dn.as<int32_t>(),
                                                                                   1.0 / h->cfg.map_voxel_size, sm->vkeys.as<unsigned long long>(),
                                                                                   sm->vhead.as<int32_t>(), sm->vcap - 1, sm->vnext.as<int32_t>(),
                                                                                   sm->pstamp.as<int32_t>(), sm->wflag.as<int32_t>(), sm->wlist.as<int32_t>(),
                                                                                   ms, h->status.as<uint32_t>(), enable_dev, sm->bbox.as<unsigned long long>());
  launch_pdl(fuse_table_dups_kernel, 4 * device_sms(), FZ_THREADS, 0, h->stream, sm->vkeys.as<unsigned long long>(), sm->vhead.as<int32_t>(), sm->vcap,
                                                               sm->vnext.as<int32_t>(), sm->dups.as<int32_t>(), ms, h->status.as<uint32_t>(), enable_dev);
  h->launches += 3;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

// live points of the map, in map order, in sm->cloud[1] (readers that leave the device: download, size)
__global__ void __launch_bounds__(FZ_THREADS) fuse_alive_flags_kernel(const double* __restrict__ mxyz, const int32_t* __restrict__ d_n, int32_t* __restrict__ flags) {
  pdl_wait();
  const int n = *d_n;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) { const double x = mxyz[3 * (size_t)i]; flags[i] = (x == x) ? 1 : 0; }
}
int32_t compact_cloud(b2s_handle* h, const b2s_cloud* in, const int32_t* flags, b2s_cloud* out, const int32_t* d_n_override = nullptr);   // voxel.cu
int32_t submap_compact_view(b2s_handle* h, b2s_submap* sm, b2s_cloud** view) {
  b2s_cloud* map = sm->cloud[0].get();
  const size_t n_max = map->n_max > 0 ? map->n_max : 1;
  B2S_TRY(h->flags.ensure((n_max + 1) * 4, h->stream));
  launch_pdl(fuse_alive_flags_kernel, grid_for(n_max, FZ_THREADS), FZ_THREADS, 0, h->stream, map->xyz.as<double>(), map->dn.as<int32_t>(), h->flags.as<int32_t>());
  h->launches++;
  B2S_TRY(compact_cloud(h, map, h->flags.as<int32_t>(), sm->cloud[1].get()));
  *view = sm->cloud[1].get();
  return B2S_OK;
}

int32_t op_submap_insert(b2s_handle* h, b2s_submap* sm, const b2s_cloud* scan, const double* T_dev, const int32_t* gate_dev) {
  B2S_REQUIRE(scan->has_normals || h->cfg.icp.reg_type == B2S_REG_POINT_TO_POINT, B2S_E_NO_NORMALS,
              "Submap::insertScan: the pre-processed scan must carry normals (isMergeScanValid) unless the registration is point-to-point");
  b2s_cloud* map = sm->cloud[0].get();
  const double v = h->cfg.map_voxel_size;
  B2S_REQUIRE(v > 0.0, B2S_E_UNSUPPORTED, "map_voxel_size <= 0 (no voxelisation) is not supported on the device path");
  B2S_TRY(fuse_reserve(h, sm));
  // host-side upper bound of the map size.  The exact size is read back asynchronously after an insertion (pinned
  // host word + event); once that copy has landed the bound becomes exact-size + what was appended since.
  if (sm->cnt_pending && !g_capturing && cudaEventQuery(sm->cnt_ev) == cudaSuccess) {   // (no event query inside a capture)
    map->n_max = (size_t)sm->pinned_cnt.as<int32_t>()[0] + sm->adds_after_readback;
    sm->cnt_pending = false;
  }
  const size_t m_max = 2 * (scan->n_max > 0 ? scan->n_max : 1);   // the duplication quirk doubles the scan
  size_t tot_max = map->n_max + m_max;
  if (sm->fixed_launch) tot_max = sm->capacity;   // graph replay: constant launch dimensions, overflow is caught on the device
  if (tot_max > sm->capacity) {
    int32_t n = 0;
    B2S_CUDA(cudaMemcpyAsync(&n, map->dn.p, 4, cudaMemcpyDeviceToHost, h->stream));
    B2S_CUDA(cudaStreamSynchronize(h->stream));
    map->n_max = (size_t)n; map->n_known = n;
    tot_max = map->n_max + m_max;
    if (tot_max > sm->capacity) tot_max = sm->capacity;   // only NEW voxels take slots: a real overflow is caught on the device
  }
  if (sm->stage_cap < m_max) {
    B2S_TRY(sm->stage_xyz.ensure(m_max * 24, h->stream));
    B2S_TRY(sm->stage_nrm.ensure(m_max * 24, h->stream));
    B2S_TRY(sm->stage_next.ensure(m_max * 4, h->stream));
    B2S_TRY(sm->stage_in.ensure(m_max * 4, h->stream));
    B2S_TRY(sm->touched.ensure(m_max * 4, h->stream));
    sm->stage_cap = m_max;
  }
  CropDev crop = make_crop(&h->cfg.scan.map_builder_cropper, T_dev);  // Submap.cpp:71 setPose(mapToRangeSensor)
  const double inv = 1.0 / v;
  int32_t* ms = sm->mstate.as<int32_t>();
  FuseView fv{map->xyz.as<double>(), map->nrm.as<double>(), sm->vnext.as<int32_t>(), sm->pstamp.as<int32_t>(), sm->stage_xyz.as<double>(),
              sm->stage_nrm.as<double>(), sm->stage_next.as<int32_t>(), sm->stage_in.as<int32_t>()};
  // B2S_RENORM_FULL=1: K3 visits every map slot, as before the worklist (A/B switch and test reference)
  static const bool renorm_full = getenv("B2S_RENORM_FULL") && atoi(getenv("B2S_RENORM_FULL")) != 0;
  const Worklist wl{renorm_full ? nullptr : sm->wflag.as<int32_t>(), sm->wlist.as<int32_t>(), sm->capacity + 1};
  // K3's grid: the worklist holds what K2 rewrote (at most one slot per staged point or queued voxel) plus the few normals that
  // cycle; after a rehash (carving, every carveSpaceEveryNscans insertions) it holds the whole map, which the grid-stride loop
  // walks in a few rounds: that insertion pays a full-map K3, as every insertion did before the worklist
  const size_t k3_items = renorm_full ? tot_max : m_max + 4096;
  {
    ProfScope prof(h, PK_FUSE);
    launch_pdl(fuse_stage_kernel, grid_for(m_max, FZ_THREADS), FZ_THREADS, 0, h->stream, 
        scan->xyz.as<double>(), scan->has_normals ? scan->nrm.as<double>() : nullptr, scan->dn.as<int32_t>(), T_dev, gate_dev, crop, inv, sm->stage_cap,
        sm->stage_xyz.as<double>(),
        sm->stage_nrm.as<double>(), sm->stage_next.as<int32_t>(), sm->stage_in.as<int32_t>(), sm->vkeys.as<unsigned long long>(),
        sm->vhead.as<int32_t>(), sm->vstamp.as<int32_t>(), sm->vcap - 1, sm->touched.as<int32_t>(), ms, h->status.as<uint32_t>());
    launch_pdl(fuse_merge_kernel, grid_for(m_max + 4096, 128), 128, 0, h->stream, gate_dev, scan->dn.as<int32_t>(), crop, fv,
                                                                         sm->vkeys.as<unsigned long long>(), inv, sm->vhead.as<int32_t>(),
                                                                         sm->vstamp.as<int32_t>(), sm->touched.as<int32_t>(), sm->dups.as<int32_t>(),
                                                                         map->dn.as<int32_t>(), sm->capacity, wl, ms, h->status.as<uint32_t>(),
                                                                         sm->bbox.as<unsigned long long>());
    launch_pdl(fuse_renorm_commit_kernel, grid_for(k3_items, FZ_THREADS), FZ_THREADS, 0, h->stream, gate_dev, scan->dn.as<int32_t>(), crop, map->xyz.as<double>(),
                                                                                         map->nrm.as<double>(), sm->pstamp.as<int32_t>(),
                                                                                         map->dn.as<int32_t>(), inv, sm->vkeys.as<unsigned long long>(),
                                                                                         sm->vhead.as<int32_t>(), sm->vcap - 1, sm->vnext.as<int32_t>(),
                                                                                         sm->dups.as<int32_t>(), wl, ms, h->status.as<uint32_t>(),
                                                                                         sm->pose.as<double>() + 5 * 16, T_dev);
    h->launches += 3;
  }
  map->n_max = tot_max;   // upper bound only; the exact count lives on the device
  map->n_known = -1;
  map->has_normals = true;
  if (!scan->has_normals) sm->no_normals = true;
  B2S_CUDA(cudaGetLastError());
  if (!sm->fixed_launch) {
    if (!sm->cnt_ev) {
      B2S_TRY(sm->pinned_cnt.alloc(64));
      B2S_CUDA(cudaEventCreateWithFlags(&sm->cnt_ev, cudaEventDisableTiming));
    }
    if (!sm->cnt_pending) {
      B2S_CUDA(cudaMemcpyAsync(sm->pinned_cnt.p, map->dn.p, 4, cudaMemcpyDeviceToHost, h->stream));
      B2S_CUDA(cudaEventRecord(sm->cnt_ev, h->stream));
      sm->cnt_pending = true;
      sm->adds_after_readback = 0;
    } else {
      sm->adds_after_readback += m_max;
    }
  }
  return B2S_OK;
}

// =====================================================================================================================
//  F3 dense map: open-addressing hash (64-bit packed key) of running position / normal sums and counts
// =====================================================================================================================
// cap: a power of two (dense_init)
__device__ __forceinline__ void dense_add_point(double x, double y, double z, double inv, unsigned long long* __restrict__ keys,
                                                double* __restrict__ sums, int32_t* __restrict__ cnts, size_t cap, int32_t* used, uint32_t* status) {
  unsigned long long key;
  if (!voxel_key_of(x, y, z, inv, inv, inv, &key)) { atomicOr(status, ST_KEY_OVERFLOW); return; }
  bool fresh;
  const long long slot = voxel_key_claim(keys, cap - 1, key, &fresh);
  if (fresh && (size_t)atomicAdd(used, 1) + 1 > cap - cap / 8) atomicOr(status, ST_HASH_FULL);
  if (slot < 0) return;
  atomicAdd(&sums[6 * slot], x); atomicAdd(&sums[6 * slot + 1], y); atomicAdd(&sums[6 * slot + 2], z);
  atomicAdd(&cnts[slot], 1);
}

// Submap::insertScanDenseMap goes through o3d_slam::transform (Submap.cpp:80), so its near-identity duplication quirk
// (helpers.cpp:275-292: |T - I|_max < 1e-4 -> the untransformed cloud is copied first and every transformed point is
// appended as well) applies: such a scan lands in the dense map twice.  Kept.
__global__ void __launch_bounds__(FZ_THREADS) dense_insert_kernel(const double* __restrict__ xyz, const int32_t* __restrict__ d_n,
                                                                  const double* __restrict__ Tdev, CropDev crop, double inv,
                                                                  unsigned long long* __restrict__ keys, double* __restrict__ sums,
                                                                  int32_t* __restrict__ cnts, size_t cap, int32_t* used, uint32_t* status,
                                                                  const int32_t* __restrict__ enable) {
  pdl_wait();
  if (enable != nullptr && *enable == 0) return;
  const int n = *d_n;
  double T[16];
#pragma unroll
  for (int i = 0; i < 16; i++) T[i] = Tdev[i];
  const bool ident = near_identity(T);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const double px = xyz[3 * i], py = xyz[3 * i + 1], pz = xyz[3 * i + 2];
    if (!(px == px && py == py && pz == pz)) continue;
    if (!crop_within(crop, px, py, pz)) continue;  // denseMapCropper_ at identity, applied in the sensor frame (Submap.cpp:78-79)
    if (ident) dense_add_point(px, py, pz, inv, keys, sums, cnts, cap, used, status);
    double x, y, z;
    transform_point(T, px, py, pz, &x, &y, &z);
    dense_add_point(x, y, z, inv, keys, sums, cnts, cap, used, status);
  }
}

__global__ void dense_init_kernel(unsigned long long* keys, double* sums, int32_t* cnts, size_t cap, int32_t* used) {
  pdl_wait();
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < cap; i += (size_t)gridDim.x * blockDim.x) {
    keys[i] = VOXEL_KEY_EMPTY; cnts[i] = 0;
    for (int k = 0; k < 6; k++) sums[6 * i + k] = 0.0;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) *used = 0;
}

int32_t dense_init(b2s_handle* h, b2s_submap* sm, size_t cap, double voxel) {
  B2S_TRY(sm->dense_keys.ensure(cap * 8, h->stream));
  B2S_TRY(sm->dense_sum.ensure(cap * 48, h->stream));
  B2S_TRY(sm->dense_cnt.ensure(cap * 4, h->stream));
  B2S_TRY(sm->dense_used.ensure(16, h->stream));
  sm->dense_cap = cap; sm->dense_voxel = voxel;
  launch_pdl(dense_init_kernel, 4 * device_sms(), 256, 0, h->stream, sm->dense_keys.as<unsigned long long>(), sm->dense_sum.as<double>(),
                                                    sm->dense_cnt.as<int32_t>(), cap, sm->dense_used.as<int32_t>());
  h->launches++;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

int32_t op_dense_insert(b2s_handle* h, b2s_submap* sm, const b2s_cloud* raw, const double* T_host, const double* T_dev, const b2s_cropper* crop,
                        const int32_t* enable_dev) {
  B2S_REQUIRE(sm->dense_cap > 0, B2S_E_INVALID, "dense map not initialised");
  const double* Td = T_dev;
  if (!Td) {
    double* slot = h->poses.as<double>() + 16 * PS_CALL;
    B2S_TRY(pose_to_device(h, T_host, slot));
    Td = slot;
  }
  b2s_cropper c0;
  memset(&c0, 0, sizeof(c0));
  if (crop) c0 = *crop;
  c0.center[0] = c0.center[1] = c0.center[2] = 0.0;  // Submap.cpp:78 setPose(Identity)
  launch_pdl(dense_insert_kernel, grid_for(raw->n_max > 0 ? raw->n_max : 1, FZ_THREADS), FZ_THREADS, 0, h->stream, 
      raw->xyz.as<double>(), raw->dn.as<int32_t>(), Td, make_crop(&c0), 1.0 / sm->dense_voxel, sm->dense_keys.as<unsigned long long>(),
      sm->dense_sum.as<double>(), sm->dense_cnt.as<int32_t>(), sm->dense_cap, sm->dense_used.as<int32_t>(), h->status.as<uint32_t>(), enable_dev);
  h->launches++;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

// VoxelizedPointCloud::toPointCloud (Voxel.cpp:90-115): flags -> scan -> gather of sum / count
__global__ void dense_flags_kernel(const int32_t* __restrict__ cnts, size_t cap, int32_t* __restrict__ flags) {
  pdl_wait();
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < cap; i += (size_t)gridDim.x * blockDim.x) flags[i] = cnts[i] > 0 ? 1 : 0;
}
__global__ void dense_gather_kernel(const unsigned long long* __restrict__ keys, const double* __restrict__ sums,
                                    const int32_t* __restrict__ cnts, size_t cap, const int32_t* __restrict__ flags,
                                    const int32_t* __restrict__ offs, double* __restrict__ oxyz, int32_t* __restrict__ okeys, int32_t* out_n) {
  pdl_wait();
  if (blockIdx.x == 0 && threadIdx.x == 0) *out_n = offs[cap];
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < cap; i += (size_t)gridDim.x * blockDim.x) {
    if (!flags[i]) continue;
    const int o = offs[i];
    const double c = (double)cnts[i];
    oxyz[3 * o] = sums[6 * i] / c; oxyz[3 * o + 1] = sums[6 * i + 1] / c; oxyz[3 * o + 2] = sums[6 * i + 2] / c;
    voxel_key_unpack(keys[i], &okeys[3 * o], &okeys[3 * o + 1], &okeys[3 * o + 2]);
  }
}

int32_t dense_to_cloud(b2s_handle* h, b2s_submap* sm, double* d_xyz, int32_t* d_keys, int32_t* d_out_n) {
  const size_t cap = sm->dense_cap;
  B2S_TRY(h->flags.ensure((cap + 1) * 4, h->stream));
  B2S_TRY(h->offs.ensure((cap + 2) * 4, h->stream));
  launch_pdl(dense_flags_kernel, 4 * device_sms(), 256, 0, h->stream, sm->dense_cnt.as<int32_t>(), cap, h->flags.as<int32_t>());
  h->launches++;
  B2S_TRY(scan_exclusive_i32(h, h->flags.as<int32_t>(), h->offs.as<int32_t>(), nullptr, cap, nullptr));
  launch_pdl(dense_gather_kernel, 4 * device_sms(), 256, 0, h->stream, sm->dense_keys.as<unsigned long long>(), sm->dense_sum.as<double>(),
                                                      sm->dense_cnt.as<int32_t>(), cap, h->flags.as<int32_t>(), h->offs.as<int32_t>(), d_xyz,
                                                      d_keys, d_out_n);
  h->launches++;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

// =====================================================================================================================
//  F2  VoxelHashMap query API on the dense map (core/include/open3d_slam/VoxelHashMap.hpp:104-158), batched:
//      hasVoxelContainingPoint / getVoxelContainingPointPtr (-> aggregated content), removeKey(getKey(p)), size, clear.
//  A removed voxel keeps its key in the table with count 0 (= absent for every reader); inserting into it again simply
//  re-populates the slot, so no tombstone handling is needed.
// =====================================================================================================================
__global__ void __launch_bounds__(FZ_THREADS) dense_query_kernel(const double* __restrict__ xyz, const int32_t* __restrict__ d_n, double inv,
                                                                 const unsigned long long* __restrict__ keys, const double* __restrict__ sums,
                                                                 const int32_t* __restrict__ cnts, size_t cap, int32_t* __restrict__ count_out,
                                                                 double* __restrict__ mean_out) {
  pdl_wait();
  const int n = *d_n;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    unsigned long long key;
    const long long s = voxel_key_of(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], inv, inv, inv, &key) ? voxel_key_find(keys, cap - 1, key) : -1;
    const int c = s >= 0 ? cnts[s] : 0;
    count_out[i] = c;
    if (mean_out) {
      const double cd = (double)c;
      for (int k = 0; k < 3; k++) mean_out[3 * i + k] = c > 0 ? sums[6 * s + k] / cd : 0.0;   // AggregatedVoxel::getAggregatedPosition
    }
  }
}

__global__ void __launch_bounds__(FZ_THREADS) dense_remove_kernel(const double* __restrict__ xyz, const int32_t* __restrict__ d_n, double inv,
                                                                  const unsigned long long* __restrict__ keys, double* __restrict__ sums,
                                                                  int32_t* __restrict__ cnts, size_t cap) {
  pdl_wait();
  const int n = *d_n;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    unsigned long long key;
    const long long s = voxel_key_of(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], inv, inv, inv, &key) ? voxel_key_find(keys, cap - 1, key) : -1;
    if (s < 0) continue;
    cnts[s] = 0;   // several points of the same voxel write the same zeros
    for (int k = 0; k < 6; k++) sums[6 * s + k] = 0.0;
  }
}

__global__ void dense_count_kernel(const int32_t* __restrict__ cnts, size_t cap, int32_t* out) {
  pdl_wait();
  int c = 0;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < cap; i += (size_t)gridDim.x * blockDim.x) c += cnts[i] > 0;
  c = warp_sum_i(c);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(out, c);
}

int32_t op_dense_query(b2s_handle* h, const b2s_submap* sm, const b2s_cloud* pts, int32_t* count_dev, double* mean_dev) {
  B2S_REQUIRE(sm->dense_cap > 0, B2S_E_INVALID, "dense map not initialised");
  launch_pdl(dense_query_kernel, grid_for(pts->n_max > 0 ? pts->n_max : 1, FZ_THREADS), FZ_THREADS, 0, h->stream, 
      pts->xyz.as<double>(), pts->dn.as<int32_t>(), 1.0 / sm->dense_voxel, sm->dense_keys.as<unsigned long long>(), sm->dense_sum.as<double>(),
      sm->dense_cnt.as<int32_t>(), sm->dense_cap, count_dev, mean_dev);
  h->launches++;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

int32_t op_dense_remove(b2s_handle* h, b2s_submap* sm, const b2s_cloud* pts) {
  B2S_REQUIRE(sm->dense_cap > 0, B2S_E_INVALID, "dense map not initialised");
  launch_pdl(dense_remove_kernel, grid_for(pts->n_max > 0 ? pts->n_max : 1, FZ_THREADS), FZ_THREADS, 0, h->stream, 
      pts->xyz.as<double>(), pts->dn.as<int32_t>(), 1.0 / sm->dense_voxel, sm->dense_keys.as<unsigned long long>(), sm->dense_sum.as<double>(),
      sm->dense_cnt.as<int32_t>(), sm->dense_cap);
  h->launches++;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

int32_t op_dense_count(b2s_handle* h, const b2s_submap* sm, int32_t* out_dev) {
  B2S_CUDA(cudaMemsetAsync(out_dev, 0, 4, h->stream));
  if (sm->dense_cap == 0) return B2S_OK;
  launch_pdl(dense_count_kernel, 4 * device_sms(), 256, 0, h->stream, sm->dense_cnt.as<int32_t>(), sm->dense_cap, out_dev);
  h->launches++;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

// =====================================================================================================================
//  C2  space carving of the dense map: Submap::carve(scan, sensorPosition, param, VoxelizedPointCloud*)
//      core/src/Submap.cpp:125-136 -> removeDuplicatePointsWithinSameVoxels (core/src/Voxel.cpp:162-192),
//      getKeysOfCarvedPoints (core/src/helpers.cpp:347-377), getVoxelsWithinPointNeighborhood (core/src/VoxelHashMap.cpp:13-45)
//  (1) first point of every voxel of the scan = the ray set (atomicMin of the index per voxel of a scratch hash);
//  (2) one thread per ray: steps of 2*radius, at every step the reference's dx/dy/dz loops (floating accumulation kept as
//      written) enumerate test points; a test point within `radius` of its voxel centre nominates that voxel; nominated
//      voxels that exist in the dense map are flagged; (3) flagged voxels are emptied (removeKey).
// =====================================================================================================================
__device__ __forceinline__ long long dense_find_key(const unsigned long long* __restrict__ keys, size_t cap, int kx, int ky, int kz) {
  if (!(abs(kx) < 1048575 && abs(ky) < 1048575 && abs(kz) < 1048575)) return -1;   // voxel_key_of's key limit
  return voxel_key_find(keys, cap - 1, voxel_key_pack(kx, ky, kz));
}

// The ray set is keyed with the full int32 range of the reference's Eigen::Vector3i, not the 21-bit fields of the map: a
// return 2^20 voxels out still casts a ray through the voxels near the sensor.  A key is three int32 in 16 bytes (z = ~0: empty
// slot) claimed by one 128-bit compare-and-swap; its home slot is the dense map's hash of the key's low 21 bits per axis, which is
// the dense map's own home slot wherever the map can key a point.
struct alignas(16) RayKey { unsigned long long xy, z; };
constexpr unsigned long long RAY_EMPTY = ~0ull;
// (int32_t)floor(v) as the reference computes it on x86-64 (cvttsd2si): NaN and values outside int32 become INT32_MIN
__device__ __forceinline__ int ray_i32(double f) { return (f >= -2147483648.0 && f < 2147483648.0) ? (int)f : INT32_MIN; }
__device__ __forceinline__ unsigned long long ray_home(int x, int y, int z) {
  const unsigned long long m = 0x1FFFFF;
  return voxel_key_hash(((((unsigned)x + 1048576u) & m) << 42) | ((((unsigned)y + 1048576u) & m) << 21) | (((unsigned)z + 1048576u) & m));
}

__global__ void __launch_bounds__(FZ_THREADS) dcarve_first_kernel(const double* __restrict__ xyz, const int32_t* __restrict__ d_n, double inv,
                                                                  RayKey* keys, int32_t* first, size_t mask,
                                                                  int32_t* __restrict__ slot_of, const int32_t* __restrict__ enable) {
  pdl_wait();
  if (enable != nullptr && *enable == 0) return;
  const int n = *d_n;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int kx = ray_i32(floor(__dmul_rn(xyz[3 * i], inv))), ky = ray_i32(floor(__dmul_rn(xyz[3 * i + 1], inv))),
              kz = ray_i32(floor(__dmul_rn(xyz[3 * i + 2], inv)));
    slot_of[i] = -1;
    const RayKey key{((unsigned long long)(unsigned)kx << 32) | (unsigned)ky, (unsigned long long)(unsigned)kz};
    const RayKey empty{RAY_EMPTY, RAY_EMPTY};
    size_t s = (size_t)ray_home(kx, ky, kz) & mask;
    for (size_t probe = 0; probe <= mask; ++probe, s = (s + 1) & mask) {
      const RayKey old = atomicCAS(&keys[s], empty, key);
      if (old.z == RAY_EMPTY || (old.xy == key.xy && old.z == key.z)) { atomicMin(&first[s], i); slot_of[i] = (int32_t)s; break; }
    }
  }
}

__global__ void dcarve_init_kernel(RayKey* keys, int32_t* first, size_t cap, int32_t* rm, size_t dense_cap,
                                   const int32_t* __restrict__ enable, int32_t* removed) {
  pdl_wait();
  if (blockIdx.x == 0 && threadIdx.x == 0 && removed) *removed = 0;
  if (enable != nullptr && *enable == 0) return;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < cap; i += (size_t)gridDim.x * blockDim.x) { keys[i] = RayKey{RAY_EMPTY, RAY_EMPTY}; first[i] = 0x7fffffff; }
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < dense_cap; i += (size_t)gridDim.x * blockDim.x) rm[i] = 0;
}

__global__ void __launch_bounds__(FZ_THREADS) dcarve_march_kernel(const double* __restrict__ xyz, const int32_t* __restrict__ d_n,
                                                                  const int32_t* __restrict__ slot_of, const int32_t* __restrict__ first,
                                                                  double sx, double sy, double sz, const double* __restrict__ sensor_dev,
                                                                  double voxel, double radius, double trunc,
                                                                  double max_len, const unsigned long long* __restrict__ dkeys,
                                                                  const int32_t* __restrict__ dcnt, size_t dcap, int32_t* __restrict__ rm,
                                                                  const int32_t* __restrict__ enable) {
  pdl_wait();
  if (enable != nullptr && *enable == 0) return;
  if (sensor_dev) { sx = sensor_dev[3]; sy = sensor_dev[7]; sz = sensor_dev[11]; }   // mapToRangeSensor.translation()
  const int n = *d_n;
  const double step = 2.0 * radius;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int so = slot_of[i];
    if (so < 0 || first[so] != i) continue;       // removeDuplicatePointsWithinSameVoxels keeps the first point of a voxel
    const double dx = xyz[3 * i] - sx, dy = xyz[3 * i + 1] - sy, dz = xyz[3 * i + 2] - sz;
    const double length = sqrt(dx * dx + dy * dy + dz * dz);
    const double ux = dx / length, uy = dy / length, uz = dz / length;
    double mp = length - trunc;
    if (max_len < mp) mp = max_len;
    if (step > mp) mp = step;
    if (!(mp == mp)) continue;
    double distance = 0.0;
    while (distance < mp) {
      const double cx = distance * ux + sx, cy = distance * uy + sy, cz = distance * uz + sz;
      const int ckx = (int)floor(cx / voxel), cky = (int)floor(cy / voxel), ckz = (int)floor(cz / voxel);
      bool center_added = false;
      if (radius > 0.0) {
        for (double ox = -radius; ox <= radius; ox += voxel)
          for (double oy = -radius; oy <= radius; oy += voxel)
            for (double oz = -radius; oz <= radius; oz += voxel) {
              const double tx = cx + ox, ty = cy + oy, tz = cz + oz;
              const int kx = (int)floor(tx / voxel), ky = (int)floor(ty / voxel), kz = (int)floor(tz / voxel);
              const double ex = tx - ((double)kx * voxel + voxel * 0.5), ey = ty - ((double)ky * voxel + voxel * 0.5),
                           ez = tz - ((double)kz * voxel + voxel * 0.5);
              if (sqrt(ex * ex + ey * ey + ez * ez) <= radius) {
                const long long s = dense_find_key(dkeys, dcap, kx, ky, kz);
                if (s >= 0 && dcnt[s] > 0) rm[s] = 1;
                if (kx == ckx && ky == cky && kz == ckz) center_added = true;
              }
            }
      }
      if (!center_added) {
        const long long s = dense_find_key(dkeys, dcap, ckx, cky, ckz);
        if (s >= 0 && dcnt[s] > 0) rm[s] = 1;
      }
      distance += step;
    }
  }
}

__global__ void dcarve_apply_kernel(const int32_t* __restrict__ rm, size_t cap, double* __restrict__ sums, int32_t* __restrict__ cnts, int32_t* removed,
                                    const int32_t* __restrict__ enable, int32_t* mstate) {
  pdl_wait();
  if (enable != nullptr && *enable == 0) return;
  if (mstate && blockIdx.x == 0 && threadIdx.x == 0) mstate[MS_NDCARVE] += 1;
  int c = 0;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < cap; i += (size_t)gridDim.x * blockDim.x) {
    if (!rm[i]) continue;
    cnts[i] = 0;
    for (int k = 0; k < 6; k++) sums[6 * i + k] = 0.0;
    c++;
  }
  c = warp_sum_i(c);
  if ((threadIdx.x & 31) == 0 && c) { atomicAdd(removed, c); if (mstate) atomicAdd(&mstate[MS_DCARVED], c); }
}

int32_t op_dense_carve(b2s_handle* h, b2s_submap* sm, const b2s_cloud* scan, const double* sensor, const double* sensor_dev, double radius,
                       double trunc, double max_len, int32_t* removed_dev, const int32_t* enable_dev) {
  B2S_REQUIRE(sm->dense_cap > 0, B2S_E_INVALID, "dense map not initialised");
  const size_t n_max = scan->n_max > 0 ? scan->n_max : 1;
  size_t cap = 1024;
  while (cap < 2 * n_max) cap <<= 1;
  B2S_TRY(h->keys.ensure(cap * sizeof(RayKey), h->stream));
  B2S_TRY(h->vals.ensure(cap * 4, h->stream));
  B2S_TRY(h->tmp_i32.ensure((n_max + 64) * 4, h->stream));
  B2S_TRY(h->offs.ensure((sm->dense_cap + 2) * 4, h->stream));   // removal flags per dense slot
  RayKey* keys = h->keys.as<RayKey>();
  int32_t* first = h->vals.as<int32_t>();
  int32_t* slot_of = h->tmp_i32.as<int32_t>();
  int32_t* rm = h->offs.as<int32_t>();
  const double voxel = sm->dense_voxel;
  const double s0 = sensor ? sensor[0] : 0.0, s1 = sensor ? sensor[1] : 0.0, s2 = sensor ? sensor[2] : 0.0;
  ProfScope prof(h, PK_FUSE);
  launch_pdl(dcarve_init_kernel, 8 * device_sms(), 256, 0, h->stream, keys, first, cap, rm, sm->dense_cap, enable_dev, removed_dev);
  launch_pdl(dcarve_first_kernel, grid_for(n_max, FZ_THREADS), FZ_THREADS, 0, h->stream, scan->xyz.as<double>(), scan->dn.as<int32_t>(), 1.0 / voxel, keys, first,
                                                                                cap - 1, slot_of, enable_dev);
  launch_pdl(dcarve_march_kernel, grid_for(n_max, FZ_THREADS), FZ_THREADS, 0, h->stream, scan->xyz.as<double>(), scan->dn.as<int32_t>(), slot_of, first, s0, s1, s2,
                                                                                sensor_dev, voxel, radius, trunc, max_len,
                                                                                sm->dense_keys.as<unsigned long long>(), sm->dense_cnt.as<int32_t>(),
                                                                                sm->dense_cap, rm, enable_dev);
  launch_pdl(dcarve_apply_kernel, 8 * device_sms(), 256, 0, h->stream, rm, sm->dense_cap, sm->dense_sum.as<double>(), sm->dense_cnt.as<int32_t>(), removed_dev, enable_dev,
                                                      sm->mstate.as<int32_t>());
  h->launches += 4;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

}  // namespace b2s
