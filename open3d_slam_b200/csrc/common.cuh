// common.cuh -- shared device helpers and the host-side runtime types of the b2s engine (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <memory>
#include <mutex>
#include <unordered_set>
#include <new>
#include <string>
#include <utility>
#include <vector>

#include "../../include/b2s.h"

namespace b2s {

// ------------------------------------------------------------------------------------------------
// error plumbing: no exception crosses the C ABI; the message is kept per host thread
// ------------------------------------------------------------------------------------------------
void set_error(const char* fmt, ...);
const char* get_error();

#define B2S_CUDA(expr)                                                                            \
  do {                                                                                            \
    cudaError_t _e = (expr);                                                                      \
    if (_e != cudaSuccess) {                                                                      \
      ::b2s::set_error("CUDA error %s at %s:%d: %s", cudaGetErrorName(_e), __FILE__, __LINE__, cudaGetErrorString(_e)); \
      return B2S_E_CUDA;                                                                          \
    }                                                                                             \
  } while (0)

#define B2S_TRY(expr)              \
  do {                             \
    int32_t _s = (expr);           \
    if (_s != B2S_OK) return _s;   \
  } while (0)

#define B2S_REQUIRE(cond, code, ...)     \
  do {                                   \
    if (!(cond)) {                       \
      ::b2s::set_error(__VA_ARGS__);     \
      return (code);                     \
    }                                    \
  } while (0)

// ------------------------------------------------------------------------------------------------
// owning buffers: the destructor frees the allocation, so an object holding them needs no release code.  They are move-only
// (declaring the move operations deletes the copies): a moved-from buffer takes over what the target held and frees it.
// ------------------------------------------------------------------------------------------------
struct DevBuf {          // grow-only device buffer
  void* p = nullptr;
  size_t cap = 0;
  bool tracked = true;   // a re-allocation invalidates captured graphs (false for clouds the caller owns: a graph never holds them)
  DevBuf() = default;
  DevBuf(DevBuf&& o) noexcept { *this = std::move(o); }
  DevBuf& operator=(DevBuf&& o) noexcept { std::swap(p, o.p); std::swap(cap, o.cap); std::swap(tracked, o.tracked); return *this; }
  ~DevBuf() { release(); }
  int32_t ensure(size_t bytes, cudaStream_t s, bool preserve = false);
  void release();
  template <typename T>
  T* as() const { return reinterpret_cast<T*>(p); }
};

struct PinnedBuf {       // page-locked host memory (cudaHostAlloc)
  void* p = nullptr;
  size_t cap = 0;
  PinnedBuf() = default;
  PinnedBuf(PinnedBuf&& o) noexcept { *this = std::move(o); }
  PinnedBuf& operator=(PinnedBuf&& o) noexcept { std::swap(p, o.p); std::swap(cap, o.cap); return *this; }
  ~PinnedBuf() { release(); }
  int32_t alloc(size_t bytes, unsigned flags = cudaHostAllocDefault);   // frees what it held first: nothing may still use that
  void release() { if (p) cudaFreeHost(p); p = nullptr; cap = 0; }
  template <typename T>
  T* as() const { return reinterpret_cast<T*>(p); }
};

// Builds a new T with init(T*) and hands it out through *out only when init succeeded; a half-built T is deleted (its members free
// what they own), so a failed create leaves nothing behind.
template <typename T, typename Init>
int32_t create_object(T** out, Init&& init) {
  T* obj = new (std::nothrow) T();
  B2S_REQUIRE(obj, B2S_E_INVALID, "out of host memory");
  const int32_t rc = init(obj);
  if (rc != B2S_OK) { delete obj; return rc; }
  *out = obj;
  return B2S_OK;
}
// Deletes an object a b2s_*_create made.  The owning handle may already be gone: wait for the whole device instead of touching it.
template <typename T>
void destroy_object(T* obj) {
  if (!obj) return;
  cudaSetDevice(obj->device);
  cudaDeviceSynchronize();
  delete obj;
}

// device-side status word: kernels OR error bits into it, the host checks it when it synchronises
enum : uint32_t { ST_KEY_OVERFLOW = 1u, ST_CAPACITY = 2u, ST_EMPTY = 4u, ST_HASH_FULL = 8u };

struct GridHeader {      // one per nearest-neighbour grid, lives in device memory; searched through the helpers after dist2_exact
  double origin[3];
  double cell, inv_cell;
  int32_t dims[3];
  int32_t ncell;
  int32_t n;             // points indexed
  int32_t pad;
};

// dense-grid nearest-neighbour index over a point set (K-index): points counting-sorted by cell
struct GridIndex {
  DevBuf hdr;            // GridHeader
  DevBuf bbox;           // 6 x uint64 ordered-double min/max
  DevBuf cell_start;     // int32 [cap_cells + 1]
  DevBuf rank;           // int32 per point: rank within its cell (-1 = not indexed)
  DevBuf pts;            // double4 per indexed point: x,y,z, bits(original index); normals are read from the cloud through it
  int32_t cap_cells = 0;
};

struct ScanScratch {     // decoupled look-back scan state
  DevBuf state;          // uint64 per tile + int32 tile counter
  int32_t cap_tiles = 0;
};

struct ScanJob {         // one array of a batched scan (scan_exclusive_i32_batch)
  const int32_t* in; int32_t* out; const int32_t* d_n; unsigned long long* state; int32_t* counter;
};

struct SortScratch {
  DevBuf hist;           // 256 x nblocks int32
  DevBuf keys_alt, vals_alt;
};

// process-wide registry of the submaps alive (by b2s_submap::uid): caches of graphs captured for a submap elsewhere drop the entries of
// submaps that are gone
void submap_register(unsigned long long uid);
void submap_forget(unsigned long long uid);
bool submap_alive(unsigned long long uid);

// A captured per-scan chain (CUDA graph) and what it was captured under.  Its launches bake in buffer addresses, the handle's
// configuration and the owner's options (key): once one of them changes the graph is destroyed, the next step runs eagerly and
// the one after re-captures.
struct GraphCache {
  cudaGraphExec_t exec = nullptr;
  int warm = 2;                       // eager steps still to run before the capture (sizes every scratch buffer)
  int64_t kernels = 0;                // kernels per replay (for the launch counter)
  unsigned long long alloc_gen = 0;   // value of b2s::g_alloc_generation when the graph was captured
  unsigned long long cfg_gen = 0;     // value of b2s_handle::cfg_gen when the graph was captured
  unsigned long long key = 0;         // the owner's options generation when the graph was captured
  GraphCache() = default;
  GraphCache(const GraphCache&) = delete;
  GraphCache& operator=(const GraphCache&) = delete;
  ~GraphCache() { if (exec) cudaGraphExecDestroy(exec); }
};

}  // namespace b2s

struct b2s_cloud {
  b2s_handle* h = nullptr;
  int device = 0;
  b2s::DevBuf xyz;       // 3 x f64 per point (the reference's AoS layout)
  b2s::DevBuf nrm;       // 3 x f64 per point
  b2s::DevBuf dn;        // int32 device-side point count
  size_t n_max = 0;      // host-side upper bound of the count (launch sizing)
  size_t fixed_cap = 0;  // non-zero: n_max is pinned to this capacity (graph replay needs constant launch dimensions)
  long long n_known = 0; // exact count when the host knows it, -1 otherwise
  bool has_normals = false;
};

struct b2s_submap {
  ~b2s_submap() { if (cnt_ev) cudaEventDestroy(cnt_ev); if (uid) b2s::submap_forget(uid); }   // the buffers, clouds and the graph free themselves
  b2s_handle* h = nullptr;
  int device = 0;
  unsigned long long uid = 0;         // unique over the process: graphs captured for this submap elsewhere are keyed by it
  std::unique_ptr<b2s_cloud> cloud[2];  // ping-pong map cloud (mapCloud_)
  int cur = 0;
  size_t capacity = 0;
  // dense map (VoxelizedPointCloud): open-addressing hash of running sums
  b2s::DevBuf dense_keys;    // uint64 packed key, EMPTY = ~0
  b2s::DevBuf dense_sum;     // 6 x f64 per slot
  b2s::DevBuf dense_cnt;     // int32 per slot
  b2s::DevBuf dense_used;    // int32 occupied-slot counter
  size_t dense_cap = 0;
  double dense_voxel = 0.0;
  bool dense_has_normals = false;
  b2s::DevBuf pose;          // 4 x (4x4 f64): [0] mapToRangeSensor_ state, [1] insertion pose, [2] odometry motion, [3] initial guess
  // asynchronous read-back of the map size (keeps the host-side launch bound tight without ever synchronising)
  b2s::PinnedBuf pinned_cnt;          // int32 map size, written by the copy cnt_ev marks
  cudaEvent_t cnt_ev = nullptr;
  bool cnt_pending = false;
  size_t adds_after_readback = 0;
  // CUDA-graph replay of the per-scan chain (b2s_mapper_graph_enable): every launch dimension is derived from fixed
  // capacities, the per-step inputs (odometry motion, result slot) come from a ring indexed by a device-side counter
  bool graph_mode = false;
  bool fixed_launch = false;           // a captured chain runs on this submap (either graph mode): launch dimensions from the capacity, no host read-backs
  b2s::GraphCache graph;
  std::unique_ptr<b2s_cloud> staging; // fixed-capacity input cloud the caller uploads each scan into
  b2s::PinnedBuf odom_ring;           // device-mapped: 64 x (4x4 f64) odometry motions
  long long host_step = 0;
  b2s::DevBuf gstate;                 // int32 [0] device step counter, [1] current result slot
  double g_min_fitness = 0.0;
  int g_ignore_fitness = 0;
  // persistent voxel hash of the map cloud (K-fuse, fuse.cu): map-voxel key -> chain of the map points inside that voxel
  b2s::DevBuf vkeys;         // uint64 [vcap] packed voxel key, EMPTY = ~0
  b2s::DevBuf vhead;         // int32 [vcap] first member of the voxel's chain (-1 = none); members >= FUSE_STAGE_BASE are staged scan points
  b2s::DevBuf vstamp;        // int32 [vcap] stamp of the last insertion that touched the voxel
  b2s::DevBuf vnext;         // int32 [capacity] chain link of every map point
  b2s::DevBuf pstamp;        // int32 [capacity] stamp of the insertion that last rewrote the point
  b2s::DevBuf stage_xyz, stage_nrm, stage_next, stage_in;   // the transformed scan of the insertion in flight
  b2s::DevBuf touched;       // int32 voxels (table slots) the insertion in flight touched
  b2s::DevBuf dups;          // int32 [2][FUSE_DUP_CAP] voxels holding more than one map point (ping-pong)
  b2s::DevBuf wflag;         // int32 [capacity + 1] 1 = the slot is on K3's renormalisation worklist
  b2s::DevBuf wlist;         // int32 [2][capacity + 1] the worklist (ping-pong): slots whose normal may not be a fixed point yet
  // uint64 [6] bounding box of the live map slots, ord_encode'd min xyz / max xyz like GridIndex::bbox.  It may hold more than the live
  // slots, never less: K2 folds in every position it writes into a slot, fuse_rehash recomputes it exactly.  The map-index build takes
  // its grid box from it (grid_build) instead of reading the whole map for one.
  b2s::DevBuf bbox;
  size_t vcap = 0;
  size_t stage_cap = 0;
  // Mapper / SubmapCollection wiring of the device chain (b2s_mapper_options) and its device-side state words (MS_*)
  b2s_mapper_options opts;
  unsigned long long opts_gen = 1;    // bumped by b2s_submap_set_mapper_options: graphs of other objects that run this chain compare it
  b2s::DevBuf mstate;                 // int32 [MS_WORDS]: gates and counters of the chain, see the MS_* indices below
  // MapperParameters::isMergeScansIntoMap_ as the chain sees it (b2s_submap_set_merge_scans): off = pure localisation, the chain
  // neither carves nor fuses (Mapper.cpp:163-167); part of the captured chain, so switching drops the graph like the options do
  bool merge_scans = true;
  // static map patch (grid_index.cu): while merge_scans is off the sparse map cannot change, so its slots are kept counting-sorted by a
  // coarse tile cell (a GridIndex built with the tile edge and no cropper) and every registration gathers its patch from the tiles the
  // cropper's box touches.  Built by the first registration after merge goes off; dropped by every call that writes the map.
  b2s::GridIndex tile;
  bool tile_valid = false;
  std::unique_ptr<b2s_cloud> patch;   // the gathered patch points (sized like the map, so the NN grid gets the full path's cell budget) ...
  b2s::DevBuf patch_idx;              // ... and each one's map slot, the original index the NN grid stores
  // the map has no normals (stored as NaN): loaded without them, or fed a scan without them.  [O3D] PointCloud::operator+= drops a
  // cloud's normals as soon as one part lacks them, so the reference's map stays without normals from then on, and so does this flag
  bool no_normals = false;
};

namespace b2s {
// Scratch of the operators that work on the whole map (b2s_assemble_map, b2s_assemble_dense_maps, assemble.cu).  Every buffer is sized to the assembled map and
// grows with it, so none is tracked: no captured chain reads them, and their growth must not make the mapper chains re-capture.
struct VoxelScratch {    // op_voxel_down_sample's own scratch instead of the handle's keys / vals / flags / offs, scan state and sort histogram
  DevBuf keys, vals, flags, offs, scan_state, sort_hist;
  VoxelScratch() { for (DevBuf* b : {&keys, &vals, &flags, &offs, &scan_state, &sort_hist}) b->tracked = false; }
};
struct AssemblyScratch {
  DevBuf tables;         // AsmJob / DenseTable + ScanJob tables, the per-job base offsets and the palette
  DevBuf slots;          // per map slot of every job: live flag, offset within the submap (A1); per dense-table tile: live voxels,
                         // their offset within the table (A2); the batched scan's tile states
  DevBuf labels;         // int32 per assembled point: palette entry (coloured call, voxel path)
  DevBuf rgb;            // 3 x f64 per output point (coloured call)
  PinnedBuf stage;       // page-locked staging of the tables
  b2s_cloud cloud;       // the assembled map in front of the voxel path
  VoxelScratch vox;
  DevBuf blob;           // A3 (state.cu): the exported blobs, laid out as on the host / the blob being imported
  AssemblyScratch() {
    for (DevBuf* b : {&tables, &slots, &labels, &rgb, &cloud.xyz, &cloud.nrm, &cloud.dn, &blob}) b->tracked = false;
  }
};
}  // namespace b2s

struct b2s_feature {
  b2s_handle* h = nullptr;
  int device = 0;
  b2s::DevBuf data;      // B2S_FEATURE_DIM x f64 per point, point after point ([O3D] Feature::data_, a column-major dim x n matrix)
  size_t n = 0;
  b2s::DevBuf nb_idx, nb_d2, nb_cnt, spfh;   // scratch of b2s_compute_fpfh: neighbour lists (knn per point) and the SPFH rows
};

namespace b2s {
// device-side state words of the mapper chain (b2s_submap::mstate)
enum MapperStateWord {
  MS_ACCEPT = 0,      // this step passed the fitness gate (Mapper.cpp:151)
  MS_INSERT = 1,      // ... and the minimum-motion gate (Mapper.cpp:170-176): F1 runs
  MS_CARVE = 2,       // sparse-map carving runs in this step (Submap.cpp:111)
  MS_DENSE = 3,       // dense-map insertion runs in this step
  MS_DCARVE = 4,      // dense-map carving runs in this step (Submap.cpp:127)
  MS_NINS = 5,        // Submap::nScansInsertedMap_
  MS_NDENSE = 6,      // Submap::nScansInsertedDenseMap_
  MS_NSTEPS = 7, MS_NACCEPT = 8, MS_NCARVE = 9, MS_CARVED = 10, MS_NDCARVE = 11, MS_DCARVED = 12,
  MS_CARVE_N = 13,    // point count the carving compaction works on (0 when carving is skipped)
  MS_TMP = 14,        // [14] grid-wide ticket, [15] dense-carve removed count
  MS_NDEAD = 16,      // tombstones among the map slots (points merged away; xyz = NaN) -- the map holds dn - NDEAD points
  MS_STAMP = 17,      // stamp of the last committed insertion
  MS_NTOUCHED = 18,   // voxels touched by the insertion in flight
  MS_DUPSEL = 19,     // which half of `dups` is current
  MS_NDUP = 20,       // [20], [21]: entries of the two halves
  MS_VUSED = 22,      // occupied slots of the voxel table
  MS_TICKET2 = 23,
  MS_WSEL = 24,       // which half of `wlist` is current
  MS_NW = 25,         // [25], [26]: entries of the two halves
  MS_NEWINIT = 27,    // Mapper::isNewInitialValueSet_: set by b2s_submap_set_initial_transform, cleared by the next step (Mapper.cpp:87-91,143-149)
  MS_IGNODOM = 28,    // Mapper::isIgnoreOdometryPrediction_: the step after a new initial value predicts without odometry (Mapper.cpp:130-138)
  MS_INITSTEP = 29,   // this step was the first after a new initial value: ICP result discarded, lastMeasurementTimestamp_ kept
  MS_WORDS = 32
};
// bumped by every DevBuf re-allocation: a captured graph holds raw pointers of the scratch buffers, so a graph captured
// under an older generation is re-captured before it is replayed again
extern unsigned long long g_alloc_generation;
// per-kernel-group device timing with CUDA events on the launching stream (bench.py's roofline numbers)
enum ProfKind { PK_ICP = 0, PK_NORMALS, PK_SORT, PK_GRID, PK_VOXEL, PK_FUSE, PK_SELECT, PK_CROP, PK_COUNT };
struct ProfRec { int kind; cudaEvent_t a, b; };
}  // namespace b2s

namespace b2s {
// set while this host thread is inside cudaStreamBeginCapture/EndCapture: growing a device buffer is impossible there
extern thread_local bool g_capturing;
extern thread_local bool g_capture_broken;
}  // namespace b2s

struct b2s_handle {
  ~b2s_handle() {   // the buffers and clouds free themselves
    for (auto& r : prof_recs) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
    for (cudaEvent_t e : prof_pool) cudaEventDestroy(e);
    if (own_stream && stream) cudaStreamDestroy(stream);
  }
  bool prof_enabled = false;
  b2s::DevBuf icp_dbg;                // optional clock64 stamps (b2s_debug_icp_clocks); unallocated while they are off
  std::vector<b2s::ProfRec> prof_recs;
  std::vector<cudaEvent_t> prof_pool;
  int device = 0;
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  std::recursive_mutex mu;            // recursive: the composite host entry points hold it across the calls they chain
  b2s_config cfg;
  unsigned long long cfg_gen = 1;     // bumped by b2s_set_config: captured graphs bake the configuration in
  int64_t launches = 0;
  int64_t captures = 0;               // CUDA graphs captured by this handle's per-scan chains (b2s_graph_capture_count)

  b2s::DevBuf status;                 // uint32 [16]: [0] device status word, the rest scratch words (b2s::SW_*)
  b2s::ScanScratch scan;
  b2s::SortScratch sort;
  b2s::GridIndex grid_a, grid_b;      // target index (ICP) / self index (normals)
  // generic scratch buffers, by role
  b2s::DevBuf keys, vals, flags, offs, tmp_i32, tmp_f64, misc, work_xyz;
  b2s::DevBuf problems;               // IcpProblem array (device)
  b2s::DevBuf results;                // b2s_result array (device)
  b2s::DevBuf slots;                  // per-slot results for the async mapper step
  b2s::DevBuf poses;                  // 64 small device-resident transforms (4x4 f64, all allocated by b2s_create); scratch slots b2s::PS_*
  b2s::PinnedBuf pinned;              // host staging of check_status and read_back (runtime.cu owns its layout)
  // temporaries for the fused chains
  std::unique_ptr<b2s_cloud> t0, t1, t2, t3;
  std::vector<std::unique_ptr<b2s::GridIndex>> batch_grids;
  b2s::DevBuf batch_jobs;             // GridJob + ScanJob tables and the scan tile states of a batched index build
  std::vector<unsigned char> batch_jobs_host;
  b2s::DevBuf lc;                     // K-ransac scratch (ransac.cu owns its layout)
  // b2s_submap_odometry_constraints (constraints.cu): the batched overlap's tables and per-slot arrays, K-info-wide's tables / tile
  // partials / records, their page-locked staging, and the overlap clouds used when the caller passes none
  b2s::DevBuf odo, odo_info;
  b2s::PinnedBuf odo_stage;
  std::vector<std::unique_ptr<b2s_cloud>> odo_clouds;
  // b2s_global_optimization (posegraph.cu owns the layouts): the dense system H and the factor of H + lambda I (padded to whole
  // tiles), the panel, the vectors and try records, the node poses and trial poses, the edge records with their per-edge scratch
  // and assembly lists, and the CUDA graph of one LM try
  b2s::DevBuf pg_A, pg_F, pg_W, pg_vec, pg_nodes, pg_edges;
  int32_t pg_edge_cap = 0;
  b2s::GraphCache pg_graph;
  b2s::AssemblyScratch assembly;      // b2s_assemble_map / _colored_map / _dense_maps (assemble.cu owns the layouts)
};

// every entry point that touches a handle's stream or buffers holds its lock and works on its device
#define LOCK(h) std::lock_guard<std::recursive_mutex> _lk((h)->mu); cudaSetDevice((h)->device)

namespace b2s {

// extra words of b2s_handle::status (uint32): removed count of b2s_submap_carve / b2s_dense_carve, voxel count of b2s_dense_size,
// point count of the chunk b2s_nearest_neighbors works on
enum StatusWord : int { SW_REMOVED = 8, SW_DENSE_SIZE = 12, SW_NN_CHUNK = 14 };
// scratch slots of b2s_handle::poses: T of b2s_voxel_map_has_voxel; sourceToTarget of b2s_overlap and the host-given pose of
// op_dense_insert (shared: each call writes the slot before its kernels read it, on the handle's stream); T of op_transform
enum PoseSlot : int { PS_VOXEL_MAP = 61, PS_CALL = 62, PS_TRANSFORM = 63 };

struct ProfScope {   // records an event pair around the launches issued during its lifetime (no-op unless enabled)
  b2s_handle* h; int idx;
  ProfScope(b2s_handle* h_, int kind);
  ~ProfScope();
};
int32_t check_status(b2s_handle* h);     // synchronises and converts device status bits into an error
struct ReadBack { void* dst; const void* src; size_t bytes; };   // host destination, device source
// small device -> host reads through pinned staging, then check_status; the destinations are written even when the device status
// reports an error, and check_status's code is returned
int32_t read_back(b2s_handle* h, std::initializer_list<ReadBack> copies);

// The scratch layout of a batched call: regions in the order they are taken, each rounded up to 256 bytes.  The same layout code runs
// twice, first on a Layout without a base, which only adds up `size`, then on one with the buffer's base, which places every region where
// the first pass counted it, so the two cannot disagree.  off() hands out a region's offset, so that a table can be written at that offset
// in a host stage and read at it in the device buffer; take() hands out base + offset (nullptr while measuring).
struct Layout {
  unsigned char* base = nullptr;
  size_t size = 0;
  size_t off(size_t bytes) { const size_t o = size; size += (bytes + 255) & ~(size_t)255; return o; }
  template <typename T>
  T* take(size_t count) { const size_t o = off(count * sizeof(T)); return base ? reinterpret_cast<T*>(base + o) : nullptr; }
};
// runs place(L) on a measuring Layout, ensures buf to the size it counted, then runs place(L) again on buf's base
template <typename F>
int32_t carve(DevBuf& buf, cudaStream_t s, F&& place) {
  Layout L;
  place(L);
  B2S_TRY(buf.ensure(L.size, s));
  L = Layout{buf.as<unsigned char>()};
  place(L);
  return B2S_OK;
}

// ---- primitives (scan.cu / radix_sort.cu / grid_index.cu / ...) : all asynchronous on h->stream ----
// exclusive scan of in[0..*d_n) into out[0..*d_n]; out[*d_n] and *d_total (optional) receive the total.  state (optional): the tile
// state buffer to use instead of the handle's
int32_t scan_exclusive_i32(b2s_handle* h, const int32_t* in, int32_t* out, const int32_t* d_n, size_t n_max, int32_t* d_total,
                           DevBuf* state = nullptr);
// njobs independent scans in one launch.  Every job's tile state comes from scan_bind_state with the same n_max and is zeroed before
// the scan: it takes the state from L and points j.state / j.counter into it (the measuring pass only counts).  A caller binds every
// job's state before its other regions, so that the states are one range that one memset clears.
void scan_bind_state(Layout& L, ScanJob& j, size_t n_max);
int32_t scan_exclusive_i32_batch(b2s_handle* h, const ScanJob* jobs_dev, int njobs, size_t n_max);
// stable LSD radix sort of (key, value) pairs, key_bits low bits significant; result ends in keys/vals
// (pointers are swapped so that keys/vals designate the sorted arrays on return, *_alt the scratch).  own (optional): the histogram and
// scan state of the multi-kernel sort come from it instead of the handle
int32_t radix_sort_pairs_u32(b2s_handle* h, uint32_t*& keys, uint32_t*& vals, uint32_t*& keys_alt, uint32_t*& vals_alt,
                             const int32_t* d_n, size_t n_max, int key_bits, VoxelScratch* own = nullptr);
int32_t radix_sort_pairs_u64(b2s_handle* h, uint64_t*& keys, uint32_t*& vals, uint64_t*& keys_alt, uint32_t*& vals_alt,
                             const int32_t* d_n, size_t n_max, int key_bits, VoxelScratch* own = nullptr);
inline const int32_t* grid_starts(const GridIndex* g) { return g->cell_start.as<int32_t>() + g->cap_cells + 4; }

// K-index: build the NN grid over cloud points (optionally only those inside `patch`, centre read from device pose)
struct CropDev {      // cropper passed by value to kernels; centre may come from a device-resident 4x4 (row-major)
  int32_t kind, invert;
  double rmin, rmax, zmin, zmax;
  double cx, cy, cz;
  const double* pose_dev;   // if non-null the centre is (pose[3], pose[7], pose[11])
};
CropDev make_crop(const b2s_cropper* c, const double* pose_dev = nullptr);
// orig (optional): per point of cloud the original index the grid stores (default: the point's own index).
// map_box, map_crop (optional, together): a box holding every point of cloud (b2s_submap::bbox) and the cropper of the patch.  The grid
// box is then map_box cut to map_crop's axis-aligned box, with no pass over the cloud for it.  B2S_GRID_BBOX_PASS=1 ignores them (A/B
// switch and test reference).
int32_t grid_build(b2s_handle* h, GridIndex* g, const b2s_cloud* cloud, double cell, const CropDev* patch, const int32_t* orig = nullptr,
                   const unsigned long long* map_box = nullptr, const CropDev* map_crop = nullptr);
// sets the six words of an ord_encode'd box (min xyz, max xyz) to the empty box
int32_t box_reset(b2s_handle* h, unsigned long long* box);
// static map patch (grid_index.cu): true when sm's merge is off, the cropper is bounded and B2S_PATCH_FULL is not set
bool tile_patch_usable(const b2s_submap* sm, const CropDev& crop);
// builds the tile table if it is not valid, gathers the tiles the cropper touches, and builds g over the gathered points that pass
// crop_within, each keeping its map slot as original index: the same indexed set, grid header and original indices as
// grid_build(map, cell, &crop)
int32_t tile_patch_build(b2s_handle* h, b2s_submap* sm, const CropDev& crop, double cell, GridIndex* g);
// every call that writes a submap's map drops its tile table (and the captured chains that read it)
int32_t tile_drop(b2s_handle* h, b2s_submap* sm);
constexpr double TILE_EDGE = 2.0;        // tile edge of the static patch table (m)
constexpr int TILE_MARGIN = 1;           // tiles added on every side of the cropper's box: rounding of the box and of crop_within
// the same for n clouds at once (batched registration: every pair brings its own target), blockIdx.y = cloud
int32_t grid_build_batch(b2s_handle* h, GridIndex* const* g, const b2s_cloud* const* clouds, int n, double cell);

int32_t pose_to_device(b2s_handle* h, const double* T, double* dst);   // host 4x4 -> device slot, no staging buffer (voxel.cu)
int32_t cloud_reserve(b2s_handle* h, b2s_cloud* c, size_t n, bool normals);
int32_t cloud_set_count(b2s_handle* h, b2s_cloud* c, size_t n);

// stages
int32_t op_crop(b2s_handle* h, const b2s_cloud* in, const CropDev& crop, b2s_cloud* out);
// fixed_key_bits > 0: key width per axis given by the caller instead of measured (no synchronisation); a voxel index outside it
// sets ST_KEY_OVERFLOW, reported by the next check_status
// own (optional): every buffer sized to `in` comes from it instead of the handle.  labels / palette / rgb_out (optional, voxel > 0 and
// no cropper): every point's colour is palette[3 labels[i] ..], averaged per voxel like the points into rgb_out (3 x f64 per voxel)
int32_t op_voxel_down_sample(b2s_handle* h, const b2s_cloud* in, const CropDev* crop, double voxel, b2s_cloud* out, int fixed_key_bits = 0,
                             VoxelScratch* own = nullptr, const int32_t* labels = nullptr, const double* palette = nullptr,
                             double* rgb_out = nullptr);
// key width per axis of the voxel down-sample for a cloud of the given extent (> 21: the extent is too wide for the voxel)
int voxel_key_bits(double extent, double voxel);
int32_t bbox_reduce(b2s_handle* h, const double* xyz, const int32_t* d_n, size_t n_max, const CropDev* crop, unsigned long long* bbox);
// A1 (assemble.cu): Mapper::getAssembledMapPointCloud / assembleColoredPointCloud, optionally voxelized; rgb (coloured call): host
// n x 3, capacity / n_out like b2s_submap_dense_download.  Validated arguments.
int32_t op_assemble_map(b2s_handle* h, int n, const b2s_submap* const* submaps, double voxel, b2s_cloud* out, bool colored, double* rgb,
                        size_t capacity, size_t* n_out);
// A2 (assemble.cu): VoxelizedPointCloud::toPointCloud of every listed submap's dense map, concatenated; offsets (optional, host): n + 1
// entries.  Validated arguments.
int32_t op_assemble_dense_maps(b2s_handle* h, int n, const b2s_submap* const* submaps, b2s_cloud* out, int64_t* offsets);
// flags (optional, one int per point of c): only flagged points get a normal.  with_prior: c's normals on entry are the priors of
// [O3D] EstimateNormals on a cloud that has normals (keep the prior for a zero solver result, flip against it otherwise)
// dbg (b2s_debug_estimate_normals only; nullptr everywhere else): rec, 10 doubles per ORIGINAL point index, receives the nine cumulants
// and the neighbour count finish_normal was given; path (one int) and sel (4 doubles) per GRID SLOT: how select2 resolved the query
// (normals.cu NPATH_*) and its selection at the last block it tried (normals_select2_kernel)
struct NormalsDebug { double* rec; int32_t* path; double* sel; };
int32_t op_estimate_normals(b2s_handle* h, b2s_cloud* c, int knn, double radius, double cell_hint, const int32_t* flags = nullptr,
                            bool with_prior = false, const NormalsDebug* dbg = nullptr);
int32_t select_flags(b2s_handle* h, const b2s_cloud* in, double ratio, uint32_t seed);
int32_t select_compact(b2s_handle* h, const b2s_cloud* in, double ratio, b2s_cloud* out);
int32_t op_random_down_sample(b2s_handle* h, const b2s_cloud* in, double ratio, uint32_t seed, b2s_cloud* out);
int32_t op_transform(b2s_handle* h, const b2s_cloud* in, const double* T_host, b2s_cloud* out);

struct IcpProblem {
  const double* src_xyz;
  const int32_t* src_n;
  const GridHeader* ghdr;
  const int32_t* cell_start;
  const double* tgt_pts;    // double4
  const double* tgt_nrm;    // the target cloud's normals (3 x f64 per point, cloud order), indexed by tgt_pts[k].w
  double* work_xyz;         // global working copy of the source (used when it does not fit in shared memory) ...
  int32_t* work_prev;       // ... and its per-point search state
  const double* init_dev;   // optional device-resident init (overrides init)
  double init[16];
  double max_corr;
  double rel_fitness, rel_rmse;
  int32_t max_iter;
  int32_t src_n_max;
  int32_t estimator;        // B2S_REG_POINT_TO_PLANE / B2S_REG_POINT_TO_POINT / EST_INFORMATION
  int32_t pad;
  b2s_result* out;
  double* info_out;         // EST_INFORMATION: 36 doubles, row-major 6x6
  const double* src_nrm;    // B2S_REG_GENERALIZED: source normals (3 x f64 per point, source order)
  double gicp_eps;          // TransformationEstimationForGeneralizedICP::epsilon_ (1e-3)
  int32_t* corr_index;      // optional: per source point the ORIGINAL index of its final correspondence (-1 = none) ...
  double* corr_d2;          // ... and its squared distance (correspondence_set_ of the last evaluation)
};
constexpr int EST_INFORMATION = 3;   // internal estimator code: a single evaluation that outputs [O3D]'s information matrix
constexpr int EST_CORRESPONDENCES = 4;   // a single evaluation whose only output is corr_index / corr_d2 (+ fitness, rmse)
// single_host != nullptr: one registration, the problem travels as a kernel argument (no copy, no sync).  A batch runs the estimator of
// the handle's configuration unless batch_estimator >= 0 names one (the odometry constraints are always point-to-plane)
int32_t icp_launch(b2s_handle* h, const IcpProblem* single_host, const IcpProblem* problems_dev, int n_problems, size_t max_src_points,
                   int batch_estimator = -1);

int32_t op_submap_insert(b2s_handle* h, b2s_submap* sm, const b2s_cloud* scan, const double* T_dev, const int32_t* gate_dev);
// K-fuse bookkeeping (fuse.cu): (re)build the persistent voxel hash from the map cloud (after set_cloud / carving / transform;
// enable_dev gates it on the device), allocate it, and the tombstone-free view of the map for readers that leave the device
constexpr int FUSE_STAGE_BASE = 1 << 30;   // chain members >= this are staged scan points (index - FUSE_STAGE_BASE)
constexpr int FUSE_DUP_CAP = 1 << 16;
int32_t fuse_reserve(b2s_handle* h, b2s_submap* sm);
int32_t fuse_rehash(b2s_handle* h, b2s_submap* sm, const int32_t* enable_dev = nullptr);
int32_t dense_init(b2s_handle* h, b2s_submap* sm, size_t cap, double voxel);   // the dense table of cap (a power of two) empty slots
size_t fuse_table_slots(const b2s_submap* sm);   // the fusion table's slots for the submap's capacity (fuse_reserve)
// b2s_submap_create's set-up of a new submap (c_api.cu)
int32_t submap_init(b2s_handle* h, b2s_submap* sm, size_t capacity);
int32_t submap_compact_view(b2s_handle* h, b2s_submap* sm, b2s_cloud** view);   // -> sm->cloud[1] holding the live points in map order
// F2 VoxelHashMap queries on the dense map (fuse.cu)
int32_t op_dense_query(b2s_handle* h, const b2s_submap* sm, const b2s_cloud* pts, int32_t* count_dev, double* mean_dev);
int32_t op_dense_remove(b2s_handle* h, b2s_submap* sm, const b2s_cloud* pts);
int32_t op_dense_count(b2s_handle* h, const b2s_submap* sm, int32_t* out_dev);
// sensor_dev != nullptr: the sensor position is the translation of that device-resident 4x4; enable_dev (optional): the
// kernels return at once unless *enable_dev != 0 (device-side schedule of the mapper chain)
int32_t op_dense_carve(b2s_handle* h, b2s_submap* sm, const b2s_cloud* scan, const double* sensor, const double* sensor_dev, double radius,
                       double trunc, double max_len, int32_t* removed_dev, const int32_t* enable_dev = nullptr);
int32_t op_submap_transform(b2s_handle* h, b2s_submap* sm, const double* T_host);
int32_t op_cloud_transform(b2s_handle* h, b2s_cloud* c, const double* T_host);     // [O3D] PointCloud::Transform in place (voxel.cu)   // Submap::transform (voxel.cu)
// D1 constant-velocity de-skew (voxel.cu)
int32_t op_undistort(b2s_handle* h, const b2s_cloud* in, const double* lin_vel, const double* ang_vel_rpy, double scan_duration, int clockwise,
                     b2s_cloud* out);
// L1 overlap selection in front of the loop-closure ICP (overlap.cu); T_dev = sourceToTarget (device, row-major)
int32_t op_overlap(b2s_handle* h, const b2s_cloud* source, const b2s_cloud* target, const double* T_dev, double voxel, int min_pts,
                   b2s_cloud* source_overlap, b2s_cloud* target_overlap);
// the same for n pairs in one set of launches (overlap.cu).  Its tables are staged in the caller's page-locked stage at the offsets
// overlap_tables carved from the caller's stage layout, and uploaded to the same offsets of h->odo.
struct OverlapTables { size_t jobs, scan, T, end; };
OverlapTables overlap_tables(Layout& stage, int n);
int32_t op_overlap_batch(b2s_handle* h, int n, const b2s_submap* const* maps, const double* inits, double voxel, int min_pts,
                         b2s_cloud* const* outs, unsigned char* stage, const OverlapTables& tb);
// L2 odometry constraints of n (parent, child) submap pairs (constraints.cu); voxel = the map voxel after getMapVoxelSize; so_out /
// to_out: the caller's overlap clouds or nullptr; out: host records.  Synchronises once.
int32_t op_odometry_constraints(b2s_handle* h, int n, const b2s_submap* const* sources, const b2s_submap* const* targets,
                                const b2s_odometry_constraint_params& p, double voxel, b2s_cloud* const* so_out, b2s_cloud* const* to_out,
                                b2s_odometry_constraint* out);
// L3 loop-closure refinement of one source against n targets at the host-given sourceToTarget guesses inits (n x 16) (constraints.cu);
// voxel = the map voxel after getMapVoxelSize.  Synchronises once.
int32_t op_loop_closure_refinement(b2s_handle* h, const b2s_submap* source, int n, const b2s_submap* const* targets, const double* inits,
                                   const b2s_loop_closure_refinement_params& p, double voxel, b2s_cloud* const* so_out, b2s_cloud* const* to_out,
                                   b2s_loop_closure_refinement* out);
// G1 (posegraph.cu): [O3D] GlobalOptimization (Levenberg-Marquardt) of a validated graph: ids in range, parameters checked
int32_t op_global_optimization(b2s_handle* h, int n_nodes, double* poses, int n_edges, const b2s_pose_graph_edge* edges,
                               const b2s_global_optimization_params& p, int32_t* kept_out, double* conf_out, b2s_global_optimization_stats* stats);
// its production launches on host-given inputs (b2s_debug_pose_graph_solve / _linearize)
int32_t op_debug_pose_graph_solve(b2s_handle* h, int n_nodes, const double* A, const double* b, double lambda, double* delta_out, double* d_out,
                                  double* L_out);
int32_t op_debug_pose_graph_linearize(b2s_handle* h, int n_nodes, const double* poses, int n_edges, const b2s_pose_graph_edge* edges,
                                      const b2s_global_optimization_params& p, const double* conf_in, double* conf_out, double* H_out,
                                      double* b_out, double* rec_out);
// K-fpfh (features.cu): [O3D] ComputeFPFHFeature of the n points of c (normals required, 1 <= knn <= B2S_FEATURE_MAX_KNN)
int32_t op_compute_fpfh(b2s_handle* h, const b2s_cloud* c, size_t n, double radius, int knn, b2s_feature* f);
// K-ransac (ransac.cu): exact feature correspondences of one source feature against n target features (device outputs; s2t[k] / t2s[k]
// hold the source size / target k's size entries), and RegistrationRANSACBasedOnFeatureMatching of one source against n targets
int32_t op_feature_correspondences(b2s_handle* h, const b2s_feature* src, int n, const b2s_feature* const* tgts, int32_t* const* s2t,
                                   int32_t* const* t2s);
int32_t op_ransac(b2s_handle* h, const b2s_cloud* src, size_t ns, const b2s_feature* src_f, int n, const b2s_cloud* const* tgts, const size_t* nts,
                  const b2s_feature* const* tgt_fs, const b2s_ransac_params& p, b2s_ransac_result* out);
// C1 space carving of the sparse map (carve.cu); removed_dev (optional) receives the number of removed points
int32_t op_submap_carve(b2s_handle* h, b2s_submap* sm, const b2s_cloud* raw_scan, const double* T_dev, const CropDev& crop,
                        const b2s_carving_params& prm, int32_t* removed_dev, const int32_t* enable_dev = nullptr);
// T_dev != nullptr: device-resident pose (T_host ignored)
int32_t op_dense_insert(b2s_handle* h, b2s_submap* sm, const b2s_cloud* raw, const double* T_host, const double* T_dev, const b2s_cropper* crop,
                        const int32_t* enable_dev = nullptr);

// ---- pieces of the per-scan chains (c_api.cu) shared with the odometry chain (odometry.cu) ----
int32_t check_icp_params(const b2s_icp_params& p);
double nn_cell(const b2s_handle* h, double max_corr);
size_t icp_work_bytes(size_t n);
void fill_problem(IcpProblem* P, const b2s_icp_params& icp, const b2s_cloud* src, const GridIndex* g, const b2s_cloud* tgt, const double* init_host,
                  const double* init_dev, double* work, b2s_result* out_dev);
// crop (sensor frame) -> voxelize -> normals (icp.knn, icp.knn_radius) -> RandomDownSample; scratch receives the voxelized cloud
int32_t preprocess_scan(b2s_handle* h, const b2s_cloud* raw, const b2s_cropper& cropper, double voxel_size, double ratio, uint32_t seed,
                        const b2s_icp_params& icp, b2s_cloud* scratch, b2s_cloud* out);
int32_t process_scan_impl(b2s_handle* h, const b2s_cloud* raw, b2s_cloud* merge, b2s_cloud* match);
int32_t register_to_submap_async(b2s_handle* h, const b2s_cloud* scan, const b2s_submap* sm, const double* sensor_pose_host,
                                 const double* sensor_pose_dev, const double* init_host, const double* init_dev, b2s_result* out_dev);
int32_t mapper_chain_tail(b2s_handle* h, b2s_submap* sm, const b2s_cloud* raw_scan, const b2s_cloud* merge, const b2s_result* res,
                          double min_fitness, int ignore_fitness, b2s_result* slots, const int32_t* gstate);
int32_t make_cloud(b2s_handle* h, size_t capacity, bool normals, bool fixed, std::unique_ptr<b2s_cloud>* out);
// one step of a graph-replayable chain: replays the captured graph, or runs chain(ctx) eagerly while warming up, or captures it.
// key: the owner's options generation (a different key drops the graph like a re-allocation or b2s_set_config does)
int32_t graph_step(b2s_handle* h, GraphCache* g, unsigned long long key, int32_t (*chain)(void*), void* ctx);
int32_t graph_drop(b2s_handle* h, GraphCache* g);

// SMs of the current device (132 on an H100 SXM), queried once per device: the grid sizes below are multiples of it
int device_sms();
// upper bound of the CTAs of a streaming kernel: 2 per SM (B2S_GRID_CAP overrides).  With many concurrent chains, few fat CTAs
// leave the SMs to the other chains' kernels; a much larger cap (16 per SM) lost throughput there
int grid_cap();
// The stand-alone operators (voxel down-sample, normals, crop of ONE large cloud: config 3) are not sharing the GPU with other chains'
// kernels: for the duration of such a call the cap is lifted so that a 2^20-point cloud fills every SM.
struct WideGridScope {
  explicit WideGridScope(size_t n);
  ~WideGridScope();
  bool on;
};
inline int grid_for(size_t n, int threads, int max_blocks = 0) {
  if (max_blocks <= 0) max_blocks = grid_cap();
  size_t b = (n + (size_t)threads - 1) / (size_t)threads;
  if (b < 1) b = 1;
  if (b > (size_t)max_blocks) b = (size_t)max_blocks;
  return (int)b;
}

bool pdl_enabled();   // runtime.cu: true inside a PdlScope unless B2S_PDL=0 (A/B)
// Launches carry the attribute only inside the per-scan mapper chain (b2s_mapper_step_*), where it was measured to help at 16 chains;
// everywhere else kernels launch exactly as before.
struct PdlScope {
  PdlScope();
  ~PdlScope();
};

#ifdef __CUDACC__
// kernel<<<grid, block, smem, stream>>>(args...) with the programmatic-stream-serialization attribute (see pdl_wait)
template <typename... KArgs, typename... Args>
inline void launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  (void)cudaLaunchKernelEx(&cfg, kernel, KArgs(static_cast<Args&&>(args))...);   // errors surface through cudaGetLastError / the next B2S_CUDA, like <<<>>>
}
#endif

}  // namespace b2s

// ------------------------------------------------------------------------------------------------
// device helpers
// ------------------------------------------------------------------------------------------------
#ifdef __CUDACC__
namespace b2s {

// Programmatic dependent launch: every kernel of the library starts with this wait and every launch carries the programmatic-stream-
// serialization attribute, so a kernel's launch (scheduling, CTA distribution, its own prologue up to here) overlaps the tail of its
// predecessor in the stream instead of starting after it -- a scan is a chain of 42 kernels of 3-50 us.  Past the wait the predecessor
// grid has completed and its writes are visible, so nothing else changes.  Without the launch attribute the instruction is a no-op.
// (An explicit early griddepcontrol.launch_dependents at the top of every kernel was measured too: the successors' CTAs become resident
// long before they can run and hold registers / shared memory that the other chains' kernels need, and throughput dropped.)
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// order-preserving map double -> uint64 so that atomicMin/atomicMax work on doubles
__host__ __device__ inline unsigned long long ord_encode(double v) {
  unsigned long long u;
#ifdef __CUDA_ARCH__
  u = (unsigned long long)__double_as_longlong(v);
#else
  memcpy(&u, &v, 8);
#endif
  return (u & 0x8000000000000000ull) ? ~u : (u | 0x8000000000000000ull);
}
__host__ __device__ inline double ord_decode(unsigned long long u) {
  u = (u & 0x8000000000000000ull) ? (u & 0x7FFFFFFFFFFFFFFFull) : ~u;
#ifdef __CUDA_ARCH__
  return __longlong_as_double((long long)u);
#else
  double v; memcpy(&v, &u, 8); return v;
#endif
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ int warp_sum_i(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_min(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmin(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Folds every thread's box (mn / mx, +-INFINITY when empty) into the ord_encode'd words box[0..5] (min xyz, max xyz): reduced over the
// block, then six atomics.  Every thread of the block must call it (it synchronises the block); THREADS = blockDim.x, a multiple of 32.
template <int THREADS>
__device__ __forceinline__ void box_fold_block(double (&mn)[3], double (&mx)[3], unsigned long long* box) {
  constexpr int nwarps = THREADS / 32;
  __shared__ double s[6][nwarps];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int d = 0; d < 3; d++) { mn[d] = warp_min(mn[d]); mx[d] = warp_max(mx[d]); }
  if (lane == 0) { for (int d = 0; d < 3; d++) { s[d][warp] = mn[d]; s[3 + d][warp] = mx[d]; } }
  __syncthreads();
  if (threadIdx.x < 6) {
    const int d = threadIdx.x;
    double v = s[d][0];
#pragma unroll 1
    for (int w = 1; w < nwarps; w++) v = d < 3 ? fmin(v, s[d][w]) : fmax(v, s[d][w]);
    if (d < 3) { if (v < INFINITY) atomicMin(&box[d], ord_encode(v)); }
    else if (v > -INFINITY) atomicMax(&box[d], ord_encode(v));
  }
}

// [O3D] TransformVector6dToMatrix4d: R = Rz(x2) Ry(x1) Rx(x0), t = x[3..5] (the ICP update and the pose-graph LM step)
__device__ __forceinline__ void vec6_to_mat4_dev(const double (&x)[6], double* T) {
  double sa, ca, sb, cb, sg, cgm;
  sincos(x[0], &sa, &ca); sincos(x[1], &sb, &cb); sincos(x[2], &sg, &cgm);
  T[0] = cgm * cb; T[1] = cgm * sb * sa - sg * ca; T[2] = cgm * sb * ca + sg * sa; T[3] = x[3];
  T[4] = sg * cb;  T[5] = sg * sb * sa + cgm * ca; T[6] = sg * sb * ca - cgm * sa; T[7] = x[4];
  T[8] = -sb;      T[9] = cb * sa;                 T[10] = cb * ca;                T[11] = x[5];
  T[12] = 0; T[13] = 0; T[14] = 0; T[15] = 1;
}

// squared distance accumulated exactly like nanoflann's L2 adaptor and the oracle: (dx*dx + dy*dy) + dz*dz,
// with explicit round-to-nearest ops so that nvcc never contracts it into FMAs (keeps argmin / strict radius
// decisions bit-identical to the CPU oracle)
__device__ __forceinline__ double dist2_exact(double ax, double ay, double az, double bx, double by, double bz) {
  double dx = __dsub_rn(ax, bx), dy = __dsub_rn(ay, by), dz = __dsub_rn(az, bz);
  return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}

// ---- Searches over a K-index grid (GridHeader, grid_index.cu) ----
// Every search follows the rules of the build and of the oracle's KD-tree, so that its neighbours match the oracle's bit for bit:
// a coordinate's cell is grid_axis_cell, a neighbour qualifies only if d2 < r2 (dist2_exact), and neighbours are ordered by
// (d2, original index).  icp.cu keeps its own tuned scan over a register copy of the header (GridView), on the same rules.

// cell of coordinate v on an axis with origin o and n cells, clamped into the grid: the build files every point with it, outside
// points into the border cells
__device__ __forceinline__ int grid_axis_cell(double v, double o, double inv_cell, int n) {
  return (int)fmin(fmax(floor((v - o) * inv_cell), 0.0), (double)(n - 1));
}

// the (d2, original index) order of neighbours: equal distances go to the lower index
__device__ __forceinline__ bool nn_key_less(double da, int ia, double db, int ib) { return da < db || (da == db && ia < ib); }

// distance from q to cell i of an axis with n cells (border cells reach to infinity), less eps and at least 0
__device__ __forceinline__ double slab_gap(double q, double o, double cell, int i, int n, double eps) {
  double g = 0.0;
  if (i > 0) { double lo = o + (double)i * cell; if (q < lo) g = lo - q; }
  if (i < n - 1) { double hi = o + (double)(i + 1) * cell; if (q > hi) g = q - hi; }
  g -= eps;  // slack: cell membership was decided with floor((p-o)*inv), which can disagree with o+i*cell by an ulp
  return g > 0.0 ? g : 0.0;
}

// distance from q to the nearest face of the (2R+1)^3 block around cell c that has cells beyond it, less eps and at least 0: every
// point outside the block lies further away.  INFINITY once the block covers the grid.
__device__ __forceinline__ double ring_bound(const GridHeader& g, const double (&q)[3], const int (&c)[3], int R, double eps) {
  double bound = INFINITY;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    if (c[a] - R > 0) bound = fmin(bound, q[a] - (g.origin[a] + (double)(c[a] - R) * g.cell));
    if (c[a] + R < g.dims[a] - 1) bound = fmin(bound, (g.origin[a] + (double)(c[a] + R + 1) * g.cell) - q[a]);
  }
  if (bound == INFINITY) return bound;
  bound -= eps;
  return bound > 0.0 ? bound : 0.0;
}

// Exact hybrid k-NN of q -- the knn nearest with d2 < r2, in (d2, index) order -- by one warp, every lane with the same query.
// Rings R = 0, 1, .. of cells around q's cell: per ring each lane first resolves ONE (y, z) row (the slab-gap test and the two
// dependent cell_start loads, the latency that dominates in empty space), then the warp walks the non-empty rows together, 32
// candidates per step.  The k best are a sorted list of ROWS * 32 entries: position p = m * 32 + lane is register row m of that
// lane, holding d2 (ed), original index (ei) and, with kSlot, slot in pts (es; left untouched without, which keeps the registers
// of a caller that does not need it); empty entries are (INFINITY, 0x7fffffff, -1).  A qualifying
// candidate is inserted with one shuffle-up of every row, lane 31 of row m - 1 carried into lane 0 of row m.  The walk ends once
// the nearest block face with cells behind it lies beyond the k-th best.  Requires 1 <= knn <= ROWS * 32.
template <int ROWS, bool kSlot>
__device__ __forceinline__ void grid_knn_walk(const GridHeader& g, const int32_t* __restrict__ cs, const double4* __restrict__ pts,
                                              double qx, double qy, double qz, int knn, double r2,
                                              double (&ed)[ROWS], int (&ei)[ROWS], int (&es)[ROWS]) {
  const unsigned FULL = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const double eps = 1e-9 * g.cell;
  const int nx = g.dims[0], ny = g.dims[1], nz = g.dims[2];
  const double q[3] = {qx, qy, qz};
  const int c[3] = {grid_axis_cell(qx, g.origin[0], g.inv_cell, nx), grid_axis_cell(qy, g.origin[1], g.inv_cell, ny),
                    grid_axis_cell(qz, g.origin[2], g.inv_cell, nz)};
  const int cx = c[0], cy = c[1], cz = c[2];
  const int km = (knn - 1) >> 5, kl = (knn - 1) & 31;   // list position of the k-th neighbour
#pragma unroll
  for (int m = 0; m < ROWS; ++m) { ed[m] = INFINITY; ei[m] = 0x7fffffff; if (kSlot) es[m] = -1; }
  double kd = INFINITY; int ki = 0x7fffffff;   // current k-th best
  for (int R = 0;; ++R) {
    const int side = 2 * R + 1;
    const int x0 = max(cx - R, 0), x1 = min(cx + R, nx - 1);
    for (int t0 = 0; t0 < side * side; t0 += 32) {
      int a0 = 0, b0 = 0, a1 = 0, b1 = 0;   // this lane's row: the whole x-run on the ring's shell, else its two end cells
      const int t = t0 + lane;
      if (t < side * side) {
        const int z = cz - R + t / side, y = cy - R + t % side;
        if (z >= 0 && z < nz && y >= 0 && y < ny) {
          const double gz = slab_gap(qz, g.origin[2], g.cell, z, nz, eps);
          const double gy = slab_gap(qy, g.origin[1], g.cell, y, ny, eps);
          if (gz * gz + gy * gy <= fmin(kd, r2)) {
            const int row = (z * ny + y) * nx;
            if (z == cz - R || z == cz + R || y == cy - R || y == cy + R) { a0 = cs[row + x0]; b0 = cs[row + x1 + 1]; }
            else {
              if (cx - R >= 0) { a0 = cs[row + cx - R]; b0 = cs[row + cx - R + 1]; }
              if (cx + R <= nx - 1) { a1 = cs[row + cx + R]; b1 = cs[row + cx + R + 1]; }
            }
          }
        }
      }
      for (int part = 0; part < 2; ++part) {
        unsigned rows = __ballot_sync(FULL, part == 0 ? (b0 > a0) : (b1 > a1));
        while (rows) {
          const int src_lane = __ffs(rows) - 1;
          rows &= rows - 1;
          const int a = __shfl_sync(FULL, part == 0 ? a0 : a1, src_lane);
          const int b = __shfl_sync(FULL, part == 0 ? b0 : b1, src_lane);
          for (int j0 = a; j0 < b; j0 += 32) {
            const int j = j0 + lane;
            double d = INFINITY; int idx = 0x7fffffff;
            if (j < b) {
              const double4 p = pts[j];
              d = dist2_exact(qx, qy, qz, p.x, p.y, p.z);
              idx = (int)__double_as_longlong(p.w);
            }
            unsigned mask = __ballot_sync(FULL, j < b && d < r2 && nn_key_less(d, idx, kd, ki));
            while (mask) {
              const int src = __ffs(mask) - 1;
              mask &= mask - 1;
              const double cd = __shfl_sync(FULL, d, src);
              const int ci = __shfl_sync(FULL, idx, src);
              if (!nn_key_less(cd, ci, kd, ki)) continue;   // an earlier insertion of this batch moved the k-th entry
              double pd[ROWS], td[ROWS]; int pi[ROWS], ti[ROWS], ps[ROWS], ts[ROWS];
#pragma unroll
              for (int m = 0; m < ROWS; ++m) {
                pd[m] = __shfl_up_sync(FULL, ed[m], 1); pi[m] = __shfl_up_sync(FULL, ei[m], 1);
                td[m] = __shfl_sync(FULL, ed[m], 31); ti[m] = __shfl_sync(FULL, ei[m], 31);
                if (kSlot) { ps[m] = __shfl_up_sync(FULL, es[m], 1); ts[m] = __shfl_sync(FULL, es[m], 31); }
              }
#pragma unroll
              for (int m = 0; m < ROWS; ++m) {   // the entry one position before this lane's: lane - 1, or lane 31 of the row above
                const bool has_prev = lane > 0 || m > 0;
                const double prd = lane > 0 ? pd[m] : (m > 0 ? td[m > 0 ? m - 1 : 0] : -INFINITY);
                const int pri = lane > 0 ? pi[m] : (m > 0 ? ti[m > 0 ? m - 1 : 0] : -1);
                if (nn_key_less(cd, ci, ed[m], ei[m])) {
                  if (has_prev && nn_key_less(cd, ci, prd, pri)) {
                    ed[m] = prd; ei[m] = pri;
                    if (kSlot) es[m] = lane > 0 ? ps[m] : ts[m > 0 ? m - 1 : 0];
                  } else {
                    ed[m] = cd; ei[m] = ci;
                    if (kSlot) es[m] = j0 + src;
                  }
                }
              }
              double kdl = ed[0]; int kil = ei[0];
#pragma unroll
              for (int m = 1; m < ROWS; ++m) if (m == km) { kdl = ed[m]; kil = ei[m]; }
              kd = __shfl_sync(FULL, kdl, kl);
              ki = __shfl_sync(FULL, kil, kl);
            }
          }
        }
      }
    }
    const double bound = ring_bound(g, q, c, R, eps);
    if (bound == INFINITY || bound * bound > fmin(kd, r2)) break;
  }
}

// Exact 1-NN of q within r: the (d2, index)-least point with d2 < r * r, or -1.  Returns its slot in pts and its d2 in *d2.
// It scans every cell of the box floor((q -+ r - o) * inv_cell -+ 1e-6): the build's cell rule, widened by a millionth of a cell on
// either side.  That holds every point with d2 < r2: such a point lies within r (1 + a few ulp) of q on every axis, and the rounding
// of its cell coordinate and of the box edge's can put it across the edge only by a few ulp of those coordinates -- far below 1e-6
// cell while points and queries lie within ~1e8 cells of the origin.  A larger box holds the same qualifying points, so any box
// that holds them all returns the same point.
__device__ __forceinline__ int grid_nearest(const GridHeader& g, const int32_t* __restrict__ cs, const double4* __restrict__ pts,
                                            double qx, double qy, double qz, double r, double* d2) {
  const double r2 = r * r, q[3] = {qx, qy, qz};
  int lo[3], hi[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const double top = (double)(g.dims[a] - 1);
    lo[a] = (int)fmin(fmax(floor((q[a] - r - g.origin[a]) * g.inv_cell - 1e-6), 0.0), top);
    hi[a] = (int)fmin(fmax(floor((q[a] + r - g.origin[a]) * g.inv_cell + 1e-6), 0.0), top);
  }
  double bd = INFINITY; int bi = 0x7fffffff, bslot = -1;
  for (int z = lo[2]; z <= hi[2]; z++)
    for (int y = lo[1]; y <= hi[1]; y++) {
      const int row = (z * g.dims[1] + y) * g.dims[0];
      const int e = cs[row + hi[0] + 1];
      for (int j = cs[row + lo[0]]; j < e; j++) {
        const double4 p = pts[j];
        const double d = dist2_exact(qx, qy, qz, p.x, p.y, p.z);
        const int idx = (int)__double_as_longlong(p.w);
        if (d < r2 && nn_key_less(d, idx, bd, bi)) { bd = d; bi = idx; bslot = j; }
      }
    }
  *d2 = bd;
  return bslot;
}

// 3x3 SVD by one-sided Jacobi (Hestenes), singular values sorted descending like Eigen's JacobiSVD (the rotation that
// umeyama builds from it is unique for rank >= 2, so the SVD algorithm itself need not be Eigen's).  One thread, a few
// hundred flops per registration iteration (icp.cu) or RANSAC hypothesis (ransac.cu).
static __device__ void svd3_dev(const double* A, double* U, double* S, double* V) {
  double W[9], Vm[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  for (int i = 0; i < 9; i++) W[i] = A[i];
  for (int sweep = 0; sweep < 60; sweep++) {
    bool rotated = false;
    for (int p = 0; p < 2; p++)
      for (int q = p + 1; q < 3; q++) {
        double alpha = 0, beta = 0, gamma = 0;
        for (int i = 0; i < 3; i++) { alpha += W[3 * i + p] * W[3 * i + p]; beta += W[3 * i + q] * W[3 * i + q]; gamma += W[3 * i + p] * W[3 * i + q]; }
        if (gamma == 0.0 || fabs(gamma) <= 1e-16 * sqrt(alpha * beta)) continue;
        rotated = true;
        const double zeta = (beta - alpha) / (2.0 * gamma);
        const double t = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
        const double c = 1.0 / sqrt(1.0 + t * t), sn = c * t;
        for (int i = 0; i < 3; i++) {
          const double wp = W[3 * i + p], wq = W[3 * i + q];
          W[3 * i + p] = c * wp - sn * wq; W[3 * i + q] = sn * wp + c * wq;
          const double vp = Vm[3 * i + p], vq = Vm[3 * i + q];
          Vm[3 * i + p] = c * vp - sn * vq; Vm[3 * i + q] = sn * vp + c * vq;
        }
      }
    if (!rotated) break;
  }
  double sv[3]; int ord[3] = {0, 1, 2};
  for (int j = 0; j < 3; j++) sv[j] = sqrt(W[j] * W[j] + W[3 + j] * W[3 + j] + W[6 + j] * W[6 + j]);
  for (int a = 0; a < 2; a++)
    for (int b = 0; b < 2 - a; b++) if (sv[ord[b]] < sv[ord[b + 1]]) { const int t = ord[b]; ord[b] = ord[b + 1]; ord[b + 1] = t; }
  const double tiny = 1e-300;
  for (int j = 0; j < 3; j++) {
    const int o = ord[j];
    S[j] = sv[o];
    for (int i = 0; i < 3; i++) { V[3 * i + j] = Vm[3 * i + o]; U[3 * i + j] = sv[o] > tiny ? W[3 * i + o] / sv[o] : 0.0; }
  }
  if (!(S[0] > tiny)) { for (int i = 0; i < 9; i++) U[i] = (i % 4 == 0) ? 1.0 : 0.0; return; }
  if (!(S[1] > tiny)) {
    const double u0[3] = {U[0], U[3], U[6]};
    const int k = fabs(u0[0]) <= fabs(u0[1]) ? (fabs(u0[0]) <= fabs(u0[2]) ? 0 : 2) : (fabs(u0[1]) <= fabs(u0[2]) ? 1 : 2);
    double e[3] = {0, 0, 0}; e[k] = 1.0;
    const double d = e[0] * u0[0] + e[1] * u0[1] + e[2] * u0[2];
    const double v[3] = {e[0] - d * u0[0], e[1] - d * u0[1], e[2] - d * u0[2]};
    const double nv = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
    U[1] = v[0] / nv; U[4] = v[1] / nv; U[7] = v[2] / nv;
  }
  // u2 = u0 x u1 also when the third column is rounding noise that is not orthogonal to the others: an exactly zero row of A keeps
  // every column of W in a plane, so W's third column can never become orthogonal to the first two (rank-2 sets such as a level
  // plane of points)
  const double c[3] = {U[3] * U[7] - U[6] * U[4], U[6] * U[1] - U[0] * U[7], U[0] * U[4] - U[3] * U[1]};
  if (!(fabs(c[0] * U[2] + c[1] * U[5] + c[2] * U[8]) > 0.5)) { U[2] = c[0]; U[5] = c[1]; U[8] = c[2]; }
}

__device__ __forceinline__ double det3_dev(const double* M) {
  return M[0] * (M[4] * M[8] - M[5] * M[7]) - M[1] * (M[3] * M[8] - M[5] * M[6]) + M[2] * (M[3] * M[7] - M[4] * M[6]);
}

// reference croppers (core/src/croppers.cpp:121-165); only the translation of the pose is used
__device__ __forceinline__ bool crop_within(const CropDev& c, double x, double y, double z) {
  double cx = c.cx, cy = c.cy, cz = c.cz;
  if (c.pose_dev) { cx = c.pose_dev[3]; cy = c.pose_dev[7]; cz = c.pose_dev[11]; }
  double dx = __dsub_rn(x, cx), dy = __dsub_rn(y, cy), dz = __dsub_rn(z, cz);
  bool w = true;
  switch (c.kind) {
    case B2S_CROP_MAX_RADIUS: w = sqrt(__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz))) <= c.rmax; break;
    case B2S_CROP_MIN_RADIUS: w = sqrt(__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz))) >= c.rmin; break;
    case B2S_CROP_MINMAX_RADIUS: {
      double d = sqrt(__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)));
      w = d <= c.rmax && d >= c.rmin;
      break;
    }
    case B2S_CROP_CYLINDER: w = z >= c.zmin && z <= c.zmax && sqrt(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy))) <= c.rmax; break;
    default: w = true;
  }
  return c.invert ? !w : w;
}

// 3 x 10-bit (u32) and 3 x 21-bit (u64) Morton interleave
__device__ __forceinline__ uint32_t morton_part10(uint32_t x) {
  x &= 0x3FFu;
  x = (x | (x << 16)) & 0x030000FFu;
  x = (x | (x << 8)) & 0x0300F00Fu;
  x = (x | (x << 4)) & 0x030C30C3u;
  x = (x | (x << 2)) & 0x09249249u;
  return x;
}
__device__ __forceinline__ uint64_t morton_part21(uint64_t x) {
  x &= 0x1FFFFFull;
  x = (x | (x << 32)) & 0x1F00000000FFFFull;
  x = (x | (x << 16)) & 0x1F0000FF0000FFull;
  x = (x | (x << 8)) & 0x100F00F00F00F00Full;
  x = (x | (x << 4)) & 0x10C30C30C30C30C3ull;
  x = (x | (x << 2)) & 0x1249249249249249ull;
  return x;
}

// ConstantVelocityMotionCompensation::undistortInputPointCloud / computePhase (core/src/MotionCompensation.cpp:82-100,120-139) for one
// point: p' = R(q) p + t with t = phase * scanDuration * v, q = fromRPY(phase * scanDuration * w).normalized() = qz * qy * qx
// (core/src/math.cpp:32-37), R(q) as Eigen::Quaternion::toRotationMatrix.  Shared by b2s_undistort (voxel.cu) and the de-skew of the
// combined chain (odometry.cu), so both give the same bits for the same velocities.
__device__ __forceinline__ void undistort_point(double px, double py, double pz, double vx, double vy, double vz, double wr, double wp,
                                                double wy, double duration, int clockwise, double* out) {
  const double two_pi = 2.0 * 3.14159265358979323846;
  const double angle = atan2(py, px);
  const double wrapped = angle < 0.0 ? (angle + two_pi) : angle;
  double phase = 0.0;
  if (wrapped != 0.0) phase = clockwise ? 1.0 - wrapped / two_pi : wrapped / two_pi;
  const double s = phase * duration;
  const double tx_ = s * vx, ty_ = s * vy, tz_ = s * vz;
  const double r = s * wr, pi_ = s * wp, yw = s * wy;
  double sr, cr, sp, cp, sy, cy;
  sincos(0.5 * r, &sr, &cr); sincos(0.5 * pi_, &sp, &cp); sincos(0.5 * yw, &sy, &cy);
  // qzy = qz * qy with qz = (cy,0,0,sy), qy = (cp,0,sp,0);  q = qzy * qx with qx = (cr,sr,0,0)   (Eigen's product, all terms kept)
  const double a0 = cy * cp - 0.0 * 0.0 - 0.0 * sp - sy * 0.0;
  const double a1 = cy * 0.0 + 0.0 * cp + 0.0 * 0.0 - sy * sp;
  const double a2 = cy * sp + 0.0 * cp + sy * 0.0 - 0.0 * 0.0;
  const double a3 = cy * 0.0 + sy * cp + 0.0 * sp - 0.0 * 0.0;
  double w = a0 * cr - a1 * sr - a2 * 0.0 - a3 * 0.0;
  double x = a0 * sr + a1 * cr + a2 * 0.0 - a3 * 0.0;
  double y = a0 * 0.0 + a2 * cr + a3 * sr - a1 * 0.0;
  double z = a0 * 0.0 + a3 * cr + a1 * 0.0 - a2 * sr;
  const double n2 = w * w + x * x + y * y + z * z;
  if (n2 > 0.0) { const double nn = sqrt(n2); w /= nn; x /= nn; y /= nn; z /= nn; }
  const double tx = 2 * x, ty = 2 * y, tz = 2 * z, twx = tx * w, twy = ty * w, twz = tz * w, txx = tx * x, txy = ty * x, txz = tz * x,
               tyy = ty * y, tyz = tz * y, tzz = tz * z;
  out[0] = ((1 - (tyy + tzz)) * px + (txy - twz) * py + (txz + twy) * pz) + tx_;
  out[1] = ((txy + twz) * px + (1 - (txx + tzz)) * py + (tyz - twx) * pz) + ty_;
  out[2] = ((txz - twy) * px + (tyz + twx) * py + (1 - (txx + tyy)) * pz) + tz_;
}

// The map-side voxel hashes (fusion and dense map in fuse.cu, carve.cu, overlap.cu, voxelmap.cu) share one key and one probe: the
// voxel index getVoxelIdx(p, inverseVoxelSize) = floor(p * inv) on the global-origin grid (VoxelHashMap.hpp:47-50), accepted while
// |index| < 2^20 - 1 on every axis, packed as three 21-bit fields offset by 2^20, hashed by the murmur3 finalizer and probed linearly
// over a power-of-two table (mask = slots - 1).  Each table keeps its own fill limit and occupancy count.  tests/voxel_hash.py restates
// these rules.
constexpr unsigned long long VOXEL_KEY_EMPTY = ~0ull;

__device__ __forceinline__ unsigned long long voxel_key_pack(int x, int y, int z) {
  return ((unsigned long long)(unsigned)(x + 1048576) << 42) | ((unsigned long long)(unsigned)(y + 1048576) << 21) |
         (unsigned long long)(unsigned)(z + 1048576);
}
__device__ __forceinline__ void voxel_key_unpack(unsigned long long k, int* x, int* y, int* z) {
  *x = (int)((k >> 42) & 0x1FFFFF) - 1048576; *y = (int)((k >> 21) & 0x1FFFFF) - 1048576; *z = (int)(k & 0x1FFFFF) - 1048576;
}
__device__ __forceinline__ unsigned long long voxel_key_hash(unsigned long long k) {
  k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
  return k;
}
// one inverse voxel size per axis (VoxelMap takes a Vector3d; every other table passes the same inverse three times)
__device__ __forceinline__ bool voxel_key_of(double x, double y, double z, double ix, double iy, double iz, unsigned long long* key) {
  const double fx = floor(__dmul_rn(x, ix)), fy = floor(__dmul_rn(y, iy)), fz = floor(__dmul_rn(z, iz));
  if (!(fabs(fx) < 1048575.0 && fabs(fy) < 1048575.0 && fabs(fz) < 1048575.0)) return false;   // also rejects NaN
  *key = voxel_key_pack((int)fx, (int)fy, (int)fz);
  return true;
}
// slot of `key`, or -1 when it is absent
__device__ __forceinline__ long long voxel_key_find(const unsigned long long* __restrict__ keys, size_t mask, unsigned long long key) {
  size_t s = (size_t)voxel_key_hash(key) & mask;
  for (size_t probe = 0; probe <= mask; ++probe, s = (s + 1) & mask) {
    const unsigned long long k = keys[s];
    if (k == VOXEL_KEY_EMPTY) return -1;
    if (k == key) return (long long)s;
  }
  return -1;
}
// slot of `key`, inserting it when absent (-1: every slot of the probe run holds another key); *fresh: this thread claimed the slot
__device__ __forceinline__ long long voxel_key_claim(unsigned long long* keys, size_t mask, unsigned long long key, bool* fresh) {
  size_t s = (size_t)voxel_key_hash(key) & mask;
  // written so that no caller needs more registers than it did with its own copy of the loop (ptxas reports)
  for (size_t probe = 0;; s = (s + 1) & mask) {
    const unsigned long long old = atomicCAS(&keys[s], VOXEL_KEY_EMPTY, key);
    if (old == key) { *fresh = false; return (long long)s; }
    if (old == VOXEL_KEY_EMPTY) { *fresh = true; return (long long)s; }
    if (++probe > mask) { *fresh = false; return -1; }
  }
}

// A row-major 4x4 T applied to one point or vector as the reference's Eigen code does it, every row summed left to right (the library
// is built with -fmad=false, and the explicit round-to-nearest ops keep the order fixed): transform_point = o3d_slam::transform /
// [O3D] TransformPoints, (T p).head3 / w; affine_point = R p + t; rotate_vector = R n ([O3D] TransformNormals).
__device__ __forceinline__ void transform_point(const double* T, double x, double y, double z, double* ox, double* oy, double* oz) {
  const double a = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[0], x), __dmul_rn(T[1], y)), __dmul_rn(T[2], z)), T[3]);
  const double b = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[4], x), __dmul_rn(T[5], y)), __dmul_rn(T[6], z)), T[7]);
  const double c = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[8], x), __dmul_rn(T[9], y)), __dmul_rn(T[10], z)), T[11]);
  const double w = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[12], x), __dmul_rn(T[13], y)), __dmul_rn(T[14], z)), T[15]);
  *ox = __ddiv_rn(a, w); *oy = __ddiv_rn(b, w); *oz = __ddiv_rn(c, w);
}
__device__ __forceinline__ void affine_point(const double* T, double x, double y, double z, double* ox, double* oy, double* oz) {
  const double a = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[0], x), __dmul_rn(T[1], y)), __dmul_rn(T[2], z)), T[3]);
  const double b = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[4], x), __dmul_rn(T[5], y)), __dmul_rn(T[6], z)), T[7]);
  const double c = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[8], x), __dmul_rn(T[9], y)), __dmul_rn(T[10], z)), T[11]);
  *ox = a; *oy = b; *oz = c;
}
__device__ __forceinline__ void rotate_vector(const double* T, double x, double y, double z, double* ox, double* oy, double* oz) {
  const double a = __dadd_rn(__dadd_rn(__dmul_rn(T[0], x), __dmul_rn(T[1], y)), __dmul_rn(T[2], z));
  const double b = __dadd_rn(__dadd_rn(__dmul_rn(T[4], x), __dmul_rn(T[5], y)), __dmul_rn(T[6], z));
  const double c = __dadd_rn(__dadd_rn(__dmul_rn(T[8], x), __dmul_rn(T[9], y)), __dmul_rn(T[10], z));
  *ox = a; *oy = b; *oz = c;
}
// o3d_slam::transform's near-identity test (helpers.cpp:275): max |T - I| < 1e-4 -> the untransformed cloud is copied first and every
// transformed point appended as well
__device__ __forceinline__ bool near_identity(const double* T) {
  double mx = 0.0;
#pragma unroll
  for (int i = 0; i < 16; i++) mx = fmax(mx, fabs(T[i] - ((i % 5 == 0) ? 1.0 : 0.0)));
  return mx < 1e-4;
}

}  // namespace b2s
#endif
