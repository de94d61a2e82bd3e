// c_api.cu -- the extern "C" boundary declared in include/b2s.h.  Host-side plumbing only: argument checks mirroring
// the reference's asserts, device staging, kernel sequencing.  No arithmetic of the hot path runs on the host.
#include <math.h>
#include <stdlib.h>

#include "common.cuh"

using namespace b2s;

namespace b2s {
int32_t pose_to_device(b2s_handle* h, const double* T, double* dst);
int32_t dense_init(b2s_handle* h, b2s_submap* sm, size_t cap, double voxel);
int32_t dense_to_cloud(b2s_handle* h, b2s_submap* sm, double* d_xyz, int32_t* d_keys, int32_t* d_out_n);

__global__ void f32_to_f64_kernel(const unsigned char* __restrict__ src, size_t stride, int n, double* __restrict__ dst) {
  pdl_wait();
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float* p = reinterpret_cast<const float*>(src + (size_t)i * stride);
    dst[3 * i] = (double)p[0]; dst[3 * i + 1] = (double)p[1]; dst[3 * i + 2] = (double)p[2];
  }
}

__global__ void write_i32_kernel(int32_t* p, int32_t v) {
  pdl_wait(); *p = v; }
__global__ void pad_kernel() {
  pdl_wait();}   // B2S_PAD_LAUNCHES=n: n empty launches per scan, to measure what a launch costs the chain (tuning aid)

__global__ void empty_check_kernel(const int32_t* a, const int32_t* b, uint32_t* status) {
  pdl_wait();
  if (*a <= 0 || *b <= 0) atomicOr(status, ST_EMPTY);
}

// guess = pose * odom ; (row-major 4x4).  After a new initial value, and in the step that follows it, the guess is the pose
// itself (Mapper.cpp:130-138: no odometry prediction while isNewInitialValueSet_ or isIgnoreOdometryPrediction_)
__global__ void compose_kernel(const double* __restrict__ A, const double* __restrict__ B, double* __restrict__ C, const int32_t* __restrict__ ms) {
  pdl_wait();
  const int i = threadIdx.x >> 2, j = threadIdx.x & 3;
  const bool hold = ms[MS_NEWINIT] || ms[MS_IGNODOM];
  if (threadIdx.x < 16) {
    double s = 0.0;
    for (int k = 0; k < 4; k++) s += A[4 * i + k] * B[4 * k + j];
    C[4 * i + j] = hold ? A[4 * i + j] : s;
  }
}

// Everything Mapper::addRangeMeasurement decides after the registration (core/src/Mapper.cpp:151-177), on the device:
//   fitness gate (:151)            accepted -> mapToRangeSensor_ = result (pose slot 0)
//   minimum-motion gate (:170-176) sensorMotion = mapToRangeSensorLastScanInsertion_^-1 * mapToRangeSensor_ (pose slot 5)
//   carving schedule               Submap::carve: map not empty and nScansInsertedMap_ % N == 1 (Submap.cpp:111)
//   dense map                      fed with every accepted scan (SlamWrapper.cpp:318-327), carved when nScansInsertedDenseMap_ % N == 1
//   new initial value (:143-149)   the first step after b2s_submap_set_initial_transform counts as accepted, keeps the pose (the ICP
//                                  result is discarded), inserts nothing and makes the next step ignore the odometry prediction
//   pure localisation (:163-167)   merge_on == 0: an accepted scan updates the pose only; no carving, no insertion
// and the copy of the result into this step's slot of the result ring (slots == nullptr: the result already sits in its slot).
struct GateArgs {
  double min_fitness, min_move;
  int ignore_fitness, carve_on, carve_n, dense_on, dcarve_n, merge_on;
};
__global__ void mapper_gate_kernel(const b2s_result* __restrict__ res, GateArgs a, double* pose, int32_t* ms, const int32_t* __restrict__ map_n,
                                   b2s_result* slots, const int32_t* __restrict__ gstate) {
  pdl_wait();
  if (threadIdx.x != 0) return;
  const int init = ms[MS_NEWINIT];
  ms[MS_NEWINIT] = 0; ms[MS_IGNODOM] = init; ms[MS_INITSTEP] = init;   // isIgnoreOdometryPrediction_ lasts exactly one step
  const bool accepted = init || a.ignore_fitness || !(res->fitness < a.min_fitness);
  if (accepted && !init) for (int i = 0; i < 16; i++) pose[i] = res->T[i];
  bool insert = accepted && !init && a.merge_on;
  if (insert && a.min_move > 0.0) {
    // Eigen: inverse of an isometry = (R^T, -(R^T t)); translation of the product A * B = A.linear() * B.translation() + A.translation()
    const double* L = pose + 5 * 16;
    const double* P = pose;
    double it[3], m[3];
    for (int i = 0; i < 3; i++) it[i] = -(L[i] * L[3] + L[4 + i] * L[7] + L[8 + i] * L[11]);
    for (int i = 0; i < 3; i++) m[i] = (L[i] * P[3] + L[4 + i] * P[7] + L[8 + i] * P[11]) + it[i];
    const double moved = sqrt(m[0] * m[0] + m[1] * m[1] + m[2] * m[2]);
    insert = !(moved < a.min_move);
  }
  const bool carve = insert && a.carve_on && a.carve_n > 0 && *map_n > 0 && (ms[MS_NINS] % a.carve_n == 1);
  const bool dense = accepted && a.dense_on;
  const bool dcarve = dense && a.dcarve_n > 0 && (ms[MS_NDENSE] % a.dcarve_n == 1);
  ms[MS_ACCEPT] = accepted; ms[MS_INSERT] = insert; ms[MS_CARVE] = carve; ms[MS_DENSE] = dense; ms[MS_DCARVE] = dcarve;
  ms[MS_NSTEPS] += 1; ms[MS_NACCEPT] += accepted ? 1 : 0;
  if (slots) slots[gstate[1]] = *res;
}
// end of a step that fed the dense map: ++nScansInsertedDenseMap_ (Submap.cpp:90)
__global__ void mapper_post_kernel(int32_t* ms) {
  pdl_wait();
  if (threadIdx.x == 0 && ms[MS_DENSE]) ms[MS_NDENSE] += 1;
}

double nn_cell(const b2s_handle* h, double max_corr) {
  if (h->cfg.nn_cell_size > 0.0) return h->cfg.nn_cell_size;
  return max_corr * 0.25;   // box queries want cells of a few map voxels; the header kernel coarsens them if the box is huge
}

int32_t check_icp_params(const b2s_icp_params& p) {
  B2S_REQUIRE(p.reg_type == B2S_REG_POINT_TO_PLANE || p.reg_type == B2S_REG_POINT_TO_POINT || p.reg_type == B2S_REG_GENERALIZED,
              B2S_E_UNSUPPORTED, "unknown registration type %d", (int)p.reg_type);
  B2S_REQUIRE(p.max_corr_dist > 0.0, B2S_E_INVALID, "[RegistrationICP] Invalid max_correspondence_distance.");
  B2S_REQUIRE(p.max_iter >= 0, B2S_E_INVALID, "max_iter must be >= 0");
  return B2S_OK;
}

// global working copy of a source of n points (positions + per-point search state); only touched by sources too large for shared memory
size_t icp_work_bytes(size_t n) { return (n + 1) * 24 + (n + 1) * 4 + 16; }

void fill_problem(IcpProblem* P, const b2s_icp_params& icp, const b2s_cloud* src, const GridIndex* g, const b2s_cloud* tgt, const double* init_host,
                  const double* init_dev, double* work, b2s_result* out_dev) {
  memset(P, 0, sizeof(*P));
  P->src_xyz = src->xyz.as<double>();
  P->src_n = src->dn.as<int32_t>();
  P->ghdr = g->hdr.as<GridHeader>();
  P->cell_start = grid_starts(g);
  P->tgt_pts = g->pts.as<double>();
  P->tgt_nrm = tgt->has_normals ? tgt->nrm.as<double>() : nullptr;
  P->work_xyz = work;
  P->work_prev = reinterpret_cast<int32_t*>(work + 3 * (src->n_max + 1));   // callers size the work buffer with icp_work_bytes()
  P->init_dev = init_dev;
  if (init_host) memcpy(P->init, init_host, 128);
  P->max_corr = icp.max_corr_dist;
  P->rel_fitness = icp.rel_fitness;
  P->rel_rmse = icp.rel_rmse;
  P->max_iter = icp.max_iter;
  P->src_n_max = (int32_t)src->n_max;
  P->estimator = icp.reg_type;
  P->src_nrm = src->has_normals ? src->nrm.as<double>() : nullptr;
  P->gicp_eps = 1e-3;   // TransformationEstimationForGeneralizedICP() default, the object the reference holds (CloudRegistration.hpp)
  P->out = out_dev;
}

int32_t preprocess_scan(b2s_handle* h, const b2s_cloud* raw, const b2s_cropper& cropper, double voxel_size, double ratio, uint32_t seed,
                        const b2s_icp_params& icp, b2s_cloud* t0, b2s_cloud* out) {
  b2s_cropper c0 = cropper;
  c0.center[0] = c0.center[1] = c0.center[2] = 0.0;   // ScanToMapIcp's and LidarOdometry's own croppers never get a pose: sensor frame
  CropDev wide = make_crop(&c0);
  const bool has_crop = c0.kind != B2S_CROP_NONE || c0.invert;
  if (voxel_size > 0.0) B2S_TRY(op_voxel_down_sample(h, raw, has_crop ? &wide : nullptr, voxel_size, t0));
  else if (has_crop) B2S_TRY(op_crop(h, raw, wide, t0));
  else B2S_TRY(op_voxel_down_sample(h, raw, nullptr, 0.0, t0));
  static const double cell_factor = getenv("B2S_NORMALS_CELL_FACTOR") ? atof(getenv("B2S_NORMALS_CELL_FACTOR")) : 4.0;   // tuning knob: index cell = factor x voxel
  const double cell_hint = voxel_size > 0.0 ? cell_factor * voxel_size : 0.0;
  if (ratio < 1.0) {
    // reference order: normals for every voxel point, then RandomDownSample.  The selection only depends on the point
    // positions, so select first and estimate normals for the survivors only (neighbours still from the full cloud).
    B2S_REQUIRE(ratio >= 0.0, B2S_E_INVALID, "[RandomDownSample] sampling_ratio must be in [0, 1]");
    B2S_TRY(select_flags(h, t0, ratio, seed));
    B2S_TRY(op_estimate_normals(h, t0, icp.knn, icp.knn_radius, cell_hint, h->flags.as<int32_t>()));
    B2S_TRY(select_compact(h, t0, ratio, out));
  } else {
    B2S_TRY(op_estimate_normals(h, t0, icp.knn, icp.knn_radius, cell_hint));
    B2S_TRY(op_random_down_sample(h, t0, ratio, seed, out));
  }
  return B2S_OK;
}

int32_t process_scan_impl(b2s_handle* h, const b2s_cloud* raw, b2s_cloud* merge, b2s_cloud* match) {
  const b2s_scan_params& sp = h->cfg.scan;
  B2S_TRY(preprocess_scan(h, raw, sp.map_builder_cropper, sp.voxel_size, sp.downsampling_ratio, sp.seed, h->cfg.icp, h->t0.get(), merge));
  b2s_cropper c1 = sp.scan_matcher_cropper;
  c1.center[0] = c1.center[1] = c1.center[2] = 0.0;   // ScanToMapRegistration.cpp:47 setPose(Identity)
  B2S_TRY(op_crop(h, merge, make_crop(&c1), match));
  launch_pdl(empty_check_kernel, 1, 1, 0, h->stream, merge->dn.as<int32_t>(), match->dn.as<int32_t>(), h->status.as<uint32_t>());
  h->launches++;
  static const int pad = getenv("B2S_PAD_LAUNCHES") ? atoi(getenv("B2S_PAD_LAUNCHES")) : 0;
  for (int i = 0; i < pad; i++) launch_pdl(pad_kernel, 1, 32, 0, h->stream);
  return B2S_OK;
}

// ---- graph replay of the per-scan chain ---------------------------------------------------------------------------
// first node of the chain: takes the step number from a device counter, fetches that step's odometry motion from the
// host-written ring (pinned, device-mapped) and publishes the result slot of this step
__global__ void graph_begin_kernel(const double* __restrict__ ring, int32_t* gstate, double* __restrict__ odom) {
  pdl_wait();
  const int step = gstate[0];
  if (threadIdx.x < 16) odom[threadIdx.x] = ring[(step & 63) * 16 + threadIdx.x];
  __syncthreads();
  if (threadIdx.x == 0) { gstate[0] = step + 1; gstate[1] = step & 255; }
}

// what follows the registration in every variant of the chain: gates, [carving], F1, [dense map]
int32_t mapper_chain_tail(b2s_handle* h, b2s_submap* sm, const b2s_cloud* raw_scan, const b2s_cloud* merge, const b2s_result* res,
                          double min_fitness, int ignore_fitness, b2s_result* slots, const int32_t* gstate) {
  const b2s_mapper_options& o = sm->opts;
  double* pose_state = sm->pose.as<double>();
  int32_t* ms = sm->mstate.as<int32_t>();
  GateArgs ga;
  ga.min_fitness = min_fitness; ga.min_move = o.min_movement_between_mapping_steps; ga.ignore_fitness = ignore_fitness;
  ga.carve_on = o.carve_enabled; ga.carve_n = o.carve_every_n_scans; ga.dense_on = o.dense_enabled; ga.dcarve_n = o.dense_carve_every_n_scans;
  ga.merge_on = sm->merge_scans ? 1 : 0;
  launch_pdl(mapper_gate_kernel, 1, 32, 0, h->stream, res, ga, pose_state, ms, sm->cloud[0]->dn.as<int32_t>(), slots, gstate);
  h->launches++;
  if (sm->merge_scans) {   // pure localisation (merge off): the sparse map is never written, so neither kernel is launched
    if (o.carve_enabled) {   // Submap::insertScan: carve BEFORE the scan is appended, cropper still at the pose of the last insertion
      B2S_REQUIRE(o.carving.voxel_size > 0.0, B2S_E_INVALID, "carving voxel size must be > 0");
      CropDev crop = make_crop(&h->cfg.scan.map_builder_cropper, pose_state + 5 * 16);
      B2S_TRY(op_submap_carve(h, sm, raw_scan, pose_state, crop, o.carving, nullptr, ms + MS_CARVE));
    }
    B2S_TRY(op_submap_insert(h, sm, merge, pose_state, ms + MS_INSERT));                                // Mapper.cpp:174
  }
  if (o.dense_enabled) {
    if (sm->dense_cap == 0) {
      B2S_REQUIRE(h->cfg.dense_voxel_size > 0.0, B2S_E_INVALID, "dense_voxel_size must be > 0");
      B2S_TRY(dense_init(h, sm, (size_t)1 << 22, h->cfg.dense_voxel_size));
    }
    B2S_TRY(op_dense_insert(h, sm, raw_scan, nullptr, pose_state, &o.dense_cropper, ms + MS_DENSE));
    if (o.dense_carve_every_n_scans > 0)
      B2S_TRY(op_dense_carve(h, sm, raw_scan, nullptr, pose_state, o.dense_carving.neighborhood_radius_dense_map, o.dense_carving.truncation_distance,
                             o.dense_carving.max_raytracing_length, ms + MS_TMP + 1, ms + MS_DCARVE));
    launch_pdl(mapper_post_kernel, 1, 32, 0, h->stream, ms);
    h->launches++;
  }
  return B2S_OK;
}

static int32_t mapper_chain_graphable(void* ctx) {
  b2s_submap* sm = static_cast<b2s_submap*>(ctx);
  b2s_handle* h = sm->h;
  double* pose_state = sm->pose.as<double>();
  double* odom = pose_state + 32;
  double* guess = pose_state + 48;
  int32_t* gstate = sm->gstate.as<int32_t>();
  b2s_result* res = h->results.as<b2s_result>();
  double* ring_dev = nullptr;
  B2S_CUDA(cudaHostGetDevicePointer(&ring_dev, sm->odom_ring.p, 0));
  launch_pdl(graph_begin_kernel, 1, 32, 0, h->stream, ring_dev, gstate, odom);
  h->launches++;
  B2S_TRY(process_scan_impl(h, sm->staging.get(), h->t1.get(), h->t2.get()));
  launch_pdl(compose_kernel, 1, 32, 0, h->stream, pose_state, odom, guess, static_cast<const int32_t*>(sm->mstate.as<int32_t>()));
  h->launches++;
  B2S_TRY(register_to_submap_async(h, h->t2.get(), sm, nullptr, pose_state, nullptr, guess, res));
  return mapper_chain_tail(h, sm, sm->staging.get(), h->t1.get(), res, sm->g_min_fitness, sm->g_ignore_fitness, h->slots.as<b2s_result>(), gstate);
}

static std::mutex g_live_mu;
static std::unordered_set<unsigned long long> g_live_submaps;
void submap_register(unsigned long long uid) { std::lock_guard<std::mutex> lk(g_live_mu); g_live_submaps.insert(uid); }
void submap_forget(unsigned long long uid) { std::lock_guard<std::mutex> lk(g_live_mu); g_live_submaps.erase(uid); }
bool submap_alive(unsigned long long uid) { std::lock_guard<std::mutex> lk(g_live_mu); return g_live_submaps.count(uid) != 0; }

int32_t graph_drop(b2s_handle* h, GraphCache* g) {
  if (!g->exec) return B2S_OK;
  B2S_CUDA(cudaStreamSynchronize(h->stream));
  cudaGraphExecDestroy(g->exec);
  g->exec = nullptr;
  g->warm = 1;
  return B2S_OK;
}

int32_t graph_step(b2s_handle* h, GraphCache* g, unsigned long long key, int32_t (*chain)(void*), void* ctx) {
  // a device buffer was re-allocated since the capture (any call that grows a scratch buffer): the graph holds the old
  // address -- or b2s_set_config / the owner's options changed what the captured launches were built from.  This step runs
  // eagerly (which also re-sizes the scratch).
  if (g->alloc_gen != __atomic_load_n(&g_alloc_generation, __ATOMIC_RELAXED) || g->cfg_gen != h->cfg_gen || g->key != key) B2S_TRY(graph_drop(h, g));
  if (g->exec) {
    B2S_CUDA(cudaGraphLaunch(g->exec, h->stream));
    h->launches += g->kernels;
    return B2S_OK;
  }
  if (g->warm > 0) {   // eager steps size every scratch buffer (no allocation may happen during capture)
    g->warm--;
    return chain(ctx);
  }
  // capture this step's chain, instantiate, replay it
  const int64_t l0 = h->launches;
  g_capturing = true; g_capture_broken = false;
  cudaError_t ce = cudaStreamBeginCapture(h->stream, cudaStreamCaptureModeThreadLocal);
  int32_t rc = B2S_E_CUDA;
  cudaGraph_t graph = nullptr;
  if (ce == cudaSuccess) {
    rc = chain(ctx);
    ce = cudaStreamEndCapture(h->stream, &graph);
  }
  g_capturing = false;
  const int64_t captured_kernels = h->launches - l0;
  h->launches = l0;
  if (ce != cudaSuccess || rc != B2S_OK || g_capture_broken || !graph) {
    // not capturable (e.g. an unbounded cropper needs a host round trip): stay eager for good
    if (graph) cudaGraphDestroy(graph);
    cudaGetLastError();
    g->warm = 1 << 30;
    return chain(ctx);
  }
  ce = cudaGraphInstantiate(&g->exec, graph, 0);
  cudaGraphDestroy(graph);
  if (ce != cudaSuccess) { g->exec = nullptr; g->warm = 1 << 30; cudaGetLastError(); return chain(ctx); }
  g->kernels = captured_kernels;
  h->captures++;
  g->alloc_gen = __atomic_load_n(&g_alloc_generation, __ATOMIC_RELAXED);
  g->cfg_gen = h->cfg_gen;
  g->key = key;
  B2S_CUDA(cudaGraphLaunch(g->exec, h->stream));
  h->launches += g->kernels;
  return B2S_OK;
}

static int32_t mapper_step_graph(b2s_handle* h, b2s_submap* sm, const b2s_cloud* raw_scan, const double* odometry_motion, int32_t slot) {
  B2S_REQUIRE(raw_scan == sm->staging.get(), B2S_E_INVALID, "graph mode: the scan must be uploaded into the staging cloud of b2s_mapper_graph_enable");
  B2S_REQUIRE(slot == (int32_t)(sm->host_step & 255), B2S_E_INVALID, "graph mode: slot must be (step count %% 256) = %d", (int)(sm->host_step & 255));
  B2S_TRY(h->results.ensure(sizeof(b2s_result), h->stream));
  // the odometry ring has 64 entries and the host may run ahead of the device: never by more than 32 steps
  if ((sm->host_step & 31) == 0) B2S_CUDA(cudaStreamSynchronize(h->stream));
  memcpy(sm->odom_ring.as<double>() + (sm->host_step & 63) * 16, odometry_motion, 128);   // read by graph_begin_kernel of this step
  sm->host_step++;
  return graph_step(h, &sm->graph, 0, mapper_chain_graphable, sm);
}

// A cloud of `capacity` points and count 0 on h's device.  normals: allocate the normals too.  fixed: n_max stays at the capacity
// (graph replay needs constant launch dimensions).  tracked = false for clouds the caller owns: a captured graph never holds them.
static int32_t make_cloud(b2s_handle* h, size_t capacity, bool normals, bool fixed, bool tracked, b2s_cloud** out) {
  return create_object(out, [&](b2s_cloud* c) -> int32_t {
    c->h = h;
    c->device = h->device;
    c->xyz.tracked = c->nrm.tracked = c->dn.tracked = tracked;
    if (fixed) c->fixed_cap = capacity;
    B2S_TRY(cloud_reserve(h, c, capacity, normals));
    return cloud_set_count(h, c, 0);
  });
}
// the same for a cloud the handle or a submap owns (tracked: its buffers may be captured in a graph)
int32_t make_cloud(b2s_handle* h, size_t capacity, bool normals, bool fixed, std::unique_ptr<b2s_cloud>* out) {
  b2s_cloud* c = nullptr;
  B2S_TRY(make_cloud(h, capacity, normals, fixed, true, &c));
  out->reset(c);
  return B2S_OK;
}

}  // namespace b2s

extern "C" {

void b2s_default_config(b2s_config* cfg) {
  memset(cfg, 0, sizeof(*cfg));
  cfg->icp.reg_type = B2S_REG_POINT_TO_PLANE;
  cfg->icp.max_iter = 50; cfg->icp.max_corr_dist = 1.0; cfg->icp.knn = 20; cfg->icp.knn_radius = 3.0;
  cfg->icp.rel_fitness = 1e-6; cfg->icp.rel_rmse = 1e-6;
  cfg->scan.voxel_size = 0.1; cfg->scan.downsampling_ratio = 0.3; cfg->scan.seed = 0;
  b2s_cropper c;
  memset(&c, 0, sizeof(c));
  c.kind = B2S_CROP_MINMAX_RADIUS; c.rmin = 2.0; c.rmax = 30.0; c.zmin = -50.0; c.zmax = 50.0;
  cfg->scan.map_builder_cropper = c;
  cfg->scan.scan_matcher_cropper = c;
  cfg->map_voxel_size = 0.1;
  cfg->dense_voxel_size = 0.05;
  cfg->nn_cell_size = 0.0;
  cfg->icp_cluster_ctas = 0;
  cfg->reserved_ = 0;
}

const char* b2s_last_error(void) { return get_error(); }
const char* b2s_version(void) { return "b2s 0.1 (sm_90a, fp64)"; }
int32_t b2s_device_count(void) { int n = 0; if (cudaGetDeviceCount(&n) != cudaSuccess) return 0; return n; }
int64_t b2s_launch_count(const b2s_handle* h) { return h ? h->launches : 0; }
int64_t b2s_graph_capture_count(const b2s_handle* h) { return h ? h->captures : 0; }

int32_t b2s_create(const b2s_config* cfg, int32_t device, void* cuda_stream_or_null, b2s_handle** out) {
  B2S_REQUIRE(out != nullptr, B2S_E_INVALID, "b2s_create: out is null");
  int ndev = 0;
  B2S_CUDA(cudaGetDeviceCount(&ndev));
  B2S_REQUIRE(ndev > 0, B2S_E_CUDA, "no CUDA device visible: the b2s engine has no CPU fallback");
  B2S_REQUIRE(device >= 0 && device < ndev, B2S_E_INVALID, "device %d out of range (%d visible)", device, ndev);
  B2S_CUDA(cudaSetDevice(device));
  return create_object(out, [&](b2s_handle* h) -> int32_t {
    h->device = device;
    if (cfg) h->cfg = *cfg; else b2s_default_config(&h->cfg);
    if (cuda_stream_or_null) h->stream = (cudaStream_t)cuda_stream_or_null;
    else { B2S_CUDA(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking)); h->own_stream = true; }
    B2S_TRY(h->status.ensure(64, h->stream));
    B2S_CUDA(cudaMemsetAsync(h->status.p, 0, 64, h->stream));
    B2S_TRY(h->poses.ensure(64 * 16 * 8, h->stream));
    B2S_TRY(h->slots.ensure(256 * sizeof(b2s_result), h->stream));
    B2S_CUDA(cudaMemsetAsync(h->slots.p, 0, 256 * sizeof(b2s_result), h->stream));
    for (std::unique_ptr<b2s_cloud>* t : {&h->t0, &h->t1, &h->t2, &h->t3}) B2S_TRY(make_cloud(h, 1, true, false, t));
    return B2S_OK;
  });
}

void b2s_destroy(b2s_handle* h) {
  if (!h) return;
  cudaSetDevice(h->device);
  if (h->stream) cudaStreamSynchronize(h->stream);
  delete h;
}

int32_t b2s_set_config(b2s_handle* h, const b2s_config* cfg) {
  B2S_REQUIRE(h && cfg, B2S_E_INVALID, "null argument");
  LOCK(h);
  h->cfg = *cfg;
  h->cfg_gen++;
  return B2S_OK;
}

int32_t b2s_profile_enable(b2s_handle* h, int32_t on) {
  B2S_REQUIRE(h, B2S_E_INVALID, "null handle");
  LOCK(h);
  h->prof_enabled = on != 0;
  return B2S_OK;
}

int32_t b2s_profile_read(b2s_handle* h, double* ms_by_kind, int64_t* count_by_kind, int32_t n_kinds) {
  B2S_REQUIRE(h && ms_by_kind && count_by_kind && n_kinds >= PK_COUNT, B2S_E_INVALID, "bad argument");
  LOCK(h);
  B2S_CUDA(cudaStreamSynchronize(h->stream));
  for (int k = 0; k < n_kinds; k++) { ms_by_kind[k] = 0.0; count_by_kind[k] = 0; }
  for (auto& r : h->prof_recs) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, r.a, r.b) == cudaSuccess) { ms_by_kind[r.kind] += (double)ms; count_by_kind[r.kind]++; }
    h->prof_pool.push_back(r.a); h->prof_pool.push_back(r.b);
  }
  h->prof_recs.clear();
  return B2S_OK;
}

// debug aid: clock64 stamps {start, search end, reduce end, solve end} of up to 64 evaluations of the next registrations
int32_t b2s_debug_icp_clocks(b2s_handle* h, int32_t enable, long long* out_1024) {
  B2S_REQUIRE(h, B2S_E_INVALID, "null handle");
  LOCK(h);
  if (enable && !h->icp_dbg.p) { B2S_TRY(h->icp_dbg.ensure(1024 * 8, h->stream)); B2S_CUDA(cudaMemset(h->icp_dbg.p, 0, 1024 * 8)); }
  if (h->icp_dbg.p && out_1024) {
    B2S_CUDA(cudaStreamSynchronize(h->stream));
    B2S_CUDA(cudaMemcpy(out_1024, h->icp_dbg.p, 1024 * 8, cudaMemcpyDeviceToHost));
  }
  if (h->icp_dbg.p) B2S_CUDA(cudaMemsetAsync(h->icp_dbg.p, 0, 1024 * 8, h->stream));
  if (!enable) h->icp_dbg.release();   // icp_launch passes nullptr again
  return B2S_OK;
}

int32_t b2s_synchronize(b2s_handle* h) {
  B2S_REQUIRE(h, B2S_E_INVALID, "null handle");
  LOCK(h);
  return check_status(h);
}

// ---- clouds ----------------------------------------------------------------------------------------------------------
int32_t b2s_cloud_create(b2s_handle* h, b2s_cloud** out) {
  B2S_REQUIRE(h && out, B2S_E_INVALID, "null argument");
  LOCK(h);
  return make_cloud(h, 1, false, false, false, out);
}

void b2s_cloud_destroy(b2s_cloud* c) { destroy_object(c); }

int32_t b2s_cloud_upload_f64(b2s_handle* h, b2s_cloud* c, const double* xyz, const double* normals, size_t n) {
  B2S_REQUIRE(h && c && (xyz || n == 0), B2S_E_INVALID, "null argument");
  B2S_REQUIRE(n < (size_t)0x7fffffff / 4, B2S_E_INVALID, "cloud too large");
  LOCK(h);
  B2S_TRY(cloud_reserve(h, c, n, normals != nullptr));
  if (n) B2S_CUDA(cudaMemcpyAsync(c->xyz.p, xyz, n * 24, cudaMemcpyHostToDevice, h->stream));
  if (n && normals) B2S_CUDA(cudaMemcpyAsync(c->nrm.p, normals, n * 24, cudaMemcpyHostToDevice, h->stream));
  c->has_normals = normals != nullptr;
  return cloud_set_count(h, c, n);
}

int32_t b2s_cloud_upload_f32(b2s_handle* h, b2s_cloud* c, const void* xyz, size_t n, size_t stride_bytes) {
  B2S_REQUIRE(h && c && (xyz || n == 0), B2S_E_INVALID, "null argument");
  B2S_REQUIRE(stride_bytes >= 12 && stride_bytes % 4 == 0, B2S_E_INVALID, "stride must be a multiple of 4 and >= 12");
  B2S_REQUIRE(n < (size_t)0x7fffffff / 4, B2S_E_INVALID, "cloud too large");
  LOCK(h);
  B2S_TRY(cloud_reserve(h, c, n, false));
  B2S_TRY(h->tmp_f64.ensure(n * stride_bytes + 16, h->stream));
  if (n) {
    B2S_CUDA(cudaMemcpyAsync(h->tmp_f64.p, xyz, n * stride_bytes, cudaMemcpyHostToDevice, h->stream));
    launch_pdl(f32_to_f64_kernel, grid_for(n, 256), 256, 0, h->stream, h->tmp_f64.as<unsigned char>(), stride_bytes, (int)n, c->xyz.as<double>());
    h->launches++;
  }
  c->has_normals = false;
  return cloud_set_count(h, c, n);
}

static int32_t cloud_count_sync(b2s_handle* h, const b2s_cloud* c, size_t* n) {
  if (c->n_known >= 0) { *n = (size_t)c->n_known; return B2S_OK; }
  int32_t v = 0;
  B2S_CUDA(cudaMemcpyAsync(&v, c->dn.p, 4, cudaMemcpyDeviceToHost, h->stream));
  B2S_CUDA(cudaStreamSynchronize(h->stream));
  *n = (size_t)v;
  const_cast<b2s_cloud*>(c)->n_known = v;
  return B2S_OK;
}

int32_t b2s_cloud_size(b2s_handle* h, const b2s_cloud* c, size_t* n, int32_t* has_normals) {
  B2S_REQUIRE(h && c && n, B2S_E_INVALID, "null argument");
  LOCK(h);
  B2S_TRY(cloud_count_sync(h, c, n));
  if (has_normals) *has_normals = c->has_normals ? 1 : 0;
  return B2S_OK;
}

int32_t b2s_cloud_download(b2s_handle* h, const b2s_cloud* c, double* xyz, double* normals, size_t capacity, size_t* n_out) {
  B2S_REQUIRE(h && c, B2S_E_INVALID, "null argument");
  LOCK(h);
  size_t n = 0;
  B2S_TRY(cloud_count_sync(h, c, &n));
  if (n_out) *n_out = n;
  B2S_REQUIRE(n <= capacity, B2S_E_CAPACITY, "download buffer too small: %zu points, capacity %zu", n, capacity);
  if (n && xyz) B2S_CUDA(cudaMemcpyAsync(xyz, c->xyz.p, n * 24, cudaMemcpyDeviceToHost, h->stream));
  if (n && normals) {
    B2S_REQUIRE(c->has_normals, B2S_E_NO_NORMALS, "cloud has no normals");
    B2S_CUDA(cudaMemcpyAsync(normals, c->nrm.p, n * 24, cudaMemcpyDeviceToHost, h->stream));
  }
  return check_status(h);
}

int32_t b2s_cloud_export_device(b2s_handle* h, const b2s_cloud* c, void* xyz_dev, void* normals_dev, size_t capacity, size_t* n_out) {
  B2S_REQUIRE(h && c && xyz_dev, B2S_E_INVALID, "null argument");
  LOCK(h);
  size_t n = 0;
  B2S_TRY(cloud_count_sync(h, c, &n));
  if (n_out) *n_out = n;
  B2S_REQUIRE(n <= capacity, B2S_E_CAPACITY, "device buffer too small: %zu points, capacity %zu", n, capacity);
  if (n) B2S_CUDA(cudaMemcpyAsync(xyz_dev, c->xyz.p, n * 24, cudaMemcpyDeviceToDevice, h->stream));
  if (n && normals_dev) {
    B2S_REQUIRE(c->has_normals, B2S_E_NO_NORMALS, "cloud has no normals");
    B2S_CUDA(cudaMemcpyAsync(normals_dev, c->nrm.p, n * 24, cudaMemcpyDeviceToDevice, h->stream));
  }
  return check_status(h);
}

int32_t b2s_cloud_import_device(b2s_handle* h, b2s_cloud* c, const void* xyz_dev, const void* normals_dev, size_t n) {
  B2S_REQUIRE(h && c && (xyz_dev || n == 0), B2S_E_INVALID, "null argument");
  B2S_REQUIRE(n < (size_t)0x7fffffff / 4, B2S_E_INVALID, "cloud too large");
  LOCK(h);
  B2S_TRY(cloud_reserve(h, c, n, normals_dev != nullptr));
  if (n) B2S_CUDA(cudaMemcpyAsync(c->xyz.p, xyz_dev, n * 24, cudaMemcpyDeviceToDevice, h->stream));
  if (n && normals_dev) B2S_CUDA(cudaMemcpyAsync(c->nrm.p, normals_dev, n * 24, cudaMemcpyDeviceToDevice, h->stream));
  c->has_normals = normals_dev != nullptr;
  return cloud_set_count(h, c, n);
}

int32_t b2s_cloud_copy(b2s_handle* h, const b2s_cloud* src, b2s_cloud* dst) {
  B2S_REQUIRE(h && src && dst, B2S_E_INVALID, "null argument");
  LOCK(h);
  B2S_REQUIRE(!dst->fixed_cap || src->n_max <= dst->fixed_cap, B2S_E_CAPACITY, "cloud larger than the fixed capacity of the destination");
  B2S_TRY(op_voxel_down_sample(h, src, nullptr, 0.0, dst));
  if (dst->fixed_cap) dst->n_max = dst->fixed_cap;
  return B2S_OK;
}

// ---- stages ----------------------------------------------------------------------------------------------------------
int32_t b2s_crop(b2s_handle* h, const b2s_cloud* in, const b2s_cropper* cropper, b2s_cloud* out) {
  B2S_REQUIRE(h && in && cropper && out && in != out, B2S_E_INVALID, "bad argument");
  LOCK(h);
  WideGridScope wide(in->n_max);
  return op_crop(h, in, make_crop(cropper), out);
}

int32_t b2s_voxel_down_sample(b2s_handle* h, const b2s_cloud* in, double voxel_size, b2s_cloud* out) {
  B2S_REQUIRE(h && in && out && in != out, B2S_E_INVALID, "bad argument");
  LOCK(h);
  WideGridScope wide(in->n_max);
  return op_voxel_down_sample(h, in, nullptr, voxel_size, out);
}

int32_t b2s_estimate_normals(b2s_handle* h, b2s_cloud* cloud, int32_t knn, double radius) {
  B2S_REQUIRE(h && cloud, B2S_E_INVALID, "null argument");
  LOCK(h);
  WideGridScope wide(cloud->n_max);
  return op_estimate_normals(h, cloud, knn, radius, h->cfg.scan.voxel_size > 0.0 ? 4.0 * h->cfg.scan.voxel_size : 0.0);
}

int32_t b2s_random_down_sample(b2s_handle* h, const b2s_cloud* in, double ratio, uint32_t seed, b2s_cloud* out) {
  B2S_REQUIRE(h && in && out && in != out, B2S_E_INVALID, "bad argument");
  LOCK(h);
  WideGridScope wide(in->n_max);
  return op_random_down_sample(h, in, ratio, seed, out);
}

int32_t b2s_transform(b2s_handle* h, const b2s_cloud* in, const double T[16], b2s_cloud* out) {
  B2S_REQUIRE(h && in && out && T && in != out, B2S_E_INVALID, "bad argument");
  LOCK(h);
  return op_transform(h, in, T, out);
}

int32_t b2s_process_scan(b2s_handle* h, const b2s_cloud* raw, b2s_cloud* merge, b2s_cloud* match) {
  B2S_REQUIRE(h && raw && merge && match && merge != match && raw != merge && raw != match, B2S_E_INVALID, "bad argument");
  LOCK(h);
  return process_scan_impl(h, raw, merge, match);
}

int32_t b2s_register(b2s_handle* h, const b2s_cloud* source, const b2s_cloud* target, const double init[16], b2s_result* out) {
  B2S_REQUIRE(h && source && target && init && out, B2S_E_INVALID, "null argument");
  LOCK(h);
  B2S_TRY(check_icp_params(h->cfg.icp));
  B2S_REQUIRE(target->has_normals || h->cfg.icp.reg_type == B2S_REG_POINT_TO_POINT, B2S_E_NO_NORMALS,
              "[RegistrationICP] TransformationEstimationPointToPlane requires target normals");
  B2S_REQUIRE(source->has_normals || h->cfg.icp.reg_type != B2S_REG_GENERALIZED, B2S_E_NO_NORMALS,
              "GeneralizedIcp on the device derives the covariances from normals: call estimateNormalsOrCovariancesIfNeeded on both clouds");
  B2S_TRY(grid_build(h, &h->grid_a, target, nn_cell(h, h->cfg.icp.max_corr_dist), nullptr));
  B2S_TRY(h->work_xyz.ensure(icp_work_bytes(source->n_max), h->stream));
  B2S_TRY(h->problems.ensure(sizeof(IcpProblem), h->stream));
  B2S_TRY(h->results.ensure(sizeof(b2s_result), h->stream));
  IcpProblem P;
  fill_problem(&P, h->cfg.icp, source, &h->grid_a, target, init, nullptr, h->work_xyz.as<double>(), h->results.as<b2s_result>());
  B2S_TRY(icp_launch(h, &P, nullptr, 1, source->n_max));
  B2S_CUDA(cudaMemcpyAsync(out, h->results.p, sizeof(b2s_result), cudaMemcpyDeviceToHost, h->stream));
  return check_status(h);
}

int32_t b2s_register_batch(b2s_handle* h, int32_t n, const b2s_cloud* const* sources, const b2s_cloud* const* targets, const double* inits,
                           b2s_result* out) {
  B2S_REQUIRE(h && sources && targets && inits && out && n >= 0, B2S_E_INVALID, "bad argument");
  if (n == 0) return B2S_OK;
  LOCK(h);
  B2S_TRY(check_icp_params(h->cfg.icp));
  std::vector<IcpProblem> probs((size_t)n);
  std::vector<const b2s_cloud*> seen;  // targets shared by several pairs are indexed once
  std::vector<GridIndex*> grids;       // seen[k]'s index
  std::vector<int> grid_of((size_t)n);
  size_t work_total = 0, max_src = 0;
  for (int i = 0; i < n; i++) {
    B2S_REQUIRE(sources[i] && targets[i], B2S_E_INVALID, "null cloud in batch");
    B2S_REQUIRE(targets[i]->has_normals || h->cfg.icp.reg_type == B2S_REG_POINT_TO_POINT, B2S_E_NO_NORMALS,
                "[RegistrationICP] target %d has no normals", i);
    B2S_REQUIRE(sources[i]->has_normals || h->cfg.icp.reg_type != B2S_REG_GENERALIZED, B2S_E_NO_NORMALS, "GeneralizedIcp: source %d has no normals", i);
    int gi = -1;
    for (size_t k = 0; k < seen.size(); k++) if (seen[k] == targets[i]) { gi = (int)k; break; }
    if (gi < 0) {
      gi = (int)seen.size();
      seen.push_back(targets[i]);
      if (h->batch_grids.size() <= (size_t)gi) h->batch_grids.push_back(std::make_unique<GridIndex>());
      grids.push_back(h->batch_grids[gi].get());
    }
    grid_of[i] = gi;
    work_total += (icp_work_bytes(sources[i]->n_max) + 7) / 8;   // in doubles
    if (sources[i]->n_max > max_src) max_src = sources[i]->n_max;
  }
  // R2 for every distinct target in one set of launches (blockIdx.y = target)
  B2S_TRY(grid_build_batch(h, grids.data(), seen.data(), (int)seen.size(), nn_cell(h, h->cfg.icp.max_corr_dist)));
  B2S_TRY(h->work_xyz.ensure(work_total * 8, h->stream));
  B2S_TRY(h->problems.ensure(sizeof(IcpProblem) * (size_t)n, h->stream));
  B2S_TRY(h->results.ensure(sizeof(b2s_result) * (size_t)n, h->stream));
  size_t woff = 0;
  for (int i = 0; i < n; i++) {
    fill_problem(&probs[i], h->cfg.icp, sources[i], grids[grid_of[i]], targets[i], inits + 16 * (size_t)i, nullptr, h->work_xyz.as<double>() + woff,
                 h->results.as<b2s_result>() + i);
    woff += (icp_work_bytes(sources[i]->n_max) + 7) / 8;
  }
  B2S_CUDA(cudaMemcpyAsync(h->problems.p, probs.data(), sizeof(IcpProblem) * (size_t)n, cudaMemcpyHostToDevice, h->stream));
  B2S_CUDA(cudaStreamSynchronize(h->stream));  // probs lives on the host stack frame
  B2S_TRY(icp_launch(h, nullptr, h->problems.as<IcpProblem>(), n, max_src));
  B2S_CUDA(cudaMemcpyAsync(out, h->results.p, sizeof(b2s_result) * (size_t)n, cudaMemcpyDeviceToHost, h->stream));
  return check_status(h);
}

int32_t b2s_dense_carve(b2s_handle* h, b2s_submap* sm, const b2s_cloud* scan, const double sensor[3], const b2s_carving_params* prm, size_t* n_removed) {
  B2S_REQUIRE(h && sm && scan && sensor && prm, B2S_E_INVALID, "null argument");
  LOCK(h);
  if (sm->dense_cap == 0) { if (n_removed) *n_removed = 0; return B2S_OK; }   // cloud->empty(): nothing to carve (Submap.cpp:127)
  int32_t* removed_dev = reinterpret_cast<int32_t*>(h->status.as<uint32_t>() + SW_REMOVED);
  B2S_TRY(op_dense_carve(h, sm, scan, sensor, nullptr, prm->neighborhood_radius_dense_map, prm->truncation_distance, prm->max_raytracing_length, removed_dev));
  if (!n_removed) return B2S_OK;
  int32_t removed = 0;
  const int32_t rc = read_back(h, {{&removed, removed_dev, 4}});
  *n_removed = (size_t)removed;
  return rc;
}

int32_t b2s_dense_query(b2s_handle* h, const b2s_submap* sm, const b2s_cloud* points, int32_t* counts, double* means_xyz, size_t capacity) {
  B2S_REQUIRE(h && sm && points && counts, B2S_E_INVALID, "null argument");
  LOCK(h);
  size_t n = 0;
  B2S_TRY(cloud_count_sync(h, points, &n));
  B2S_REQUIRE(n <= capacity, B2S_E_CAPACITY, "output arrays hold %zu entries, the cloud has %zu points", capacity, n);
  if (n == 0) return B2S_OK;
  B2S_TRY(h->tmp_i32.ensure((n + 64) * 4, h->stream));
  if (means_xyz) B2S_TRY(h->tmp_f64.ensure((n + 1) * 24, h->stream));
  B2S_TRY(op_dense_query(h, sm, points, h->tmp_i32.as<int32_t>(), means_xyz ? h->tmp_f64.as<double>() : nullptr));
  B2S_CUDA(cudaMemcpyAsync(counts, h->tmp_i32.p, n * 4, cudaMemcpyDeviceToHost, h->stream));
  if (means_xyz) B2S_CUDA(cudaMemcpyAsync(means_xyz, h->tmp_f64.p, n * 24, cudaMemcpyDeviceToHost, h->stream));
  return check_status(h);
}

int32_t b2s_dense_remove(b2s_handle* h, b2s_submap* sm, const b2s_cloud* points) {
  B2S_REQUIRE(h && sm && points, B2S_E_INVALID, "null argument");
  LOCK(h);
  return op_dense_remove(h, sm, points);
}

int32_t b2s_dense_size(b2s_handle* h, const b2s_submap* sm, size_t* n_voxels) {
  B2S_REQUIRE(h && sm && n_voxels, B2S_E_INVALID, "null argument");
  LOCK(h);
  int32_t* d = reinterpret_cast<int32_t*>(h->status.as<uint32_t>() + SW_DENSE_SIZE);
  B2S_TRY(op_dense_count(h, sm, d));
  int32_t count = 0;
  const int32_t rc = read_back(h, {{&count, d, 4}});
  *n_voxels = (size_t)count;
  return rc;
}

int32_t b2s_dense_clear(b2s_handle* h, b2s_submap* sm) {
  B2S_REQUIRE(h && sm, B2S_E_INVALID, "null argument");
  LOCK(h);
  if (sm->dense_cap == 0) return B2S_OK;
  return dense_init(h, sm, sm->dense_cap, sm->dense_voxel);
}

int32_t b2s_undistort(b2s_handle* h, const b2s_cloud* in, const double lin_vel[3], const double ang_vel_rpy[3], double scan_duration,
                      int32_t clockwise, b2s_cloud* out) {
  B2S_REQUIRE(h && in && out && lin_vel && ang_vel_rpy && in != out, B2S_E_INVALID, "bad argument");
  B2S_REQUIRE(scan_duration > 0.0, B2S_E_INVALID, "lidar scanDuration_: must be > 0");   // assert_gt at MotionCompensation.cpp:61
  LOCK(h);
  return op_undistort(h, in, lin_vel, ang_vel_rpy, scan_duration, clockwise ? 1 : 0, out);
}

int32_t b2s_overlap(b2s_handle* h, const b2s_cloud* source, const b2s_cloud* target, const double T[16], double voxel, int32_t min_pts,
                    b2s_cloud* source_overlap, b2s_cloud* target_overlap) {
  B2S_REQUIRE(h && source && target && T && source_overlap && target_overlap, B2S_E_INVALID, "null argument");
  B2S_REQUIRE(source_overlap != target_overlap && source_overlap != source && target_overlap != target, B2S_E_INVALID, "aliased clouds");
  B2S_REQUIRE(voxel > 0.0, B2S_E_INVALID, "voxel size must be > 0");
  B2S_REQUIRE(min_pts >= 1, B2S_E_INVALID, "minNumPointsPerVoxel must be >= 1");   // assert_ge at helpers.cpp:310
  LOCK(h);
  double* Td = h->poses.as<double>() + 16 * PS_CALL;
  B2S_TRY(pose_to_device(h, T, Td));
  return op_overlap(h, source, target, Td, voxel, min_pts, source_overlap, target_overlap);
}

int32_t b2s_information_matrix(b2s_handle* h, const b2s_cloud* source, const b2s_cloud* target, double max_corr, const double T[16],
                               double info_out[36]) {
  B2S_REQUIRE(h && source && target && T && info_out, B2S_E_INVALID, "null argument");
  B2S_REQUIRE(max_corr > 0.0, B2S_E_INVALID, "[GetInformationMatrixFromPointClouds] Invalid max_correspondence_distance.");
  LOCK(h);
  B2S_TRY(grid_build(h, &h->grid_a, target, max_corr * 0.25, nullptr));
  B2S_TRY(h->work_xyz.ensure(icp_work_bytes(source->n_max), h->stream));
  B2S_TRY(h->results.ensure(sizeof(b2s_result) + 36 * 8 + 64, h->stream));
  IcpProblem P;
  fill_problem(&P, h->cfg.icp, source, &h->grid_a, target, T, nullptr, h->work_xyz.as<double>(), h->results.as<b2s_result>());
  P.max_corr = max_corr;
  P.max_iter = 0;
  P.estimator = EST_INFORMATION;
  P.info_out = reinterpret_cast<double*>(h->results.as<b2s_result>() + 1);
  B2S_TRY(icp_launch(h, &P, nullptr, 1, source->n_max));
  B2S_CUDA(cudaMemcpyAsync(info_out, P.info_out, 36 * 8, cudaMemcpyDeviceToHost, h->stream));
  return check_status(h);
}

int32_t b2s_nearest_neighbors(b2s_handle* h, const b2s_cloud* queries, const b2s_cloud* target, double max_corr, const double T[16], int32_t* index_out,
                              double* d2_out, size_t capacity, size_t* n_queries) {
  B2S_REQUIRE(h && queries && target && index_out, B2S_E_INVALID, "null argument");
  B2S_REQUIRE(max_corr > 0.0, B2S_E_INVALID, "[RegistrationICP] Invalid max_correspondence_distance.");
  LOCK(h);
  size_t n = 0;
  B2S_TRY(cloud_count_sync(h, queries, &n));
  if (n_queries) *n_queries = n;
  B2S_REQUIRE(n <= capacity, B2S_E_CAPACITY, "output arrays hold %zu entries, the cloud has %zu points", capacity, n);
  if (n == 0) return B2S_OK;
  B2S_TRY(grid_build(h, &h->grid_a, target, nn_cell(h, max_corr), nullptr));
  constexpr size_t CHUNK = 36864;   // what one launch keeps in shared memory (8 CTAs x 72 tiles of 64 points at 40 bytes per point)
  B2S_TRY(h->work_xyz.ensure(icp_work_bytes(CHUNK), h->stream));
  B2S_TRY(h->results.ensure(sizeof(b2s_result) + 36 * 8 + 64, h->stream));
  B2S_TRY(h->tmp_i32.ensure((n + 64) * 4, h->stream));
  B2S_TRY(h->tmp_f64.ensure((n + 1) * 8, h->stream));
  const double I[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  int32_t* d_cnt = reinterpret_cast<int32_t*>(h->status.as<uint32_t>() + SW_NN_CHUNK);
  for (size_t off = 0; off < n; off += CHUNK) {
    const size_t cnt = n - off < CHUNK ? n - off : CHUNK;
    launch_pdl(write_i32_kernel, 1, 1, 0, h->stream, d_cnt, (int32_t)cnt);
    h->launches++;
    IcpProblem P;
    fill_problem(&P, h->cfg.icp, queries, &h->grid_a, target, T ? T : I, nullptr, h->work_xyz.as<double>(), h->results.as<b2s_result>());
    P.src_xyz = queries->xyz.as<double>() + 3 * off;
    P.work_prev = reinterpret_cast<int32_t*>(h->work_xyz.as<double>() + 3 * (CHUNK + 1));   // the work buffer is sized for a chunk, not for the cloud
    P.src_n = d_cnt;
    P.max_corr = max_corr;
    P.max_iter = 0;
    P.estimator = EST_CORRESPONDENCES;
    P.info_out = nullptr;
    P.src_n_max = (int32_t)cnt;
    P.corr_index = h->tmp_i32.as<int32_t>() + off;
    P.corr_d2 = h->tmp_f64.as<double>() + off;
    B2S_TRY(icp_launch(h, &P, nullptr, 1, cnt));
  }
  B2S_CUDA(cudaMemcpyAsync(index_out, h->tmp_i32.p, n * 4, cudaMemcpyDeviceToHost, h->stream));
  if (d2_out) B2S_CUDA(cudaMemcpyAsync(d2_out, h->tmp_f64.p, n * 8, cudaMemcpyDeviceToHost, h->stream));
  return check_status(h);
}

int32_t b2s_register_host(b2s_handle* h, const double* src_xyz, size_t n_src, const double* tgt_xyz, const double* tgt_normals, size_t n_tgt,
                          const double init[16], b2s_result* out) {
  B2S_REQUIRE(h && init && out, B2S_E_INVALID, "null argument");
  B2S_REQUIRE(tgt_normals != nullptr || h->cfg.icp.reg_type != B2S_REG_POINT_TO_PLANE, B2S_E_NO_NORMALS,
              "[RegistrationICP] TransformationEstimationPointToPlane requires target normals");
  LOCK(h);   // held across the three calls (recursive mutex): another thread cannot touch t2 / t3 in between
  B2S_TRY(b2s_cloud_upload_f64(h, h->t2.get(), src_xyz, nullptr, n_src));
  B2S_TRY(b2s_cloud_upload_f64(h, h->t3.get(), tgt_xyz, tgt_normals, n_tgt));
  return b2s_register(h, h->t2.get(), h->t3.get(), init, out);
}

// ---- submap ----------------------------------------------------------------------------------------------------------
int32_t b2s_submap_create(b2s_handle* h, size_t capacity_points, b2s_submap** out) {
  B2S_REQUIRE(h && out && capacity_points > 0, B2S_E_INVALID, "bad argument");
  LOCK(h);
  static unsigned long long next_uid = 0;
  return create_object(out, [&](b2s_submap* sm) -> int32_t {
    sm->h = h;
    sm->device = h->device;
    sm->uid = __atomic_add_fetch(&next_uid, 1ull, __ATOMIC_RELAXED);
    submap_register(sm->uid);
    sm->capacity = capacity_points;
    for (std::unique_ptr<b2s_cloud>& c : sm->cloud) {
      B2S_TRY(make_cloud(h, capacity_points, true, false, &c));
      c->has_normals = true;
    }
    // pose slots: [0] mapToRangeSensor_, [1] pose of a host-driven insertion, [2] odometry motion, [3] initial guess, [4] carving pose,
    //             [5] pose of the last insertion (= mapToRangeSensorLastScanInsertion_ = mapBuilderCropper_'s pose; Identity before the first)
    B2S_TRY(sm->pose.ensure(8 * 16 * 8, h->stream));
    const double I[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    B2S_TRY(pose_to_device(h, I, sm->pose.as<double>()));
    B2S_TRY(pose_to_device(h, I, sm->pose.as<double>() + 5 * 16));
    B2S_TRY(sm->mstate.ensure(MS_WORDS * 4, h->stream));
    B2S_CUDA(cudaMemsetAsync(sm->mstate.p, 0, MS_WORDS * 4, h->stream));
    b2s_default_mapper_options(&sm->opts);
    return B2S_OK;
  });
}

void b2s_submap_destroy(b2s_submap* sm) { destroy_object(sm); }

int32_t b2s_submap_set_pose(b2s_handle* h, b2s_submap* sm, const double T[16]) {
  B2S_REQUIRE(h && sm && T, B2S_E_INVALID, "null argument");
  LOCK(h);
  return pose_to_device(h, T, sm->pose.as<double>());
}

int32_t b2s_cloud_transform_inplace(b2s_handle* h, b2s_cloud* c, const double T[16]) {
  B2S_REQUIRE(h && c && T, B2S_E_INVALID, "null argument");
  B2S_REQUIRE(c->h == h, B2S_E_INVALID, "the cloud belongs to another handle");
  LOCK(h);
  return op_cloud_transform(h, c, T);
}

int32_t b2s_submap_transform(b2s_handle* h, b2s_submap* sm, const double T[16]) {
  B2S_REQUIRE(h && sm && T, B2S_E_INVALID, "null argument");
  LOCK(h);
  B2S_TRY(tile_drop(h, sm));
  return op_submap_transform(h, sm, T);
}

int32_t b2s_submap_get_pose(b2s_handle* h, const b2s_submap* sm, double T[16]) {
  B2S_REQUIRE(h && sm && T, B2S_E_INVALID, "null argument");
  LOCK(h);
  B2S_CUDA(cudaMemcpyAsync(T, sm->pose.p, 128, cudaMemcpyDeviceToHost, h->stream));
  return check_status(h);
}

int32_t b2s_submap_insert(b2s_handle* h, b2s_submap* sm, const b2s_cloud* scan, const double T[16]) {
  B2S_REQUIRE(h && sm && scan && T, B2S_E_INVALID, "null argument");
  LOCK(h);
  B2S_TRY(tile_drop(h, sm));
  double* Td = sm->pose.as<double>() + 16;  // slot 1: pose used by this insertion
  B2S_TRY(pose_to_device(h, T, Td));
  return op_submap_insert(h, sm, scan, Td, nullptr);
}

int32_t b2s_submap_carve(b2s_handle* h, b2s_submap* sm, const b2s_cloud* raw_scan, const double T[16], const double cropper_pose[16],
                         const b2s_carving_params* prm, size_t* n_removed) {
  B2S_REQUIRE(h && sm && raw_scan && T && cropper_pose && prm, B2S_E_INVALID, "null argument");
  B2S_REQUIRE(prm->voxel_size > 0.0, B2S_E_INVALID, "carving voxel size must be > 0");
  LOCK(h);
  B2S_TRY(tile_drop(h, sm));
  double* Td = sm->pose.as<double>() + 64;   // slot 4: pose of the carving scan
  B2S_TRY(pose_to_device(h, T, Td));
  b2s_cropper c = h->cfg.scan.map_builder_cropper;   // mapBuilderCropper_ at the pose of the previous insertion
  c.center[0] = cropper_pose[3]; c.center[1] = cropper_pose[7]; c.center[2] = cropper_pose[11];
  int32_t* removed_dev = reinterpret_cast<int32_t*>(h->status.as<uint32_t>() + SW_REMOVED);
  B2S_TRY(op_submap_carve(h, sm, raw_scan, Td, make_crop(&c), *prm, removed_dev));
  if (!n_removed) return B2S_OK;
  int32_t removed = 0;
  const int32_t rc = read_back(h, {{&removed, removed_dev, 4}});
  *n_removed = (size_t)removed;
  return rc;
}

int32_t b2s_submap_insert_dense(b2s_handle* h, b2s_submap* sm, const b2s_cloud* raw, const double T[16], const b2s_cropper* crop) {
  B2S_REQUIRE(h && sm && raw && T, B2S_E_INVALID, "null argument");
  LOCK(h);
  if (sm->dense_cap == 0) {
    B2S_REQUIRE(h->cfg.dense_voxel_size > 0.0, B2S_E_INVALID, "dense_voxel_size must be > 0");
    B2S_TRY(dense_init(h, sm, (size_t)1 << 22, h->cfg.dense_voxel_size));
  }
  return op_dense_insert(h, sm, raw, T, nullptr, crop);
}

int32_t b2s_submap_size(b2s_handle* h, const b2s_submap* sm, size_t* n) {
  B2S_REQUIRE(h && sm && n, B2S_E_INVALID, "null argument");
  LOCK(h);
  // slots in use minus the tombstones the fusion left behind (fuse.cu)
  int32_t used = 0, dead = 0;
  const int32_t rc = read_back(h, {{&used, sm->cloud[0]->dn.p, 4}, {&dead, sm->mstate.as<int32_t>() + MS_NDEAD, 4}});
  *n = (size_t)(used - dead);
  return rc;
}

int32_t b2s_submap_download(b2s_handle* h, const b2s_submap* sm_c, double* xyz, double* normals, size_t capacity, size_t* n_out) {
  B2S_REQUIRE(h && sm_c, B2S_E_INVALID, "null argument");
  b2s_submap* sm = const_cast<b2s_submap*>(sm_c);
  b2s_cloud* view = nullptr;
  {
    LOCK(h);
    sm->cloud[0]->n_known = -1;
    size_t n = 0;
    B2S_TRY(cloud_count_sync(h, sm->cloud[0].get(), &n));
    sm->cloud[0]->n_max = n;
    B2S_TRY(submap_compact_view(h, sm, &view));   // the live points, in map order
    view->n_known = -1;
  }
  return b2s_cloud_download(h, view, xyz, normals, capacity, n_out);
}

int32_t b2s_submap_to_cloud(b2s_handle* h, const b2s_submap* sm_c, b2s_cloud* out) {
  B2S_REQUIRE(h && sm_c && out, B2S_E_INVALID, "null argument");
  b2s_submap* sm = const_cast<b2s_submap*>(sm_c);
  LOCK(h);
  b2s_cloud* view = nullptr;
  B2S_TRY(submap_compact_view(h, sm, &view));            // live points, map order, in the submap's scratch cloud
  return op_voxel_down_sample(h, view, nullptr, 0.0, out);   // voxel <= 0: plain device copy
}

int32_t b2s_submap_dense_download(b2s_handle* h, const b2s_submap* sm_c, double* xyz, double* normals, int32_t* keys, size_t capacity,
                                  size_t* n_out) {
  B2S_REQUIRE(h && sm_c, B2S_E_INVALID, "null argument");
  (void)normals;
  b2s_submap* sm = const_cast<b2s_submap*>(sm_c);
  LOCK(h);
  if (sm->dense_cap == 0) { if (n_out) *n_out = 0; return B2S_OK; }
  B2S_TRY(h->tmp_f64.ensure(sm->dense_cap * 24 + 64, h->stream));
  B2S_TRY(h->tmp_i32.ensure(sm->dense_cap * 12 + 64, h->stream));
  int32_t* d_keys = h->tmp_i32.as<int32_t>() + 16;
  int32_t* d_n = h->tmp_i32.as<int32_t>();
  B2S_TRY(dense_to_cloud(h, sm, h->tmp_f64.as<double>(), d_keys, d_n));
  int32_t n = 0;
  B2S_CUDA(cudaMemcpyAsync(&n, d_n, 4, cudaMemcpyDeviceToHost, h->stream));
  B2S_CUDA(cudaStreamSynchronize(h->stream));
  if (n_out) *n_out = (size_t)n;
  B2S_REQUIRE((size_t)n <= capacity, B2S_E_CAPACITY, "download buffer too small");
  if (n && xyz) B2S_CUDA(cudaMemcpyAsync(xyz, h->tmp_f64.p, (size_t)n * 24, cudaMemcpyDeviceToHost, h->stream));
  if (n && keys) B2S_CUDA(cudaMemcpyAsync(keys, d_keys, (size_t)n * 12, cudaMemcpyDeviceToHost, h->stream));
  return check_status(h);
}

int32_t b2s_submap_set_cloud(b2s_handle* h, b2s_submap* sm, const b2s_cloud* cloud) {
  B2S_REQUIRE(h && sm && cloud, B2S_E_INVALID, "null argument");
  // the point-to-plane and generalized estimators read the map's normals; a point-to-point pipeline may load a map without
  // (the reference accepts it: isMergeScanValid is only asked of scans) -- "no normal" is stored as NaN
  B2S_REQUIRE(cloud->has_normals || h->cfg.icp.reg_type == B2S_REG_POINT_TO_POINT, B2S_E_NO_NORMALS, "map cloud needs normals for this registration type");
  B2S_REQUIRE(cloud->n_max <= sm->capacity, B2S_E_CAPACITY, "cloud larger than the submap capacity");
  LOCK(h);
  B2S_TRY(tile_drop(h, sm));
  b2s_cloud* m = sm->cloud[0].get();
  if (cloud->n_max) {
    B2S_CUDA(cudaMemcpyAsync(m->xyz.p, cloud->xyz.p, cloud->n_max * 24, cudaMemcpyDeviceToDevice, h->stream));
    if (cloud->has_normals) B2S_CUDA(cudaMemcpyAsync(m->nrm.p, cloud->nrm.p, cloud->n_max * 24, cudaMemcpyDeviceToDevice, h->stream));
    else B2S_CUDA(cudaMemsetAsync(m->nrm.p, 0xFF, cloud->n_max * 24, h->stream));   // all-ones = NaN
  }
  B2S_CUDA(cudaMemcpyAsync(m->dn.p, cloud->dn.p, 4, cudaMemcpyDeviceToDevice, h->stream));
  m->n_max = cloud->n_max; m->n_known = cloud->n_known; m->has_normals = true;
  sm->no_normals = !cloud->has_normals;
  sm->cnt_pending = false; sm->adds_after_readback = 0;
  B2S_CUDA(cudaMemsetAsync(sm->mstate.as<int32_t>() + MS_NDEAD, 0, 4, h->stream));
  return fuse_rehash(h, sm);
}

// Submap::insertScan's initial-map branch (src/Submap.cpp:47-52): mapCloud_ = cloud; voxelize(mapVoxelSize) -- [O3D] VoxelDownSample on
// the data-dependent grid, normals averaged, no carving, no fusion; nScansInsertedMap_ is not counted.  voxelize returns early for a voxel
// size <= 0 (helpers.cpp:107-113): the cloud is then loaded as it is.
int32_t b2s_submap_set_initial_map(b2s_handle* h, b2s_submap* sm, const b2s_cloud* cloud, double map_voxel_size) {
  B2S_REQUIRE(h && sm && cloud, B2S_E_INVALID, "null argument");
  B2S_REQUIRE(sm->h == h && cloud->h == h, B2S_E_INVALID, "the submap or the cloud belongs to another handle");
  LOCK(h);
  b2s_cloud* v = h->t3.get();
  {
    WideGridScope wide(cloud->n_max);
    B2S_TRY(op_voxel_down_sample(h, cloud, nullptr, map_voxel_size, v));   // voxel <= 0: plain device copy
  }
  size_t n = 0;
  v->n_known = -1;
  B2S_TRY(cloud_count_sync(h, v, &n));   // one-off load: the exact size bounds every later launch over the map
  v->n_max = n;
  return b2s_submap_set_cloud(h, sm, v);
}

// Mapper::setMapToRangeSensorInitial (src/Mapper.cpp:87-91): mapToRangeSensor_ = mapToRangeSensorPrev_ = T, isNewInitialValueSet_ = true.
// The pose slot and the flag are device words the captured chains read, so a replayed graph picks both up.
int32_t b2s_submap_set_initial_transform(b2s_handle* h, b2s_submap* sm, const double T[16]) {
  B2S_REQUIRE(h && sm && T, B2S_E_INVALID, "null argument");
  LOCK(h);
  B2S_TRY(pose_to_device(h, T, sm->pose.as<double>()));
  launch_pdl(write_i32_kernel, 1, 1, 0, h->stream, sm->mstate.as<int32_t>() + MS_NEWINIT, (int32_t)1);
  h->launches++;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

// MapperParameters::isMergeScansIntoMap_ for the chain on this submap (Mapper.cpp:163-167).  Off: accepted scans move the pose only.
int32_t b2s_submap_set_merge_scans(b2s_handle* h, b2s_submap* sm, int32_t on) {
  B2S_REQUIRE(h && sm, B2S_E_INVALID, "null argument");
  LOCK(h);
  if (sm->merge_scans == (on != 0)) return B2S_OK;
  sm->merge_scans = on != 0;
  if (on) B2S_TRY(tile_drop(h, sm));   // the chain writes the map again: the table would go stale
  sm->opts_gen++;   // the combined chain's graphs compare it
  return graph_drop(h, &sm->graph);
}

}  // extern "C"

int32_t b2s::register_to_submap_async(b2s_handle* h, const b2s_cloud* scan, const b2s_submap* sm, const double* sensor_pose_host,
                                      const double* sensor_pose_dev, const double* init_host, const double* init_dev, b2s_result* out_dev) {
  B2S_TRY(check_icp_params(h->cfg.icp));
  B2S_REQUIRE(scan->has_normals || h->cfg.icp.reg_type != B2S_REG_GENERALIZED, B2S_E_NO_NORMALS, "GeneralizedIcp: the scan has no normals");
  const b2s_cloud* map = sm->cloud[0].get();
  b2s_cropper c = h->cfg.scan.scan_matcher_cropper;  // ScanToMapRegistration.cpp:58 setPose(mapToRangeSensor)
  if (sensor_pose_host) { c.center[0] = sensor_pose_host[3]; c.center[1] = sensor_pose_host[7]; c.center[2] = sensor_pose_host[11]; }
  CropDev patch = make_crop(&c, sensor_pose_dev);
  if (tile_patch_usable(sm, patch))   // frozen map: the patch from the tiles the cropper touches (K-patch, grid_index.cu)
    B2S_TRY(tile_patch_build(h, const_cast<b2s_submap*>(sm), patch, nn_cell(h, h->cfg.icp.max_corr_dist), &h->grid_a));
  else
    B2S_TRY(grid_build(h, &h->grid_a, map, nn_cell(h, h->cfg.icp.max_corr_dist), &patch));
  B2S_TRY(h->work_xyz.ensure(icp_work_bytes(scan->n_max), h->stream));
  B2S_TRY(h->problems.ensure(sizeof(IcpProblem), h->stream));
  IcpProblem P;
  fill_problem(&P, h->cfg.icp, scan, &h->grid_a, map, init_host, init_dev, h->work_xyz.as<double>(), out_dev);
  return icp_launch(h, &P, nullptr, 1, scan->n_max);
}

extern "C" {

int32_t b2s_register_to_submap(b2s_handle* h, const b2s_cloud* scan, const b2s_submap* sm, const double map_to_sensor[16],
                               const double init[16], b2s_result* out) {
  B2S_REQUIRE(h && scan && sm && map_to_sensor && init && out, B2S_E_INVALID, "null argument");
  LOCK(h);
  B2S_TRY(h->results.ensure(sizeof(b2s_result), h->stream));
  B2S_TRY(register_to_submap_async(h, scan, sm, map_to_sensor, nullptr, init, nullptr, h->results.as<b2s_result>()));
  B2S_CUDA(cudaMemcpyAsync(out, h->results.p, sizeof(b2s_result), cudaMemcpyDeviceToHost, h->stream));
  GridHeader gh;
  B2S_CUDA(cudaMemcpyAsync(&gh, h->grid_a.hdr.p, sizeof(gh), cudaMemcpyDeviceToHost, h->stream));
  B2S_TRY(check_status(h));
  B2S_REQUIRE(gh.n > 0, B2S_E_EMPTY, "map patch size is zero");  // ScanToMapRegistration.cpp:60
  return B2S_OK;
}

int32_t b2s_mapper_step_async(b2s_handle* h, b2s_submap* sm, const b2s_cloud* raw_scan, const double odometry_motion[16],
                              double min_refinement_fitness, int32_t ignore_min_fitness, int32_t slot) {
  B2S_REQUIRE(h && sm && raw_scan && odometry_motion, B2S_E_INVALID, "null argument");
  B2S_REQUIRE(slot >= 0 && slot < 256, B2S_E_INVALID, "slot out of range");
  LOCK(h);
  PdlScope pdl;   // the chain's launches (eager and captured) overlap their predecessors' tails: see pdl_wait in common.cuh
  if (sm->graph_mode) return mapper_step_graph(h, sm, raw_scan, odometry_motion, slot);
  double* pose_state = sm->pose.as<double>();        // mapToRangeSensor_ (== mapToRangeSensorPrev_ in steady state)
  double* odom = pose_state + 32;
  double* guess = pose_state + 48;
  b2s_result* res = h->slots.as<b2s_result>() + slot;
  B2S_TRY(process_scan_impl(h, raw_scan, h->t1.get(), h->t2.get()));          // Mapper.cpp:139
  B2S_TRY(pose_to_device(h, odometry_motion, odom));
  launch_pdl(compose_kernel, 1, 32, 0, h->stream, pose_state, odom, guess, static_cast<const int32_t*>(sm->mstate.as<int32_t>()));   // Mapper.cpp:130-138
  h->launches++;
  B2S_TRY(register_to_submap_async(h, h->t2.get(), sm, nullptr, pose_state, nullptr, guess, res));  // Mapper.cpp:140-141
  return mapper_chain_tail(h, sm, raw_scan, h->t1.get(), res, min_refinement_fitness, ignore_min_fitness, nullptr, nullptr);   // Mapper.cpp:151-177
}

void b2s_default_mapper_options(b2s_mapper_options* o) {
  memset(o, 0, sizeof(*o));
  o->min_movement_between_mapping_steps = 0.0;
  o->carve_enabled = 0; o->carve_every_n_scans = 10;
  o->carving.voxel_size = 0.1; o->carving.max_raytracing_length = 20.0; o->carving.truncation_distance = 0.1;
  o->carving.min_dot_product_with_normal = 0.5; o->carving.neighborhood_radius_dense_map = 0.1;
  o->dense_enabled = 0; o->dense_carve_every_n_scans = 0;
  o->dense_carving = o->carving;
  o->dense_cropper.kind = B2S_CROP_NONE;
}

int32_t b2s_submap_set_mapper_options(b2s_handle* h, b2s_submap* sm, const b2s_mapper_options* o) {
  B2S_REQUIRE(h && sm && o, B2S_E_INVALID, "null argument");
  B2S_REQUIRE(!o->carve_enabled || (o->carve_every_n_scans > 0 && o->carving.voxel_size > 0.0), B2S_E_INVALID, "invalid carving parameters");
  B2S_REQUIRE(o->dense_carve_every_n_scans >= 0 && o->min_movement_between_mapping_steps >= 0.0, B2S_E_INVALID, "invalid mapper options");
  LOCK(h);
  sm->opts = *o;
  sm->opts_gen++;
  return graph_drop(h, &sm->graph);
}

int32_t b2s_submap_get_mapper_counters(b2s_handle* h, const b2s_submap* sm, b2s_mapper_counters* out) {
  B2S_REQUIRE(h && sm && out, B2S_E_INVALID, "null argument");
  LOCK(h);
  int32_t pw[MS_WORDS] = {};
  const int32_t rc = read_back(h, {{pw, sm->mstate.p, sizeof(pw)}});
  out->steps = pw[MS_NSTEPS]; out->accepted = pw[MS_NACCEPT]; out->inserted_map = pw[MS_NINS]; out->inserted_dense = pw[MS_NDENSE];
  out->carve_runs = pw[MS_NCARVE]; out->carved_points_total = pw[MS_CARVED]; out->dense_carve_runs = pw[MS_NDCARVE];
  out->carved_voxels_total = pw[MS_DCARVED];
  return rc;
}

// Turns b2s_mapper_step_async into a CUDA-graph replay for this submap: the ~45 kernel launches of one scan collapse
// into one cudaGraphLaunch.  Returns the fixed-capacity staging cloud every scan has to be uploaded / copied into.
int32_t b2s_mapper_graph_enable(b2s_handle* h, b2s_submap* sm, size_t raw_capacity_points, double min_refinement_fitness,
                                int32_t ignore_min_fitness, b2s_cloud** staging_out) {
  B2S_REQUIRE(h && sm && staging_out && raw_capacity_points > 0, B2S_E_INVALID, "bad argument");
  LOCK(h);
  if (!sm->staging) {   // staging cloud, odometry ring and step counter: all three or none
    std::unique_ptr<b2s_cloud> staging;
    B2S_TRY(make_cloud(h, raw_capacity_points, false, true, &staging));
    PinnedBuf ring;
    B2S_TRY(ring.alloc(64 * 16 * sizeof(double), cudaHostAllocMapped));
    DevBuf gstate;
    B2S_TRY(gstate.ensure(64, h->stream));
    sm->staging = std::move(staging); sm->odom_ring = std::move(ring); sm->gstate = std::move(gstate);
  }
  B2S_TRY(graph_drop(h, &sm->graph));
  sm->g_min_fitness = min_refinement_fitness;
  sm->g_ignore_fitness = ignore_min_fitness;
  sm->graph_mode = true;
  sm->fixed_launch = true;
  sm->graph.warm = 2;
  sm->host_step = 0;
  B2S_CUDA(cudaMemsetAsync(sm->gstate.p, 0, 64, h->stream));
  *staging_out = sm->staging.get();
  return B2S_OK;
}

// upload of a float32 host scan into the chain's input cloud, then one step; *slot receives the result slot of the step
static int32_t mapper_step_upload(b2s_handle* h, b2s_submap* sm, const void* xyz_f32, size_t n, size_t stride_bytes, const double* odometry_motion,
                                  double min_refinement_fitness, int32_t ignore_min_fitness, int32_t* slot) {
  b2s_cloud* dst = sm->graph_mode ? sm->staging.get() : h->t3.get();
  B2S_REQUIRE(!dst->fixed_cap || n <= dst->fixed_cap, B2S_E_CAPACITY, "scan larger than the staging capacity");
  B2S_TRY(b2s_cloud_upload_f32(h, dst, xyz_f32, n, stride_bytes));
  *slot = sm->graph_mode ? (int32_t)(sm->host_step & 255) : 0;
  return b2s_mapper_step_async(h, sm, dst, odometry_motion, min_refinement_fitness, ignore_min_fitness, *slot);
}

// End-to-end form of the per-scan chain with HOST buffers: float32 xyz in (pinned memory makes the copy asynchronous),
// RegistrationResult out.  One call = upload + S1 + S2 + gate + F1 + read-back; synchronises on the result.
int32_t b2s_mapper_step_host(b2s_handle* h, b2s_submap* sm, const void* xyz_f32, size_t n, size_t stride_bytes,
                             const double odometry_motion[16], double min_refinement_fitness, int32_t ignore_min_fitness,
                             b2s_result* out) {
  B2S_REQUIRE(h && sm && xyz_f32 && odometry_motion && out, B2S_E_INVALID, "null argument");
  LOCK(h);   // upload + chain + fetch as one unit
  int32_t slot = 0;
  B2S_TRY(mapper_step_upload(h, sm, xyz_f32, n, stride_bytes, odometry_motion, min_refinement_fitness, ignore_min_fitness, &slot));
  return b2s_scan_result_fetch(h, slot, out);
}

int32_t b2s_mapper_step_host_async(b2s_handle* h, b2s_submap* sm, const void* xyz_f32, size_t n, size_t stride_bytes,
                                   const double odometry_motion[16], double min_refinement_fitness, int32_t ignore_min_fitness,
                                   b2s_result* out_pinned) {
  B2S_REQUIRE(h && sm && xyz_f32 && odometry_motion && out_pinned, B2S_E_INVALID, "null argument");
  LOCK(h);   // upload + chain + result copy as one unit
  int32_t slot = 0;
  B2S_TRY(mapper_step_upload(h, sm, xyz_f32, n, stride_bytes, odometry_motion, min_refinement_fitness, ignore_min_fitness, &slot));
  B2S_CUDA(cudaMemcpyAsync(out_pinned, h->slots.as<b2s_result>() + slot, sizeof(b2s_result), cudaMemcpyDeviceToHost, h->stream));
  return B2S_OK;
}

int32_t b2s_mapper_processed_scan(b2s_handle* h, b2s_cloud* merge_out, b2s_cloud* match_out) {
  B2S_REQUIRE(h, B2S_E_INVALID, "null handle");
  LOCK(h);
  if (merge_out) B2S_TRY(op_voxel_down_sample(h, h->t1.get(), nullptr, 0.0, merge_out));   // voxel <= 0: plain copy
  if (match_out) B2S_TRY(op_voxel_down_sample(h, h->t2.get(), nullptr, 0.0, match_out));
  return B2S_OK;
}

int32_t b2s_scan_result_fetch(b2s_handle* h, int32_t slot, b2s_result* out) {
  B2S_REQUIRE(h && out && slot >= 0 && slot < 256, B2S_E_INVALID, "bad argument");
  LOCK(h);
  return read_back(h, {{out, h->slots.as<b2s_result>() + slot, sizeof(b2s_result)}});
}

// ---- loop-closure features ---------------------------------------------------------------------------------------------
int32_t b2s_feature_create(b2s_handle* h, b2s_feature** out) {
  B2S_REQUIRE(h && out, B2S_E_INVALID, "null argument");
  LOCK(h);
  return create_object(out, [&](b2s_feature* f) -> int32_t {
    f->h = h;
    f->device = h->device;
    f->data.tracked = f->nb_idx.tracked = f->nb_d2.tracked = f->nb_cnt.tracked = f->spfh.tracked = false;   // caller-owned, never in a graph
    return B2S_OK;
  });
}

void b2s_feature_destroy(b2s_feature* f) { destroy_object(f); }

int32_t b2s_feature_size(b2s_handle* h, const b2s_feature* f, size_t* n) {
  B2S_REQUIRE(h && f && n, B2S_E_INVALID, "null argument");
  B2S_REQUIRE(f->h == h, B2S_E_INVALID, "the feature belongs to another handle");
  LOCK(h);
  *n = f->n;
  return B2S_OK;
}

int32_t b2s_feature_download(b2s_handle* h, const b2s_feature* f, double* data, size_t capacity_points, size_t* n_out) {
  B2S_REQUIRE(h && f && (data || f->n == 0), B2S_E_INVALID, "null argument");
  B2S_REQUIRE(f->h == h, B2S_E_INVALID, "the feature belongs to another handle");
  LOCK(h);
  if (n_out) *n_out = f->n;
  B2S_REQUIRE(f->n <= capacity_points, B2S_E_CAPACITY, "download buffer too small: %zu points, capacity %zu", f->n, capacity_points);
  if (f->n) B2S_CUDA(cudaMemcpyAsync(data, f->data.p, f->n * B2S_FEATURE_DIM * 8, cudaMemcpyDeviceToHost, h->stream));
  return check_status(h);
}

int32_t b2s_feature_upload(b2s_handle* h, b2s_feature* f, const double* data, size_t n) {
  B2S_REQUIRE(h && f && (data || n == 0), B2S_E_INVALID, "null argument");
  B2S_REQUIRE(n < (size_t)0x7fffffff / B2S_FEATURE_DIM, B2S_E_INVALID, "feature too large");
  B2S_REQUIRE(f->h == h, B2S_E_INVALID, "the feature belongs to another handle");
  LOCK(h);
  if (n) {
    B2S_TRY(f->data.ensure(n * B2S_FEATURE_DIM * 8, h->stream));
    B2S_CUDA(cudaMemcpyAsync(f->data.p, data, n * B2S_FEATURE_DIM * 8, cudaMemcpyHostToDevice, h->stream));
  }
  f->n = n;
  return B2S_OK;
}

int32_t b2s_compute_fpfh(b2s_handle* h, const b2s_cloud* cloud, double radius, int32_t knn, b2s_feature* feature) {
  B2S_REQUIRE(h && cloud && feature, B2S_E_INVALID, "null argument");
  B2S_REQUIRE(feature->h == h, B2S_E_INVALID, "the feature belongs to another handle");
  B2S_REQUIRE(cloud->device == h->device, B2S_E_INVALID, "the cloud lives on device %d, the handle on device %d", cloud->device, h->device);
  B2S_REQUIRE(radius > 0.0, B2S_E_INVALID, "ComputeFPFHFeature: radius must be > 0");
  B2S_REQUIRE(knn > 0, B2S_E_INVALID, "ComputeFPFHFeature: max_nn must be > 0");
  B2S_REQUIRE(knn <= B2S_FEATURE_MAX_KNN, B2S_E_UNSUPPORTED, "ComputeFPFHFeature: max_nn %d > %d is not supported", knn, B2S_FEATURE_MAX_KNN);
  LOCK(h);
  size_t n = 0;
  B2S_TRY(cloud_count_sync(h, cloud, &n));
  B2S_REQUIRE(n == 0 || cloud->has_normals, B2S_E_NO_NORMALS, "ComputeFPFHFeature: the point cloud has no normals");
  return op_compute_fpfh(h, cloud, n, radius, knn, feature);
}

void b2s_default_feature_params(b2s_feature_params* p) {   // parameter_structure_definitions.lua:155-159
  memset(p, 0, sizeof(*p));
  p->feature_voxel_size = 0.5; p->normal_estimation_radius = 2.0; p->normal_knn = 20; p->feature_radius = 2.5; p->feature_knn = 100;
}

// Submap::computeFeatures (src/Submap.cpp:239-244) without the host: map -> sparse cloud -> normals (the voxel-mean normals as
// priors) -> FPFH.  The map's count is never read; the one synchronisation reads the sparse cloud's count for the FPFH launch
// and reports a voxel key beyond the fixed width.
int32_t b2s_submap_compute_features(b2s_handle* h, b2s_submap* sm, const b2s_feature_params* p, b2s_cloud* sparse, b2s_feature* f) {
  B2S_REQUIRE(h && sm && p && sparse && f, B2S_E_INVALID, "null argument");
  B2S_REQUIRE(sm->h == h, B2S_E_INVALID, "the submap belongs to another handle");
  B2S_REQUIRE(sparse->h == h, B2S_E_INVALID, "the sparse cloud belongs to another handle");
  B2S_REQUIRE(f->h == h, B2S_E_INVALID, "the feature belongs to another handle");
  B2S_REQUIRE(!sparse->fixed_cap, B2S_E_INVALID, "the sparse cloud must not be a fixed-capacity staging cloud");
  B2S_REQUIRE(p->feature_voxel_size > 0.0 && p->normal_estimation_radius > 0.0 && p->feature_radius > 0.0, B2S_E_INVALID,
              "computeFeatures: featureVoxelSize_, normalEstimationRadius_ and featureRadius_ must be > 0");
  B2S_REQUIRE(p->normal_knn > 0 && p->feature_knn > 0, B2S_E_INVALID, "computeFeatures: normalKnn_ and featureKnn_ must be > 0");
  B2S_REQUIRE(p->normal_knn <= 32, B2S_E_UNSUPPORTED, "computeFeatures: normalKnn_ %d > 32 is not supported", p->normal_knn);
  B2S_REQUIRE(p->feature_knn <= B2S_FEATURE_MAX_KNN, B2S_E_UNSUPPORTED, "computeFeatures: featureKnn_ %d > %d is not supported", p->feature_knn,
              B2S_FEATURE_MAX_KNN);
  LOCK(h);
  b2s_cloud* view = nullptr;
  B2S_TRY(submap_compact_view(h, sm, &view));   // getMapPointCloudCopy: the live points in map order, normals included (NaN = none)
  // VoxelDownSample: the full key width, so that the extent need not be read back; a map wider than 2^21 voxels is reported below
  B2S_TRY(op_voxel_down_sample(h, view, nullptr, p->feature_voxel_size, sparse, 21));
  B2S_TRY(op_estimate_normals(h, sparse, p->normal_knn, p->normal_estimation_radius, 0.0, nullptr, sparse->has_normals));
  int32_t n = 0;
  B2S_TRY(read_back(h, {{&n, sparse->dn.p, 4}}));
  sparse->n_known = n;
  return op_compute_fpfh(h, sparse, (size_t)n, p->feature_radius, p->feature_knn, f);
}

// ---- loop-closure proposal (PlaceRecognition.cpp:81-86) --------------------------------------------------------------------
void b2s_default_ransac_params(b2s_ransac_params* p) {   // parameter_structure_definitions.lua:156-161
  memset(p, 0, sizeof(*p));
  p->mutual_filter = 1; p->ransac_n = 3; p->max_correspondence_distance = 0.75; p->checker_distance = 0.8; p->checker_edge_length = 0.6;
  p->max_iteration = 10000000; p->confidence = 0.999; p->seed = 1;
}

// RegistrationRANSACBasedOnFeatureMatching(sourceSparse, targetSparse, sourceFeature, targetFeature, true, ...) for every candidate
// of PlaceRecognition.cpp:71 in one call.  Synchronises for the cloud sizes, then once per batch of hypotheses.
int32_t b2s_ransac_feature_matching(b2s_handle* h, const b2s_cloud* src, const b2s_feature* src_f, int32_t n, const b2s_cloud* const* tgts,
                                    const b2s_feature* const* tgt_fs, const b2s_ransac_params* p, b2s_ransac_result* out) {
  B2S_REQUIRE(n >= 0, B2S_E_INVALID, "n_targets must be >= 0");
  B2S_REQUIRE(h && src && src_f && p && (n == 0 || (tgts && tgt_fs && out)), B2S_E_INVALID, "null argument");
  B2S_REQUIRE(p->confidence > 0.0 && p->confidence < 1.0, B2S_E_INVALID, "RANSACConvergenceCriteria: confidence must be in (0, 1)");
  B2S_REQUIRE(p->max_iteration >= 0, B2S_E_INVALID, "RANSACConvergenceCriteria: max_iteration must be >= 0");
  B2S_REQUIRE(p->ransac_n <= B2S_RANSAC_MAX_N, B2S_E_UNSUPPORTED, "ransac_n %d > %d is not supported", p->ransac_n, B2S_RANSAC_MAX_N);
  B2S_REQUIRE(src->h == h && src_f->h == h, B2S_E_INVALID, "the source belongs to another handle");
  for (int32_t k = 0; k < n; ++k) {
    B2S_REQUIRE(tgts[k] && tgt_fs[k], B2S_E_INVALID, "null target %d", k);
    B2S_REQUIRE(tgts[k]->h == h && tgt_fs[k]->h == h, B2S_E_INVALID, "target %d belongs to another handle", k);
  }
  LOCK(h);
  size_t ns = 0;
  B2S_TRY(cloud_count_sync(h, src, &ns));
  B2S_REQUIRE(ns == src_f->n, B2S_E_INVALID, "the source feature has %zu points, its cloud %zu", src_f->n, ns);
  std::vector<size_t> nts((size_t)n);
  for (int32_t k = 0; k < n; ++k) {
    B2S_TRY(cloud_count_sync(h, tgts[k], &nts[k]));
    B2S_REQUIRE(nts[k] == tgt_fs[k]->n, B2S_E_INVALID, "target %d: the feature has %zu points, its cloud %zu", k, tgt_fs[k]->n, nts[k]);
  }
  if (n == 0) return B2S_OK;
  B2S_TRY(op_ransac(h, src, ns, src_f, n, tgts, nts.data(), tgt_fs, *p, out));
  return check_status(h);
}

int32_t b2s_feature_correspondences(b2s_handle* h, const b2s_feature* src_f, const b2s_feature* tgt_f, int32_t* s2t, size_t s_cap, int32_t* t2s,
                                    size_t t_cap) {
  B2S_REQUIRE(h && src_f && tgt_f && (s2t || src_f->n == 0) && (t2s || tgt_f->n == 0), B2S_E_INVALID, "null argument");
  B2S_REQUIRE(src_f->h == h && tgt_f->h == h, B2S_E_INVALID, "the feature belongs to another handle");
  B2S_REQUIRE(src_f->n <= s_cap && tgt_f->n <= t_cap, B2S_E_CAPACITY, "output arrays hold %zu / %zu entries, the features have %zu / %zu points",
              s_cap, t_cap, src_f->n, tgt_f->n);
  LOCK(h);
  B2S_TRY(h->tmp_i32.ensure((src_f->n + tgt_f->n + 1) * 4, h->stream));
  int32_t* d_s2t = h->tmp_i32.as<int32_t>();
  int32_t* d_t2s = d_s2t + src_f->n;
  B2S_TRY(op_feature_correspondences(h, src_f, 1, &tgt_f, &d_s2t, &d_t2s));
  if (src_f->n) B2S_CUDA(cudaMemcpyAsync(s2t, d_s2t, src_f->n * 4, cudaMemcpyDeviceToHost, h->stream));
  if (tgt_f->n) B2S_CUDA(cudaMemcpyAsync(t2s, d_t2s, tgt_f->n * 4, cudaMemcpyDeviceToHost, h->stream));
  return check_status(h);
}

// ---- odometry constraints (src/constraint_builders.cpp:33-118) ---------------------------------------------------------------
void b2s_default_odometry_constraint_params(b2s_odometry_constraint_params* p) {   // magic.hpp:12-15, Lua map_builder / mapper defaults
  memset(p, 0, sizeof(*p));
  p->map_voxel_size = 0.1; p->voxel_if_zero = 0.04; p->overlap_factor = 20.0; p->icp_factor = 1.5; p->min_points_per_voxel = 1;
  p->refine = 0; p->max_iter = 100; p->rel_fitness = 1e-6; p->rel_rmse = 1e-6;
}

int32_t b2s_submap_odometry_constraints(b2s_handle* h, int32_t n, const b2s_submap* const* sources, const b2s_submap* const* targets,
                                        const b2s_odometry_constraint_params* p, b2s_cloud* const* so, b2s_cloud* const* to,
                                        b2s_odometry_constraint* out) {
  B2S_REQUIRE(h && p && n >= 0, B2S_E_INVALID, "bad argument");
  if (n == 0) return B2S_OK;
  B2S_REQUIRE(sources && targets && out, B2S_E_INVALID, "null argument");
  const double voxel = fabs(p->map_voxel_size) <= 1e-3 ? p->voxel_if_zero : p->map_voxel_size;   // getMapVoxelSize, helpers.cpp:343-345
  B2S_REQUIRE(voxel > 0.0, B2S_E_INVALID, "map voxel size %g after getMapVoxelSize: must be > 0", voxel);
  B2S_REQUIRE(p->overlap_factor > 0.0 && p->icp_factor > 0.0, B2S_E_INVALID, "overlap_factor and icp_factor must be > 0");
  B2S_REQUIRE(p->min_points_per_voxel >= 1, B2S_E_INVALID, "minNumPointsPerVoxel must be >= 1");   // assert_ge at helpers.cpp:310
  B2S_REQUIRE(p->max_iter >= 0, B2S_E_INVALID, "max_iter must be >= 0");
  for (int32_t k = 0; k < n; k++) {
    B2S_REQUIRE(sources[k] && targets[k], B2S_E_INVALID, "null submap in pair %d", k);
    B2S_REQUIRE(sources[k]->h == h && targets[k]->h == h, B2S_E_INVALID, "pair %d: a submap belongs to another handle", k);
    for (b2s_cloud* const* c : {so, to})
      if (c) {
        B2S_REQUIRE(c[k] && c[k]->h == h, B2S_E_INVALID, "pair %d: an overlap cloud is null or belongs to another handle", k);
        B2S_REQUIRE(!c[k]->fixed_cap, B2S_E_INVALID, "pair %d: an overlap cloud must not be a fixed-capacity staging cloud", k);
      }
    B2S_REQUIRE(!so || !to || so[k] != to[k], B2S_E_INVALID, "pair %d: the two overlap clouds are the same object", k);
  }
  for (int32_t k = 0; k < n; k++)   // RegistrationICP's point-to-plane estimator needs the target's normals ([O3D] LogError)
    B2S_REQUIRE(!p->refine || !targets[k]->no_normals, B2S_E_NO_NORMALS,
                "[RegistrationICP] pair %d: TransformationEstimationPointToPlane requires target normals, the child map has none", k);
  LOCK(h);
  return op_odometry_constraints(h, n, sources, targets, *p, voxel, so, to, out);
}

// ---- pose-graph optimisation (src/OptimizationProblem.cpp:25-44 -> [O3D] GlobalOptimization, LM) -------------------------------
void b2s_default_global_optimization_params(b2s_global_optimization_params* p) {   // parameter_structure_definitions.lua:45-50, [O3D] criteria
  memset(p, 0, sizeof(*p));
  p->max_correspondence_distance = 1000.0; p->edge_prune_threshold = 0.2; p->preference_loop_closure = 2.0; p->reference_node = 0;
  p->max_iteration = 100; p->min_relative_increment = 1e-6; p->min_relative_residual_increment = 1e-6; p->min_right_term = 1e-6;
  p->min_residual = 1e-6; p->max_iteration_lm = 20; p->upper_scale_factor = 2.0 / 3.0; p->lower_scale_factor = 1.0 / 3.0;
}

int32_t b2s_global_optimization(b2s_handle* h, int32_t n_nodes, double* node_poses, int32_t n_edges, const b2s_pose_graph_edge* edges,
                                const b2s_global_optimization_params* p, int32_t* edge_kept_out, double* edge_confidence_out,
                                b2s_global_optimization_stats* stats_out) {
  B2S_REQUIRE(h && p && node_poses, B2S_E_INVALID, "null argument");
  B2S_REQUIRE(n_nodes >= 1 && n_edges >= 0, B2S_E_INVALID, "n_nodes %d must be >= 1 and n_edges %d >= 0", (int)n_nodes, (int)n_edges);
  B2S_REQUIRE(n_edges == 0 || edges, B2S_E_INVALID, "null edges");
  B2S_REQUIRE(p->min_relative_increment > 0.0 && p->min_relative_residual_increment > 0.0 && p->min_right_term > 0.0 && p->min_residual > 0.0,
              B2S_E_INVALID, "the convergence tolerances must be > 0");
  B2S_REQUIRE(p->max_iteration >= 1 && p->max_iteration_lm >= 1, B2S_E_INVALID, "max_iteration and max_iteration_lm must be >= 1");
  for (int32_t e = 0; e < n_edges; e++)   // ValidatePoseGraph's id check
    B2S_REQUIRE(edges[e].source >= 0 && edges[e].source < n_nodes && edges[e].target >= 0 && edges[e].target < n_nodes, B2S_E_INVALID,
                "edge %d: node ids (%d, %d) outside [0, %d)", (int)e, (int)edges[e].source, (int)edges[e].target, (int)n_nodes);
  LOCK(h);
  return op_global_optimization(h, n_nodes, node_poses, n_edges, edges, *p, edge_kept_out, edge_confidence_out, stats_out);
}

// debug aid for tests: the header, cell starts and original indices of the NN index the last registration built (h->grid_a).
// dims_n = {dims[0..2], ncell, n}; cell_start (ncell + 1 entries) and orig (n entries) are skipped when null or too small.
int32_t b2s_debug_nn_index(b2s_handle* h, double origin_cell[4], int32_t dims_n[5], int32_t* cell_start, size_t cap_cells, int32_t* orig,
                           size_t cap_pts) {
  B2S_REQUIRE(h && origin_cell && dims_n, B2S_E_INVALID, "null argument");
  LOCK(h);
  B2S_REQUIRE(h->grid_a.hdr.p, B2S_E_INVALID, "no NN index has been built yet");
  GridHeader gh;
  B2S_TRY(read_back(h, {{&gh, h->grid_a.hdr.p, sizeof(gh)}}));
  for (int d = 0; d < 3; d++) { origin_cell[d] = gh.origin[d]; dims_n[d] = gh.dims[d]; }
  origin_cell[3] = gh.cell; dims_n[3] = gh.ncell; dims_n[4] = gh.n;
  if (cell_start && cap_cells >= (size_t)gh.ncell + 1)
    B2S_CUDA(cudaMemcpy(cell_start, grid_starts(&h->grid_a), ((size_t)gh.ncell + 1) * 4, cudaMemcpyDeviceToHost));
  if (orig && cap_pts >= (size_t)gh.n && gh.n > 0) {
    std::vector<double> p4((size_t)gh.n * 4);
    B2S_CUDA(cudaMemcpy(p4.data(), h->grid_a.pts.p, p4.size() * 8, cudaMemcpyDeviceToHost));
    for (int32_t k = 0; k < gh.n; k++) { long long v; memcpy(&v, &p4[4 * (size_t)k + 3], 8); orig[k] = (int32_t)v; }
  }
  return B2S_OK;
}

}  // extern "C"
