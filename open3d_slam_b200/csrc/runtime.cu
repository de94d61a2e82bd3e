// runtime.cu -- host runtime (errors, buffers) and the two device-wide primitives everything else is built
// from: a single-pass decoupled-look-back exclusive scan and a stable LSD radix sort (8-bit digits,
// match_any warp ranking).  Hand-written for sm_90a; no CUB/Thrust on the product path.
#include <cooperative_groups.h>
#include <stdarg.h>
#include <stdlib.h>

#include "common.cuh"

namespace b2s {

static thread_local char g_err[1024] = {0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
const char* get_error() { return g_err; }

unsigned long long g_alloc_generation = 1;
static int g_device_sms[64] = {0};
int device_sms() {
  int d = 0;
  if (cudaGetDevice(&d) != cudaSuccess || d < 0 || d >= 64) d = 0;
  int v = __atomic_load_n(&g_device_sms[d], __ATOMIC_RELAXED);
  if (v <= 0) {
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, d) != cudaSuccess || v <= 0) v = 132;
    __atomic_store_n(&g_device_sms[d], v, __ATOMIC_RELAXED);
  }
  return v;
}
static thread_local int g_grid_cap_override = 0;
int grid_cap() {
  if (g_grid_cap_override > 0) return g_grid_cap_override;
  static const int v = getenv("B2S_GRID_CAP") ? atoi(getenv("B2S_GRID_CAP")) : 0;
  return v > 0 ? v : 2 * device_sms();
}
WideGridScope::WideGridScope(size_t n) : on(n >= ((size_t)1 << 19) && g_grid_cap_override == 0) { if (on) g_grid_cap_override = 16 * device_sms(); }
WideGridScope::~WideGridScope() { if (on) g_grid_cap_override = 0; }
static thread_local int g_pdl_depth = 0;
bool pdl_enabled() {
  static const bool on = !(getenv("B2S_PDL") && atoi(getenv("B2S_PDL")) == 0);
  return on && g_pdl_depth > 0;
}
PdlScope::PdlScope() { g_pdl_depth++; }
PdlScope::~PdlScope() { g_pdl_depth--; }
thread_local bool g_capturing = false;
thread_local bool g_capture_broken = false;

int32_t DevBuf::ensure(size_t bytes, cudaStream_t s, bool preserve) {
  if (bytes <= cap && p) return B2S_OK;
  if (g_capturing) {   // cannot allocate / synchronise inside a stream capture: the caller falls back to eager launches
    g_capture_broken = true;
    set_error("device buffer would have to grow during CUDA graph capture");
    return B2S_E_CAPACITY;
  }
  // 25 % headroom on every (re)allocation: scan sizes jitter by a few percent from scan to scan and a re-allocation
  // is a device-wide synchronisation (cudaMalloc / cudaFree), so steady state must never re-allocate
  size_t ncap = cap + cap / 2;
  const size_t want = bytes > 4096 ? bytes + bytes / 4 : bytes;
  if (ncap < want) ncap = want;
  ncap = (ncap + 255) & ~(size_t)255;
  if (ncap < 256) ncap = 256;
  void* np = nullptr;
  const cudaError_t me = cudaMalloc(&np, ncap);
  // the runtime also keeps the failure as this thread's last error: clear it, so that this call reports it and no later one does
  if (me != cudaSuccess) { cudaGetLastError(); B2S_CUDA(me); }
  if (p) {
    if (preserve) B2S_CUDA(cudaMemcpyAsync(np, p, cap, cudaMemcpyDeviceToDevice, s));
    B2S_CUDA(cudaStreamSynchronize(s));  // earlier kernels may still read the old allocation
    B2S_CUDA(cudaFree(p));
  }
  if (p && tracked) __atomic_add_fetch(&g_alloc_generation, 1ull, __ATOMIC_RELAXED);   // captured graphs may hold the old address
  p = np;
  cap = ncap;
  return B2S_OK;
}
void DevBuf::release() {
  if (p) cudaFree(p);
  p = nullptr;
  cap = 0;
}
int32_t PinnedBuf::alloc(size_t bytes, unsigned flags) {
  release();
  const cudaError_t me = cudaHostAlloc(&p, bytes, flags);
  if (me != cudaSuccess) { p = nullptr; cudaGetLastError(); B2S_CUDA(me); }   // last error cleared as in DevBuf::ensure
  cap = bytes;
  return B2S_OK;
}

ProfScope::ProfScope(b2s_handle* h_, int kind) : h(h_), idx(-1) {
  if (!h->prof_enabled || g_capturing) return;
  ProfRec r;
  r.kind = kind;
  cudaEvent_t* ev[2] = {&r.a, &r.b};
  for (int i = 0; i < 2; i++) {
    if (!h->prof_pool.empty()) { *ev[i] = h->prof_pool.back(); h->prof_pool.pop_back(); }
    else if (cudaEventCreate(ev[i]) != cudaSuccess) return;
  }
  cudaEventRecord(r.a, h->stream);
  idx = (int)h->prof_recs.size();
  h->prof_recs.push_back(r);
}
ProfScope::~ProfScope() {
  if (idx >= 0) cudaEventRecord(h->prof_recs[(size_t)idx].b, h->stream);
}

constexpr size_t PINNED_READ_BACK = 256;   // layout of h->pinned: the status word at byte 0, read_back's copies from here on

static int32_t ensure_pinned(b2s_handle* h, size_t bytes) {
  if (bytes <= h->pinned.cap) return B2S_OK;
  if (h->pinned.p) B2S_CUDA(cudaStreamSynchronize(h->stream));
  return h->pinned.alloc((bytes + 4095) & ~(size_t)4095);
}

int32_t check_status(b2s_handle* h) {
  // through pinned memory: a pageable device->host copy goes through a driver staging path that serialises the host
  // threads of all chains
  B2S_TRY(ensure_pinned(h, 4096));
  volatile uint32_t* pst = h->pinned.as<volatile uint32_t>();
  B2S_CUDA(cudaMemcpyAsync(h->pinned.p, h->status.p, 4, cudaMemcpyDeviceToHost, h->stream));
  B2S_CUDA(cudaStreamSynchronize(h->stream));
  const uint32_t st = pst[0];
  if (st == 0) return B2S_OK;
  B2S_CUDA(cudaMemsetAsync(h->status.p, 0, 4, h->stream));
  if (st & ST_CAPACITY) { set_error("device structure capacity exceeded (status 0x%x)", st); return B2S_E_CAPACITY; }
  if (st & ST_HASH_FULL) { set_error("dense voxel hash is full (status 0x%x)", st); return B2S_E_CAPACITY; }
  if (st & ST_KEY_OVERFLOW) { set_error("voxel key out of range for the chosen key width (status 0x%x)", st); return B2S_E_INVALID; }
  if (st & ST_EMPTY) { set_error("cloud is empty where the reference asserts a non-empty cloud (status 0x%x)", st); return B2S_E_EMPTY; }
  set_error("unknown device status 0x%x", st);
  return B2S_E_INVALID;
}

int32_t read_back(b2s_handle* h, std::initializer_list<ReadBack> copies) {
  size_t end = PINNED_READ_BACK;
  for (const ReadBack& c : copies) end += c.bytes;
  B2S_TRY(ensure_pinned(h, end));   // rounded up to whole pages, so check_status keeps this allocation
  char* stage = h->pinned.as<char>() + PINNED_READ_BACK;
  for (const ReadBack& c : copies) { B2S_CUDA(cudaMemcpyAsync(stage, c.src, c.bytes, cudaMemcpyDeviceToHost, h->stream)); stage += c.bytes; }
  const int32_t rc = check_status(h);   // synchronises
  stage = h->pinned.as<char>() + PINNED_READ_BACK;
  for (const ReadBack& c : copies) { memcpy(c.dst, stage, c.bytes); stage += c.bytes; }
  return rc;
}

// =================================================================================================
//  exclusive scan, single pass, decoupled look-back
// =================================================================================================
constexpr int SCAN_THREADS = 256;
constexpr int SCAN_ITEMS = 16;
constexpr int SCAN_TILE = SCAN_THREADS * SCAN_ITEMS;
#define FLAG_AGG (1ull << 62)
#define FLAG_PREFIX (2ull << 62)

__device__ __forceinline__ void scan_lookback_body(const int32_t* __restrict__ in, int32_t* __restrict__ out,
                                                   const int32_t* __restrict__ d_n, int32_t n_host, unsigned long long* state,
                                                   int32_t* tile_counter, int32_t* d_total) {
  __shared__ int s_tile;
  __shared__ int s_warp[SCAN_THREADS / 32];
  __shared__ int s_prefix;
  if (threadIdx.x == 0) s_tile = atomicAdd(tile_counter, 1);
  __syncthreads();
  const int tile = s_tile;
  const int n = d_n ? *d_n : n_host;
  const int ntiles = (n + SCAN_TILE - 1) / SCAN_TILE;
  if (tile >= ntiles) {
    if (tile == 0 && threadIdx.x == 0) { out[0] = 0; if (d_total) *d_total = 0; }
    return;
  }
  const int base = tile * SCAN_TILE + threadIdx.x * SCAN_ITEMS;
  int v[SCAN_ITEMS];
  const bool vec_ok = ((((size_t)in | (size_t)out) & 15) == 0);
  if (vec_ok && base + SCAN_ITEMS <= n) {
    const int4* p = reinterpret_cast<const int4*>(in + base);
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS / 4; k++) { int4 q = p[k]; v[4 * k] = q.x; v[4 * k + 1] = q.y; v[4 * k + 2] = q.z; v[4 * k + 3] = q.w; }
  } else {
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; k++) v[k] = (base + k < n) ? in[base + k] : 0;
  }
  int tsum = 0;
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; k++) tsum += v[k];
  // block exclusive scan of the per-thread sums
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int inc = tsum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { int t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
  if (lane == 31) s_warp[warp] = inc;
  __syncthreads();
  int woff = 0, agg = 0;
#pragma unroll
  for (int w = 0; w < SCAN_THREADS / 32; w++) { int t = s_warp[w]; if (w < warp) woff += t; agg += t; }
  int texcl = woff + inc - tsum;
  // decoupled look-back (warp 0)
  if (warp == 0) {
    volatile unsigned long long* vs = state;
    if (tile == 0) {
      if (lane == 0) { vs[0] = FLAG_PREFIX | (unsigned long long)(unsigned)agg; s_prefix = 0; }
    } else {
      if (lane == 0) vs[tile] = FLAG_AGG | (unsigned long long)(unsigned)agg;
      int look = tile - 1, excl = 0;
      while (true) {
        int idx = look - lane;
        unsigned long long s = (idx >= 0) ? vs[idx] : FLAG_PREFIX;
        unsigned flag = (unsigned)(s >> 62);
        if (__any_sync(0xffffffffu, flag == 0)) continue;
        unsigned pmask = __ballot_sync(0xffffffffu, flag == 2);
        int val = (int)(unsigned)(s & 0xffffffffull);
        if (pmask) {
          int first = __ffs(pmask) - 1;
          excl += warp_sum_i(lane <= first ? val : 0);
          excl = __shfl_sync(0xffffffffu, excl, 0);
          break;
        }
        excl += warp_sum_i(val);
        excl = __shfl_sync(0xffffffffu, excl, 0);
        look -= 32;
      }
      if (lane == 0) { vs[tile] = FLAG_PREFIX | (unsigned long long)(unsigned)(excl + agg); s_prefix = excl; }
    }
  }
  __syncthreads();
  int run = s_prefix + texcl;
  if (vec_ok && base + SCAN_ITEMS <= n) {
    int o[SCAN_ITEMS];
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; k++) { o[k] = run; run += v[k]; }
    int4* p = reinterpret_cast<int4*>(out + base);
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS / 4; k++) p[k] = make_int4(o[4 * k], o[4 * k + 1], o[4 * k + 2], o[4 * k + 3]);
  } else {
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; k++) { if (base + k < n) out[base + k] = run; run += v[k]; }
  }
  if (tile == ntiles - 1 && threadIdx.x == SCAN_THREADS - 1) {
    out[n] = s_prefix + agg;
    if (d_total) *d_total = s_prefix + agg;
  }
}

__global__ void __launch_bounds__(SCAN_THREADS) scan_lookback_kernel(const int32_t* __restrict__ in, int32_t* __restrict__ out,
                                                                     const int32_t* __restrict__ d_n, int32_t n_host,
                                                                     unsigned long long* state, int32_t* tile_counter,
                                                                     int32_t* d_total) {
  pdl_wait();
  scan_lookback_body(in, out, d_n, n_host, state, tile_counter, d_total);
}

// blockIdx.y = job: independent scans of different arrays in one launch (batched index builds)
__global__ void __launch_bounds__(SCAN_THREADS) scan_lookback_batch_kernel(const ScanJob* __restrict__ jobs) {
  pdl_wait();
  const ScanJob j = jobs[blockIdx.y];
  scan_lookback_body(j.in, j.out, j.d_n, 0, j.state, j.counter, nullptr);
}

// A scan's tile state: one uint64 per tile, then the tile counter in the 64 bytes after them.
static int scan_tiles(size_t n_max) {
  const size_t ntiles = (n_max + SCAN_TILE - 1) / SCAN_TILE;
  return ntiles < 1 ? 1 : (int)ntiles;
}
static size_t scan_state_bytes(size_t n_max) { return (size_t)scan_tiles(n_max) * 8 + 64; }
static int32_t* scan_counter(unsigned long long* state, size_t n_max) { return reinterpret_cast<int32_t*>(state + scan_tiles(n_max)); }

void scan_bind_state(Layout& L, ScanJob& j, size_t n_max) {
  unsigned char* s = L.take<unsigned char>(scan_state_bytes(n_max));
  if (!s) return;
  j.state = reinterpret_cast<unsigned long long*>(s);
  j.counter = scan_counter(j.state, n_max);
}

int32_t scan_exclusive_i32_batch(b2s_handle* h, const ScanJob* jobs_dev, int njobs, size_t n_max) {
  launch_pdl(scan_lookback_batch_kernel, dim3(scan_tiles(n_max), njobs), SCAN_THREADS, 0, h->stream, jobs_dev);
  h->launches++;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

static int32_t scan_impl(b2s_handle* h, const int32_t* in, int32_t* out, const int32_t* d_n, int32_t n_host, size_t n_max,
                         int32_t* d_total, DevBuf* state) {
  const int ntiles = scan_tiles(n_max);
  DevBuf& sb = state ? *state : h->scan.state;
  B2S_TRY(sb.ensure(scan_state_bytes(n_max), h->stream));
  B2S_CUDA(cudaMemsetAsync(sb.p, 0, scan_state_bytes(n_max), h->stream));
  unsigned long long* st = sb.as<unsigned long long>();
  int32_t* counter = scan_counter(st, n_max);
  launch_pdl(scan_lookback_kernel, ntiles, SCAN_THREADS, 0, h->stream, in, out, d_n, n_host, st, counter, d_total);
  h->launches++;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

int32_t scan_exclusive_i32(b2s_handle* h, const int32_t* in, int32_t* out, const int32_t* d_n, size_t n_max, int32_t* d_total, DevBuf* state) {
  return scan_impl(h, in, out, d_n, (int32_t)n_max, n_max, d_total, state);
}

// =================================================================================================
//  stable LSD radix sort, 8-bit digits: per pass  histogram -> scan -> ranked scatter
// =================================================================================================
constexpr int RS_THREADS = 256;
constexpr int RS_ITEMS = 8;
constexpr int RS_TILE = RS_THREADS * RS_ITEMS;
constexpr int RS_WARPS = RS_THREADS / 32;

template <typename K>
__global__ void __launch_bounds__(RS_THREADS) rs_hist_kernel(const K* __restrict__ keys, const int32_t* __restrict__ d_n, int shift,
                                                             int32_t* __restrict__ hist, int nblocks) {
  pdl_wait();
  __shared__ int s_h[256];
  s_h[threadIdx.x] = 0;
  __syncthreads();
  const int n = *d_n;
  const int base = blockIdx.x * RS_TILE;
#pragma unroll
  for (int k = 0; k < RS_ITEMS; k++) {
    int i = base + k * RS_THREADS + threadIdx.x;
    if (i < n) atomicAdd(&s_h[(int)((keys[i] >> shift) & 0xFF)], 1);
  }
  __syncthreads();
  hist[threadIdx.x * nblocks + blockIdx.x] = s_h[threadIdx.x];
}

template <typename K>
__global__ void __launch_bounds__(RS_THREADS) rs_scatter_kernel(const K* __restrict__ keys_in, const uint32_t* __restrict__ vals_in,
                                                                K* __restrict__ keys_out, uint32_t* __restrict__ vals_out,
                                                                const int32_t* __restrict__ d_n, int shift,
                                                                const int32_t* __restrict__ offs, int nblocks) {
  pdl_wait();
  __shared__ int s_cnt[RS_WARPS][256];
  __shared__ int s_base[256];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int i = threadIdx.x; i < RS_WARPS * 256; i += RS_THREADS) (&s_cnt[0][0])[i] = 0;
  __syncthreads();
  const int n = *d_n;
  // warp w owns the contiguous slice [base + w*32*ITEMS, +32*ITEMS) processed in ITEMS rounds of 32 keys:
  // the (round, lane) order equals the input order, which makes the pass stable
  const int wbase = blockIdx.x * RS_TILE + warp * 32 * RS_ITEMS;
  K key[RS_ITEMS];
  int lrank[RS_ITEMS];
#pragma unroll
  for (int k = 0; k < RS_ITEMS; k++) {
    int i = wbase + k * 32 + lane;
    bool valid = i < n;
    key[k] = valid ? keys_in[i] : (K)0;
    int d = valid ? (int)((key[k] >> shift) & 0xFF) : 256 + lane;  // invalid lanes match nobody
    unsigned peers = __match_any_sync(0xffffffffu, d);
    int prior = valid ? s_cnt[warp][d] : 0;
    __syncwarp();
    lrank[k] = prior + __popc(peers & ((1u << lane) - 1u));
    if (valid && (peers & ((1u << lane) - 1u)) == 0) s_cnt[warp][d] = prior + __popc(peers);
    __syncwarp();
  }
  __syncthreads();
  {  // per digit: exclusive scan over the warps, add the global base of this (digit, block)
    const int d = threadIdx.x;
    int run = offs[d * nblocks + blockIdx.x];
#pragma unroll
    for (int w = 0; w < RS_WARPS; w++) { int c = s_cnt[w][d]; s_cnt[w][d] = run; run += c; }
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < RS_ITEMS; k++) {
    int i = wbase + k * 32 + lane;
    if (i < n) {
      int d = (int)((key[k] >> shift) & 0xFF);
      int pos = s_cnt[warp][d] + lrank[k];
      keys_out[pos] = key[k];
      vals_out[pos] = vals_in[i];
    }
  }
  (void)s_base;
}

// =================================================================================================
//  single-launch radix sort: one thread-block cluster does ALL passes
// =================================================================================================
// The multi-kernel sort above costs 3 launches + a memset per pass (12-24 launches per sort, three sorts per scan); at
// the sizes of this workload (5e4 .. 4e5 keys) every one of them is launch-latency bound.  Here one cluster of CS_CTAS
// CTAs owns the whole sort: per pass each CTA histograms its contiguous chunk in shared memory, a cluster barrier
// publishes the histograms, every CTA derives its per-digit base offsets from ALL histograms through distributed shared
// memory, scatters its chunk tile by tile with the same stable warp ranking as rs_scatter_kernel, and a second cluster
// barrier (release/acquire at cluster scope) makes the scattered keys visible to the peers before the next pass.
constexpr int CS_CTAS = 8;
constexpr int CS_THREADS = 1024;
constexpr int CS_WARPS = CS_THREADS / 32;
constexpr int CS_ITEMS = 8;
constexpr int CS_TILE = CS_THREADS * CS_ITEMS;

template <typename K>
__global__ void __cluster_dims__(CS_CTAS, 1, 1) __launch_bounds__(CS_THREADS, 1)
    cluster_sort_kernel(K* __restrict__ keys_a, uint32_t* __restrict__ vals_a, K* __restrict__ keys_b, uint32_t* __restrict__ vals_b,
                        const int32_t* __restrict__ d_n, int passes) {
  pdl_wait();
  namespace cg = cooperative_groups;
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  extern __shared__ int cs_smem[];
  int* s_hist = cs_smem;                 // [256]   this CTA's digit counts (read by the peers)
  int* s_base = s_hist + 256;            // [256]   running global offset per digit for this CTA
  int* s_scan = s_base + 256;            // [CS_WARPS] scratch of the 256-wide block scan
  int* s_cnt = s_scan + CS_WARPS;        // [CS_WARPS][256] per-warp digit counters of the current tile
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int n = *d_n;
  // contiguous chunk per CTA, tile-aligned so that the (CTA, tile, warp, round, lane) order is the input order
  const int tiles_total = (n + CS_TILE - 1) / CS_TILE;
  const int tiles_per = (tiles_total + CS_CTAS - 1) / CS_CTAS;
  const int lo = min(rank * tiles_per * CS_TILE, n), hi = min(lo + tiles_per * CS_TILE, n);
  for (int p = 0; p < passes; ++p) {
    const K* kin = (p & 1) ? keys_b : keys_a;
    const uint32_t* vin = (p & 1) ? vals_b : vals_a;
    K* kout = (p & 1) ? keys_a : keys_b;
    uint32_t* vout = (p & 1) ? vals_a : vals_b;
    const int shift = 8 * p;
    if (tid < 256) s_hist[tid] = 0;
    __syncthreads();
    for (int i = lo + tid; i < hi; i += CS_THREADS) atomicAdd(&s_hist[(int)((kin[i] >> shift) & 0xFF)], 1);
    cluster.sync();
    {  // base[d] = (keys with a smaller digit, all CTAs) + (keys with digit d in lower-ranked CTAs)
      int tot = 0, mine = 0;
      if (tid < 256) {
        for (int r = 0; r < CS_CTAS; ++r) {
          const int c = cluster.map_shared_rank(s_hist, r)[tid];
          if (r < rank) mine += c;
          tot += c;
        }
      }
      int inc = tot;   // inclusive scan over the 256 digits (threads 0..255 = warps 0..7)
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
      if (lane == 31 && warp < 8) s_scan[warp] = inc;
      __syncthreads();
      if (tid < 256) {
        int woff = 0;
        for (int w = 0; w < warp; ++w) woff += s_scan[w];
        s_base[tid] = woff + inc - tot + mine;
      }
    }
    __syncthreads();
    for (int t0 = lo; t0 < hi; t0 += CS_TILE) {
      for (int i = tid; i < CS_WARPS * 256; i += CS_THREADS) s_cnt[i] = 0;
      __syncthreads();
      const int wbase = t0 + warp * 32 * CS_ITEMS;
      K key[CS_ITEMS];
      int lrank[CS_ITEMS];
#pragma unroll
      for (int k = 0; k < CS_ITEMS; k++) {   // all loads first: the ranking rounds below are separated by warp barriers
        const int i = wbase + k * 32 + lane;
        key[k] = (i < hi) ? kin[i] : (K)0;
      }
#pragma unroll
      for (int k = 0; k < CS_ITEMS; k++) {
        const int i = wbase + k * 32 + lane;
        const bool valid = i < hi;
        const int d = valid ? (int)((key[k] >> shift) & 0xFF) : 256 + lane;
        const unsigned peers = __match_any_sync(0xffffffffu, d);
        const int prior = valid ? s_cnt[warp * 256 + d] : 0;
        __syncwarp();
        lrank[k] = prior + __popc(peers & ((1u << lane) - 1u));
        if (valid && (peers & ((1u << lane) - 1u)) == 0) s_cnt[warp * 256 + d] = prior + __popc(peers);
        __syncwarp();
      }
      __syncthreads();
      if (tid < 256) {  // exclusive scan over the warps, seeded with the running base of this digit
        int run = s_base[tid];
        for (int w = 0; w < CS_WARPS; w++) { const int c = s_cnt[w * 256 + tid]; s_cnt[w * 256 + tid] = run; run += c; }
        s_base[tid] = run;
      }
      __syncthreads();
#pragma unroll
      for (int k = 0; k < CS_ITEMS; k++) {
        const int i = wbase + k * 32 + lane;
        if (i < hi) {
          const int d = (int)((key[k] >> shift) & 0xFF);
          const int pos = s_cnt[warp * 256 + d] + lrank[k];
          kout[pos] = key[k];
          vout[pos] = vin[i];
        }
      }
      __syncthreads();
    }
    __threadfence();
    cluster.sync();
  }
}

static bool g_cs_attr32 = false, g_cs_attr64 = false;

template <typename K>
static int32_t cluster_sort_impl(b2s_handle* h, K*& keys, uint32_t*& vals, K*& keys_alt, uint32_t*& vals_alt, const int32_t* d_n, int key_bits) {
  int passes = (key_bits + 7) / 8;
  if (passes < 1) passes = 1;
  const size_t smem = (size_t)(256 + 256 + CS_WARPS + CS_WARPS * 256) * sizeof(int);
  bool& attr = sizeof(K) == 4 ? g_cs_attr32 : g_cs_attr64;
  if (!attr) {
    B2S_CUDA(cudaFuncSetAttribute(cluster_sort_kernel<K>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr = true;
  }
  ProfScope prof(h, PK_SORT);
  launch_pdl(cluster_sort_kernel<K>, CS_CTAS, CS_THREADS, smem, h->stream, keys, vals, keys_alt, vals_alt, d_n, passes);
  h->launches++;
  B2S_CUDA(cudaGetLastError());
  if (passes & 1) {
    K* tk = keys; keys = keys_alt; keys_alt = tk;
    uint32_t* tv = vals; vals = vals_alt; vals_alt = tv;
  }
  return B2S_OK;
}

static bool use_multi_kernel_sort() {
  static const bool v = getenv("B2S_SORT") && strcmp(getenv("B2S_SORT"), "multi") == 0;
  return v;
}

// returns 0 when the result is in (keys, vals), 1 when it is in (keys_alt, vals_alt) -- callers get the
// pointers swapped so that (keys, vals) always designate the sorted arrays afterwards
template <typename K>
static int32_t radix_sort_impl(b2s_handle* h, K*& keys, uint32_t*& vals, K*& keys_alt, uint32_t*& vals_alt, const int32_t* d_n,
                               size_t n_max, int key_bits, VoxelScratch* own) {
  // one cluster (8 SMs) wins while the sort is launch-latency bound; from ~1e6 keys on the whole GPU has to work on it
  if (!use_multi_kernel_sort() && n_max <= ((size_t)3 << 18)) return cluster_sort_impl<K>(h, keys, vals, keys_alt, vals_alt, d_n, key_bits);
  int nblocks = (int)((n_max + RS_TILE - 1) / RS_TILE);
  if (nblocks < 1) nblocks = 1;
  size_t hist_n = (size_t)256 * nblocks;
  DevBuf& hb = own ? own->sort_hist : h->sort.hist;
  B2S_TRY(hb.ensure((hist_n + 8) * 4 * 2, h->stream));
  int32_t* hist = hb.as<int32_t>();
  int32_t* offs = hist + ((hist_n + 4) & ~(size_t)3);
  int passes = (key_bits + 7) / 8;
  if (passes < 1) passes = 1;
  ProfScope prof(h, PK_SORT);
  for (int p = 0; p < passes; p++) {
    int shift = 8 * p;
    launch_pdl(rs_hist_kernel<K>, nblocks, RS_THREADS, 0, h->stream, keys, d_n, shift, hist, nblocks);
    h->launches++;
    B2S_TRY(scan_impl(h, hist, offs, nullptr, (int32_t)hist_n, hist_n, nullptr, own ? &own->scan_state : nullptr));
    launch_pdl(rs_scatter_kernel<K>, nblocks, RS_THREADS, 0, h->stream, keys, vals, keys_alt, vals_alt, d_n, shift, offs, nblocks);
    h->launches++;
    K* tk = keys; keys = keys_alt; keys_alt = tk;
    uint32_t* tv = vals; vals = vals_alt; vals_alt = tv;
  }
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

int32_t radix_sort_pairs_u32(b2s_handle* h, uint32_t*& keys, uint32_t*& vals, uint32_t*& keys_alt, uint32_t*& vals_alt,
                             const int32_t* d_n, size_t n_max, int key_bits, VoxelScratch* own) {
  return radix_sort_impl<uint32_t>(h, keys, vals, keys_alt, vals_alt, d_n, n_max, key_bits, own);
}
int32_t radix_sort_pairs_u64(b2s_handle* h, uint64_t*& keys, uint32_t*& vals, uint64_t*& keys_alt, uint32_t*& vals_alt,
                             const int32_t* d_n, size_t n_max, int key_bits, VoxelScratch* own) {
  return radix_sort_impl<uint64_t>(h, keys, vals, keys_alt, vals_alt, d_n, n_max, key_bits, own);
}

}  // namespace b2s
