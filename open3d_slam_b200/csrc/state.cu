// state.cu -- A3: every listed submap's device state exported as self-contained host blobs in one batched call, and a blob imported into
// a new submap on any handle (include/b2s.h "session state", DESIGN.md row A3).
//
// Export is one set of launches over every listed submap, on A2's machinery: tile_count_kernel counts the non-EMPTY keys of every tile
// of every fusion and dense table (blockIdx.y = table), the batched scan turns the counts into tile offsets, state_size_kernel derives
// each blob's section lengths from its device counters, and asm_base_kernel scans the sizes into byte offsets.  After the one
// synchronisation for the sizes, state_sections_kernel writes each blob's header and contiguous sections and state_records_kernel the
// (slot, key, payload) record of every live table slot into one staging buffer laid out exactly as the blobs; one copy takes it to the
// host.  A table is mostly empty, so nothing is kept per slot: the scratch scales with tiles.
// Import checks the header on the host, allocates the submap as b2s_submap_create / fuse_reserve / dense_init do, uploads the blob, and
// state_validate_kernel checks every value that is later used as an index: a record claims its slot with atomicCAS(EMPTY -> key), so a
// second record of the slot fails; every link lies in [-1, dn); and the walk of every voxel's chain counts one arrival per member (in the
// new submap's worklist flags, which the sections overwrite afterwards), so a slot reached twice -- a cycle or two merged chains, which
// would hang fusion's chain walks -- fails.  Only a clean error word lets state_scatter_kernel and the copies write the payloads.
#include "assemble.cuh"

namespace b2s {

static_assert(MS_WORDS == B2S_STATE_MSTATE_WORDS, "a blob holds every MS_* word");
static_assert(sizeof(b2s_state_voxel_record) == 24 && sizeof(b2s_state_dense_record) == 64, "record layouts of include/b2s.h");

constexpr long long ST_MAX_BYTES = 1LL << 46;   // one export's total, far above any device memory
constexpr int ST_HDR_WORDS = B2S_STATE_HEADER_BYTES / 8;

__host__ __device__ inline long long st_pad8(long long b) { return (b + 7) & ~7LL; }

struct SubmapCounts { long long dn, nv, ndup, nw, nd; };   // map slots, fusion records, duplicates, worklist entries, dense records

// the byte length of every section of a submap blob (B2S_SS_*); returns the blob's total
__host__ __device__ inline long long submap_sections(const SubmapCounts& c, bool fused, bool dense, long long* len) {
  len[B2S_SS_POSE] = B2S_STATE_POSE_SLOTS * 16 * 8;
  len[B2S_SS_OPTIONS] = st_pad8((long long)sizeof(b2s_mapper_options));
  len[B2S_SS_MSTATE] = B2S_STATE_MSTATE_WORDS * 4;
  len[B2S_SS_BBOX] = 48;
  len[B2S_SS_MAP_XYZ] = len[B2S_SS_MAP_NORMALS] = 24 * c.dn;
  len[B2S_SS_VNEXT] = len[B2S_SS_PSTAMP] = len[B2S_SS_WFLAG] = fused ? st_pad8(4 * c.dn) : 0;
  len[B2S_SS_DUPS] = st_pad8(4 * c.ndup);
  len[B2S_SS_WLIST] = st_pad8(4 * c.nw);
  len[B2S_SS_VOXELS] = (long long)sizeof(b2s_state_voxel_record) * c.nv;
  len[B2S_SS_DENSE_USED] = dense ? 8 : 0;
  len[B2S_SS_DENSE] = (long long)sizeof(b2s_state_dense_record) * c.nd;
  long long total = B2S_STATE_HEADER_BYTES;
  for (int k = 0; k < B2S_SS_COUNT; k++) total += len[k];
  return total;
}
__host__ __device__ inline void section_offsets(const long long* len, long long* off) {
  long long o = B2S_STATE_HEADER_BYTES;
  for (int k = 0; k < B2S_SS_COUNT; k++) { off[k] = o; o += len[k]; }
}

// ---- export -----------------------------------------------------------------------------------------------------------------------------
struct StateJob {                    // one listed submap
  const double* xyz; const double* nrm; const int32_t* d_n;                  // map slots
  const int32_t* ms; const double* pose; const unsigned long long* bbox;
  const int32_t* vnext; const int32_t* pstamp; const int32_t* wflag;        // [capacity (+ 1)]
  const int32_t* dups; const int32_t* wlist; long long wstride;              // both halves; wlist's half stride
  const int32_t* dense_used;
  const int32_t* vlive; const int32_t* dlive;   // live slots of its fusion / dense table (the table's toffs[ntiles]), or a zero word
  long long* c;                                 // device: [0] blob bytes, [1..5] SubmapCounts (state_size_kernel)
  int32_t fused, dense;
  unsigned long long hdr[ST_HDR_WORDS];         // the header words the host knows (magic .. parameters); the rest is filled on the device
  b2s_mapper_options opts;
  __device__ long long live() const { return c[0]; }
  __device__ bool lacks_normals() const { return false; }
  __device__ SubmapCounts counts() const { return SubmapCounts{c[1], c[2], c[3], c[4], c[5]}; }
};

struct KeyTable {                    // one fusion or dense table of a listed submap
  const unsigned long long* keys;
  const int32_t* head; const int32_t* stamp;    // fusion table payload
  const double* sum; const int32_t* cnt;        // dense table payload
  int32_t* tiles; int32_t* toffs;               // per tile: live slots; their exclusive scan
  long long cap;                                // slots (a power of two, a multiple of DX_TILE)
  int32_t ntiles, job, dense, pad;
  __device__ unsigned live_mask(long long s0) const {
    unsigned m = 0;
    if (s0 + DX_ITEMS <= cap) {
      const ulonglong2* k2 = reinterpret_cast<const ulonglong2*>(keys + s0);
#pragma unroll
      for (int q = 0; q < DX_ITEMS / 2; q++) {
        const ulonglong2 v = k2[q];
        m |= (v.x != VOXEL_KEY_EMPTY ? 1u : 0u) << (2 * q);
        m |= (v.y != VOXEL_KEY_EMPTY ? 1u : 0u) << (2 * q + 1);
      }
    } else {
      for (int k = 0; k < DX_ITEMS; k++) if (s0 + k < cap && keys[s0 + k] != VOXEL_KEY_EMPTY) m |= 1u << k;
    }
    return m;
  }
};

__global__ void state_size_kernel(const StateJob* __restrict__ jobs, int n) {
  pdl_wait();
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const StateJob& j = jobs[k];
  SubmapCounts c{*j.d_n, *j.vlive, 0, 0, *j.dlive};
  if (j.fused) {
    c.ndup = min(max(j.ms[MS_NDUP + (j.ms[MS_DUPSEL] & 1)], 0), FUSE_DUP_CAP);
    c.nw = min((long long)max(j.ms[MS_NW + (j.ms[MS_WSEL] & 1)], 0), j.wstride);
  }
  long long len[B2S_SS_COUNT];
  j.c[0] = submap_sections(c, j.fused, j.dense, len);
  j.c[1] = c.dn; j.c[2] = c.nv; j.c[3] = c.ndup; j.c[4] = c.nw; j.c[5] = c.nd;
}

// bytes from src to dst (8-aligned), then zeros up to len; words of 8 bytes when bytes allows, else of 4
__device__ __forceinline__ void st_copy(unsigned char* dst, const void* src, long long bytes, long long len, long long t, long long stride) {
  if ((bytes & 7) == 0 && (reinterpret_cast<uintptr_t>(src) & 7) == 0) {
    unsigned long long* d = reinterpret_cast<unsigned long long*>(dst);
    const unsigned long long* s = static_cast<const unsigned long long*>(src);
    for (long long i = t; i < len / 8; i += stride) d[i] = i < bytes / 8 ? s[i] : 0ull;
  } else {
    uint32_t* d = reinterpret_cast<uint32_t*>(dst);
    const uint32_t* s = static_cast<const uint32_t*>(src);
    for (long long i = t; i < len / 4; i += stride) d[i] = i < bytes / 4 ? s[i] : 0u;
  }
}

// the header and the contiguous sections of blob blockIdx.y
__global__ void __launch_bounds__(AS_THREADS) state_sections_kernel(const StateJob* __restrict__ jobs, const long long* __restrict__ base,
                                                                    unsigned char* __restrict__ out) {
  pdl_wait();
  const StateJob& j = jobs[blockIdx.y];
  const SubmapCounts c = j.counts();
  long long len[B2S_SS_COUNT], off[B2S_SS_COUNT];
  const long long total = submap_sections(c, j.fused, j.dense, len);
  section_offsets(len, off);
  unsigned char* b = out + base[blockIdx.y];
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x, stride = (long long)gridDim.x * blockDim.x;
  if (t < ST_HDR_WORDS) {
    unsigned long long w = j.hdr[t];
    if (t == B2S_STATE_W_TOTAL_BYTES) w = (unsigned long long)total;
    if (t >= B2S_STATE_W_SECTIONS && t < B2S_STATE_W_SECTIONS + B2S_SS_COUNT) w = (unsigned long long)len[t - B2S_STATE_W_SECTIONS];
    if (t == B2S_SP_DN) w = c.dn;
    if (t == B2S_SP_N_VOXELS) w = c.nv;
    if (t == B2S_SP_N_DUPS) w = c.ndup;
    if (t == B2S_SP_N_WLIST) w = c.nw;
    if (t == B2S_SP_N_DENSE) w = c.nd;
    reinterpret_cast<unsigned long long*>(b)[t] = w;
  }
  st_copy(b + off[B2S_SS_POSE], j.pose, len[B2S_SS_POSE], len[B2S_SS_POSE], t, stride);
  st_copy(b + off[B2S_SS_OPTIONS], &j.opts, sizeof(b2s_mapper_options), len[B2S_SS_OPTIONS], t, stride);
  st_copy(b + off[B2S_SS_MSTATE], j.ms, len[B2S_SS_MSTATE], len[B2S_SS_MSTATE], t, stride);
  st_copy(b + off[B2S_SS_BBOX], j.bbox, 48, 48, t, stride);
  st_copy(b + off[B2S_SS_MAP_XYZ], j.xyz, 24 * c.dn, len[B2S_SS_MAP_XYZ], t, stride);
  st_copy(b + off[B2S_SS_MAP_NORMALS], j.nrm, 24 * c.dn, len[B2S_SS_MAP_NORMALS], t, stride);
  if (j.fused) {
    st_copy(b + off[B2S_SS_VNEXT], j.vnext, 4 * c.dn, len[B2S_SS_VNEXT], t, stride);
    st_copy(b + off[B2S_SS_PSTAMP], j.pstamp, 4 * c.dn, len[B2S_SS_PSTAMP], t, stride);
    st_copy(b + off[B2S_SS_WFLAG], j.wflag, 4 * c.dn, len[B2S_SS_WFLAG], t, stride);
    st_copy(b + off[B2S_SS_DUPS], j.dups + (size_t)(j.ms[MS_DUPSEL] & 1) * FUSE_DUP_CAP, 4 * c.ndup, len[B2S_SS_DUPS], t, stride);
    st_copy(b + off[B2S_SS_WLIST], j.wlist + (size_t)(j.ms[MS_WSEL] & 1) * j.wstride, 4 * c.nw, len[B2S_SS_WLIST], t, stride);
  }
  if (j.dense) st_copy(b + off[B2S_SS_DENSE_USED], j.dense_used, 4, 8, t, stride);
}

// the record of every live slot of table blockIdx.y, in slot order
__global__ void __launch_bounds__(AS_THREADS) state_records_kernel(const KeyTable* __restrict__ tabs, const StateJob* __restrict__ jobs,
                                                                   const long long* __restrict__ base, unsigned char* __restrict__ out) {
  pdl_wait();
  const KeyTable t = tabs[blockIdx.y];
  if ((int)blockIdx.x >= t.ntiles) return;
  const long long s0 = (long long)blockIdx.x * DX_TILE + threadIdx.x * DX_ITEMS;
  const unsigned m = t.live_mask(s0);
  const int rank = tile_rank(__popc(m));
  if (m == 0) return;
  const StateJob& j = jobs[t.job];
  long long len[B2S_SS_COUNT], off[B2S_SS_COUNT];
  submap_sections(j.counts(), j.fused, j.dense, len);
  section_offsets(len, off);
  unsigned char* b = out + base[t.job] + off[t.dense ? B2S_SS_DENSE : B2S_SS_VOXELS];
  long long r = t.toffs[blockIdx.x] + rank;
#pragma unroll
  for (int k = 0; k < DX_ITEMS; k++) {
    if (!((m >> k) & 1u)) continue;
    const long long s = s0 + k;
    if (t.dense) {
      b2s_state_dense_record* d = reinterpret_cast<b2s_state_dense_record*>(b) + r;
      d->key = t.keys[s];
      for (int q = 0; q < 6; q++) d->sum[q] = t.sum[6 * s + q];
      d->slot = (int32_t)s; d->count = t.cnt[s];
    } else {
      b2s_state_voxel_record* v = reinterpret_cast<b2s_state_voxel_record*>(b) + r;
      v->key = t.keys[s]; v->slot = (int32_t)s; v->head = t.head[s]; v->stamp = t.stamp[s]; v->reserved_ = 0;
    }
    r++;
  }
}

static unsigned long long dbits(double v) { unsigned long long u; memcpy(&u, &v, 8); return u; }

int32_t op_export_submap_states(b2s_handle* h, int n, const b2s_submap* const* submaps, void* host, size_t capacity, size_t* offsets) {
  if (n == 0) { if (offsets) offsets[0] = 0; return B2S_OK; }
  AssemblyScratch& A = h->assembly;
  auto tiles_of = [](size_t cap) { return (cap + DX_TILE - 1) / DX_TILE; };
  int m = 0;   // tables
  size_t max_tiles = 1, max_words = 1;
  for (int k = 0; k < n; k++) {
    const b2s_submap* sm = submaps[k];
    for (const size_t cap : {sm->vcap, sm->dense_cap}) {
      if (cap == 0) continue;
      if (tiles_of(cap) > max_tiles) max_tiles = tiles_of(cap);
      m++;
    }
    const size_t w = 3 * (sm->cloud[0]->n_max > sm->capacity ? sm->capacity : sm->cloud[0]->n_max);
    if (w > max_words) max_words = w;
  }
  // tables: [StateJob x n][KeyTable x m][ScanJob x m][zero word] staged from the host; then [base x (n + 1)][c x 6n][words] on the device
  Layout L;
  const size_t t_jobs = L.off((size_t)n * sizeof(StateJob)), t_tabs = L.off((size_t)m * sizeof(KeyTable));
  const size_t t_scan = L.off((size_t)m * sizeof(ScanJob)), t_zero = L.off(4), staged = L.size;
  const size_t t_base = L.off(((size_t)n + 1) * 8), t_c = L.off((size_t)n * 48), t_words = L.off(8);
  B2S_TRY(A.tables.ensure(L.size, h->stream));
  if (A.stage.cap < t_c) B2S_TRY(A.stage.alloc(2 * t_c));   // it also receives the bases; every earlier call synchronised after its upload
  unsigned char* st = A.stage.as<unsigned char>();
  unsigned char* tab = A.tables.as<unsigned char>();
  StateJob* hj = reinterpret_cast<StateJob*>(st + t_jobs);
  KeyTable* ht = reinterpret_cast<KeyTable*>(st + t_tabs);
  ScanJob* hs = reinterpret_cast<ScanJob*>(st + t_scan);
  memset(st + t_zero, 0, 4);
  const int32_t* zero = reinterpret_cast<const int32_t*>(tab + t_zero);
  long long* base = reinterpret_cast<long long*>(tab + t_base);
  long long* cdev = reinterpret_cast<long long*>(tab + t_c);
  int32_t* words = reinterpret_cast<int32_t*>(tab + t_words);
  // slots: the tile states of every table (the region zeroed below), then the tables' tile counts and offsets
  memset(ht, 0, (size_t)m * sizeof(KeyTable));
  size_t state_bytes = 0;
  B2S_TRY(carve(A.slots, h->stream, [&](Layout& S) {
    int t = 0;
    for (int k = 0; k < n; k++)
      for (const size_t cap : {submaps[k]->vcap, submaps[k]->dense_cap})
        if (cap) scan_bind_state(S, hs[t++], tiles_of(cap));
    state_bytes = S.size;
    t = 0;
    for (int k = 0; k < n; k++)
      for (const size_t cap : {submaps[k]->vcap, submaps[k]->dense_cap})
        if (cap) { ht[t].tiles = S.take<int32_t>(tiles_of(cap)); ht[t].toffs = S.take<int32_t>(tiles_of(cap) + 2); t++; }
  }));
  const double mv = h->cfg.map_voxel_size;
  for (int k = 0, t = 0; k < n; k++) {
    const b2s_submap* sm = submaps[k];
    StateJob& J = hj[k];
    memset(&J, 0, sizeof(J));
    const b2s_cloud* map = sm->cloud[0].get();
    J.xyz = map->xyz.as<double>(); J.nrm = map->nrm.as<double>(); J.d_n = map->dn.as<int32_t>();
    J.ms = sm->mstate.as<int32_t>(); J.pose = sm->pose.as<double>(); J.bbox = sm->bbox.as<unsigned long long>();
    J.fused = sm->vcap > 0; J.dense = sm->dense_cap > 0;
    J.vnext = sm->vnext.as<int32_t>(); J.pstamp = sm->pstamp.as<int32_t>(); J.wflag = sm->wflag.as<int32_t>();
    J.dups = sm->dups.as<int32_t>(); J.wlist = sm->wlist.as<int32_t>(); J.wstride = (long long)sm->capacity + 1;
    J.dense_used = sm->dense_used.as<int32_t>();
    J.vlive = J.dlive = zero;
    J.c = cdev + 6 * (size_t)k;
    J.opts = sm->opts;
    unsigned long long* w = J.hdr;
    w[B2S_STATE_W_MAGIC] = B2S_STATE_MAGIC_SUBMAP; w[B2S_STATE_W_VERSION] = B2S_STATE_VERSION; w[B2S_STATE_W_BYTE_ORDER] = B2S_STATE_BYTE_ORDER;
    w[B2S_STATE_W_MAP_VOXEL] = dbits(mv); w[B2S_STATE_W_N_SECTIONS] = B2S_SS_COUNT;
    w[B2S_SP_CAPACITY] = sm->capacity; w[B2S_SP_VCAP] = sm->vcap; w[B2S_SP_STAGE_CAP] = sm->stage_cap; w[B2S_SP_DENSE_CAP] = sm->dense_cap;
    w[B2S_SP_DENSE_VOXEL] = dbits(sm->dense_voxel);
    w[B2S_SP_FLAGS] = (map->has_normals ? B2S_STATE_F_HAS_NORMALS : 0) | (sm->no_normals ? B2S_STATE_F_NO_NORMALS : 0) |
                      (sm->merge_scans ? B2S_STATE_F_MERGE_SCANS : 0) | (sm->dense_has_normals ? B2S_STATE_F_DENSE_HAS_NORMALS : 0);
    for (int d = 0; d < 2; d++) {
      const size_t cap = d ? sm->dense_cap : sm->vcap;
      if (cap == 0) continue;
      const size_t nt = tiles_of(cap);
      KeyTable& T = ht[t];
      T.keys = (d ? sm->dense_keys : sm->vkeys).as<unsigned long long>();
      T.head = sm->vhead.as<int32_t>(); T.stamp = sm->vstamp.as<int32_t>();
      T.sum = sm->dense_sum.as<double>(); T.cnt = sm->dense_cnt.as<int32_t>();
      T.cap = (long long)cap; T.ntiles = (int32_t)nt; T.job = k; T.dense = d;
      hs[t].in = T.tiles; hs[t].out = T.toffs;
      hs[t].d_n = reinterpret_cast<const int32_t*>(tab + t_tabs + (size_t)t * sizeof(KeyTable) + offsetof(KeyTable, ntiles));
      (d ? J.dlive : J.vlive) = T.toffs + nt;
      t++;
    }
  }
  B2S_CUDA(cudaMemcpyAsync(tab, st, staged, cudaMemcpyHostToDevice, h->stream));
  if (state_bytes) B2S_CUDA(cudaMemsetAsync(A.slots.p, 0, state_bytes, h->stream));
  const StateJob* dj = reinterpret_cast<const StateJob*>(tab + t_jobs);
  const KeyTable* dt = reinterpret_cast<const KeyTable*>(tab + t_tabs);
  const ScanJob* ds = reinterpret_cast<const ScanJob*>(tab + t_scan);
  if (m > 0) {
    launch_pdl(tile_count_kernel<KeyTable>, dim3((unsigned)max_tiles, (unsigned)m), AS_THREADS, 0, h->stream, dt);
    h->launches++;
    B2S_TRY(scan_exclusive_i32_batch(h, ds, m, max_tiles));
  }
  launch_pdl(state_size_kernel, (n + 255) / 256, 256, 0, h->stream, dj, n);
  launch_pdl(asm_base_kernel<StateJob, ST_MAX_BYTES>, 1, AS_BASE_THREADS, 0, h->stream, dj, n, base, words, words + 1, h->status.as<uint32_t>());
  h->launches += 2;
  B2S_CUDA(cudaGetLastError());

  // synchronisation 1: the byte offsets
  long long* hb = reinterpret_cast<long long*>(st + t_base);
  B2S_CUDA(cudaMemcpyAsync(hb, base, ((size_t)n + 1) * 8, cudaMemcpyDeviceToHost, h->stream));
  B2S_TRY(check_status(h));
  const size_t total = (size_t)hb[n];
  if (offsets) for (int k = 0; k <= n; k++) offsets[k] = (size_t)hb[k];
  if (!host) return B2S_OK;
  B2S_REQUIRE(total <= capacity, B2S_E_CAPACITY, "the blobs take %zu bytes, the buffer holds %zu (a submap changed since the size call?)",
              total, capacity);
  B2S_TRY(A.blob.ensure(total, h->stream));
  const int bx = grid_for(max_words, AS_THREADS, 2 * device_sms());
  launch_pdl(state_sections_kernel, dim3((unsigned)bx, (unsigned)n), AS_THREADS, 0, h->stream, dj, static_cast<const long long*>(base),
             A.blob.as<unsigned char>());
  h->launches++;
  if (m > 0) {
    launch_pdl(state_records_kernel, dim3((unsigned)max_tiles, (unsigned)m), AS_THREADS, 0, h->stream, dt, dj, static_cast<const long long*>(base),
               A.blob.as<unsigned char>());
    h->launches++;
  }
  B2S_CUDA(cudaGetLastError());
  // synchronisation 2: the data
  B2S_CUDA(cudaMemcpyAsync(host, A.blob.p, total, cudaMemcpyDeviceToHost, h->stream));
  return check_status(h);
}

// ---- import -----------------------------------------------------------------------------------------------------------------------------
enum : uint32_t { SV_SLOT = 1u, SV_KEY = 2u, SV_DUP_SLOT = 4u, SV_LINK = 8u, SV_TWICE = 16u, SV_FLAG = 32u, SV_DUPS = 64u, SV_WLIST = 128u };

struct ImportView {                  // the uploaded blob and the new submap
  const unsigned char* blob; long long off[B2S_SS_COUNT];
  long long dn, nv, ndup, nw, nd, vcap, dcap;
  unsigned long long* vkeys; int32_t* vhead; int32_t* vstamp;
  unsigned long long* dkeys; double* dsum; int32_t* dcnt;
  int32_t* arrivals;                 // one word per map slot, zeroed (the new submap's worklist flags)
  uint32_t* err;
};

// every item of the blob that becomes an index: items [0, nv) voxel records, then dense records, chain links, worklist flags,
// duplicates, worklist entries
__global__ void state_validate_kernel(ImportView v) {
  pdl_wait();
  const b2s_state_voxel_record* vr = reinterpret_cast<const b2s_state_voxel_record*>(v.blob + v.off[B2S_SS_VOXELS]);
  const b2s_state_dense_record* dr = reinterpret_cast<const b2s_state_dense_record*>(v.blob + v.off[B2S_SS_DENSE]);
  const int32_t* vnext = reinterpret_cast<const int32_t*>(v.blob + v.off[B2S_SS_VNEXT]);
  const int32_t* wflag = reinterpret_cast<const int32_t*>(v.blob + v.off[B2S_SS_WFLAG]);
  const int32_t* dups = reinterpret_cast<const int32_t*>(v.blob + v.off[B2S_SS_DUPS]);
  const int32_t* wlist = reinterpret_cast<const int32_t*>(v.blob + v.off[B2S_SS_WLIST]);
  const long long nlinks = v.vcap ? v.dn : 0;
  const long long items = v.nv + v.nd + 2 * nlinks + v.ndup + v.nw;
  uint32_t e = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < items; i += (long long)gridDim.x * blockDim.x) {
    long long r = i;
    if (r < v.nv) {
      const b2s_state_voxel_record x = vr[r];
      if (x.key == VOXEL_KEY_EMPTY) { e |= SV_KEY; continue; }
      if (x.slot < 0 || x.slot >= v.vcap) { e |= SV_SLOT; continue; }
      if (atomicCAS(&v.vkeys[x.slot], VOXEL_KEY_EMPTY, x.key) != VOXEL_KEY_EMPTY) e |= SV_DUP_SLOT;
      // the voxel's chain: every member a map slot that no walk reached before (chains are disjoint and end in -1), so the walks
      // together take at most dn steps and a cycle or two merged chains stop at the first repeat
      for (int32_t to = x.head; to != -1; to = vnext[to]) {
        if (to < 0 || to >= v.dn) { e |= SV_LINK; break; }
        if (atomicAdd(&v.arrivals[to], 1) != 0) { e |= SV_TWICE; break; }
      }
      continue;
    }
    r -= v.nv;
    if (r < v.nd) {
      const unsigned long long key = dr[r].key;
      const int32_t slot = dr[r].slot;
      if (key == VOXEL_KEY_EMPTY) { e |= SV_KEY; continue; }
      if (slot < 0 || slot >= v.dcap) { e |= SV_SLOT; continue; }
      if (atomicCAS(&v.dkeys[slot], VOXEL_KEY_EMPTY, key) != VOXEL_KEY_EMPTY) e |= SV_DUP_SLOT;
      continue;
    }
    r -= v.nd;
    if (r < nlinks) { if (vnext[r] < -1 || vnext[r] >= v.dn) e |= SV_LINK; continue; }   // links of slots in no chain (tombstones) too
    r -= nlinks;
    if (r < nlinks) { if (wflag[r] != 0 && wflag[r] != 1) e |= SV_FLAG; continue; }
    r -= nlinks;
    if (r < v.ndup) { if (dups[r] < 0 || dups[r] >= v.vcap) e |= SV_DUPS; continue; }
    r -= v.ndup;
    if (wlist[r] < 0 || wlist[r] >= v.dn) e |= SV_WLIST;
  }
  if (e) atomicOr(v.err, e);
}

// the records' payloads into their (claimed) slots
__global__ void state_scatter_kernel(ImportView v) {
  pdl_wait();
  const b2s_state_voxel_record* vr = reinterpret_cast<const b2s_state_voxel_record*>(v.blob + v.off[B2S_SS_VOXELS]);
  const b2s_state_dense_record* dr = reinterpret_cast<const b2s_state_dense_record*>(v.blob + v.off[B2S_SS_DENSE]);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < v.nv + v.nd; i += (long long)gridDim.x * blockDim.x) {
    if (i < v.nv) {
      const b2s_state_voxel_record x = vr[i];
      v.vhead[x.slot] = x.head; v.vstamp[x.slot] = x.stamp;
    } else {
      const b2s_state_dense_record& d = dr[i - v.nv];
      for (int q = 0; q < 6; q++) v.dsum[6 * (size_t)d.slot + q] = d.sum[q];
      v.dcnt[d.slot] = d.count;
    }
  }
}

static unsigned long long word(const void* blob, int k) { unsigned long long w; memcpy(&w, static_cast<const unsigned char*>(blob) + 8 * k, 8); return w; }

int32_t op_import_submap_state(b2s_handle* h, const void* blob, size_t n_bytes, b2s_submap** out) {
  // the header, on the host: everything that sizes an allocation or bounds an index
  B2S_REQUIRE(n_bytes >= B2S_STATE_HEADER_BYTES, B2S_E_INVALID, "state blob: %zu bytes, shorter than its header", n_bytes);
  B2S_REQUIRE(word(blob, B2S_STATE_W_MAGIC) == B2S_STATE_MAGIC_SUBMAP, B2S_E_INVALID, "state blob: not a submap blob (magic)");
  B2S_REQUIRE(word(blob, B2S_STATE_W_VERSION) == B2S_STATE_VERSION, B2S_E_INVALID, "state blob: format version %llu, this library reads %d",
              word(blob, B2S_STATE_W_VERSION), B2S_STATE_VERSION);
  B2S_REQUIRE(word(blob, B2S_STATE_W_BYTE_ORDER) == B2S_STATE_BYTE_ORDER, B2S_E_INVALID, "state blob: foreign byte order");
  B2S_REQUIRE(word(blob, B2S_STATE_W_TOTAL_BYTES) == n_bytes, B2S_E_INVALID, "state blob: %zu bytes, its header says %llu", n_bytes,
              word(blob, B2S_STATE_W_TOTAL_BYTES));
  B2S_REQUIRE(word(blob, B2S_STATE_W_MAP_VOXEL) == dbits(h->cfg.map_voxel_size), B2S_E_INVALID,
              "state blob: exported under another map_voxel_size than this handle's %g (the fusion hash is keyed by it)", h->cfg.map_voxel_size);
  B2S_REQUIRE(word(blob, B2S_STATE_W_N_SECTIONS) == B2S_SS_COUNT, B2S_E_INVALID, "state blob: %llu sections, a submap blob has %d",
              word(blob, B2S_STATE_W_N_SECTIONS), (int)B2S_SS_COUNT);
  const unsigned long long capacity = word(blob, B2S_SP_CAPACITY), vcap = word(blob, B2S_SP_VCAP), stage_cap = word(blob, B2S_SP_STAGE_CAP);
  const unsigned long long dcap = word(blob, B2S_SP_DENSE_CAP), flags = word(blob, B2S_SP_FLAGS);
  double dvox;
  { const unsigned long long u = word(blob, B2S_SP_DENSE_VOXEL); memcpy(&dvox, &u, 8); }
  const unsigned long long dn = word(blob, B2S_SP_DN), nv = word(blob, B2S_SP_N_VOXELS), ndup = word(blob, B2S_SP_N_DUPS);
  const unsigned long long nw = word(blob, B2S_SP_N_WLIST), nd = word(blob, B2S_SP_N_DENSE);
  B2S_REQUIRE(capacity >= 1 && capacity <= (1ull << 30), B2S_E_INVALID, "state blob: capacity %llu", capacity);
  B2S_REQUIRE(stage_cap <= (1ull << 30), B2S_E_INVALID, "state blob: stage capacity %llu", stage_cap);
  B2S_REQUIRE(dcap == 0 || (dcap >= (unsigned long long)DX_TILE && dcap <= (1ull << 28) && (dcap & (dcap - 1)) == 0 && dvox > 0.0 &&
                            dvox < INFINITY), B2S_E_INVALID, "state blob: dense table of %llu slots, voxel %g", dcap, dvox);
  B2S_REQUIRE(flags < 16, B2S_E_INVALID, "state blob: flags %llu", flags);
  B2S_REQUIRE(dn <= capacity, B2S_E_INVALID, "state blob: %llu map slots, capacity %llu", dn, capacity);
  B2S_REQUIRE(nv <= vcap && nd <= dcap && ndup <= (unsigned long long)(vcap ? FUSE_DUP_CAP : 0) && nw <= (vcap ? capacity + 1 : 0),
              B2S_E_INVALID, "state blob: counts (%llu voxels, %llu dense voxels, %llu duplicates, %llu worklist entries) beyond the tables",
              nv, nd, ndup, nw);
  long long len[B2S_SS_COUNT], off[B2S_SS_COUNT];
  const SubmapCounts c{(long long)dn, (long long)nv, (long long)ndup, (long long)nw, (long long)nd};
  const long long total = submap_sections(c, vcap > 0, dcap > 0, len);
  for (int k = 0; k < B2S_SS_COUNT; k++)
    B2S_REQUIRE(word(blob, B2S_STATE_W_SECTIONS + k) == (unsigned long long)len[k], B2S_E_INVALID,
                "state blob: section %d holds %llu bytes, its counts give %lld", k, word(blob, B2S_STATE_W_SECTIONS + k), len[k]);
  B2S_REQUIRE((unsigned long long)total == n_bytes, B2S_E_INVALID, "state blob: sections of %lld bytes in %zu", total, n_bytes);
  section_offsets(len, off);
  int32_t ms[MS_WORDS];
  memcpy(ms, static_cast<const unsigned char*>(blob) + off[B2S_SS_MSTATE], sizeof(ms));
  const int dsel = ms[MS_DUPSEL], wsel = ms[MS_WSEL];
  B2S_REQUIRE((dsel == 0 || dsel == 1) && (wsel == 0 || wsel == 1) && (unsigned long long)min(max(ms[MS_NDUP + dsel], 0), FUSE_DUP_CAP) == ndup &&
                  ms[MS_NDUP + dsel] >= 0 && ms[MS_NDUP + (dsel ^ 1)] == 0 && (unsigned long long)(long long)ms[MS_NW + wsel] == nw &&
                  ms[MS_NW + (wsel ^ 1)] == 0 && ms[MS_NTOUCHED] == 0 && ms[MS_TICKET2] == 0 && ms[MS_TMP] == 0,
              B2S_E_INVALID, "state blob: the mapper's state words disagree with the sections");

  return create_object(out, [&](b2s_submap* sm) -> int32_t {
    B2S_TRY(submap_init(h, sm, (size_t)capacity));
    B2S_REQUIRE(vcap == 0 || vcap == fuse_table_slots(sm), B2S_E_INVALID, "state blob: fusion table of %llu slots for capacity %llu", vcap,
                capacity);
    if (vcap) B2S_TRY(fuse_reserve(h, sm));   // the empty table, zero worklist flags (the arrival counters below)
    if (dcap) B2S_TRY(dense_init(h, sm, (size_t)dcap, dvox));
    if (stage_cap) {
      B2S_TRY(sm->stage_xyz.ensure(stage_cap * 24, h->stream));
      B2S_TRY(sm->stage_nrm.ensure(stage_cap * 24, h->stream));
      B2S_TRY(sm->stage_next.ensure(stage_cap * 4, h->stream));
      B2S_TRY(sm->stage_in.ensure(stage_cap * 4, h->stream));
      B2S_TRY(sm->touched.ensure(stage_cap * 4, h->stream));
      sm->stage_cap = stage_cap;
    }
    AssemblyScratch& A = h->assembly;
    B2S_TRY(A.blob.ensure(n_bytes, h->stream));
    B2S_TRY(A.tables.ensure(256, h->stream));
    const unsigned char* d = A.blob.as<unsigned char>();
    uint32_t* err = A.tables.as<uint32_t>();
    B2S_CUDA(cudaMemcpyAsync(A.blob.p, blob, n_bytes, cudaMemcpyHostToDevice, h->stream));
    B2S_CUDA(cudaMemsetAsync(err, 0, 4, h->stream));
    ImportView v;
    memset(&v, 0, sizeof(v));
    v.blob = d;
    for (int k = 0; k < B2S_SS_COUNT; k++) v.off[k] = off[k];
    v.dn = (long long)dn; v.nv = (long long)nv; v.ndup = (long long)ndup; v.nw = (long long)nw; v.nd = (long long)nd;
    v.vcap = (long long)vcap; v.dcap = (long long)dcap;
    v.vkeys = sm->vkeys.as<unsigned long long>(); v.vhead = sm->vhead.as<int32_t>(); v.vstamp = sm->vstamp.as<int32_t>();
    v.dkeys = sm->dense_keys.as<unsigned long long>(); v.dsum = sm->dense_sum.as<double>(); v.dcnt = sm->dense_cnt.as<int32_t>();
    v.arrivals = sm->wflag.as<int32_t>();
    v.err = err;
    const long long items = (long long)(nv + nd + ndup + nw) + (vcap ? 2 * (long long)dn : 0);
    if (items > 0) {
      launch_pdl(state_validate_kernel, grid_for((size_t)items, 256, 4 * device_sms()), 256, 0, h->stream, v);
      h->launches++;
    }
    uint32_t e = 0;
    B2S_TRY(read_back(h, {{&e, err, 4}}));
    B2S_REQUIRE(e == 0, B2S_E_INVALID, "state blob refused (%s%s%s%s%s%s%s%s)", e & SV_SLOT ? " record slot beyond its table" : "",
                e & SV_KEY ? " EMPTY key" : "", e & SV_DUP_SLOT ? " two records of one slot" : "", e & SV_LINK ? " chain link out of range" : "",
                e & SV_TWICE ? " map slot linked twice" : "", e & SV_FLAG ? " worklist flag" : "", e & SV_DUPS ? " duplicate entry out of range" : "",
                e & SV_WLIST ? " worklist entry out of range" : "");
    if (nv + nd > 0) {
      launch_pdl(state_scatter_kernel, grid_for((size_t)(nv + nd), 256, 4 * device_sms()), 256, 0, h->stream, v);
      h->launches++;
    }
    b2s_cloud* map = sm->cloud[0].get();
    auto copy = [&](void* dst, int s, size_t bytes) -> int32_t {
      if (bytes) B2S_CUDA(cudaMemcpyAsync(dst, d + off[s], bytes, cudaMemcpyDeviceToDevice, h->stream));
      return B2S_OK;
    };
    B2S_TRY(copy(sm->pose.p, B2S_SS_POSE, len[B2S_SS_POSE]));
    B2S_TRY(copy(sm->mstate.p, B2S_SS_MSTATE, len[B2S_SS_MSTATE]));
    B2S_TRY(copy(sm->bbox.p, B2S_SS_BBOX, 48));
    B2S_TRY(copy(map->xyz.p, B2S_SS_MAP_XYZ, 24 * dn));
    B2S_TRY(copy(map->nrm.p, B2S_SS_MAP_NORMALS, 24 * dn));
    if (vcap) {
      B2S_TRY(copy(sm->vnext.p, B2S_SS_VNEXT, 4 * dn));
      B2S_TRY(copy(sm->pstamp.p, B2S_SS_PSTAMP, 4 * dn));
      B2S_TRY(copy(sm->wflag.p, B2S_SS_WFLAG, 4 * dn));   // over the arrival counts: past dn they stayed 0
      B2S_TRY(copy(sm->dups.as<int32_t>() + (size_t)dsel * FUSE_DUP_CAP, B2S_SS_DUPS, 4 * ndup));
      B2S_TRY(copy(sm->wlist.as<int32_t>() + (size_t)wsel * (capacity + 1), B2S_SS_WLIST, 4 * nw));
    }
    if (dcap) B2S_TRY(copy(sm->dense_used.p, B2S_SS_DENSE_USED, 4));
    B2S_TRY(cloud_set_count(h, map, (size_t)dn));
    map->has_normals = (flags & B2S_STATE_F_HAS_NORMALS) != 0;
    sm->no_normals = (flags & B2S_STATE_F_NO_NORMALS) != 0;
    sm->merge_scans = (flags & B2S_STATE_F_MERGE_SCANS) != 0;
    sm->dense_has_normals = (flags & B2S_STATE_F_DENSE_HAS_NORMALS) != 0;
    memcpy(&sm->opts, static_cast<const unsigned char*>(blob) + off[B2S_SS_OPTIONS], sizeof(b2s_mapper_options));
    B2S_CUDA(cudaGetLastError());
    return check_status(h);   // the blob's upload buffer is reused by the next call: the copies are done when this returns
  });
}

}  // namespace b2s

using namespace b2s;

extern "C" {

int32_t b2s_submaps_export_state(b2s_handle* h, int32_t n, const b2s_submap* const* submaps, void* host_or_null, size_t capacity,
                                 size_t* offsets_out) {
  B2S_REQUIRE(h && offsets_out, B2S_E_INVALID, "null argument");
  B2S_REQUIRE(n >= 0, B2S_E_INVALID, "n must be >= 0");
  B2S_REQUIRE(n == 0 || submaps, B2S_E_INVALID, "null submap array");
  for (int32_t k = 0; k < n; k++) {
    B2S_REQUIRE(submaps[k], B2S_E_INVALID, "null submap %d", k);
    B2S_REQUIRE(submaps[k]->h == h, B2S_E_INVALID, "submap %d belongs to another handle", k);
  }
  B2S_REQUIRE(n <= B2S_ASSEMBLY_MAX_SUBMAPS, B2S_E_UNSUPPORTED, "%d submaps: one export takes at most %d", n, B2S_ASSEMBLY_MAX_SUBMAPS);
  LOCK(h);
  return op_export_submap_states(h, n, submaps, host_or_null, capacity, offsets_out);
}

int32_t b2s_submap_import_state(b2s_handle* h, const void* blob, size_t n_bytes, b2s_submap** out) {
  B2S_REQUIRE(h && blob && out, B2S_E_INVALID, "null argument");
  LOCK(h);
  return op_import_submap_state(h, blob, n_bytes, out);
}

}  // extern "C"
