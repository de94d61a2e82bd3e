// assemble.cuh -- the batched-export machinery shared by A1 / A2 (assemble.cu) and A3 (state.cu): the per-job base scan with its
// capacity check, and the live-slot count of hash tables cut into tiles.  Templates and inline functions only: every file that
// includes it instantiates its own.
#pragma once
#include "common.cuh"

namespace b2s {

constexpr int AS_THREADS = 256;
constexpr int AS_BASE_THREADS = 1024;                  // the base scan walks the jobs 1024 at a time
constexpr long long AS_MAX_POINTS = 0x7fffffffLL / 3;   // the kernels downstream index 3 i in int32

// one CTA: base[k] = live units of the jobs before k (int64, job order), base[njobs] = their total; words[0] = *out_n = the total as
// int32 (0 above MAX_TOTAL, which is reported as ST_CAPACITY), words[1] = a job that contributes a unit has no normals.
// Job: AsmJob (A1), DenseJob (A2) or StateJob (A3, bytes), read through live() and lacks_normals()
template <typename Job, long long MAX_TOTAL = AS_MAX_POINTS>
__global__ void __launch_bounds__(AS_BASE_THREADS) asm_base_kernel(const Job* __restrict__ jobs, int njobs, long long* __restrict__ base,
                                                                   int32_t* out_n, int32_t* words, uint32_t* status) {
  pdl_wait();
  __shared__ long long s_warp[AS_BASE_THREADS / 32];
  __shared__ long long s_carry;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) s_carry = 0;
  int mixed = 0;
  for (int r0 = 0; r0 < njobs; r0 += AS_BASE_THREADS) {
    __syncthreads();
    const int k = r0 + tid;
    long long t = 0;
    if (k < njobs) {
      t = jobs[k].live();
      if (t > 0 && jobs[k].lacks_normals()) mixed = 1;
    }
    long long inc = t;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const long long v = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += v; }
    if (lane == 31) s_warp[warp] = inc;
    __syncthreads();
    long long woff = 0, agg = 0;
    for (int w = 0; w < AS_BASE_THREADS / 32; w++) { const long long v = s_warp[w]; if (w < warp) woff += v; agg += v; }
    const long long carry = s_carry;
    if (k < njobs) base[k] = carry + woff + inc - t;
    __syncthreads();
    if (tid == 0) s_carry = carry + agg;
  }
  mixed = __syncthreads_or(mixed);
  if (tid == 0) {
    const long long total = s_carry;
    base[njobs] = total;
    int32_t cnt = (int32_t)total;
    if (total > MAX_TOTAL) { atomicOr(status, ST_CAPACITY); cnt = 0; }
    *out_n = cnt;
    words[0] = cnt;
    words[1] = mixed;
  }
}

// Live slots of hash tables, tile by tile: a table of `cap` slots is cut into tiles of DX_TILE slots, one CTA per tile (blockIdx.y =
// table), and thread t of a tile looks at the DX_ITEMS consecutive slots s0 = tile * DX_TILE + t * DX_ITEMS ...  Table::live_mask(s0)
// says which of them are live (bit k: slot s0 + k; 0 past the table).  The count pass writes every tile's live slots, the batched scan
// turns them into tile offsets, and a gather recomputes a live slot's rank within its tile with tile_rank.
constexpr int DX_ITEMS = 8;                        // consecutive slots per thread
constexpr int DX_TILE = AS_THREADS * DX_ITEMS;     // slots per CTA

template <typename Table>
__global__ void __launch_bounds__(AS_THREADS) tile_count_kernel(const Table* __restrict__ tabs) {
  pdl_wait();
  const Table t = tabs[blockIdx.y];
  if ((int)blockIdx.x >= t.ntiles) return;
  __shared__ int s_warp[AS_THREADS / 32];
  const int live = warp_sum_i(__popc(t.live_mask((long long)blockIdx.x * DX_TILE + threadIdx.x * DX_ITEMS)));
  if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = live;
  __syncthreads();
  if (threadIdx.x == 0) {
    int s = 0;
    for (int w = 0; w < AS_THREADS / 32; w++) s += s_warp[w];
    t.tiles[blockIdx.x] = s;
  }
}

// the live slots of the threads before this one in its tile (every thread of the CTA calls it with its own count)
__device__ __forceinline__ int tile_rank(int live) {
  __shared__ int s_warp[AS_THREADS / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int inc = live;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += v; }
  if (lane == 31) s_warp[warp] = inc;
  __syncthreads();
  int woff = 0;
  for (int w = 0; w < warp; w++) woff += s_warp[w];
  return woff + inc - live;
}

}  // namespace b2s
