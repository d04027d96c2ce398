// Hand-written device primitives for the integration pipeline: a stable LSD radix sort of
// (key, value) pairs whose element count lives in DEVICE memory, and an exclusive prefix sum.
//
// Both are single-pass "chained scan" designs (ONE kernel for the whole sort, one kernel for the
// scan): a tile publishes its local aggregate, looks back over its predecessors' status words
// until it meets an inclusive prefix, publishes its own inclusive prefix and scatters.  Tiles are
// handed out through an atomic ticket, so every predecessor of a running tile is itself running
// or finished (no deadlock regardless of block scheduling).  A status word packs a 2-bit flag and
// a 30-bit count, so flag and value travel in one 32-bit store and no fence is needed.
//
// Why not a library sort: (1) the number of update records K is only known on the device; a
// library call needs it on the host, which costs a stream synchronisation in the middle of every
// integratePointCloud call; (2) passes whose digit is the same for every key (typical for the
// compact bundle keys and for small maps) are detected on the device and skipped.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace vbx {

constexpr int kSortThreads = 256;
constexpr int kSortItems = 16;                              // per thread
constexpr int kSortTile = kSortThreads * kSortItems;        // 4096 elements
constexpr int kSortWarps = kSortThreads / 32;
constexpr int kRadix = 256;
constexpr int kMaxPasses = 8;
constexpr uint32_t kFlagAggregate = 1u << 30, kFlagPrefix = 2u << 30, kValueMask = (1u << 30) - 1u;

struct SortPlan {  // device resident; zeroed by the host before every sort
  uint32_t n;
  uint32_t n_tiles;
  uint32_t final_buf;                 // 0: sorted data is in buffer A (the input), 1: in buffer B
  uint32_t hist_ticket;               // histogram phase: tiles handed out / tiles finished
  uint32_t hist_done;
  uint32_t plan_ready;                // set (after a fence) by the block that finished the last histogram tile
  uint32_t active[kMaxPasses];
  uint32_t src_buf[kMaxPasses];
  uint32_t tile_counter[kMaxPasses];  // radix passes: tiles handed out / tiles scattered
  uint32_t tiles_done[kMaxPasses];
  uint32_t hist[kMaxPasses][kRadix];  // global digit histograms
};

__device__ __forceinline__ uint32_t ld_status(const uint32_t* p) { return *reinterpret_cast<const volatile uint32_t*>(p); }
__device__ __forceinline__ void st_status(uint32_t* p, uint32_t v) { *reinterpret_cast<volatile uint32_t*>(p) = v; }
// thread 0 of the block waits until *p reaches `want`; every thread returns with the writers' data visible
__device__ __forceinline__ void block_wait_for(const uint32_t* p, uint32_t want) {
  if (threadIdx.x == 0) {
    while (ld_status(p) < want) __nanosleep(40);
    __threadfence();
  }
  __syncthreads();
}

// Decoupled look-back of tile `tile` (> 0): the sum of the predecessors' aggregates back to (and including) the
// nearest inclusive prefix.  base[t * stride] is tile t's status word.  The words of kLookBatch predecessors
// are requested together -- independent loads, one L2 round trip for the batch instead of one per tile --
// and then consumed in order; a word that is not published yet is polled.
constexpr int kLookBatch = 8;
__device__ __forceinline__ uint32_t look_back(const uint32_t* base, uint32_t stride, uint32_t tile) {
  uint32_t excl = 0;
  uint32_t t = tile;  // predecessors t-1, t-2, ... 0
  while (t > 0) {
    uint32_t v[kLookBatch];
    const uint32_t nb = t < (uint32_t)kLookBatch ? t : (uint32_t)kLookBatch;
#pragma unroll
    for (int i = 0; i < kLookBatch; ++i) {
      if ((uint32_t)i < nb) v[i] = ld_status(base + (size_t)(t - 1u - (uint32_t)i) * stride);
    }
#pragma unroll
    for (int i = 0; i < kLookBatch; ++i) {
      if ((uint32_t)i < nb) {
        uint32_t x = v[i];
        while ((x & ~kValueMask) == 0u) x = ld_status(base + (size_t)(t - 1u - (uint32_t)i) * stride);
        excl += x & kValueMask;
        if (x & kFlagPrefix) return excl;
      }
    }
    t -= nb;
  }
  return excl;  // (not reached: tile 0 always publishes a prefix)
}

// exclusive scan of one value per thread over a 256-thread block; returns the exclusive prefix
__device__ __forceinline__ uint32_t block_exclusive_scan_256(uint32_t v, uint32_t* warp_sums /* [8] shared */) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  if (lane == 31) warp_sums[warp] = inc;
  __syncthreads();
  uint32_t base = 0;
#pragma unroll
  for (int w = 0; w < kSortWarps; ++w) {
    if (w < warp) base += warp_sums[w];
  }
  __syncthreads();
  return base + inc - v;
}

// The whole sort in ONE launch: digit histograms of every pass (one read of the keys), the plan
// (which passes are needed, which buffer feeds each), the radix passes, and the final copy back
// into buffer A for callers that want the result there.  Phases are separated by counters in
// device memory instead of kernel boundaries.  That is deadlock free for any grid size because
// ALL work is handed out by ticket: a block only ever waits for tiles whose tickets were taken by
// blocks that are already running (look-back inside a pass, "all tiles of the previous phase
// done" between phases); a block that is scheduled late finds the tickets gone and walks through.
// Data written by one phase is read by the next on other SMs: loads go through L2 (__ldcg), the
// writers fence before they count themselves done.
// Stable: tiles, warps inside a tile and items inside a warp are all ranked in element order.
template <typename KeyT>
__global__ void __launch_bounds__(kSortThreads, 2)
k_sort(KeyT* keys_a, uint32_t* vals_a, KeyT* keys_b, uint32_t* vals_b, const unsigned long long* d_n, uint32_t n_fixed,
       int passes, const uint32_t* d_key_bits, SortPlan* plan, uint32_t* status_all, uint32_t tiles_cap, int result_in_a) {
  __shared__ uint32_t digit_base[kRadix];             // global exclusive prefix of the digit counts
  __shared__ uint32_t warp_hist[kSortWarps][kRadix];  // phase 1: digit counts of all passes; passes: per-warp counts
  __shared__ uint32_t tile_excl[kRadix];
  __shared__ uint32_t warp_sums[kSortWarps];
  __shared__ uint32_t cur_tile, s_flag;
  // staging of one tile in digit order (32-bit keys only; a one-element dummy otherwise)
  constexpr int kStage = sizeof(KeyT) == 4 ? kSortTile : 1;
  __shared__ uint32_t stage_k[kStage];
  __shared__ uint32_t stage_v[kStage];
  __shared__ uint32_t digit_base_tile[sizeof(KeyT) == 4 ? kRadix : 1];
  static_assert(kSortWarps == kMaxPasses, "the histogram phase reuses warp_hist as hist[pass][digit]");
  // the number of key bits in use may be known on the device only: passes beyond them are not even histogrammed
  if (d_key_bits) passes = min(passes, (int)((*d_key_bits + 7u) / 8u));
  const uint32_t n = d_n ? (uint32_t)min(*d_n, (unsigned long long)tiles_cap * kSortTile) : n_fixed;
  const uint32_t n_tiles = (n + kSortTile - 1) / kSortTile;
  if (n_tiles == 0) {
    if (blockIdx.x == 0 && threadIdx.x == 0) {
      plan->n = 0;
      plan->n_tiles = 0;
      plan->final_buf = 0;
    }
    return;
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned lt_mask = (1u << lane) - 1u;

  // ---- phase 1: histograms (ticketed tiles), status words of the used tiles cleared
  {
    uint32_t(*hist)[kRadix] = warp_hist;
    for (int i = threadIdx.x; i < kMaxPasses * kRadix; i += kSortThreads) (&hist[0][0])[i] = 0;
    uint32_t mine = 0;
    while (true) {
      __syncthreads();
      if (threadIdx.x == 0) cur_tile = atomicAdd(&plan->hist_ticket, 1u);
      __syncthreads();
      const uint32_t tile = cur_tile;
      if (tile >= n_tiles) break;
      ++mine;
      for (int p = 0; p < passes; ++p) status_all[((size_t)p * tiles_cap + tile) * kRadix + threadIdx.x] = 0;
      const uint32_t base = tile * kSortTile;
#pragma unroll 4
      for (int j = 0; j < kSortItems; ++j) {
        const uint32_t e = base + j * kSortThreads + threadIdx.x;
        if (e < n) {
          const KeyT k = keys_a[e];
          for (int p = 0; p < passes; ++p) atomicAdd(&hist[p][(uint32_t)(k >> (8 * p)) & 0xffu], 1u);
        }
      }
    }
    if (mine) {  // (uniform over the block)
      for (int i = threadIdx.x; i < passes * kRadix; i += kSortThreads) {
        const uint32_t v = (&hist[0][0])[i];
        if (v) atomicAdd(&plan->hist[0][0] + i, v);
      }
      __threadfence();
      __syncthreads();
      if (threadIdx.x == 0) s_flag = (atomicAdd(&plan->hist_done, mine) + mine == n_tiles) ? 1u : 0u;
      __syncthreads();
      if (s_flag) {
        // this block finished the last tile: it writes the plan.  A pass whose digit is identical for
        // all keys is the identity permutation and is skipped.
        __threadfence();
        __shared__ uint32_t uniform[kMaxPasses];
        if (threadIdx.x < kMaxPasses) uniform[threadIdx.x] = 0;
        __syncthreads();
        for (int p = 0; p < passes; ++p) {
          if (ld_status(&plan->hist[p][threadIdx.x]) == n) uniform[p] = 1;
        }
        __syncthreads();
        if (threadIdx.x == 0) {
          uint32_t buf = 0;
          for (int p = 0; p < kMaxPasses; ++p) {  // (passes beyond the bits in use stay inactive)
            const uint32_t act = (p < passes && n > 1 && !uniform[p]) ? 1u : 0u;
            plan->active[p] = act;
            plan->src_buf[p] = buf;
            if (act) buf ^= 1u;
          }
          plan->final_buf = buf;
          plan->n = n;
          plan->n_tiles = n_tiles;
          __threadfence();
          st_status(&plan->plan_ready, 1u);
        }
      }
    }
    block_wait_for(&plan->plan_ready, 1u);
  }

  // ---- phase 2: the radix passes
  for (int pass = 0; pass < passes; ++pass) {
    if (!ld_status(&plan->active[pass])) continue;
    const bool from_a = ld_status(&plan->src_buf[pass]) == 0;
    const KeyT* src_k = from_a ? keys_a : keys_b;
    const uint32_t* src_v = from_a ? vals_a : vals_b;
    KeyT* dst_k = from_a ? keys_b : keys_a;
    uint32_t* dst_v = from_a ? vals_b : vals_a;
    uint32_t* status = status_all + (size_t)pass * tiles_cap * kRadix;
    {
      const uint32_t h = ld_status(&plan->hist[pass][threadIdx.x]);
      const uint32_t ex = block_exclusive_scan_256(h, warp_sums);
      digit_base[threadIdx.x] = ex;
    }
    while (true) {
      __syncthreads();
      if (threadIdx.x == 0) cur_tile = atomicAdd(&plan->tile_counter[pass], 1u);
      for (int w = 0; w < kSortWarps; ++w) warp_hist[w][threadIdx.x] = 0;
      __syncthreads();
      const uint32_t tile = cur_tile;
      if (tile >= n_tiles) break;
      const uint32_t base = tile * kSortTile + warp * (32 * kSortItems);
      KeyT key[kSortItems];
      uint32_t val[kSortItems];
      uint32_t rank[kSortItems];
#pragma unroll
      for (int j = 0; j < kSortItems; ++j) {
        const uint32_t e = base + j * 32 + lane;
        key[j] = e < n ? __ldcg(&src_k[e]) : (KeyT)0;
        val[j] = e < n ? __ldcg(&src_v[e]) : 0u;
      }
#pragma unroll
      for (int j = 0; j < kSortItems; ++j) {
        const uint32_t e = base + j * 32 + lane;
        const uint32_t d = e < n ? ((uint32_t)(key[j] >> (8 * pass)) & 0xffu) : 0xffffffffu;
        const unsigned peers = __match_any_sync(0xffffffffu, d);
        const int leader = __ffs(peers) - 1;
        uint32_t before = 0;
        if (lane == leader && d != 0xffffffffu) {
          before = warp_hist[warp][d];
          warp_hist[warp][d] = before + (uint32_t)__popc(peers);
        }
        before = __shfl_sync(0xffffffffu, before, leader);
        rank[j] = before + (uint32_t)__popc(peers & lt_mask);
        __syncwarp();
      }
      __syncthreads();
      // thread d: exclusive offsets of digit d over the warps of this tile, and the tile total
      uint32_t total = 0;
#pragma unroll
      for (int w = 0; w < kSortWarps; ++w) {
        const uint32_t c = warp_hist[w][threadIdx.x];
        warp_hist[w][threadIdx.x] = total;
        total += c;
      }
      // chained scan over the tiles, one digit per thread
      uint32_t* mine = status + (size_t)tile * kRadix + threadIdx.x;
      uint32_t excl = 0;
      if (tile == 0) {
        st_status(mine, kFlagPrefix | total);
      } else {
        st_status(mine, kFlagAggregate | total);
        excl = look_back(status + threadIdx.x, kRadix, tile);
        st_status(mine, kFlagPrefix | (excl + total));
      }
      if constexpr (sizeof(KeyT) == 4) {
        // 32-bit keys (the update records: up to millions per scan): the tile is first put in digit order
        // in shared memory, then written out by consecutive threads -- every digit's elements leave as one
        // contiguous run instead of 32 scattered sectors per store instruction
        const uint32_t tstart = block_exclusive_scan_256(total, warp_sums);  // digit's first position inside the tile
        tile_excl[threadIdx.x] = digit_base[threadIdx.x] + excl - tstart;    // global position of tile position q: + q
        digit_base_tile[threadIdx.x] = tstart;
        __syncthreads();
#pragma unroll
        for (int j = 0; j < kSortItems; ++j) {
          const uint32_t e = base + j * 32 + lane;
          if (e < n) {
            const uint32_t d = (uint32_t)(key[j] >> (8 * pass)) & 0xffu;
            const uint32_t p = digit_base_tile[d] + warp_hist[warp][d] + rank[j];
            stage_k[p] = (uint32_t)key[j];
            stage_v[p] = val[j];
          }
        }
        __syncthreads();
        const uint32_t in_tile = min((uint32_t)kSortTile, n - tile * kSortTile);
#pragma unroll 4
        for (int i = 0; i < kSortItems; ++i) {
          const uint32_t q = i * kSortThreads + threadIdx.x;
          if (q < in_tile) {
            const uint32_t k = stage_k[q];
            const uint32_t pos = tile_excl[(k >> (8 * pass)) & 0xffu] + q;
            dst_k[pos] = (KeyT)k;
            dst_v[pos] = stage_v[q];
          }
        }
      } else {
        tile_excl[threadIdx.x] = excl;
        __syncthreads();
#pragma unroll
        for (int j = 0; j < kSortItems; ++j) {
          const uint32_t e = base + j * 32 + lane;
          if (e < n) {
            const uint32_t d = (uint32_t)(key[j] >> (8 * pass)) & 0xffu;
            const uint32_t pos = digit_base[d] + tile_excl[d] + warp_hist[warp][d] + rank[j];
            dst_k[pos] = key[j];
            dst_v[pos] = val[j];
          }
        }
      }
      // this tile is scattered: visible to every SM before it is counted
      __threadfence();
      __syncthreads();
      if (threadIdx.x == 0) atomicAdd(&plan->tiles_done[pass], 1u);
    }
    block_wait_for(&plan->tiles_done[pass], n_tiles);
  }

  // ---- phase 3: callers that read buffer A get the result there (nobody waits for this phase)
  if (result_in_a && ld_status(&plan->final_buf) != 0) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
      keys_a[i] = __ldcg(&keys_b[i]);
      vals_a[i] = __ldcg(&vals_b[i]);
    }
  }
}

// Exclusive prefix sum of n uint32 (n = *d_n, or n_fixed), chained scan over tiles of 2048.  With a
// permutation the summand at position i is in[perm[i]] for i < *d_limit and 0 beyond (the record
// offsets of the Merged integrator: counts are stored per bundle id, offsets are needed in rank order;
// a few thousand bundles out of a launch sized for every point its own bundle).
constexpr int kScanItems = 8;
constexpr int kScanTile = kSortThreads * kScanItems;
static __global__ void __launch_bounds__(kSortThreads)
k_exclusive_scan(const uint32_t* __restrict__ in, const uint32_t* __restrict__ perm, const uint32_t* __restrict__ d_limit,
                 uint32_t* __restrict__ out, const uint32_t* __restrict__ d_n, uint32_t n_fixed, uint32_t* status,
                 uint32_t* tile_counter, unsigned long long* total_out, unsigned long long* total_ok_out,
                 uint32_t* error_word, unsigned long long total_max, uint32_t error_bit) {
  const uint32_t n = d_n ? *d_n : n_fixed;
  const uint32_t limit = d_limit ? *d_limit : 0xffffffffu;
  // with a limit only positions [0, limit] are scanned (position `limit` holds the total: its summand is 0);
  // the total is also stored at out[n - 1], where the callers read it -- positions in between are not written
  const uint32_t n_eff = (d_limit && limit < n - 1u) ? limit + 1u : n;
  __shared__ uint32_t warp_sums[kSortWarps];
  __shared__ uint32_t cur_tile, tile_base;
  const uint32_t n_tiles = (n_eff + kScanTile - 1) / kScanTile;
  while (true) {
    __syncthreads();
    if (threadIdx.x == 0) cur_tile = atomicAdd(tile_counter, 1u);
    __syncthreads();
    const uint32_t tile = cur_tile;
    if (tile >= n_tiles) break;
    const uint32_t base = tile * kScanTile + threadIdx.x * kScanItems;
    uint32_t v[kScanItems];
    uint32_t sum = 0;
#pragma unroll
    for (int j = 0; j < kScanItems; ++j) {
      const uint32_t e = base + j;
      v[j] = (e < n_eff && e < limit) ? in[perm ? perm[e] : e] : 0u;
      sum += v[j];
    }
    const uint32_t excl_in_tile = block_exclusive_scan_256(sum, warp_sums);
    if (threadIdx.x == kSortThreads - 1) {
      const uint32_t total = excl_in_tile + sum;
      uint32_t excl = 0;
      if (tile == 0) {
        st_status(status, kFlagPrefix | total);
      } else {
        st_status(status + tile, kFlagAggregate | total);
        excl = look_back(status, 1, tile);
        st_status(status + tile, kFlagPrefix | (excl + total));
      }
      tile_base = excl;
    }
    __syncthreads();
    uint32_t run = tile_base + excl_in_tile;
#pragma unroll
    for (int j = 0; j < kScanItems; ++j) {
      if (base + j < n_eff) out[base + j] = run;
      if (base + j == n_eff - 1u) {
        // the last scanned position: its exclusive prefix is the sum of everything (its own summand is 0 by
        // the callers' construction).  What the integration pipeline does with the total (its update-record
        // count): too many for one pass is an error, and nothing downstream runs on a failed call.
        if (n_eff < n) out[n - 1u] = run;
        if (total_out) {
          unsigned long long total = run;
          if (total > total_max) atomicOr(error_word, error_bit);
          *total_out = total;
          if (*reinterpret_cast<volatile uint32_t*>(error_word) != 0u || total > total_max) total = 0;
          *total_ok_out = total;
        }
      }
      run += v[j];
    }
  }
}

}  // namespace vbx
