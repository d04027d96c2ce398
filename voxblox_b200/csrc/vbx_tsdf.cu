// TSDF integration on the device: the Simple / Merged / Fast integrators of
// voxblox/src/integrator/tsdf_integrator.cc re-designed as a data-parallel pipeline.
//
//   k_point_keys     transform + validate every point, key it by its end voxel
//                    (bundleRays, cc:340-371)
//   sort             stable radix sort of the point keys: bundles become runs, in the
//                    reference's point order inside a run
//   k_heads          dense list of bundle heads
//   k_merge          the reference's sequential weighted mean (integrateVoxel
//                    cc:387-405) by a TRIPLE of warps: a producer prepares each bundle's
//                    members 32 at a time, a mean and a colour consumer run the two
//                    dependent chains in list order
//   k_rays_count     one thread per ray: the number of voxels the ray will update (from
//                    its DDA set-up, or a DDA walk (RayCaster) for Fast and anti-grazing)
//   scan             offsets of every ray's update records
//   k_rays_emit      DDA walk writing (block id, voxel) -> ray records at the end of the
//                    front half, keyed by local block ids of a scan-private table, without
//                    reading the map; the Merged single walk casts a warp per ray
//                    (k_rays_emit_warp)
//   k_assign         the scan's local ids found or created in the hash, in submission order
//                    (allocateStorageAndGetVoxelPtr cc:91-134); pool slots for new blocks
//   sort             stable radix sort by voxel id: every voxel's updates become one
//                    run, ordered by ray rank
//   k_apply_prep     per sorted record: sdf, weight, colour and a keep bit; the list
//                    of runs longer than 32 updates -- no voxel is read, so it runs
//                    on the sort stream
//   k_apply          updateTsdfVoxel (cc:150-209) applied sequentially per voxel --
//                    clamp-after-every-update semantics preserved exactly, with no
//                    locks and no atomics on voxels.  A warp per long run (free space
//                    near the sensor), then a thread per short run.
//
// Update order.  The reference applies a voxel's updates in whatever order its
// threads reach the voxel's mutex (cc:186); with one thread that is point order for
// Simple / Fast and unordered_map iteration order for Merged.  The device applies
// them in ray-rank order, and the rank IS the reference's one-thread order: point
// order (integration_order_mode) for Simple / Fast; for Merged the iteration order
// of the reference's libstdc++ unordered_map (k_bundle_order, vbx_order.cuh), normal
// bundles before clearing bundles (cc:323-335).  See DESIGN.md "update order".
#include <algorithm>
#include <cassert>
#include <chrono>
#include <cstdio>
#include <cstring>
#include <numeric>
#include <utility>
#include <unordered_map>  // std::__detail::_Prime_rehash_policy: the growth schedule the reference's map follows

#include <cooperative_groups.h>

#include "vbx_engine.h"
#include "vbx_hash.cuh"
#include "vbx_sort.cuh"
#include "vbx_order.cuh"

namespace cg = cooperative_groups;

namespace vbx {

constexpr int kShortRun = 32;  // a voxel run of at most this many updates is applied by one thread, a longer one by a warp

struct ScanParams {
  Pose T;
  F3 origin;
  float voxel_size, voxel_size_inv;
  float trunc, min_ray, max_ray;
  UpdateParams up;
  int L;  // log2(voxels per side)
  int kind;
  int freespace, use_const_weight, allow_clear, carving, anti_grazing;
  int order_mode;      // 0 mixed, 1 sorted (order array)
  uint32_t n;          // points in the cloud
  uint32_t n_groups;   // n / 1024 (MixedThreadSafeIndex)
  float start_inv;     // start_voxel_subsampling_factor * voxel_size_inv
  int max_collisions;
  uint32_t set_offset;  // slot offset of the Fast integrator's approximate sets (ApproxHashSet::offset_)
  uint64_t max_updates;
  // block-ownership sharding (multi-GPU, one map over the GPUs of a box): this rank applies the
  // updates of the voxels in blocks it owns (block_owner() == own_rank) and creates only those
  // blocks; everything before the apply is identical on all ranks
  int own_world, own_rank;
  // the number of voxels a ray updates is known from its DDA set-up alone (no anti-grazing, not the
  // Fast integrator): the ray is walked once, by the emit that writes its update records
  int single_walk;
  // a call whose update records do not fit max_updates_per_pass is emitted and applied in several
  // passes over contiguous ray-slot ranges [emit_lo, emit_hi); emit_base = off[emit_lo]
  uint32_t emit_lo, emit_hi, emit_base;
};

// Everything a scan's kernels take that changes from scan to scan, in device memory (one block per hand-off
// set, ScratchSet::d_args): the kernel nodes of a scan's CUDA graph are built once and read it at run time.
struct ScanArgs {
  ScanParams P;
  const float* xyz;
  const uint8_t* rgba;
  unsigned long long n;  // P.n: the point sort's element count
  uint32_t n_scan;       // P.n + 1: positions of the record-offset scan
  uint32_t nb_cur;       // k_assign reads d_nblocks[nb_cur], writes d_nblocks[nb_cur ^ 1]
  uint32_t count_paths;  // k_apply counts its paths into ScanState::apply_paths (vbx_debug_count_apply_paths)
};

// MixedThreadSafeIndex::getNextIndexImpl, integrator_utils.cc:54-63
__device__ __forceinline__ uint32_t point_order(const ScanParams& P, const uint32_t* order, uint32_t s) {
  if (P.order_mode == 1) return order[s];
  if (P.n_groups * 1024u <= s) return s;
  return (s % P.n_groups) * 1024u + s / P.n_groups;
}

__device__ __forceinline__ F3 load_point(const float* xyz, uint32_t idx) {
  return f3(__ldg(xyz + 3 * idx), __ldg(xyz + 3 * idx + 1), __ldg(xyz + 3 * idx + 2));
}
__device__ __forceinline__ uint32_t load_color(const uint8_t* rgba, uint32_t idx) {
  return __ldg(reinterpret_cast<const uint32_t*>(rgba) + idx);
}

// ------------------------------------------------------- block ownership (multi-GPU)
// One map over the GPUs of a box: rank r owns the blocks with block_owner() == r -- a 2 x 2 x 2
// brick pattern for 8 ranks, so the blocks around the sensor (where most updates land) spread
// over all ranks.  See DESIGN.md "multi-GPU".
__device__ __forceinline__ bool owns_block(const ScanParams& P, int bx, int by, int bz) {
  return P.own_world <= 1 || block_owner(bx, by, bz, P.own_world) == P.own_rank;
}
// An update record's key: (touched id of the block in this call, voxel inside the block) -- e.g.
// 6 + 12 bits when a scan touches ~50 blocks, so the record sort runs three 8-bit passes whatever
// the size of the map.  Records of blocks another rank owns keep their place in the ray's record
// range (offsets are fixed before the walk) under the key 0xffffffff, which sorts behind every
// real key and is skipped by the apply.
constexpr uint32_t kNotOwned = 0xfffffffeu;
constexpr uint32_t kSkipRecord = 0xffffffffu;
__device__ __forceinline__ uint32_t record_key(uint32_t touched_id, uint32_t lin, int L) {
  return touched_id >= kNotOwned ? kSkipRecord : ((touched_id << (3 * L)) | lin);
}

// ------------------------------------------------------------------ bundle keys
// key = [clearing | z | y | x] with the voxel coordinates taken relative to the bounding box of
// the scan's valid points' voxels (k_point_bounds), each axis in exactly the bits its extent
// needs.  Any scan fits 64 bits (|voxel coordinate| < 2^20: at most 21 bits per axis + 1), a
// 640 x 480 room scan needs ~22 -- and the sort only runs the radix passes those bits span.
// Ascending key order = (clearing, z, y, x).
constexpr uint32_t kBoundBias = 1u << 30;
struct KeyLayout {
  int minx, miny, minz;
  int bx, by, bz;  // bits per axis
  bool any;        // the scan has at least one valid point
};
__device__ __forceinline__ int bits_of(uint32_t extent) { return 32 - __clz(extent); }
__device__ __forceinline__ KeyLayout key_layout(const ScanState* st) {
  KeyLayout k;
  const uint32_t mx = st->kb_max[0];
  k.any = mx != 0u;
  k.minx = (int)(0xffffffffu - st->kb_min[0] - kBoundBias);
  k.miny = (int)(0xffffffffu - st->kb_min[1] - kBoundBias);
  k.minz = (int)(0xffffffffu - st->kb_min[2] - kBoundBias);
  k.bx = k.any ? bits_of((uint32_t)((int)(mx - kBoundBias) - k.minx)) : 0;
  k.by = k.any ? bits_of((uint32_t)((int)(st->kb_max[1] - kBoundBias) - k.miny)) : 0;
  k.bz = k.any ? bits_of((uint32_t)((int)(st->kb_max[2] - kBoundBias) - k.minz)) : 0;
  return k;
}
__device__ __forceinline__ uint64_t make_point_key(const KeyLayout& k, I3 v, bool clearing, bool* in_range) {
  const int rx = v.x - k.minx, ry = v.y - k.miny, rz = v.z - k.minz;
  *in_range = k.any && rx >= 0 && ry >= 0 && rz >= 0 && (rx >> k.bx) == 0 && (ry >> k.by) == 0 && (rz >> k.bz) == 0;
  return (uint64_t)(uint32_t)rx | ((uint64_t)(uint32_t)ry << k.bx) | ((uint64_t)(uint32_t)rz << (k.bx + k.by)) |
         ((uint64_t)clearing << (k.bx + k.by + k.bz));
}
// the key a NORMAL bundle ending in voxel v would have (anti-grazing lookup)
__device__ __forceinline__ uint64_t normal_key_of(const KeyLayout& k, int x, int y, int z, bool* in_range) {
  return make_point_key(k, i3(x, y, z), false, in_range);
}
__device__ __forceinline__ bool key_is_clearing(const KeyLayout& k, uint64_t key) {
  return ((key >> (k.bx + k.by + k.bz)) & 1ull) != 0;
}
// the voxel a bundle key stands for
__device__ __forceinline__ I3 key_voxel(const KeyLayout& k, uint64_t key) {
  return i3((int)(key & ((1ull << k.bx) - 1ull)) + k.minx, (int)((key >> k.bx) & ((1ull << k.by) - 1ull)) + k.miny,
            (int)((key >> (k.bx + k.by)) & ((1ull << k.bz) - 1ull)) + k.minz);
}

// ------------------------------------------------------------------- kernels
// Merged, pass 1 over the cloud: the bounding box of the valid points' voxels (and their count).
// Grid-stride over the points, one set of atomics per thread block.
__global__ void __launch_bounds__(256)
k_point_bounds(const ScanArgs* __restrict__ A, uint32_t* __restrict__ first_bits, SortPlan* plan,
               uint32_t* __restrict__ scan_status, uint32_t scan_words, ScanState* st) {
  const ScanParams P = A->P;
  const float* __restrict__ xyz = A->xyz;
  __shared__ uint32_t s_red[7];
  if (threadIdx.x < 7) s_red[threadIdx.x] = 0u;
  const uint32_t words2 = 2u * ((P.n + 31u) >> 5);
  for (uint32_t w = blockIdx.x * blockDim.x + threadIdx.x; w < words2; w += gridDim.x * blockDim.x) {
    first_bits[w] = 0u;  // the first-occurrence bitmaps k_heads fills
  }
  // (the first kernel of the front half also clears what later kernels of its lane count in: the point sort's
  // plan and the status words of the offset scan)
  for (uint32_t w = blockIdx.x * blockDim.x + threadIdx.x; w < (uint32_t)(sizeof(SortPlan) / 4); w += gridDim.x * blockDim.x) {
    reinterpret_cast<uint32_t*>(plan)[w] = 0u;
  }
  for (uint32_t w = blockIdx.x * blockDim.x + threadIdx.x; w < scan_words; w += gridDim.x * blockDim.x) scan_status[w] = 0u;
  __syncthreads();
  // both ends encoded so that the zero-initialised status block means "empty" and atomicMax serves both
  uint32_t hi_x = 0, hi_y = 0, hi_z = 0, lo_x = 0, lo_y = 0, lo_z = 0, n_valid = 0;
  const int lim = kCoordBias - 1;
  for (uint32_t s = blockIdx.x * blockDim.x + threadIdx.x; s < P.n; s += gridDim.x * blockDim.x) {
    const F3 p = load_point(xyz, s);  // (the bounding box does not depend on the point order)
    if (classify_point(p, P.min_ray, P.max_ray, P.allow_clear != 0, P.freespace != 0) == 0) continue;
    const I3 v = grid_index(transform(P.T, p), P.voxel_size_inv);
    if (v.x < -lim || v.x > lim || v.y < -lim || v.y > lim || v.z < -lim || v.z > lim) {
      atomicOr(&st->error, kErrCoordRange);
      continue;
    }
    ++n_valid;
    hi_x = max(hi_x, (uint32_t)v.x + kBoundBias);
    hi_y = max(hi_y, (uint32_t)v.y + kBoundBias);
    hi_z = max(hi_z, (uint32_t)v.z + kBoundBias);
    lo_x = max(lo_x, 0xffffffffu - ((uint32_t)v.x + kBoundBias));
    lo_y = max(lo_y, 0xffffffffu - ((uint32_t)v.y + kBoundBias));
    lo_z = max(lo_z, 0xffffffffu - ((uint32_t)v.z + kBoundBias));
  }
  hi_x = __reduce_max_sync(0xffffffffu, hi_x);
  hi_y = __reduce_max_sync(0xffffffffu, hi_y);
  hi_z = __reduce_max_sync(0xffffffffu, hi_z);
  lo_x = __reduce_max_sync(0xffffffffu, lo_x);
  lo_y = __reduce_max_sync(0xffffffffu, lo_y);
  lo_z = __reduce_max_sync(0xffffffffu, lo_z);
  n_valid = __reduce_add_sync(0xffffffffu, n_valid);
  if ((threadIdx.x & 31) == 0) {
    atomicMax(&s_red[0], hi_x);
    atomicMax(&s_red[1], hi_y);
    atomicMax(&s_red[2], hi_z);
    atomicMax(&s_red[3], lo_x);
    atomicMax(&s_red[4], lo_y);
    atomicMax(&s_red[5], lo_z);
    atomicAdd(&s_red[6], n_valid);
  }
  __syncthreads();
  if (threadIdx.x < 3 && s_red[threadIdx.x]) atomicMax(&st->kb_max[threadIdx.x], s_red[threadIdx.x]);
  if (threadIdx.x >= 3 && threadIdx.x < 6 && s_red[threadIdx.x]) atomicMax(&st->kb_min[threadIdx.x - 3], s_red[threadIdx.x]);
  if (threadIdx.x == 6 && s_red[6]) atomicAdd(&st->n_valid_points, s_red[6]);
}

// Merged, pass 2: key every point by its end voxel (bundleRays, cc:340-371), in the reference's
// point order (position s of that order holds point point_order(s)).
__global__ void k_point_keys(const ScanArgs* __restrict__ A, const uint32_t* __restrict__ order,
                             uint64_t* __restrict__ keys, uint32_t* __restrict__ vals, ScanState* st) {
  const ScanParams P = A->P;
  const float* __restrict__ xyz = A->xyz;
  const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  const KeyLayout kl = key_layout(st);
  if (s == 0) st->key_bits = (uint32_t)(kl.bx + kl.by + kl.bz + 1);
  if (s < P.n) {
    const uint32_t idx = point_order(P, order, s);
    const F3 p = load_point(xyz, idx);
    const int cls = classify_point(p, P.min_ray, P.max_ray, P.allow_clear != 0, P.freespace != 0);
    uint64_t key = kInvalidPointKey;
    if (cls != 0) {
      const I3 v = grid_index(transform(P.T, p), P.voxel_size_inv);
      bool in_range;
      const uint64_t k = make_point_key(kl, v, cls == 2, &in_range);
      if (in_range) key = k;  // (out of range only beyond +-2^20 voxels: flagged by k_point_bounds)
    }
    keys[s] = key;
    vals[s] = idx;
  }
}

// "sorted" integration order: key = |p|^2 (float, widened to double like
// SortedThreadSafeIndex, integrator_utils.cc:24-37); non-negative doubles order as integers.
__global__ void k_sqnorm_keys(uint32_t n, const float* __restrict__ xyz, uint64_t* __restrict__ keys,
                              uint32_t* __restrict__ vals) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const F3 p = load_point(xyz, i);
  const double d = (double)dot3(p, p);
  keys[i] = (uint64_t)__double_as_longlong(d);
  vals[i] = i;
}

// point index -> its position in the reference's point order (the inverse of point_order)
__device__ __forceinline__ uint32_t point_order_inv(const ScanParams& P, const uint32_t* order_inv, uint32_t idx) {
  if (P.order_mode == 1) return order_inv[idx];
  if (P.n_groups * 1024u <= idx) return idx;
  return (idx % 1024u) * P.n_groups + idx / 1024u;
}
__global__ void k_invert_order(uint32_t n, const uint32_t* __restrict__ order, uint32_t* __restrict__ order_inv) {
  const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s < n) order_inv[order[s]] = s;
}

// A bundle's id is its position j in head_list (unordered, dense): the per-ray tables (ray_p / ray_a /
// ray_c / cnt) are indexed by j, update records carry j, and ray_list[rank] = j gives the order.
constexpr uint32_t kBigBundle = 256;         // members from which a bundle is folded before the others
constexpr uint32_t kHeadBig = 0x80000000u;   // head_list entry: sorted position of the head | this flag

// Dense (unordered) list of bundle heads, and the first-occurrence bitmaps: bit t of map m
// (0 normal, 1 clearing) is set when the point at position t of the reference's point order is the
// first of its bundle, i.e. the point whose operator[] inserts the bundle's key into the reference's
// voxel_map / clear_map (bundleRays, cc:340-371).  k_bundle_order turns them into the maps'
// iteration order.
__global__ void k_heads(const ScanArgs* __restrict__ A, const uint64_t* __restrict__ keys, const uint32_t* __restrict__ vals,
                        const uint32_t* __restrict__ order_inv, uint32_t* __restrict__ head_list,
                        uint32_t* __restrict__ big_list, uint32_t* __restrict__ first_bits, uint32_t* __restrict__ cnt,
                        ScanState* st) {
  const ScanParams P = A->P;
  const uint32_t n = P.n;
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  const KeyLayout kl = key_layout(st);
  bool head = false;
  if (i <= n) cnt[i] = 0;
  if (i < n) {
    const uint64_t key = keys[i];
    head = key != kInvalidPointKey && (i == 0 || keys[i - 1] != key);
    if (head) {
      // the stable sort keeps point order inside a bundle: its first member is its first occurrence
      const uint32_t t0 = point_order_inv(P, order_inv, vals[i]);
      const uint32_t words = (n + 31u) >> 5;
      atomicOr(first_bits + (key_is_clearing(kl, (uint64_t)key) ? words : 0u) + (t0 >> 5), 1u << (t0 & 31u));
    }
  }
  const unsigned b = __ballot_sync(0xffffffffu, head);
  if (b) {
    const int lane = threadIdx.x & 31;
    uint32_t base = 0;
    if (lane == 0) base = atomicAdd(&st->n_ray_list, (uint32_t)__popc(b));
    base = __shfl_sync(0xffffffffu, base, 0);
    if (head) {
      // the fold of a bundle is one dependent chain: the long ones are started first (k_merge)
      const bool big = i + kBigBundle < n && keys[i + kBigBundle] == keys[i];
      const uint32_t j = base + __popc(b & ((1u << lane) - 1u));
      head_list[j] = i | (big ? kHeadBig : 0u);
      if (big) big_list[atomicAdd(&st->n_big, 1u)] = j;
    }
  }
}

// LongIndexHash, core/block_hash.h:52-64 (32-bit wrap of x + 17191 y + 17191^2 z)
__device__ __forceinline__ uint32_t long_index_hash(int x, int y, int z) {
  return (uint32_t)x + (uint32_t)y * 17191u + (uint32_t)z * 295530481u;
}
// ---- The reference's bundle order (vbx_order.cuh) in three kernels:
//   k_order_prefix  per-word popcount prefixes of the two first-occurrence bitmaps (one thread block);
//                   the bundle counts B0 (normal map) and B1 (clearing map)
//   k_order_heads   one thread per bundle: its insertion index e into the reference's map (= number of
//                   earlier first occurrences), LongIndexHash of its voxel -> h[map][e], head_of[map][e]
//   k_bundle_order  the iteration order of each map; writes ray_list[rank] = bundle id.  Ranks are
//                   dense: normal bundles 0 .. B0-1 in voxel_map's iteration order, clearing bundles
//                   B0 .. B0+B1-1 in clear_map's (integrateRays(false) runs before integrateRays(true),
//                   cc:323-335).  When a map's tables fit shared memory (16-bit tables: up to ~18 k
//                   bundles; 640 x 480 scans have a few thousand) one block does everything alone -- an
//                   ordinary one-block launch when recent scans say so, see launch_bundle_order; larger
//                   maps (LiDAR: ~50 k bundles) run their late rehash stages grid-wide on global tables
//                   (cooperative launch), the early (small) stages still in block 0's shared memory.
// The clearing map's arrays follow the normal map's at offset g.cap.
__global__ void __launch_bounds__(kOrderThreads)
k_order_prefix(const ScanArgs* __restrict__ A, const uint32_t* __restrict__ first_bits, OrderScratch g, ScanState* st) {
  const uint32_t n = A->P.n;
  __shared__ uint32_t warp_sums[33];
  const uint32_t tid = threadIdx.x;
  const uint32_t words = (n + 31u) >> 5;
  const uint32_t per = (words + kOrderThreads - 1) / kOrderThreads;
  const uint32_t lo = min(tid * per, words), hi = min(lo + per, words);
  for (int mp = 0; mp < 2; ++mp) {
    const uint32_t* bits = first_bits + (mp ? words : 0u);
    uint32_t* wp = g.wp + (mp ? words : 0u);
    uint32_t sum = 0;
    for (uint32_t w = lo; w < hi; ++w) sum += (uint32_t)__popc(bits[w]);  // (independent loads: all in flight together)
    uint32_t total;
    uint32_t run = order_block_scan(sum, warp_sums, &total);
    for (uint32_t w = lo; w < hi; ++w) {
      wp[w] = run;
      run += (uint32_t)__popc(bits[w]);
    }
    if (tid == 0) {
      if (mp == 0) st->n_rays = total; else st->n_clear_rays = total;
    }
  }
}

__global__ void k_order_heads(const ScanArgs* __restrict__ A, const uint64_t* __restrict__ keys, const uint32_t* __restrict__ vals,
                              const uint32_t* __restrict__ order_inv, const uint32_t* __restrict__ head_list,
                              const uint32_t* __restrict__ first_bits, OrderScratch g, const ScanState* st) {
  const ScanParams P = A->P;
  const uint32_t words = (P.n + 31u) >> 5;
  const uint32_t n_heads = st->n_ray_list;
  const KeyLayout kl = key_layout(st);
  for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n_heads; j += gridDim.x * blockDim.x) {
    const uint32_t i = head_list[j] & ~kHeadBig;
    const uint64_t key = (uint64_t)keys[i];
    const uint32_t mp = key_is_clearing(kl, key) ? 1u : 0u;
    const uint32_t t0 = point_order_inv(P, order_inv, vals[i]);
    const uint32_t w = (mp ? words : 0u) + (t0 >> 5);
    const uint32_t e = g.wp[w] + (uint32_t)__popc(first_bits[w] & ((1u << (t0 & 31u)) - 1u));
    if (e >= g.cap) continue;  // (cannot happen: cap = max_points_per_scan)
    const I3 v = key_voxel(kl, key);
    g.h[mp * g.cap + e] = long_index_hash(v.x, v.y, v.z);
    g.head_of[mp * g.cap + e] = j;
  }
}

// A one-block grid needs no cooperative launch: its grid barrier is the block barrier.
__device__ __forceinline__ void order_grid_sync(cg::grid_group& grid) {
  if (gridDim.x == 1) {
    __syncthreads();
  } else {
    grid.sync();
  }
}

// grid-wide version of order_positions (vbx_order.cuh) on global tables; every block of the cooperative
// grid calls it.  cta_tot: one word per block.
__device__ void order_positions_grid(cg::grid_group& grid, const uint32_t* h, const uint32_t* tau, uint32_t* tau_out,
                                     uint32_t* next, uint32_t* bkt, uint32_t* A, uint32_t* bhead, uint32_t m, uint32_t n,
                                     uint32_t tag, uint32_t B, uint32_t* cta_tot, uint32_t* warp_sums) {
  const uint32_t gtid = blockIdx.x * blockDim.x + threadIdx.x, gthreads = gridDim.x * blockDim.x;
  const uint32_t tg = tag << 20;
  for (uint32_t b = gtid; b < m; b += gthreads) {
    const uint32_t gb = h[b] % n;
    bkt[b] = gb;
    const uint32_t old = atomicExch(&bhead[gb], tg | b);
    next[b] = (old >> 20) == tag ? (old & 0xfffffu) : kOrderNil;
  }
  order_grid_sync(grid);
  for (uint32_t b = gtid; b < m; b += gthreads) {
    const uint32_t tb = __ldcg(&tau[b]);
    uint32_t cmin = kOrderNil, size = 0;
    for (uint32_t c = __ldcg(&bhead[bkt[b]]) & 0xfffffu; c != kOrderNil; c = __ldcg(&next[c])) {
      cmin = min(cmin, __ldcg(&tau[c]));
      ++size;
    }
    A[tb] = cmin == tb ? size : 0u;
  }
  order_grid_sync(grid);
  // exclusive suffix sum of A over times: block c owns a contiguous range of times (block 0 the highest),
  // thread t of it a contiguous run inside
  {
    const uint32_t per_cta = (m + gridDim.x - 1) / gridDim.x;
    const uint32_t chi = m > blockIdx.x * per_cta ? m - blockIdx.x * per_cta : 0u;
    const uint32_t clo = chi > per_cta ? chi - per_cta : 0u;
    const uint32_t per = (per_cta + kOrderThreads - 1) / kOrderThreads;
    const uint32_t hi = chi > clo + threadIdx.x * per ? chi - threadIdx.x * per : clo;
    const uint32_t lo = hi > clo + per ? hi - per : clo;
    uint32_t sum = 0;
    for (uint32_t t = lo; t < hi; ++t) sum += __ldcg(&A[t]);
    uint32_t total;
    uint32_t run = order_block_scan(sum, warp_sums, &total);
    if (threadIdx.x == 0) cta_tot[blockIdx.x] = total;
    order_grid_sync(grid);
    uint32_t above = 0;  // elements at times above this block's range
    for (uint32_t c = 0; c < blockIdx.x; ++c) above += __ldcg(&cta_tot[c]);
    run += above;
    for (uint32_t t = hi; t-- > lo;) {
      const uint32_t v = __ldcg(&A[t]);
      A[t] = run;
      run += v;
    }
  }
  order_grid_sync(grid);
  for (uint32_t b = gtid; b < B; b += gthreads) {
    if (b >= m) {  // inserted after this rehash: the insertion index stays its time
      tau_out[b] = b;
      continue;
    }
    const uint32_t tb = __ldcg(&tau[b]);
    uint32_t cmin = kOrderNil, later = 0;
    for (uint32_t c = __ldcg(&bhead[bkt[b]]) & 0xfffffu; c != kOrderNil; c = __ldcg(&next[c])) {
      const uint32_t tc = __ldcg(&tau[c]);
      cmin = min(cmin, tc);
      later += tc > tb ? 1u : 0u;
    }
    tau_out[b] = __ldcg(&A[cmin]) + later;
  }
  order_grid_sync(grid);
}

__global__ void __launch_bounds__(kOrderThreads)
k_bundle_order(RehashSchedule rs, OrderScratch g, uint32_t smem_words, uint32_t* __restrict__ ray_list, uint32_t* cta_tot,
               ScanState* st) {
  extern __shared__ uint32_t order_smem[];
  __shared__ uint32_t warp_sums[33];
  cg::grid_group grid = cg::this_grid();
  const uint32_t tid = threadIdx.x;
  const uint32_t B_of[2] = {st->n_rays, st->n_clear_rays};
  uint32_t n_of[2];
  bool small = true, bad = false;
  for (int mp = 0; mp < 2; ++mp) {
    uint32_t nf = 1;
    for (int k = 0; k < rs.count && rs.m[k] < B_of[mp]; ++k) nf = rs.n[k];
    n_of[mp] = nf;
    if (order_smem_words_needed(B_of[mp], nf) > smem_words) small = false;
    // bucket heads pack the element into 20 bits; cap = max_points_per_scan
    if (B_of[mp] > g.cap || B_of[mp] > (1u << 20) || nf > g.bucket_cap) bad = true;
  }
  if (bad) {
    if (blockIdx.x == 0 && tid == 0) atomicOr(&st->error, kErrUpdatesFull);
    return;
  }
  if (small && blockIdx.x != 0) return;  // (every block takes the same decision: nobody waits at a grid barrier)
  uint32_t base_rank = 0;
  for (int mp = 0; mp < 2; ++mp) {
    const uint32_t B = B_of[mp], n_final = n_of[mp];
    if (B == 0) continue;
    const uint32_t* gh = g.h + mp * g.cap;
    const uint32_t* head_of = g.head_of + mp * g.cap;
    uint32_t *h = order_smem, *tau = h, *tau2 = h, *next = h, *bkt = h, *A = h, *bhead = h;
    if (small) {
      // one block, 16-bit tables in shared memory (the hashes are read from global memory, once per stage)
      const uint32_t pad = (B + 1u) & ~1u;
      uint16_t* t16 = reinterpret_cast<uint16_t*>(order_smem);
      bhead = order_smem + 5u * pad / 2u;
      const uint16_t* pos = order_run<uint16_t>(rs, B, gh, t16, t16 + pad, t16 + 2u * pad, t16 + 3u * pad, t16 + 4u * pad, bhead,
                                                n_final, warp_sums);
      for (uint32_t e = tid; e < B; e += kOrderThreads) ray_list[base_rank + pos[e]] = head_of[e];
      __syncthreads();
      base_rank += B;
      continue;
    }
    // ---- a large map.  Stages whose tables fit shared memory run in block 0 alone ...
    int k_small = 0;       // rehash events [0, k_small) are handled in shared memory
    uint32_t m_small = 0;  // elements present at the last of them
    uint32_t n_small = 1;  // bucket count after it
    for (int k = 0; k < rs.count && rs.m[k] < B; ++k) {
      if (6u * rs.m[k] + (k > 0 ? rs.n[k - 1] : 1u) > smem_words) break;
      k_small = k + 1;
      m_small = rs.m[k];
      n_small = rs.n[k];
    }
    uint32_t* cur = g.tau;   // global arrays of the grid-wide stages
    uint32_t* oth = g.tau2;
    if (blockIdx.x == 0) {
      // the first m_small elements through rehash events 0 .. k_small-1: order_run's loop on a prefix
      h = order_smem;
      tau = h + m_small;
      tau2 = tau + m_small;
      next = tau2 + m_small;
      bkt = next + m_small;
      A = bkt + m_small;
      bhead = A + m_small;
      for (uint32_t e = tid; e < m_small; e += kOrderThreads) {
        h[e] = gh[e];
        tau[e] = e;
      }
      const uint32_t n_clear = k_small > 1 ? rs.n[k_small - 2] : 1u;
      for (uint32_t j = tid; j < n_clear; j += kOrderThreads) bhead[j] = 0u;
      __syncthreads();
      uint32_t n_cur = 1, tag = 1;
      uint32_t* c0 = tau;
      uint32_t* c1 = tau2;
      for (int k = 0; k < k_small; ++k) {
        const uint32_t mk = rs.m[k];
        if (mk > 0) {
          order_positions<uint32_t>(h, c0, c1, next, bkt, A, bhead, mk, n_cur, tag++, warp_sums);
          for (uint32_t e = mk + tid; e < m_small; e += kOrderThreads) c1[e] = e;
          __syncthreads();
          uint32_t* t = c0;
          c0 = c1;
          c1 = t;
        }
        n_cur = rs.n[k];
      }
      for (uint32_t e = tid; e < m_small; e += kOrderThreads) cur[e] = c0[e];
    }
    // ... the rest grid-wide.  Times of elements not yet inserted = their insertion index.
    const uint32_t gtid = blockIdx.x * blockDim.x + tid, gthreads = gridDim.x * blockDim.x;
    for (uint32_t e = m_small + gtid; e < B; e += gthreads) cur[e] = e;
    for (uint32_t j = gtid; j < n_final; j += gthreads) g.bhead[j] = 0u;
    order_grid_sync(grid);
    uint32_t n_cur = n_small, tag = 1;
    for (int k = k_small; k < rs.count && rs.m[k] < B; ++k) {
      order_positions_grid(grid, gh, cur, oth, g.next, g.bkt, g.A, g.bhead, rs.m[k], n_cur, tag++, B, cta_tot, warp_sums);
      uint32_t* t = cur;
      cur = oth;
      oth = t;
      n_cur = rs.n[k];
    }
    order_positions_grid(grid, gh, cur, oth, g.next, g.bkt, g.A, g.bhead, B, n_cur, tag, B, cta_tot, warp_sums);
    for (uint32_t e = gtid; e < B; e += gthreads) ray_list[base_rank + __ldcg(&oth[e])] = head_of[e];
    order_grid_sync(grid);  // the arrays are reused by the other map
    base_rank += B;
  }
}

// Correctly rounded a / b in three dependent operations, given y = RN(1 / b):
//   q = RN(a y);  r = a - q b (exact, one FMA);  a / b = RN(q + r y)
// (Markstein's division step; checked against IEEE division on 8e8 random and adversarial
// operand pairs by tests/exact_div_check.c).  It is only trusted for operands in a
// comfortable exponent band with a non-zero dividend (sign of zero) and a divisor whose
// mantissa is not all ones; anything else is flagged and the bundle's mean is folded again with
// the IEEE division instruction.
__device__ __forceinline__ bool exact_div_operand_ok(float v) {
  const float a = fabsf(v);
  return a > 1e-18f && a < 1e18f;
}
__device__ __forceinline__ float recip_for_exact_div(float b, bool* ok) {
  *ok = exact_div_operand_ok(b) && (__float_as_uint(b) & 0x7fffffu) != 0x7fffffu;
  return __frcp_rn(b);
}

// float4 per staged member: roles 0-2 (the mean's x, y, z) and 3-6 (the colour's r, g, b, a), padded
// to an odd stride so that the lanes' row stores are free of bank conflicts
constexpr int kStageStride = 9;

// One member's step of the fold, as two separate chains (k_merge runs them in separate warps, so that
// neither pays for the other's instructions): the running mean's  state = (state*A + B) / C  with the
// three-operation division (D = RN(1/C); operands it does not trust are recorded in *suspect), and a
// colour channel's  state = round(state*A + B).
__device__ __forceinline__ float fold_step_mean(float state, float4 abcd, bool* suspect) {
  const float tt = fadd(fmul(state, abcd.x), abcd.y);
  const float q = __fmul_rn(tt, abcd.w);
  *suspect |= !exact_div_operand_ok(tt);
  return __fmaf_rn(__fmaf_rn(-q, abcd.z, tt), abcd.w, q);
}
// C round() (half away from zero) of t in [0, 2^22): nearest-even via the 2^23 trick, then bump exact
// ties that went down
__device__ __forceinline__ float fold_step_colour(float state, float4 abcd) {
  const float tt = fadd(fmul(state, abcd.x), abcd.y);
  const float m = fadd(fadd(tt, 8388608.0f), -8388608.0f);
  return (fsub(tt, m) == 0.5f) ? fadd(m, 1.0f) : m;
}

// Up to 32 consecutive members of one bundle, member L of the chunk on lane L (list order).
struct Chunk {
  F3 p;           // the member's point (camera frame) and colour
  uint32_t col;
  float w;        // its weight (0 on lanes past the bundle's end)
  float wl;       // w, or 0 below kEpsilon: such members are skipped (cc:391-393)
  float wb;       // the merged weight the member sees: W + wl_0 + ... + wl_{L-1}, added in list order
  unsigned live;  // the members the fold takes: those that carry weight, or a clearing bundle's first one
};

// One warp's walk over a bundle (the run of equal keys from sorted position i), a chunk per next(), with
// the weight chain W <- W + w of the reference's merge (cc:387-405) that links the chunks.  Loads run
// three deep: when a chunk is handed out, the points of the next one are being gathered (their keys and
// point indices arrived one chunk ago) and the keys of the one after it requested, so no load is waited
// for right after it was issued.  k_merge's producer and its refold of a suspect bundle both walk
// bundles through it.
struct ChunkSource {
  uint32_t n;  // points in the cloud
  bool const_weight;
  const float* __restrict__ xyz;
  const uint8_t* __restrict__ rgba;
  const uint64_t* __restrict__ keys;
  const uint32_t* __restrict__ vals;
  uint64_t key;
  bool clearing;
  uint32_t j0;  // sorted position of the chunk whose keys are in flight
  bool in;      // the next chunk: this lane's member is in the bundle, and its point and colour
  F3 p;
  uint32_t col;
  bool inb_next;  // the chunk after it: key and point index of this lane's position
  uint64_t k_next;
  uint32_t idx_next;
  float mw;   // the bundle's merged weight after the chunks handed out so far
  bool done;  // the bundle's last chunk has been handed out

  __device__ __forceinline__ ChunkSource(const ScanParams& P, const float* __restrict__ xyz_,
                                         const uint8_t* __restrict__ rgba_, const uint64_t* __restrict__ keys_,
                                         const uint32_t* __restrict__ vals_, const KeyLayout& kl, uint32_t i)
      : n(P.n), const_weight(P.use_const_weight != 0), xyz(xyz_), rgba(rgba_), keys(keys_), vals(vals_), mw(0.0f),
        done(false) {
    const int lane = threadIdx.x & 31;
    key = keys[i];
    clearing = key_is_clearing(kl, key);
    const uint32_t jj = i + lane;
    const bool inb = jj < n;
    const uint64_t kk = inb ? keys[jj] : kInvalidPointKey;
    const uint32_t idx = inb ? vals[jj] : 0u;
    j0 = i + 32;
    const uint32_t jn = j0 + lane;
    inb_next = jn < n;
    k_next = inb_next ? keys[jn] : kInvalidPointKey;
    idx_next = inb_next ? vals[jn] : 0u;
    in = inb && kk == key;
    p = f3(0.f, 0.f, 0.f);
    col = 0u;
    if (in) {
      p = load_point(xyz, idx);
      col = load_color(rgba, idx);
    }
  }

  __device__ __forceinline__ Chunk next() {
    const int lane = threadIdx.x & 31;
    Chunk c;
    const int n_in = __popc(__ballot_sync(0xffffffffu, in));  // members form a prefix
    c.p = p;
    c.col = col;
    const bool inc = in;
    if (n_in == 32) {
      in = inb_next && k_next == key;
      if (in) {
        p = load_point(xyz, idx_next);
        col = load_color(rgba, idx_next);
      }
      j0 += 32;
      const uint32_t jn = j0 + lane;
      inb_next = jn < n;
      k_next = inb_next ? keys[jn] : kInvalidPointKey;
      idx_next = inb_next ? vals[jn] : 0u;
    }
    c.w = inc ? point_weight(c.p.z, const_weight) : 0.f;
    c.wl = (inc && !(c.w < VBX_EPS)) ? c.w : 0.f;  // adding +0.0f to W is the identity
    c.wb = mw;
#pragma unroll
    for (int k = 0; k < 31; ++k) {
      const float wk = __shfl_sync(0xffffffffu, c.wl, k);
      if (k < lane) c.wb = fadd(c.wb, wk);
    }
    mw = __shfl_sync(0xffffffffu, fadd(c.wb, c.wl), 31);
    c.live = __ballot_sync(0xffffffffu, c.wl != 0.f);
    if (clearing && c.live) {  // "only take first point when clearing", cc:401-404
      const int k = __ffs(c.live) - 1;
      c.live = 1u << k;
      mw = fadd(__shfl_sync(0xffffffffu, c.wb, k), __shfl_sync(0xffffffffu, c.w, k));
      done = true;
    }
    if (n_in < 32) done = true;
    return c;
  }
};

// Per-ray records.  ray_p (point_G, flags) feeds the two DDA walks; ray_a (point_G - origin and
// its norm, the per-ray half of computeDistance cc:216-228) and ray_c (colour, weight) feed the
// apply kernels, so that an update costs one division and no square root.
__device__ __forceinline__ void store_ray(const ScanParams& P, uint32_t i, F3 point_G, float weight, uint32_t color,
                                          bool clearing, float4* ray_p, float4* ray_a, uint2* ray_c) {
  const F3 po = sub3(point_G, P.origin);
  ray_p[i] = make_float4(point_G.x, point_G.y, point_G.z, __uint_as_float(clearing ? 1u : 0u));
  ray_a[i] = make_float4(po.x, po.y, po.z, norm3(po));
  ray_c[i] = make_uint2(color, __float_as_uint(weight));
}

// One chunk (up to 32 consecutive members of one bundle) handed from the producer warp to the
// consumer warp of a pair through shared memory.
struct ChunkDesc {
  uint32_t live;   // members that carry weight, in list order
  uint32_t head;   // sorted position of the bundle's first member
  uint32_t slot;   // the bundle's ray slot = its rank in the reference's bundle order
  uint32_t flags;
  float mw;        // merged weight after this chunk (final on the bundle's last chunk)
};
constexpr uint32_t kChunkFirst = 1u, kChunkLast = 2u, kChunkSuspect = 4u, kChunkEnd = 8u;

// named barriers of one warp triple (producer, mean consumer, colour consumer): ids 1 / 2 = the chunk
// hand-over of triple 0 / 1 (96 threads), ids 3 / 4 = the two consumers among themselves (64 threads);
// 0 is __syncthreads'.  Literal ids so that ptxas reserves five barriers, not all sixteen.
__device__ __forceinline__ void pair_barrier(int triple_in_block) {
  if (triple_in_block == 0) {
    asm volatile("bar.sync 1, 96;" ::: "memory");
  } else {
    asm volatile("bar.sync 2, 96;" ::: "memory");
  }
}
__device__ __forceinline__ void consumer_barrier(int triple_in_block) {
  if (triple_in_block == 0) {
    asm volatile("bar.sync 3, 64;" ::: "memory");
  } else {
    asm volatile("bar.sync 4, 64;" ::: "memory");
  }
}

// The merge of integrateVoxel (cc:384-407): every bundle's points folded in list order.  The fold
// is one dependent chain per bundle, so the kernel's duration is the largest bundle's chain (up to
// ~3000 points on this workload).  Warps work in TRIPLES on a stream of 32-member chunks:
//   producer         takes the chunks from a ChunkSource (the members and the weight chain W <- W + w,
//                    the only thing a chunk needs from its predecessor besides the running state),
//                    computes everything else that does not depend on the running mean -- p*w, W+w,
//                    RN(1/(W+w)), blendTwoColors' normalised weights -- and stages it per role
//   mean consumer    runs the dependent chain state = (state*A + B) / C over the staged operands (lanes 0-2: x, y, z)
//   colour consumer  runs state = round(state*A + B) (lanes 0-3: r, g, b, a)
// so the preparation of chunk c+1 overlaps the chains of chunk c (two shared-memory slots, one
// named barrier per chunk), also across bundle boundaries, and each chain issues only its own
// instructions (~5 dependent operations per member for the mean, ~7 for a colour channel).
// Launched as 4 blocks per SM; the bound keeps ptxas from spilling to fit a fifth.
__global__ void __launch_bounds__(192, 4)
k_merge(const ScanArgs* __restrict__ A,
        const uint64_t* __restrict__ keys, const uint32_t* __restrict__ vals, const uint32_t* __restrict__ head_list,
        const uint32_t* __restrict__ big_list,
        float4* __restrict__ ray_p, float4* __restrict__ ray_a, uint2* __restrict__ ray_c, uint32_t* __restrict__ cnt,
        ScanState* st) {
  const ScanParams P = A->P;
  const float* __restrict__ xyz = A->xyz;
  const uint8_t* __restrict__ rgba = A->rgba;
  __shared__ float4 stage[2][2][32 * kStageStride];  // [pair in block][slot][member][role]
  __shared__ ChunkDesc desc[2][2];
  const int lane = threadIdx.x & 31;
  __shared__ uint32_t s_col[2];
  const int warp_in_block = threadIdx.x >> 5;
  const int pair_in_block = warp_in_block / 3;  // (the triple this warp belongs to)
  const int warp_role = warp_in_block % 3;      // 0 producer, 1 mean consumer, 2 colour consumer
  const bool producer = warp_role == 0;
  const int bar_id = pair_in_block;
  const uint32_t n_bundles = st->n_ray_list;
  const uint32_t n_big = st->n_big;
  const KeyLayout kl = key_layout(st);
  uint32_t seq = 0;
  if (producer) {
    // Work is handed out by ticket: first the big bundles (their chains bound the kernel's duration, so
    // they start at once), then every other bundle in head_list order.
    while (true) {
      uint32_t ticket = 0;
      if (lane == 0) ticket = atomicAdd(&st->merge_ticket, 1u);
      ticket = __shfl_sync(0xffffffffu, ticket, 0);
      if (ticket >= n_big + n_bundles) break;
      uint32_t b, hl;
      if (ticket < n_big) {
        b = big_list[ticket];
        hl = head_list[b];
      } else {
        b = ticket - n_big;
        hl = head_list[b];
        if (hl & kHeadBig) continue;  // folded through the big list
      }
      const uint32_t i = hl & ~kHeadBig;
      ChunkSource src(P, xyz, rgba, keys, vals, kl, i);
      for (bool first = true; !src.done; first = false) {
        const Chunk c = src.next();
        const float tot = fadd(c.wb, c.w);
        const F3 pw = scale3(c.p, c.w);
        float w1 = 0.f, w2 = 0.f, rtot = 1.f;
        bool bad = false;
        if (c.wl != 0.f) {
          w1 = fdiv(c.wb, tot);  // blendTwoColors' normalised weights, core/common.h:112-113
          w2 = fdiv(c.w, tot);
          bool ok;
          rtot = recip_for_exact_div(tot, &ok);
          bad = !ok;
        }
        const bool any_bad = __any_sync(0xffffffffu, bad);
        // (the slot was released by the consumer two barriers ago)
        const int slot = (int)(seq & 1u);
        float4* st_row = stage[pair_in_block][slot] + lane * kStageStride;
        st_row[0] = make_float4(c.wb, pw.x, tot, rtot);
        st_row[1] = make_float4(c.wb, pw.y, tot, rtot);
        st_row[2] = make_float4(c.wb, pw.z, tot, rtot);
        st_row[3] = make_float4(w1, fmul((float)(int)(c.col & 0xffu), w2), 1.f, 1.f);
        st_row[4] = make_float4(w1, fmul((float)(int)((c.col >> 8) & 0xffu), w2), 1.f, 1.f);
        st_row[5] = make_float4(w1, fmul((float)(int)((c.col >> 16) & 0xffu), w2), 1.f, 1.f);
        st_row[6] = make_float4(w1, fmul((float)(int)(c.col >> 24), w2), 1.f, 1.f);
        if (lane == 0) {
          ChunkDesc d;
          d.live = c.live;
          d.head = i;
          d.slot = b;
          d.flags = (first ? kChunkFirst : 0u) | (src.done ? kChunkLast : 0u) | (any_bad ? kChunkSuspect : 0u);
          d.mw = src.mw;
          desc[pair_in_block][slot] = d;
        }
        pair_barrier(bar_id);
        ++seq;
      }
    }
    if (lane == 0) {
      ChunkDesc d;
      d.live = 0u;
      d.head = 0u;
      d.slot = 0u;
      d.flags = kChunkEnd;
      d.mw = 0.f;
      desc[pair_in_block][seq & 1u] = d;
    }
    pair_barrier(bar_id);
  } else if (warp_role == 2) {
    // ---- colour consumer: lanes 0-3 carry r, g, b, a (floats holding exact integers 0..255)
    const int role = 3 + (lane < 4 ? lane : 3);
    float state = 0.f;
    for (;; ++seq) {
      pair_barrier(bar_id);
      const int slot = (int)(seq & 1u);
      const ChunkDesc d = desc[pair_in_block][slot];
      if (d.flags & kChunkEnd) break;
      if (d.flags & kChunkFirst) state = 0.f;
      const float4* st_col = stage[pair_in_block][slot] + role;
      if (d.live == 0xffffffffu) {
        float4 cur = st_col[0];
#pragma unroll
        for (int k = 0; k < 32; ++k) {
          const float4 nxt = st_col[((k + 1) & 31) * kStageStride];
          state = fold_step_colour(state, cur);
          cur = nxt;
        }
      } else if (d.live) {
        unsigned m = d.live;
        float4 cur = st_col[(__ffs(m) - 1) * kStageStride];
        while (m) {
          m &= m - 1;
          const float4 nxt = st_col[(m ? __ffs(m) - 1 : 0) * kStageStride];
          state = fold_step_colour(state, cur);
          cur = nxt;
        }
      }
      if (d.flags & kChunkLast) {
        const uint32_t mcol = ((uint32_t)(int)__shfl_sync(0xffffffffu, state, 0) & 0xffu) |
                              (((uint32_t)(int)__shfl_sync(0xffffffffu, state, 1) & 0xffu) << 8) |
                              (((uint32_t)(int)__shfl_sync(0xffffffffu, state, 2) & 0xffu) << 16) |
                              (((uint32_t)(int)__shfl_sync(0xffffffffu, state, 3) & 0xffu) << 24);
        if (lane == 0) s_col[pair_in_block] = mcol;
        consumer_barrier(pair_in_block);  // the mean consumer picks the colour up and finishes the bundle
      }
    }
  } else {
    // ---- mean consumer: lanes 0-2 carry x, y, z of the running mean; it also finishes every bundle
    const int role = lane < 3 ? lane : 2;
    float state = 0.f;
    bool suspect = false;
    for (;; ++seq) {
      pair_barrier(bar_id);
      const int slot = (int)(seq & 1u);
      const ChunkDesc d = desc[pair_in_block][slot];
      if (d.flags & kChunkEnd) break;
      if (d.flags & kChunkFirst) {
        state = 0.f;
        suspect = false;
      }
      suspect |= (d.flags & kChunkSuspect) != 0u;
      const float4* st_col = stage[pair_in_block][slot] + role;
      if (d.live == 0xffffffffu) {
        float4 cur = st_col[0];
#pragma unroll
        for (int k = 0; k < 32; ++k) {
          const float4 nxt = st_col[((k + 1) & 31) * kStageStride];
          state = fold_step_mean(state, cur, &suspect);
          cur = nxt;
        }
      } else if (d.live) {
        unsigned m = d.live;
        float4 cur = st_col[(__ffs(m) - 1) * kStageStride];
        while (m) {
          m &= m - 1;
          const float4 nxt = st_col[(m ? __ffs(m) - 1 : 0) * kStageStride];  // the next operand's load overlaps the step
          state = fold_step_mean(state, cur, &suspect);
          cur = nxt;
        }
      }
      if (d.flags & kChunkLast) {
        consumer_barrier(pair_in_block);  // the colour consumer is done with this slot and has published the colour
        const uint32_t i = d.head;
        if (__any_sync(0xffffffffu, suspect)) {
          // the fast division met an operand it does not trust: fold this bundle's mean again with the
          // IEEE division (this warp alone, the slot just consumed as its staging area).  The weight and
          // colour involve no division of the running mean: d.mw and s_col are final.
          state = 0.f;
          float4* st_row = stage[pair_in_block][slot] + lane * kStageStride;
          ChunkSource src(P, xyz, rgba, keys, vals, kl, i);
          while (!src.done) {
            const Chunk c = src.next();
            const float tot = fadd(c.wb, c.w);
            const F3 pw = scale3(c.p, c.w);
            __syncwarp();  // the previous chunk's readers are done
            st_row[0] = make_float4(c.wb, pw.x, tot, 0.f);
            st_row[1] = make_float4(c.wb, pw.y, tot, 0.f);
            st_row[2] = make_float4(c.wb, pw.z, tot, 0.f);
            __syncwarp();
            for (unsigned m = c.live; m; m &= m - 1) {
              const float4 abc = st_col[(__ffs(m) - 1) * kStageStride];
              state = fdiv(fadd(fmul(state, abc.x), abc.y), abc.z);
            }
          }
          if (lane == 0) {
            atomicAdd(&st->n_refold, 1u);
            uint32_t lo = i, hi = P.n;  // first sorted position with a larger key
            const uint64_t k = keys[i];
            while (lo < hi) {
              const uint32_t mid = (lo + hi) >> 1;
              if (keys[mid] <= k) lo = mid + 1; else hi = mid;
            }
            atomicAdd(&st->refold_members, lo - i);
          }
        }
        const F3 mp = f3(__shfl_sync(0xffffffffu, state, 0), __shfl_sync(0xffffffffu, state, 1),
                         __shfl_sync(0xffffffffu, state, 2));
        const uint32_t mcol = s_col[pair_in_block];
        if (lane == 0) {
          const bool clearing = key_is_clearing(kl, (uint64_t)keys[i]);
          const F3 pg = transform(P.T, mp);
          store_ray(P, d.slot, pg, d.mw, mcol, clearing, ray_p, ray_a, ray_c);
          if (P.single_walk) {
            Dda dd;
            dda_setup(dd, P.origin, pg, clearing, P.carving != 0, P.max_ray, P.voxel_size_inv, P.trunc, true);
            cnt[d.slot] = dd.len + 1u;  // RayCaster emits ray_length_in_steps_ + 1 voxels (integrator_utils.cc:111-125)
          }
        }
      }
    }
  }
}

// binary search over the sorted point keys: is there a NORMAL bundle ending in this voxel?
// (the voxel_map.find() of the anti-grazing test, cc:415-422)
__device__ bool bundle_exists(const uint64_t* keys, uint32_t n, uint64_t key) {
  uint32_t lo = 0, hi = n;
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    if (keys[mid] < key) {
      lo = mid + 1;
    } else {
      hi = mid;
    }
  }
  return lo < n && keys[lo] == key;
}

__device__ __forceinline__ bool grazing_skip(const ScanParams& P, const KeyLayout& kl, const uint64_t* keys, uint64_t own,
                                             bool clearing, int x, int y, int z) {
  bool in_range;
  const uint64_t vkey = normal_key_of(kl, x, y, z, &in_range);
  if (!in_range) return false;
  const uint64_t own_normal = clearing ? kInvalidPointKey : own;
  return (clearing || vkey != own_normal) && bundle_exists(keys, P.n, vkey);
}

// ApproxHashSet::replaceHash, utils/approx_hash_array.h:125-134: hash h lives in slot (h & mask) + offset,
// and the reference's load, compare and store there are one exchange.  A slot no hash has been stored in
// since the last clear holds 0, so hash 0 reads as present there, as in the reference (reset_fast_sets).
__device__ __forceinline__ bool replace_hash(unsigned long long* set, uint32_t h, uint32_t offset) {
  return atomicExch(set + (h & kApproxSetMask) + offset, (unsigned long long)h) != h;
}

// The update count of ray t: from its DDA set-up, or (not a single walk) by a first DDA walk.  Merged rays
// come from k_merge's records through the dense ray list; Simple / Fast build their ray from point slot t
// (integrateFunction, cc:269-305 / :488-553).
__device__ __forceinline__ void ray_count(const ScanParams& P, const ScanArgs* __restrict__ A,
                                          const uint32_t* __restrict__ order, const uint64_t* __restrict__ keys,
                                          const uint32_t* __restrict__ head_list, float4* __restrict__ ray_p,
                                          float4* __restrict__ ray_a, uint2* __restrict__ ray_c,
                                          uint32_t* __restrict__ cnt, unsigned long long* set_start,
                                          unsigned long long* set_observed, ScanState* st, uint32_t t) {
  const float* __restrict__ xyz = A->xyz;
  const uint8_t* __restrict__ rgba = A->rgba;
  uint32_t i;
  F3 point_G;
  bool clearing;
  uint64_t own = 0;
  if (P.kind == VBX_MERGED) {
    if (t >= st->n_ray_list) return;
    i = t;  // bundle id j (the count does not depend on the order); head_list[j] = sorted position of its head
    const float4 rp = ray_p[i];
    point_G = f3(rp.x, rp.y, rp.z);
    clearing = (__float_as_uint(rp.w) & 1u) != 0;
    own = keys[head_list[t] & ~kHeadBig];
  } else {
    i = t;
    if (i > P.n) return;
    if (i == P.n) {
      cnt[i] = 0;
      return;
    }
    const uint32_t idx = point_order(P, order, i);
    const F3 p = load_point(xyz, idx);
    const int cls = classify_point(p, P.min_ray, P.max_ray, P.allow_clear != 0, P.freespace != 0);
    if (cls == 0) {
      cnt[i] = 0;
      return;
    }
    point_G = transform(P.T, p);
    clearing = (cls == 2);
    if (P.kind == VBX_FAST) {
      // start-voxel subsampling, cc:507-519
      const I3 g = grid_index(point_G, P.start_inv);
      if (!replace_hash(set_start, long_index_hash(g.x, g.y, g.z), P.set_offset)) {
        cnt[i] = 0;
        return;
      }
    }
    store_ray(P, i, point_G, point_weight(p.z, P.use_const_weight != 0), load_color(rgba, idx), clearing, ray_p,
              ray_a, ray_c);
  }
  if (P.kind != VBX_MERGED) atomicAdd(clearing ? &st->n_clear_rays : &st->n_rays, 1u);  // (Merged: k_bundle_order)

  Dda d;
  dda_setup(d, P.origin, point_G, clearing, P.carving != 0, P.max_ray, P.voxel_size_inv, P.trunc,
            P.kind != VBX_FAST);
  if (P.single_walk) {
    cnt[i] = d.len + 1u;
    return;
  }
  uint32_t count = 0;
  int collisions = 0;
  const int lim = (kCoordBias - 1) << P.L;
  for (unsigned int s = 0; s <= d.len; ++s, dda_advance(d)) {
    if (P.kind == VBX_MERGED && P.anti_grazing) {
      if (grazing_skip(P, key_layout(st), keys, own, clearing, d.cx, d.cy, d.cz)) continue;
    }
    if (P.kind == VBX_FAST) {
      // cc:531-543: stop once the ray runs through voxels other rays already observed
      if (!replace_hash(set_observed, long_index_hash(d.cx, d.cy, d.cz), P.set_offset)) {
        ++collisions;
      } else {
        collisions = 0;
      }
      if (collisions > P.max_collisions) break;
    }
    if (d.cx < -lim || d.cx > lim || d.cy < -lim || d.cy > lim || d.cz < -lim || d.cz > lim) {
      atomicOr(&st->error, kErrCoordRange);
      break;
    }
    ++count;
  }
  cnt[i] = count;
}

// One thread per ray (10 blocks per SM: at most 48 registers, no spills).
__global__ void __launch_bounds__(128, 10)
k_rays_count(const ScanArgs* __restrict__ A, const uint32_t* __restrict__ order, const uint64_t* __restrict__ keys,
             const uint32_t* __restrict__ head_list, float4* __restrict__ ray_p, float4* __restrict__ ray_a,
             uint2* __restrict__ ray_c, uint32_t* __restrict__ cnt, unsigned long long* set_start,
             unsigned long long* set_observed, ScanState* st) {
  const ScanParams P = A->P;
  ray_count(P, A, order, keys, head_list, ray_p, ray_a, ray_c, cnt, set_start, set_observed, st,
            blockIdx.x * blockDim.x + threadIdx.x);
}

// One thread walks slots 0..n in rank order: the reference's one-thread FastTsdfIntegrator schedule, so
// its approximate sets see the same sequence of lookups (vbx_debug_serial_fast; Simple / Fast only).
__global__ void k_rays_count_serial(const ScanArgs* __restrict__ A, const uint32_t* __restrict__ order,
                                    float4* __restrict__ ray_p, float4* __restrict__ ray_a, uint2* __restrict__ ray_c,
                                    uint32_t* __restrict__ cnt, unsigned long long* set_start,
                                    unsigned long long* set_observed, ScanState* st) {
  const ScanParams P = A->P;
  for (uint32_t t = 0; t <= P.n; ++t) {
    ray_count(P, A, order, nullptr, nullptr, ray_p, ray_a, ray_c, cnt, set_start, set_observed, st, t);
  }
}

// A call that is applied in several passes (K > max_updates_per_pass): before each pass.  Blocks
// created by earlier passes already own their slots; the apply work lists restart.
__global__ void k_pass_begin(ScanState* st, unsigned long long pass_updates) {
  st->error &= ~kErrUpdatesFull;
  st->total_updates = st->error ? 0ull : pass_updates;
  st->n_new = 0;
  st->n_long = 0;
  st->long_ticket = 0;
  st->tile_ticket = 0;
}

// First kernel of an asynchronously submitted scan's back half (walk stream: submission order).
__global__ void k_back_begin(ScanState* st, uint32_t* hold) {
  if (*hold) {
    st->error |= kSkipped;  // queued behind a scan that must be redone: do nothing, the host redoes both in order
    st->total_updates = 0;
  } else if (st->error & kErrUpdatesFull) {
    *hold = 1u;
  }
}

// The walk stage's own work, in submission order: one thread block, and the only place blocks are created.
// The ray walk (front half), an upload or a robot-position sphere gave every block it met a local id in the
// hand-off set's private table; here each id listed since the last pass finds or creates its block in the
// hash (allocateStorageAndGetVoxelPtr's find-or-emplace, cc:109-124), becomes the touched id the apply
// resolves, and an existing block's slot_updated becomes touch_bits (cc:128; 0 leaves it alone).  The call's
// last pass clears the table.  Then pool slots for the blocks created by this call
// (updateLayerWithStoredBlocks, cc:137-147), whose slot_updated starts at new_bits: a scan's new block is born
// with all updated bits set (cc:128).
constexpr int kAssignThreads = 512;
__global__ void __launch_bounds__(kAssignThreads)
k_assign(Tables tab, ScanBlocks sb, const ScanArgs* __restrict__ A, uint32_t* __restrict__ nb, SortPlan* record_plan,
         ScanState* st, uint8_t touch_bits, uint8_t new_bits) {
  const uint32_t* __restrict__ nb_in = nb + A->nb_cur;
  uint32_t* __restrict__ nb_out = nb + (A->nb_cur ^ 1u);
  const uint32_t t = threadIdx.x;
  for (uint32_t j = t; j < (uint32_t)(sizeof(SortPlan) / 4); j += blockDim.x) {
    reinterpret_cast<uint32_t*>(record_plan)[j] = 0u;  // for the record sort that follows
  }
  const uint32_t n_ids = min(st->n_touch_ids, sb.cap);
  // a scan skipped behind the hold flag creates nothing (the host redoes it); its table is still cleared
  const bool create = !(st->error & kSkipped);
  // (a call in one pass has emit_hi = 0xffffffff; of the passes of apply_in_passes only the last ends at n)
  const bool last_pass = A->P.emit_hi >= A->P.n;
  if (create) {
    // the blocks this call creates are listed (and take pool slots) in local-id order: a block-wide
    // scan over each round of ids instead of a counter the threads race for
    __shared__ uint32_t warp_new[kAssignThreads / 32];
    const uint32_t lane = t & 31u, w = t >> 5;
    uint32_t n_new = st->n_new;  // (0 in every pass: only this kernel creates blocks)
    uint32_t touched = 0;
    for (uint32_t id0 = st->ids_resolved; id0 < n_ids; id0 += blockDim.x) {
      const uint32_t id = id0 + t;
      const uint64_t key = id < n_ids ? sb.keys[id] : 0ull;
      bool created = false;
      uint32_t hp = 0xffffffffu;
      if (key != 0ull) {
        hp = find_or_insert_block(tab, key, &created, st);
        tab.touched_list[id] = hp;
        if (hp != 0xffffffffu) {
          const int32_t slot = tab.hslot[hp];
          if (slot >= 0 && touch_bits) tab.slot_updated[slot] = touch_bits;  // (*last_block)->updated().set(), cc:128
          ++touched;
        }
      }
      const unsigned int ballot = __ballot_sync(0xffffffffu, created);
      if (lane == 0) warp_new[w] = __popc(ballot);
      __syncthreads();
      uint32_t j = n_new + __popc(ballot & ((1u << lane) - 1u));
      for (uint32_t v = 0; v < blockDim.x / 32; ++v) {
        if (v < w) j += warp_new[v];
        n_new += warp_new[v];
      }
      if (created) {
        if (j < tab.max_blocks) {
          tab.new_list[j] = hp;
        } else {
          atomicOr(&st->error, kErrPoolFull);
        }
      }
      __syncthreads();  // (warp_new is reused by the next round)
    }
    if (touched) atomicAdd(&st->n_touched, touched);
    if (t == 0) st->n_new = n_new;
  }
  if (last_pass) {
    for (uint32_t id = t; id < n_ids; id += blockDim.x) {
      if (sb.keys[id] != 0ull) sb.table[sb.pos[id]] = 0u;
    }
  }
  __syncthreads();  // every new block is in new_list and counted in n_new
  const uint32_t n_blocks_before = *nb_in;
  const uint32_t n_new_all = *reinterpret_cast<volatile uint32_t*>(&st->n_new);
  const uint32_t n_new = min(n_new_all, tab.max_blocks);
  for (uint32_t j = t; j < n_new; j += blockDim.x) {
    const uint32_t slot = n_blocks_before + j;
    if (slot < tab.max_blocks) {
      const uint32_t hp = tab.new_list[j];
      tab.hslot[hp] = (int32_t)slot;
      tab.slot_key[slot] = tab.hkeys[hp];
      tab.slot_updated[slot] = new_bits;
    } else {
      atomicOr(&st->error, kErrPoolFull);
    }
  }
  if (t == 0) {
    const uint32_t after = min(n_blocks_before + n_new_all, tab.max_blocks);
    st->n_blocks = after;
    *nb_out = after;
    st->ids_resolved = n_ids;
    // what the record sort has to look at: voxel bits + the bits of the touched ids handed out
    uint32_t vb = 0;
    while ((tab.vox_per_block >> vb) > 1u) ++vb;
    st->rec_key_bits = vb + (uint32_t)(32 - __clz(st->n_touch_ids));
  }
}

// How a block-run head of a walk becomes the id its update records are keyed by: its local id in the scan's
// private table; k_assign creates the blocks and marks them updated later, in submission order.  in_range: the
// voxel passed the +-2^20-block coordinate check.  0xffffffff when the block has no id (an error is raised).
__device__ __forceinline__ uint32_t walk_block_id(const ScanBlocks& sb, int bx, int by, int bz, bool in_range,
                                                  ScanState* st) {
  if (!in_range) {
    atomicOr(&st->error, kErrCoordRange);
    return 0xffffffffu;
  }
  return scan_block_id(sb, pack3(bx, by, bz), st);
}

// One ray, walked sequentially by the calling thread: RayCaster's loop (integrator_utils.cc:106-125), with
// allocateStorageAndGetVoxelPtr's per-block lookup (cc:91-134) a local id at each block change (walk_block_id).
__device__ void emit_ray_sequential(const ScanParams& P, const ScanBlocks& sb, const uint64_t* __restrict__ keys,
                                    uint32_t i, uint32_t rank, uint32_t head_pos, const float4* __restrict__ ray_p,
                                    const uint32_t* __restrict__ cnt,
                                    const uint32_t* __restrict__ off, uint32_t* __restrict__ ckeys,
                                    uint32_t* __restrict__ cvals, ScanState* st) {
  const uint32_t c = cnt[i];
  if (c == 0 || st->total_updates == 0) return;  // (a failed / to-be-redone call emits nothing)
  if (rank < P.emit_lo || rank >= P.emit_hi) return;   // (not in this pass)
  const float4 rp = ray_p[i];
  const bool clearing = (__float_as_uint(rp.w) & 1u) != 0;
  const F3 point_G = f3(rp.x, rp.y, rp.z);
  Dda d;
  dda_setup(d, P.origin, point_G, clearing, P.carving != 0, P.max_ray, P.voxel_size_inv, P.trunc,
            P.kind != VBX_FAST);
  const uint64_t own = (P.kind == VBX_MERGED) ? keys[head_pos] : 0;
  uint32_t emitted = 0;
  int lbx = INT_MIN, lby = INT_MIN, lbz = INT_MIN;
  uint32_t tid = 0;
  const uint32_t base = off[rank] - P.emit_base;
  const int mask = (1 << P.L) - 1;
  const int lim = (kCoordBias - 1) << P.L;
  for (unsigned int s = 0; s <= d.len && emitted < c; ++s, dda_advance(d)) {
    if (P.kind == VBX_MERGED && P.anti_grazing) {
      if (grazing_skip(P, key_layout(st), keys, own, clearing, d.cx, d.cy, d.cz)) continue;
    }
    const int bx = d.cx >> P.L, by = d.cy >> P.L, bz = d.cz >> P.L;
    if (bx != lbx || by != lby || bz != lbz) {
      if (!owns_block(P, bx, by, bz)) {
        tid = kNotOwned;  // another rank's block: the record keeps its place and is skipped by the apply
      } else {
        const bool in_range = !(d.cx < -lim || d.cx > lim || d.cy < -lim || d.cy > lim || d.cz < -lim || d.cz > lim);
        tid = walk_block_id(sb, bx, by, bz, in_range, st);  // (0xffffffff passes through: the record is skipped)
      }
      lbx = bx;
      lby = by;
      lbz = bz;
    }
    const uint32_t lin = (uint32_t)(d.cx & mask) | ((uint32_t)(d.cy & mask) << P.L) |
                         ((uint32_t)(d.cz & mask) << (2 * P.L));
    // a record = (local id of the block, voxel inside the block) -> ray.  A ray whose block has no
    // id still fills its slots so that offsets stay valid; the error flag set above stops the apply
    // kernels.
    ckeys[base + emitted] = record_key(tid, lin, P.L);
    cvals[base + emitted] = i;
    ++emitted;
  }
}

// One thread per ray, at the end of the front half: like the warp form below, it does not touch the map.
__global__ void k_rays_emit(const ScanArgs* __restrict__ A, ScanBlocks sb, const uint64_t* __restrict__ keys,
                            const uint32_t* __restrict__ ray_list, const uint32_t* __restrict__ head_list,
                            const float4* __restrict__ ray_p, const uint32_t* __restrict__ cnt,
                            const uint32_t* __restrict__ off, uint32_t* __restrict__ ckeys,
                            uint32_t* __restrict__ cvals, ScanState* st) {
  const ScanParams P = A->P;
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t i;
  uint32_t head_pos = 0;
  if (P.kind == VBX_MERGED) {
    if (t >= st->n_ray_list) return;
    i = ray_list[t];  // rank t -> bundle id
    head_pos = head_list[i] & ~kHeadBig;
  } else {
    i = t;
    if (i >= P.n) return;
  }
  emit_ray_sequential(P, sb, keys, i, t, head_pos, ray_p, cnt, off, ckeys, cvals, st);
}

// The same walk cast by a WARP per ray: the trace of the Merged integrator's single walk (a few
// thousand rays of 100-300 steps each, far too few threads for a thread-per-ray walk).  It runs at the
// end of the front half and does not touch the map (it takes no Tables): a block-run head takes its
// block's local id from the scan's private table (walk_block_id), and k_assign resolves those ids
// against the block hash in the walk stage.  The walk is the stable three-way merge of the per-axis
// boundary-crossing chains (vbx_math.cuh, dda_rank):
//   1. lanes 0-2 build the chains T_a(k+1) = RN(T_a(k) + dt_a) in shared memory -- the only
//      sequential part, and plain additions;
//   2. all lanes rank the chain elements (two binary searches each) and scatter the voxel each
//      step reaches into a shared walk list;
//   3. the walk list is turned into records 32 at a time: block changes are found by comparing
//      neighbouring lanes, only the first lane of each block run looks its block up, and the
//      records leave the warp coalesced.
// Bit-identical to the sequential walk (tests/dda_merge_check.cc proves the merge against
// dda_advance on the host); rays the merge form does not cover (axis-parallel components,
// non-finite increments, more than kChainCap crossings on an axis) are walked by lane 0.
constexpr int kChainCap = 256;
constexpr int kWalkCap = 3 * kChainCap;

__global__ void __launch_bounds__(128)
k_rays_emit_warp(const ScanArgs* __restrict__ A, ScanBlocks sb, const uint64_t* __restrict__ keys, const uint32_t* __restrict__ ray_list,
                 const uint32_t* __restrict__ head_list, const float4* __restrict__ ray_p, const uint32_t* __restrict__ cnt, const uint32_t* __restrict__ off,
                 uint32_t* __restrict__ ckeys, uint32_t* __restrict__ cvals, ScanState* st) {
  const ScanParams P = A->P;
  __shared__ float chain_s[4][3][kChainCap];
  __shared__ uint32_t walk_s[4][kWalkCap];
  const int lane = threadIdx.x & 31;
  const int w = threadIdx.x >> 5;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t n_warps = (gridDim.x * blockDim.x) >> 5;
  const uint32_t n_rays = st->n_ray_list;
  if (st->total_updates == 0) return;  // (a failed / to-be-redone call emits nothing)
  const int mask = (1 << P.L) - 1;
  const int lim = (kCoordBias - 1) << P.L;
  for (uint32_t b = warp; b < n_rays; b += n_warps) {
    const uint32_t i = ray_list[b];  // rank b in the reference's bundle order -> bundle id
    const uint32_t c = cnt[i];
    if (c == 0 || b < P.emit_lo || b >= P.emit_hi) continue;
    const float4 rp = ray_p[i];
    const bool clearing = (__float_as_uint(rp.w) & 1u) != 0;
    Dda d;
    dda_setup(d, P.origin, f3(rp.x, rp.y, rp.z), clearing, P.carving != 0, P.max_ray, P.voxel_size_inv, P.trunc, true);
    const unsigned int len = d.len;
    int K[3];
    K[0] = (int)dda_chain_len(d.nx, len);
    K[1] = (int)dda_chain_len(d.ny, len);
    K[2] = (int)dda_chain_len(d.nz, len);
    bool merge_ok = dda_is_regular(d) && K[0] <= kChainCap && K[1] <= kChainCap && K[2] <= kChainCap &&
                    len + 1u <= (unsigned int)kWalkCap && c == len + 1u;
    if (merge_ok) {
      // 1. the chains
      if (lane < 3) {
        float t = lane == 0 ? d.tx : (lane == 1 ? d.ty : d.tz);
        const float dt = lane == 0 ? d.dx : (lane == 1 ? d.dy : d.dz);
        const int kk = K[lane];
        float* dst = chain_s[w][lane];
        for (int k = 0; k < kk; ++k) {
          dst[k] = t;
          t = fadd(t, dt);
        }
      }
      if (lane == 0) walk_s[w][0] = 0u;
      __syncwarp();
      // 2. rank every chain element, scatter the voxel it leads to
      const float* const T[3] = {chain_s[w][0], chain_s[w][1], chain_s[w][2]};
      const int total = K[0] + K[1] + K[2];
      unsigned int emitted = 0;
      bool trusted_all = true;
      for (int e = lane; e < total; e += 32) {
        const int a = e < K[0] ? 0 : (e < K[0] + K[1] ? 1 : 2);
        const int k = e - (a == 0 ? 0 : (a == 1 ? K[0] : K[0] + K[1]));
        unsigned int rank;
        int c3[3];
        const bool trusted = dda_rank(T, K, len, a, k, &rank, c3);
        if (rank < len) {
          trusted_all &= trusted;
          walk_s[w][rank + 1u] = (uint32_t)c3[0] | ((uint32_t)c3[1] << 10) | ((uint32_t)c3[2] << 20);
          ++emitted;
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) emitted += __shfl_xor_sync(0xffffffffu, emitted, o);
      merge_ok = __all_sync(0xffffffffu, trusted_all) && emitted == len;
      __syncwarp();
    }
    if (!merge_ok) {
      if (lane == 0) {
        emit_ray_sequential(P, sb, keys, i, b, head_list[i] & ~kHeadBig, ray_p, cnt, off, ckeys, cvals, st);
      }
      __syncwarp();
      continue;
    }
    // 3. records, 32 steps at a time
    const uint32_t base = off[b] - P.emit_base;
    int cbx = INT_MIN, cby = INT_MIN, cbz = INT_MIN;  // block of the previous chunk's last step
    uint32_t chp = 0u;
    for (unsigned int r0 = 0; r0 <= len; r0 += 32u) {
      const unsigned int r = r0 + (unsigned int)lane;
      const bool valid = r <= len;
      const uint32_t pk = valid ? walk_s[w][r] : 0u;
      const int vx = d.cx + d.sx * (int)(pk & 1023u);
      const int vy = d.cy + d.sy * (int)((pk >> 10) & 1023u);
      const int vz = d.cz + d.sz * (int)(pk >> 20);
      const int bx = vx >> P.L, by = vy >> P.L, bz = vz >> P.L;
      int pbx = __shfl_up_sync(0xffffffffu, bx, 1), pby = __shfl_up_sync(0xffffffffu, by, 1),
          pbz = __shfl_up_sync(0xffffffffu, bz, 1);
      if (lane == 0) {
        pbx = cbx;
        pby = cby;
        pbz = cbz;
      }
      const bool head = valid && (bx != pbx || by != pby || bz != pbz);
      uint32_t hp = 0u;  // the block's local id
      if (head) {
        // the first step inside a block: allocateStorageAndGetVoxelPtr's find-or-create (cc:91-134) happens
        // in k_assign; here the block gets its id in the scan's table
        if (!owns_block(P, bx, by, bz)) {
          hp = kNotOwned;
        } else {
          hp = walk_block_id(sb, bx, by, bz, !(vx < -lim || vx > lim || vy < -lim || vy > lim || vz < -lim || vz > lim), st);
        }
      }
      const unsigned int heads = __ballot_sync(0xffffffffu, head);
      const unsigned int below = heads & (0xffffffffu >> (31 - lane));  // heads at or below this lane
      const int src = below ? 31 - __clz(below) : 0;
      const uint32_t hp_run = __shfl_sync(0xffffffffu, hp, src);
      const uint32_t hp_l = below ? hp_run : chp;
      if (valid) {
        const uint32_t lin = (uint32_t)(vx & mask) | ((uint32_t)(vy & mask) << P.L) | ((uint32_t)(vz & mask) << (2 * P.L));
        ckeys[base + r] = record_key(hp_l, lin, P.L);
        cvals[base + r] = i;
      }
      // carry the last step's block into the next chunk (a full chunk whenever there is a next one)
      cbx = __shfl_sync(0xffffffffu, bx, 31);
      cby = __shfl_sync(0xffffffffu, by, 31);
      cbz = __shfl_sync(0xffffffffu, bz, 31);
      chp = __shfl_sync(0xffffffffu, hp_l, 31);
    }
    __syncwarp();  // the walk list is reused by this warp's next ray
  }
}

// ----------------------------------------------------------------------- apply
struct VoxelRef {
  TsdfVoxel* ptr;
  F3 vo;  // voxel centre - sensor origin
};

__device__ __forceinline__ VoxelRef locate_voxel(const ScanParams& P, const Tables& tab, uint32_t key) {
  const uint32_t hp = tab.touched_list[key >> (3 * P.L)];  // touched id -> hash position
  const uint32_t lin = key & ((1u << (3 * P.L)) - 1u);
  int bx, by, bz;
  unpack3(tab.hkeys[hp], &bx, &by, &bz);
  const int mask = (1 << P.L) - 1;
  const int vx = (bx << P.L) + (int)(lin & mask);
  const int vy = (by << P.L) + (int)((lin >> P.L) & mask);
  const int vz = (bz << P.L) + (int)(lin >> (2 * P.L));
  VoxelRef r;
  // (a block that found no pool slot -- kErrPoolFull -- has hslot < 0: nothing to update)
  const int32_t slot = tab.hslot[hp];
  r.ptr = slot >= 0 ? tab.tsdf + (((size_t)slot) << (3 * P.L)) + lin : nullptr;
  const F3 c = f3(center_coord(vx, P.voxel_size), center_coord(vy, P.voxel_size), center_coord(vz, P.voxel_size));
  r.vo = sub3(c, P.origin);
  return r;
}

// computeDistance (cc:216-228) with both sides hoisted: vo = voxel centre - origin (per voxel),
// ra = (point_G - origin, |point_G - origin|) (per ray):  sdf = |po| - (vo . po) / |po|
__device__ __forceinline__ float sdf_from(F3 vo, float4 ra) {
  return fsub(ra.w, fdiv(dot3(vo, f3(ra.x, ra.y, ra.z)), ra.w));
}

// The sorted update records as the apply kernels see them: with the library sort the host knows
// which buffer holds the result and how many records there are; with the engine's own sort both
// live in device memory (SortPlan::final_buf, ScanState::total_updates).
struct RecordView {
  uint32_t* keys[2];
  uint32_t* vals[2];
  const SortPlan* plan;                 // nullptr: buffer 0 holds the sorted records
  const unsigned long long* d_total;    // nullptr: total_fixed
  unsigned long long total_fixed;
};

// What k_apply_prep hands to k_apply besides the records themselves: the voxel runs longer than
// kShortRun updates and one keep bit per record.  Both are private to the scan's hand-off set.
constexpr int kApplyTile = 256;  // records per work item of k_apply's short-run phase
constexpr int kApplyWarps = 4;   // warps per thread block of k_apply
struct LongRuns {
  unsigned long long* start;   // [n_long] first record of the run
  unsigned long long* end;     // [n_long] one past its last record
  uint32_t* keep;              // bit j of word j / 32: record j's update maps (+T, max_weight) onto itself
  unsigned long long cap;      // entries of start / end and words of keep: max_updates / 32 + 1
};

// The prepared form of the sorted records.  After the sort only one of the two buffer pairs holds
// records; k_apply_prep writes each record's sdf and weight into the other pair and its colour over
// its ray id, so no buffer is added and everything stays private to the scan.
struct Prepared {
  const uint32_t* key;
  const float* sdf;
  const float* w;
  const uint32_t* col;
  unsigned long long total;
};
__device__ __forceinline__ Prepared open_prepared(const RecordView& rv) {
  const uint32_t sel = rv.plan ? rv.plan->final_buf : 0u;
  Prepared r;
  r.key = rv.keys[sel];
  r.sdf = reinterpret_cast<const float*>(rv.keys[sel ^ 1u]);
  r.w = reinterpret_cast<const float*>(rv.vals[sel ^ 1u]);
  r.col = rv.vals[sel];
  r.total = rv.d_total ? *rv.d_total : rv.total_fixed;
  return r;
}

// The per-record half of the apply; it reads no voxel, so it runs on the sort stream, beside the
// previous scan's apply.  One thread per sorted record: gather its ray, form sdf, weight and colour
// exactly as updateTsdfVoxel will use them (cc:150-209), and set its keep bit.  The bit is set when
// the update maps a voxel at (+T, max_weight) onto itself: sdf >= T (no colour blend), the new
// distance clamps back to +T and the weight back to max_weight -- the reference's own arithmetic,
// so "unchanged" is exact, not approximate.  Run heads count the distinct voxels (U) and list the
// runs longer than kShortRun updates with their [start, end).  Records of blocks this rank does not
// own (kSkipRecord) sort to the end and are skipped.
//
// kGiven (vbx_debug_apply only): a record's value is its ordinal into caller-given sdf / weight / colour
// arrays instead of a ray id, so that a test can drive the production apply with any update sequence.
struct GivenRecords {
  const float* sdf;
  const float* w;
  const uint32_t* col;
};
template <bool kGiven>
__global__ void __launch_bounds__(256, 6)
k_apply_prep(const ScanArgs* __restrict__ A, Tables tab, RecordView rv, const float4* __restrict__ ray_a,
             const uint2* __restrict__ ray_c, LongRuns lr, ScanState* st, GivenRecords given) {
  const ScanParams P = A->P;
  const uint32_t sel = rv.plan ? rv.plan->final_buf : 0u;
  const uint32_t* __restrict__ keys = rv.keys[sel];
  uint32_t* __restrict__ vals = rv.vals[sel];
  float* __restrict__ rec_sdf = reinterpret_cast<float*>(rv.keys[sel ^ 1u]);
  float* __restrict__ rec_w = reinterpret_cast<float*>(rv.vals[sel ^ 1u]);
  const unsigned long long total = rv.d_total ? *rv.d_total : rv.total_fixed;
  if (st->error & kFatalErrors) return;
  const float T = P.up.trunc, W = P.up.max_weight;
  const unsigned long long n_tiles = (total + 255ull) / 256ull;
  for (unsigned long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const unsigned long long e = tile * 256ull + threadIdx.x;
    const uint32_t key = e < total ? keys[e] : kSkipRecord;
    bool keep = false, head = false;
    if (key != kSkipRecord) {
      const uint32_t r = vals[e];
      const VoxelRef vr = locate_voxel(P, tab, key);
      float sdf, w;
      if (kGiven) {
        sdf = given.sdf[r];
        w = given.w[r];
        vals[e] = given.col[r];
      } else {
        const float4 ra = ray_a[r];
        const uint2 rc = ray_c[r];
        sdf = sdf_from(vr.vo, ra);
        w = update_weight(sdf, __uint_as_float(rc.y), P.up);
        vals[e] = rc.x;
      }
      rec_sdf[e] = sdf;
      rec_w[e] = w;
      const float nw = fadd(W, w);
      keep = sdf >= T && !(nw < VBX_EPS) && !(nw < W);
      if (keep) {
        const float ns = fdiv(fadd(fmul(sdf, w), fmul(T, W)), nw);
        keep = (ns > 0.0f) && !(ns < T);
      }
      // (a block that found no pool slot has no voxel to update: kErrPoolFull stops the next scan's apply)
      head = (e == 0 || keys[e - 1] != key) && vr.ptr != nullptr;
      if (head && e + kShortRun < total && keys[e + kShortRun] == key) {
        // the first record past the run: galloping from the record known to be in it, then bisection
        unsigned long long lo = e + kShortRun + 1, step = 2 * kShortRun;
        while (e + step < total && keys[e + step] == key) {
          lo = e + step + 1;
          step *= 2;
        }
        unsigned long long hi = min(e + step, total);
        while (lo < hi) {
          const unsigned long long mid = (lo + hi) >> 1;
          if (keys[mid] <= key) {
            lo = mid + 1;
          } else {
            hi = mid;
          }
        }
        const uint32_t q = atomicAdd(&st->n_long, 1u);
        assert(q < lr.cap);
        lr.start[q] = e;
        lr.end[q] = lo;
      }
    }
    const unsigned kb = __ballot_sync(0xffffffffu, keep);
    const unsigned hb = __ballot_sync(0xffffffffu, head);
    if ((threadIdx.x & 31) == 0) {
      if (e < total) {
        assert((e >> 5) < lr.cap);
        lr.keep[e >> 5] = kb;
      }
      if (hb) atomicAdd(&st->n_voxels, (uint32_t)__popc(hb));
    }
  }
}

// The first record p of [start, end) such that every record of [p, end) keeps (+T, max_weight):
// one warp reads the keep bits from the end of the run backwards, 32 words per step.
__device__ __forceinline__ unsigned long long keep_suffix(const uint32_t* __restrict__ keep, unsigned long long start,
                                                          unsigned long long end, int lane) {
  const long long w0 = (long long)(start >> 5), w1 = (long long)((end - 1) >> 5);
  for (long long top = w1; top >= w0; top -= 32) {
    const long long wi = top - lane;
    uint32_t bad = 0u;
    if (wi >= w0) {
      uint32_t m = 0xffffffffu;
      if (wi == w0) m &= 0xffffffffu << (start & 31u);
      if (wi == w1) m &= 0xffffffffu >> (31u - ((end - 1) & 31u));
      bad = ~keep[wi] & m;
    }
    const unsigned b = __ballot_sync(0xffffffffu, bad != 0u);
    if (b) {
      const int src = __ffs(b) - 1;  // the lowest lane holds the highest word with a record that does not keep
      const uint32_t bw = __shfl_sync(0xffffffffu, bad, src);
      return (unsigned long long)(top - src) * 32ull + (unsigned long long)(31 - __clz(bw)) + 1ull;
    }
  }
  return start;
}

// The read-modify-write chains of updateTsdfVoxel (cc:150-209), applied sequentially per voxel --
// clamp-after-every-update semantics preserved exactly, with no locks and no atomics on voxels --
// over the records k_apply_prep prepared.  Warps first take the long runs by ticket, so the longest
// chains start at once; then they take kApplyTile-record tiles of the short runs, one thread per
// run.  Every voxel has exactly one owner and no warp waits on another.
//
// A long run is one warp's from its first record.  kG x 32 records are loaded per step (and the next
// step's are prefetched) so that the loads of a step are all in flight together.  Free space far in
// front of any surface is the common long run: there every update has sdf >= T and the voxel already
// sits at +T, so after computing the exact sequential weight chain each lane checks that ITS update
// maps +T to +T; if all do, the sequential result is (+T, chained weight) without walking the
// distance chain.  Once the voxel rests at (+T, max_weight) and every remaining record's keep bit is
// set, the rest of the run leaves it unchanged and is skipped.
__global__ void __launch_bounds__(32 * kApplyWarps, 8)
k_apply(const ScanArgs* __restrict__ A, Tables tab, RecordView rv, LongRuns lr, ScanState* st) {
  const ScanParams P = A->P;
  const Prepared pr = open_prepared(rv);
  if (st->error & kFatalErrors) return;
  const uint32_t* __restrict__ keys = pr.key;
  const float* __restrict__ rec_sdf = pr.sdf;
  const float* __restrict__ rec_w = pr.w;
  const uint32_t* __restrict__ rec_col = pr.col;
  const unsigned long long total = pr.total;
  const int lane = threadIdx.x & 31;
  const uint32_t n_long = st->n_long;
  const float T = P.up.trunc;
  const bool can_rest = P.up.max_weight >= VBX_EPS;
  const int wb = threadIdx.x >> 5;
  // How often each path ran (ApplyPath), only when asked for (ScanArgs::count_paths: tests and diagnostics),
  // added to the status block once per warp when it leaves.  The long-run paths are decided per warp: lane 0
  // counts them in the warp's row of s_paths (in shared memory, so that they take no registers from the
  // chains).  Short runs are counted per lane in two registers.
  const bool counting = A->count_paths != 0u;
  __shared__ uint32_t s_paths[kApplyWarps][kApplyPaths];
  if (counting && lane < kApplyPaths) s_paths[wb][lane] = 0u;
  __syncwarp();
  auto count = [&](int path) {
    if (counting && lane == 0) ++s_paths[wb][path];
  };
  uint32_t n_short = 0, n_crossed = 0;
  for (;;) {
    uint32_t q = 0;
    if (lane == 0) q = atomicAdd(&st->long_ticket, 1u);
    q = __shfl_sync(0xffffffffu, q, 0);
    if (q >= n_long) break;
    const unsigned long long start = lr.start[q], end = lr.end[q];
    count(kPathLongRun);
    const VoxelRef vr = locate_voxel(P, tab, keys[start]);
    TsdfVoxel v = *vr.ptr;
    unsigned long long keep_from = ~0ull;  // found on first need
    unsigned long long j0 = start;
    constexpr int kG = 4;
    bool in_n[kG];
    float sdf_n[kG], w_n[kG];
#pragma unroll
    for (int g = 0; g < kG; ++g) {
      const unsigned long long j = j0 + 32ull * g + lane;
      in_n[g] = j < end;
      sdf_n[g] = in_n[g] ? rec_sdf[j] : 0.f;
      w_n[g] = in_n[g] ? rec_w[j] : 0.f;
    }
    for (;;) {
      if (can_rest && v.distance == T && v.weight == P.up.max_weight) {
        if (keep_from == ~0ull) keep_from = keep_suffix(lr.keep, start, end, lane);
        if (j0 >= keep_from) {
          count(kPathLongRested);
          break;
        }
      }
      bool in_c[kG];
      float sdf_c[kG], w_c[kG];
#pragma unroll
      for (int g = 0; g < kG; ++g) {
        in_c[g] = in_n[g];
        sdf_c[g] = sdf_n[g];
        w_c[g] = w_n[g];
      }
      const bool more = j0 + 32ull * kG < end;
      if (more) {
#pragma unroll
        for (int g = 0; g < kG; ++g) {
          const unsigned long long j = j0 + 32ull * (kG + g) + lane;
          in_n[g] = j < end;
          sdf_n[g] = in_n[g] ? rec_sdf[j] : 0.f;
          w_n[g] = in_n[g] ? rec_w[j] : 0.f;
        }
      }
      // The common long run -- free space far in front of any surface, the voxel already at +T -- is decided
      // for all kG chunks at once: ONE exact in-order weight chain over the step's records, then every
      // lane checks that its updates map +T onto +T, one vote.  (Same arithmetic as the per-chunk path
      // below, which remains for everything else and redoes the step from the unchanged voxel if a
      // check fails.)
      bool step_done = false;
      {
        bool ff = true;
        float wl[kG];
#pragma unroll
        for (int g = 0; g < kG; ++g) {
          ff = ff && (!in_c[g] || sdf_c[g] >= T);
          wl[g] = in_c[g] ? w_c[g] : 0.f;
        }
        if (__all_sync(0xffffffffu, ff) && v.distance == T) {
          float ws = (wl[0] + wl[1]) + (wl[2] + wl[3]);  // any-order sum, used only as a bound
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) ws += __shfl_xor_sync(0xffffffffu, ws, o);
          const bool saturated = v.weight == P.up.max_weight && P.up.max_weight >= VBX_EPS;
          const bool no_clamp = v.weight >= VBX_EPS && (v.weight + ws) * 1.0001f < P.up.max_weight;
          float mb[kG];
          float w_end = v.weight;
          bool have = true;
          int path = kPathStepSaturated;
          if (saturated) {
            // W + w >= max_weight for every w >= 0: the clamp returns max_weight at every step
#pragma unroll
            for (int g = 0; g < kG; ++g) mb[g] = v.weight;
          } else if (no_clamp) {
            // neither the 1e-6 guard nor the max_weight clamp can fire: the chain is plain in-order addition
            bool ints = v.weight == truncf(v.weight) && (v.weight + ws) < 16777216.0f;
#pragma unroll
            for (int g = 0; g < kG; ++g) ints = ints && wl[g] == truncf(wl[g]);
            if (__all_sync(0xffffffffu, ints)) {
              path = kPathStepIntScan;
              // integer-valued weights (use_const_weight: a bundle's weight is its point count) on an
              // integer-valued W, everything below 2^24: every partial sum is exact, so any order gives
              // the in-order chain -- a warp scan per chunk
              float base = v.weight;
#pragma unroll
              for (int g = 0; g < kG; ++g) {
                float inc = wl[g];
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                  const float t = __shfl_up_sync(0xffffffffu, inc, o);
                  if (lane >= o) inc += t;
                }
                mb[g] = base + (inc - wl[g]);
                base = base + __shfl_sync(0xffffffffu, inc, 31);
              }
              w_end = base;
            } else {
              path = kPathStepPrefix;
              float base = v.weight;
#pragma unroll
              for (int g = 0; g < kG; ++g) {
                float before = base;
#pragma unroll
                for (int k = 0; k < 31; ++k) {
                  const float wk = __shfl_sync(0xffffffffu, wl[g], k);
                  if (k < lane) before = fadd(before, wk);
                }
                mb[g] = before;
                base = __shfl_sync(0xffffffffu, fadd(before, wl[g]), 31);
              }
              w_end = base;
            }
          } else {
            have = false;
          }
          if (have) {
            bool keeps_T = true;
#pragma unroll
            for (int g = 0; g < kG; ++g) {
              if (in_c[g]) {
                const float nw = fadd(mb[g], w_c[g]);
                if (!(nw < VBX_EPS)) {
                  const float ns = fdiv(fadd(fmul(sdf_c[g], w_c[g]), fmul(T, mb[g])), nw);
                  const float clamped = (ns > 0.0f) ? ((ns < T) ? ns : T) : ((-T < ns) ? ns : -T);
                  keeps_T = keeps_T && (clamped == T);
                }
              }
            }
            if (__all_sync(0xffffffffu, keeps_T)) {
              v.weight = w_end;
              step_done = true;
              count(path);
            }
          }
        }
      }
#pragma unroll
      for (int g = 0; g < kG; ++g) {
        if (step_done) break;
        const bool in = in_c[g];
        const float sdf = sdf_c[g], w = w_c[g];
        const int cnt = __popc(__ballot_sync(0xffffffffu, in));
        if (cnt == 0) break;
        const bool far_free = !in || sdf >= T;
        bool fast = __all_sync(0xffffffffu, far_free) && v.distance == T;
        float w_end = v.weight;
        int path = kPathChunkSaturated;
        if (fast) {
          // exact sequential weight chain: W <- min(W + w, max_weight) unless W + w < 1e-6
          float my_before = 0.f;
          float wsum = in ? w : 0.f;  // any-order sum, used only as a bound
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) wsum += __shfl_xor_sync(0xffffffffu, wsum, o);
          const bool no_clamp = v.weight >= VBX_EPS && (v.weight + wsum) * 1.0001f < P.up.max_weight;
          if (v.weight == P.up.max_weight && P.up.max_weight >= VBX_EPS) {
            // the weight already sits at max_weight: W + w >= max_weight for every w >= 0, so the
            // clamp returns max_weight at every step
            my_before = v.weight;
          } else if (no_clamp && v.weight < 4194304.0f && v.weight == truncf(v.weight) &&
                     __all_sync(0xffffffffu, !in || w == 1.0f)) {
            // constant weights (use_const_weight) on an integer-valued W below 2^22: every partial
            // sum is an integer that float represents exactly, so the in-order chain is W + k
            path = kPathChunkConst;
            my_before = v.weight + (float)lane;
            w_end = v.weight + (float)cnt;
          } else if (no_clamp) {
            // neither the 1e-6 guard nor the max_weight clamp can fire in this chunk: the
            // chain is plain in-order addition; lane L forms its own prefix
            path = kPathChunkPrefix;
            const float wl = in ? w : 0.f;
            my_before = v.weight;
#pragma unroll
            for (int k = 0; k < 31; ++k) {
              const float wk = __shfl_sync(0xffffffffu, wl, k);
              if (k < lane) my_before = fadd(my_before, wk);
            }
            w_end = __shfl_sync(0xffffffffu, fadd(my_before, wl), 31);
          } else {
            path = kPathChunkSequential;
            for (int k = 0; k < cnt; ++k) {
              const float wk = __shfl_sync(0xffffffffu, w, k);
              if (lane == k) my_before = w_end;
              const float nw = fadd(w_end, wk);
              w_end = (nw < VBX_EPS) ? w_end : ((nw < P.up.max_weight) ? nw : P.up.max_weight);
            }
          }
          bool keeps_T = true;
          if (in) {
            const float nw = fadd(my_before, w);
            if (!(nw < VBX_EPS)) {
              const float ns = fdiv(fadd(fmul(sdf, w), fmul(T, my_before)), nw);
              const float clamped = (ns > 0.0f) ? ((ns < T) ? ns : T) : ((-T < ns) ? ns : -T);
              keeps_T = (clamped == T);
            }
          }
          fast = __all_sync(0xffffffffu, keeps_T);
        }
        if (fast) {
          v.weight = w_end;
          count(path);
        } else {
          count(kPathChunkExact);
          const uint32_t col = in ? rec_col[j0 + 32ull * g + lane] : 0u;
          for (int k = 0; k < cnt; ++k) {
            apply_update(v, __shfl_sync(0xffffffffu, sdf, k), __shfl_sync(0xffffffffu, w, k),
                         __shfl_sync(0xffffffffu, col, k), P.up);
          }
        }
      }
      j0 += 32ull * kG;
      if (!more) break;
    }
    if (lane == 0) *vr.ptr = v;
  }
  // The short runs.  A warp stages its tile's records in shared memory (all loads in flight together),
  // lists the tile's run heads, and gives each lane a head: the tile's chains run side by side.
  __shared__ uint32_t s_key[kApplyWarps][kApplyTile];
  __shared__ float s_sdf[kApplyWarps][kApplyTile];
  __shared__ float s_w[kApplyWarps][kApplyTile];
  __shared__ uint32_t s_col[kApplyWarps][kApplyTile];
  __shared__ uint8_t s_head[kApplyWarps][kApplyTile];
  const uint32_t n_tiles = (uint32_t)((total + kApplyTile - 1) / kApplyTile);
  for (;;) {
    uint32_t t = 0;
    if (lane == 0) t = atomicAdd(&st->tile_ticket, 1u);
    t = __shfl_sync(0xffffffffu, t, 0);
    if (t >= n_tiles) break;
    const unsigned long long base = (unsigned long long)t * kApplyTile;
#pragma unroll
    for (int s = 0; s < kApplyTile / 32; ++s) {
      const int o = 32 * s + lane;
      const bool in = base + o < total;
      s_key[wb][o] = in ? keys[base + o] : kSkipRecord;
      s_sdf[wb][o] = in ? rec_sdf[base + o] : 0.f;
      s_w[wb][o] = in ? rec_w[base + o] : 0.f;
      s_col[wb][o] = in ? rec_col[base + o] : 0u;
    }
    __syncwarp();
    uint32_t n_heads = 0;
    for (int s = 0; s < kApplyTile / 32; ++s) {
      const int o = 32 * s + lane;
      const unsigned long long e = base + o;
      const uint32_t key = s_key[wb][o];
      bool head = key != kSkipRecord && (o > 0 ? s_key[wb][o - 1] != key : (e == 0 || keys[e - 1] != key));
      if (head && e + kShortRun < total) {
        // a run longer than kShortRun belongs to a warp of the first phase
        head = (o + kShortRun < kApplyTile ? s_key[wb][o + kShortRun] : keys[e + kShortRun]) != key;
      }
      const unsigned m = __ballot_sync(0xffffffffu, head);
      if (head) s_head[wb][n_heads + __popc(m & ((1u << lane) - 1u))] = (uint8_t)o;
      n_heads += __popc(m);
    }
    __syncwarp();
    for (uint32_t h = lane; h < n_heads; h += 32) {
      const int o = s_head[wb][h];
      const uint32_t key = s_key[wb][o];
      const VoxelRef vr = locate_voxel(P, tab, key);
      if (vr.ptr == nullptr) continue;
      ++n_short;
      TsdfVoxel v = *vr.ptr;
      int k = o;
      for (; k < kApplyTile && s_key[wb][k] == key; ++k) apply_update(v, s_sdf[wb][k], s_w[wb][k], s_col[wb][k], P.up);
      if (k == kApplyTile) {
        // a run that crosses the tile's end continues from global memory
        ++n_crossed;
        for (unsigned long long j = base + kApplyTile; j < total && keys[j] == key; ++j) {
          apply_update(v, rec_sdf[j], rec_w[j], rec_col[j], P.up);
        }
      }
      *vr.ptr = v;
    }
    __syncwarp();  // the staging arrays are reused by the warp's next tile
  }
  if (counting) {
    n_short = __reduce_add_sync(0xffffffffu, n_short);
    n_crossed = __reduce_add_sync(0xffffffffu, n_crossed);
    if (lane == 0) {
      s_paths[wb][kPathShortRun] = n_short;
      s_paths[wb][kPathShortCrossed] = n_crossed;
    }
    __syncwarp();
    if (lane < kApplyPaths && s_paths[wb][lane]) atomicAdd(&st->apply_paths[lane], s_paths[wb][lane]);
  }
}

// --------------------------------------------------------------------- host side
// The growth schedule of a default-constructed std::unordered_map (max_load_factor 1) under
// one-by-one insertion, taken from the C++ library's own policy object: operator[] asks
// _M_need_rehash(bucket_count, element_count, 1) before every insertion of a new key
// (bits/hashtable.h _M_insert_unique_node).
int init_bundle_order(vbx_ctx* c) {
  RehashSchedule& rs = c->rehash;
  std::memset(&rs, 0, sizeof(rs));
  std::__detail::_Prime_rehash_policy pol;
  size_t buckets = 1;
  size_t e = 0;
  const size_t limit = (size_t)c->max_points + 1;
  while (e < limit && rs.count < 30) {
    const auto r = pol._M_need_rehash(buckets, e, 1);
    if (r.first) {
      buckets = r.second;
      rs.m[rs.count] = (uint32_t)e;
      rs.n[rs.count] = (uint32_t)buckets;
      ++rs.count;
    }
    // no rehash can happen before the element count exceeds the policy's next threshold
    const size_t next = (size_t)pol._M_next_resize;
    e = std::max(e + 1, next);
  }
  if (e < limit) return fail(c, VBX_E_INVALID, "unordered_map growth schedule longer than expected");
  int dev = 0, max_optin = 0;
  VBX_CUDA(c, cudaGetDevice(&dev));
  VBX_CUDA(c, cudaDeviceGetAttribute(&max_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  c->order_smem_bytes = (size_t)std::max(0, max_optin - 2048) & ~(size_t)15;
  VBX_CUDA(c, cudaFuncSetAttribute(k_bundle_order, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)c->order_smem_bytes));
  return VBX_OK;
}

int check_state_errors(vbx_ctx* c, const ScanState& h) {
  const uint32_t err = h.error & kFatalErrors;
  if (!err) return VBX_OK;
  if (err & kErrPoolFull) {
    // the surplus hash entries of this call have no pool slot: drop them, or later calls would find them
    if (h.n_blocks) c->n_blocks = h.n_blocks;
    rebuild_hash(c);
  }
  std::string m = "device reported:";
  if (err & kErrPoolFull) m += " block pool full (raise vbx_engine_options.max_blocks);";
  if (err & kErrHashFull) m += " block hash full;";
  if (err & kErrCoordRange) m += " voxel coordinate outside +-2^20 blocks;";
  if (err & kErrUpdatesFull) m += " ray-voxel updates exceed max_updates_per_pass;";
  return fail(c, VBX_E_CAPACITY, m);
}

namespace {
// The back half's streams and hand-off events while a pipelined scan's graph is captured (capture_scan)
struct Capture {
  cudaStream_t sort, apply;
  cudaEvent_t walked, sorted, applied;   // this scan's stage ends: later scans' graphs wait for them
  cudaEvent_t prev_sorted, prev_applied; // the record sort two scans back, the previous scan's apply
  cudaEvent_t edge[2];                   // capture-internal: walk -> sort, sort -> apply
};
}  // namespace

// The map's tables as a scan's kernels see them: with the hand-off set's touched-id list
static Tables scan_tables(const vbx_ctx* c, const vbx_ctx::ScratchSet& S) {
  Tables t = c->tab;
  t.touched_list = S.touched_list;
  return t;
}

static unsigned int sort_grid(const vbx_ctx* c, int which, uint64_t n_hint, unsigned int sms) {
  const uint64_t tiles_hint = std::max<uint64_t>(1, (n_hint + kSortTile - 1) / kSortTile);
  return (unsigned int)std::min<uint64_t>(std::min<uint64_t>(c->sort_tiles_cap[which], tiles_hint), (uint64_t)sms * 2);
}

// The engine's own stable radix sort (vbx_sort.cuh): one launch.  n lives on the device (d_n) or is n_fixed;
// n_hint sizes the grid (tiles are handed out by ticket, so any grid sorts any n).  result_in_a: the sorted
// pairs end in buffer A whatever the number of passes (otherwise SortPlan::final_buf says where they are).
// which: 0 the point sort (the front lane's plan), 1 the record sort (the hand-off set's).
template <typename KeyT>
static int own_sort(vbx_ctx* c, const ScanRoute& x, int which, KeyT* keys_a, uint32_t* vals_a, KeyT* keys_b,
                    uint32_t* vals_b, const unsigned long long* d_n, uint32_t n_fixed, uint64_t n_hint, int key_bits,
                    bool result_in_a, Tally& tally, const uint32_t* d_key_bits = nullptr, bool plan_cleared = false) {
  cudaStream_t s = x.s;
  const int passes = std::min(kMaxPasses, (key_bits + 7) / 8);
  SortPlan* plan = which ? x.S.sort_plan1 : x.F.sort_plan0;
  uint32_t* status = which ? x.S.sort_status1 : x.F.sort_status0;
  const uint32_t tiles_cap = c->sort_tiles_cap[which];
  if (!plan_cleared) VBX_CUDA(c, cudaMemsetAsync(plan, 0, sizeof(SortPlan), s));  // (else: an earlier kernel of the stream did)
  const unsigned int grid = sort_grid(c, which, n_hint, x.sms);
  k_sort<KeyT><<<grid, kSortThreads, 0, s>>>(keys_a, vals_a, keys_b, vals_b, d_n, n_fixed, passes, d_key_bits, plan, status,
                                              tiles_cap, result_in_a ? 1 : 0);
  ++tally.launches;
  return VBX_OK;
}

// k_order_prefix, k_order_heads, k_bundle_order on stream `so` (see the kernels).
constexpr int kOrderGrid = 32;  // blocks of the cooperative k_bundle_order launch (only large maps use more than one)
// The shared memory asked for is what the bundle count of recent scans needs (plus a margin), not the whole
// SM: a block that wants 200 KB can only start on an SM that holds nothing else, and in the pipelined path
// -- every SM busy with other scans' kernels -- it waits for one to drain.  A scan with more bundles than the
// request covers is still ordered correctly: the kernel falls back to its global-memory stages.
struct OrderLaunch {
  unsigned int grid;  // 1: the one-block form, else the cooperative one
  size_t smem_bytes;
};
static OrderLaunch order_launch(const vbx_ctx* c, uint32_t n) {
  OrderLaunch o{(unsigned int)kOrderGrid, c->order_smem_bytes};
  if (c->bundle_hint) {
    const RehashSchedule& rs = c->rehash;
    const uint32_t B = (uint32_t)std::min<uint64_t>(c->bundle_hint + c->bundle_hint / 4 + 512, n);
    uint32_t nf = 1;
    for (int k = 0; k < rs.count && rs.m[k] < B; ++k) nf = rs.n[k];
    const uint32_t words = order_smem_words_needed(B, nf);
    const size_t need = ((size_t)words * 4 + 1023) & ~(size_t)1023;
    if (words != 0xffffffffu && need <= c->order_smem_bytes) {
      o.smem_bytes = need;
      o.grid = 1;  // the single-block form; block 0 is the only one that would work
    }
  }
  return o;
}

static int launch_bundle_order(vbx_ctx* c, const ScanRoute& x, cudaStream_t so, uint32_t n, Tally& tally) {
  const vbx_ctx::ScratchSet& S = x.S;
  const vbx_ctx::FrontLane& F = x.F;
  k_order_prefix<<<1, kOrderThreads, 0, so>>>(S.d_args, F.first_bits, F.order_scratch, S.d_state);
  ++tally.launches;
  k_order_heads<<<std::min<unsigned int>(grid_for(c->max_points, 256), x.sms * 2), 256, 0, so>>>(
      S.d_args, S.pkeys0, F.pvals[0], c->order_inv, S.head_list, F.first_bits, F.order_scratch, S.d_state);
  ++tally.launches;
  // Always a cooperative launch (the one-block form is a cooperative grid of one block), so that a scan
  // graph's node switches between the two forms by its grid and shared memory alone (update_scan_graph).
  const OrderLaunch o = order_launch(c, n);
  const uint32_t smem_words = (uint32_t)(o.smem_bytes / 4);
  cudaLaunchConfig_t lc = {};
  lc.gridDim = dim3(o.grid);
  lc.blockDim = dim3(kOrderThreads);
  lc.dynamicSmemBytes = o.smem_bytes;
  lc.stream = so;
  cudaLaunchAttribute coop;
  coop.id = cudaLaunchAttributeCooperative;
  coop.val.cooperative = 1;
  lc.attrs = &coop;
  lc.numAttrs = 1;
  VBX_CUDA(c, cudaLaunchKernelEx(&lc, k_bundle_order, c->rehash, F.order_scratch, smem_words, S.ray_list,
                                 F.order_scratch.cta_tot, S.d_state));
  ++tally.launches;
  return VBX_OK;
}

// The ray walk that writes the update records (of the pass in P.emit_lo .. P.emit_hi) against the scan's
// private block table: it needs nothing of the map.
static void launch_emit(const vbx_ctx* c, const ScanRoute& x, const ScanParams& P, Tally& tally) {
  const vbx_ctx::ScratchSet& S = x.S;
  if (P.kind == VBX_MERGED && P.single_walk) {
    // a few thousand bundles of 100-300 steps: one warp per ray
    k_rays_emit_warp<<<x.sms * 8, 128, 0, x.s>>>(S.d_args, S.blocks, S.pkeys0, S.ray_list, S.head_list, S.ray_p, S.cnt,
                                                 S.off, S.ckeys[0], S.cvals[0], S.d_state);
  } else {
    k_rays_emit<<<grid_for(c->max_points, 128), 128, 0, x.s>>>(S.d_args, S.blocks, S.pkeys0, S.ray_list, S.head_list,
                                                               S.ray_p, S.cnt, S.off, S.ckeys[0], S.cvals[0], S.d_state);
  }
  ++tally.launches;
  tally.mark(kStageRayEmit);
}

// Stages up to the record offsets and the ray walk that writes the update records: everything that decides
// WHICH voxels are updated, without touching the map.  The per-scan values
// come from the set's argument block (S.d_args), and the grids are sized for max_points_per_scan -- surplus threads
// exit at once -- so that one captured graph serves scans of any size (the point sort's grid, whose surplus
// blocks would wait between passes, is set per scan instead: update_scan_graph).
static int front_half(vbx_ctx* c, const ScanRoute& x, const ScanParams& P, const uint32_t* order, Tally& tally) {
  cudaStream_t s = x.s;
  const vbx_ctx::ScratchSet& S = x.S;
  const vbx_ctx::FrontLane& F = x.F;
  const ScanArgs* A = S.d_args;
  const uint32_t n = P.n;
  const uint32_t gn = c->max_points;
  const int TB = 256;
  const uint32_t* scan_perm = nullptr;
  const uint32_t* scan_limit = nullptr;
  const uint32_t scan_tiles = (gn + 1 + kScanTile - 1) / kScanTile;
  if (P.kind == VBX_MERGED) {
    k_point_bounds<<<std::min<unsigned int>(grid_for(gn, TB), x.sms * 4), TB, 0, s>>>(
        A, F.first_bits, F.sort_plan0, F.scan_status, scan_tiles + 1, S.d_state);
    ++tally.launches;
    k_point_keys<<<grid_for(gn, TB), TB, 0, s>>>(A, order, S.pkeys0, F.pvals[0], S.d_state);
    ++tally.launches;
    tally.mark(kStagePointKeys);
    // the bits in use are known on the device only (ScanState::key_bits): passes beyond them exit at once
    if (int rc = own_sort(c, x, 0, S.pkeys0, F.pvals[0], F.pkeys1, F.pvals[1], &A->n, 0, n, 64, true, tally,
                          &S.d_state->key_bits, /*plan_cleared=*/true)) {
      return rc;
    }
    tally.mark(kStagePointSort);
    k_heads<<<grid_for((uint64_t)gn + 1, TB), TB, 0, s>>>(A, S.pkeys0, F.pvals[0], c->order_inv, S.head_list, F.big_list,
                                                          F.first_bits, S.cnt, S.d_state);
    ++tally.launches;
    // The reference's bundle order (ray_list[rank] = bundle id, vbx_order.cuh) is one thread block's work
    // and the fold (k_merge) does not need it: the two run side by side.  (With stage profiling on they
    // run one after the other so that each gets its own time.)
    cudaStream_t so = tally.on ? s : F.side;
    if (so != s) {
      VBX_CUDA(c, cudaEventRecord(F.ev_fork, s));
      VBX_CUDA(c, cudaStreamWaitEvent(so, F.ev_fork, 0));
    }
    if (int rc = launch_bundle_order(c, x, so, P.n, tally)) return rc;
    if (so != s) VBX_CUDA(c, cudaEventRecord(F.ev_join, so));
    tally.mark(kStageBundleOrder);
    k_merge<<<x.sms * 4, 192, 0, s>>>(A, S.pkeys0, F.pvals[0], S.head_list, F.big_list, S.ray_p, S.ray_a, S.ray_c, S.cnt,
                                      S.d_state);
    ++tally.launches;
    tally.mark(kStageBundleMerge);
    if (!P.single_walk) {
      // the bundle count is only known on the device: launch for the worst case (every
      // point its own bundle); surplus threads exit on the first load
      k_rays_count<<<grid_for(gn, 128), 128, 0, s>>>(A, order, S.pkeys0, S.head_list, S.ray_p, S.ray_a, S.ray_c,
                                                     S.cnt, c->set_start, c->set_observed, S.d_state);
      ++tally.launches;
    }
    if (so != s) VBX_CUDA(c, cudaStreamWaitEvent(s, F.ev_join, 0));
    // record offsets in RANK order: off[rank] = sum of cnt[ray_list[r]] over r < rank
    scan_perm = S.ray_list;
    scan_limit = &S.d_state->n_ray_list;
  } else if (P.kind == VBX_FAST && c->serial_fast) {
    k_rays_count_serial<<<1, 1, 0, s>>>(A, order, S.ray_p, S.ray_a, S.ray_c, S.cnt, c->set_start, c->set_observed,
                                        S.d_state);
    ++tally.launches;
  } else {
    k_rays_count<<<grid_for((uint64_t)gn + 1, 128), 128, 0, s>>>(A, order, S.pkeys0, S.head_list, S.ray_p, S.ray_a,
                                                                 S.ray_c, S.cnt, c->set_start, c->set_observed,
                                                                 S.d_state);
    ++tally.launches;
  }
  tally.mark(kStageRayCount);
  {
    // record offsets; the scan's last position also settles the call's update count (total_found, total_updates,
    // kErrUpdatesFull: too many for one pass; nothing downstream runs on a call that failed)
    if (P.kind != VBX_MERGED) VBX_CUDA(c, cudaMemsetAsync(F.scan_status, 0, (size_t)(scan_tiles + 1) * sizeof(uint32_t), s));  // (Merged: k_point_bounds did)
    k_exclusive_scan<<<std::min<uint32_t>(scan_tiles, x.sms * 4), kSortThreads, 0, s>>>(
        S.cnt, scan_perm, scan_limit, S.off, &A->n_scan, 0u, F.scan_status + 1, F.scan_status, &S.d_state->total_found,
        &S.d_state->total_updates, &S.d_state->error, (unsigned long long)c->max_updates, kErrUpdatesFull);
    ++tally.launches;
  }
  tally.mark(kStageScan);
  // (a call whose records do not fit one pass emits nothing here: apply_in_passes emits each pass)
  launch_emit(c, x, P, tally);
  return VBX_OK;
}

// update-record sort + the apply kernels.  cap: a pipelined scan's graph is being captured.  given: the records'
// values are ordinals into these arrays, not ray ids (debug_apply)
static int sort_and_apply(vbx_ctx* c, const ScanRoute& x, Tally& tally, const Capture* cap,
                          const GivenRecords* given = nullptr) {
  ScanRoute r = x;
  const vbx_ctx::ScratchSet& S = x.S;
  const Tables tab = scan_tables(c, S);
  RecordView rv;
  {
    // K and the number of touched blocks are only known on the device: sort on every bit a
    // record key can have; passes whose digit is uniform are skipped on the device
    const int key_bits = 32;
    if (cap) {
      // pipelined submission: the record sort works on buffers private to this scan, so it leaves
      // the walk stream (which the next scan's ray walk is waiting for)
      VBX_CUDA(c, cudaEventRecordWithFlags(cap->walked, r.s, cudaEventRecordExternal));
      VBX_CUDA(c, cudaEventRecord(cap->edge[0], r.s));
      VBX_CUDA(c, cudaStreamWaitEvent(cap->sort, cap->edge[0], 0));
      VBX_CUDA(c, cudaStreamWaitEvent(cap->sort, cap->prev_sorted, cudaEventWaitExternal));
      r.s = cap->sort;
    }
    if (int rc = own_sort(c, r, 1, S.ckeys[0], S.cvals[0], S.ckeys[1], S.cvals[1], &S.d_state->total_updates, 0,
                          c->record_hint, key_bits, false, tally, &S.d_state->rec_key_bits, /*plan_cleared=*/true)) {
      return rc;
    }
    rv.keys[0] = S.ckeys[0];
    rv.keys[1] = S.ckeys[1];
    rv.vals[0] = S.cvals[0];
    rv.vals[1] = S.cvals[1];
    rv.plan = S.sort_plan1;
    rv.d_total = &S.d_state->total_updates;
    rv.total_fixed = 0;
  }
  LongRuns lr;
  lr.start = S.long_list;
  lr.end = S.long_end;
  lr.keep = S.keep_bits;
  lr.cap = c->max_updates / 32 + 1;
  // everything of the apply that does not depend on the map, on the (pipelined: scan-private) sort stream
  cudaStream_t s = r.s;
  if (given) {
    k_apply_prep<true><<<x.sms * 8, 256, 0, s>>>(S.d_args, tab, rv, S.ray_a, S.ray_c, lr, S.d_state, *given);
  } else {
    k_apply_prep<false><<<x.sms * 8, 256, 0, s>>>(S.d_args, tab, rv, S.ray_a, S.ray_c, lr, S.d_state, GivenRecords{});
  }
  ++tally.launches;
  tally.mark(kStageUpdateSort);
  if (cap) {
    // pipelined submission: the apply kernel runs behind the previous scan's apply, so the next scan's
    // ray walk can start while this scan's voxels are still being written
    VBX_CUDA(c, cudaEventRecordWithFlags(cap->sorted, s, cudaEventRecordExternal));
    VBX_CUDA(c, cudaEventRecord(cap->edge[1], s));
    VBX_CUDA(c, cudaStreamWaitEvent(cap->apply, cap->edge[1], 0));
    VBX_CUDA(c, cudaStreamWaitEvent(cap->apply, cap->prev_applied, cudaEventWaitExternal));
    s = cap->apply;
  }
  k_apply<<<x.sms * 8, 32 * kApplyWarps, 0, s>>>(S.d_args, tab, rv, lr, S.d_state);
  ++tally.launches;
  if (cap) VBX_CUDA(c, cudaEventRecordWithFlags(cap->applied, s, cudaEventRecordExternal));
  tally.mark(kStageApply);
  return VBX_OK;
}

// k_assign on x.s for the blocks listed in the hand-off set's table; the block count moves to the other word
// of d_nblocks.
static void assign_blocks(vbx_ctx* c, const ScanRoute& x, uint8_t touch_bits, uint8_t new_bits) {
  const vbx_ctx::ScratchSet& S = x.S;
  k_assign<<<1, kAssignThreads, 0, x.s>>>(scan_tables(c, S), S.blocks, S.d_args, c->d_nblocks, S.sort_plan1,
                                          S.d_state, touch_bits, new_bits);
  c->nb_cur ^= 1;
}

// Block creation (k_assign, in submission order), then the record sort and the apply.
static int back_half(vbx_ctx* c, const ScanRoute& x, Tally& tally, const Capture* cap = nullptr) {
  assign_blocks(c, x, kTouchedBits, kTouchedBits);
  ++tally.launches;
  tally.mark(kStageAssign);
  return sort_and_apply(c, x, tally, cap);
}

static void fill_args(const vbx_ctx* c, const ScanParams& P, const float* xyz, const uint8_t* rgba, ScanArgs* a) {
  a->P = P;
  a->xyz = xyz;
  a->rgba = rgba;
  a->n = P.n;
  a->n_scan = P.n + 1;
  a->nb_cur = (uint32_t)c->nb_cur;
  a->count_paths = c->count_apply_paths ? 1u : 0u;
}

// The synchronous calls' argument block goes through the set's page-locked copy: the host writes it
// only when the stream has finished every earlier upload.
static int upload_args(vbx_ctx* c, const ScanRoute& x, const ScanArgs& a) {
  *x.S.h_args = a;
  VBX_CUDA(c, cudaMemcpyAsync(x.S.d_args, x.S.h_args, sizeof(ScanArgs), cudaMemcpyHostToDevice, x.s));
  return VBX_OK;
}

int create_listed_blocks(vbx_ctx* c, uint8_t new_bits) {
  const ScanRoute x = sync_route(c);
  ScanArgs a;
  std::memset(&a, 0, sizeof(a));
  a.P.emit_hi = 0xffffffffu;  // (>= P.n: k_assign clears the table, as a scan's last pass does)
  a.nb_cur = (uint32_t)c->nb_cur;
  if (int rc = upload_args(c, x, a)) return rc;
  assign_blocks(c, x, 0, new_bits);
  return VBX_OK;
}

int alloc_scan_args(vbx_ctx* c, Holdings& h, vbx_ctx::ScratchSet& S) {
  VBX_CUDA(c, h.dev(&S.d_args, 1));
  VBX_CUDA(c, h.host(&S.h_args, 1));
  return VBX_OK;
}

// The back half of a call whose K exceeds max_updates_per_pass, in passes (see integrate_device).
static int apply_in_passes(vbx_ctx* c, const ScanRoute& x, ScanArgs a, Tally& tally, uint32_t* passes) {
  cudaStream_t s = x.s;
  const uint32_t n = a.P.n;
  std::vector<uint32_t> off(n + 1);
  VBX_CUDA(c, cudaMemcpyAsync(off.data(), x.S.off, (size_t)(n + 1) * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
  VBX_CUDA(c, cudaStreamSynchronize(s));
  if (a.P.kind == VBX_MERGED) {
    // the scan wrote the offsets of the bundles and, at [n], the total; ranks past the last bundle hold nothing
    const uint32_t nr = std::min(x.S.h_state->n_ray_list, n);
    for (uint32_t i = nr + 1; i < n; ++i) off[i] = off[n];
  }
  // every pass's slot range first: a call that cannot be split is refused before any pass runs (the
  // passes share the scan's block table, which only a call's last pass clears)
  std::vector<std::pair<uint32_t, uint32_t>> ranges;
  for (uint32_t lo = 0; lo < n;) {
    // the longest slot range starting at lo whose records fit
    const uint64_t room = (uint64_t)off[lo] + c->max_updates;
    uint32_t hi = (uint32_t)(std::upper_bound(off.begin() + lo, off.end(), room,
                                              [](uint64_t v, uint32_t o) { return v < (uint64_t)o; }) -
                             off.begin());
    hi = hi > 0 ? hi - 1 : 0;  // off[hi] <= room
    if (hi <= lo) return fail(c, VBX_E_CAPACITY, "a single ray has more updates than max_updates_per_pass");
    if (off[hi] > off[lo]) ranges.emplace_back(lo, hi);
    lo = hi;
  }
  *passes = (uint32_t)ranges.size();
  for (const auto& r : ranges) {
    const uint32_t lo = r.first, hi = r.second;
    const unsigned long long kp = (unsigned long long)off[hi] - off[lo];
    a.P.emit_lo = lo;
    a.P.emit_hi = hi;  // (the last range ends at n: its k_assign clears the scan's block table)
    a.P.emit_base = off[lo];
    a.nb_cur = (uint32_t)c->nb_cur;
    VBX_CUDA(c, cudaStreamSynchronize(s));  // (the previous pass has read its arguments)
    if (int rc = upload_args(c, x, a)) return rc;
    k_pass_begin<<<1, 1, 0, s>>>(x.S.d_state, kp);
    ++tally.launches;
    launch_emit(c, x, a.P, tally);
    if (int rc = back_half(c, x, tally)) return rc;
  }
  return VBX_OK;
}

// ScanParams::single_walk: a ray's update count is known from its DDA set-up alone (not Fast, no
// anti-grazing).  Otherwise the front half walks every ray twice, once to count its updates and once to emit
// them, and Fast's counting walk reads its approximate sets, which must see the scans in schedule order; only
// single walks are pipelined (integrate_async).
static bool single_walk(const vbx_tsdf_config& cfg, int kind) {
  return kind != VBX_FAST && !(kind == VBX_MERGED && cfg.enable_anti_grazing);
}

static void fill_params(vbx_ctx* c, int kind, const float q[4], const float t[3], uint32_t n, int freespace,
                        ScanParams& P) {
  const vbx_tsdf_config& cfg = c->cfg;
  std::memset(&P, 0, sizeof(P));
  P.T.w = q[0];
  P.T.x = q[1];
  P.T.y = q[2];
  P.T.z = q[3];
  P.T.t = f3(t[0], t[1], t[2]);
  P.origin = P.T.t;  // T_G_C.getPosition()
  P.voxel_size = c->voxel_size;
  P.voxel_size_inv = c->voxel_size_inv;
  P.trunc = cfg.default_truncation_distance;
  P.min_ray = cfg.min_ray_length_m;
  P.max_ray = cfg.max_ray_length_m;
  P.up.trunc = cfg.default_truncation_distance;
  P.up.max_weight = cfg.max_weight;
  P.up.voxel_size = c->voxel_size;
  P.up.use_weight_dropoff = cfg.use_weight_dropoff;
  P.up.use_sparsity = cfg.use_sparsity_compensation_factor;
  P.up.sparsity_factor = cfg.sparsity_compensation_factor;
  P.L = c->L;
  P.kind = kind;
  P.freespace = freespace;
  P.use_const_weight = cfg.use_const_weight;
  P.allow_clear = cfg.allow_clear;
  P.carving = cfg.voxel_carving_enabled;
  P.anti_grazing = cfg.enable_anti_grazing;
  P.order_mode = cfg.integration_order_mode;
  P.n = n;
  P.n_groups = n / 1024u;
  P.start_inv = cfg.start_voxel_subsampling_factor * c->voxel_size_inv;
  P.max_collisions = cfg.max_consecutive_ray_collisions;
  P.max_updates = c->max_updates;
  P.set_offset = c->set_offset;
  P.own_world = c->opt.world_size > 1 ? c->opt.world_size : 1;
  P.own_rank = c->opt.rank;
  P.emit_lo = 0;
  P.emit_hi = 0xffffffffu;
  P.emit_base = 0;
  P.single_walk = single_walk(cfg, kind) ? 1 : 0;
}

// Both approximate sets as ApproxHashSet's constructor and full reset leave them: every slot 0 but word 0,
// which holds a value no hash has, so that hash 0 does not read as present there (approx_hash_array.h:155-168).
int init_fast_sets(vbx_ctx* c, cudaStream_t s) {
  for (unsigned long long* set : {c->set_start, c->set_observed}) {
    VBX_CUDA(c, cudaMemsetAsync(set, 0, kApproxSetWords * sizeof(unsigned long long), s));
    VBX_CUDA(c, cudaMemsetAsync(set, 0xff, sizeof(unsigned long long), s));
  }
  return VBX_OK;
}

// FastTsdfIntegrator::integratePointCloud: resetApproxSet every clear_checks_every_n_frames calls (cc:563-568),
// which moves the sets' slot offset on by one and clears them once it reaches kApproxSetResets.  The slots
// the new offset reaches keep what earlier calls stored.  The call counter is the context's own; the
// reference's is one function-level static shared by every Fast integrator of the process (cc:564).
static int reset_fast_sets(vbx_ctx* c, cudaStream_t s) {
  if (++c->fast_reset_counter < c->cfg.clear_checks_every_n_frames) return VBX_OK;
  c->fast_reset_counter = 0;
  if (++c->set_offset < kApproxSetResets) return VBX_OK;
  c->set_offset = 0;
  return init_fast_sets(c, s);
}

int integrate_device(vbx_ctx* c, const ScanRoute& x, int kind, const float q[4], const float t[3], const float* d_xyz,
                     const uint8_t* d_rgba, uint64_t n64, int freespace) {
  if (kind < VBX_SIMPLE || kind > VBX_FAST) return fail(c, VBX_E_INVALID, "Unknown TSDF integrator type");
  if (n64 > c->max_points) return fail(c, VBX_E_CAPACITY, "cloud larger than max_points_per_scan");
  cudaStream_t s = x.s;
  const vbx_ctx::ScratchSet& S = x.S;
  const vbx_ctx::FrontLane& F = x.F;
  const vbx_tsdf_config& cfg = c->cfg;
  std::memset(c->counters, 0, sizeof(c->counters));
  if (kind == VBX_FAST) {
    if (int rc = reset_fast_sets(c, s)) return rc;
  }
  // Fast checks max_integration_time_s before each point, after the reset (cc:496-500): at 0 or less, or
  // NaN, it integrates no point.  A positive limit is wall-clock time and is not enforced.
  const uint32_t n = (kind == VBX_FAST && !(cfg.max_integration_time_s > 0.f)) ? 0u : (uint32_t)n64;

  ScanParams P;
  fill_params(c, kind, q, t, n, freespace, P);

  VBX_CUDA(c, cudaEventRecord(c->ev0, s));
  VBX_CUDA(c, cudaMemsetAsync(S.d_state, 0, sizeof(ScanState), s));
  if (n == 0) {
    VBX_CUDA(c, cudaEventRecord(c->ev1, s));
    VBX_CUDA(c, cudaStreamSynchronize(s));
    c->last_ms = 0.f;
    return VBX_OK;
  }
  ScanArgs a;
  fill_args(c, P, d_xyz, d_rgba, &a);
  if (int rc = upload_args(c, x, a)) return rc;
  const int TB = 256;
  Tally tally{c, s, x.marks};
  tally.begin();

  const uint32_t* order = nullptr;
  if (cfg.integration_order_mode == 1) {
    // SortedThreadSafeIndex: ascending |p|^2 (stable here; std::sort leaves ties unspecified)
    k_sqnorm_keys<<<grid_for(n, TB), TB, 0, s>>>(n, d_xyz, S.pkeys0, F.pvals[0]);
    ++tally.launches;
    if (int rc = own_sort(c, x, 0, S.pkeys0, F.pvals[0], F.pkeys1, F.pvals[1], nullptr, n, n, 64, true, tally)) return rc;
    VBX_CUDA(c, cudaMemcpyAsync(c->order, F.pvals[0], n * sizeof(uint32_t), cudaMemcpyDeviceToDevice, s));
    k_invert_order<<<grid_for(n, TB), TB, 0, s>>>(n, c->order, c->order_inv);
    ++tally.launches;
    order = c->order;
  }

  if (int rc = front_half(c, x, P, order, tally)) return rc;
  // own sort: K stays on the device, the whole call is enqueued without a host round trip
  if (int rc = back_half(c, x, tally)) return rc;
  VBX_CUDA(c, cudaEventRecord(c->ev1, s));
  VBX_CUDA(c, cudaMemcpyAsync(S.h_state, S.d_state, sizeof(ScanState), cudaMemcpyDeviceToHost, s));
  VBX_CUDA(c, cudaStreamSynchronize(s));
  const ScanState& h = *S.h_state;
  const uint32_t blocks_before = c->n_blocks;
  const bool chunked = h.error == kErrUpdatesFull;
  uint32_t passes = 1;
  if (chunked) {
    // More update records than one pass holds.  Nothing was emitted or applied; the per-ray
    // tables, counts and offsets of the front half stand.  Apply the call in passes over
    // contiguous ray-slot ranges: every voxel still sees its updates in ray-rank order, so
    // the result is the one-pass result bit for bit.
    if (int rc = apply_in_passes(c, x, a, tally, &passes)) return rc;
    VBX_CUDA(c, cudaEventRecord(c->ev1, s));
    VBX_CUDA(c, cudaMemcpyAsync(S.h_state, S.d_state, sizeof(ScanState), cudaMemcpyDeviceToHost, s));
    VBX_CUDA(c, cudaStreamSynchronize(s));
  }
  if (int rc = check_state_errors(c, h)) return rc;
  c->n_blocks = h.n_blocks;
  VBX_CUDA(c, cudaGetLastError());
  VBX_CUDA(c, cudaEventElapsedTime(&c->last_ms, c->ev0, c->ev1));
  tally.collect();
  c->launches += tally.launches;
  report_scan(c, h, kind, tally.launches, passes, chunked ? (uint64_t)(c->n_blocks - blocks_before) : (uint64_t)h.n_new);
  return VBX_OK;
}

static void report_apply_paths(vbx_ctx* c, const ScanState& h) {
  for (int i = 0; i < kApplyPaths; ++i) c->apply_paths[i] = h.apply_paths[i];
}

// The status block of a synchronous call (integrate_device) or a collected asynchronous scan (harvest_async)
void report_scan(vbx_ctx* c, const ScanState& h, int kind, uint64_t launches, uint64_t passes,
                 uint64_t blocks_allocated) {
  uint64_t* cnt = c->counters;
  std::memset(cnt, 0, sizeof(c->counters));
  cnt[kCntRays] = h.n_rays;
  cnt[kCntClearRays] = h.n_clear_rays;
  cnt[kCntUpdates] = h.total_found;
  cnt[kCntVoxels] = h.n_voxels;
  cnt[kCntBlocksTouched] = h.n_touched;
  cnt[kCntBlocksAllocated] = blocks_allocated;
  cnt[kCntValidPoints] = kind == VBX_MERGED ? h.n_valid_points : (uint64_t)h.n_rays + h.n_clear_rays;
  cnt[kCntLaunches] = launches;
  cnt[kCntRefoldedBundles] = h.n_refold;
  cnt[kCntRefoldedPoints] = h.refold_members;
  cnt[kCntPasses] = passes;
  cnt[kCntBundleKeyBits] = h.key_bits;
  // (vbx_get_counters adds the context's totals)
  if (h.total_found) c->record_hint = h.total_found;
  if (kind == VBX_MERGED && !(h.error & kFatalErrors)) c->bundle_hint = std::max(h.n_rays, h.n_clear_rays);
  report_apply_paths(c, h);
}

// ------------------------------------------------------------- asynchronous submission
// integratePointCloud without the host round trip: the call enqueues the scan and returns.  A scan
// passes through four stages:
//   front   (Merged: keys, bundle sort, bundle fold) record offsets and the ray walk that writes the
//           update records against the scan's private block table -- touches nothing of the map; the
//           front lanes alternate, so several front halves can run side by side
//   walk    block creation (k_assign resolves the ray walk's local ids), slot assignment
//   sort    record sort and apply preparation on scan-private buffers
//   apply   the per-voxel updates
// Stages that touch the map run in submission order (the walk of scan i+1 only inserts new hash
// entries and never moves existing ones, so it can overlap the apply of scan i).  Up to kSets scans
// are in flight, each with its own hand-off buffers; results (counters, errors) of a scan are
// collected when its set is reused or at the next synchronous call / vbx_sync.
//
// A scan is one launch of a CUDA graph: the kernels and hand-offs the enqueue code above issues,
// captured once per (hand-off set, front lane, kind) and kept until vbx_destroy.  What changes from
// scan to scan is in the set's argument block (uploaded by the graph's first node) or in three kernel
// nodes updated in place (the two sorts' grids, k_bundle_order's form and shared memory).  The order between
// scans is carried by events: the front half waits for the lane's previous front half, the walk for
// the previous scan's walk, the record sort for the one two scans back, the apply for the previous
// scan's apply.  An event-record node of an earlier launched graph is the event's most recent record
// for a later one (tests/test_async_graph_gpu.py checks the maps bit for bit against synchronous calls).
// sms: the grid unit of the graph's kernels.
static int capture_scan(vbx_ctx* c, vbx_ctx::ScratchSet& S, vbx_ctx::FrontLane& F, const ScanParams& P,
                        vbx_ctx::ScanGraph& G, unsigned int sms) {
  const int k = (int)(&S - c->set), sets = c->pipe.sets_in_use;
  const vbx_ctx::ScratchSet& prev = c->set[(k + sets - 1) % sets];
  const vbx_ctx::ScratchSet& prev2 = c->set[(k + 2 * sets - 2) % sets];
  const Capture cap{c->pipe.stream_s, c->stream, S.walked, S.sorted, S.applied, prev2.sorted, prev.applied,
                    {c->pipe.cap_ev[2], c->pipe.cap_ev[3]}};
  const ScanRoute front{S, F, F.stream, sms, false}, walk{S, F, c->pipe.stream_e, sms, false};
  cudaStream_t o = S.stream;
  Tally tally{c, F.stream, false};  // (the graph's kernel nodes are counted below)
  auto enqueue = [&]() -> int {
    VBX_CUDA(c, cudaMemcpyAsync(S.d_args, S.h_args, sizeof(ScanArgs), cudaMemcpyHostToDevice, o));
    VBX_CUDA(c, cudaStreamWaitEvent(o, S.copy_done, cudaEventWaitExternal));  // a host cloud's copy
    VBX_CUDA(c, cudaStreamWaitEvent(o, F.done, cudaEventWaitExternal));       // the lane's previous front half
    // ---- front half on the lane's stream
    VBX_CUDA(c, cudaEventRecord(c->pipe.cap_ev[0], o));
    VBX_CUDA(c, cudaStreamWaitEvent(F.stream, c->pipe.cap_ev[0], 0));
    VBX_CUDA(c, cudaMemsetAsync(S.d_state, 0, sizeof(ScanState), F.stream));
    if (c->pipe.timeline) VBX_CUDA(c, cudaEventRecordWithFlags(S.front_start, F.stream, cudaEventRecordExternal));
    if (int rc = front_half(c, front, P, nullptr, tally)) return rc;
    VBX_CUDA(c, cudaEventRecordWithFlags(F.done, F.stream, cudaEventRecordExternal));
    if (c->pipe.timeline) VBX_CUDA(c, cudaEventRecordWithFlags(S.front_done, F.stream, cudaEventRecordExternal));
    // ---- walk, record sort and apply (sort_and_apply hands off between their streams)
    VBX_CUDA(c, cudaEventRecord(c->pipe.cap_ev[1], F.stream));
    VBX_CUDA(c, cudaStreamWaitEvent(c->pipe.stream_e, c->pipe.cap_ev[1], 0));
    VBX_CUDA(c, cudaStreamWaitEvent(c->pipe.stream_e, prev.walked, cudaEventWaitExternal));
    // Scans run their map-touching stages in submission order.  A scan that cannot be applied
    // asynchronously (more update records than one pass holds) raises the context's hold flag here;
    // every scan queued behind it then skips its back half, and the host redoes all of them
    // synchronously, in order, from the retained inputs (recover_async, vbx_capi.cu).
    k_back_begin<<<1, 1, 0, c->pipe.stream_e>>>(S.d_state, c->pipe.d_hold);
    if (int rc = back_half(c, walk, tally, &cap)) return rc;
    VBX_CUDA(c, cudaMemcpyAsync(S.h_state, S.d_state, sizeof(ScanState), cudaMemcpyDeviceToHost, cap.apply));
    // every stream of the capture joins its origin
    const cudaStream_t joined[4] = {F.stream, c->pipe.stream_e, c->pipe.stream_s, c->stream};
    for (int j = 0; j < 4; ++j) {
      VBX_CUDA(c, cudaEventRecord(c->pipe.cap_ev[4 + j], joined[j]));
      VBX_CUDA(c, cudaStreamWaitEvent(o, c->pipe.cap_ev[4 + j], 0));
    }
    return VBX_OK;
  };
  VBX_CUDA(c, cudaStreamBeginCapture(o, cudaStreamCaptureModeThreadLocal));
  int rc = enqueue();
  cudaGraph_t g = nullptr;
  cudaGraphExec_t x = nullptr;
  Holdings pending;  // the graph and its exec until they are complete and handed to the context
  pending.graph(&g, &x);
  const cudaError_t e = cudaStreamEndCapture(o, &g);
  if (rc == VBX_OK && e != cudaSuccess) rc = cuda_fail(c, e, "cudaStreamEndCapture");
  // Per-node stage priorities (apply > walk > sort > front, as the streams of the unpipelined stages had)
  // and the nodes whose launch shape follows the scan or the hints.
  cudaGraphNode_t point_sort = nullptr, record_sort = nullptr, order = nullptr;
  cudaKernelNodeParams pp = {}, rp = {}, op = {};
  uint64_t launches = 0;
  if (rc == VBX_OK) {
    const int walk_prio = std::min(c->prio_lo, c->prio_hi + 1), sort_prio = std::min(c->prio_lo, c->prio_hi + 2);
    size_t nn = 0;
    cudaGraphGetNodes(g, nullptr, &nn);
    std::vector<cudaGraphNode_t> nodes(nn);
    cudaGraphGetNodes(g, nodes.data(), &nn);
    for (cudaGraphNode_t nd : nodes) {
      cudaGraphNodeType ty;
      cudaKernelNodeParams kp;
      if (cudaGraphNodeGetType(nd, &ty) != cudaSuccess || ty != cudaGraphNodeTypeKernel ||
          cudaGraphKernelNodeGetParams(nd, &kp) != cudaSuccess) {
        continue;
      }
      ++launches;
      cudaLaunchAttributeValue prio = {};
      prio.priority = c->prio_lo;
      // (the ray walk, k_rays_emit / k_rays_emit_warp, is a front-half node: it keeps the front priority)
      if (kp.func == (void*)k_back_begin || kp.func == (void*)k_assign) {
        prio.priority = walk_prio;
      } else if (kp.func == (void*)k_sort<uint32_t> || kp.func == (void*)k_apply_prep<false>) {
        prio.priority = sort_prio;
      } else if (kp.func == (void*)k_apply) {
        prio.priority = c->prio_hi;
      }
      if (cudaGraphKernelNodeSetAttribute(nd, cudaLaunchAttributePriority, &prio) != cudaSuccess) {
        rc = fail(c, VBX_E_CUDA, "cudaGraphKernelNodeSetAttribute(priority)");
      }
      if (kp.func == (void*)k_sort<uint64_t>) {
        point_sort = nd;
        pp = kp;
      } else if (kp.func == (void*)k_sort<uint32_t>) {
        record_sort = nd;
        rp = kp;
      } else if (kp.func == (void*)k_bundle_order) {
        order = nd;
        op = kp;
      }
    }
    if (rc == VBX_OK && (!record_sort || (P.kind == VBX_MERGED) != (order != nullptr && point_sort != nullptr))) {
      rc = fail(c, VBX_E_CUDA, "captured scan graph: sort / bundle order node not found");
    }
  }
  if (rc == VBX_OK) {
    const cudaError_t ei = cudaGraphInstantiateWithFlags(&x, g, cudaGraphInstantiateFlagUseNodePriority);
    if (ei != cudaSuccess) rc = cuda_fail(c, ei, "cudaGraphInstantiateWithFlags");
  }
  if (rc == VBX_OK) {
    // (otherwise the graph's first launch uploads it, in the middle of a stream of scans)
    const cudaError_t eu = cudaGraphUpload(x, o);
    if (eu != cudaSuccess) rc = cuda_fail(c, eu, "cudaGraphUpload");
  }
  if (rc != VBX_OK) return rc;
  G.graph = std::exchange(g, nullptr);
  G.exec = std::exchange(x, nullptr);
  c->pipe.own.graph(&G.graph, &G.exec);
  G.launches = launches;
  G.point_sort = point_sort;
  G.point_grid = pp.gridDim.x;
  G.record_sort = record_sort;
  G.record_grid = rp.gridDim.x;
  G.order = order;
  G.order_grid = op.gridDim.x;
  G.order_smem = op.sharedMemBytes;
  return VBX_OK;
}

static int set_grid(vbx_ctx* c, vbx_ctx::ScanGraph& G, cudaGraphNode_t node, unsigned int grid, unsigned int* now) {
  if (grid == *now) return VBX_OK;
  cudaKernelNodeParams p;
  VBX_CUDA(c, cudaGraphKernelNodeGetParams(node, &p));
  p.gridDim.x = grid;
  VBX_CUDA(c, cudaGraphExecKernelNodeSetParams(G.exec, node, &p));
  *now = grid;
  return VBX_OK;
}

// Brings the kernel nodes of a scan graph whose launch shape varies up to date (a no-op unless it moved):
// the point sort's grid (a grid larger than the scan's tiles keeps blocks waiting between passes), the
// record sort's grid, k_bundle_order's form (grid) and shared memory.  sms: the grid unit the graph was captured with.
static int update_scan_graph(vbx_ctx* c, vbx_ctx::ScanGraph& G, uint32_t n, unsigned int sms) {
  if (G.point_sort) {
    if (int rc = set_grid(c, G, G.point_sort, sort_grid(c, 0, n, sms), &G.point_grid)) return rc;
  }
  if (int rc = set_grid(c, G, G.record_sort, sort_grid(c, 1, c->record_hint, sms), &G.record_grid)) return rc;
  if (G.order) {
    const OrderLaunch o = order_launch(c, n);
    if (o.grid != G.order_grid || o.smem_bytes != G.order_smem) {
      cudaKernelNodeParams p;
      VBX_CUDA(c, cudaGraphKernelNodeGetParams(G.order, &p));
      uint32_t smem_words = (uint32_t)(o.smem_bytes / 4);
      void* args[6];
      std::copy(p.kernelParams, p.kernelParams + 6, args);
      args[2] = &smem_words;
      p.kernelParams = args;
      p.gridDim.x = o.grid;
      p.sharedMemBytes = (unsigned int)o.smem_bytes;
      VBX_CUDA(c, cudaGraphExecKernelNodeSetParams(G.exec, G.order, &p));
      G.order_grid = o.grid;
      G.order_smem = o.smem_bytes;
    }
  }
  return VBX_OK;
}

// sync: where a synchronous call goes (sync_route): the fallback for scans that cannot be overlapped, and the
// grid unit the graphs' share of the GPU is taken from.
int integrate_async(vbx_ctx* c, const ScanRoute& sync, int kind, const float q[4], const float t[3], const float* xyz,
                    const uint8_t* rgba, uint64_t n64, int freespace, int on_device) {
  if (kind < VBX_SIMPLE || kind > VBX_FAST) return fail(c, VBX_E_INVALID, "Unknown TSDF integrator type");
  if (n64 > c->max_points) return fail(c, VBX_E_CAPACITY, "cloud larger than max_points_per_scan");
  const vbx_tsdf_config& cfg = c->cfg;
  const bool overlappable = single_walk(cfg, kind) && cfg.integration_order_mode == 0 && n64 > 0;
  if (!overlappable) {
    // scans that are not a single walk (counted and emitted by separate walks; Fast's count reads its
    // approximate sets in schedule order) or that follow the sorted integration order run in order
    if (int rc = drain_async(c)) return rc;
    const float* dx = xyz;
    const uint8_t* dr = rgba;
    if (!on_device && n64) {
      VBX_CUDA(c, cudaMemcpyAsync(sync.S.d_xyz, xyz, n64 * 3 * sizeof(float), cudaMemcpyHostToDevice, sync.s));
      VBX_CUDA(c, cudaMemcpyAsync(sync.S.d_rgba, rgba, n64 * 4, cudaMemcpyHostToDevice, sync.s));
      dx = sync.S.d_xyz;
      dr = sync.S.d_rgba;
    }
    return integrate_device(c, sync, kind, q, t, dx, dr, n64, freespace);
  }
  if (int rc = ensure_async(c)) return rc;
  const uint32_t n = (uint32_t)n64;
  const int k = (int)(c->pipe.seq % c->pipe.sets_in_use);
  const int l = (int)(c->pipe.seq % c->pipe.lanes_in_use);
  vbx_ctx::ScratchSet& S = c->set[k];
  const auto t_enter = std::chrono::steady_clock::now();
  if (S.in_flight) {  // bounded run-ahead: wait for the scan that used this hand-off set
    VBX_CUDA(c, cudaEventSynchronize(S.back_done));
    c->pipe.wait_ns += (uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t_enter).count();
    harvest_async(c, S);
    if (S.redo) {
      // it (and every scan queued behind it) did not run its back half: redo them now, in order
      if (int rc = drain_async(c)) return rc;
    }
  }
  ScanParams P;
  fill_params(c, kind, q, t, n, freespace, P);
  const float* dx = xyz;
  const uint8_t* dr = rgba;
  if (!on_device) {
    // the copy engine works ahead of the front half on a stream of its own
    // (two copy streams alternate, so two scans' clouds can be in flight on the copy engines at once)
    cudaStream_t sc = (c->pipe.seq & 1u) ? c->stream_c2 : c->stream_c;
    if (cudaMemcpyAsync(S.d_xyz, xyz, (size_t)n * 3 * sizeof(float), cudaMemcpyHostToDevice, sc) != cudaSuccess ||
        cudaMemcpyAsync(S.d_rgba, rgba, (size_t)n * 4, cudaMemcpyHostToDevice, sc) != cudaSuccess ||
        cudaEventRecord(S.copy_done, sc) != cudaSuccess) {
      return fail(c, VBX_E_CUDA, "asynchronous host-to-device copy failed");
    }
    dx = S.d_xyz;
    dr = S.d_rgba;
  }
  // the set's previous scan has finished (back_done), so its page-locked argument block is free
  fill_args(c, P, dx, dr, S.h_args);
  const int nb = c->nb_cur;
  const int variant = kind == VBX_MERGED ? vbx_ctx::kGraphMerged : vbx_ctx::kGraphSimple;
  vbx_ctx::ScanGraph& G = S.graph[l][variant];
  int rc = VBX_OK;
  // The pipeline runs the kernels of several scans at once (front halves, a walk, a record sort, an apply):
  // a persistent grid sized for the whole GPU only holds SM slots that the other scans' kernels need.  The
  // graphs' grids are sized for a quarter of the SMs (DESIGN.md §5b: the pace against the grid scale).
  const unsigned int sms = std::max(1u, sync.sms / 4);
  if (!G.exec) {
    // the first scan of its kind captures the graphs of every (set, lane) pair the submission order
    // reaches (set = seq % sets, lane = seq % lanes), so that no later scan waits for a capture
    const int pairs = std::lcm(c->pipe.sets_in_use, c->pipe.lanes_in_use);
    for (int j = 0; j < pairs && rc == VBX_OK; ++j) {
      const int kj = j % c->pipe.sets_in_use, lj = j % c->pipe.lanes_in_use;
      rc = capture_scan(c, c->set[kj], c->lane[lj], P, c->set[kj].graph[lj][variant], sms);
    }
  }
  if (rc == VBX_OK) rc = update_scan_graph(c, G, n, sms);
  if (rc == VBX_OK && (cudaGraphLaunch(G.exec, S.stream) != cudaSuccess || cudaEventRecord(S.back_done, S.stream) != cudaSuccess)) {
    rc = fail(c, VBX_E_CUDA, "launching the scan's graph failed");
  }
  c->nb_cur = rc == VBX_OK ? nb ^ 1 : nb;  // k_assign of the scan moves the block count to the other word
  if (rc != VBX_OK) return rc;
  S.in_flight = true;
  S.kind = kind;
  S.launches = G.launches;
  S.seq = c->pipe.seq;
  S.redo = false;
  std::memcpy(S.q, q, sizeof(S.q));
  std::memcpy(S.t, t, sizeof(S.t));
  S.n = n64;
  S.freespace = freespace;
  S.in_xyz = dx;   // (the set's private copy of a host cloud, or the caller's device buffers)
  S.in_rgba = dr;
  c->pipe.submit_ns += (uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t_enter).count();
  c->launches += G.launches;
  c->pipe.seq += 1;
  if (c->pipe.deferred_rc) {
    rc = c->pipe.deferred_rc;
    c->err = c->pipe.deferred_msg;
    c->pipe.deferred_rc = 0;
    return rc;
  }
  return VBX_OK;
}

// ------------------------------------------------------------------ test hooks
// k_bundle_order on caller-supplied hashes (element e = e-th inserted key, hash hashes[e]): out[p] = the
// element at iteration position p.  tests/test_order_gpu.py compares it with a real std::unordered_map.
// force_global: pretend there is no shared memory, i.e. run every stage grid-wide on the global tables.
__global__ void k_debug_order_setup(OrderScratch g, uint32_t n, ScanState* st) {
  const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e < n) g.head_of[e] = e;
  if (e == 0) {
    st->n_rays = n;
    st->n_clear_rays = 0;
  }
}

int debug_bundle_order(vbx_ctx* c, const uint32_t* hashes, uint32_t n, int force_global, uint32_t* out) {
  cudaStream_t s = c->stream;
  const vbx_ctx::ScratchSet& S = c->set[0];
  if (n > c->max_points) return fail(c, VBX_E_CAPACITY, "debug_bundle_order: n > max_points_per_scan");
  if (n == 0) return VBX_OK;
  RehashSchedule rs = c->rehash;
  OrderScratch g = c->lane[0].order_scratch;
  VBX_CUDA(c, cudaMemsetAsync(S.d_state, 0, sizeof(ScanState), s));
  VBX_CUDA(c, cudaMemcpyAsync(g.h, hashes, (size_t)n * 4, cudaMemcpyHostToDevice, s));
  k_debug_order_setup<<<grid_for(n, 256), 256, 0, s>>>(g, n, S.d_state);
  uint32_t smem_words = force_global ? 0u : (uint32_t)(c->order_smem_bytes / 4);
  uint32_t* ray_list = S.ray_list;
  uint32_t* cta_tot = g.cta_tot;
  ScanState* st = S.d_state;
  void* args[] = {&rs, &g, &smem_words, &ray_list, &cta_tot, &st};
  VBX_CUDA(c, cudaLaunchCooperativeKernel((void*)k_bundle_order, dim3(kOrderGrid), dim3(kOrderThreads), args,
                                          c->order_smem_bytes, s));
  VBX_CUDA(c, cudaMemcpyAsync(out, S.ray_list, (size_t)n * 4, cudaMemcpyDeviceToHost, s));
  VBX_CUDA(c, cudaMemcpyAsync(S.h_state, S.d_state, sizeof(ScanState), cudaMemcpyDeviceToHost, s));
  VBX_CUDA(c, cudaStreamSynchronize(s));
  VBX_CUDA(c, cudaGetLastError());
  if (S.h_state->error) return fail(c, VBX_E_CAPACITY, "debug_bundle_order: table capacity");
  return VBX_OK;
}

__global__ void k_iota(uint32_t* v, uint32_t n) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) v[i] = i;
}

// Sorts n host keys with the engine's radix sort and returns the sorted keys and the permutation
// (tests/test_sort_gpu.py checks it against a stable host sort).  key_bytes 4 uses the update-
// record buffers with the count in device memory, 8 the point-key buffers with a host count.
int debug_sort(vbx_ctx* c, const void* keys, int key_bytes, uint32_t n, int key_bits, void* keys_out,
               uint32_t* vals_out) {
  const ScanRoute x = sync_route(c);
  const vbx_ctx::ScratchSet& S = x.S;
  const vbx_ctx::FrontLane& F = x.F;
  cudaStream_t s = x.s;
  Tally tally{c, s, false};
  if (key_bytes == 4) {
    if (n > c->max_updates) return fail(c, VBX_E_CAPACITY, "debug_sort: n > max_updates_per_pass");
    VBX_CUDA(c, cudaMemcpyAsync(S.ckeys[0], keys, (size_t)n * 4, cudaMemcpyHostToDevice, s));
    k_iota<<<c->grid_sms, 256, 0, s>>>(S.cvals[0], n);
    VBX_CUDA(c, cudaMemsetAsync(S.d_state, 0, sizeof(ScanState), s));
    const unsigned long long nn = n;
    VBX_CUDA(c, cudaMemcpyAsync(&S.d_state->total_updates, &nn, sizeof(nn), cudaMemcpyHostToDevice, s));
    if (int rc = own_sort(c, x, 1, S.ckeys[0], S.cvals[0], S.ckeys[1], S.cvals[1], &S.d_state->total_updates, 0, n,
                          key_bits, true, tally)) {
      return rc;
    }
    VBX_CUDA(c, cudaMemcpyAsync(keys_out, S.ckeys[0], (size_t)n * 4, cudaMemcpyDeviceToHost, s));
    VBX_CUDA(c, cudaMemcpyAsync(vals_out, S.cvals[0], (size_t)n * 4, cudaMemcpyDeviceToHost, s));
  } else if (key_bytes == 8) {
    if (n > c->max_points) return fail(c, VBX_E_CAPACITY, "debug_sort: n > max_points_per_scan");
    VBX_CUDA(c, cudaMemcpyAsync(S.pkeys0, keys, (size_t)n * 8, cudaMemcpyHostToDevice, s));
    k_iota<<<c->grid_sms, 256, 0, s>>>(F.pvals[0], n);
    if (int rc = own_sort(c, x, 0, S.pkeys0, F.pvals[0], F.pkeys1, F.pvals[1], nullptr, n, n, key_bits, true, tally)) {
      return rc;
    }
    VBX_CUDA(c, cudaMemcpyAsync(keys_out, S.pkeys0, (size_t)n * 8, cudaMemcpyDeviceToHost, s));
    VBX_CUDA(c, cudaMemcpyAsync(vals_out, F.pvals[0], (size_t)n * 4, cudaMemcpyDeviceToHost, s));
  } else {
    return fail(c, VBX_E_INVALID, "debug_sort: key_bytes must be 4 or 8");
  }
  VBX_CUDA(c, cudaStreamSynchronize(s));
  VBX_CUDA(c, cudaGetLastError());
  return VBX_OK;
}

// vbx_debug_apply: touched id i -> hash position of block i, the records' keys (touched id, voxel) and
// ordinals, and what the record sort and k_apply_prep otherwise learn from k_assign and the offset scan.
// A block that is not a TSDF block of the map sets *bad.
__global__ void k_debug_apply_setup(Tables tab, const uint64_t* __restrict__ bkeys, uint32_t nb,
                                    const uint32_t* __restrict__ rec_block, const uint32_t* __restrict__ rec_voxel,
                                    unsigned long long n, int L, uint32_t* keys, uint32_t* vals, ScanState* st,
                                    uint32_t* bad) {
  const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < nb) {
    const uint32_t hp = find_block(tab, bkeys[i]);
    const int32_t slot = hp == 0xffffffffu ? -1 : tab.hslot[hp];
    if (slot < 0 || (tab.slot_updated[slot] & kSlotNoTsdf)) *bad = 1u;
    tab.touched_list[i] = hp;
  }
  if (i < n) {
    keys[i] = (rec_block[i] << (3 * L)) | rec_voxel[i];
    vals[i] = (uint32_t)i;
  }
  if (i == 0) {
    st->total_updates = n;
    st->total_found = n;
    st->rec_key_bits = 3u * (uint32_t)L + (uint32_t)(32 - __clz(nb));
  }
}

// Runs the production record sort, k_apply_prep (on the given values) and k_apply over caller-given
// update records of blocks already in the map.  Record r belongs to block idx3[rec_block[r]], voxel
// rec_voxel[r]; its sdf and weight are the final ones updateTsdfVoxel uses (after drop-off and sparsity).
// Records of one voxel are applied in the order given.  Block updated() bits are left alone.
int debug_apply(vbx_ctx* c, const int32_t* idx3, uint32_t nb, uint64_t n, const uint32_t* rec_block,
                const uint32_t* rec_voxel, const float* sdf, const float* w, const uint8_t* rgba, uint64_t paths[16]) {
  const ScanRoute x = sync_route(c);
  const vbx_ctx::ScratchSet& S = x.S;
  cudaStream_t s = x.s;
  if (n > c->max_updates) return fail(c, VBX_E_INVALID, "debug_apply: more records than max_updates_per_pass");
  if (nb > c->tab.touched_cap) return fail(c, VBX_E_INVALID, "debug_apply: too many blocks");
  for (uint64_t r = 0; r < n; ++r) {
    if (rec_block[r] >= nb) return fail(c, VBX_E_INVALID, "debug_apply: block ordinal out of range");
    if (rec_voxel[r] >= c->vox_per_block) return fail(c, VBX_E_INVALID, "debug_apply: voxel index >= voxels_per_side^3");
  }
  std::vector<uint64_t> bkeys(nb);
  for (uint32_t i = 0; i < nb; ++i) bkeys[i] = pack3(idx3[3 * i], idx3[3 * i + 1], idx3[3 * i + 2]);
  {
    // a block listed twice would give one voxel two runs under different keys, applied side by side
    std::vector<uint64_t> sorted = bkeys;
    std::sort(sorted.begin(), sorted.end());
    if (std::adjacent_find(sorted.begin(), sorted.end()) != sorted.end()) {
      return fail(c, VBX_E_INVALID, "debug_apply: a block is listed twice");
    }
  }
  // scratch: block keys, the records' block / voxel, sdf, weight, colour, and the "not in the map" flag
  const size_t n4 = (size_t)n * 4;
  char* buf = nullptr;
  const size_t bytes = (size_t)nb * 8 + 5 * n4 + 4;
  Holdings scratch;
  VBX_CUDA(c, scratch.dev(&buf, bytes));
  uint64_t* d_bkeys = reinterpret_cast<uint64_t*>(buf);
  uint32_t* d_block = reinterpret_cast<uint32_t*>(buf + (size_t)nb * 8);
  uint32_t* d_voxel = d_block + n;
  float* d_sdf = reinterpret_cast<float*>(d_voxel + n);
  float* d_w = d_sdf + n;
  uint32_t* d_col = reinterpret_cast<uint32_t*>(d_w + n);
  uint32_t* d_bad = d_col + n;
  VBX_CUDA(c, cudaMemcpyAsync(d_bkeys, bkeys.data(), (size_t)nb * 8, cudaMemcpyHostToDevice, s));
  VBX_CUDA(c, cudaMemcpyAsync(d_block, rec_block, n4, cudaMemcpyHostToDevice, s));
  VBX_CUDA(c, cudaMemcpyAsync(d_voxel, rec_voxel, n4, cudaMemcpyHostToDevice, s));
  VBX_CUDA(c, cudaMemcpyAsync(d_sdf, sdf, n4, cudaMemcpyHostToDevice, s));
  VBX_CUDA(c, cudaMemcpyAsync(d_w, w, n4, cudaMemcpyHostToDevice, s));
  VBX_CUDA(c, cudaMemcpyAsync(d_col, rgba, n4, cudaMemcpyHostToDevice, s));
  VBX_CUDA(c, cudaMemsetAsync(d_bad, 0, 4, s));
  ScanParams P;
  const float q[4] = {1.f, 0.f, 0.f, 0.f}, t[3] = {0.f, 0.f, 0.f};
  fill_params(c, VBX_SIMPLE, q, t, 0, 0, P);
  ScanArgs a;
  fill_args(c, P, nullptr, nullptr, &a);
  a.count_paths = 1u;
  if (int rc = upload_args(c, x, a)) return rc;
  VBX_CUDA(c, cudaMemsetAsync(S.d_state, 0, sizeof(ScanState), s));
  VBX_CUDA(c, cudaMemsetAsync(S.sort_plan1, 0, sizeof(SortPlan), s));  // (sort_and_apply expects it cleared)
  const uint64_t m = std::max<uint64_t>(n, nb);
  if (m) {
    k_debug_apply_setup<<<grid_for(m, 256), 256, 0, s>>>(scan_tables(c, S), d_bkeys, nb, d_block, d_voxel, n, c->L,
                                                         S.ckeys[0], S.cvals[0], S.d_state, d_bad);
  }
  uint32_t bad = 0;
  VBX_CUDA(c, cudaMemcpyAsync(&bad, d_bad, 4, cudaMemcpyDeviceToHost, s));
  VBX_CUDA(c, cudaStreamSynchronize(s));
  if (bad) return fail(c, VBX_E_INVALID, "debug_apply: a block is not in the TSDF layer");
  Tally tally{c, s, x.marks};
  const GivenRecords given{d_sdf, d_w, d_col};
  if (int rc = sort_and_apply(c, x, tally, nullptr, &given)) return rc;
  VBX_CUDA(c, cudaMemcpyAsync(S.h_state, S.d_state, sizeof(ScanState), cudaMemcpyDeviceToHost, s));
  VBX_CUDA(c, cudaStreamSynchronize(s));
  VBX_CUDA(c, cudaGetLastError());
  if (int rc = check_state_errors(c, *S.h_state)) return rc;
  report_apply_paths(c, *S.h_state);
  if (paths) std::memcpy(paths, c->apply_paths, sizeof(c->apply_paths));
  return VBX_OK;
}

// exclusive prefix sum of n host uint32 through the engine's scan kernel
int debug_scan(vbx_ctx* c, const uint32_t* in, uint32_t n, uint32_t* out) {
  cudaStream_t s = c->stream;
  const vbx_ctx::ScratchSet& S = c->set[0];
  uint32_t* status = c->lane[0].scan_status;
  if (n > c->max_points + 1) return fail(c, VBX_E_CAPACITY, "debug_scan: n > max_points_per_scan + 1");
  VBX_CUDA(c, cudaMemcpyAsync(S.cnt, in, (size_t)n * 4, cudaMemcpyHostToDevice, s));
  const uint32_t tiles = (n + kScanTile - 1) / kScanTile;
  VBX_CUDA(c, cudaMemsetAsync(status, 0, (size_t)(tiles + 1) * sizeof(uint32_t), s));
  if (n) {
    k_exclusive_scan<<<std::min<uint32_t>(tiles, c->grid_sms * 4), kSortThreads, 0, s>>>(S.cnt, nullptr, nullptr, S.off, nullptr, n,
                                                                               status + 1, status, nullptr,
                                                                               nullptr, nullptr, 0ull, 0u);
  }
  VBX_CUDA(c, cudaMemcpyAsync(out, S.off, (size_t)n * 4, cudaMemcpyDeviceToHost, s));
  VBX_CUDA(c, cudaStreamSynchronize(s));
  VBX_CUDA(c, cudaGetLastError());
  return VBX_OK;
}

}  // namespace vbx
