// Internal declarations shared by the engine's translation units (not installed;
// the public boundary is include/voxblox_b200.h).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <string>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "../../include/voxblox_b200.h"
#include "vbx_math.cuh"
#include "vbx_order.cuh"

namespace vbx {
struct SortPlan;
struct ScanArgs;  // a scan's per-call kernel arguments in device memory (vbx_tsdf.cu)
}

namespace vbx {

constexpr uint64_t kEmptyKey = ~0ull;
constexpr uint64_t kInvalidPointKey = ~0ull;
constexpr int kCoordBias = 1 << 20;  // block / voxel coordinates are packed 21 bits per axis
// The Fast integrator's approximate sets, laid out as ApproxHashSet<20, 10000> (utils/approx_hash_array.h:75-179):
// hash h lives in slot (h & kApproxSetMask) + offset; the offset moves on by one per reset, and the set is
// cleared when it reaches kApproxSetResets.
constexpr uint32_t kApproxSetMask = (1u << 20) - 1u, kApproxSetResets = 10000u;
constexpr size_t kApproxSetWords = (1u << 20) + kApproxSetResets;
// Internal bits of the per-slot flag bytes (never reported through the C-ABI):
//   slot_updated bit 7: the slot holds an ESDF block only -- the TSDF layer has no block at this
//     index (blocks allocated by EsdfIntegrator::addNewRobotPosition or uploaded into the ESDF layer).
//     Any TSDF touch writes the byte to 7 (Block::updated().set()), which turns the slot into a TSDF block
//     that starts from zeroed voxels, exactly like a freshly allocated one.
//   slot_esdf_updated bit 7: member of EsdfIntegrator::updated_blocks_ (esdf_integrator.h:172-175).
constexpr uint8_t kEngineBit = 0x80;  // bit 7 of either byte: no caller selects, clears or is told about it
constexpr uint8_t kSlotNoTsdf = kEngineBit, kEsdfPending = kEngineBit;
//   bit 3 of both flag bytes (VBX_UPDATED_MIRROR): the block changed since a vbx_mirror_updated /
//     vbx_serialize_updated call last cleared this bit -- the engine's own dirty mark for the incremental
//     host mirror, independent of the three Block::updated() bits (which their consumers clear).
constexpr uint8_t kTouchedBits = 0x0F;  // what a TSDF update writes: Block::updated().set() + the mirror mark
constexpr uint8_t kReportedBits = 0x07;  // Block::updated() (kMap | kMesh | kEsdf): the bits the C-ABI reports
constexpr uint8_t kMirrorBits = 0x7F;    // what a mirror call may select on or clear: all but kEngineBit

struct EsdfVoxel {  // core/voxel.h:18-37
  float distance;
  uint8_t observed, hallucinated, in_queue, fixed;
  int32_t parent[3];
};
static_assert(sizeof(TsdfVoxel) == 12 && sizeof(EsdfVoxel) == 20, "voxel layouts");

// Error bits raised on the device (ScanState::error)
enum : uint32_t {
  kErrPoolFull = 1u,        // more blocks than max_blocks
  kErrHashFull = 2u,        // block hash probe wrapped around
  kErrCoordRange = 4u,      // |voxel coordinate| >= 2^20 * vps
  kErrUpdatesFull = 8u,     // ray-voxel updates exceed max_updates_per_pass
  kFatalErrors = 15u,       // any of the above
  kSkipped = 32u,           // not an error: the scan was queued behind a scan that must be redone (vbx_capi.cu)
};

// The paths of k_apply, counted per call in ScanState::apply_paths (vbx_debug_apply_paths reports them).
// Each path claims the sequential updateTsdfVoxel result bit for bit; the counts show which of them a
// call exercised.
enum ApplyPath : int {
  kPathLongRun = 0,        // runs longer than kShortRun updates, one warp each
  kPathLongRested,         // ... of which the rest was skipped: the voxel rests at (+T, max_weight), every later record keeps
  kPathStepSaturated,      // 4 x 32-record steps decided in one go: weight already at max_weight
  kPathStepIntScan,        // ... integer weights below 2^24: a warp scan forms the weight chain
  kPathStepPrefix,         // ... an in-order prefix sum forms it
  kPathChunkSaturated,     // 32-record chunks decided fast: weight already at max_weight
  kPathChunkConst,         // ... unit weights on an integer weight below 2^22
  kPathChunkPrefix,        // ... an in-order prefix sum
  kPathChunkSequential,    // ... the clamped weight chain, one record after the other
  kPathChunkExact,         // 32-record chunks applied with the exact per-record update
  kPathShortRun,           // runs of at most kShortRun updates, one thread each
  kPathShortCrossed,       // ... that continue past the end of their shared-memory tile
  kApplyPaths
};

// Device-resident per-call state; the host reads it back through pinned memory.
struct ScanState {
  uint32_t n_new;            // hash entries created by this call
  uint32_t n_touched;        // distinct blocks touched by this call
  uint32_t error;
  uint32_t n_rays;           // normal rays / bundles cast
  uint32_t n_clear_rays;     // clearing rays / bundles cast
  uint32_t n_valid_points;
  uint32_t n_voxels;         // distinct voxels updated (U)
  uint32_t n_blocks;         // pool slots in use after the call
  unsigned long long total_updates;  // K the back half runs on (0 when the call failed / is redone)
  unsigned long long total_found;    // K as counted
  uint32_t n_ray_list;       // bundle heads (Merged)
  uint32_t n_long;           // voxel runs longer than kShortRun updates (k_apply_prep's long-run list)
  uint32_t long_ticket;      // k_apply: long runs handed out
  uint32_t n_refold;         // bundles folded a second time with IEEE division (diagnostic)
  uint32_t refold_members;   // ... and the points they hold
  uint32_t tile_ticket;      // k_apply: record tiles of the short runs handed out
  uint32_t apply_paths[12];  // k_apply: how often each arithmetic path ran, summed over the call (ApplyPath)
  // Merged: bounding box of the valid points' voxels, both ends atomicMax'ed (so that an all-zero
  // block means "no valid point"): kb_max = v + 2^30, kb_min = 0xffffffff - (v + 2^30); the bundle
  // keys are packed relative to it (vbx_tsdf.cu, KeyLayout)
  uint32_t kb_max[3];
  uint32_t kb_min[3];
  uint32_t key_bits;         // bits a bundle key uses
  uint32_t n_big;            // Merged: bundles of at least kBigBundle members (folded first)
  uint32_t merge_ticket;     // Merged: work hand-out counter of k_merge
  uint32_t n_touch_ids;      // touched-block ids handed out: one per block the call touches (vbx_hash.cuh)
  uint32_t rec_key_bits;     // bits an update-record key uses: voxel-in-block bits + bits of the touched ids
  uint32_t ids_resolved;     // local block ids k_assign has resolved so far in this call (all passes)
};
static_assert(sizeof(ScanState) == 168, "the status block the host reads back is 168 bytes");
static_assert(offsetof(ScanState, total_updates) % 8 == 0 && offsetof(ScanState, total_found) % 8 == 0,
              "64-bit counters stay 8-byte aligned");
static_assert(sizeof(ScanState::apply_paths) / 4 == kApplyPaths, "one word per apply path");

// Error bits raised on the device (EsdfState::error)
enum : uint32_t {
  kEsdfErrQueueFull = 1u,    // a wavefront / raise / seed queue append past its capacity
  kEsdfErrParentRange = 2u,  // full-Euclidean mode: a parent vector component outside [-512, 511]
};

// The ESDF's per-call status block (vbx_esdf.cu), device-resident; the host reads it back through pinned memory.
struct EsdfState {
  uint32_t error;
  uint32_t counts[7];      // [0] blocks listed, [1..6] the VLOG counters (vbx_esdf_get_counters)
  // The queue kernels rotate through three counters per queue: sweep k reads [k % 3], appends to
  // [(k + 1) % 3] and zeroes [(k + 2) % 3], so a sweep needs one grid-wide barrier.
  uint32_t frontier_n[3];  // the open queue (wavefront)
  uint32_t raise_n[3];     // the raise queue
  uint32_t seed_n;         // new free voxels waiting for updateVoxelFromNeighbors
  uint32_t lowered_n;      // voxels lowered by the wavefront
};

// The GPU-resident block hash + voxel pools (the device mirror of Layer<T>::block_map_,
// core/layer.h:30-32,292).
struct Tables {
  uint64_t* hkeys;        // [hcap] packed block index, kEmptyKey when free
  int32_t* hslot;         // [hcap] pool slot
  uint32_t hmask;         // hcap - 1
  uint32_t max_blocks;
  uint32_t vox_per_block;
  uint32_t* new_list;     // [max_blocks] hash positions created by this call
  uint32_t* touched_list; // [touched_cap] touched id -> hash position (0xffffffff: unused id); hand-off set private
  uint32_t touched_cap;
  uint64_t* slot_key;     // [max_blocks] packed block index per pool slot
  uint8_t* slot_updated;  // [max_blocks] TSDF Block::updated() bits
  uint8_t* slot_esdf_updated;  // [max_blocks] ESDF Block::updated() bits
  uint8_t* slot_has_esdf;      // [max_blocks] 1 once the ESDF layer holds this block
  TsdfVoxel* tsdf;        // [max_blocks << 3L]
  EsdfVoxel* esdf;        // [max_blocks << 3L] (allocated by vbx_esdf_create)
};

// A scan's private block table (hand-off set private, beside touched_list).  The ray walk that writes the
// update records runs in the front half, beside other scans' map-touching stages, so it must not read the
// block hash: it gives the blocks it meets dense local ids here instead, and k_assign (walk stage, submission
// order) resolves each id against the hash, creating the blocks that are missing.  Uploads and robot-position
// spheres list their blocks in hand-off set 0's table the same way.  Open addressing keyed by pack3(block),
// value = local id + 1 (0: free).  The table is zeroed once when it is allocated; k_assign clears the
// positions a call used.
struct ScanBlocks {
  uint32_t* table;            // [mask + 1], a power of two >= 2 * cap
  unsigned long long* keys;   // [cap] local id -> packed block index
  uint32_t* pos;              // [cap] local id -> its table position
  uint32_t mask;
  uint32_t cap;               // = Tables::touched_cap
};

__host__ __device__ inline uint64_t pack3(int x, int y, int z) {
  return ((uint64_t)(uint32_t)(z + kCoordBias) << 42) | ((uint64_t)(uint32_t)(y + kCoordBias) << 21) |
         (uint64_t)(uint32_t)(x + kCoordBias);
}
__host__ __device__ inline void unpack3(uint64_t k, int* x, int* y, int* z) {
  *x = (int)(k & 0x1fffffu) - kCoordBias;
  *y = (int)((k >> 21) & 0x1fffffu) - kCoordBias;
  *z = (int)((k >> 42) & 0x1fffffu) - kCoordBias;
}
// block-ownership sharding: the rank that owns a block (2 x 2 x 2 brick pattern for 8 ranks)
__host__ __device__ inline int block_owner(int bx, int by, int bz, int world) {
  const int a = (bx + 2 * by + 4 * bz) % world;
  return a < 0 ? a + world : a;
}
__host__ __device__ inline uint32_t hash64(uint64_t k) {
  k ^= k >> 33;
  k *= 0xff51afd7ed558ccdULL;
  k ^= k >> 33;
  k *= 0xc4ceb9fe1a85ec53ULL;
  k ^= k >> 33;
  return (uint32_t)k;
}

}  // namespace vbx

struct vbx_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;      // main stream: synchronous calls, ESDF, block management, pipelined applies
  cudaStream_t stream_c = nullptr;    // host-to-device cloud copies of asynchronously submitted scans
  cudaStream_t stream_c2 = nullptr;   // ... alternating with this one
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  vbx_tsdf_config cfg;
  vbx_engine_options opt;
  float voxel_size = 0, voxel_size_inv = 0;
  int vps = 16, L = 4;         // voxels per side and log2
  uint32_t vox_per_block = 4096;
  uint32_t hcap = 0;
  unsigned int grid_sms = 132;  // persistent-kernel grids are multiples of this (the device's SM count, queried at create; VBX_GRID_SMS overrides: tuning aid)
  vbx::Tables tab;  // the map (touched_list is null: each hand-off set owns its own)
  // scratch
  uint32_t max_points = 0;
  uint64_t max_updates = 0;
  bool timeline = false;            // VBX_ASYNC_TIMELINE: the hand-off events carry timestamps
  cudaEvent_t timeline_ref = nullptr;
  uint32_t bundle_hint = 0;         // bundles (the larger of the two maps) of the most recent Merged scan whose counters reached the host
  uint64_t record_hint = 1u << 20;  // update records of the most recent scan whose count reached the host: sizes the record sort's grid
  uint32_t* order = nullptr;               // [max_points] "sorted" integration order
  uint32_t* order_inv = nullptr;           // [max_points] inverse of `order`
  vbx::RehashSchedule rehash{};            // libstdc++'s unordered_map growth schedule (vbx_create)
  size_t order_smem_bytes = 0;             // dynamic shared memory of k_bundle_order
  // tiles of the engine's own radix sorts (vbx_sort.cuh): [0] point keys, [1] update records
  uint32_t sort_tiles_cap[2] = {0, 0};
  // the Fast integrator's approximate sets, kApproxSetWords each, and their slot offset (init_fast_sets)
  unsigned long long* set_start = nullptr;
  unsigned long long* set_observed = nullptr;
  uint32_t set_offset = 0;
  int64_t fast_reset_counter = 0;  // calls since the last reset (the reference's is process-wide)
  uint32_t n_blocks = 0;              // pool slots in use (host copy, exact after a drain)
  uint32_t* d_nblocks = nullptr;      // [2] device copy, ping-pong: k_assign reads [nb_cur], writes [nb_cur ^ 1]
  int nb_cur = 0;
  // Asynchronous submission (vbx_tsdf_integrate_async): a scan passes through four stages -- front half
  // (keys, bundle sort, bundle fold, offsets, the ray walk that writes the update records; does not touch
  // the map) on one of kLanes
  // front lanes, block creation, record sort, apply -- so up to kSets scans are in flight, each owning one set
  // of hand-off buffers.  Map-touching stages run in submission order.  Each scan is one launch of a CUDA
  // graph per (hand-off set, front lane, kind), captured before its first use.  The sets and lanes are the
  // only owners of per-scan scratch: set 0 / lane 0 (allocated by vbx_create) are the buffers the synchronous
  // calls use, the others are allocated on the first asynchronous submission (alloc_set / alloc_lane).
  static constexpr int kSets = 16, kLanes = 8;  // upper bounds
  int sets_in_use = 10, lanes_in_use = 6;  // (tuning aids: VBX_ASYNC_SETS, VBX_ASYNC_LANES)
  enum { kGraphSimple, kGraphMerged, kGraphVariants };
  struct ScanGraph {
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t exec = nullptr;
    uint64_t launches = 0;                  // kernel nodes
    cudaGraphNode_t point_sort = nullptr;   // grid sized by the scan's point count
    unsigned int point_grid = 0;
    cudaGraphNode_t record_sort = nullptr;  // grid sized by record_hint
    unsigned int record_grid = 0;
    cudaGraphNode_t order = nullptr;        // k_bundle_order: form and shared memory follow bundle_hint
    unsigned int order_grid = 0;
    size_t order_smem = 0;
  };
  struct ScratchSet {
    float4* ray_p = nullptr;         // [max_points] point_G.xyz, flags (bit 0: clearing ray)
    float4* ray_a = nullptr;         // [max_points] point_G - origin, |point_G - origin|
    uint2* ray_c = nullptr;          // [max_points] colour, weight bits
    uint32_t* ray_list = nullptr;    // [max_points] Merged: ray slot (rank in the reference's bundle order) -> head
    uint32_t* head_list = nullptr;   // bundle id -> sorted position of its head (read again by the ray walk)
    uint32_t* touched_list = nullptr;  // touched id -> hash position (written by k_assign, read by the apply)
    vbx::ScanBlocks blocks{};          // local block ids of the ray walk (written by the front half, read by k_assign)
    uint32_t* cnt = nullptr;         // [max_points + 1]
    uint32_t* off = nullptr;         // [max_points + 1]
    vbx::ScanState* d_state = nullptr;
    vbx::ScanState* h_state = nullptr;  // page-locked
    vbx::ScanArgs* d_args = nullptr;
    vbx::ScanArgs* h_args = nullptr;  // page-locked: the graph's first node uploads it
    float* d_xyz = nullptr;          // a host cloud's device copy
    uint8_t* d_rgba = nullptr;
    uint64_t* pkeys0 = nullptr;  // sorted bundle keys (read again by the ray walk)
    uint32_t* ckeys[2] = {nullptr, nullptr};  // update records (written by the walk, read by apply)
    uint32_t* cvals[2] = {nullptr, nullptr};
    // [max_updates / 32 + 1] each: the long voxel runs' first record and end, and per sorted record a bit
    // "the update keeps (+T, max_weight)" (k_apply_prep -> k_apply)
    unsigned long long* long_list = nullptr;
    unsigned long long* long_end = nullptr;
    uint32_t* keep_bits = nullptr;
    vbx::SortPlan* sort_plan1 = nullptr;  // the record sort's plan and status words
    uint32_t* sort_status1 = nullptr;
    cudaEvent_t copy_done = nullptr, walked = nullptr, sorted = nullptr, applied = nullptr, back_done = nullptr;
    cudaEvent_t front_start = nullptr, front_done = nullptr;  // only with VBX_ASYNC_TIMELINE (vbx_debug_async_timeline)
    cudaStream_t stream = nullptr;  // the scan's graph is launched here (one stream per set: graphs in one stream run one after the other)
    ScanGraph graph[kLanes][kGraphVariants];
    bool in_flight = false;
    int kind = 0;
    uint64_t launches = 0;
    // what the scan was submitted with, kept until it is known to be in the map: a scan that cannot
    // be applied asynchronously is redone from here (recover_async)
    uint64_t seq = 0;
    bool redo = false;
    float q[4] = {1, 0, 0, 0}, t[3] = {0, 0, 0};
    uint64_t n = 0;
    int freespace = 0;
    const float* in_xyz = nullptr;
    const uint8_t* in_rgba = nullptr;
  } set[kSets];
  struct FrontLane {  // scratch private to one front-half stream
    cudaStream_t stream = nullptr;
    uint64_t* pkeys1 = nullptr;  // the point sort's second key buffer
    uint32_t* pvals[2] = {nullptr, nullptr};
    vbx::SortPlan* sort_plan0 = nullptr;  // the point sort's plan and status words
    uint32_t* sort_status0 = nullptr;
    uint32_t* scan_status = nullptr;  // the offset scan's tile status words
    uint32_t* big_list = nullptr;     // [max_points / 256 + 1] ids of the big bundles
    uint32_t* first_bits = nullptr;   // [2][max_points / 32 + 1] first-occurrence bitmaps
    vbx::OrderScratch order_scratch{};  // k_bundle_order's global tables
    cudaStream_t side = nullptr;      // k_bundle_order runs here, beside k_merge
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    cudaEvent_t done = nullptr;  // the lane's last front half
  } lane[kLanes];
  bool async_ready = false;
  int prio_lo = 0, prio_hi = 0;  // stream priority range of the device
  // the streams a scan's graph is captured from (besides the front lane's and the main stream)
  cudaStream_t stream_e = nullptr;  // block creation: k_back_begin, k_assign
  cudaStream_t stream_s = nullptr;  // record sort + apply preparation
  cudaEvent_t cap_ev[8] = {};  // capture-internal edges (fork, front -> walk, walk -> sort, sort -> apply, joins)
  uint64_t async_seq = 0;
  uint32_t* d_hold = nullptr;           // device flag: a queued scan must be redone, later scans skip their back half
  uint64_t async_redone = 0;            // scans redone synchronously since vbx_create (reporting)
  bool hash_dirty = false;              // an asynchronous scan ran out of pool slots: rebuild the hash at the next drain
  int deferred_rc = 0;
  std::string deferred_msg;
  // incremental device -> host mirror (vbx_mirror_updated): gather staging on both sides
  void* mirror_dev = nullptr;
  void* mirror_host = nullptr;  // page-locked
  uint32_t* mirror_slots = nullptr;
  size_t mirror_cap_bytes = 0, mirror_cap_slots = 0;
  // device-to-device block transfer (vbx_gather_updated_device): the gathered blocks' slots, device only
  uint32_t* xfer_slots = nullptr;
  size_t xfer_cap_slots = 0;
  // host mirror of slot_key (refreshed lazily)
  std::vector<uint64_t> host_slot_key;
  std::unordered_map<uint64_t, int32_t> host_key2slot;
  // Block::has_data_ (core/block.h:206): never set by the integrators, carried by BlockProto; blocks loaded
  // from a .vxblx file with has_data = true are remembered per layer so that a re-save writes the flag back
  std::unordered_set<uint64_t> has_data_keys[2];
  // ESDF
  bool has_esdf = false;
  vbx_esdf_config ecfg;
  uint32_t* frontier[2] = {nullptr, nullptr};
  uint32_t* raise_q[2] = {nullptr, nullptr};
  uint64_t frontier_cap = 0;
  uint32_t* esdf_block_list = nullptr;
  uint32_t* esdf_seed_list = nullptr;
  float* esdf_seed_val = nullptr;
  uint32_t* esdf_touched = nullptr;
  // full-Euclidean mode only (allocated by its first update): every voxel's distance and parent as one 64-bit
  // word, so that the wavefront lowers both in a single atomicMin (vbx_esdf.cu, fe_pack)
  unsigned long long* esdf_fe = nullptr;
  vbx::EsdfState* esdf_d_state = nullptr;
  vbx::EsdfState* esdf_h_state = nullptr;  // page-locked
  int esdf_sms = 0, esdf_ctas_wide = 1;
  uint32_t esdf_pending_raise = 0, esdf_pending_open = 0;  // raise_ / open_ entries queued by addNewRobotPosition
  bool maybe_esdf_only = false;                            // some slot may carry kSlotNoTsdf
  // mesher (vbx_mesh.cu): the result of the last vbx_mesh_generate stays on the device until the next one
  uint32_t* mesh_slots = nullptr;
  uint16_t* mesh_cube_off = nullptr;
  uint32_t* mesh_block_nv = nullptr;
  unsigned long long* mesh_first = nullptr;
  float* mesh_vertices = nullptr;
  float* mesh_normals = nullptr;
  uint32_t* mesh_colors = nullptr;
  uint64_t mesh_cap_blocks = 0, mesh_cap_vertices = 0, mesh_launches = 0;
  std::vector<int32_t> mesh_idx;
  std::vector<uint64_t> mesh_first_host = std::vector<uint64_t>(1, 0);
  bool mesh_use_color = false;
  // ICP (vbx_icp.cu): shuffled point order (host page-locked + device), host-cloud staging, result block
  uint32_t* icp_perm_dev = nullptr;
  uint32_t* icp_perm_host = nullptr;
  float* icp_points_dev = nullptr;
  float* icp_out_dev = nullptr;
  float* icp_out_host = nullptr;
  uint64_t icp_cap = 0;
  // reporting
  uint64_t counters[16] = {0};
  uint64_t apply_paths[16] = {0};  // ScanState::apply_paths of the last call whose status reached the host
  bool count_apply_paths = false;  // k_apply counts its paths (vbx_debug_count_apply_paths; vbx_debug_apply always does)
  bool serial_fast = false;        // Fast calls walk their rays on one thread, in rank order (vbx_debug_serial_fast)
  uint64_t async_wait_ns = 0, async_submit_ns = 0;  // host time of vbx_tsdf_integrate_async: waiting for a hand-off set / enqueueing
  uint64_t esdf_counters[16] = {0};
  float last_ms = 0.f;
  uint64_t launches = 0;
  cudaEvent_t tev0 = nullptr, tev1 = nullptr;  // vbx_timer_*
  bool profiling = false;
  cudaEvent_t sev[20] = {nullptr};             // stage boundaries
  double stage_ms[16] = {0};
  uint64_t stage_calls[16] = {0};
  std::string err;
};

namespace vbx {
int fail(vbx_ctx* c, int code, const std::string& msg);
int cuda_fail(vbx_ctx* c, cudaError_t e, const char* what);
int refresh_host_mirror(vbx_ctx* c);

// One layer's view of the pool slots (read_layer_slots): every host caller that asks which slots hold a
// block of the layer, with which flag bits, reads it here.  The TSDF and the ESDF layer share pool slots; a
// slot belongs to the TSDF layer unless its slot_updated carries kSlotNoTsdf, and to the ESDF layer when
// slot_has_esdf is set (a slot may hold both, either or, after a batch ESDF update wiped an ESDF-only
// block, neither).  Valid until the next call that changes the pool.
struct LayerSlots {
  struct Entry {
    int x, y, z;
    uint32_t slot;
  };
  const vbx_ctx* c = nullptr;
  std::vector<uint8_t> flags;   // [n_blocks] the layer's raw flag byte (slot_updated / slot_esdf_updated)
  std::vector<uint8_t> member;  // [n_blocks] 1: the layer holds a block in this slot
  // The member slots with (flags & select_bits & mask) != 0, or every member when mask == 0, by (x, y, z)
  std::vector<Entry> sorted(uint8_t select_bits, int mask) const;
  // slots_out[i] = the slot of block idx3[i], or -1 when the layer holds no block there
  void find(const int32_t* idx3, uint64_t m, int32_t* slots_out) const;
};
// The host mirror of slot_key brought up to date, then the layer's flag bytes (and slot_has_esdf) in one read
int read_layer_slots(vbx_ctx* c, int layer, LayerSlots* view);
// flags[s] &= keep over the slots in use, on the main stream
int keep_flag_bits(vbx_ctx* c, uint8_t* flags, uint8_t keep);
int mirror_updated(vbx_ctx* c, int layer, int updated_mask, int clear_mask, int32_t* idx3, void* voxels,
                   uint8_t* updated_bits, uint64_t cap, uint64_t* n, int serialized);
int gather_updated_device(vbx_ctx* c, int layer, int updated_mask, int clear_mask, int owned_only, int32_t* d_idx3,
                          void* d_voxels, uint64_t cap, uint64_t* n);
int upload_blocks_device(vbx_ctx* c, int layer, const int32_t* d_idx3, uint64_t m, const void* d_voxels,
                         uint8_t updated_bits);
int esdf_destroy(vbx_ctx* c);
void mesh_destroy(vbx_ctx* c);
void icp_destroy(vbx_ctx* c);
int icp_debug_solve(vbx_ctx* c, uint32_t n, int refine_roll_pitch, const float* h, const float* m, const float* q,
                    const float* w, float* r_out, int32_t* valid_out, float* q_out, float* log_out, float* exp_out);
int icp_run(vbx_ctx* c, const vbx_icp_config* cfg, const float* points, int on_device, uint64_t n, const float q[4],
            const float t[3], uint32_t seed, float out_q[4], float out_t[3], uint64_t* num_updates);
int mesh_generate(vbx_ctx* c, const vbx_mesh_config* cfg, int only_updated, int clear_flag, uint64_t* n_blocks_out,
                  uint64_t* n_vertices_out);
int mesh_download(vbx_ctx* c, int32_t* idx3, uint64_t* first_vertex, float* vertices, float* normals, uint8_t* colors);
int esdf_add_robot_position(vbx_ctx* c, const float p[3]);
int esdf_clear_state(vbx_ctx* c);
int ensure_async(vbx_ctx* c);          // allocate the extra hand-off sets / front lanes
int drain_async(vbx_ctx* c);           // wait for every asynchronously submitted scan, collect its results
int set_n_blocks(vbx_ctx* c, uint32_t n);
int init_bundle_order(vbx_ctx* c);     // rehash schedule + shared-memory opt-in of k_bundle_order
int rebuild_hash(vbx_ctx* c);          // block hash rebuilt from slot_key (after removals / a pool overflow)
void harvest_async(vbx_ctx* c, vbx_ctx::ScratchSet& S);  // collect a finished asynchronous scan's results
int alloc_scan_args(vbx_ctx* c, vbx_ctx::ScratchSet& S);  // the set's argument block, device + page-locked host

// Where a scan's work is enqueued (vbx_tsdf.cu): its hand-off set and front lane, the stream of the stage
// being enqueued, the unit of the persistent kernels' grids and whether stage marks are recorded.
struct ScanRoute {
  vbx_ctx::ScratchSet& S;
  vbx_ctx::FrontLane& F;
  cudaStream_t s;
  unsigned int sms;  // an SM count: the whole GPU, or a share of it in the pipelined graphs
  bool marks;        // vbx_set_stage_profiling
};
// The synchronous calls: hand-off set 0 and front lane 0 on the main stream, grids for the whole GPU.
inline ScanRoute sync_route(vbx_ctx* c) { return {c->set[0], c->lane[0], c->stream, c->grid_sms, c->profiling}; }
int init_fast_sets(vbx_ctx* c, cudaStream_t s);  // both sets cleared and word 0 marked, as a fresh ApproxHashSet
// The blocks an upload or a robot-position sphere listed in hand-off set 0's table (scan_block_id), created by
// k_assign as a scan's are, on the main stream: blocks that exist keep their updated bits, a new slot's start
// at new_bits, and the block count moves as after a scan.
int create_listed_blocks(vbx_ctx* c, uint8_t new_bits);
// A finished call's status block: VBX_E_CAPACITY for a device error; a full pool also takes h.n_blocks and
// rebuilds the hash (the call's surplus entries have no slot)
int check_state_errors(vbx_ctx* c, const ScanState& h);
int integrate_device(vbx_ctx* c, const ScanRoute& x, int kind, const float q[4], const float t[3], const float* d_xyz,
                     const uint8_t* d_rgba, uint64_t n, int freespace);

// The slots of vbx_get_stage_ms, in the order of api.py's STAGE_NAMES (the C-ABI's order)
enum Stage : int {
  kStagePointKeys, kStagePointSort, kStageRayCount, kStageScan, kStageAssign, kStageRayEmit, kStageUpdateSort,
  kStageApply, kStageBundleMerge, kStageEsdfPropagate, kStageEsdfRaise, kStageEsdfLower, kStageBundleOrder
};

// One call's bookkeeping: the kernels it launched, counted where each is launched, and with stage profiling
// on an event at the end of each stage on stream s (off while a graph is captured: stage events would
// serialise the streams).
struct Tally {
  vbx_ctx* c;
  cudaStream_t s;
  bool on;
  uint64_t launches = 0;
  int n = 0;
  Stage stage[19];
  void begin() {
    if (on) cudaEventRecord(c->sev[0], s);
  }
  void mark(Stage just_finished) {
    if (on && n < 19) {
      cudaEventRecord(c->sev[n + 1], s);
      stage[n++] = just_finished;
    }
  }
  void collect() {
    for (int m = 0; m < n; ++m) {
      float ms = 0.f;
      if (cudaEventElapsedTime(&ms, c->sev[m], c->sev[m + 1]) == cudaSuccess) {
        c->stage_ms[stage[m]] += ms;
        c->stage_calls[stage[m]] += 1;
      }
    }
  }
};

// The slots of vbx_get_counters (include/voxblox_b200.h)
enum Counter : int {
  kCntRays, kCntClearRays, kCntUpdates, kCntVoxels, kCntBlocksTouched, kCntBlocksAllocated, kCntValidPoints,
  kCntLaunches, kCntLaunchesTotal, kCntRefoldedBundles, kCntRefoldedPoints, kCntPasses, kCntBundleKeyBits,
  kCntAsyncRedone, kCntAsyncWaitNs, kCntAsyncSubmitNs
};
// A finished TSDF call's status block -> its counters, the grid hints of later scans and the apply-path counts
void report_scan(vbx_ctx* c, const ScanState& h, int kind, uint64_t launches, uint64_t passes, uint64_t blocks_allocated);
}  // namespace vbx

#define VBX_CUDA(c, expr)                                          \
  do {                                                             \
    cudaError_t _e = (expr);                                       \
    if (_e != cudaSuccess) return vbx::cuda_fail((c), _e, #expr);  \
  } while (0)
