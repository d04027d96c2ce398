// The C-ABI of include/voxblox_b200.h: context life cycle, the host<->device block
// mirror (Layer<T> on the host side stays the reference's own container; see
// INTEGRATION.md) and the entry points that dispatch into the device pipelines.
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "vbx_engine.h"
#include "vbx_sort.cuh"

namespace vbx {

int debug_sort(vbx_ctx* c, const void* keys, int key_bytes, uint32_t n, int key_bits, void* keys_out,
               uint32_t* vals_out);
int debug_scan(vbx_ctx* c, const uint32_t* in, uint32_t n, uint32_t* out);
int debug_bundle_order(vbx_ctx* c, const uint32_t* hashes, uint32_t n, int force_global, uint32_t* out);
int debug_apply(vbx_ctx* c, const int32_t* idx3, uint32_t nb, uint64_t n, const uint32_t* rec_block,
                const uint32_t* rec_voxel, const float* sdf, const float* w, const uint8_t* rgba, uint64_t paths[16]);
int upload_blocks(vbx_ctx* c, int layer, const int32_t* idx3, uint64_t m, const void* voxels,
                  const uint8_t* updated_bits, int serialized);
int remove_blocks(vbx_ctx* c, int layer, const int32_t* idx3, uint64_t m);
int clear_layer(vbx_ctx* c, int layer);
int integrate_async(vbx_ctx* c, const ScanRoute& sync, int kind, const float q[4], const float t[3], const float* xyz,
                    const uint8_t* rgba, uint64_t n, int freespace, int on_device);
int esdf_create(vbx_ctx* c, const vbx_esdf_config* cfg);
int esdf_update(vbx_ctx* c, int batch, int clear_updated_flag);
int esdf_update_blocks(vbx_ctx* c, const int32_t* idx3, uint64_t m, int incremental);
int esdf_add_robot_position(vbx_ctx* c, const float p[3]);
int esdf_clear_state(vbx_ctx* c);

int fail(vbx_ctx* c, int code, const std::string& msg) {
  if (c) c->err = msg;
  return code;
}
int cuda_fail(vbx_ctx* c, cudaError_t e, const char* what) {
  if (c) c->err = std::string("CUDA error: ") + cudaGetErrorString(e) + " in " + what;
  return VBX_E_CUDA;
}

// Bring the host copy of slot -> block index up to date (new blocks are appended to
// slot_key by k_assign; removal rebuilds it).
int refresh_host_mirror(vbx_ctx* c) {
  const size_t have = c->host_slot_key.size();
  if (have < c->n_blocks) {
    c->host_slot_key.resize(c->n_blocks);
    VBX_CUDA(c, cudaMemcpyAsync(c->host_slot_key.data() + have, c->tab.slot_key + have,
                                (c->n_blocks - have) * sizeof(uint64_t), cudaMemcpyDeviceToHost, c->stream));
    VBX_CUDA(c, cudaStreamSynchronize(c->stream));
    for (size_t s = have; s < c->n_blocks; ++s) c->host_key2slot[c->host_slot_key[s]] = (int32_t)s;
  }
  return VBX_OK;
}

int set_n_blocks(vbx_ctx* c, uint32_t n) {
  c->n_blocks = n;
  VBX_CUDA(c, cudaMemcpyAsync(c->d_nblocks + c->nb_cur, &c->n_blocks, sizeof(uint32_t), cudaMemcpyHostToDevice,
                              c->stream));
  VBX_CUDA(c, cudaStreamSynchronize(c->stream));
  return VBX_OK;
}

// Collect a finished asynchronous scan: its counters, the block count, and any error it raised
// (reported by the next call that can return one).
void harvest_async(vbx_ctx* c, vbx_ctx::ScratchSet& S) {
  S.in_flight = false;
  const ScanState& h = *S.h_state;
  c->n_blocks = std::max(c->n_blocks, h.n_blocks);
  report_scan(c, h, S.kind, S.launches, 1, h.n_new);
  const uint32_t fatal = h.error & kFatalErrors & ~kErrUpdatesFull;
  if (!fatal && (h.error & (kErrUpdatesFull | kSkipped))) {
    // more update records than one pass holds (or queued behind such a scan): nothing was applied;
    // recover_async redoes it synchronously, in passes, in submission order
    S.redo = true;
    return;
  }
  if (fatal & kErrPoolFull) c->pipe.hash_dirty = true;  // surplus hash entries without a pool slot
  if (fatal && !c->pipe.deferred_rc) {
    c->pipe.deferred_rc = VBX_E_CAPACITY;
    c->pipe.deferred_msg = "an asynchronously submitted scan failed on the device (error bits " + std::to_string(h.error) +
                           (fatal & kErrPoolFull ? ": block pool full, raise vbx_engine_options.max_blocks" : "") + ")";
  }
}

// Every queued scan has been waited for.  Scans that could not be applied asynchronously (and the
// scans queued behind them, which skipped their back halves) are redone synchronously from their
// retained inputs, in submission order -- no scan is lost and the update order is the callers'.  The redo
// runs on hand-off set 0's scratch and only reads set k's input cloud.
static int recover_async(vbx_ctx* c) {
  if (c->pipe.hash_dirty) {
    c->pipe.hash_dirty = false;
    if (int rc = rebuild_hash(c)) return rc;
  }
  std::vector<vbx_ctx::ScratchSet*> todo;
  for (int k = 0; k < vbx_ctx::kSets; ++k) {
    if (c->set[k].redo) todo.push_back(&c->set[k]);
  }
  if (todo.empty()) return VBX_OK;
  std::sort(todo.begin(), todo.end(), [](const vbx_ctx::ScratchSet* a, const vbx_ctx::ScratchSet* b) { return a->seq < b->seq; });
  VBX_CUDA(c, cudaMemsetAsync(c->pipe.d_hold, 0, sizeof(uint32_t), c->stream));
  int first_rc = VBX_OK;
  std::string first_msg;
  for (vbx_ctx::ScratchSet* S : todo) {
    S->redo = false;
    const int rc = integrate_device(c, sync_route(c), S->kind, S->q, S->t, S->in_xyz, S->in_rgba, S->n, S->freespace);
    c->pipe.redone += 1;
    if (rc != VBX_OK && first_rc == VBX_OK) {
      first_rc = rc;
      first_msg = c->err;
    }
  }
  if (first_rc != VBX_OK) c->err = first_msg;
  return first_rc;
}

int drain_async(vbx_ctx* c) {
  for (int k = 0; k < c->pipe.sets_in_use; ++k) {
    vbx_ctx::ScratchSet& S = c->set[(c->pipe.seq + k) % c->pipe.sets_in_use];  // oldest submission first
    if (!S.in_flight) continue;
    VBX_CUDA(c, cudaEventSynchronize(S.back_done));
    harvest_async(c, S);
  }
  if (int rc = recover_async(c)) {
    if (!c->pipe.deferred_rc) return rc;
  }
  if (c->pipe.deferred_rc) {
    const int rc = c->pipe.deferred_rc;
    c->err = c->pipe.deferred_msg;
    c->pipe.deferred_rc = 0;
    return rc;
  }
  return VBX_OK;
}

// Everything a hand-off set owns except the pipeline's streams and events (ensure_async).  Its private block
// table is zeroed here, once; afterwards every call clears the positions it used.
static int alloc_set(vbx_ctx* c, Holdings& h, vbx_ctx::ScratchSet& S) {
  const size_t np = c->max_points, nu = c->max_updates;
  VBX_CUDA(c, h.dev(&S.ray_p, np));
  VBX_CUDA(c, h.dev(&S.ray_a, np));
  VBX_CUDA(c, h.dev(&S.ray_c, np));
  VBX_CUDA(c, h.dev(&S.ray_list, np));
  VBX_CUDA(c, h.dev(&S.head_list, np));
  VBX_CUDA(c, h.dev(&S.touched_list, c->tab.touched_cap));
  VBX_CUDA(c, h.dev(&S.cnt, np + 1));
  VBX_CUDA(c, h.dev(&S.off, np + 1));
  VBX_CUDA(c, h.dev(&S.d_state, 1));
  VBX_CUDA(c, h.host(&S.h_state, 1));
  if (int rc = alloc_scan_args(c, h, S)) return rc;
  VBX_CUDA(c, h.dev(&S.d_xyz, 3 * np));
  VBX_CUDA(c, h.dev(&S.d_rgba, 4 * np));
  VBX_CUDA(c, h.dev(&S.pkeys0, np));
  for (int i = 0; i < 2; ++i) {
    VBX_CUDA(c, h.dev(&S.ckeys[i], nu));
    VBX_CUDA(c, h.dev(&S.cvals[i], nu));
  }
  VBX_CUDA(c, h.dev(&S.long_list, nu / 32 + 1));
  VBX_CUDA(c, h.dev(&S.long_end, nu / 32 + 1));
  VBX_CUDA(c, h.dev(&S.keep_bits, nu / 32 + 1));
  VBX_CUDA(c, h.dev(&S.sort_plan1, 1));
  VBX_CUDA(c, h.dev(&S.sort_status1, (size_t)4 * c->sort_tiles_cap[1] * kRadix));
  ScanBlocks& b = S.blocks;
  b.cap = c->tab.touched_cap;
  uint32_t size = 1;
  while (size < 2 * b.cap) size <<= 1;
  b.mask = size - 1;
  VBX_CUDA(c, h.dev(&b.table, size));
  VBX_CUDA(c, h.dev(&b.keys, b.cap));
  VBX_CUDA(c, h.dev(&b.pos, b.cap));
  VBX_CUDA(c, cudaMemsetAsync(b.table, 0, (size_t)size * sizeof(uint32_t), c->stream));
  VBX_CUDA(c, cudaMemsetAsync(S.d_state, 0, sizeof(ScanState), c->stream));
  VBX_CUDA(c, cudaStreamSynchronize(c->stream));
  return VBX_OK;
}

// Everything a front lane owns except the pipeline's stream and event (ensure_async).
static int alloc_lane(vbx_ctx* c, Holdings& h, vbx_ctx::FrontLane& F) {
  const size_t np = c->max_points;
  VBX_CUDA(c, h.dev(&F.pkeys1, np));
  VBX_CUDA(c, h.dev(&F.pvals[0], np));
  VBX_CUDA(c, h.dev(&F.pvals[1], np));
  VBX_CUDA(c, h.dev(&F.sort_plan0, 1));
  VBX_CUDA(c, h.dev(&F.sort_status0, (size_t)8 * c->sort_tiles_cap[0] * kRadix));
  VBX_CUDA(c, h.dev(&F.scan_status, (np + 1) / kScanTile + 4));
  VBX_CUDA(c, h.dev(&F.big_list, np / 256 + 2));
  VBX_CUDA(c, h.dev(&F.first_bits, 2 * (np / 32 + 2)));
  VBX_CUDA(c, cudaMemsetAsync(F.first_bits, 0, 2 * (np / 32 + 2) * sizeof(uint32_t), c->stream));
  // k_bundle_order's tables (vbx_order.cuh), for the bucket count after np insertions
  OrderScratch& g = F.order_scratch;
  g.cap = (uint32_t)np;
  uint32_t buckets = 1;
  for (int k = 0; k < c->rehash.count && c->rehash.m[k] < np; ++k) buckets = c->rehash.n[k];
  g.bucket_cap = buckets;
  VBX_CUDA(c, h.dev(&g.h, 2 * np));
  VBX_CUDA(c, h.dev(&g.tau, np));
  VBX_CUDA(c, h.dev(&g.tau2, np));
  VBX_CUDA(c, h.dev(&g.next, np));
  VBX_CUDA(c, h.dev(&g.bkt, np));
  VBX_CUDA(c, h.dev(&g.A, np));
  VBX_CUDA(c, h.dev(&g.bhead, (size_t)buckets));
  VBX_CUDA(c, h.dev(&g.head_of, 2 * np));
  VBX_CUDA(c, h.dev(&g.wp, 2 * (np / 32 + 2)));
  VBX_CUDA(c, h.dev(&g.cta_tot, 64));
  VBX_CUDA(c, h.stream(&F.side, cudaStreamNonBlocking, c->prio_lo));
  VBX_CUDA(c, h.event(&F.ev_fork, cudaEventDisableTiming));
  VBX_CUDA(c, h.event(&F.ev_join, cudaEventDisableTiming));
  return VBX_OK;
}

}  // namespace vbx

using namespace vbx;

// every synchronous entry point first waits for asynchronously submitted scans (and reports a
// deferred error of theirs)
#define VBX_DRAIN(c)                          \
  do {                                        \
    if (int _rc = drain_async(c)) return _rc; \
  } while (0)

extern "C" {

const char* vbx_version(void) { return "voxblox_b200 0.1 (sm_90a)"; }

const char* vbx_last_error(const vbx_ctx* ctx) { return ctx ? ctx->err.c_str() : "null context"; }

int vbx_create(const vbx_tsdf_config* cfg, float voxel_size, int voxels_per_side,
               const vbx_engine_options* opt_in, vbx_ctx** out) {
  if (!cfg || !out) return VBX_E_INVALID;
  *out = nullptr;
  if (!(voxel_size > 0.0f)) return VBX_E_INVALID;  // CHECK_GT(voxel_size_, 0.0f), core/layer.h:38
  if (voxels_per_side <= 0 || voxels_per_side > 16 || (voxels_per_side & (voxels_per_side - 1))) {
    return VBX_E_INVALID;  // CHECK(isPowerOfTwo(voxels_per_side)), core/common.h:239
  }
  vbx_ctx* c = new vbx_ctx;
  c->cfg = *cfg;
  // TsdfIntegratorBase ctor, tsdf_integrator.cc:57-64
  if (c->cfg.integrator_threads == 0) c->cfg.integrator_threads = 1;
  if (c->cfg.allow_clear && !c->cfg.voxel_carving_enabled) c->cfg.allow_clear = 0;
  vbx_engine_options o;
  std::memset(&o, 0, sizeof(o));
  if (opt_in) o = *opt_in;
  int cur = 0;
  cudaError_t e = cudaGetDevice(&cur);
  if (e != cudaSuccess) {
    delete c;
    return VBX_E_CUDA;
  }
  if (!opt_in || opt_in->device < 0) o.device = cur;
  if (o.max_blocks == 0) o.max_blocks = 32768;
  if (o.max_points_per_scan == 0) o.max_points_per_scan = 1u << 20;
  if (o.max_updates_per_pass == 0) o.max_updates_per_pass = 1ull << 26;
  if (o.world_size <= 0) o.world_size = 1;
  c->opt = o;
  c->device = o.device;
  c->voxel_size = voxel_size;
  c->voxel_size_inv = (float)(1.0 / voxel_size);  // setLayer, tsdf_integrator.cc:77
  c->vps = voxels_per_side;
  c->L = 0;
  while ((1 << c->L) < voxels_per_side) ++c->L;
  c->vox_per_block = 1u << (3 * c->L);
  c->max_points = o.max_points_per_scan;
  c->max_updates = std::min<uint64_t>(o.max_updates_per_pass, 0x7fffffffull);
  int rb = 0;
  for (uint32_t v = o.max_blocks; v; v >>= 1) ++rb;
  // an update record's key = (touched id, voxel in block) in 32 bits with 0xffffffff reserved: a single
  // call may touch up to 2^(32 - 3L) - 1 blocks; the pool itself is only bounded by memory
  if (rb > 30) {
    delete c;
    return VBX_E_INVALID;
  }
  if (o.world_size > 1 && (o.rank < 0 || o.rank >= o.world_size)) {
    delete c;
    return VBX_E_INVALID;
  }
  *out = c;  // from here on the caller can read vbx_last_error and must vbx_destroy
  Holdings& h = c->own_core;
  VBX_CUDA(c, cudaSetDevice(c->device));
  {
    int sms = 0;
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, c->device) == cudaSuccess && sms > 0) c->grid_sms = (unsigned int)sms;
    if (const char* e = std::getenv("VBX_GRID_SMS")) c->grid_sms = (unsigned int)std::max(1, std::atoi(e));
  }
  // stream priorities for the pipelined path: the stages that run in submission order (apply, then
  // the ray walk) are the pipeline's bottleneck, so their thread blocks go first
  int prio_lo = 0, prio_hi = 0;
  VBX_CUDA(c, cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi));  // numerically lower = higher priority
  c->prio_lo = prio_lo;
  c->prio_hi = prio_hi;
  VBX_CUDA(c, h.stream(&c->stream, cudaStreamNonBlocking, prio_hi));
  VBX_CUDA(c, h.stream(&c->stream_c, cudaStreamNonBlocking));
  VBX_CUDA(c, h.stream(&c->stream_c2, cudaStreamNonBlocking));
  VBX_CUDA(c, h.event(&c->ev0));
  VBX_CUDA(c, h.event(&c->ev1));
  VBX_CUDA(c, h.event(&c->tev0));
  VBX_CUDA(c, h.event(&c->tev1));
  for (int i = 0; i < 20; ++i) VBX_CUDA(c, h.event(&c->sev[i]));
  uint32_t hcap = 1;
  while (hcap < 2 * o.max_blocks) hcap <<= 1;
  c->hcap = hcap;
  Tables& t = c->tab;
  std::memset(&t, 0, sizeof(t));
  t.hmask = hcap - 1;
  t.max_blocks = o.max_blocks;
  VBX_CUDA(c, h.dev(&t.hkeys, hcap));
  VBX_CUDA(c, h.dev(&t.hslot, hcap));
  VBX_CUDA(c, h.dev(&t.new_list, o.max_blocks));
  // one local id per block a call touches (vbx_hash.cuh, scan_block_id), with headroom past the pool;
  // (id, voxel) must fit a 32-bit record key
  t.touched_cap = (uint32_t)std::min<uint64_t>((uint64_t)o.max_blocks + 65536u, (0xffffffffull >> (3 * c->L)) - 1);
  t.vox_per_block = c->vox_per_block;
  VBX_CUDA(c, h.dev(&t.slot_key, o.max_blocks));
  VBX_CUDA(c, h.dev(&t.slot_updated, o.max_blocks));
  VBX_CUDA(c, h.dev(&t.slot_esdf_updated, o.max_blocks));
  VBX_CUDA(c, h.dev(&t.slot_has_esdf, o.max_blocks));
  VBX_CUDA(c, h.dev(&t.tsdf, (size_t)o.max_blocks * c->vox_per_block));
  VBX_CUDA(c, cudaMemsetAsync(t.hkeys, 0xff, (size_t)hcap * sizeof(uint64_t), c->stream));
  VBX_CUDA(c, cudaMemsetAsync(t.hslot, 0xff, (size_t)hcap * sizeof(int32_t), c->stream));
  VBX_CUDA(c, cudaMemsetAsync(t.slot_updated, 0, o.max_blocks, c->stream));
  VBX_CUDA(c, cudaMemsetAsync(t.slot_esdf_updated, 0, o.max_blocks, c->stream));
  VBX_CUDA(c, cudaMemsetAsync(t.slot_has_esdf, 0, o.max_blocks, c->stream));
  // new Block: voxels default-constructed = all zero bytes (core/voxel.h:12-16)
  VBX_CUDA(c, cudaMemsetAsync(t.tsdf, 0, (size_t)o.max_blocks * c->vox_per_block * sizeof(TsdfVoxel), c->stream));
  const size_t np = c->max_points;
  VBX_CUDA(c, h.dev(&c->order, np));
  VBX_CUDA(c, h.dev(&c->order_inv, np));
  if (int rc = init_bundle_order(c)) return rc;
  c->sort_tiles_cap[0] = (uint32_t)((np + kSortTile - 1) / kSortTile);
  c->sort_tiles_cap[1] = (uint32_t)((c->max_updates + kSortTile - 1) / kSortTile);
  VBX_CUDA(c, h.dev(&c->set_start, kApproxSetWords));
  VBX_CUDA(c, h.dev(&c->set_observed, kApproxSetWords));
  if (int rc = init_fast_sets(c, c->stream)) return rc;
  VBX_CUDA(c, h.dev(&c->d_nblocks, 2));
  VBX_CUDA(c, cudaMemsetAsync(c->d_nblocks, 0, 2 * sizeof(uint32_t), c->stream));
  // the synchronous calls' scratch; ensure_async allocates the other sets and lanes
  if (int rc = alloc_set(c, h, c->set[0])) return rc;
  if (int rc = alloc_lane(c, h, c->lane[0])) return rc;
  VBX_CUDA(c, cudaStreamSynchronize(c->stream));
  return VBX_OK;
}

}  // extern "C" (reopened below)

namespace vbx {
// First asynchronous submission: the remaining hand-off sets, the second front lane, streams, events.
int ensure_async(vbx_ctx* c) {
  if (c->pipe.ready) return VBX_OK;
  Holdings& h = c->pipe.own;
  h.release();  // whatever a failed earlier call made
  if (const char* e = std::getenv("VBX_ASYNC_SETS")) c->pipe.sets_in_use = std::max(2, std::min(std::atoi(e), (int)vbx_ctx::kSets));
  if (const char* e = std::getenv("VBX_ASYNC_LANES")) c->pipe.lanes_in_use = std::max(1, std::min(std::atoi(e), (int)vbx_ctx::kLanes));
  VBX_CUDA(c, h.stream(&c->pipe.stream_e, cudaStreamNonBlocking, std::min(c->prio_lo, c->prio_hi + 1)));
  VBX_CUDA(c, h.stream(&c->pipe.stream_s, cudaStreamNonBlocking, std::min(c->prio_lo, c->prio_hi + 2)));
  for (cudaEvent_t& e : c->pipe.cap_ev) VBX_CUDA(c, h.event(&e, cudaEventDisableTiming));
  VBX_CUDA(c, h.dev(&c->pipe.d_hold, 1));
  VBX_CUDA(c, cudaMemsetAsync(c->pipe.d_hold, 0, sizeof(uint32_t), c->stream));  // (alloc_set synchronises the stream)
  for (int l = 0; l < c->pipe.lanes_in_use; ++l) {
    vbx_ctx::FrontLane& F = c->lane[l];
    VBX_CUDA(c, h.stream(&F.stream, cudaStreamNonBlocking, c->prio_lo));
    VBX_CUDA(c, h.event(&F.done, cudaEventDisableTiming));
    if (l == 0) continue;
    if (int rc = alloc_lane(c, h, F)) return rc;
  }
  // diagnostic: with VBX_ASYNC_TIMELINE set the hand-off events keep timestamps (vbx_debug_async_timeline)
  c->pipe.timeline = std::getenv("VBX_ASYNC_TIMELINE") != nullptr;
  const unsigned int evf = c->pipe.timeline ? cudaEventDefault : cudaEventDisableTiming;
  if (c->pipe.timeline) {
    VBX_CUDA(c, h.event(&c->pipe.timeline_ref));
    VBX_CUDA(c, cudaEventRecord(c->pipe.timeline_ref, c->stream));
  }
  for (int k = 0; k < c->pipe.sets_in_use; ++k) {
    vbx_ctx::ScratchSet& S = c->set[k];
    VBX_CUDA(c, h.stream(&S.stream, cudaStreamNonBlocking));
    VBX_CUDA(c, h.event(&S.copy_done, evf));
    VBX_CUDA(c, h.event(&S.walked, evf));
    VBX_CUDA(c, h.event(&S.sorted, evf));
    VBX_CUDA(c, h.event(&S.back_done, evf));
    VBX_CUDA(c, h.event(&S.applied, evf));
    if (c->pipe.timeline) {
      VBX_CUDA(c, h.event(&S.front_start));
      VBX_CUDA(c, h.event(&S.front_done));
    }
    if (k == 0) continue;
    if (int rc = alloc_set(c, h, S)) return rc;
  }
  c->pipe.ready = true;
  return VBX_OK;
}
}  // namespace vbx

extern "C" {

void vbx_destroy(vbx_ctx* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  // every stream's work ends before the context's owners free what it reads
  for (cudaStream_t s : {c->stream, c->stream_c, c->stream_c2}) {
    if (s) cudaStreamSynchronize(s);
  }
  for (const vbx_ctx::ScratchSet& S : c->set) {
    if (S.stream) cudaStreamSynchronize(S.stream);
  }
  for (const vbx_ctx::FrontLane& F : c->lane) {
    if (F.stream) cudaStreamSynchronize(F.stream);
    if (F.side) cudaStreamSynchronize(F.side);
  }
  delete c;
}

int vbx_get_tsdf_config(const vbx_ctx* c, vbx_tsdf_config* out) {
  if (!c || !out) return VBX_E_INVALID;
  *out = c->cfg;
  return VBX_OK;
}

int vbx_tsdf_integrate_device(vbx_ctx* c, int kind, const float q[4], const float t[3], const float* d_xyz,
                              const uint8_t* d_rgba, uint64_t n, int freespace) {
  if (!c || !q || !t || (n && (!d_xyz || !d_rgba))) return fail(c, VBX_E_INVALID, "null argument");
  VBX_CUDA(c, cudaSetDevice(c->device));
  VBX_DRAIN(c);
  return integrate_device(c, sync_route(c), kind, q, t, d_xyz, d_rgba, n, freespace);
}

int vbx_tsdf_integrate(vbx_ctx* c, int kind, const float q[4], const float t[3], const float* xyz,
                       const uint8_t* rgba, uint64_t n, int freespace) {
  if (!c || !q || !t || (n && (!xyz || !rgba))) return fail(c, VBX_E_INVALID, "null argument");
  if (n > c->max_points) return fail(c, VBX_E_CAPACITY, "cloud larger than max_points_per_scan");
  VBX_CUDA(c, cudaSetDevice(c->device));
  VBX_DRAIN(c);
  const vbx_ctx::ScratchSet& S = c->set[0];
  if (n) {
    VBX_CUDA(c, cudaMemcpyAsync(S.d_xyz, xyz, n * 3 * sizeof(float), cudaMemcpyHostToDevice, c->stream));
    VBX_CUDA(c, cudaMemcpyAsync(S.d_rgba, rgba, n * 4, cudaMemcpyHostToDevice, c->stream));
  }
  return integrate_device(c, sync_route(c), kind, q, t, S.d_xyz, S.d_rgba, n, freespace);
}

int vbx_tsdf_integrate_async(vbx_ctx* c, int kind, const float q[4], const float t[3], const float* xyz,
                             const uint8_t* rgba, uint64_t n, int freespace, int inputs_on_device) {
  if (!c || !q || !t || (n && (!xyz || !rgba))) return fail(c, VBX_E_INVALID, "null argument");
  if (cudaSetDevice(c->device) != cudaSuccess) return fail(c, VBX_E_CUDA, "cudaSetDevice");
  return integrate_async(c, sync_route(c), kind, q, t, xyz, rgba, n, freespace, inputs_on_device);
}

int vbx_block_owner(const vbx_ctx* c, const int32_t block_index[3], int32_t* owner) {
  if (!c || !block_index || !owner) return VBX_E_INVALID;
  *owner = c->opt.world_size > 1 ? block_owner(block_index[0], block_index[1], block_index[2], c->opt.world_size) : 0;
  return VBX_OK;
}

int vbx_debug_sort(vbx_ctx* c, const void* keys, int key_bytes, uint32_t n, int key_bits, void* keys_out,
                   uint32_t* vals_out) {
  if (!c || (n && (!keys || !keys_out || !vals_out))) return fail(c, VBX_E_INVALID, "null argument");
  VBX_CUDA(c, cudaSetDevice(c->device));
  VBX_DRAIN(c);
  return debug_sort(c, keys, key_bytes, n, key_bits, keys_out, vals_out);
}

int vbx_debug_async_timeline(vbx_ctx* c, uint64_t* seq, float* ms, int cap_sets) {
  if (!c || !seq || !ms) return VBX_E_INVALID;
  if (!c->pipe.ready || !c->pipe.timeline) return fail(c, VBX_E_STATE, "set VBX_ASYNC_TIMELINE before the first asynchronous submission");
  for (int k = 0; k < cap_sets; ++k) {
    if (k >= c->pipe.sets_in_use) {
      seq[k] = ~0ull;
      continue;
    }
    vbx_ctx::ScratchSet& S = c->set[k];
    seq[k] = S.seq;
    cudaEvent_t ev[5] = {S.front_start, S.front_done, S.walked, S.sorted, S.applied};
    for (int j = 0; j < 5; ++j) {
      float t = -1.f;
      if (cudaEventSynchronize(ev[j]) != cudaSuccess || cudaEventElapsedTime(&t, c->pipe.timeline_ref, ev[j]) != cudaSuccess) {
        t = -1.f;
        cudaGetLastError();
      }
      ms[5 * k + j] = t;
    }
  }
  return VBX_OK;
}

int vbx_debug_scan(vbx_ctx* c, const uint32_t* in, uint32_t n, uint32_t* out) {
  if (!c || (n && (!in || !out))) return fail(c, VBX_E_INVALID, "null argument");
  VBX_CUDA(c, cudaSetDevice(c->device));
  VBX_DRAIN(c);
  return debug_scan(c, in, n, out);
}

int vbx_debug_bundle_order(vbx_ctx* c, const uint32_t* hashes, uint32_t n, int force_global, uint32_t* out) {
  if (!c || (n && (!hashes || !out))) return fail(c, VBX_E_INVALID, "null argument");
  VBX_CUDA(c, cudaSetDevice(c->device));
  VBX_DRAIN(c);
  return debug_bundle_order(c, hashes, n, force_global, out);
}

int vbx_debug_apply(vbx_ctx* c, const int32_t* idx3, uint32_t n_blocks, uint64_t n, const uint32_t* rec_block,
                    const uint32_t* rec_voxel, const float* sdf, const float* weight, const uint8_t* rgba,
                    uint64_t paths[16]) {
  if (!c || (n_blocks && !idx3) || (n && (!rec_block || !rec_voxel || !sdf || !weight || !rgba))) {
    return fail(c, VBX_E_INVALID, "null argument");
  }
  VBX_CUDA(c, cudaSetDevice(c->device));
  VBX_DRAIN(c);
  return debug_apply(c, idx3, n_blocks, n, rec_block, rec_voxel, sdf, weight, rgba, paths);
}

int vbx_debug_count_apply_paths(vbx_ctx* c, int enabled) {
  if (!c) return VBX_E_INVALID;
  VBX_CUDA(c, cudaSetDevice(c->device));
  VBX_DRAIN(c);  // (scans already queued keep the setting they were submitted with)
  c->count_apply_paths = enabled != 0;
  return VBX_OK;
}

int vbx_debug_serial_fast(vbx_ctx* c, int enabled) {
  if (!c) return VBX_E_INVALID;
  VBX_CUDA(c, cudaSetDevice(c->device));
  VBX_DRAIN(c);
  c->serial_fast = enabled != 0;
  return VBX_OK;
}

int vbx_debug_apply_paths(const vbx_ctx* c, uint64_t out[16]) {
  if (!c || !out) return VBX_E_INVALID;
  std::memcpy(out, c->apply_paths, sizeof(c->apply_paths));
  return VBX_OK;
}

int vbx_get_counters(const vbx_ctx* c, uint64_t out[16]) {
  if (!c || !out) return VBX_E_INVALID;
  std::memcpy(out, c->counters, sizeof(c->counters));
  out[kCntLaunchesTotal] = c->launches;
  out[kCntAsyncRedone] = c->pipe.redone;
  out[kCntAsyncWaitNs] = c->pipe.wait_ns;
  out[kCntAsyncSubmitNs] = c->pipe.submit_ns;
  return VBX_OK;
}

int vbx_esdf_get_counters(const vbx_ctx* c, uint64_t out[16]) {
  if (!c || !out) return VBX_E_INVALID;
  std::memcpy(out, c->esdf.counters, sizeof(c->esdf.counters));
  return VBX_OK;
}

int vbx_last_device_ms(const vbx_ctx* c, float* ms) {
  if (!c || !ms) return VBX_E_INVALID;
  *ms = c->last_ms;
  return VBX_OK;
}

int vbx_host_alloc(vbx_ctx* c, size_t bytes, void** out) {
  if (!c || !out) return VBX_E_INVALID;
  VBX_CUDA(c, cudaSetDevice(c->device));
  VBX_DRAIN(c);
  VBX_CUDA(c, cudaHostAlloc(out, bytes, cudaHostAllocPortable));
  return VBX_OK;
}

int vbx_host_free(vbx_ctx* c, void* p) {
  if (!c) return VBX_E_INVALID;
  VBX_CUDA(c, cudaFreeHost(p));
  return VBX_OK;
}

int vbx_host_copy_ms(vbx_ctx* c, const void* src, size_t bytes, float* ms) {
  if (!c || !src || !ms) return VBX_E_INVALID;
  if (bytes > (size_t)c->max_points * 12) return fail(c, VBX_E_CAPACITY, "copy larger than the staging buffer");
  VBX_CUDA(c, cudaSetDevice(c->device));
  VBX_DRAIN(c);
  VBX_CUDA(c, cudaEventRecord(c->tev0, c->stream));
  VBX_CUDA(c, cudaMemcpyAsync(c->set[0].d_xyz, src, bytes, cudaMemcpyHostToDevice, c->stream));
  VBX_CUDA(c, cudaEventRecord(c->tev1, c->stream));
  VBX_CUDA(c, cudaEventSynchronize(c->tev1));
  VBX_CUDA(c, cudaEventElapsedTime(ms, c->tev0, c->tev1));
  return VBX_OK;
}

int vbx_timer_start(vbx_ctx* c) {
  if (!c) return VBX_E_INVALID;
  VBX_CUDA(c, cudaSetDevice(c->device));
  VBX_DRAIN(c);
  VBX_CUDA(c, cudaEventRecord(c->tev0, c->stream));
  return VBX_OK;
}

int vbx_timer_stop_ms(vbx_ctx* c, float* ms) {
  if (!c || !ms) return VBX_E_INVALID;
  VBX_CUDA(c, cudaSetDevice(c->device));
  VBX_DRAIN(c);
  VBX_CUDA(c, cudaEventRecord(c->tev1, c->stream));
  VBX_CUDA(c, cudaEventSynchronize(c->tev1));
  VBX_CUDA(c, cudaEventElapsedTime(ms, c->tev0, c->tev1));
  return VBX_OK;
}

int vbx_set_stage_profiling(vbx_ctx* c, int enabled) {
  if (!c) return VBX_E_INVALID;
  c->profiling = enabled != 0;
  std::memset(c->stage_ms, 0, sizeof(c->stage_ms));
  std::memset(c->stage_calls, 0, sizeof(c->stage_calls));
  return VBX_OK;
}

int vbx_get_stage_ms(const vbx_ctx* c, double ms[16], uint64_t calls[16]) {
  if (!c || !ms || !calls) return VBX_E_INVALID;
  std::memcpy(ms, c->stage_ms, sizeof(c->stage_ms));
  std::memcpy(calls, c->stage_calls, sizeof(c->stage_calls));
  return VBX_OK;
}

int vbx_sync(vbx_ctx* c) {
  if (!c) return VBX_E_INVALID;
  VBX_CUDA(c, cudaSetDevice(c->device));
  VBX_DRAIN(c);
  VBX_CUDA(c, cudaStreamSynchronize(c->stream));  // (the drain above already waited for every queued scan)
  return VBX_OK;
}

int vbx_num_blocks(vbx_ctx* c, int layer, uint64_t* n) {
  if (!c || !n) return VBX_E_INVALID;
  VBX_CUDA(c, cudaSetDevice(c->device));
  VBX_DRAIN(c);
  if (layer == VBX_LAYER_TSDF && !c->maybe_esdf_only) {
    *n = c->n_blocks;
    return VBX_OK;
  }
  LayerSlots view;  // (no members in the ESDF layer before vbx_esdf_create)
  if (int rc = read_layer_slots(c, layer, &view)) return rc;
  *n = (uint64_t)std::count(view.member.begin(), view.member.end(), 1);
  return VBX_OK;
}

int vbx_list_blocks(vbx_ctx* c, int layer, int updated_mask, int32_t* idx3, uint64_t cap, uint64_t* n) {
  if (!c || !n) return VBX_E_INVALID;
  VBX_CUDA(c, cudaSetDevice(c->device));
  VBX_DRAIN(c);
  *n = 0;
  LayerSlots view;
  if (int rc = read_layer_slots(c, layer, &view)) return rc;
  // selected on the reported bits only: VBX_UPDATED_MIRROR lists nothing here
  const std::vector<LayerSlots::Entry> keys = view.sorted(kReportedBits, updated_mask);
  *n = keys.size();
  if (idx3) {
    const uint64_t m = std::min<uint64_t>(cap, keys.size());
    for (uint64_t i = 0; i < m; ++i) {
      idx3[3 * i] = keys[i].x;
      idx3[3 * i + 1] = keys[i].y;
      idx3[3 * i + 2] = keys[i].z;
    }
  }
  return VBX_OK;
}

int vbx_download_blocks(vbx_ctx* c, int layer, const int32_t* idx3, uint64_t m, void* voxels,
                        uint8_t* updated_bits) {
  if (!c || (m && (!idx3 || !voxels))) return fail(c, VBX_E_INVALID, "null argument");
  VBX_CUDA(c, cudaSetDevice(c->device));
  VBX_DRAIN(c);
  if (layer == VBX_LAYER_ESDF && !c->esdf.ready) return fail(c, VBX_E_STATE, "no ESDF layer");
  LayerSlots view;
  if (int rc = read_layer_slots(c, layer, &view)) return rc;
  std::vector<int32_t> slots(m);
  view.find(idx3, m, slots.data());
  const size_t vbytes = (layer == VBX_LAYER_TSDF) ? sizeof(TsdfVoxel) : sizeof(EsdfVoxel);
  const size_t bbytes = vbytes * c->vox_per_block;
  const char* pool = (layer == VBX_LAYER_TSDF) ? reinterpret_cast<const char*>(c->tab.tsdf)
                                               : reinterpret_cast<const char*>(c->tab.esdf);
  for (uint64_t i = 0; i < m; ++i) {
    if (slots[i] < 0) return fail(c, VBX_E_NOT_FOUND, "block not allocated");
    // one copy per block: the mirror's gather kernels are tested against this path
    VBX_CUDA(c, cudaMemcpyAsync(static_cast<char*>(voxels) + i * bbytes, pool + (size_t)slots[i] * bbytes,
                                bbytes, cudaMemcpyDeviceToHost, c->stream));
    if (updated_bits) updated_bits[i] = view.flags[slots[i]] & kReportedBits;
  }
  VBX_CUDA(c, cudaStreamSynchronize(c->stream));
  return VBX_OK;
}

int vbx_mirror_updated(vbx_ctx* c, int layer, int updated_mask, int clear_mask, int32_t* idx3, void* voxels,
                       uint8_t* updated_bits, uint64_t cap, uint64_t* n) {
  if (!c || !n || (cap && (!idx3 || !voxels))) return fail(c, VBX_E_INVALID, "null argument");
  VBX_CUDA(c, cudaSetDevice(c->device));
  VBX_DRAIN(c);
  *n = 0;
  if (layer == VBX_LAYER_ESDF && !c->esdf.ready) return VBX_OK;
  return mirror_updated(c, layer, updated_mask, clear_mask, idx3, voxels, updated_bits, cap, n, 0);
}

int vbx_serialize_updated(vbx_ctx* c, int layer, int updated_mask, int clear_mask, int32_t* idx3, uint32_t* words,
                          uint8_t* updated_bits, uint64_t cap, uint64_t* n) {
  if (!c || !n || (cap && (!idx3 || !words))) return fail(c, VBX_E_INVALID, "null argument");
  VBX_CUDA(c, cudaSetDevice(c->device));
  VBX_DRAIN(c);
  *n = 0;
  if (layer == VBX_LAYER_ESDF && !c->esdf.ready) return VBX_OK;
  return mirror_updated(c, layer, updated_mask, clear_mask, idx3, words, updated_bits, cap, n, 1);
}

int vbx_deserialize_blocks(vbx_ctx* c, int layer, const int32_t* idx3, uint64_t m, const uint32_t* words,
                           const uint8_t* updated_bits) {
  if (!c || (m && (!idx3 || !words))) return fail(c, VBX_E_INVALID, "null argument");
  VBX_CUDA(c, cudaSetDevice(c->device));
  VBX_DRAIN(c);
  return upload_blocks(c, layer, idx3, m, words, updated_bits, 1);
}

int vbx_clear_updated(vbx_ctx* c, int layer, int updated_mask) {
  if (!c) return VBX_E_INVALID;
  VBX_CUDA(c, cudaSetDevice(c->device));
  VBX_DRAIN(c);
  return keep_flag_bits(c, (layer == VBX_LAYER_TSDF) ? c->tab.slot_updated : c->tab.slot_esdf_updated,
                        (uint8_t)(~updated_mask | kEngineBit));
}

int vbx_upload_blocks(vbx_ctx* c, int layer, const int32_t* idx3, uint64_t m, const void* voxels,
                      const uint8_t* updated_bits) {
  if (!c || (m && (!idx3 || !voxels))) return fail(c, VBX_E_INVALID, "null argument");
  VBX_CUDA(c, cudaSetDevice(c->device));
  VBX_DRAIN(c);
  return upload_blocks(c, layer, idx3, m, voxels, updated_bits, 0);
}

// device memory of this process (cudaMalloc, or managed), 4-byte aligned: the transfer kernels read and write
// 32-bit words
static bool device_words(const void* p) {
  cudaPointerAttributes a;
  const bool dev = cudaPointerGetAttributes(&a, p) == cudaSuccess &&
                   (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged);
  cudaGetLastError();  // (an unregistered host pointer may leave an error code behind)
  return dev && reinterpret_cast<uintptr_t>(p) % 4 == 0;
}

int vbx_gather_updated_device(vbx_ctx* c, int layer, int updated_mask, int clear_mask, int owned_only, int32_t* d_idx3,
                              void* d_voxels, uint64_t cap, uint64_t* n) {
  if (!c || !n || (cap && (!d_idx3 || !d_voxels))) return fail(c, VBX_E_INVALID, "null argument");
  VBX_CUDA(c, cudaSetDevice(c->device));
  if (cap && (!device_words(d_idx3) || !device_words(d_voxels))) {
    return fail(c, VBX_E_INVALID, "d_idx3 / d_voxels must be 4-byte aligned device memory");
  }
  VBX_DRAIN(c);
  *n = 0;
  if (layer == VBX_LAYER_ESDF && !c->esdf.ready) return VBX_OK;
  return gather_updated_device(c, layer, updated_mask, clear_mask, owned_only, d_idx3, d_voxels, cap, n);
}

int vbx_upload_blocks_device(vbx_ctx* c, int layer, const int32_t* d_idx3, uint64_t m, const void* d_voxels,
                             uint8_t updated_bits) {
  if (!c || (m && (!d_idx3 || !d_voxels))) return fail(c, VBX_E_INVALID, "null argument");
  VBX_CUDA(c, cudaSetDevice(c->device));
  if (m && (!device_words(d_idx3) || !device_words(d_voxels))) {
    return fail(c, VBX_E_INVALID, "d_idx3 / d_voxels must be 4-byte aligned device memory");
  }
  VBX_DRAIN(c);
  return upload_blocks_device(c, layer, d_idx3, m, d_voxels, updated_bits);
}

int vbx_debug_staging_bytes(const vbx_ctx* c, uint64_t* host_bytes) {
  if (!c || !host_bytes) return VBX_E_INVALID;
  *host_bytes = c->mirror.host ? c->mirror.cap_bytes : 0;
  return VBX_OK;
}

int vbx_remove_blocks(vbx_ctx* c, int layer, const int32_t* idx3, uint64_t m) {
  if (!c || (m && !idx3)) return fail(c, VBX_E_INVALID, "null argument");
  VBX_CUDA(c, cudaSetDevice(c->device));
  VBX_DRAIN(c);
  return remove_blocks(c, layer, idx3, m);
}

int vbx_clear(vbx_ctx* c, int layer) {
  if (!c) return VBX_E_INVALID;
  VBX_CUDA(c, cudaSetDevice(c->device));
  VBX_DRAIN(c);
  return clear_layer(c, layer);
}

int vbx_esdf_create(vbx_ctx* c, const vbx_esdf_config* cfg) {
  if (!c || !cfg) return VBX_E_INVALID;
  VBX_CUDA(c, cudaSetDevice(c->device));
  VBX_DRAIN(c);
  return esdf_create(c, cfg);
}

int vbx_esdf_update(vbx_ctx* c, int batch, int clear_updated_flag) {
  if (!c) return VBX_E_INVALID;
  VBX_CUDA(c, cudaSetDevice(c->device));
  VBX_DRAIN(c);
  if (!c->esdf.ready) return fail(c, VBX_E_STATE, "vbx_esdf_update before vbx_esdf_create");
  return esdf_update(c, batch, clear_updated_flag);
}

int vbx_esdf_update_blocks(vbx_ctx* c, const int32_t* idx3, uint64_t m, int incremental) {
  if (!c || (m && !idx3)) return fail(c, VBX_E_INVALID, "null argument");
  VBX_CUDA(c, cudaSetDevice(c->device));
  VBX_DRAIN(c);
  if (!c->esdf.ready) return fail(c, VBX_E_STATE, "vbx_esdf_update_blocks before vbx_esdf_create");
  return esdf_update_blocks(c, idx3, m, incremental);
}

int vbx_mesh_generate(vbx_ctx* c, const vbx_mesh_config* cfg, int only_mesh_updated_blocks, int clear_updated_flag,
                      uint64_t* n_blocks, uint64_t* n_vertices) {
  if (!c || !cfg) return fail(c, VBX_E_INVALID, "null argument");
  VBX_CUDA(c, cudaSetDevice(c->device));
  VBX_DRAIN(c);
  return mesh_generate(c, cfg, only_mesh_updated_blocks, clear_updated_flag, n_blocks, n_vertices);
}

int vbx_icp_run(vbx_ctx* c, const vbx_icp_config* cfg, const float* points_C, uint64_t n, const float q_wxyz[4],
                const float t[3], uint32_t seed, float out_q_wxyz[4], float out_t[3], uint64_t* num_updates) {
  if (!c || !cfg || (n && !points_C) || !q_wxyz || !t || !out_q_wxyz || !out_t) return fail(c, VBX_E_INVALID, "null argument");
  VBX_CUDA(c, cudaSetDevice(c->device));
  VBX_DRAIN(c);
  return icp_run(c, cfg, points_C, 0, n, q_wxyz, t, seed, out_q_wxyz, out_t, num_updates);
}

int vbx_icp_run_device(vbx_ctx* c, const vbx_icp_config* cfg, const float* d_points_C, uint64_t n, const float q_wxyz[4],
                       const float t[3], uint32_t seed, float out_q_wxyz[4], float out_t[3], uint64_t* num_updates) {
  if (!c || !cfg || (n && !d_points_C) || !q_wxyz || !t || !out_q_wxyz || !out_t) return fail(c, VBX_E_INVALID, "null argument");
  VBX_CUDA(c, cudaSetDevice(c->device));
  VBX_DRAIN(c);
  return icp_run(c, cfg, d_points_C, 1, n, q_wxyz, t, seed, out_q_wxyz, out_t, num_updates);
}

int vbx_debug_icp_solve(vbx_ctx* c, uint32_t n, int refine_roll_pitch, const float* h, const float* m, const float* q,
                        const float* w, float* r_out, int32_t* valid_out, float* q_out, float* log_out, float* exp_out) {
  if (!c || (n && (!h || !m || !q || !w || !r_out || !valid_out || !q_out || !log_out || !exp_out)))
    return fail(c, VBX_E_INVALID, "null argument");
  VBX_CUDA(c, cudaSetDevice(c->device));
  VBX_DRAIN(c);
  return icp_debug_solve(c, n, refine_roll_pitch, h, m, q, w, r_out, valid_out, q_out, log_out, exp_out);
}

int vbx_mesh_download(vbx_ctx* c, int32_t* idx3, uint64_t* first_vertex, float* vertices, float* normals,
                      uint8_t* colors) {
  if (!c) return VBX_E_INVALID;
  VBX_CUDA(c, cudaSetDevice(c->device));
  return mesh_download(c, idx3, first_vertex, vertices, normals, colors);
}

int vbx_esdf_add_robot_position(vbx_ctx* c, const float position[3]) {
  if (!c || !position) return fail(c, VBX_E_INVALID, "null argument");
  VBX_CUDA(c, cudaSetDevice(c->device));
  VBX_DRAIN(c);
  if (!c->esdf.ready) return fail(c, VBX_E_STATE, "vbx_esdf_add_robot_position before vbx_esdf_create");
  return esdf_add_robot_position(c, position);
}

int vbx_esdf_clear(vbx_ctx* c) {
  if (!c) return VBX_E_INVALID;
  VBX_CUDA(c, cudaSetDevice(c->device));
  VBX_DRAIN(c);
  if (!c->esdf.ready) return fail(c, VBX_E_STATE, "no ESDF integrator");
  return esdf_clear_state(c);
}

int vbx_esdf_set_max_distance(vbx_ctx* c, float max_distance_m) {
  if (!c) return VBX_E_INVALID;
  if (!c->esdf.ready) return fail(c, VBX_E_STATE, "no ESDF integrator");
  // setEsdfMaxDistance, esdf_integrator.h:140-145: the default distance follows upwards
  c->esdf.cfg.max_distance_m = max_distance_m;
  if (c->esdf.cfg.default_distance_m < max_distance_m) c->esdf.cfg.default_distance_m = max_distance_m;
  return VBX_OK;
}

int vbx_esdf_set_full_euclidean(vbx_ctx* c, int full_euclidean) {
  if (!c) return VBX_E_INVALID;
  if (!c->esdf.ready) return fail(c, VBX_E_STATE, "no ESDF integrator");
  c->esdf.cfg.full_euclidean_distance = full_euclidean ? 1 : 0;  // esdf_integrator.h:147-149
  return VBX_OK;
}

int vbx_esdf_get_config(const vbx_ctx* c, vbx_esdf_config* out) {
  if (!c || !out) return VBX_E_INVALID;
  if (!c->esdf.ready) return VBX_E_STATE;
  *out = c->esdf.cfg;
  return VBX_OK;
}

}  // extern "C"
