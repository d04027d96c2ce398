// Host-driven block management of the device map: the counterparts of Layer::insertBlock /
// allocateBlockPtrByIndex (+ voxel copy), removeBlock and removeAllBlocks
// (voxblox/include/voxblox/core/layer.h:103-111,152-164).  None of this is on the per-scan hot
// path; it exists so that host code which edits the Layer between scans (loading a map,
// TsdfServer's removeDistantBlocks, voxblox_ros/src/tsdf_server.cc:314-316) can keep the HBM map
// of record in step.
#include <algorithm>
#include <cstring>
#include <numeric>
#include <vector>

#include "vbx_engine.h"
#include "vbx_hash.cuh"

namespace vbx {

// an uploaded block's local id in the hand-off set's table (k_assign creates the missing blocks)
__global__ void k_list_keys(ScanBlocks sb, const uint64_t* __restrict__ keys, uint32_t m, uint32_t* __restrict__ ids,
                            ScanState* st) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  ids[i] = scan_block_id(sb, keys[i], st);
}

// ... and its pool slot once k_assign has resolved the id to a hash position (touched_list)
__global__ void k_slots_of(const int32_t* __restrict__ hslot, const uint32_t* __restrict__ touched_list,
                           const uint32_t* __restrict__ ids, uint32_t m, int32_t* __restrict__ slot_out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  const uint32_t hp = ids[i] == 0xffffffffu ? 0xffffffffu : touched_list[ids[i]];
  slot_out[i] = hp == 0xffffffffu ? -1 : hslot[hp];
}

// rebuild the hash from the per-slot keys (after blocks were removed and the pool compacted)
__global__ void k_rebuild_hash(Tables tab, uint32_t n_blocks) {
  const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n_blocks) return;
  const uint64_t key = tab.slot_key[s];
  uint32_t hp = hash64(key) & tab.hmask;
  while (true) {
    const unsigned long long old = atomicCAS(reinterpret_cast<unsigned long long*>(tab.hkeys + hp),
                                             (unsigned long long)kEmptyKey, (unsigned long long)key);
    if (old == kEmptyKey) {
      tab.hslot[hp] = (int32_t)s;
      return;
    }
    hp = (hp + 1) & tab.hmask;
  }
}

// The block transfer kernels take the block number from blockIdx.y, which is capped at 65,535: larger
// batches are launched in slices of at most that many blocks.
static constexpr uint64_t kMaxGridY = 65535;

// The block hash rebuilt from slot_key: after removals, and after a call that ran out of pool slots
// (its surplus hash entries have no slot and must not be found by later calls).
int rebuild_hash(vbx_ctx* c) {
  cudaStream_t s = c->stream;
  VBX_CUDA(c, cudaMemsetAsync(c->tab.hkeys, 0xff, (size_t)c->hcap * sizeof(uint64_t), s));
  VBX_CUDA(c, cudaMemsetAsync(c->tab.hslot, 0xff, (size_t)c->hcap * sizeof(int32_t), s));
  if (c->n_blocks) k_rebuild_hash<<<grid_for(c->n_blocks, 256), 256, 0, s>>>(c->tab, c->n_blocks);
  VBX_CUDA(c, cudaStreamSynchronize(s));
  VBX_CUDA(c, cudaGetLastError());
  return VBX_OK;
}

// ---- serialised block payloads (SURVEY.md section 8f N2), voxblox/src/core/block.cc:
//   TsdfVoxel -> 3 words: distance bits, weight bits, a | b<<8 | g<<16 | r<<24      (cc:159-183, :65-90)
//   EsdfVoxel -> 2 words: distance bits, parent x,y,z as int8 in bytes 3,2,1 | flag byte
//                (observed 1, hallucinated 2, in_queue 4, fixed 8)                (cc:203-234, :110-135)
// serializeDirection (cc:8-41) ORs `int8 << shift` as a sign-extended int, so a negative y or z
// also sets every byte above it; reproduced bit for bit.
__device__ __forceinline__ uint32_t tsdf_word(uint32_t w, uint32_t k) { return k == 2u ? __byte_perm(w, 0, 0x0123) : w; }

__device__ __forceinline__ uint2 esdf_pack(const uint32_t* v) {
  auto clamp8 = [](int32_t x) { return (int)max(-128, min(127, x)); };
  uint32_t d = 0;
  d |= (uint32_t)(clamp8((int32_t)v[2]) << 24);
  d |= (uint32_t)(clamp8((int32_t)v[3]) << 16);
  d |= (uint32_t)(clamp8((int32_t)v[4]) << 8);
  const uint32_t f = v[1];  // four bool bytes: observed, hallucinated, in_queue, fixed
  uint32_t flag = 0;
  if (f & 0x000000ffu) flag |= 1u;
  if (f & 0x0000ff00u) flag |= 2u;
  if (f & 0x00ff0000u) flag |= 4u;
  if (f & 0xff000000u) flag |= 8u;
  return make_uint2(v[0], d | flag);
}

__device__ __forceinline__ void esdf_unpack(uint2 w, uint32_t* v) {
  v[0] = w.x;
  v[1] = ((w.y & 1u) ? 0x00000001u : 0u) | ((w.y & 2u) ? 0x00000100u : 0u) | ((w.y & 4u) ? 0x00010000u : 0u) |
         ((w.y & 8u) ? 0x01000000u : 0u);
  v[2] = (uint32_t)(int32_t)(int8_t)((w.y >> 24) & 0xffu);  // deserializeDirection, cc:43-63
  v[3] = (uint32_t)(int32_t)(int8_t)((w.y >> 16) & 0xffu);
  v[4] = (uint32_t)(int32_t)(int8_t)((w.y >> 8) & 0xffu);
}

// device pool -> contiguous words in block.cc's format; one thread per output word (TSDF) / voxel (ESDF)
__global__ void k_serialize_blocks(int layer, const uint32_t* __restrict__ pool, const uint32_t* __restrict__ slots,
                                   uint32_t m, uint32_t vox_per_block, uint32_t* __restrict__ out,
                                   uint8_t* __restrict__ flags, uint8_t clear_mask) {
  const uint32_t b = blockIdx.y;
  if (b >= m) return;
  const uint32_t slot = slots[b];
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (layer == VBX_LAYER_TSDF) {
    const uint32_t nw = 3u * vox_per_block;
    if (i < nw) out[(size_t)b * nw + i] = tsdf_word(__ldcs(pool + (size_t)slot * nw + i), i % 3u);
  } else if (i < vox_per_block) {
    const uint32_t* v = pool + ((size_t)slot * vox_per_block + i) * 5u;
    uint32_t w[5] = {v[0], v[1], v[2], v[3], v[4]};
    reinterpret_cast<uint2*>(out)[(size_t)b * vox_per_block + i] = esdf_pack(w);
  }
  if (i == 0 && clear_mask) flags[slot] &= (uint8_t)~clear_mask;
}

// contiguous payloads (raw voxel structs or block.cc words) -> pool slots; also the per-slot flags
__global__ void k_scatter_blocks(int layer, int serialized, const uint32_t* __restrict__ in,
                                 const int32_t* __restrict__ slots, uint32_t m, uint32_t vox_per_block,
                                 uint32_t* __restrict__ pool, const uint8_t* __restrict__ upd_in, uint8_t upd_all,
                                 uint8_t* __restrict__ flags, uint8_t* __restrict__ has_esdf) {
  const uint32_t b = blockIdx.y;
  if (b >= m) return;
  const int32_t slot = slots[b];
  if (slot < 0) return;
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t wpv = (layer == VBX_LAYER_TSDF) ? 3u : 5u;
  if (!serialized || layer == VBX_LAYER_TSDF) {
    const uint32_t nw = wpv * vox_per_block;
    if (i < nw) {
      const uint32_t w = in[(size_t)b * nw + i];
      pool[(size_t)slot * nw + i] = (serialized ? tsdf_word(w, i % 3u) : w);  // the byte reversal is its own inverse
    }
  } else if (i < vox_per_block) {
    uint32_t v[5];
    esdf_unpack(reinterpret_cast<const uint2*>(in)[(size_t)b * vox_per_block + i], v);
    uint32_t* dst = pool + ((size_t)slot * vox_per_block + i) * 5u;
#pragma unroll
    for (int k = 0; k < 5; ++k) dst[k] = v[k];
  }
  if (i == 0) {
    // (bit 7 is the engine's own; a TSDF upload clears kSlotNoTsdf)
    flags[slot] = (uint8_t)((upd_in ? upd_in[b] : upd_all) & kReportedBits);
    if (has_esdf) has_esdf[slot] = 1;
  }
}

static int ensure_staging(vbx_ctx* c, size_t bytes, size_t slots) {
  if (bytes <= c->mirror.cap_bytes && slots <= c->mirror.cap_slots) return VBX_OK;
  Holdings& h = c->mirror.own;
  h.release();
  c->mirror.cap_bytes = c->mirror.cap_slots = 0;
  const size_t want_b = std::max<size_t>(2 * bytes, 16u << 20), want_s = std::max<size_t>(2 * slots, 1024);
  VBX_CUDA(c, h.dev(&c->mirror.dev, want_b));
  VBX_CUDA(c, h.host(&c->mirror.host, want_b));
  VBX_CUDA(c, h.dev(&c->mirror.slots, want_s));
  c->mirror.cap_bytes = want_b;
  c->mirror.cap_slots = want_s;
  return VBX_OK;
}

static size_t payload_bytes(const vbx_ctx* c, int layer, int serialized) {
  if (layer == VBX_LAYER_TSDF) return sizeof(TsdfVoxel) * c->vox_per_block;  // 3 words either way
  return (serialized ? 8u : sizeof(EsdfVoxel)) * c->vox_per_block;
}

// The packed keys of an upload's block indices; VBX_E_INVALID (before anything is written) for an index
// outside +-2^20
static int upload_keys(vbx_ctx* c, const int32_t* idx3, uint64_t m, std::vector<uint64_t>* keys) {
  keys->resize(m);
  for (uint64_t i = 0; i < m; ++i) {
    const int32_t* p = idx3 + 3 * i;
    const int lim = kCoordBias - 1;
    if (p[0] < -lim || p[0] > lim || p[1] < -lim || p[1] > lim || p[2] < -lim || p[2] > lim) {
      return fail(c, VBX_E_INVALID, "block index outside +-2^20");
    }
    (*keys)[i] = pack3(p[0], p[1], p[2]);
  }
  return VBX_OK;
}

// Find-or-create an upload's blocks.  Every block is created by k_assign, in rounds of at most as many keys as
// hand-off set 0's table has ids (the point-key buffer holds the keys, the ray list their local ids); the slots
// end in set 0's cnt.  *listed = the keys whose slots are known (a round that fails ends the listing), *err =
// that round's state error (DESIGN.md section 9: the blocks created before the pool ran out stay).
static int create_upload_blocks(vbx_ctx* c, int layer, const std::vector<uint64_t>& keys, uint64_t* listed, int* err) {
  cudaStream_t s = c->stream;
  const uint64_t m = keys.size();
  const vbx_ctx::ScratchSet& S = c->set[0];
  VBX_CUDA(c, cudaMemcpyAsync(S.pkeys0, keys.data(), m * sizeof(uint64_t), cudaMemcpyHostToDevice, s));
  // a block inserted into the ESDF layer at an index the TSDF layer does not hold occupies a slot of its own
  const uint8_t new_bits = layer == VBX_LAYER_ESDF ? kSlotNoTsdf : (uint8_t)0;
  *err = VBX_OK;
  *listed = 0;
  while (*listed < m && *err == VBX_OK) {
    const uint32_t rn = (uint32_t)std::min<uint64_t>(S.blocks.cap, m - *listed);
    VBX_CUDA(c, cudaMemsetAsync(S.d_state, 0, sizeof(ScanState), s));
    k_list_keys<<<grid_for(rn, 256), 256, 0, s>>>(S.blocks, S.pkeys0 + *listed, rn, S.ray_list + *listed, S.d_state);
    if (int rc = create_listed_blocks(c, new_bits)) return rc;
    k_slots_of<<<grid_for(rn, 256), 256, 0, s>>>(c->tab.hslot, S.touched_list, S.ray_list + *listed, rn,
                                                  reinterpret_cast<int32_t*>(S.cnt) + *listed);
    VBX_CUDA(c, cudaMemcpyAsync(S.h_state, S.d_state, sizeof(ScanState), cudaMemcpyDeviceToHost, s));
    VBX_CUDA(c, cudaStreamSynchronize(s));
    const ScanState& h = *S.h_state;
    c->n_blocks = h.n_blocks;
    if (layer == VBX_LAYER_ESDF && h.n_new) c->maybe_esdf_only = true;
    *err = check_state_errors(c, h);
    *listed += rn;
  }
  return VBX_OK;
}

// k_scatter_blocks of listed blocks [at, at + k) from the contiguous device payloads at `src`, in slices of
// kMaxGridY blocks; the flags become d_upd[b] (device, per block) or, when d_upd is null, upd_all
static int scatter_listed(vbx_ctx* c, int layer, int serialized, const void* src, uint64_t at, uint64_t k,
                          const uint8_t* d_upd, uint8_t upd_all) {
  const size_t bbytes = payload_bytes(c, layer, serialized);
  const uint32_t wpv = (layer == VBX_LAYER_TSDF) ? 3u : (serialized ? 1u : 5u);  // threads per voxel along x
  uint32_t* pool = layer == VBX_LAYER_TSDF ? reinterpret_cast<uint32_t*>(c->tab.tsdf) : reinterpret_cast<uint32_t*>(c->tab.esdf);
  uint8_t* flags = layer == VBX_LAYER_TSDF ? c->tab.slot_updated : c->tab.slot_esdf_updated;
  const int32_t* slots = reinterpret_cast<const int32_t*>(c->set[0].cnt) + at;
  for (uint64_t b0 = 0; b0 < k; b0 += kMaxGridY) {
    const uint64_t kb = std::min<uint64_t>(kMaxGridY, k - b0);
    const dim3 grid(grid_for((uint64_t)wpv * c->vox_per_block, 256), (unsigned int)kb);
    k_scatter_blocks<<<grid, 256, 0, c->stream>>>(
        layer, serialized, reinterpret_cast<const uint32_t*>(static_cast<const char*>(src) + b0 * bbytes), slots + b0,
        (uint32_t)kb, (uint32_t)c->vox_per_block, pool, d_upd ? d_upd + b0 : nullptr, upd_all, flags,
        layer == VBX_LAYER_ESDF ? c->tab.slot_has_esdf : nullptr);
    VBX_CUDA(c, cudaGetLastError());
  }
  return VBX_OK;
}

// Layer::insertBlock / allocateBlockPtrByIndex + voxel copy, or Block(BlockProto) + deserializeFromIntegers
// (core/block_inl.h:73-109) when `serialized`: find-or-create the blocks, then ONE staged copy per
// chunk and a scatter kernel.
int upload_blocks(vbx_ctx* c, int layer, const int32_t* idx3, uint64_t m, const void* voxels,
                  const uint8_t* updated_bits, int serialized) {
  if (m == 0) return VBX_OK;
  if (layer == VBX_LAYER_ESDF && !c->esdf.ready) return fail(c, VBX_E_STATE, "no ESDF layer");
  if (m > c->tab.max_blocks) return fail(c, VBX_E_CAPACITY, "more blocks than the pool holds");
  cudaStream_t s = c->stream;
  std::vector<uint64_t> keys;
  if (int rc = upload_keys(c, idx3, m, &keys)) return rc;
  if (m > c->max_points) return fail(c, VBX_E_CAPACITY, "upload more than max_points_per_scan blocks at once");
  uint64_t listed = 0;
  int err = VBX_OK;
  if (int rc = create_upload_blocks(c, layer, keys, &listed, &err)) return rc;
  // The payloads of the blocks that have slots, also when the pool ran out: every block the call created
  // holds what was uploaded for it (an ESDF block becomes one only here, by slot_has_esdf)
  const size_t bbytes = payload_bytes(c, layer, serialized);
  const uint64_t chunk = std::max<uint64_t>(1, std::min<uint64_t>(listed, (256ull << 20) / bbytes));
  if (int rc = ensure_staging(c, chunk * bbytes + chunk, chunk)) return rc;
  uint8_t* d_upd = static_cast<uint8_t*>(c->mirror.dev) + chunk * bbytes;
  for (uint64_t at = 0; at < listed; at += chunk) {
    const uint64_t k = std::min<uint64_t>(chunk, listed - at);
    VBX_CUDA(c, cudaMemcpyAsync(c->mirror.dev, static_cast<const char*>(voxels) + at * bbytes, k * bbytes,
                                cudaMemcpyHostToDevice, s));
    if (updated_bits) VBX_CUDA(c, cudaMemcpyAsync(d_upd, updated_bits + at, k, cudaMemcpyHostToDevice, s));
    if (int rc = scatter_listed(c, layer, serialized, c->mirror.dev, at, k, updated_bits ? d_upd : nullptr, 0)) return rc;
    VBX_CUDA(c, cudaStreamSynchronize(s));  // the staging buffer is reused by the next chunk
  }
  if (err) return err;
  return refresh_host_mirror(c);
}

// upload_blocks with the raw voxel payloads already in device memory: the blocks are created the same way and
// scattered straight from `d_voxels`, every written slot's flags set to `updated_bits` (reported bits only).
// k_list_keys takes packed keys, and the range and ownership checks must pass before anything is written, so
// the indices (12 B per block, never a payload byte) are read to the host once.  On a sharded engine a block
// this rank owns is refused: its copy of record is the one the integrators update here.
int upload_blocks_device(vbx_ctx* c, int layer, const int32_t* d_idx3, uint64_t m, const void* d_voxels,
                         uint8_t updated_bits) {
  if (m == 0) return VBX_OK;
  if (layer == VBX_LAYER_ESDF && !c->esdf.ready) return fail(c, VBX_E_STATE, "no ESDF layer");
  if (m > c->tab.max_blocks) return fail(c, VBX_E_CAPACITY, "more blocks than the pool holds");
  std::vector<int32_t> idx(3 * m);
  VBX_CUDA(c, cudaMemcpyAsync(idx.data(), d_idx3, 3 * m * sizeof(int32_t), cudaMemcpyDeviceToHost, c->stream));
  VBX_CUDA(c, cudaStreamSynchronize(c->stream));
  std::vector<uint64_t> keys;
  if (int rc = upload_keys(c, idx.data(), m, &keys)) return rc;
  if (c->opt.world_size > 1) {
    for (uint64_t i = 0; i < m; ++i) {
      if (block_owner(idx[3 * i], idx[3 * i + 1], idx[3 * i + 2], c->opt.world_size) == c->opt.rank) {
        return fail(c, VBX_E_INVALID, "a replica upload names a block this rank owns");
      }
    }
  }
  if (m > c->max_points) return fail(c, VBX_E_CAPACITY, "upload more than max_points_per_scan blocks at once");
  uint64_t listed = 0;
  int err = VBX_OK;
  if (int rc = create_upload_blocks(c, layer, keys, &listed, &err)) return rc;
  if (int rc = scatter_listed(c, layer, 0, d_voxels, 0, listed, nullptr, updated_bits)) return rc;
  VBX_CUDA(c, cudaStreamSynchronize(c->stream));
  if (err) return err;
  return refresh_host_mirror(c);
}

int remove_blocks(vbx_ctx* c, int layer, const int32_t* idx3, uint64_t m);

// Layer::removeAllBlocks (core/layer.h:164) of ONE layer; the other layer keeps its blocks
int clear_layer(vbx_ctx* c, int layer) {
  cudaStream_t s = c->stream;
  if (layer == VBX_LAYER_ESDF && !c->esdf.ready) return VBX_OK;
  if (c->esdf.ready && c->n_blocks) {
    // the layers share pool slots: remove this layer's block from every slot (slots that end up
    // empty are given back)
    if (int rc = refresh_host_mirror(c)) return rc;
    std::vector<int32_t> idx(3 * (size_t)c->n_blocks);
    for (uint32_t sl = 0; sl < c->n_blocks; ++sl)
      unpack3(c->host_slot_key[sl], &idx[3 * sl], &idx[3 * sl + 1], &idx[3 * sl + 2]);
    return remove_blocks(c, layer, idx.data(), c->n_blocks);
  }
  c->has_data_keys[0].clear();
  c->has_data_keys[1].clear();
  // no ESDF layer: reset the whole map
  const size_t used = (size_t)c->n_blocks * c->vox_per_block;
  c->esdf.pending_raise = c->esdf.pending_open = 0;
  c->maybe_esdf_only = false;
  VBX_CUDA(c, cudaMemsetAsync(c->tab.tsdf, 0, used * sizeof(TsdfVoxel), s));
  VBX_CUDA(c, cudaMemsetAsync(c->tab.hkeys, 0xff, (size_t)c->hcap * sizeof(uint64_t), s));
  VBX_CUDA(c, cudaMemsetAsync(c->tab.hslot, 0xff, (size_t)c->hcap * sizeof(int32_t), s));
  VBX_CUDA(c, cudaMemsetAsync(c->tab.slot_updated, 0, c->tab.max_blocks, s));
  VBX_CUDA(c, cudaMemsetAsync(c->tab.slot_esdf_updated, 0, c->tab.max_blocks, s));
  VBX_CUDA(c, cudaMemsetAsync(c->tab.slot_has_esdf, 0, c->tab.max_blocks, s));
  VBX_CUDA(c, cudaStreamSynchronize(s));
  if (int rc = set_n_blocks(c, 0)) return rc;
  c->host_slot_key.clear();
  c->host_key2slot.clear();
  return VBX_OK;
}

// One item of a removal's pool compaction: the block in slot `src`, with the halves in `clear` cleared, is
// written to slot `dst` (-1: nowhere); a src at or above the new block count is then zeroed, so that it reads
// as a freshly constructed block for its next owner.  No two items touch the same slot.
struct SlotMove {
  int32_t src, dst;
  uint32_t clear;
};
constexpr uint32_t kClearTsdf = 1u, kClearEsdf = 2u;  // (a cleared TSDF half leaves slot_updated = kSlotNoTsdf)

__global__ void k_compact_pool(Tables tab, const SlotMove* __restrict__ moves, uint32_t n_blocks, int has_esdf) {
  const SlotMove mv = moves[blockIdx.x];
  const bool zero_src = (uint32_t)mv.src >= n_blocks;
  const size_t src = (size_t)mv.src, dst = (size_t)mv.dst;
  const bool clear_t = mv.clear & kClearTsdf, clear_e = mv.clear & kClearEsdf;
  auto move = [&](uint32_t* pool, uint32_t words, bool clear) {  // words: 32-bit words per block
    for (uint32_t i = threadIdx.x; i < words; i += blockDim.x) {
      if (mv.dst >= 0) pool[dst * words + i] = clear ? 0u : pool[src * words + i];
      if (zero_src) pool[src * words + i] = 0u;
    }
  };
  move(reinterpret_cast<uint32_t*>(tab.tsdf), 3u * tab.vox_per_block, clear_t);
  if (has_esdf) move(reinterpret_cast<uint32_t*>(tab.esdf), 5u * tab.vox_per_block, clear_e);
  if (threadIdx.x != 0) return;
  if (mv.dst >= 0) {
    tab.slot_key[dst] = tab.slot_key[src];
    tab.slot_updated[dst] = clear_t ? kSlotNoTsdf : tab.slot_updated[src];
    tab.slot_esdf_updated[dst] = clear_e ? (uint8_t)0 : tab.slot_esdf_updated[src];
    tab.slot_has_esdf[dst] = clear_e ? (uint8_t)0 : tab.slot_has_esdf[src];
  }
  if (zero_src) tab.slot_updated[src] = tab.slot_esdf_updated[src] = tab.slot_has_esdf[src] = 0;
}

int remove_blocks(vbx_ctx* c, int layer, const int32_t* idx3, uint64_t m) {
  if (m == 0) return VBX_OK;
  cudaStream_t s = c->stream;
  const bool esdf = layer == VBX_LAYER_ESDF;
  // The two layers are independent in the reference (Layer::removeBlock = block_map_.erase, core/layer.h:163)
  // but share pool slots here: a slot is given back only when NEITHER layer holds a block in it.
  LayerSlots tv, ev;
  if (int rc = read_layer_slots(c, VBX_LAYER_TSDF, &tv)) return rc;
  if (int rc = read_layer_slots(c, VBX_LAYER_ESDF, &ev)) return rc;
  const LayerSlots& own = esdf ? ev : tv;
  const LayerSlots& other = esdf ? tv : ev;
  bool names_slot = false;
  for (uint64_t i = 0; i < m; ++i) {
    const uint64_t key = pack3(idx3[3 * i], idx3[3 * i + 1], idx3[3 * i + 2]);
    c->has_data_keys[esdf ? 1 : 0].erase(key);
    names_slot = names_slot || c->host_key2slot.count(key);
  }
  if (!names_slot || (esdf && !c->esdf.ready)) return VBX_OK;  // erasing a missing block is a no-op
  // queue entries of addNewRobotPosition address voxels by slot: they are dropped once the call names an
  // allocated slot, whichever layer holds it
  c->esdf.pending_raise = c->esdf.pending_open = 0;
  std::vector<int32_t> victims(m);
  own.find(idx3, m, victims.data());
  victims.erase(std::remove(victims.begin(), victims.end(), -1), victims.end());
  std::sort(victims.begin(), victims.end());
  victims.erase(std::unique(victims.begin(), victims.end()), victims.end());
  const uint32_t n0 = c->n_blocks;
  std::vector<uint32_t> clear(n0, 0), drop;  // the halves cleared per slot; the slots that become free
  for (int32_t v : victims) {
    if (!other.member[v]) {
      drop.push_back((uint32_t)v);
    } else {
      // the other layer's block stays; a TSDF half reads as never allocated from now on
      clear[v] = esdf ? kClearEsdf : kClearTsdf;
      if (!esdf) c->maybe_esdf_only = true;
    }
  }
  // The swap-remove of one victim at a time (highest first, each filled from the current last slot),
  // replayed on slot numbers: at[d] ends as the slot whose block lands in slot d.  So every block ends where
  // that removal put it (the ESDF walks its blocks in slot order, DESIGN.md section 6), every moved block
  // comes from at or above the new count and goes below it, and the moves are independent of each other.
  std::vector<uint32_t> at(n0);
  std::iota(at.begin(), at.end(), 0u);
  uint32_t n = n0;
  for (auto it = drop.rbegin(); it != drop.rend(); ++it) at[*it] = at[--n];
  std::vector<SlotMove> moves;
  for (uint32_t d = 0; d < n; ++d) {
    if (at[d] != d || clear[d]) moves.push_back({(int32_t)at[d], (int32_t)d, clear[at[d]]});
  }
  for (uint32_t v : drop) {
    if (v >= n) moves.push_back({(int32_t)v, -1, 0u});  // a freed slot that no block moves out of
  }
  if (moves.empty()) return VBX_OK;
  if (int rc = ensure_staging(c, moves.size() * sizeof(SlotMove), 0)) return rc;
  VBX_CUDA(c, cudaMemcpyAsync(c->mirror.dev, moves.data(), moves.size() * sizeof(SlotMove), cudaMemcpyHostToDevice, s));
  k_compact_pool<<<(unsigned int)moves.size(), 256, 0, s>>>(c->tab, static_cast<const SlotMove*>(c->mirror.dev), n,
                                                             c->esdf.ready ? 1 : 0);
  VBX_CUDA(c, cudaGetLastError());
  VBX_CUDA(c, cudaStreamSynchronize(s));  // (moves lives on this stack frame)
  if (drop.empty()) return VBX_OK;
  // then the hash is rebuilt from slot_key
  if (int rc = set_n_blocks(c, n)) return rc;
  if (int rc = rebuild_hash(c)) return rc;
  c->host_slot_key.clear();
  c->host_key2slot.clear();
  return refresh_host_mirror(c);
}

int read_layer_slots(vbx_ctx* c, int layer, LayerSlots* v) {
  if (int rc = refresh_host_mirror(c)) return rc;
  const uint32_t n = c->n_blocks;
  v->c = c;
  v->flags.assign(n, 0);
  v->member.assign(n, 0);
  if (n == 0 || (layer == VBX_LAYER_ESDF && !c->esdf.ready)) return VBX_OK;
  const bool tsdf = layer == VBX_LAYER_TSDF;
  VBX_CUDA(c, cudaMemcpyAsync(v->flags.data(), tsdf ? c->tab.slot_updated : c->tab.slot_esdf_updated, n,
                              cudaMemcpyDeviceToHost, c->stream));
  if (!tsdf) VBX_CUDA(c, cudaMemcpyAsync(v->member.data(), c->tab.slot_has_esdf, n, cudaMemcpyDeviceToHost, c->stream));
  VBX_CUDA(c, cudaStreamSynchronize(c->stream));
  if (tsdf) {
    for (uint32_t s = 0; s < n; ++s) v->member[s] = !(v->flags[s] & kSlotNoTsdf);
  }
  return VBX_OK;
}

std::vector<LayerSlots::Entry> LayerSlots::sorted(uint8_t select_bits, int mask) const {
  std::vector<Entry> out;
  for (uint32_t s = 0; s < member.size(); ++s) {
    if (!member[s] || (mask && !(flags[s] & select_bits & mask))) continue;
    Entry e;
    unpack3(c->host_slot_key[s], &e.x, &e.y, &e.z);
    e.slot = s;
    out.push_back(e);
  }
  std::sort(out.begin(), out.end(), [](const Entry& a, const Entry& b) {
    if (a.x != b.x) return a.x < b.x;
    if (a.y != b.y) return a.y < b.y;
    return a.z < b.z;
  });
  return out;
}

void LayerSlots::find(const int32_t* idx3, uint64_t m, int32_t* slots_out) const {
  for (uint64_t i = 0; i < m; ++i) {
    auto it = c->host_key2slot.find(pack3(idx3[3 * i], idx3[3 * i + 1], idx3[3 * i + 2]));
    slots_out[i] = (it != c->host_key2slot.end() && member[it->second]) ? it->second : -1;
  }
}

__global__ void k_keep_flag_bits(uint8_t* __restrict__ flags, uint32_t n, uint8_t keep) {
  const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s < n) flags[s] &= keep;
}

int keep_flag_bits(vbx_ctx* c, uint8_t* flags, uint8_t keep) {
  if (c->n_blocks == 0) return VBX_OK;
  k_keep_flag_bits<<<grid_for(c->n_blocks, 256), 256, 0, c->stream>>>(flags, c->n_blocks, keep);
  VBX_CUDA(c, cudaGetLastError());
  VBX_CUDA(c, cudaStreamSynchronize(c->stream));
  return VBX_OK;
}

// ------------------------------------------------------------------ incremental host mirror
// SURVEY.md section 8(f) N1: what every host consumer of the Layer does after a scan --
// getAllUpdatedBlocks(bit) (core/layer.h:194-203), read the blocks, updated().reset(bit)
// (e.g. mesh_integrator.h:168-183, esdf_integrator.cc:113-121) -- as ONE call: the dirty blocks
// are gathered into a contiguous staging buffer by a kernel, leave the device in one copy into
// page-locked memory, and their bits are cleared on the device.
__global__ void k_gather_blocks(const uint4* __restrict__ pool, const uint32_t* __restrict__ slots, uint32_t m,
                                uint32_t vec_per_block, uint4* __restrict__ out, uint8_t* __restrict__ flags,
                                uint8_t clear_mask) {
  // one CTA per (block, 1/8 of its payload): 16-byte loads, fully coalesced both ways
  const uint32_t b = blockIdx.x >> 3, part = blockIdx.x & 7u;
  if (b >= m) return;
  const uint32_t slot = slots[b];
  const uint32_t per = (vec_per_block + 7u) / 8u;
  const uint32_t lo = part * per, hi = min(vec_per_block, lo + per);
  const uint4* src = pool + (size_t)slot * vec_per_block;
  uint4* dst = out + (size_t)b * vec_per_block;
  for (uint32_t i = lo + threadIdx.x; i < hi; i += blockDim.x) dst[i] = __ldcs(src + i);
  if (part == 0 && threadIdx.x == 0 && clear_mask) flags[slot] &= (uint8_t)~clear_mask;
}

// The same for payloads that are not a multiple of 16 B (one-voxel blocks: 12 B TSDF, 20 B ESDF): one
// thread per output word, consecutive threads on consecutive words
__global__ void k_gather_words(const uint32_t* __restrict__ pool, const uint32_t* __restrict__ slots, uint32_t m,
                               uint32_t words_per_block, uint32_t* __restrict__ out, uint8_t* __restrict__ flags,
                               uint8_t clear_mask) {
  const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= (uint64_t)m * words_per_block) return;
  const uint32_t b = (uint32_t)(g / words_per_block), i = (uint32_t)(g % words_per_block);
  const uint32_t slot = slots[b];
  out[g] = __ldcs(pool + (size_t)slot * words_per_block + i);
  if (i == 0 && clear_mask) flags[slot] &= (uint8_t)~clear_mask;
}

int mirror_updated(vbx_ctx* c, int layer, int updated_mask, int clear_mask, int32_t* idx3, void* voxels,
                   uint8_t* updated_bits, uint64_t cap, uint64_t* n, int serialized) {
  cudaStream_t s = c->stream;
  *n = 0;
  if (c->n_blocks == 0) return VBX_OK;
  // the flags are one byte per block: a single small copy decides what is dirty (VBX_UPDATED_MIRROR may be
  // selected; it is not reported)
  LayerSlots view;
  if (int rc = read_layer_slots(c, layer, &view)) return rc;
  const std::vector<LayerSlots::Entry> items = view.sorted(kMirrorBits, updated_mask);
  *n = items.size();
  if (items.empty() || items.size() > cap) return VBX_OK;  // (too small a buffer: the caller grows it and retries)
  const size_t m = items.size();
  uint8_t* flags = (layer == VBX_LAYER_TSDF) ? c->tab.slot_updated : c->tab.slot_esdf_updated;
  const size_t raw_bytes = ((layer == VBX_LAYER_TSDF) ? sizeof(TsdfVoxel) : sizeof(EsdfVoxel)) * c->vox_per_block;
  const size_t bbytes = payload_bytes(c, layer, serialized);
  if (int rc = ensure_staging(c, m * bbytes, m)) return rc;
  std::vector<uint32_t> slots(m);
  for (size_t i = 0; i < m; ++i) {
    slots[i] = items[i].slot;
    if (idx3) {
      idx3[3 * i] = items[i].x;
      idx3[3 * i + 1] = items[i].y;
      idx3[3 * i + 2] = items[i].z;
    }
    if (updated_bits) updated_bits[i] = view.flags[items[i].slot] & kReportedBits;
  }
  VBX_CUDA(c, cudaMemcpyAsync(c->mirror.slots, slots.data(), m * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
  const char* pool = (layer == VBX_LAYER_TSDF) ? reinterpret_cast<const char*>(c->tab.tsdf)
                                               : reinterpret_cast<const char*>(c->tab.esdf);
  if (serialized) {
    const uint32_t tpv = (layer == VBX_LAYER_TSDF) ? 3u : 1u;
    for (size_t b0 = 0; b0 < m; b0 += kMaxGridY) {
      const size_t kb = std::min<size_t>(kMaxGridY, m - b0);
      const dim3 grid(grid_for((uint64_t)tpv * c->vox_per_block, 256), (unsigned int)kb);
      k_serialize_blocks<<<grid, 256, 0, s>>>(
          layer, reinterpret_cast<const uint32_t*>(pool), c->mirror.slots + b0, (uint32_t)kb, (uint32_t)c->vox_per_block,
          reinterpret_cast<uint32_t*>(static_cast<char*>(c->mirror.dev) + b0 * bbytes), flags,
          (uint8_t)(clear_mask & kMirrorBits));
      VBX_CUDA(c, cudaGetLastError());
    }
  } else if (raw_bytes % 16 == 0) {
    k_gather_blocks<<<(unsigned int)(m * 8), 256, 0, s>>>(reinterpret_cast<const uint4*>(pool), c->mirror.slots,
                                                           (uint32_t)m, (uint32_t)(raw_bytes / 16),
                                                           reinterpret_cast<uint4*>(c->mirror.dev), flags,
                                                           (uint8_t)(clear_mask & kMirrorBits));
    VBX_CUDA(c, cudaGetLastError());
  } else {
    k_gather_words<<<grid_for((uint64_t)m * (raw_bytes / 4), 256), 256, 0, s>>>(
        reinterpret_cast<const uint32_t*>(pool), c->mirror.slots, (uint32_t)m, (uint32_t)(raw_bytes / 4),
        static_cast<uint32_t*>(c->mirror.dev), flags, (uint8_t)(clear_mask & kMirrorBits));
    VBX_CUDA(c, cudaGetLastError());
  }
  // straight into the caller's buffer when it is page-locked (vbx_host_alloc / cudaHostRegister),
  // otherwise through the engine's page-locked staging buffer
  cudaPointerAttributes attr;
  const bool direct = voxels && cudaPointerGetAttributes(&attr, voxels) == cudaSuccess && attr.type == cudaMemoryTypeHost;
  cudaGetLastError();  // (an unregistered pointer may leave a sticky-free error code behind)
  void* dst = direct ? voxels : c->mirror.host;
  VBX_CUDA(c, cudaMemcpyAsync(dst, c->mirror.dev, m * bbytes, cudaMemcpyDeviceToHost, s));
  VBX_CUDA(c, cudaStreamSynchronize(s));
  VBX_CUDA(c, cudaGetLastError());
  if (!direct && voxels) std::memcpy(voxels, c->mirror.host, m * bbytes);
  return VBX_OK;
}

// The gather half of mirror_updated into caller-owned device memory (the payloads of one GPU's blocks handed
// to another GPU).  The ownership filter and the (x, y, z) order are taken on the host view of the slots: it is
// one flag byte per block that every layer call reads anyway, and the keys are already in the host mirror,
// whereas a device compaction would need a device sort to give the same order.  The indices travel host ->
// device; only the flag bytes come back, never a payload byte.
int gather_updated_device(vbx_ctx* c, int layer, int updated_mask, int clear_mask, int owned_only, int32_t* d_idx3,
                          void* d_voxels, uint64_t cap, uint64_t* n) {
  cudaStream_t s = c->stream;
  *n = 0;
  if (c->n_blocks == 0) return VBX_OK;
  LayerSlots view;
  if (int rc = read_layer_slots(c, layer, &view)) return rc;
  std::vector<LayerSlots::Entry> items = view.sorted(kMirrorBits, updated_mask);
  if (owned_only && c->opt.world_size > 1) {
    const int w = c->opt.world_size, r = c->opt.rank;
    items.erase(std::remove_if(items.begin(), items.end(),
                               [&](const LayerSlots::Entry& e) { return block_owner(e.x, e.y, e.z, w) != r; }),
                items.end());
  }
  *n = items.size();
  if (items.empty() || items.size() > cap) return VBX_OK;  // (too small a buffer: nothing copied or cleared)
  const size_t m = items.size();
  if (m > c->xfer.cap_slots) {
    c->xfer.own.release();
    c->xfer.cap_slots = 0;
    const size_t want = std::max<size_t>(2 * m, 1024);
    VBX_CUDA(c, c->xfer.own.dev(&c->xfer.slots, want));
    c->xfer.cap_slots = want;
  }
  std::vector<int32_t> idx(3 * m);
  std::vector<uint32_t> slots(m);
  for (size_t i = 0; i < m; ++i) {
    slots[i] = items[i].slot;
    idx[3 * i] = items[i].x;
    idx[3 * i + 1] = items[i].y;
    idx[3 * i + 2] = items[i].z;
  }
  VBX_CUDA(c, cudaMemcpyAsync(d_idx3, idx.data(), 3 * m * sizeof(int32_t), cudaMemcpyHostToDevice, s));
  VBX_CUDA(c, cudaMemcpyAsync(c->xfer.slots, slots.data(), m * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
  uint8_t* flags = (layer == VBX_LAYER_TSDF) ? c->tab.slot_updated : c->tab.slot_esdf_updated;
  const size_t raw_bytes = ((layer == VBX_LAYER_TSDF) ? sizeof(TsdfVoxel) : sizeof(EsdfVoxel)) * c->vox_per_block;
  const char* pool = (layer == VBX_LAYER_TSDF) ? reinterpret_cast<const char*>(c->tab.tsdf)
                                               : reinterpret_cast<const char*>(c->tab.esdf);
  const uint8_t clear = (uint8_t)(clear_mask & kMirrorBits);
  if (raw_bytes % 16 == 0 && reinterpret_cast<uintptr_t>(d_voxels) % 16 == 0) {
    k_gather_blocks<<<(unsigned int)(m * 8), 256, 0, s>>>(reinterpret_cast<const uint4*>(pool), c->xfer.slots,
                                                           (uint32_t)m, (uint32_t)(raw_bytes / 16),
                                                           static_cast<uint4*>(d_voxels), flags, clear);
  } else {
    k_gather_words<<<grid_for((uint64_t)m * (raw_bytes / 4), 256), 256, 0, s>>>(
        reinterpret_cast<const uint32_t*>(pool), c->xfer.slots, (uint32_t)m, (uint32_t)(raw_bytes / 4),
        static_cast<uint32_t*>(d_voxels), flags, clear);
  }
  VBX_CUDA(c, cudaGetLastError());
  VBX_CUDA(c, cudaStreamSynchronize(s));  // (idx and slots live on this stack frame)
  return VBX_OK;
}

}  // namespace vbx
