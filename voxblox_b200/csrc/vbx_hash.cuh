// Device-side access to the GPU-resident block hash (the device mirror of
// Layer<T>::block_map_, voxblox/include/voxblox/core/layer.h:30-32,292).
#pragma once

#include "vbx_engine.h"

namespace vbx {

// ------------------------------------------------------------------ block hash
// Find the hash position of a block, creating the entry if it is missing
// (allocateStorageAndGetVoxelPtr's find-or-emplace, cc:109-124, without the mutex:
// one CAS decides the winner).  Pool slots are assigned later by k_assign.
// *created: this call inserted the key (the caller lists the new entry for a pool slot).
__device__ inline uint32_t find_or_insert_block(const Tables& t, uint64_t key, bool* created, ScanState* st) {
  *created = false;
  uint32_t hp = hash64(key) & t.hmask;
  for (uint32_t probe = 0; probe <= t.hmask; ++probe) {
    const uint64_t k = *reinterpret_cast<volatile uint64_t*>(t.hkeys + hp);
    if (k == key) return hp;
    if (k == kEmptyKey) {
      const unsigned long long old = atomicCAS(reinterpret_cast<unsigned long long*>(t.hkeys + hp),
                                               (unsigned long long)kEmptyKey, (unsigned long long)key);
      if (old == kEmptyKey) {
        *created = true;
        return hp;
      }
      if (old == key) return hp;
    }
    hp = (hp + 1) & t.hmask;
  }
  atomicOr(&st->error, kErrHashFull);
  return 0xffffffffu;
}

__device__ __forceinline__ uint32_t find_block(const Tables& t, uint64_t key) {
  uint32_t hp = hash64(key) & t.hmask;
  for (uint32_t probe = 0; probe <= t.hmask; ++probe) {
    const uint64_t k = t.hkeys[hp];
    if (k == key) return hp;
    if (k == kEmptyKey) return 0xffffffffu;
    hp = (hp + 1) & t.hmask;
  }
  return 0xffffffffu;
}

__device__ __forceinline__ uint32_t ld_acquire_gpu(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// ------------------------------------------------------ scan-private block table
// A table position that a thread has claimed and not yet filled in: the thread that wins a block draws its
// id only after its claim succeeded, so a race for a block's first touch draws ONE id, however many threads
// take part.  (At voxels_per_side 1 every walk step is a new block and thousands of rays leave the sensor
// together: drawing before the claim would burn an id per racing thread, ~100x the blocks a scan touches.)
constexpr uint32_t kPendingId = 0xffffffffu;

// The local id of a block in the scan's private table (ScanBlocks), drawn from ScanState::n_touch_ids, without
// reading the block hash: blocks touched by the call get dense ids 0, 1, 2, ... (update records are keyed by
// (local id, voxel in block): a handful of bits instead of a hash position).  The first thread to meet a free
// position claims it with one CAS (kPendingId), draws an id, lists its key and position under it and then
// publishes id + 1 at the position.  A reader that meets a claimed position waits for the id, then compares
// the key listed under it.  Every id drawn names a block (ids drawn past the capacity raise kErrPoolFull and
// free the position again).
__device__ inline uint32_t scan_block_id(const ScanBlocks& b, uint64_t key, ScanState* st) {
  uint32_t pos = hash64(key) & b.mask;
  for (uint32_t probe = 0; probe <= b.mask;) {
    uint32_t v = ld_acquire_gpu(b.table + pos);
    if (v == 0u) {
      v = atomicCAS(b.table + pos, 0u, kPendingId);
      if (v == 0u) {
        const uint32_t id = atomicAdd(&st->n_touch_ids, 1u);
        if (id >= b.cap) {
          atomicOr(&st->error, kErrPoolFull);
          atomicExch(b.table + pos, 0u);
          return 0xffffffffu;
        }
        b.keys[id] = key;
        b.pos[id] = pos;
        __threadfence();  // the key is visible before the id can be found
        atomicExch(b.table + pos, id + 1u);
        return id;
      }
    }
    while (v == kPendingId) v = ld_acquire_gpu(b.table + pos);
    if (v == 0u) continue;  // (a claim that ran past the capacity was given back: try the position again)
    if (*reinterpret_cast<volatile unsigned long long*>(b.keys + (v - 1u)) == key) return v - 1u;
    pos = (pos + 1u) & b.mask;
    ++probe;
  }
  atomicOr(&st->error, kErrHashFull);
  return 0xffffffffu;
}

}  // namespace vbx
