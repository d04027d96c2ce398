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

__device__ inline uint32_t ensure_block(const Tables& t, uint64_t key, ScanState* st) {
  bool created;
  const uint32_t hp = find_or_insert_block(t, key, &created, st);
  if (created) {
    const uint32_t j = atomicAdd(&st->n_new, 1u);
    if (j < t.max_blocks) {
      t.new_list[j] = hp;
    } else {
      atomicOr(&st->error, kErrPoolFull);
    }
  }
  return hp;
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

// Blocks touched by the current call get dense ids 0, 1, 2, ... (update records are keyed by
// (touched id, voxel in block): a handful of bits instead of a hash position).  The per-position
// word packs (call id, touched id); the first toucher of a block in this call installs it with one
// CAS.  A thread that loses the CAS race has drawn an id nobody uses: it is marked as a hole in
// touched_list (0xffffffff) -- ids stay dense enough, n_touched counts the blocks exactly.
__device__ __forceinline__ uint32_t touch_block(const Tables& t, uint32_t hp, uint32_t epoch, ScanState* st) {
  unsigned long long* w = t.htouch + hp;
  const unsigned long long cur = *reinterpret_cast<volatile unsigned long long*>(w);
  if ((uint32_t)(cur >> 32) == epoch) return (uint32_t)cur;
  const uint32_t id = atomicAdd(&st->n_touch_ids, 1u);
  if (id >= t.touched_cap) {
    atomicOr(&st->error, kErrPoolFull);
    return 0u;
  }
  const unsigned long long want = ((unsigned long long)epoch << 32) | id;
  const unsigned long long old = atomicCAS(w, cur, want);
  if (old == cur) {
    t.touched_list[id] = hp;
    atomicAdd(&st->n_touched, 1u);
    return id;
  }
  t.touched_list[id] = 0xffffffffu;  // a hole
  return (uint32_t)old;              // (only this call's walk writes these words: the winner carries this call's id)
}

// ------------------------------------------------------ scan-private block table
// The local id of a block in the scan's private table (ScanBlocks), drawn from the same counter and installed
// the same way as touch_block's ids, without reading the block hash: an id is drawn and its key written to
// the block list first, then one CAS installs (id + 1) at a free position.  A reader that meets an occupied
// position compares the key listed under its id (published before the CAS).  A thread whose key another
// thread installed first leaves its drawn id as a hole (key 0; a block index packs to a non-zero key).
__device__ __forceinline__ uint32_t ld_acquire_gpu(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

__device__ inline uint32_t scan_block_id(const ScanBlocks& b, uint64_t key, ScanState* st) {
  uint32_t pos = hash64(key) & b.mask;
  uint32_t drawn = 0xffffffffu;
  for (uint32_t probe = 0; probe <= b.mask; ++probe) {
    uint32_t v = ld_acquire_gpu(b.table + pos);
    if (v == 0u) {
      if (drawn == 0xffffffffu) {
        drawn = atomicAdd(&st->n_touch_ids, 1u);
        if (drawn >= b.cap) {
          atomicOr(&st->error, kErrPoolFull);
          return 0xffffffffu;
        }
        b.keys[drawn] = key;
        __threadfence();  // the key is visible before the id can be found
      }
      v = atomicCAS(b.table + pos, 0u, drawn + 1u);
      if (v == 0u) {
        b.pos[drawn] = pos;
        return drawn;
      }
      __threadfence();  // (the winner's key was published before its CAS)
    }
    if (*reinterpret_cast<volatile unsigned long long*>(b.keys + (v - 1u)) == key) {
      if (drawn != 0xffffffffu) b.keys[drawn] = 0ull;  // a hole
      return v - 1u;
    }
    pos = (pos + 1u) & b.mask;
  }
  if (drawn != 0xffffffffu) b.keys[drawn] = 0ull;
  atomicOr(&st->error, kErrHashFull);
  return 0xffffffffu;
}

}  // namespace vbx
