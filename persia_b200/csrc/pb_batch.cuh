// pb_batch.cuh — bookkeeping of a batch's work lists, shared by the single-GPU forward (pb_dedup.cu) and the sharded
// requester (pb_shard.cu) (internal).
#pragma once
#include "pb_device.cuh"

namespace pb {

// the scratch set's region of a slot (k_dedup, pb_dedup.cu): linear probing from a hash over `size` cells
__device__ __forceinline__ uint32_t set_region(const SlotsDev& sl, uint32_t slot, uint32_t& size) {
  size = 2u * (sl.occ_off[slot + 1] - sl.occ_off[slot]) + 1u;  // the reserved cell (sign == KEY_EMPTY) follows
  return 2u * sl.occ_off[slot] + 2u * slot;
}

// block-level list bookkeeping shared by k_probe_items and k_route_items (pb_shard.cu): every thread of the block
// calls it once, converged.  `head`: this thread speaks for an item; cnt its multiplicity (0 = keep nothing);
// returns through the references the item's list position and the base of its occurrence list.
// One global atomic per block and list instead of one per warp (they all hit the same few words).
struct ItemSlots {
  uint32_t cls;   // 0 none, 1 cold, 2 warm, 3 hot
  uint32_t pos;   // position in the class's list
  uint32_t base;  // first entry of the occurrence list (cnt > 1)
};
// hot_nwords: words of a bitmap over the item's slot (one bit per sample); a hot item gets one from the pool when
// it fits (base = bit 31 | word offset) and an occurrence list otherwise.
__device__ __forceinline__ ItemSlots block_item_slots(const BatchDev& b, bool head, uint32_t cnt, uint32_t hot_nwords) {
  __shared__ uint32_t s_n[6], s_g[6];  // cold, warm, hot, huge, giant, occurrence-list entries
  if (threadIdx.x < 6) s_n[threadIdx.x] = 0;
  __syncthreads();
  const uint32_t lane = threadIdx.x & 31;
  ItemSlots r;
  // list: 1 cold, 2 warm, 3 hot, 4 huge, 5 giant (the long chains are numbered apart and listed from the end of `hot`:
  // the reducing kernel starts them first)
  const uint32_t list = !head || cnt == 0 ? 0u : (cnt == 1 ? 1u : (cnt <= PB_WARM_MAX ? 2u : (cnt <= PB_HUGE_MIN ? 3u : (cnt <= PB_GIANT_MIN ? 4u : 5u))));
  r.cls = list > 3u ? 3u : list;
  r.pos = r.base = 0;
  uint32_t off = 0, seg = 0;
#pragma unroll
  for (uint32_t c = 1; c <= 5; ++c) {
    const uint32_t m = __ballot_sync(0xffffffffu, list == c);
    uint32_t w = 0;
    if (m && lane == 0) w = atomicAdd(&s_n[c - 1], (uint32_t)__popc(m));
    w = __shfl_sync(0xffffffffu, w, 0);
    if (list == c) off = w + __popc(m & ((1u << lane) - 1u));
  }
  bool bitmap = false;
  uint32_t bm_off = 0;
  if (r.cls == 3 && hot_nwords && hot_nwords <= b.hot_words) {  // a few hundred per batch: one global atomic each
    bm_off = atomicAdd(&b.cnt[BC_HOTW], hot_nwords);
    bitmap = bm_off + hot_nwords <= b.hot_words;
  }
  if (r.cls >= 2 && !bitmap) seg = atomicAdd(&s_n[5], cnt);
  __syncthreads();
  if (threadIdx.x < 6 && s_n[threadIdx.x]) {
    const uint32_t which = threadIdx.x == 0 ? BC_COLD : threadIdx.x == 1 ? BC_WARM : threadIdx.x == 2 ? BC_HOT
                           : threadIdx.x == 3 ? BC_HUGE : threadIdx.x == 4 ? BC_GIANT : BC_SEG;
    s_g[threadIdx.x] = atomicAdd(&b.cnt[which], s_n[threadIdx.x]);
  }
  __syncthreads();
  if (list) r.pos = s_g[list - 1] + off;
  if (list == 5) r.pos = b.hot_cap - 1u - r.pos;  // (a batch holds at most n / PB_GIANT_MIN giants: giant_cap)
  else if (list == 4) r.pos = b.hot_cap - 1u - b.giant_cap - r.pos;
  if (r.cls >= 2) r.base = bitmap ? (0x80000000u | bm_off) : s_g[5] + seg;
  return r;
}

// what the gather needs of an occurrence's set cell: one 16 B load (target, base) + count/cursor when filing
struct OccRef {
  uint32_t row, base, count;
};
__device__ __forceinline__ OccRef occ_ref(const BatchDev& b, uint32_t cell) {
  const uint4 lo = *reinterpret_cast<const uint4*>(&b.set[cell]);           // key (2 words), count, cursor
  const uint4 hi = *(reinterpret_cast<const uint4*>(&b.set[cell]) + 1);     // target, base, first, item
  OccRef r;
  r.row = hi.x;
  r.base = hi.y;
  r.count = lo.z;
  return r;
}
__device__ __forceinline__ void file_occurrence(const BatchDev& b, const SlotsDev& sl, uint32_t cell, const OccRef& r, uint32_t occ) {
  if (r.count <= 1) return;
  if (r.base & 0x80000000u) {  // hot item in bitmap mode: one bit per sample of the slot
    const uint32_t rel = occ - sl.occ_off[slot_of_occ(sl, occ)];
    atomicOr(&b.hot_bits[(r.base & 0x7FFFFFFFu) + (rel >> 5)], 1u << (rel & 31u));
  } else {
    b.seg_occ[r.base + atomicAdd(&b.set[cell].cursor, 1u)] = occ;
  }
}
// the same for 32 consecutive occurrences at once, one per lane: occurrences of one sign share ONE atomic (a sign
// repeated thousands of times would otherwise serialise thousands of atomics on its cursor)
__device__ __forceinline__ void file_occurrences_warp(const BatchDev& b, const SlotsDev& sl, uint32_t occ, bool valid) {
  const uint32_t lane = threadIdx.x & 31;
  uint32_t cell = 0xFFFFFFFFu;
  OccRef r;
  r.row = r.base = r.count = 0;
  if (valid) {
    cell = b.occ_set[occ];
    r = occ_ref(b, cell);
    if (r.count <= 1) cell = 0xFFFFFFFFu;
  }
  // hot items in bitmap mode: the lanes of one sign AND one bitmap word OR their bits together
  uint32_t word = 0xFFFFFFFFu, bit = 0;
  if (cell != 0xFFFFFFFFu && (r.base & 0x80000000u)) {
    const uint32_t rel = occ - sl.occ_off[slot_of_occ(sl, occ)];
    word = (r.base & 0x7FFFFFFFu) + (rel >> 5);
    bit = 1u << (rel & 31u);
  }
  const uint32_t wpeers = __match_any_sync(0xffffffffu, word);
  if (word != 0xFFFFFFFFu) {
    const uint32_t bits = __reduce_or_sync(wpeers, bit);
    if (lane == (uint32_t)(__ffs(wpeers) - 1)) atomicOr(&b.hot_bits[word], bits);
    cell = 0xFFFFFFFFu;  // filed
  }
  const uint32_t peers = __match_any_sync(0xffffffffu, cell);
  if (cell == 0xFFFFFFFFu) return;
  const uint32_t leader = __ffs(peers) - 1;
  uint32_t at = 0;
  if (lane == leader) at = atomicAdd(&b.set[cell].cursor, (uint32_t)__popc(peers));
  at = __shfl_sync(peers, at, leader);
  b.seg_occ[r.base + at + __popc(peers & ((1u << lane) - 1u))] = occ;
}

}  // namespace pb
