// pb_dedup.cu — forward of the batched path (SURVEY.md §8a rows A0, A2, A4, A5):
//
//   k_dedup         FeatureBatch::new on the device (persia-common/src/lib.rs:45-82): per slot, the distinct signs of
//                   the batch and how often each occurs, in a scratch set kept in L2; indices_add_prefix fused in.
//   k_probe_items   batched_lookup over the DISTINCT signs only (PS mod.rs:162-262): find / refresh / admit + init,
//                   then sorts the items into the backward's work lists by multiplicity.
//   k_gather_items  lookup_batched_all_slots_postprocess for summation slots (mod.rs:486-629): every output row is
//                   the f32 sum of its occurrences' rows in sample order, optional sqrt scaling, RNE to f16; also
//                   files every occurrence of a repeated sign into that sign's occurrence list for the backward.
//   k_clear_items   returns the scratch set to all-empty (only the cells the batch used).
//
// Everything downstream of k_dedup works on U distinct signs instead of N occurrences (Criteo batches: U/N ~ 0.3), and
// nothing here depends on thread timing in a way that reaches a result: item numbers and list orders do, values do not
// (a sign's gradient is summed in ascending occurrence order whatever order its list was filled in, pb_reduce.cu).
#include "pb_batch.cuh"
#include "pb_probe.cuh"

namespace pb {

// ------------------------------------------------------------------------------------------------
// A0 + A2.  One thread per id occurrence: prefix, insert-or-find in the slot's region (linear probing, CAS on
// the key), count.  Counting and item numbering are aggregated per warp (__match_any_sync / ballot): a sign
// repeated thousands of times in a tiny-cardinality slot costs one atomic per warp, not one per occurrence.
// ------------------------------------------------------------------------------------------------
template <bool PREFIX>
__global__ void __launch_bounds__(256) k_dedup(SlotsDev sl, BatchDev b, const uint64_t* __restrict__ ids) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t lane = threadIdx.x & 31;
  const bool valid = i < b.n;
  uint32_t idx = 0xFFFFFFFFu;
  bool won = false, special_sign = false;
  // the warp's occurrences of one (slot, sign) go to the set ONCE: a tiny-cardinality slot repeats a sign thousands of
  // times, and same-address atomics serialise in L2.  (32 consecutive occurrences span at most two slots; the slot
  // number is part of the match through the prefix or, without one, through a second match on the slot.)
  uint64_t sign = 0ULL;
  uint32_t slot = 0xFFFFFFFFu;
  if (valid) {
    sign = ids[i];
    slot = slot_of_occ(sl, i);
    if (PREFIX) {
      const uint64_t p = sl.prefix[slot];
      if (p) sign = mod_mersenne(sign, sl.spacing_bits) + p;  // indices_add_prefix, mod.rs:402-429
    }
  }
  const uint32_t peers = __match_any_sync(0xffffffffu, sign) & __match_any_sync(0xffffffffu, slot);
  const uint32_t leader = __ffs(peers) - 1;
  if (valid && lane == leader) {
    uint32_t size;
    const uint32_t off = set_region(sl, slot, size);
    const bool special = sign == KEY_EMPTY;
    special_sign = special;
    const unsigned long long stored = special ? 0ULL : sign;
    idx = special ? off + size : off + __umulhi((uint32_t)(mix64(sign) >> 32), size);
    for (;;) {  // one round trip per probed cell: the CAS returns what the cell holds
      const unsigned long long old = atomicCAS(&b.set[idx].key, KEY_EMPTY, stored);
      if (old == KEY_EMPTY) {
        won = true;
        break;
      }
      if (old == stored) break;
      if (!special) idx = (idx + 1 == off + size) ? off : idx + 1;  // the region has more cells than the slot has ids
    }
    atomicAdd(&b.set[idx].count, (uint32_t)__popc(peers));
  }
  idx = __shfl_sync(0xffffffffu, idx, leader);
  if (valid) b.occ_set[i] = idx;
  // item numbers: one global atomic per BLOCK (same-address atomics with a return serialise in L2 at several cycles
  // each: one per warp — thousands on one word — was most of this kernel's time)
  __shared__ uint32_t s_won, s_base;
  if (threadIdx.x == 0) s_won = 0;
  __syncthreads();
  const uint32_t wm = __ballot_sync(0xffffffffu, won);
  uint32_t woff = 0;
  if (wm && lane == 0) woff = atomicAdd(&s_won, (uint32_t)__popc(wm));
  woff = __shfl_sync(0xffffffffu, woff, 0);
  __syncthreads();
  if (threadIdx.x == 0 && s_won) s_base = atomicAdd(&b.cnt[BC_ITEMS], s_won);
  __syncthreads();
  if (won) {
    const uint32_t u = s_base + woff + __popc(wm & ((1u << lane) - 1u));
    b.item_cell[u] = idx;
    b.set[idx].first = i;
    b.set[idx].item = u | (special_sign ? 0x80000000u : 0u);  // the reserved cell stores 0 for the sign KEY_EMPTY
  }
}

// ------------------------------------------------------------------------------------------------
// A4 over the distinct signs.  Eight lanes per item (pb_probe.cuh).  Then lane 0 of the group records where the
// sign lives, reserves the sign's occurrence list and appends the item to the list of its class:
//   cold  one occurrence (the majority): (row, that occurrence) — complete here, the gather has nothing to file
//   warm  2..PB_WARM_MAX occurrences, hot: more — (row, list base, count)
// Persistent grid: the number of items lives on the device.
// ------------------------------------------------------------------------------------------------
template <int MODE>
__global__ void __launch_bounds__(256, 4) k_probe_items(TableDev t, HyperDev hy, OptimDev op, SlotsDev slots, BatchDev b) {
  const uint32_t tick = t.counters[CTR_TICK];
  const uint32_t n_items = b.cnt[BC_ITEMS];
  const uint32_t sub = threadIdx.x % BUCKET;
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t gshift = lane & ~(BUCKET - 1);
  constexpr uint32_t PER_BLOCK = 256u / BUCKET;
  // a few blocks per SM stride over the items (their number lives on the device); whole blocks leave together
  for (uint32_t u0 = blockIdx.x * PER_BLOCK; u0 < n_items; u0 += gridDim.x * PER_BLOCK) {
    const uint32_t u = u0 + threadIdx.x / BUCKET;
    const bool valid = u < n_items;
    uint64_t sign = 0ULL;
    uint32_t cell = 0, cnt = 0, first = 0;
    if (valid && sub == 0) {
      cell = b.item_cell[u];
      const uint4 lo = *reinterpret_cast<const uint4*>(&b.set[cell]);        // key (2 words), count, cursor
      const uint4 hi = *(reinterpret_cast<const uint4*>(&b.set[cell]) + 1);  // target, base, first, item
      sign = (hi.w >> 31) ? KEY_EMPTY : ((uint64_t)lo.x | ((uint64_t)lo.y << 32));
      cnt = lo.z;
      first = hi.z;
    }
    sign = __shfl_sync(0xffffffffu, sign, gshift);
    const ProbeOut r = probe_group<MODE>(t, hy, op, sign, valid, tick, sub, gshift);
    const bool head = valid && sub == 0;
    if (MODE != MODE_TRAIN) cnt = 0;  // inference: nothing is kept for a backward
    uint32_t slot = 0, hot_nwords = 0;
    if (head && cnt > PB_WARM_MAX) {
      slot = slot_of_occ(slots, first);
      hot_nwords = (slots.occ_off[slot + 1] - slots.occ_off[slot] + 31u) / 32u;
    }
    const ItemSlots sl = block_item_slots(b, head, cnt, hot_nwords);
    if (head) {
      *(reinterpret_cast<uint2*>(&b.set[cell]) + 2) = make_uint2(r.row, sl.base);  // target, base
      if (r.row == ROW_NONE && MODE != MODE_SET) atomicAdd(&t.counters[CTR_MISS], 1u);  // index_miss_count, per distinct sign
      if (sl.cls == 1) b.cold[sl.pos] = make_uint2(r.row, first);
      else if (sl.cls == 2) b.warm[sl.pos] = make_uint4(r.row, sl.base, cnt, 0u);
      else if (sl.cls == 3) b.hot[sl.pos] = make_uint4(r.row, sl.base, cnt, slot);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// A4 + A5: gather + pool.  A group of G lanes owns output rows; lanes stride over VEC-float chunks of the
// embedding.  f32 accumulate in sample order, optional 1/sqrt(max(n,1)), RNE to f16 (mod.rs:547-579,
// persia-common lib.rs:157-161).  TRAIN: an occurrence of a repeated sign is filed into the sign's list.
// ------------------------------------------------------------------------------------------------
template <int VEC>
__device__ __forceinline__ void store_f16(__half* dst, const float (&acc)[VEC], float scale) {
  if (VEC == 4) {
    __half2 a = __floats2half2_rn(__fmul_rn(acc[0], scale), __fmul_rn(acc[VEC > 1 ? 1 : 0], scale));
    __half2 b2 = __floats2half2_rn(__fmul_rn(acc[VEC > 1 ? 2 : 0], scale), __fmul_rn(acc[VEC > 1 ? 3 : 0], scale));
    uint2 pk;
    pk.x = *reinterpret_cast<uint32_t*>(&a);
    pk.y = *reinterpret_cast<uint32_t*>(&b2);
    *reinterpret_cast<uint2*>(dst) = pk;
  } else {
    dst[0] = __float2half_rn(__fmul_rn(acc[0], scale));
  }
}

constexpr int GATHER_ITEM_ROWS = 4;  // output rows per group in the one-id-per-sample layout (independent loads in flight)

// TIER (inference with a host tier attached, pb_tier.cu): an item whose target is capacity + r reads row r of the tier
// in place, tier_rows = the tier's mapped rows (same stride), tier_cap its rows
template <int VEC, int G, bool TRAIN, bool TIER>
__global__ void __launch_bounds__(256) k_gather_items(TableDev t, SlotsDev sl, BatchDev b,
                                                      const uint32_t* __restrict__ row_off, uint32_t n_out,
                                                      uint32_t batch, __half* __restrict__ out,
                                                      const float* __restrict__ tier_rows, uint32_t tier_cap) {
  const uint32_t group = (blockIdx.x * blockDim.x + threadIdx.x) / G;
  const uint32_t lane = threadIdx.x % G;
  const uint32_t nvec = t.dim / VEC;
  if (!row_off) {
    // one occurrence per output row: GATHER_ITEM_ROWS rows per group, every stage issued for all rows before use
    if (TRAIN) {  // one occurrence per thread first: the grid has at least n_out threads
      const uint32_t gt = blockIdx.x * blockDim.x + threadIdx.x;
      if ((gt & ~31u) < n_out) file_occurrences_warp(b, sl, gt, gt < n_out);
    }
    const uint32_t r0 = group * GATHER_ITEM_ROWS;
    if (r0 >= n_out) return;
    uint32_t cell[GATHER_ITEM_ROWS];
    OccRef ref[GATHER_ITEM_ROWS];
#pragma unroll
    for (int k = 0; k < GATHER_ITEM_ROWS; ++k) cell[k] = (r0 + k < n_out) ? b.occ_set[r0 + k] : 0xFFFFFFFFu;
#pragma unroll
    for (int k = 0; k < GATHER_ITEM_ROWS; ++k) {
      if (cell[k] != 0xFFFFFFFFu) {
        ref[k] = occ_ref(b, cell[k]);
      } else {
        ref[k].row = ROW_NONE;
        ref[k].base = 0;
        ref[k].count = 0;
      }
    }
    for (uint32_t c = lane; c < nvec; c += G) {
      float v[GATHER_ITEM_ROWS][VEC];
#pragma unroll
      for (int k = 0; k < GATHER_ITEM_ROWS; ++k) {
        if (ref[k].row < t.capacity) {
          load_vec<VEC>(t.rows + (size_t)ref[k].row * t.stride + c * VEC, v[k]);
        } else if (TIER && ref[k].row - t.capacity < tier_cap) {
          load_vec<VEC>(tier_rows + (size_t)(ref[k].row - t.capacity) * t.stride + c * VEC, v[k]);
        } else {
#pragma unroll
          for (int e = 0; e < VEC; ++e) v[k][e] = 0.0f;
        }
      }
#pragma unroll
      for (int k = 0; k < GATHER_ITEM_ROWS; ++k)
        if (r0 + k < n_out) {
#pragma unroll
          for (int e = 0; e < VEC; ++e) v[k][e] = __fadd_rn(0.0f, v[k][e]);  // the EW adds into a zeroed row (mod.rs:555-561)
          store_f16<VEC>(out + (size_t)(r0 + k) * t.dim + c * VEC, v[k], 1.0f);  // 1/sqrt(max(1,1)) = 1
        }
    }
    return;
  }
  const uint32_t gid = group;
  if (gid >= n_out) return;
  const uint32_t beg = row_off[gid], end = row_off[gid + 1];
  float scale = 1.0f;
  if (batch && sl.sqrt_scaling[gid / batch]) {
    uint32_t cnt = end - beg;
    scale = __fdiv_rn(1.0f, __fsqrt_rn((float)(cnt > 1 ? cnt : 1)));
  }
  if (TRAIN && lane == 0) {
    for (uint32_t j = beg; j < end; ++j) {
      const uint32_t cell = b.occ_set[j];
      file_occurrence(b, sl, cell, occ_ref(b, cell), j);
    }
  }
  for (uint32_t c = lane; c < nvec; c += G) {
    float acc[VEC];
#pragma unroll
    for (int k = 0; k < VEC; ++k) acc[k] = 0.0f;
    for (uint32_t j = beg; j < end; ++j) {
      const uint32_t row = b.set[b.occ_set[j]].target;
      float v[VEC];
      if (row < t.capacity) load_vec<VEC>(t.rows + (size_t)row * t.stride + c * VEC, v);
      else if (TIER && row - t.capacity < tier_cap) load_vec<VEC>(tier_rows + (size_t)(row - t.capacity) * t.stride + c * VEC, v);
      else continue;
#pragma unroll
      for (int k = 0; k < VEC; ++k) acc[k] = __fadd_rn(acc[k], v[k]);
    }
    store_f16<VEC>(out + (size_t)gid * t.dim + c * VEC, acc, scale);
  }
}

// the cells the batch used go back to empty (the set is all-empty between batches)
__global__ void __launch_bounds__(256) k_clear_items(BatchDev b) {
  const uint32_t n_items = b.cnt[BC_ITEMS];
  const uint4 e0 = make_uint4(0xFFFFFFFFu, 0xFFFFFFFFu, 0u, 0u);  // key = KEY_EMPTY, count = cursor = 0
  const uint4 e1 = make_uint4(ROW_NONE, 0u, 0u, 0u);
  for (uint32_t u = blockIdx.x * blockDim.x + threadIdx.x; u < n_items; u += gridDim.x * blockDim.x) {
    uint4* c = reinterpret_cast<uint4*>(&b.set[b.item_cell[u]]);
    c[0] = e0;
    c[1] = e1;
  }
}

// a batch whose gradients never came leaves the bits its forward set in the hot-item bitmap pool
__global__ void __launch_bounds__(256) k_clear_hot_bits(BatchDev b) {
  const unsigned long long asked = *hot_words_asked(b);
  const uint32_t used = asked < b.hot_words ? (uint32_t)asked : b.hot_words;
  for (uint32_t w = blockIdx.x * blockDim.x + threadIdx.x; w < used; w += gridDim.x * blockDim.x) b.hot_bits[w] = 0u;
}

__global__ void k_fill_set(DCell* set, uint64_t n) {
  const uint4 e0 = make_uint4(0xFFFFFFFFu, 0xFFFFFFFFu, 0u, 0u);
  const uint4 e1 = make_uint4(ROW_NONE, 0u, 0u, 0u);
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    uint4* c = reinterpret_cast<uint4*>(&set[i]);
    c[0] = e0;
    c[1] = e1;
  }
}

// ------------------------------------------------------------------------------------------------
// launchers (host)
// ------------------------------------------------------------------------------------------------
void launch_fill_set(DCell* set, uint64_t n, cudaStream_t st) { PB_LAUNCH(k_fill_set, PB_NUM_SMS * 4, 256, 0, st, set, n); }

void launch_dedup(const SlotsDev& sl, const BatchDev& b, const uint64_t* ids, cudaStream_t st) {
  if (b.n) PB_LAUNCH_F(FAM_DEDUP, (k_dedup<true>), cdiv(b.n, 256), 256, 0, st, sl, b, ids);
}

void launch_probe_items(bool training, const TableDev& t, const HyperDev& hy, const OptimDev& op, const SlotsDev& sl,
                        const BatchDev& b, cudaStream_t st) {
  if (!b.n) return;
  uint32_t grid = cdiv((uint64_t)b.n * BUCKET, 256);  // worst case U = N
  if (grid > PB_NUM_SMS * 4u) grid = PB_NUM_SMS * 4u;  // the blocks stride over the items
  if (training) PB_LAUNCH_F(FAM_PROBE, (k_probe_items<MODE_TRAIN>), grid, 256, 0, st, t, hy, op, sl, b);
  else PB_LAUNCH_F(FAM_PROBE, (k_probe_items<MODE_FIND>), grid, 256, 0, st, t, hy, op, sl, b);
}

template <int VEC, bool TRAIN, bool TIER>
static void gather_items_dispatch(int G, const TableDev& t, const SlotsDev& sl, const BatchDev& b, const uint32_t* row_off,
                                  uint32_t n_out, uint32_t batch, __half* out, const float* tier_rows, uint32_t tier_cap,
                                  cudaStream_t st) {
  uint32_t grid;
#define PB_G(GG)                                                                                                  \
  case GG:                                                                                                        \
    grid = cdiv((uint64_t)(row_off ? n_out : cdiv(n_out, GATHER_ITEM_ROWS)) * GG, 256);                           \
    if (!row_off && grid < cdiv(n_out, 256)) grid = cdiv(n_out, 256);                                             \
    PB_LAUNCH_F(FAM_GATHER, (k_gather_items<VEC, GG, TRAIN, TIER>), grid, 256, 0, st, t, sl, b, row_off, n_out, batch, out, \
                tier_rows, tier_cap);                                                                              \
    break;
  switch (G) { PB_G(1) PB_G(2) PB_G(4) PB_G(8) PB_G(16) PB_G(32) }
#undef PB_G
}

void launch_gather_items(const TableDev& t, const SlotsDev& sl, const BatchDev& b, const uint32_t* row_off,
                         uint32_t n_out, uint32_t batch, bool training, void* out_f16, cudaStream_t st,
                         const float* tier_rows, uint32_t tier_cap) {
  if (!n_out) return;
  int vec, G;
  vec_group(t.dim, vec, G);
  __half* out = reinterpret_cast<__half*>(out_f16);
  const bool tier = !training && tier_rows;
  if (vec == 4) {
    if (training) gather_items_dispatch<4, true, false>(G, t, sl, b, row_off, n_out, batch, out, nullptr, 0, st);
    else if (tier) gather_items_dispatch<4, false, true>(G, t, sl, b, row_off, n_out, batch, out, tier_rows, tier_cap, st);
    else gather_items_dispatch<4, false, false>(G, t, sl, b, row_off, n_out, batch, out, nullptr, 0, st);
  } else {
    if (training) gather_items_dispatch<1, true, false>(G, t, sl, b, row_off, n_out, batch, out, nullptr, 0, st);
    else if (tier) gather_items_dispatch<1, false, true>(G, t, sl, b, row_off, n_out, batch, out, tier_rows, tier_cap, st);
    else gather_items_dispatch<1, false, false>(G, t, sl, b, row_off, n_out, batch, out, nullptr, 0, st);
  }
}

void launch_clear_hot_bits(const BatchDev& b, cudaStream_t st) { PB_LAUNCH(k_clear_hot_bits, PB_NUM_SMS, 256, 0, st, b); }

void launch_clear_items(const BatchDev& b, cudaStream_t st) {
  if (!b.n) return;
  const uint32_t full = cdiv(b.n, 256);
  PB_LAUNCH(k_clear_items, full < PB_NUM_SMS * 4u ? full : PB_NUM_SMS * 4u, 256, 0, st, b);
}

}  // namespace pb
