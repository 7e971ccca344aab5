// pb_inc.cu — the set of updated signs behind incremental updates (DESIGN.md §4 "Incremental update").
//
// The reference's parameter server hands every sign an update_gradient_mixed stepped to its incremental-update manager,
// which collects them in a HashSet<u64> and dumps their entries once it holds more than incremental_buffer_size signs
// (embedding_parameter_service/mod.rs:366-424, persia-incremental-update-manager/src/lib.rs:251-312).  A step touches
// ~2e5 distinct signs, so the set lives on the device and the training calls fill it:
//   k_inc_mark_items  pb_backward: the context's distinct (slot, sign) items whose slot was applied and that had a row;
//                     it also empties the context's scratch set (the work k_clear_items does when no set is enabled)
//   k_inc_mark_raw    pb_backward_raw: the raw slot's distinct signs that had a row, unless the NaN rule dropped them
//   k_inc_mark_signs  pb_update: the signs found in HBM or in the host tier
//   k_inc_mark_owner  the owner's side of pb_backward_sharded / pb_backward_raw_sharded: every received entry whose apply
//                     word is set and that had a row (the entries of a chain included: the set dedups)
//   k_inc_take        compacts the set into the caller's buffer and empties it, when it fits
// Every mark runs after the optimizer step it reports, on the same stream: a captured step stays one graph.
#include "pb_device.cuh"

namespace pb {

namespace {

constexpr uint32_t FULL = 0xffffffffu;

// the reserved cell of a sign that equals a marker (>= KEY_TOMB, as in the index); its `row` word is 1 while held
__device__ __forceinline__ bool inc_special(uint64_t sign) { return sign >= KEY_TOMB; }

// Where `sign` is, or would go: true = held; else `at` = the first EMPTY cell of its probe path.  The path runs from the
// first cell of the home bucket (mix64, as the index) along whole 128 B lines.  Cells only go from EMPTY to a sign while
// marks run (takes, which empty them, are ordered apart), so a sign is always found before the first EMPTY cell.
__device__ __forceinline__ bool inc_find(const IncDev& s, uint64_t sign, uint32_t& at) {
  if (inc_special(sign)) {
    at = s.n_cells + (uint32_t)(sign - KEY_TOMB);
    return __ldcg(&s.cells[at].row) == 1u;
  }
  uint32_t i = ((uint32_t)mix64(sign) & s.bucket_mask) * BUCKET;
  for (;;) {
    const unsigned long long k = __ldcg(&s.cells[i].key);
    if (k == sign) return true;
    if (k == KEY_EMPTY) {
      at = i;
      return false;
    }
    i = (i + 1u) & (s.n_cells - 1u);
  }
}

// claims `at` or the next EMPTY cell after it: true = inserted here, false = another thread inserted the sign first
__device__ __forceinline__ bool inc_claim(const IncDev& s, uint64_t sign, uint32_t at) {
  if (inc_special(sign)) return atomicCAS(&s.cells[at].row, 0u, 1u) == 0u;
  for (;;) {
    const unsigned long long old = atomicCAS(&s.cells[at].key, KEY_EMPTY, (unsigned long long)sign);
    if (old == KEY_EMPTY) return true;
    if (old == sign) return false;
    at = (at + 1u) & (s.n_cells - 1u);
  }
}

// Every lane of the warp calls it, converged; the valid lanes insert their sign.  A sign several lanes carry (slots of one
// feature group) goes to the set once.  The held count is reserved a warp at a time, with one atomic: the warp gets
// min(n, capacity - old) places (none once old >= capacity) and gives the rest back.  The first warp to overflow fills
// the set to exactly `capacity`, so whoever reads the overshoot before it is given back finds the set full anyway: the
// drops are exact, except for a claim that finds its sign inserted meanwhile by another warp (one sign racing itself
// across the slots of a feature group), whose place goes back after the others were refused.  A sign that finds no
// room is dropped and counted; a mark never blocks.
__device__ __forceinline__ void inc_insert_warp(const IncDev& s, uint64_t sign, bool valid) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t vmask = __ballot_sync(FULL, valid);
  const uint32_t peers = __match_any_sync(FULL, sign) & vmask;
  const bool lead = valid && lane == (uint32_t)(__ffs(peers) - 1);
  uint32_t at = 0;
  const bool need = lead && !inc_find(s, sign, at);
  const uint32_t m = __ballot_sync(FULL, need);
  uint32_t grant = 0;
  if (m) {
    if (lane == 0) {
      const unsigned long long n = (unsigned long long)__popc(m);
      const unsigned long long old = atomicAdd(&s.ctr[INC_HELD], n);
      const unsigned long long room = old < s.capacity ? s.capacity - old : 0ull;
      grant = (uint32_t)(room < n ? room : n);
      if (grant < n) atomicAdd(&s.ctr[INC_HELD], (unsigned long long)(-(long long)(n - grant)));
    }
    grant = __shfl_sync(FULL, grant, 0);
  }
  const uint32_t rank = __popc(m & ((1u << lane) - 1u));
  bool ins = false, back = false;
  if (need && rank < grant) {
    ins = inc_claim(s, sign, at);
    back = !ins;  // another warp inserted it meanwhile: its reservation stands, this one goes back
  }
  const uint32_t mi = __ballot_sync(FULL, ins), mb = __ballot_sync(FULL, back);
  const uint32_t md = __ballot_sync(FULL, need && rank >= grant);
  if (lane == 0) {
    if (mi) atomicAdd(&s.ctr[INC_INSERTED], (unsigned long long)__popc(mi));
    if (md) atomicAdd(&s.ctr[INC_DROPPED], (unsigned long long)__popc(md));
    if (mb) atomicAdd(&s.ctr[INC_HELD], (unsigned long long)(-(long long)__popc(mb)));
  }
}

// the last block of a mark publishes the held count to the mapped host word (pb_inc_held reads it without a sync)
__device__ __forceinline__ void inc_publish(const IncDev& s) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(&s.ctr[INC_DONE], 1ull) == gridDim.x - 1u) {
      *reinterpret_cast<volatile unsigned long long*>(s.mirror) = atomicAdd(&s.ctr[INC_HELD], 0ull);
      s.ctr[INC_DONE] = 0ull;
    }
  }
}

__device__ __forceinline__ bool slot_on(const uint32_t (&mask)[PB_MAX_SLOTS / 32], uint32_t slot) {
  return (mask[slot >> 5] >> (slot & 31u)) & 1u;
}

// pb_backward: the batch's items (item_cell) in uniform warp strides.  applied: slots with a gradient (not skipped); a
// slot whose gradient held a NaN this request (nan_tick == tick) is not applied either.  clear: the item's scratch-set
// cell goes back to empty once read (k_clear_items' work).
__global__ void __launch_bounds__(256) k_inc_mark_items(IncDev s, BatchDev b, SlotsDev sl, IncSlots on,
                                                        const uint32_t* __restrict__ tick_ptr,
                                                        const uint32_t* __restrict__ nan_tick, int clear) {
  const uint32_t n_items = b.cnt[BC_ITEMS];
  const uint32_t tick = *tick_ptr;
  const uint4 e0 = make_uint4(0xFFFFFFFFu, 0xFFFFFFFFu, 0u, 0u);
  const uint4 e1 = make_uint4(ROW_NONE, 0u, 0u, 0u);
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t u0 = blockIdx.x * blockDim.x + (threadIdx.x & ~31u); u0 < n_items; u0 += stride) {
    const uint32_t u = u0 + (threadIdx.x & 31u);
    bool valid = false;
    uint64_t sign = 0ULL;
    if (u < n_items) {
      uint4* c = reinterpret_cast<uint4*>(&b.set[b.item_cell[u]]);
      const uint4 lo = c[0];  // key (2 words), count, cursor
      const uint4 hi = c[1];  // target, base, first, item
      sign = (hi.w >> 31) ? KEY_EMPTY : ((uint64_t)lo.x | ((uint64_t)lo.y << 32));
      const uint32_t slot = slot_of_occ(sl, hi.z);
      valid = hi.x != ROW_NONE && slot_on(on.applied, slot) && nan_tick[slot] != tick;
      if (clear) {
        c[0] = e0;
        c[1] = e1;
      }
    }
    inc_insert_warp(s, sign, valid);
  }
  inc_publish(s);
}

// pb_backward_raw: the first occurrence of every distinct sign speaks for it
__global__ void __launch_bounds__(256) k_inc_mark_raw(IncDev s, RawWork w, uint32_t n, const uint32_t* __restrict__ tick_ptr,
                                                      const uint32_t* __restrict__ nan_tick) {
  const bool dropped = nan_tick[0] == *tick_ptr;  // the NaN rule dropped the whole request
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t i0 = blockIdx.x * blockDim.x + (threadIdx.x & ~31u); i0 < n; i0 += stride) {
    const uint32_t i = i0 + (threadIdx.x & 31u);
    bool valid = false;
    uint64_t sign = 0ULL;
    if (i < n && !dropped) {
      const uint32_t h = w.occ_set[i];
      const RawCell c = w.set[h];
      sign = h == w.set_mask + 1u ? KEY_EMPTY : c.key;  // the sign KEY_EMPTY owns the extra cell
      valid = c.first == i && w.target[c.rank] != ROW_NONE;
    }
    inc_insert_warp(s, sign, valid);
  }
  inc_publish(s);
}

// pb_update: occ_cell = the HBM index cell each sign was found in; where (with a tier) = its tier cell
__global__ void __launch_bounds__(256) k_inc_mark_signs(IncDev s, TableDev h, const uint64_t* __restrict__ signs,
                                                        const uint32_t* __restrict__ occ_cell, uint32_t n, TableDev t,
                                                        const uint32_t* __restrict__ where) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t i0 = blockIdx.x * blockDim.x + (threadIdx.x & ~31u); i0 < n; i0 += stride) {
    const uint32_t i = i0 + (threadIdx.x & 31u);
    bool valid = false;
    uint64_t sign = 0ULL;
    if (i < n) {
      sign = signs[i];
      const uint32_t c = occ_cell[i];
      valid = c < h.n_cells + N_SPECIAL && h.cells[c].row < h.capacity;
      if (!valid && where) {
        const uint32_t tc = where[i];
        valid = tc < t.n_cells + N_SPECIAL && t.cells[tc].row < t.capacity;
      }
    }
    inc_insert_warp(s, sign, valid);
  }
  inc_publish(s);
}

// the owner's side of a sharded backward: the step's R requests as received (sign area, own_row, apply words)
__global__ void __launch_bounds__(256) k_inc_mark_owner(IncDev s, XchgDev x, uint32_t capacity) {
  const uint32_t total = x.R * x.cap;
  const uint64_t* sg = reinterpret_cast<const uint64_t*>(x.base[x.rank] + x.off_sign);
  const uint32_t* gok = reinterpret_cast<const uint32_t*>(x.base[x.rank] + x.off_gok);
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t j0 = blockIdx.x * blockDim.x + (threadIdx.x & ~31u); j0 < total; j0 += stride) {
    const uint32_t j = j0 + (threadIdx.x & 31u);
    bool valid = false;
    uint64_t sign = 0ULL;
    if (j < total) {
      const uint32_t src = j / x.cap, k = j % x.cap;
      if (k < x.own_cnt[src] && gok[j] != 0u && x.own_row[j] < capacity) {
        valid = true;
        sign = sg[j];
      }
    }
    inc_insert_warp(s, sign, valid);
  }
  inc_publish(s);
}

// The take: when the set holds at most max_n signs, every held cell is written out (warp-aggregated cursor) and emptied
// in the same pass; otherwise nothing is touched.  *count = signs held, either way.
__global__ void __launch_bounds__(256) k_inc_take(IncDev s, uint64_t* __restrict__ out, uint32_t max_n,
                                                  uint32_t* __restrict__ count) {
  const unsigned long long held = s.ctr[INC_HELD];
  if (blockIdx.x == 0 && threadIdx.x == 0) *count = (uint32_t)held;
  if (held > max_n) return;
  const uint32_t total = s.n_cells + N_SPECIAL;
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t i0 = blockIdx.x * blockDim.x + (threadIdx.x & ~31u); i0 < total; i0 += stride) {
    const uint32_t i = i0 + lane;
    bool have = false;
    uint64_t sign = 0ULL;
    if (i < s.n_cells) {
      sign = s.cells[i].key;
      have = sign != KEY_EMPTY;
      if (have) s.cells[i].key = KEY_EMPTY;
    } else if (i < total) {
      have = s.cells[i].row == 1u;
      sign = KEY_TOMB + (i - s.n_cells);
      if (have) s.cells[i].row = 0u;
    }
    const uint32_t m = __ballot_sync(FULL, have);
    if (!m) continue;
    unsigned long long base = 0;
    if (lane == 0) base = atomicAdd(&s.ctr[INC_CURSOR], (unsigned long long)__popc(m));
    base = __shfl_sync(FULL, base, 0);
    const unsigned long long at = base + __popc(m & ((1u << lane) - 1u));
    if (have && at < max_n) out[at] = sign;  // (cells beyond the count: a mark not ordered with this take; never written)
  }
}

__global__ void k_inc_take_end(IncDev s, uint32_t max_n) {
  const unsigned long long held = s.ctr[INC_HELD];
  if (held > max_n) return;
  s.ctr[INC_TAKEN] += held;
  s.ctr[INC_HELD] = 0ull;
  s.ctr[INC_CURSOR] = 0ull;
  *reinterpret_cast<volatile unsigned long long*>(s.mirror) = 0ull;
}

__global__ void k_inc_fill(IncDev s) {
  const uint32_t total = s.n_cells + N_SPECIAL;
  Cell e;
  e.key = KEY_EMPTY;
  e.row = 0u;
  e.aux = 0u;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) s.cells[i] = e;
  if (blockIdx.x == 0 && threadIdx.x < INC_WORDS) s.ctr[threadIdx.x] = 0ull;
}

// a persistent grid for n work items (at most four blocks per SM: a mark runs after the step, on a short list)
uint32_t mark_grid(uint64_t n) {
  const uint32_t g = cdiv(n ? n : 1, 256);
  return g < PB_NUM_SMS * 4u ? g : PB_NUM_SMS * 4u;
}

}  // namespace

void launch_inc_fill(const IncDev& s, cudaStream_t st) { PB_LAUNCH(k_inc_fill, PB_NUM_SMS * 4, 256, 0, st, s); }

void launch_inc_mark_items(const IncDev& s, const BatchDev& b, const SlotsDev& sl, const IncSlots& on,
                           const uint32_t* tick, const uint32_t* nan_tick, bool clear, cudaStream_t st) {
  PB_LAUNCH(k_inc_mark_items, mark_grid(b.n), 256, 0, st, s, b, sl, on, tick, nan_tick, clear ? 1 : 0);
}

void launch_inc_mark_raw(const IncDev& s, const RawWork& w, uint32_t n, const uint32_t* tick, const uint32_t* nan_tick,
                         cudaStream_t st) {
  PB_LAUNCH(k_inc_mark_raw, mark_grid(n), 256, 0, st, s, w, n, tick, nan_tick);
}

void launch_inc_mark_signs(const IncDev& s, const TableDev& h, const uint64_t* signs, const uint32_t* occ_cell,
                           uint32_t n, const TableDev& t, const uint32_t* where, cudaStream_t st) {
  PB_LAUNCH(k_inc_mark_signs, mark_grid(n), 256, 0, st, s, h, signs, occ_cell, n, t, where);
}

void launch_inc_mark_owner(const IncDev& s, const XchgDev& x, uint32_t capacity, cudaStream_t st) {
  PB_LAUNCH(k_inc_mark_owner, mark_grid((uint64_t)x.R * x.cap), 256, 0, st, s, x, capacity);
}

void launch_inc_take(const IncDev& s, uint64_t* out, uint32_t max_n, uint32_t* count, cudaStream_t st) {
  PB_LAUNCH(k_inc_take, mark_grid((uint64_t)s.n_cells + N_SPECIAL), 256, 0, st, s, out, max_n, count);
  PB_LAUNCH(k_inc_take_end, 1, 1, 0, st, s, max_n);
}

}  // namespace pb
