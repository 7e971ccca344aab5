// pb_tier.cu — the host-memory tier behind an HBM table (pb_table_attach_tier, include/persia_b200.h).
//
// The tier is a second table whose rows live in mapped pinned host memory; its index cells, row_tick, free-row stack,
// counters and rebuild buffers live in HBM like any table's, so the probe, admission, sweep and rebuild code is the
// same, and every claim is a CAS on an HBM index cell (no atomic ever targets host memory).  The kernels here only move
// whole entries (embedding ++ optimizer state) between the two tables, eight lanes per sign with 16-byte accesses:
//   out      an eviction check's victims: tier row + cell claimed (MODE_MOVE), entry copied, tier cell published, and
//            only then the HBM cell tombstoned and its row freed
//   restore  before the probe of a training request (and of pb_set_rows; on R GPUs, before the owner's probe of the
//            signs its peers sent): a sign the HBM index lacks and the tier holds gets a row from the HBM free pool, its
//            entry is copied back and published (MODE_MOVE), the tier row is freed
//   in place inference lookups (on R GPUs too: k_owner_lookup_tier, pb_shard.cu), pb_update and pb_get_rows read (or
//            step) tier-held rows where they are: nothing moves, so they never depend on free HBM rows
//   stage    pb_tier_stage, one batch ahead on a stream of its own: the eviction check the next training request would
//            run, then the restores of its signs, so that request finds them in HBM and its own check and restore have
//            (usually) nothing left to do.  On R GPUs (pb_tier_stage_sharded) every rank first sends the next batch's
//            signs to their owners' stage areas (k_stage_route, pb_shard.cu); each owner runs the check and restores
//            what it received (k_tier_restore_recv<true>).  A staged row is stamped with the current batch number (age 0), so the next
//            check keeps it; a stage that finds no free row leaves the entry in the tier for the request's own restore.
// A moved entry keeps its row_tick (a staged restore excepted), and the tier ages its rows by the HBM table's batch
// number: the union of the two tables evicts least recently used first, at batch granularity.  A sign lives in at most
// one of the two tables.
#include "pb_probe.cuh"

namespace pb {

namespace {

// one entry (stride floats, a multiple of 4, 16-byte aligned rows) by the eight lanes of a group
__device__ __forceinline__ void copy_entry(float* __restrict__ dst, const float* __restrict__ src, uint32_t stride,
                                           uint32_t sub) {
  for (uint32_t e = sub * 4; e < stride; e += BUCKET * 4)
    *reinterpret_cast<float4*>(dst + e) = __ldcg(reinterpret_cast<const float4*>(src + e));
}

// releases a cell and its row: tombstone (a reserved cell: EMPTY) unless the caller's CAS already did, row onto the free stack
__device__ __forceinline__ void free_row(const TableDev& t, uint32_t cell, uint32_t row, bool key_done = false) {
  if (!key_done) *reinterpret_cast<volatile unsigned long long*>(&t.cells[cell].key) = cell < t.n_cells ? KEY_TOMB : KEY_EMPTY;
  t.cells[cell].row = ROW_PENDING;
  t.row_tick[row] = 0u;
  const uint32_t f = atomicAdd(&t.counters[CTR_FREE], 1u);
  t.free_rows[f] = row;
}

// A sign (valid: this group has one) the HBM index lacks and the tier holds is moved into a free HBM row.  Called by all
// 32 lanes of a warp.  Duplicates of a sign in one launch: the group whose CAS turns the tier cell into a tombstone
// restores it, the others leave it (the probe that follows finds it in HBM).  No free HBM row: the tier cell gets its
// sign back, the entry stays where it is and the refusal is counted; the probe's admission then finds no row either.
// STAGE (pb_tier_stage): the moved row is stamped with the current batch number instead of keeping its tier recency (age
// 0: the next check keeps it), and a want of free rows is counted as a skipped stage, not as a refused restore.
template <bool STAGE>
__device__ __forceinline__ void restore_group(const TableDev& h, const TableDev& t, const HyperDev& hy, const OptimDev& op,
                                              uint64_t sign, bool valid, uint32_t tick, uint32_t sub, uint32_t gshift) {
  const ProbeOut in_hbm = probe_group<MODE_FIND>(h, hy, op, sign, valid, tick, sub, gshift);
  valid = valid && in_hbm.cell == h.n_cells + N_SPECIAL;
  const ProbeOut in_tier = probe_group<MODE_FIND>(t, hy, op, sign, valid, tick, sub, gshift);
  valid = valid && in_tier.cell != t.n_cells + N_SPECIAL;
  const bool special = sign >= KEY_TOMB;  // a reserved cell holds 0 for its sign and goes back to EMPTY
  const unsigned long long stored = special ? 0ULL : sign;
  unsigned long long old = ~stored;
  if (valid && sub == 0) old = atomicCAS(&t.cells[in_tier.cell].key, stored, special ? KEY_EMPTY : KEY_TOMB);
  old = __shfl_sync(0xffffffffu, old, gshift);
  valid = valid && old == stored;
  const ProbeOut to = probe_group<MODE_MOVE>(h, hy, op, sign, valid, tick, sub, gshift);
  if (!valid) return;
  if (to.row == ROW_NONE) {
    if (sub == 0) {
      *reinterpret_cast<volatile unsigned long long*>(&t.cells[in_tier.cell].key) = stored;
      atomicAdd(&t.counters[STAGE ? CTR_STAGE_SKIP : CTR_TIER_REFUSED], 1u);
    }
    return;
  }
  copy_entry(h.rows + (size_t)to.row * h.stride, t.rows + (size_t)in_tier.row * t.stride, h.stride, sub);
  if (sub == 0) h.row_tick[to.row] = STAGE ? tick : t.row_tick[in_tier.row];
  __threadfence();
  __syncwarp(0xFFu << gshift);
  if (sub == 0) {
    *reinterpret_cast<volatile uint32_t*>(&h.cells[to.cell].row) = to.row;  // published: the entry is complete
    free_row(t, in_tier.cell, in_tier.row, true);  // (the CAS above tombstoned the tier cell)
    atomicAdd(&t.counters[CTR_TIER_IN], 1u);
    if (STAGE) atomicAdd(&t.counters[CTR_STAGE_IN], 1u);
  }
}

}  // namespace

template <bool PREFIX>
__global__ void __launch_bounds__(256) k_tier_restore(TableDev h, TableDev t, HyperDev hy, OptimDev op, SlotsDev sl,
                                                      const uint64_t* __restrict__ ids, uint32_t n) {
  const uint32_t tick = h.counters[CTR_TICK];
  const uint32_t i = (blockIdx.x * 256 + threadIdx.x) / BUCKET;
  const uint32_t sub = threadIdx.x % BUCKET;
  const uint32_t gshift = (threadIdx.x & 31) & ~(BUCKET - 1);
  const bool valid = i < n;
  uint64_t sign = 0ULL;
  if (valid && sub == 0) {
    sign = ids[i];
    if (PREFIX) {
      const uint64_t p = sl.prefix[slot_of_occ(sl, i)];
      if (p) sign = mod_mersenne(sign, sl.spacing_bits) + p;
    }
  }
  sign = __shfl_sync(0xffffffffu, sign, gshift);
  restore_group<false>(h, t, hy, op, sign, valid, tick, sub, gshift);
}

// pb_tier_stage: the signs of an upcoming training request (slot-prefixed here, as k_tier_restore<true> does), grid-stride
// over a fixed number of blocks.  Never admits a sign and never refreshes an HBM-resident one.  (One block per SM is all
// its small grid needs: the register budget that allows keeps it from spilling.)
__global__ void __launch_bounds__(256, 1) k_tier_stage(TableDev h, TableDev t, HyperDev hy, OptimDev op, SlotsDev sl,
                                                    const uint64_t* __restrict__ ids, uint32_t n) {
  const uint32_t tick = h.counters[CTR_TICK];
  const uint32_t sub = threadIdx.x % BUCKET;
  const uint32_t gshift = (threadIdx.x & 31) & ~(BUCKET - 1);
  constexpr uint32_t PER_BLOCK = 256u / BUCKET;
  for (uint32_t u0 = blockIdx.x * PER_BLOCK; u0 < n; u0 += gridDim.x * PER_BLOCK) {
    const uint32_t i = u0 + threadIdx.x / BUCKET;
    const bool valid = i < n;
    uint64_t sign = 0ULL;
    if (valid && sub == 0) {
      sign = ids[i];
      const uint64_t p = sl.prefix[slot_of_occ(sl, i)];
      if (p) sign = mod_mersenne(sign, sl.spacing_bits) + p;
    }
    sign = __shfl_sync(0xffffffffu, sign, gshift);
    restore_group<true>(h, t, hy, op, sign, valid, tick, sub, gshift);
  }
}

// pb_forward: over the batch's distinct (slot, sign) items, after k_dedup (their number lives on the device)
__global__ void __launch_bounds__(256) k_tier_restore_items(TableDev h, TableDev t, HyperDev hy, OptimDev op, BatchDev b) {
  const uint32_t tick = h.counters[CTR_TICK];
  const uint32_t n_items = b.cnt[BC_ITEMS];
  const uint32_t sub = threadIdx.x % BUCKET;
  const uint32_t gshift = (threadIdx.x & 31) & ~(BUCKET - 1);
  constexpr uint32_t PER_BLOCK = 256u / BUCKET;
  for (uint32_t u0 = blockIdx.x * PER_BLOCK; u0 < n_items; u0 += gridDim.x * PER_BLOCK) {
    const uint32_t u = u0 + threadIdx.x / BUCKET;
    const bool valid = u < n_items;
    uint64_t sign = 0ULL;
    if (valid && sub == 0) {
      const DCell& c = b.set[b.item_cell[u]];
      sign = (c.item >> 31) ? KEY_EMPTY : c.key;  // the scratch set's reserved cell stores 0 for the sign KEY_EMPTY
    }
    sign = __shfl_sync(0xffffffffu, sign, gshift);
    restore_group<false>(h, t, hy, op, sign, valid, tick, sub, gshift);
  }
}

// sharded training forward (PB_PHASE_SERVE), before k_owner_lookup: the R x cap signs of this owner's receive area, each
// source's up to its count.  A sign that several sources sent is restored once (the tier cell's CAS); one that finds no
// free HBM row stays in the tier, counted, and the probe that follows reads zeros for it (its gradient is a miss).
// STAGE (pb_tier_stage_sharded's SERVE): the same walk over a stage exchange's area, whose signs the sources sent one
// batch ahead; restored as k_tier_stage restores (age 0; no free row: a skipped stage, left to the forward's restore).
template <bool STAGE>
__global__ void __launch_bounds__(256) k_tier_restore_recv(TableDev h, TableDev t, HyperDev hy, OptimDev op, XchgDev x) {
  const uint32_t tick = h.counters[CTR_TICK];
  const uint32_t sub = threadIdx.x % BUCKET;
  const uint32_t gshift = (threadIdx.x & 31) & ~(BUCKET - 1);
  const uint32_t total = x.R * x.cap;
  const uint32_t* ctrl = reinterpret_cast<const uint32_t*>(x.base[x.rank]);
  const uint64_t* signs = reinterpret_cast<const uint64_t*>(x.base[x.rank] + x.off_sign);
  constexpr uint32_t PER_BLOCK = 256u / BUCKET;
  for (uint32_t j0 = blockIdx.x * PER_BLOCK; j0 < total; j0 += gridDim.x * PER_BLOCK) {
    const uint32_t j = j0 + threadIdx.x / BUCKET;
    const bool valid = j < total && j % x.cap < ctrl[XC_COUNT * PB_MAX_RANKS + j / x.cap];
    if (!__any_sync(0xffffffffu, valid)) continue;  // (warp-uniform)
    uint64_t sign = 0ULL;
    if (valid && sub == 0) sign = signs[j];
    sign = __shfl_sync(0xffffffffu, sign, gshift);
    restore_group<STAGE>(h, t, hy, op, sign, valid, tick, sub, gshift);
  }
}

// Eviction check, between the HBM threshold and the tier's sweep: the tier ages its rows by the HBM batch number, and
// must free as many rows as the HBM sweep has victims (the entries of ages >= the threshold).
__global__ void __launch_bounds__(256) k_tier_plan(TableDev h, TableDev t, const uint32_t* __restrict__ ev,
                                                   uint32_t* __restrict__ tev) {
  __shared__ uint32_t s_victims;
  if (threadIdx.x == 0) s_victims = 0;
  __syncthreads();
  const bool go = ev[2] && ev[0] != 0xFFFFFFFFu;
  uint32_t v = 0;
  for (uint32_t a = threadIdx.x; a < EV_BINS; a += blockDim.x) {
    if (go && a >= ev[0]) v += ev[3 + a];
    tev[3 + a] = 0;
  }
  atomicAdd(&s_victims, v);
  __syncthreads();
  if (threadIdx.x == 0) {
    t.counters[CTR_TICK] = h.counters[CTR_TICK];
    const uint32_t used = min(t.counters[CTR_ROWS], t.capacity);
    const uint32_t free_now = (t.capacity - used) + t.counters[CTR_FREE];
    const uint32_t victims = s_victims;
    tev[2] = victims > free_now ? 1u : 0u;
    tev[1] = victims > free_now ? victims - free_now : 0u;
    tev[0] = 0xFFFFFFFFu;
    tev[EV_MOVE] = 0u;
  }
}

// the HBM sweep's victims (the cells k_evict_sweep would release), listed for the move
__global__ void __launch_bounds__(256) k_tier_collect(TableDev h, const uint32_t* __restrict__ ev, uint32_t* __restrict__ tev,
                                                      uint64_t* __restrict__ keys, uint32_t* __restrict__ rows,
                                                      uint32_t* __restrict__ cells) {
  if (!ev[2] || ev[0] == 0xFFFFFFFFu) return;
  const uint32_t tick = h.counters[CTR_TICK], thr = ev[0];
  const uint64_t n = (uint64_t)h.n_cells + N_SPECIAL;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const Cell c = h.cells[i];
    if (!cell_live(h, i, c)) continue;
    if (tick - h.row_tick[c.row] < thr) continue;
    const uint32_t at = atomicAdd(&tev[EV_MOVE], 1u);  // < capacity: every live cell holds a row of its own
    keys[at] = cell_sign(h, i, c);
    rows[at] = c.row;
    cells[at] = (uint32_t)i;
  }
}

__global__ void __launch_bounds__(256) k_tier_move(TableDev h, TableDev t, HyperDev hy, OptimDev op,
                                                   const uint32_t* __restrict__ tev, const uint64_t* __restrict__ keys,
                                                   const uint32_t* __restrict__ rows, const uint32_t* __restrict__ cells) {
  const uint32_t tick = h.counters[CTR_TICK];
  const uint32_t n = tev[EV_MOVE];
  const uint32_t sub = threadIdx.x % BUCKET;
  const uint32_t gshift = (threadIdx.x & 31) & ~(BUCKET - 1);
  constexpr uint32_t PER_BLOCK = 256u / BUCKET;
  for (uint32_t u0 = blockIdx.x * PER_BLOCK; u0 < n; u0 += gridDim.x * PER_BLOCK) {
    const uint32_t u = u0 + threadIdx.x / BUCKET;
    const bool valid = u < n;
    const uint64_t sign = valid ? keys[u] : 0ULL;
    const ProbeOut to = probe_group<MODE_MOVE>(t, hy, op, sign, valid, tick, sub, gshift);
    if (valid) {
      const uint32_t row = rows[u];
      if (to.row != ROW_NONE) {
        copy_entry(t.rows + (size_t)to.row * t.stride, h.rows + (size_t)row * h.stride, t.stride, sub);
        if (sub == 0) t.row_tick[to.row] = h.row_tick[row];  // the entry keeps its recency
        __threadfence();
        __syncwarp(0xFFu << gshift);
        if (sub == 0) {
          *reinterpret_cast<volatile uint32_t*>(&t.cells[to.cell].row) = to.row;
          atomicAdd(&t.counters[CTR_TIER_OUT], 1u);
        }
      } else if (sub == 0) {
        atomicAdd(&t.counters[CTR_TIER_LOST], 1u);
      }
      if (sub == 0) {  // only now does the HBM copy go
        free_row(h, cells[u], row);
        atomicAdd(&h.counters[CTR_EVICT], 1u);
      }
    }
  }
}

// pb_get_rows (len = entry length) and inference pb_lookup (len = dim): what the tier holds of the signs the HBM probe
// did not find, read where it is
__global__ void __launch_bounds__(256) k_tier_get(TableDev h, TableDev t, const uint64_t* __restrict__ signs,
                                                  const uint32_t* __restrict__ occ_cell, uint32_t n, uint32_t len,
                                                  float* __restrict__ entries, uint8_t* __restrict__ found,
                                                  uint32_t* __restrict__ miss_ctr) {
  const uint32_t i = (blockIdx.x * 256 + threadIdx.x) / BUCKET;
  const uint32_t sub = threadIdx.x % BUCKET;
  const uint32_t gshift = (threadIdx.x & 31) & ~(BUCKET - 1);
  const bool valid = i < n && occ_cell[i] == h.n_cells + N_SPECIAL;
  const uint64_t sign = valid ? signs[i] : 0ULL;
  const ProbeOut r = probe_group<MODE_FIND>(t, HyperDev{}, OptimDev{}, sign, valid, 0u, sub, gshift);
  if (!valid || r.row == ROW_NONE) return;
  const float* src = t.rows + (size_t)r.row * t.stride;
  for (uint32_t e = sub; e < len; e += BUCKET) entries[(size_t)i * len + e] = src[e];
  if (found && sub == 0) found[i] = 1;
  if (miss_ctr && sub == 0) atomicSub(miss_ctr, 1u);  // the probe counted a lookup miss: the sign was found after all
}

// inference pb_forward: an item the HBM probe did not find and the tier holds is read where it is (k_gather_items<TIER>)
__global__ void __launch_bounds__(256) k_tier_find_items(TableDev h, TableDev t, BatchDev b) {
  const uint32_t n_items = b.cnt[BC_ITEMS];
  const uint32_t sub = threadIdx.x % BUCKET;
  const uint32_t gshift = (threadIdx.x & 31) & ~(BUCKET - 1);
  constexpr uint32_t PER_BLOCK = 256u / BUCKET;
  for (uint32_t u0 = blockIdx.x * PER_BLOCK; u0 < n_items; u0 += gridDim.x * PER_BLOCK) {
    const uint32_t u = u0 + threadIdx.x / BUCKET;
    uint32_t cell = 0;
    bool valid = false;
    uint64_t sign = 0ULL;
    if (u < n_items && sub == 0) {
      cell = b.item_cell[u];
      const DCell& c = b.set[cell];
      valid = c.target == ROW_NONE;
      sign = (c.item >> 31) ? KEY_EMPTY : c.key;
    }
    valid = __shfl_sync(0xffffffffu, valid, gshift);
    sign = __shfl_sync(0xffffffffu, sign, gshift);
    const ProbeOut r = probe_group<MODE_FIND>(t, HyperDev{}, OptimDev{}, sign, valid, 0u, sub, gshift);
    if (valid && sub == 0 && r.row != ROW_NONE) {
      b.set[cell].target = h.capacity + r.row;
      atomicSub(&h.counters[CTR_MISS], 1u);  // k_probe_items counted the item as a lookup miss
    }
  }
}

// inference pb_forward_raw: distinct sign u (first occurrence i) that the HBM probe did not find and the tier holds:
// table row u + 1 = f16(its tier row), rounded as k_raw_table rounds HBM rows
__global__ void __launch_bounds__(256) k_tier_raw_fill(TableDev h, TableDev t, SlotsDev sl, const uint64_t* __restrict__ ids,
                                                       uint32_t n, const uint32_t* __restrict__ occ_cell, RawWork w,
                                                       __half* __restrict__ out) {
  const uint32_t i = (blockIdx.x * 256 + threadIdx.x) / BUCKET;
  const uint32_t sub = threadIdx.x % BUCKET;
  const uint32_t gshift = (threadIdx.x & 31) & ~(BUCKET - 1);
  const bool valid = i < n && occ_cell[i] == h.n_cells + N_SPECIAL;
  uint64_t sign = 0ULL;
  if (valid) {
    sign = ids[i];
    const uint64_t p = sl.prefix[0];
    if (p) sign = mod_mersenne(sign, sl.spacing_bits) + p;
  }
  const ProbeOut r = probe_group<MODE_FIND>(t, HyperDev{}, OptimDev{}, sign, valid, 0u, sub, gshift);
  if (!valid || r.row == ROW_NONE) return;
  if (sub == 0) atomicSub(&h.counters[CTR_MISS], 1u);  // k_probe counted the occurrence as a lookup miss
  const RawCell& c = w.set[w.occ_set[i]];
  if (c.first != i) return;  // one occurrence writes the sign's row
  const float* src = t.rows + (size_t)r.row * t.stride;
  __half* o = out + (size_t)(c.rank + 1) * t.dim;
  for (uint32_t e = sub; e < t.dim; e += BUCKET) o[e] = __float2half_rn(src[e]);
}

// pb_update: the tier cell of every sign the HBM probe did not find and the tier holds (its gradient steps the tier row
// in place); else none.  The HBM update counts a gradient miss for such a sign: it is given back here.
__global__ void __launch_bounds__(256) k_tier_where(TableDev h, TableDev t, const uint64_t* __restrict__ signs,
                                                    const uint32_t* __restrict__ occ_cell, uint32_t n,
                                                    uint32_t* __restrict__ where) {
  const uint32_t i = (blockIdx.x * 256 + threadIdx.x) / BUCKET;
  const uint32_t sub = threadIdx.x % BUCKET;
  const uint32_t gshift = (threadIdx.x & 31) & ~(BUCKET - 1);
  const bool valid = i < n && occ_cell[i] == h.n_cells + N_SPECIAL;
  const uint64_t sign = valid ? signs[i] : 0ULL;
  const ProbeOut r = probe_group<MODE_FIND>(t, HyperDev{}, OptimDev{}, sign, valid, 0u, sub, gshift);
  if (i >= n || sub != 0) return;
  where[i] = valid ? r.cell : t.n_cells + N_SPECIAL;
  if (valid && r.row != ROW_NONE) atomicSub(&h.counters[CTR_GRAD_MISS], 1u);
}

// pb_set_rows: the entries the HBM table had no row for go to the tier (set_embedding beyond the HBM rows)
__global__ void __launch_bounds__(256) k_tier_set(TableDev h, TableDev t, HyperDev hy, OptimDev op,
                                                  const uint64_t* __restrict__ signs, const uint32_t* __restrict__ occ_cell,
                                                  uint32_t n, const float* __restrict__ entries) {
  const uint32_t tick = h.counters[CTR_TICK];
  const uint32_t i = (blockIdx.x * 256 + threadIdx.x) / BUCKET;
  const uint32_t sub = threadIdx.x % BUCKET;
  const uint32_t gshift = (threadIdx.x & 31) & ~(BUCKET - 1);
  const bool valid = i < n && occ_cell[i] == h.n_cells + N_SPECIAL;
  const uint64_t sign = valid ? signs[i] : 0ULL;
  const ProbeOut r = probe_group<MODE_SET>(t, hy, op, sign, valid, tick, sub, gshift);
  if (!valid) return;
  if (sub == 0) {
    // the HBM admission that failed counted CTR_FULL: the entry is stored after all, here; if the tier has no row either
    // it is dropped, counted as such (and the tier's own CTR_FULL is given back)
    atomicSub(&h.counters[CTR_FULL], 1u);
    if (r.row == ROW_NONE) {
      atomicSub(&t.counters[CTR_FULL], 1u);
      atomicAdd(&t.counters[CTR_TIER_LOST], 1u);
    }
  }
  if (r.row == ROW_NONE) return;
  const uint32_t elen = t.dim + t.state_floats;
  float* dst = t.rows + (size_t)r.row * t.stride;
  for (uint32_t e = sub; e < t.stride; e += BUCKET) dst[e] = e < elen ? entries[(size_t)i * elen + e] : 0.0f;
}

// ------------------------------------------------------------------------------------------------
// launchers (host)
// ------------------------------------------------------------------------------------------------
void launch_tier_plan(const TableDev& h, const TableDev& t, const uint32_t* ev, uint32_t* tev, cudaStream_t st) {
  PB_LAUNCH(k_tier_plan, 1, 256, 0, st, h, t, ev, tev);
}

void launch_tier_move(const TableDev& h, const TableDev& t, const HyperDev& hy, const OptimDev& op, const uint32_t* ev,
                      uint32_t* tev, uint64_t* keys, uint32_t* rows, uint32_t* cells, cudaStream_t st, uint32_t blocks) {
  PB_LAUNCH(k_tier_collect, blocks ? blocks : PB_NUM_SMS * 8, 256, 0, st, h, ev, tev, keys, rows, cells);
  PB_LAUNCH(k_tier_move, blocks ? blocks : PB_NUM_SMS * 4, 256, 0, st, h, t, hy, op, tev, keys, rows, cells);
}

void launch_tier_restore(const TableDev& h, const TableDev& t, const HyperDev& hy, const OptimDev& op, const SlotsDev& sl,
                         bool prefix, const uint64_t* ids, uint32_t n, cudaStream_t st) {
  if (!n) return;
  const uint32_t g = cdiv((uint64_t)n * BUCKET, 256);
  if (prefix) PB_LAUNCH(k_tier_restore<true>, g, 256, 0, st, h, t, hy, op, sl, ids, n);
  else PB_LAUNCH(k_tier_restore<false>, g, 256, 0, st, h, t, hy, op, sl, ids, n);
}

void launch_tier_stage(const TableDev& h, const TableDev& t, const HyperDev& hy, const OptimDev& op, const SlotsDev& sl,
                       const uint64_t* ids, uint32_t n, uint32_t blocks, cudaStream_t st) {
  if (n) PB_LAUNCH(k_tier_stage, blocks, 256, 0, st, h, t, hy, op, sl, ids, n);
}

void launch_tier_restore_items(const TableDev& h, const TableDev& t, const HyperDev& hy, const OptimDev& op,
                               const BatchDev& b, cudaStream_t st) {
  if (!b.n) return;
  uint32_t grid = cdiv((uint64_t)b.n * BUCKET, 256);  // worst case U = N
  if (grid > PB_NUM_SMS * 4u) grid = PB_NUM_SMS * 4u;
  PB_LAUNCH(k_tier_restore_items, grid, 256, 0, st, h, t, hy, op, b);
}

void launch_tier_restore_recv(const TableDev& h, const TableDev& t, const HyperDev& hy, const OptimDev& op,
                              const XchgDev& x, cudaStream_t st, uint32_t stage_blocks) {
  uint32_t grid = cdiv((uint64_t)x.R * x.cap * BUCKET, 256);
  if (stage_blocks) {
    PB_LAUNCH(k_tier_restore_recv<true>, grid < stage_blocks ? grid : stage_blocks, 256, 0, st, h, t, hy, op, x);
    return;
  }
  if (grid > PB_NUM_SMS * 4u) grid = PB_NUM_SMS * 4u;
  PB_LAUNCH(k_tier_restore_recv<false>, grid, 256, 0, st, h, t, hy, op, x);
}

void launch_tier_get(const TableDev& h, const TableDev& t, const uint64_t* signs, const uint32_t* occ_cell, uint32_t n,
                     uint32_t len, float* entries, uint8_t* found, uint32_t* miss_ctr, cudaStream_t st) {
  if (n)
    PB_LAUNCH(k_tier_get, cdiv((uint64_t)n * BUCKET, 256), 256, 0, st, h, t, signs, occ_cell, n, len, entries, found, miss_ctr);
}

void launch_tier_find_items(const TableDev& h, const TableDev& t, const BatchDev& b, cudaStream_t st) {
  if (!b.n) return;
  uint32_t grid = cdiv((uint64_t)b.n * BUCKET, 256);
  if (grid > PB_NUM_SMS * 4u) grid = PB_NUM_SMS * 4u;
  PB_LAUNCH(k_tier_find_items, grid, 256, 0, st, h, t, b);
}

void launch_tier_raw_fill(const TableDev& h, const TableDev& t, const SlotsDev& sl, const uint64_t* ids, uint32_t n,
                          const uint32_t* occ_cell, const RawWork& w, void* table_f16, cudaStream_t st) {
  if (n)
    PB_LAUNCH(k_tier_raw_fill, cdiv((uint64_t)n * BUCKET, 256), 256, 0, st, h, t, sl, ids, n, occ_cell, w,
              reinterpret_cast<__half*>(table_f16));
}

void launch_tier_where(const TableDev& h, const TableDev& t, const uint64_t* signs, const uint32_t* occ_cell, uint32_t n,
                       uint32_t* where, cudaStream_t st) {
  if (n) PB_LAUNCH(k_tier_where, cdiv((uint64_t)n * BUCKET, 256), 256, 0, st, h, t, signs, occ_cell, n, where);
}

void launch_tier_set(const TableDev& h, const TableDev& t, const HyperDev& hy, const OptimDev& op, const uint64_t* signs,
                     const uint32_t* occ_cell, uint32_t n, const float* entries, cudaStream_t st) {
  if (n) PB_LAUNCH(k_tier_set, cdiv((uint64_t)n * BUCKET, 256), 256, 0, st, h, t, hy, op, signs, occ_cell, n, entries);
}

}  // namespace pb
