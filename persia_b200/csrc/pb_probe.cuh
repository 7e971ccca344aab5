// pb_probe.cuh — find-or-admit in the shard's hash index, eight lanes per sign (internal; SURVEY.md §8a row A4).
// Shared by k_probe (flat id lists, pb_index.cu) and k_probe_items (a batch's distinct signs, pb_dedup.cu).
#pragma once
#include "pb_device.cuh"

namespace pb {

#ifndef PB_PROBE_BLOCKS
#define PB_PROBE_BLOCKS 5  // resident blocks per SM the probing kernels are compiled for (48 registers; 6 and 8 measured no faster)
#endif

// ------------------------------------------------------------------------------------------------
// A4 (admission part): initialise a newly admitted row, eight lanes cooperating.
// emb_entry.rs:28-68 + optim.rs:299-302.  The value stream restates rand 0.8.4 SmallRng (Xoshiro256++
// seeded through rand_core's PCG32 expansion) + UniformFloat<f32> — PARITY UNPINNED (no reference test
// asserts an initial value); the oracle carries the same restatement.
// ------------------------------------------------------------------------------------------------
static __device__ __noinline__ void init_row(const TableDev& t, const HyperDev& hy, const OptimDev& op, uint64_t seed,
                                             uint32_t row_idx, uint32_t sub) {
  // rand_core::SeedableRng::seed_from_u64 (PCG32 stream) -> 4 x u64 state
  uint64_t st = seed;
  uint32_t wds[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    st = st * 6364136223846793005ULL + 11634580027462260723ULL;
    uint32_t xs = (uint32_t)(((st >> 18) ^ st) >> 27);
    uint32_t rot = (uint32_t)(st >> 59);
    wds[k] = (xs >> rot) | (xs << ((32 - rot) & 31));
  }
  uint64_t s0 = wds[0] | ((uint64_t)wds[1] << 32), s1 = wds[2] | ((uint64_t)wds[3] << 32);
  uint64_t s2 = wds[4] | ((uint64_t)wds[5] << 32), s3 = wds[6] | ((uint64_t)wds[7] << 32);
  float* row = t.rows + (size_t)row_idx * t.stride;
  // every lane walks the whole stream (it is sequential) and keeps the elements it owns
  for (uint32_t e = 0; e < t.dim; ++e) {
    uint64_t sum = s0 + s3;
    uint64_t r = ((sum << 23) | (sum >> 41)) + s0;
    uint64_t tt = s1 << 17;
    s2 ^= s0;
    s3 ^= s1;
    s1 ^= s2;
    s0 ^= s3;
    s2 ^= tt;
    s3 = (s3 << 45) | (s3 >> 19);
    if ((e & (BUCKET - 1)) == sub) {
      uint32_t bits = ((uint32_t)(r >> 32) >> 9) | 0x3f800000u;
      float v01 = __fsub_rn(__uint_as_float(bits), 1.0f);
      row[e] = __fadd_rn(__fmul_rn(v01, hy.scale), hy.lo);
    }
  }
  float sv = (op.kind == PB_OPT_ADAGRAD || op.kind == PB_OPT_ADAGRAD_VW) ? op.init_acc : 0.0f;
  for (uint32_t e = t.dim + sub; e < t.stride; e += BUCKET) row[e] = (e < t.dim + t.state_floats) ? sv : 0.0f;
}

// ------------------------------------------------------------------------------------------------
// A4 (index part): the eight lanes of a group read one 128 B bucket per step.
//   MODE_FIND   read-only probe (inference lookup, update, get_rows)
//   MODE_TRAIN  find, refresh recency (get_refresh, eviction_map.rs:48-60), admit + initialise on miss
//               (emb_entry.rs:28-68 + optim.rs:299-302)
//   MODE_SET    find or force-admit without initialisation (set_embedding)
//   MODE_MOVE   admit an entry that moves between an HBM table and its host tier (pb_tier.cu): as MODE_SET, but the
//               row number stays unpublished (ROW_PENDING) for the caller to store once the entry is copied, and a
//               refusal is not counted as CTR_FULL (the caller counts it)
// Must be called by all 32 lanes of a warp (four groups, each with its own sign; `valid` false = no work).
// Returns, to every lane of the group, the index cell (n_cells + N_SPECIAL = the sign has no storage) and the row
// (ROW_NONE likewise).
// Invariant that makes "an empty cell in the bucket => the sign is absent" true: a sign is stored no later
// in its probe sequence than the first bucket that had an EMPTY cell when it was admitted, and between rebuilds
// a cell never returns to EMPTY: eviction leaves a tombstone, which lookups walk past and admissions reuse (after
// having seen an EMPTY cell further on, i.e. knowing the sign is absent).  A sign admitted when the shard is out of
// row storage is rolled back to a tombstone (the reference would have evicted its LRU entry; here the sweep between
// batches does), so it can be admitted again later.
// So EMPTY cells only ever get fewer: an admission whose probe path holds no tombstone uses one up, and under
// eviction churn they would run out (every admission then fails, every miss walks the whole index).  CTR_USED counts
// the normal cells that are not EMPTY; every eviction check rebuilds the index when it passes 7/8 of them
// (pb_index.cu, k_rebuild_*): live signs are re-inserted into an index of EMPTY cells, tombstones are dropped.
// ------------------------------------------------------------------------------------------------
struct ProbeOut {
  uint32_t cell, row;
};

template <int MODE>
__device__ __forceinline__ ProbeOut probe_group(const TableDev& t, const HyperDev& hy, const OptimDev& op, uint64_t sign,
                                                bool valid, uint32_t tick, uint32_t sub, uint32_t gshift) {
  const uint32_t h_none = t.n_cells + N_SPECIAL;
  uint32_t bucket = (uint32_t)(mix64(sign)) & t.bucket_mask;
  const bool special = (sign >= KEY_TOMB);  // the three signs that collide with a marker have their own cells
  const uint32_t special_cell = t.n_cells + (uint32_t)(KEY_EMPTY - sign);
  const unsigned long long stored = special ? 0ULL : sign;
  bool admit = true;
  if (MODE == MODE_TRAIN && hy.admit_p < 1.0f) {  // reference: unseeded thread_rng draw (unpinned)
    float u = (float)(mix64(sign ^ (0x9E3779B97F4A7C15ULL * (tick + 1))) >> 40) * (1.0f / 16777216.0f);
    admit = u < hy.admit_p;
  }
  uint32_t result = h_none, row_res = ROW_NONE;
  bool done = !valid;
  const uint32_t home = bucket;
  uint32_t tomb_cell = 0xFFFFFFFFu;  // first tombstone met on the probe path (admissions reuse it)
  for (uint32_t step = 0; step <= 2u * (t.bucket_mask + 1u); ++step) {
    if (!__any_sync(0xffffffffu, !done)) break;
    const bool look = !done && (!special || sub == 0);
    const uint32_t cell = special ? special_cell : bucket * BUCKET + sub;
    uint4 c = make_uint4(0xFFFFFFFEu, 0xFFFFFFFFu, ROW_PENDING, 0u);  // neither empty, tombstone nor any sign's low word pair
    if (look) c = __ldcg(reinterpret_cast<const uint4*>(t.cells + cell));
    const unsigned long long kk = (unsigned long long)c.x | ((unsigned long long)c.y << 32);
    const uint32_t mm = (__ballot_sync(0xffffffffu, look && kk == stored) >> gshift) & 0xffu;
    const uint32_t em = (__ballot_sync(0xffffffffu, look && kk == KEY_EMPTY) >> gshift) & 0xffu;
    const uint32_t tm = (__ballot_sync(0xffffffffu, look && kk == KEY_TOMB && !special) >> gshift) & 0xffu;
    const uint32_t lm = mm ? __ffs(mm) - 1 : 0;  // lane of the match
    const uint32_t mrow = __shfl_sync(0xffffffffu, c.z, gshift + lm);  // its row (may still be ROW_PENDING)
    if (!done && !mm && tm && tomb_cell == 0xFFFFFFFFu) tomb_cell = bucket * BUCKET + (__ffs(tm) - 1);
    // an EMPTY cell in this bucket (and no match so far) proves the sign absent: admit it into the first tombstone
    // seen on the way, else into the first empty cell here
    const bool try_ins = !done && !mm && em && MODE != MODE_FIND && admit;
    const bool use_tomb = try_ins && tomb_cell != 0xFFFFFFFFu;
    const uint32_t le = em ? __ffs(em) - 1 : 0;  // lane of the first free cell
    const uint32_t free_cell = special ? special_cell : (use_tomb ? tomb_cell : bucket * BUCKET + le);
    unsigned long long old = 0ULL;
    if (try_ins && sub == le) old = atomicCAS(&t.cells[free_cell].key, use_tomb ? KEY_TOMB : KEY_EMPTY, stored);
    old = __shfl_sync(0xffffffffu, old, gshift + le);
    const bool won_cas = try_ins && old == (use_tomb ? KEY_TOMB : KEY_EMPTY);  // lane `le` of this group admitted the sign
    uint32_t row = 0;
    if (won_cas && sub == le) {
      if (!use_tomb && !special) atomicAdd(&t.counters[CTR_USED], 1u);  // an EMPTY cell is used up (rollback leaves a tombstone)
      // storage: a row released by eviction if there is one, else the next never-used row
      uint32_t f = atomicSub(&t.counters[CTR_FREE], 1u);
      if (f > 0 && f <= t.capacity) {
        row = t.free_rows[f - 1];
      } else {
        atomicAdd(&t.counters[CTR_FREE], 1u);
        row = atomicAdd(&t.counters[CTR_ROWS], 1u);
      }
      if (row >= t.mapped) {  // (mapped <= capacity) a row past the backed ones is refused like a full shard's
        if (row < t.capacity) atomicAdd(&t.counters[CTR_UNMAPPED], 1u);
        else if (MODE != MODE_MOVE) atomicAdd(&t.counters[CTR_FULL], 1u);
        row = ROW_NONE;
      } else {
        atomicAdd(&t.counters[CTR_ADMIT], 1u);
        t.row_tick[row] = tick;  // recency of a fresh row
      }
      if (row == ROW_NONE) {  // no storage: give the cell back (duplicates that matched meanwhile read ROW_NONE)
        *reinterpret_cast<volatile uint32_t*>(&t.cells[free_cell].row) = row;
        __threadfence();
        *reinterpret_cast<volatile unsigned long long*>(&t.cells[free_cell].key) = special ? KEY_EMPTY : KEY_TOMB;
      } else if (MODE == MODE_SET) {
        *reinterpret_cast<volatile uint32_t*>(&t.cells[free_cell].row) = row;  // set_embedding: the caller fills the row
      }
    }
    row = __shfl_sync(0xffffffffu, row, gshift + le);
    if (MODE == MODE_TRAIN && won_cas && row != ROW_NONE) {
      // the row number is published only once all eight lanes have initialised the row: whoever finds the sign in the
      // index meanwhile (a duplicate in this launch, another requester's lookup) waits for it below instead of reading
      // a half-written row
      init_row(t, hy, op, sign, row, sub);
      __threadfence();
      __syncwarp(0xFFu << gshift);
      if (sub == le) *reinterpret_cast<volatile uint32_t*>(&t.cells[free_cell].row) = row;
    }
    if (!done) {
      if (mm) {
        result = special ? special_cell : bucket * BUCKET + lm;
        row_res = mrow;
        done = true;
      } else if (em) {
        if (!try_ins) {
          done = true;  // absent (and not admitted)
        } else if (won_cas) {
          result = (row == ROW_NONE) ? h_none : free_cell;
          row_res = row;
          done = true;
        } else if (old == stored) {  // a duplicate occurrence won the race for the same cell
          result = free_cell;
          row_res = ROW_PENDING;
          done = true;
        } else {
          // another sign took the cell (possibly this very sign took a different one): search again from home
          bucket = home;
          tomb_cell = 0xFFFFFFFFu;
        }
      } else {
        if (special) done = true;  // cannot happen: a reserved cell only ever holds its sign
        bucket = (bucket + 1) & t.bucket_mask;  // no match and no empty cell: next line
      }
    }
  }
  // a duplicate admitted concurrently: its row is published right after its CAS (no warp-level call in this loop)
  if (result != h_none && row_res == ROW_PENDING) {
    volatile uint32_t* pr = reinterpret_cast<volatile uint32_t*>(&t.cells[result].row);
    uint32_t spins = 0;
    while ((row_res = *pr) == ROW_PENDING && ++spins < (1u << 24)) {
    }
    if (row_res == ROW_PENDING) row_res = ROW_NONE;
  }
  if (row_res >= t.capacity) {  // ROW_NONE / rolled back
    row_res = ROW_NONE;
    result = h_none;
  } else if (MODE == MODE_TRAIN && sub == 0) {
    t.row_tick[row_res] = tick;  // get_refresh (a store, never a dependent load: probing is latency-bound)
  }
  ProbeOut o;
  o.cell = result;
  o.row = row_res;
  return o;
}

// Whole-index scans (eviction, checkpoint export, the tier's move) visit all n_cells + N_SPECIAL cells `i` holding `c`.
// live: the cell holds a sign with a row (a reserved cell holds 0 for its sign, KEY_EMPTY when it is free)
__device__ __forceinline__ bool cell_live(const TableDev& t, uint64_t i, const Cell& c) {
  return (i < t.n_cells ? c.key < KEY_TOMB : c.key == 0ULL) && c.row < t.capacity;
}

// the sign a live cell holds: reserved cell n_cells + k holds the marker-valued sign KEY_EMPTY - k
__device__ __forceinline__ uint64_t cell_sign(const TableDev& t, uint64_t i, const Cell& c) {
  return i < t.n_cells ? c.key : KEY_EMPTY - (i - t.n_cells);
}

}  // namespace pb
