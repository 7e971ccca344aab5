// pb_index.cu — the shard's hash index and row store behind the single-request entry points (pb_lookup, pb_update,
// pb_set_rows, pb_get_rows), capacity sweeps, checkpoint export and the small id-preprocessing kernels (A2, A3 hash).
// The batched path is pb_dedup.cu (forward) + pb_reduce.cu (backward).
#include "pb_probe.cuh"

namespace pb {

// A2 + A4 over a flat list of ids (pb_lookup / pb_update / pb_set_rows / pb_get_rows, raw slots): eight lanes per id,
// see pb_probe.cuh.  Output: the index cell of every id (n_cells + N_SPECIAL when the sign has no storage).
template <int MODE, bool PREFIX>
__global__ void __launch_bounds__(256, PB_PROBE_BLOCKS) k_probe(TableDev t, HyperDev hy, OptimDev op, SlotsDev sl,
                                               const uint64_t* __restrict__ ids, uint32_t n,
                                               uint32_t* __restrict__ occ_cell) {
  const uint32_t tick = t.counters[CTR_TICK];
  const uint32_t i = (blockIdx.x * 256 + threadIdx.x) / BUCKET;
  const uint32_t sub = threadIdx.x % BUCKET;
  const uint32_t gshift = (threadIdx.x & 31) & ~(BUCKET - 1);  // this group's bit offset in a warp ballot
  const bool valid = i < n;
  // lane 0 of the group derives the sign (prefix arithmetic); the other seven take it by shuffle
  uint64_t sign = 0ULL;
  if (valid && sub == 0) {
    sign = ids[i];
    if (PREFIX) {
      uint64_t p = sl.prefix[slot_of_occ(sl, i)];
      if (p) sign = mod_mersenne(sign, sl.spacing_bits) + p;  // indices_add_prefix, mod.rs:402-429
    }
  }
  sign = __shfl_sync(0xffffffffu, sign, gshift);
  const ProbeOut r = probe_group<MODE>(t, hy, op, sign, valid, tick, sub, gshift);
  if (valid && sub == 0) {
    if (MODE != MODE_SET && r.cell == t.n_cells + N_SPECIAL) atomicAdd(&t.counters[CTR_MISS], 1u);
    occ_cell[i] = r.cell;
  }
}

// ------------------------------------------------------------------------------------------------
// pb_lookup's gather: one resident row per sign, plain f32 (lookup_mixed returns the f32 rows, PS mod.rs:344-357).
// GATHER_ROWS rows per lane group, every stage issued for all rows before use.
// ------------------------------------------------------------------------------------------------
constexpr int GATHER_ROWS = 4;

template <int VEC, int G>
__global__ void __launch_bounds__(256) k_gather_rows(TableDev t, const uint32_t* __restrict__ occ_cell, uint32_t n_out,
                                                     float* __restrict__ out) {
  const uint32_t group = (blockIdx.x * blockDim.x + threadIdx.x) / G;
  const uint32_t lane = threadIdx.x % G;
  const uint32_t nvec = t.dim / VEC;
  const uint32_t r0 = group * GATHER_ROWS;
  if (r0 >= n_out) return;
  uint32_t cell[GATHER_ROWS], row[GATHER_ROWS];
#pragma unroll
  for (int k = 0; k < GATHER_ROWS; ++k) cell[k] = (r0 + k < n_out) ? occ_cell[r0 + k] : 0xFFFFFFFFu;
#pragma unroll
  for (int k = 0; k < GATHER_ROWS; ++k) row[k] = (cell[k] < t.n_cells + N_SPECIAL) ? t.cells[cell[k]].row : ROW_NONE;
  for (uint32_t c = lane; c < nvec; c += G) {
    float v[GATHER_ROWS][VEC];
#pragma unroll
    for (int k = 0; k < GATHER_ROWS; ++k) {
      if (row[k] < t.capacity) {
        load_vec<VEC>(t.rows + (size_t)row[k] * t.stride + c * VEC, v[k]);
      } else {
#pragma unroll
        for (int e = 0; e < VEC; ++e) v[k][e] = 0.0f;
      }
    }
#pragma unroll
    for (int k = 0; k < GATHER_ROWS; ++k)
      if (r0 + k < n_out) store_vec<VEC>(out + (size_t)(r0 + k) * t.dim + c * VEC, v[k]);
  }
}

// set_embedding / get_rows: whole entries (emb ++ state), one group per sign.
template <bool WRITE>
__global__ void __launch_bounds__(256) k_copy_entries(TableDev t, const uint32_t* __restrict__ occ_cell, uint32_t n,
                                                      float* __restrict__ entries, uint8_t* __restrict__ found) {
  uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= n) return;
  uint32_t h = occ_cell[warp];
  uint32_t elen = t.dim + t.state_floats;
  uint32_t row = (h < t.n_cells + N_SPECIAL) ? t.cells[h].row : ROW_NONE;
  bool ok = row < t.capacity;
  if (!WRITE && found && lane == 0) found[warp] = ok ? 1 : 0;
  float* e = entries + (size_t)warp * elen;
  if (WRITE) {
    if (!ok) return;
    float* dst = t.rows + (size_t)row * t.stride;
    for (uint32_t i = lane; i < t.stride; i += 32) dst[i] = (i < elen) ? e[i] : 0.0f;
  } else {
    const float* src = t.rows + (size_t)row * t.stride;
    for (uint32_t i = lane; i < elen; i += 32) e[i] = ok ? src[i] : 0.0f;
  }
}

// CSR row offsets -> output row of every occurrence (multi-id slots)
__global__ void __launch_bounds__(256) k_expand_rows(const uint32_t* __restrict__ row_off, uint32_t n_out,
                                                     uint32_t* __restrict__ occ_outrow) {
  uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_out) return;
  for (uint32_t j = row_off[r]; j < row_off[r + 1]; ++j) occ_outrow[j] = r;
}

__global__ void __launch_bounds__(256) k_add_prefix(SlotsDev sl, const uint64_t* __restrict__ ids, uint32_t n,
                                                    uint64_t* __restrict__ out) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint64_t p = sl.prefix[slot_of_occ(sl, i)];
  uint64_t v = ids[i];
  out[i] = p ? mod_mersenne(v, sl.spacing_bits) + p : v;
}

__global__ void __launch_bounds__(256) k_shard_of(const uint64_t* __restrict__ signs, uint32_t n, uint32_t R,
                                                  uint32_t* __restrict__ shard, uint64_t* __restrict__ hash) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint64_t h = farmhash64_u64(signs[i]);
  if (shard) shard[i] = (uint32_t)(h % R);
  if (hash) hash[i] = h;
}

// Opens a training request on the device: bumps the table's batch number (recency, leader election) and the
// context's own request number, by which the backward of this batch recognises its NaN marks.  The latter never
// repeats within a context, whatever tables it serves and whenever they are cleared.
__global__ void k_begin_batch(uint32_t* counters, uint32_t* ctx_tick, uint32_t* batch_cnt, int bump) {
  if (threadIdx.x == 0 && bump) {
    counters[CTR_TICK] = counters[CTR_TICK] + 1;
    if (ctx_tick) *ctx_tick = *ctx_tick + 1;
  }
  if (batch_cnt)  // list lengths and work cursors of the batch context
    for (uint32_t i = threadIdx.x; i < BC_COUNT; i += blockDim.x) batch_cnt[i] = 0;
}

__global__ void k_fill_cells(Cell* cells, uint64_t n) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  Cell e;
  e.key = KEY_EMPTY;
  e.row = ROW_PENDING;
  e.aux = 0;
  for (; i < n; i += stride) cells[i] = e;
}

// ------------------------------------------------------------------------------------------------
// Capacity: the reference's EvictionMap drops the least recently used entry whenever an insert pushes it over
// capacity (eviction_map.rs:76-97).  Here recency is the batch number kept in row_tick and
// eviction is a sweep run between batches when free storage is low: (1) histogram of row ages over the occupied
// cells, (2) the age threshold that releases `want` rows (never rows touched in the last `keep` batches),
// (3) tombstone those cells and push their rows on the free stack.  ev[0] = threshold age, ev[1] = want,
// ev[2] = go flag, ev[3..] = age histogram (EV_BINS bins, last bin = older).
// ------------------------------------------------------------------------------------------------
constexpr uint32_t EV_BINS = 1024;
__global__ void k_evict_plan(TableDev t, uint32_t low_water, uint32_t target_free, uint32_t* __restrict__ ev) {
  // one block: decide whether a sweep is needed and clear the histogram
  uint32_t used = min(t.counters[CTR_ROWS], t.capacity);
  uint32_t free_now = (t.capacity - used) + t.counters[CTR_FREE];
  bool go = free_now < low_water;
  for (uint32_t i = threadIdx.x; i < EV_BINS; i += blockDim.x) ev[3 + i] = 0;
  if (threadIdx.x == 0) {
    ev[2] = go ? 1u : 0u;
    ev[1] = go ? (target_free > free_now ? target_free - free_now : 0u) : 0u;
    ev[0] = 0xFFFFFFFFu;
  }
}

__global__ void __launch_bounds__(256) k_evict_hist(TableDev t, uint32_t* __restrict__ ev) {
  if (!ev[2]) return;
  const uint32_t tick = t.counters[CTR_TICK];
  const uint64_t n = (uint64_t)t.n_cells + N_SPECIAL;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    Cell c = t.cells[i];
    bool occupied = (i < t.n_cells) ? (c.key < KEY_TOMB) : (c.key == 0ULL);
    if (!occupied || c.row >= t.capacity) continue;
    uint32_t age = tick - t.row_tick[c.row];
    atomicAdd(&ev[3 + min(age, EV_BINS - 1)], 1u);
  }
}

__global__ void k_evict_threshold(uint32_t keep, uint32_t* __restrict__ ev) {
  if (threadIdx.x || !ev[2]) return;
  uint32_t want = ev[1], got = 0, thr = 0xFFFFFFFFu;
  for (uint32_t a = EV_BINS; a-- > 0 && a > keep;) {  // oldest first; ages <= keep are protected
    got += ev[3 + a];
    thr = a;
    if (got >= want) break;
  }
  ev[0] = got ? thr : 0xFFFFFFFFu;
}

__global__ void __launch_bounds__(256) k_evict_sweep(TableDev t, uint32_t* __restrict__ ev) {
  if (!ev[2] || ev[0] == 0xFFFFFFFFu) return;
  const uint32_t tick = t.counters[CTR_TICK], thr = ev[0];
  const uint64_t n = (uint64_t)t.n_cells + N_SPECIAL;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    Cell c = t.cells[i];
    bool occupied = (i < t.n_cells) ? (c.key < KEY_TOMB) : (c.key == 0ULL);
    if (!occupied || c.row >= t.capacity) continue;
    uint32_t age = tick - t.row_tick[c.row];
    if (age < thr) continue;
    t.cells[i].key = (i < t.n_cells) ? KEY_TOMB : KEY_EMPTY;  // reserved cells have no probe chain behind them
    t.cells[i].row = ROW_PENDING;
    t.row_tick[c.row] = 0u;
    uint32_t f = atomicAdd(&t.counters[CTR_FREE], 1u);
    t.free_rows[f] = c.row;
    atomicAdd(&t.counters[CTR_EVICT], 1u);
  }
}

// the same sweep for a table backed by a host tier (pb_table_spill): every released row is first written out — sign
// and whole entry (embedding ++ optimizer state) — and only the victims that fit the caller's buffers are released
__global__ void __launch_bounds__(256) k_evict_sweep_spill(TableDev t, uint32_t* __restrict__ ev, uint64_t* __restrict__ signs,
                                                           float* __restrict__ entries, uint32_t max_n,
                                                           uint32_t* __restrict__ count) {
  if (!ev[2] || ev[0] == 0xFFFFFFFFu) return;
  const uint32_t tick = t.counters[CTR_TICK], thr = ev[0];
  const uint64_t n = (uint64_t)t.n_cells + N_SPECIAL;
  const uint32_t entry_len = t.dim + t.state_floats;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    Cell c = t.cells[i];
    bool occupied = (i < t.n_cells) ? (c.key < KEY_TOMB) : (c.key == 0ULL);
    if (!occupied || c.row >= t.capacity) continue;
    uint32_t age = tick - t.row_tick[c.row];
    if (age < thr) continue;
    const uint32_t at = atomicAdd(count, 1u);
    if (at >= max_n) continue;  // no room to write it out: it stays resident (count tells the caller)
    signs[at] = (i < t.n_cells) ? c.key : KEY_EMPTY;  // (the reserved cell holds the sign KEY_EMPTY)
    const float* row = t.rows + (size_t)c.row * t.stride;
    for (uint32_t e = 0; e < entry_len; ++e) entries[(size_t)at * entry_len + e] = row[e];
    t.cells[i].key = (i < t.n_cells) ? KEY_TOMB : KEY_EMPTY;
    t.cells[i].row = ROW_PENDING;
    t.row_tick[c.row] = 0u;
    uint32_t f = atomicAdd(&t.counters[CTR_FREE], 1u);
    t.free_rows[f] = c.row;
    atomicAdd(&t.counters[CTR_EVICT], 1u);
  }
}

// ------------------------------------------------------------------------------------------------
// launchers (host)
// ------------------------------------------------------------------------------------------------
void launch_fill_cells(Cell* cells, uint64_t n, cudaStream_t st) { PB_LAUNCH(k_fill_cells, PB_NUM_SMS * 8, 256, 0, st, cells, n); }

void launch_begin_batch(const TableDev& t, uint32_t* ctx_tick, uint32_t* batch_cnt, cudaStream_t st, bool bump) {
  PB_LAUNCH(k_begin_batch, 1, batch_cnt ? 256 : 32, 0, st, t.counters, ctx_tick, batch_cnt, bump ? 1 : 0);
}

void launch_probe(int mode, bool prefix, const TableDev& t, const HyperDev& hy, const OptimDev& op, const SlotsDev& sl,
                  const uint64_t* ids, uint32_t n, uint32_t* occ_cell, cudaStream_t st) {
  if (!n) return;
  uint32_t g = cdiv((uint64_t)n * BUCKET, 256);
  if (mode == MODE_FIND) {
    if (prefix) PB_LAUNCH_F(FAM_PROBE, (k_probe<MODE_FIND, true>), g, 256, 0, st, t, hy, op, sl, ids, n, occ_cell);
    else PB_LAUNCH_F(FAM_PROBE, (k_probe<MODE_FIND, false>), g, 256, 0, st, t, hy, op, sl, ids, n, occ_cell);
  } else if (mode == MODE_TRAIN) {
    if (prefix) PB_LAUNCH_F(FAM_PROBE, (k_probe<MODE_TRAIN, true>), g, 256, 0, st, t, hy, op, sl, ids, n, occ_cell);
    else PB_LAUNCH_F(FAM_PROBE, (k_probe<MODE_TRAIN, false>), g, 256, 0, st, t, hy, op, sl, ids, n, occ_cell);
  } else {
    PB_LAUNCH_F(FAM_PROBE, (k_probe<MODE_SET, false>), g, 256, 0, st, t, hy, op, sl, ids, n, occ_cell);
  }
}

void launch_gather(const TableDev& t, const uint32_t* occ_cell, uint32_t n_out, float* out, cudaStream_t st) {
  if (!n_out) return;
  int vec, G;
  vec_group(t.dim, vec, G);
  uint32_t grid;
#define PB_G(V, GG)                                                                                          \
  if (vec == V && G == GG) {                                                                                 \
    grid = cdiv((uint64_t)cdiv(n_out, GATHER_ROWS) * GG, 256);                                               \
    PB_LAUNCH_F(FAM_GATHER, (k_gather_rows<V, GG>), grid, 256, 0, st, t, occ_cell, n_out, out);             \
  }
  PB_G(4, 1) PB_G(4, 2) PB_G(4, 4) PB_G(4, 8) PB_G(4, 16) PB_G(4, 32)
  PB_G(1, 1) PB_G(1, 2) PB_G(1, 4) PB_G(1, 8) PB_G(1, 16) PB_G(1, 32)
#undef PB_G
}

void launch_copy_entries(bool write, const TableDev& t, const uint32_t* occ_cell, uint32_t n, float* entries,
                         uint8_t* found, cudaStream_t st) {
  if (!n) return;
  uint32_t grid = cdiv((uint64_t)n * 32, 256);
  if (write) PB_LAUNCH(k_copy_entries<true>, grid, 256, 0, st, t, occ_cell, n, entries, found);
  else PB_LAUNCH(k_copy_entries<false>, grid, 256, 0, st, t, occ_cell, n, entries, found);
}

void launch_expand_rows(const uint32_t* row_off, uint32_t n_out, uint32_t* occ_outrow, cudaStream_t st) {
  if (n_out) PB_LAUNCH(k_expand_rows, cdiv(n_out, 256), 256, 0, st, row_off, n_out, occ_outrow);
}

void launch_add_prefix(const SlotsDev& sl, const uint64_t* ids, uint32_t n, uint64_t* out, cudaStream_t st) {
  if (n) PB_LAUNCH(k_add_prefix, cdiv(n, 256), 256, 0, st, sl, ids, n, out);
}

// Checkpointing (persia-model-manager dump_internal_shard_embeddings, lib.rs:242-257): the resident signs and the
// batch number each was last used in (the reference walks its LRU list; this is the same order up to ties inside
// a batch).  Writes at most `max_n` pairs in index order; *count receives the number of resident signs.
__global__ void __launch_bounds__(256) k_export_signs(TableDev t, uint64_t* __restrict__ signs,
                                                      uint32_t* __restrict__ recency, uint32_t max_n,
                                                      uint32_t* __restrict__ count) {
  const uint64_t n = (uint64_t)t.n_cells + N_SPECIAL;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    Cell c = t.cells[i];
    const bool occupied = (i < t.n_cells) ? (c.key < KEY_TOMB) : (c.key == 0ULL);
    if (!occupied || c.row >= t.capacity) continue;
    const uint32_t k = atomicAdd(count, 1u);
    if (k < max_n) {
      signs[k] = (i < t.n_cells) ? c.key : KEY_EMPTY - (i - t.n_cells);  // the three marker-valued signs
      recency[k] = t.row_tick[c.row];
    }
  }
}

void launch_export_signs(const TableDev& t, uint64_t* signs, uint32_t* recency, uint32_t max_n, uint32_t* count,
                         cudaStream_t st) {
  cudaMemsetAsync(count, 0, sizeof(uint32_t), st);
  PB_LAUNCH(k_export_signs, PB_NUM_SMS * 8, 256, 0, st, t, signs, recency, max_n, count);
}

void launch_spill(const TableDev& t, uint32_t want_free, uint32_t keep, uint32_t* ev, uint64_t* signs, float* entries,
                  uint32_t max_n, uint32_t* count, cudaStream_t st) {
  PB_LAUNCH(k_evict_plan, 1, 256, 0, st, t, want_free, want_free, ev);
  PB_LAUNCH(k_evict_hist, PB_NUM_SMS * 8, 256, 0, st, t, ev);
  PB_LAUNCH(k_evict_threshold, 1, 32, 0, st, keep, ev);
  PB_LAUNCH(k_evict_sweep_spill, PB_NUM_SMS * 8, 256, 0, st, t, ev, signs, entries, max_n, count);
}

void launch_evict(const TableDev& t, uint32_t low_water, uint32_t target_free, uint32_t keep, uint32_t* ev, cudaStream_t st) {
  PB_LAUNCH(k_evict_plan, 1, 256, 0, st, t, low_water, target_free, ev);
  PB_LAUNCH(k_evict_hist, PB_NUM_SMS * 8, 256, 0, st, t, ev);
  PB_LAUNCH(k_evict_threshold, 1, 32, 0, st, keep, ev);
  PB_LAUNCH(k_evict_sweep, PB_NUM_SMS * 8, 256, 0, st, t, ev);
}

void launch_shard_of(const uint64_t* signs, uint32_t n, uint32_t R, uint32_t* shard, uint64_t* hash, cudaStream_t st) {
  if (n) PB_LAUNCH(k_shard_of, cdiv(n, 256), 256, 0, st, signs, n, R, shard, hash);
}

// A1: indices_to_hashstack_indices (embedding_worker_service/mod.rs:347-400) as an id expansion: every id becomes
// `rounds` keys, key_r = farmhash64^(r+1)(id) % embedding_size + r * embedding_size, laid out id-major so that a
// sample's ids stay together (sample_num_signs grows by the same factor, :393-397).  The regrouping of occurrences
// per hashed key that the reference does next is the per-batch dedup of the forward (pb_dedup.cu).
__global__ void __launch_bounds__(256) k_hash_stack(const uint64_t* __restrict__ ids, uint32_t n, uint32_t rounds,
                                                    uint64_t size, uint64_t* __restrict__ out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint64_t h = ids[i];
  for (uint32_t r = 0; r < rounds; ++r) {
    h = farmhash64_u64(h);
    out[(size_t)i * rounds + r] = h % size + (uint64_t)r * size;
  }
}
void launch_hash_stack(const uint64_t* ids, uint32_t n, uint32_t rounds, uint64_t size, uint64_t* out, cudaStream_t st) {
  if (n) PB_LAUNCH(k_hash_stack, cdiv(n, 256), 256, 0, st, ids, n, rounds, size, out);
}

}  // namespace pb
