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
// A live-exported table (pb_table_export_live_view) keeps training while peers read its index and rows in place
// (pb_remote.cu).  A sweep tombstones cells and frees rows the next admission hands to another sign; a rebuild empties
// the index and fills it again.  So the table's write-sequence word `seq` is odd from before the first cell either
// changes to after the last, and a reader whose probe or row read overlapped that window reads the item again.  The
// word moves inside kernels the check launches anyway, so a live table's step launches what any other table's does and
// stays one graph: the one-thread plan kernels that decide the sweep and the rebuild raise it (a grid's first block is
// not ordered before its other blocks, the kernel before the grid is), and the last block of the rebuild's re-insert
// lowers it.  seq null (every other table): none of this runs.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void seq_step(uint32_t* seq) {
  __threadfence_system();  // (lowering: every cell and row written before)
  *reinterpret_cast<volatile uint32_t*>(seq) = *seq + 1u;
  __threadfence_system();  // (raising: before any cell or row is written)
}

// ------------------------------------------------------------------------------------------------
// Capacity: the reference's EvictionMap drops the least recently used entry whenever an insert pushes it over
// capacity (eviction_map.rs:76-97).  Here recency is the batch number kept in row_tick and
// eviction is a sweep run between batches when free storage is low: (1) histogram of row ages over the occupied
// cells, (2) the age threshold that releases `want` rows (never rows touched in the last `keep` batches),
// (3) tombstone those cells and push their rows on the free stack.  ev[0] = threshold age, ev[1] = want,
// ev[2] = go flag, ev[3..] = age histogram (EV_BINS bins, last bin = older).
// ------------------------------------------------------------------------------------------------
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
    if (!cell_live(t, i, c)) continue;
    uint32_t age = tick - t.row_tick[c.row];
    atomicAdd(&ev[3 + min(age, EV_BINS - 1)], 1u);
  }
}

__global__ void k_evict_threshold(uint32_t keep, uint32_t* __restrict__ ev, uint32_t* __restrict__ seq) {
  if (threadIdx.x || !ev[2]) return;
  uint32_t want = ev[1], got = 0, thr = 0xFFFFFFFFu;
  for (uint32_t a = EV_BINS; a-- > 0 && a > keep;) {  // oldest first; ages <= keep are protected
    got += ev[3 + a];
    thr = a;
    if (got >= want) break;
  }
  ev[0] = got ? thr : 0xFFFFFFFFu;
  if (seq && got) seq_step(seq);  // the sweep below runs: odd (k_rebuild_plan or the rebuild lowers it)
}

__global__ void __launch_bounds__(256) k_evict_sweep(TableDev t, uint32_t* __restrict__ ev) {
  if (!ev[2] || ev[0] == 0xFFFFFFFFu) return;
  const uint32_t tick = t.counters[CTR_TICK], thr = ev[0];
  const uint64_t n = (uint64_t)t.n_cells + N_SPECIAL;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    Cell c = t.cells[i];
    if (!cell_live(t, i, c)) continue;
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

// ------------------------------------------------------------------------------------------------
// Index rebuild (pb_probe.cuh): EMPTY cells only get fewer between rebuilds, so after every eviction check, swept or
// not, the index is rebuilt once more than 7/8 of its normal cells are used (CTR_USED).  Every step is gated on the
// flag the plan sets (no host sync; a captured step stays capturable).  The live (sign, row) pairs of the normal cells
// are compacted into a buffer of `capacity` entries, the normal cells refilled with EMPTY and every pair re-inserted
// at the first EMPTY cell of its probe sequence; the reserved cells stay as they are.  Rows and row_tick do not move,
// so rows held by pending batches stay valid.  After a rebuild at most capacity <= 2/3 n_cells cells are used.
// ev[EV_RB] = rebuild flag, ev[EV_RB + 1] = pairs compacted.
// ------------------------------------------------------------------------------------------------
static_assert(EV_RB + 2 <= EVICT_WS_WORDS, "eviction workspace too small");

__global__ void k_rebuild_plan(TableDev t, uint32_t* __restrict__ ev, uint32_t* __restrict__ seq) {
  if (threadIdx.x) return;
  const uint32_t rb = t.counters[CTR_USED] > t.n_cells - t.n_cells / 8 ? 1u : 0u;
  ev[EV_RB] = rb;
  ev[EV_RB + 1] = 0u;
  if (!seq) return;
  ev[EV_DONE] = 0u;
  // the word is odd iff a sweep ran (k_evict_threshold): a rebuild keeps it odd or raises it, else the sweep is over
  const bool swept = ev[2] && ev[0] != 0xFFFFFFFFu;
  if (swept != (rb != 0u)) seq_step(seq);
}

__global__ void __launch_bounds__(256) k_rebuild_compact(TableDev t, uint32_t* __restrict__ ev, uint64_t* __restrict__ keys,
                                                         uint32_t* __restrict__ rows) {
  if (!ev[EV_RB]) return;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < t.n_cells; i += gridDim.x * blockDim.x) {
    const Cell c = t.cells[i];
    if (c.key >= KEY_TOMB || c.row >= t.capacity) continue;
    const uint32_t at = atomicAdd(&ev[EV_RB + 1], 1u);
    if (at < t.capacity) {  // (always: every live cell holds a row of its own)
      keys[at] = c.key;
      rows[at] = c.row;
    }
  }
}

__global__ void __launch_bounds__(256) k_rebuild_clear(TableDev t, const uint32_t* __restrict__ ev) {
  if (!ev[EV_RB]) return;
  Cell e;
  e.key = KEY_EMPTY;
  e.row = ROW_PENDING;
  e.aux = 0;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < t.n_cells; i += gridDim.x * blockDim.x) t.cells[i] = e;
}

// keys are distinct and no cell is a tombstone: a CAS on EMPTY is all an insertion needs
__global__ void __launch_bounds__(256) k_rebuild_insert(TableDev t, uint32_t* __restrict__ ev,
                                                        const uint64_t* __restrict__ keys, const uint32_t* __restrict__ rows,
                                                        uint32_t* __restrict__ seq) {
  if (!ev[EV_RB]) return;
  const uint32_t n = min(ev[EV_RB + 1], t.capacity);
  if (blockIdx.x == 0 && threadIdx.x == 0) t.counters[CTR_USED] = n;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const unsigned long long key = keys[i];
    uint32_t bucket = (uint32_t)mix64(key) & t.bucket_mask;
    for (bool done = false; !done; bucket = (bucket + 1) & t.bucket_mask) {  // n < n_cells: an EMPTY cell exists
      for (uint32_t s = 0; s < BUCKET && !done; ++s) {
        Cell* c = t.cells + (size_t)bucket * BUCKET + s;
        if (c->key == KEY_EMPTY && atomicCAS(&c->key, KEY_EMPTY, key) == KEY_EMPTY) {
          c->row = rows[i];
          done = true;
        }
      }
    }
  }
  if (seq) {  // the last block to finish lowers the word once every block's cells are written
    __syncthreads();
    if (threadIdx.x == 0) {
      __threadfence();
      if (atomicAdd(&ev[EV_DONE], 1u) == gridDim.x - 1) seq_step(seq);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Growth of a growable table's index (launch_grow_index): the rebuild above with a larger target.  k_grow_plan forces
// the rebuild flag; k_rebuild_compact runs with the old masks; k_grow_specials copies the reserved cells to the new end
// before k_rebuild_clear (new n_cells) overwrites where they were; k_rebuild_insert re-inserts with the new masks.
// ------------------------------------------------------------------------------------------------
__global__ void k_grow_plan(uint32_t* __restrict__ ev) {
  if (threadIdx.x) return;
  ev[EV_RB] = 1u;
  ev[EV_RB + 1] = 0u;
}

__global__ void k_grow_specials(Cell* cells, uint32_t from_n, uint32_t to_n) {
  if (threadIdx.x < N_SPECIAL) cells[(size_t)to_n + threadIdx.x] = cells[(size_t)from_n + threadIdx.x];
}

__global__ void k_grow_readback(const uint32_t* __restrict__ counters, uint32_t* out, uint32_t stamp) {
  if (threadIdx.x) return;
  volatile uint32_t* o = out;
  o[0] = counters[CTR_ROWS];
  o[1] = counters[CTR_USED];
  __threadfence_system();
  o[2] = stamp;
}

// diagnostic (pb_table_index_stats): live, tombstone and EMPTY cells among the n_cells normal cells
__global__ void __launch_bounds__(256) k_index_stats(TableDev t, uint32_t* __restrict__ out) {
  uint32_t live = 0, tomb = 0, empty = 0;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < t.n_cells; i += gridDim.x * blockDim.x) {
    const Cell c = t.cells[i];
    if (c.key == KEY_EMPTY) ++empty;
    else if (c.key == KEY_TOMB) ++tomb;
    else if (c.row < t.capacity) ++live;
  }
  for (int o = 16; o > 0; o >>= 1) {
    live += __shfl_down_sync(0xffffffffu, live, o);
    tomb += __shfl_down_sync(0xffffffffu, tomb, o);
    empty += __shfl_down_sync(0xffffffffu, empty, o);
  }
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(&out[0], live);
    atomicAdd(&out[1], tomb);
    atomicAdd(&out[2], empty);
  }
}

// ------------------------------------------------------------------------------------------------
// launchers (host)
// ------------------------------------------------------------------------------------------------
void launch_rebuild(const TableDev& t, uint32_t* ev, uint64_t* keys, uint32_t* rows, cudaStream_t st, uint32_t blocks,
                    uint32_t* seq) {
  const uint32_t g = blocks ? blocks : PB_NUM_SMS * 8;
  PB_LAUNCH(k_rebuild_plan, 1, 32, 0, st, t, ev, seq);
  PB_LAUNCH(k_rebuild_compact, g, 256, 0, st, t, ev, keys, rows);
  PB_LAUNCH(k_rebuild_clear, g, 256, 0, st, t, ev);
  PB_LAUNCH(k_rebuild_insert, g, 256, 0, st, t, ev, keys, rows, seq);
}

void launch_grow_index(const TableDev& from, const TableDev& to, uint32_t* ev, uint64_t* keys, uint32_t* rows,
                       cudaStream_t st) {
  const uint32_t g = PB_NUM_SMS * 8;
  PB_LAUNCH(k_grow_plan, 1, 32, 0, st, ev);
  PB_LAUNCH(k_rebuild_compact, g, 256, 0, st, from, ev, keys, rows);
  PB_LAUNCH(k_grow_specials, 1, 32, 0, st, to.cells, from.n_cells, to.n_cells);
  PB_LAUNCH(k_rebuild_clear, g, 256, 0, st, to, ev);
  PB_LAUNCH(k_rebuild_insert, g, 256, 0, st, to, ev, keys, rows, nullptr);
}

void launch_grow_readback(const uint32_t* counters, uint32_t* out, uint32_t stamp, cudaStream_t st) {
  PB_LAUNCH(k_grow_readback, 1, 32, 0, st, counters, out, stamp);
}

void launch_index_stats(const TableDev& t, uint32_t* out, cudaStream_t st) {
  cudaMemsetAsync(out, 0, 3 * sizeof(uint32_t), st);
  PB_LAUNCH(k_index_stats, PB_NUM_SMS * 8, 256, 0, st, t, out);
}

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
    if (!cell_live(t, i, c)) continue;
    const uint32_t k = atomicAdd(count, 1u);
    if (k < max_n) {
      signs[k] = cell_sign(t, i, c);
      recency[k] = t.row_tick[c.row];
    }
  }
}

void launch_export_signs(const TableDev& t, uint64_t* signs, uint32_t* recency, uint32_t max_n, uint32_t* count,
                         cudaStream_t st) {
  cudaMemsetAsync(count, 0, sizeof(uint32_t), st);
  PB_LAUNCH(k_export_signs, PB_NUM_SMS * 8, 256, 0, st, t, signs, recency, max_n, count);
}

void launch_evict(const TableDev& t, uint32_t low_water, uint32_t target_free, uint32_t keep, uint32_t* ev, uint64_t* rb_keys,
                  uint32_t* rb_rows, uint32_t* seq, cudaStream_t st) {
  PB_LAUNCH(k_evict_plan, 1, 256, 0, st, t, low_water, target_free, ev);
  PB_LAUNCH(k_evict_hist, PB_NUM_SMS * 8, 256, 0, st, t, ev);
  PB_LAUNCH(k_evict_threshold, 1, 32, 0, st, keep, ev, seq);
  PB_LAUNCH(k_evict_sweep, PB_NUM_SMS * 8, 256, 0, st, t, ev);
  launch_rebuild(t, ev, rb_keys, rb_rows, st, 0, seq);
}

// The HBM table's plan and threshold count its victims; the tier's own sweep (gated on the flag launch_tier_plan sets)
// drops as many of the tier's oldest entries as it takes to hold them; the victims then move (launch_tier_move) instead
// of being swept.  Every step reads its sizes from the device: no host sync, a captured step stays capturable.
void launch_evict_tier(const TableDev& h, const TableDev& t, const HyperDev& hy, const OptimDev& op, uint32_t low_water,
                       uint32_t target_free, uint32_t keep, uint32_t* ev, uint64_t* rb_keys, uint32_t* rb_rows, uint32_t* tev,
                       uint64_t* trb_keys, uint32_t* trb_rows, uint32_t* move_cells, cudaStream_t st, uint32_t blocks) {
  const uint32_t g = blocks ? blocks : PB_NUM_SMS * 8;
  PB_LAUNCH(k_evict_plan, 1, 256, 0, st, h, low_water, target_free, ev);
  PB_LAUNCH(k_evict_hist, g, 256, 0, st, h, ev);
  PB_LAUNCH(k_evict_threshold, 1, 32, 0, st, keep, ev, nullptr);
  launch_tier_plan(h, t, ev, tev, st);
  PB_LAUNCH(k_evict_hist, g, 256, 0, st, t, tev);
  PB_LAUNCH(k_evict_threshold, 1, 32, 0, st, 0u, tev, nullptr);  // no batch holds a tier row: only the current batch number's stay
  PB_LAUNCH(k_evict_sweep, g, 256, 0, st, t, tev);
  launch_tier_move(h, t, hy, op, ev, tev, rb_keys, rb_rows, move_cells, st, blocks);  // (rebuild buffers free until below)
  launch_rebuild(h, ev, rb_keys, rb_rows, st, blocks);
  launch_rebuild(t, tev, trb_keys, trb_rows, st, blocks);
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
