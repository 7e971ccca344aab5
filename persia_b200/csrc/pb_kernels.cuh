// pb_kernels.cuh — kernel-side parameter blocks and launcher prototypes (internal).
#pragma once
#include <atomic>
#include <string>
#include <vector>

#include "pb_common.cuh"

namespace pb {

// per-batch slot table, passed by value in kernel-parameter memory
struct SlotsDev {
  uint64_t prefix[PB_MAX_SLOTS];
  uint32_t occ_off[PB_MAX_SLOTS + 1];  // slot boundaries in the flat id array
  uint8_t sqrt_scaling[PB_MAX_SLOTS];
  uint32_t n_slots;
  uint64_t spacing;  // 2^(64-prefix_bit) - 1
  uint32_t spacing_bits;  // 64 - prefix_bit
  uint32_t uniform;       // occurrences per slot when every slot holds the same number (one id per sample), else 0
};

// per-batch gradient table (GradientBatch, persia-core/src/backward.rs:74-106)
struct GradsDev {
  const void* ptr[PB_MAX_SLOTS];  // nullptr = skipped slot
  float inv_scale[PB_MAX_SLOTS];  // 1/scale_factor
  uint8_t do_scale[PB_MAX_SLOTS]; // |scale-1| > f32::EPSILON (mod.rs:751)
  const float* adam_pow;          // Adam: accumulated (beta1^t, beta2^t) pairs on the device, one per feature group
  uint8_t pow_idx[PB_MAX_SLOTS];  // the slot's pair
};

// ---- the batch context on the device (what the EW keeps in post_forward_buffer, mod.rs:1087-1098) ------------------
// Filled by the forward (dedup -> probe -> gather), consumed by the backward.  A distinct (sign, slot) pair of the
// batch is an "item"; the occurrences of an item with count > 1 are listed in seg_occ[base, base + count) in
// arbitrary order (the reducing kernels put them in ascending order, the reference's summation order).
constexpr uint32_t PB_GIANT_MIN = 1024;  // the few longest chains of a batch: listed in the top giant_cap entries of `hot`
constexpr uint32_t PB_HUGE_MIN = 256;  // hot items above this are the long poles of the backward: they start first
constexpr uint32_t PB_WARM_MAX = 32;  // items of 2..PB_WARM_MAX occurrences are reduced by a lane group, larger ones by a CTA
enum {
  BC_ITEMS = 0,  // distinct items of the batch
  BC_COLD,       // items of one occurrence
  BC_WARM,       // items of 2..PB_WARM_MAX occurrences
  BC_HOT,        // items of more
  BC_SEG,        // entries of seg_occ handed out
  BC_HUGE,       // hot items of more than PB_HUGE_MIN occurrences: listed from the END of `hot`, reduced first
  BC_GIANT,      // hot items of more than PB_GIANT_MIN occurrences: the very first to be reduced
  BC_PEER = 8,
  BC_NEXT = 24,  // work cursors of the reducing kernels: [round] warm, [PB_MAX_SLOTS + round] hot
  // words of the hot-item bitmap pool asked for, a u64 over two words (8-byte aligned): every hot item adds its slot's
  // bitmap words, also once the pool is used up, and a batch can ask for up to n / 33 x n / 32 words (2^38 at 2^24)
  BC_HOTW = BC_NEXT + 2 * PB_MAX_SLOTS,
  BC_COUNT = BC_HOTW + 2
};
static_assert(BC_HOTW % 2 == 0, "BC_HOTW is a u64");
struct BatchDev {
  DCell* set;           // scratch set: region of slot s = [2*occ_off[s] + 2*s, +2*n_s + 1), then its reserved cell
  uint32_t* occ_set;    // [n] set cell of every occurrence
  uint32_t* item_cell;  // [n] set cell of every item
  uint32_t* seg_occ;    // [n] occurrence lists
  uint2* cold;          // [n]   (target, occurrence)
  uint4* warm;          // [n/2] (target, base, count, -)
  uint4* hot;           // [n/PB_WARM_MAX] (target, base | bitmap word offset + bit 31, count, slot)
  uint32_t* hot_bits;   // [hot_words] one bit per sample of the slot for hot items in bitmap mode (all zero between batches)
  uint32_t hot_words;
  uint32_t hot_cap;     // entries of `hot`
  uint32_t giant_cap;   // of which the top ones are reserved for the giants (n / PB_GIANT_MIN + 1)
  uint32_t* cnt;        // BC_* words
  uint32_t n;           // id occurrences of the batch
};
__device__ __forceinline__ unsigned long long* hot_words_asked(const BatchDev& b) {
  return reinterpret_cast<unsigned long long*>(b.cnt + BC_HOTW);
}

// ---- the shard exchange (pb_shard.cu): one endpoint per rank, buffers in peer-mapped memory -----------------------
// Every rank is an embedding worker for its own batches (requester) and parameter server `rank` (owner).  Rank r owns
// one receive area, written by its peers over NVLink with plain stores; `base[q]` is rank q's area as mapped here.
//   ctrl   [XC_WORDS][16] u32   flags (one word per phase and source, written by that source) and sign counts
//   sign   [R][cap] u64         signs requested of this rank, by source
//   row    [R][cap][dim]        rows returned to this rank, by owner (f16, or f32 for ragged layouts)
//   grad   [R][cap][dim] f32    reduced gradients sent to this rank, by source
//   gok    [R][cap] u32         1 = apply the gradient, 0 = the slot was skipped / held a NaN
//   chain  [R][cap] u32         requests with slots sharing a feature group: CHAIN_CONT | the sign's next entry
// ctrl word XC_CHAIN of a source equals its XC_FLAG_SIGN word when that source's request of the step carries chain words.
// A stage exchange (pb_xchg_create_stage) has the ctrl and sign parts only: XC_FLAG_SIGN and XC_COUNT carry the signs
// of the next batch that each source sends the owner a step early (pb_tier_stage_sharded).
enum { XC_FLAG_SIGN = 0, XC_FLAG_ROW, XC_FLAG_GRAD, XC_COUNT, XC_CHAIN, XC_WORDS };
// chain word of an entry: a sign that several slots of one feature group hold is one entry per slot; the first (the
// head, in slot order) carries the step, the others follow it.  CHAIN_CONT: not a head; low bits: the request's next
// entry of the sign (CHAIN_END: none).
constexpr uint32_t CHAIN_CONT = 0x80000000u;
constexpr uint32_t CHAIN_END = 0x7FFFFFFFu;
// the slots of a context's feature groups in slot order: prev / next slot of the same group (0xFF: none)
struct GroupLinks {
  uint8_t prev[PB_MAX_SLOTS];
  uint8_t next[PB_MAX_SLOTS];
};
constexpr uint32_t PB_MAX_RANKS = 16;
constexpr uint32_t PB_ADAM_KEYS = 256;  // beta-power pairs per table; the last one serves pb_update
// owner side, one step: the distinct rows the R requests touch (k_owner_lookup fills it, k_owner_update_all empties it)
struct __align__(16) UCell {
  uint32_t row;               // ROW_NONE = empty
  uint32_t mask;              // sources that asked for the row
  uint32_t k[PB_MAX_RANKS];   // the row's index in each such source's request
  uint32_t pad[2];
};
struct XchgDev {
  uint64_t base[PB_MAX_RANKS];
  uint64_t off_sign, off_row, off_grad, off_gok, off_chain;  // byte offsets inside an area (ctrl at 0)
  uint32_t R, rank, cap, row_f32;
  uint32_t* epoch;     // [XC_WORDS] phases signalled so far (device side: CUDA-graph safe)
  uint32_t* waited;    // [XC_WORDS][PB_MAX_RANKS] phases waited for so far, per source
  uint32_t* own_row;   // [R][cap] row of every received sign (forward -> backward)
  uint32_t* own_cnt;   // [R] signs received per source (copied out of ctrl: the next request may overwrite it early)
  uint32_t* err;       // [0] a pair needed more than cap slots, [1] a wait gave up
  UCell* ucell;        // [ucells] rows of the step's requests, hashed by row number
  uint32_t* uwin;      // [R][cap] the cell a request's sign opened (it was the first to ask for the row), else ROW_NONE
  uint32_t ucells;     // a power of two >= 2 R cap
  uint32_t* chained;   // [1] bit per source: its request of this step carries chain words (forward -> backward)
  uint32_t* own_link;  // [R][cap] chain word of every received sign of such a request (forward -> backward)
  // Adam on the owner: feature groups (index prefixes) of the table, the groups each request holds, and the (beta1^t,
  // beta2^t) pair every request's signs of a group use (get_batch_level_state, optim.rs:151-197)
  const uint64_t* akeys;  // [n_akeys] prefixes, position = pair number of the table
  uint32_t n_akeys;
  uint64_t amask;         // the prefix bits of a sign
  uint32_t* apresent;     // [R][PB_ADAM_KEYS / 32] groups among the signs request s applies
  float* apow;            // [R][PB_ADAM_KEYS][2]
};

// a remote read (pb_remote.cu): every owner's index and rows as this GPU reaches them (its own table directly, a peer's
// through a pb_view), and the owner's write-sequence word (null: no insert can run beside the read)
struct RemoteDev {
  TableDev t[PB_MAX_RANKS];
  const uint32_t* seq[PB_MAX_RANKS];
  uint32_t R;
};
// k_remote_lookup<TIER>'s argument: the owners' tables and each owner's shared host tier (cells null: none)
struct RemoteTierDev {
  RemoteDev rv;
  TableDev tier[PB_MAX_RANKS];
};
// k_remote_lookup<GROW>'s argument: owners whose tables are exportable growable ones.  geo[q]: owner q's published
// index cell count (its write-sequence word's second word; null: the geometry in rv.t[q] holds); rows[q] / cells[q]:
// the rows and index cell slots (with the N_SPECIAL reserved ones) this process has mapped of owner q.  An item whose
// owner's index has more cells than are mapped here, or whose row is not mapped here, is stale: not read, its target
// set to ROW_STALE and counted in *stale.  only_stale: items whose target is not ROW_STALE are skipped (a retry)
struct RemoteGrowDev {
  RemoteDev rv;
  const uint32_t* geo[PB_MAX_RANKS];
  uint32_t rows[PB_MAX_RANKS], cells[PB_MAX_RANKS];
  uint32_t* stale;
  uint32_t only_stale;
};
constexpr uint32_t ROW_STALE = 0xFFFFFFFDu;  // an item a remote read must read again once more chunks are mapped

// arguments of the backward kernels (pb_reduce.cu)
struct ReduceArgs {
  BatchDev b;
  const uint32_t* occ_outrow;  // nullptr: one id per sample per slot (output row == occurrence)
  const uint32_t* row_off;
  const uint32_t* tick_ptr;
  const uint32_t* nan_tick;
  float* vw_stage;             // Adagrad vectorwise: one reduced gradient per item
  float* hot_stage;            // [hot_cap][dim]: the sum of every hot item at its entry of b.hot (k_reduce_hot -> k_step_hot)
  uint32_t batch, round, quiet_miss;
  uint32_t short_max;          // hot items of up to this many occurrences are k_reduce_hot_short's (0: none)
  uint32_t round_mask[PB_MAX_SLOTS / 32];  // slots stepped by this launch (slots of one feature group take turns)
  XchgDev x;                   // sharded: the reduced gradient is stored into the owner's receive area instead
};

// raw slots (pb_raw.cu): per-batch scratch set of distinct signs and its workspace
struct RawCell {
  uint64_t key;
  uint32_t first;  // first occurrence of the sign in the flat id array
  uint32_t rank;   // number of the sign among the batch's distinct signs (first-occurrence order)
};
struct RawWork {
  RawCell* set;      // set_mask + 2 cells
  uint32_t set_mask;
  uint32_t* occ_set;        // set cell of every occurrence
  uint32_t* flag;           // scan input / second scan output
  uint32_t* rank;           // scan output
  uint32_t* tiles;          // scan spine
  uint32_t* distinct_cell;  // index cell of every distinct sign (forward -> backward); sharded: its scratch-set cell
  uint32_t* counts;         // [0] distinct signs, [1] ids placed in `index`
  // sharded path (pb_forward_raw_sharded): where every distinct sign went, owner * cap + slot (ROW_NONE: over cap);
  // local path (pb_forward_raw): the table row of every distinct sign (ROW_NONE: no storage), forward -> backward
  uint32_t* target;         // [n]
  uint32_t* peer;           // [PB_MAX_RANKS] distinct signs routed to each owner
};

// the set of signs stepped since the last take (pb_inc.cu, pb_table_enable_incremental): an open-addressing set of
// n_cells cells keyed by sign (a power of two >= 2 x capacity), BUCKET cells per 128 B line, home bucket from mix64 as in
// the index; the signs >= KEY_TOMB (equal to a marker) own the N_SPECIAL reserved cells after them (row == 1: held)
enum { INC_HELD = 0, INC_INSERTED, INC_DROPPED, INC_TAKEN, INC_CURSOR, INC_DONE, INC_WORDS };
struct IncDev {
  Cell* cells;                  // n_cells + N_SPECIAL
  unsigned long long* ctr;      // INC_* words
  unsigned long long* mirror;   // device address of the mapped pinned host word that mirrors ctr[INC_HELD]
  unsigned long long capacity;  // signs the set may hold
  uint32_t n_cells, bucket_mask;
};
struct IncSlots {
  uint32_t applied[PB_MAX_SLOTS / 32];  // slots the request gave a gradient (the NaN rule is read on the device)
};
void launch_inc_fill(const IncDev& s, cudaStream_t st);
void launch_inc_mark_items(const IncDev& s, const BatchDev& b, const SlotsDev& sl, const IncSlots& on,
                           const uint32_t* tick, const uint32_t* nan_tick, bool clear, cudaStream_t st);
void launch_inc_mark_raw(const IncDev& s, const RawWork& w, uint32_t n, const uint32_t* tick, const uint32_t* nan_tick,
                         cudaStream_t st);
void launch_inc_mark_signs(const IncDev& s, const TableDev& h, const uint64_t* signs, const uint32_t* occ_cell,
                           uint32_t n, const TableDev& t, const uint32_t* where, cudaStream_t st);
void launch_inc_mark_owner(const IncDev& s, const XchgDev& x, uint32_t capacity, cudaStream_t st);
void launch_inc_take(const IncDev& s, uint64_t* out, uint32_t max_n, uint32_t* count, cudaStream_t st);

void launch_fill_cells(Cell* cells, uint64_t n, cudaStream_t st);
void launch_fill_set(DCell* set, uint64_t n, cudaStream_t st);
// bump: a training request (advances the table's batch number and the context's request number)
void launch_begin_batch(const TableDev& t, uint32_t* ctx_tick, uint32_t* batch_cnt, cudaStream_t st, bool bump = true);
void launch_probe(int mode, bool prefix, const TableDev& t, const HyperDev& hy, const OptimDev& op, const SlotsDev& sl,
                  const uint64_t* ids, uint32_t n, uint32_t* occ_cell, cudaStream_t st);
void launch_gather(const TableDev& t, const uint32_t* occ_cell, uint32_t n_out, float* out, cudaStream_t st);
// batched path (pb_dedup.cu)
void launch_dedup(const SlotsDev& sl, const BatchDev& b, const uint64_t* ids, cudaStream_t st);
void launch_probe_items(bool training, const TableDev& t, const HyperDev& hy, const OptimDev& op, const SlotsDev& sl,
                        const BatchDev& b, cudaStream_t st);
// tier_rows / tier_cap (inference with a host tier): targets >= capacity name tier rows, read in place
void launch_gather_items(const TableDev& t, const SlotsDev& sl, const BatchDev& b, const uint32_t* row_off,
                         uint32_t n_out, uint32_t batch, bool training, void* out_f16, cudaStream_t st,
                         const float* tier_rows = nullptr, uint32_t tier_cap = 0);
void launch_clear_items(const BatchDev& b, cudaStream_t st);
void launch_clear_hot_bits(const BatchDev& b, cudaStream_t st);  // of a batch whose backward never came
void launch_copy_entries(bool write, const TableDev& t, const uint32_t* occ_cell, uint32_t n, float* entries,
                         uint8_t* found, cudaStream_t st);
void launch_nan_scan(const GradsDev& gr, uint32_t n_slots, uint32_t elems_per_slot, bool f16, const uint32_t* tick,
                     uint32_t* nan_tick, int32_t* status, cudaStream_t st);
// pb_reduce.cu, the backward's reduces.  send: sharded requester — a.x names the owners' receive areas, no row is
// touched here.
// cold items on `st`, warm items on `st_warm` (may equal st)
void launch_reduce_items(const TableDev& t, const OptimDev& op, const HyperDev& hy, const SlotsDev& sl,
                         const GradsDev& gr, bool f16, const ReduceArgs& a, cudaStream_t st, cudaStream_t st_warm,
                         bool send = false);
// hot items: the ordered sums (to a.hot_stage unless send; reads no NaN mark unless send), then, local path only, the
// step of their rows (after the NaN scan and the Adam power advance)
void launch_reduce_hot(const TableDev& t, const SlotsDev& sl, const GradsDev& gr, bool f16, const ReduceArgs& a,
                       cudaStream_t st, bool send = false);
// local path: the sums of the hot items of up to a.short_max occurrences (k_reduce_hot_short), staged as
// launch_reduce_hot stages the others'; a.short_max = hot_short_max(batch), 0 when k_reduce_hot takes every hot item
uint32_t hot_short_max(uint32_t batch);
void launch_reduce_hot_short(const TableDev& t, const SlotsDev& sl, const GradsDev& gr, bool f16, const ReduceArgs& a,
                             cudaStream_t st);
void launch_step_hot(const TableDev& t, const OptimDev& op, const HyperDev& hy, const SlotsDev& sl, const GradsDev& gr,
                     const ReduceArgs& a, cudaStream_t st);
// diagnostic (pb_hot_geometry): the geometry launch_reduce_hot gives k_reduce_hot
void hot_geometry(uint32_t dim, bool f16, bool ragged, uint32_t out[12]);
// pb_shard.cu
void launch_route_items(bool training, const SlotsDev& sl, const BatchDev& b, const XchgDev& x, cudaStream_t st);
void launch_link_items(const SlotsDev& sl, const BatchDev& b, const XchgDev& x, const GroupLinks& gl, cudaStream_t st);
void launch_signal(const XchgDev& x, int phase, const uint32_t* counts, cudaStream_t st);
void launch_wait(const XchgDev& x, int phase, int src /* -1: every source */, cudaStream_t st);
void launch_signal_wait(const XchgDev& x, int phase, const uint32_t* counts, cudaStream_t st);
// tier: the table's host tier (null: none); an inference request then reads the signs it holds in place
void launch_owner_lookup(bool training, const TableDev& t, const TableDev* tier, const HyperDev& hy, const OptimDev& op,
                         const XchgDev& x, cudaStream_t st);
// rows: the f16 or f32 (row_f32) rows the items' set-cell targets index (the receive area, or a remote read's staging)
void launch_expand_items(const TableDev& t, const SlotsDev& sl, const BatchDev& b, const void* rows, bool row_f32,
                         const uint32_t* row_off, uint32_t n_out, uint32_t batch, bool training, void* out_f16,
                         cudaStream_t st);
void launch_hash_stack(const uint64_t* ids, uint32_t n, uint32_t rounds, uint64_t size, uint64_t* out, cudaStream_t st);
void launch_owner_adam(const XchgDev& x, float* table_pow, float b1, float b2, cudaStream_t st);
void launch_uclear(const XchgDev& x, cudaStream_t st);
void launch_owner_update_all(const TableDev& t, const OptimDev& op, const HyperDev& hy, const XchgDev& x, cudaStream_t st);
void launch_owner_update(const TableDev& t, const OptimDev& op, const HyperDev& hy, const XchgDev& x, uint32_t src,
                         cudaStream_t st);
// n_ptr (optional): the live count on the device (<= n); tick/nan_tick (optional): skip everything when equal;
// by_row: `where` holds table rows (ROW_NONE: no storage) rather than index cells
void launch_update_direct(const TableDev& t, const OptimDev& op, const HyperDev& hy, const uint32_t* where,
                          const float* grads, uint32_t n, const float* adam_pair, cudaStream_t st,
                          const uint32_t* n_ptr = nullptr, const uint32_t* tick = nullptr,
                          const uint32_t* nan_tick = nullptr, bool by_row = false);
struct AdamKeys {
  uint8_t idx[PB_MAX_SLOTS];
  uint32_t n;
};
void launch_adam_fill(float* pow, float b1, float b2, cudaStream_t st);
void launch_adam_advance(float* pow, const AdamKeys& keys, float b1, float b2, cudaStream_t st, const GradsDev* gr = nullptr,
                         uint32_t n_slots = 0, const uint32_t* tick = nullptr, const uint32_t* nan_tick = nullptr);
uint32_t raw_scan_tiles(uint32_t n);
// numbering of the distinct signs, index / non_empty / sample_id_num; occ_cell null: distinct_cell = scratch-set cells
void launch_raw_number(const SlotsDev& sl, const uint64_t* ids, uint32_t n, const uint32_t* row_off,
                       const uint32_t* occ_sample, uint32_t batch, uint32_t fixed, const uint32_t* occ_cell,
                       const RawWork& w, long long* index, long long* non_empty, uint32_t* sample_id_num,
                       cudaStream_t st);
// pb_shard.cu, PB_PHASE_PREPARE: need[q] += the prepared batch's distinct items owned by q (the dedup's items of `b`, or
// the raw numbering's distinct signs of `w` when raw; n: worst-case U)
void launch_count_owners(bool raw, const BatchDev& b, const RawWork& w, uint32_t n, uint32_t R, uint32_t* need,
                         cudaStream_t st);
// pb_remote.cu: the distinct items of the context's batch (raw: its numbered distinct signs) read from their owners into
// `stage` at the item's number, f16(0 + row) or f32 rows (raw: f32), targets set to the item's number; err counts the
// items whose read gave up (n: worst-case U)
// tiers: the owners' host tiers (null: no owner has one, and the untiered kernels run); grow: the owners' growth
// (null: no owner grows, and the kernels without the stale check run; its `rv` is ignored: `rv` is used)
void launch_remote_lookup(bool raw, bool row_f32, const RemoteDev& rv, const TableDev* tiers, const RemoteGrowDev* grow,
                          const BatchDev& b, const RawWork& w, uint32_t n, void* stage, uint32_t dim, uint32_t* err,
                          cudaStream_t st);
// an exported table's write-sequence word: odd from `begin` to the end of the writes that follow.  cells (at the
// end, nonzero): the index's new cell count, published in the word after it before it is even again
void launch_seq_bump(uint32_t* seq, bool begin, cudaStream_t st, uint32_t cells = 0);
// pb_shard.cu, raw slot over R shards: requester's route, table fill and gradient send (n: worst-case U)
void launch_raw_route(const RawWork& w, uint32_t n, const XchgDev& x, cudaStream_t st);
void launch_raw_fill(const RawWork& w, uint32_t n, uint32_t dim, const float* rows, void* table_f16, cudaStream_t st);
void launch_raw_send(const void* grad, bool f16, const RawWork& w, uint32_t n, uint32_t dim, float inv_scale,
                     bool do_scale, const uint32_t* tick, const uint32_t* nan_tick, const XchgDev& x, cudaStream_t st);
void launch_raw_forward(const TableDev& t, const SlotsDev& sl, const uint64_t* ids, uint32_t n,
                        const uint32_t* row_off, const uint32_t* occ_sample, uint32_t batch, uint32_t fixed,
                        const uint32_t* occ_cell, const RawWork& w, void* table_f16, long long* index,
                        long long* non_empty, uint32_t* sample_id_num, cudaStream_t st);
void launch_raw_nan(const void* grad, bool f16, const uint32_t* n_distinct, uint32_t dim, const uint32_t* tick,
                    uint32_t* nan_tick, cudaStream_t st);
void launch_raw_stage(const void* grad, bool f16, const uint32_t* n_distinct, uint32_t dim, float inv_scale,
                      bool do_scale, float* out, cudaStream_t st);
void launch_slot_status(const GradsDev& gr, uint32_t n_slots, const uint32_t* tick, const uint32_t* nan_tick,
                        int32_t* status, cudaStream_t st);
uint32_t radix_tile(uint32_t n);
uint32_t radix_hist_words();
uint32_t radix_hist_zero_words(uint32_t n);
void launch_zero_words(uint32_t* p, uint32_t n_words, cudaStream_t st);
uint64_t partition_workspace_bytes(uint32_t n);
void launch_partition_by_shard(const uint64_t* signs, uint32_t n, uint32_t R, uint32_t* perm, uint32_t* counts,
                               uint32_t* work, cudaStream_t st);
void launch_expand_rows(const uint32_t* row_off, uint32_t n_out, uint32_t* occ_outrow, cudaStream_t st);
void launch_add_prefix(const SlotsDev& sl, const uint64_t* ids, uint32_t n, uint64_t* out, cudaStream_t st);
void launch_shard_of(const uint64_t* signs, uint32_t n, uint32_t R, uint32_t* shard, uint64_t* hash, cudaStream_t st);
void launch_export_signs(const TableDev& t, uint64_t* signs, uint32_t* recency, uint32_t max_n, uint32_t* count,
                         cudaStream_t st);
// capacity sweeps (pb_index.cu): ev = EVICT_WS_WORDS words; rb_keys / rb_rows = `capacity` entries each, where the index
// rebuild that follows every sweep check compacts the live pairs
constexpr uint32_t EV_BINS = 1024;        // ev[3..]: age histogram (last bin = older)
constexpr uint32_t EV_RB = 3 + EV_BINS;   // ev[EV_RB] rebuild flag, ev[EV_RB + 1] pairs compacted
constexpr uint32_t EV_MOVE = EV_RB + 2;   // a tier's ev[EV_MOVE]: HBM victims listed for the move (pb_tier.cu)
constexpr uint32_t EV_DONE = EV_MOVE + 1;  // ev[EV_DONE]: blocks of the rebuild's re-insert that finished (seq != null)
constexpr uint32_t EVICT_WS_WORDS = EV_DONE + 1;
// seq: a live-exported table's write-sequence word (pb_table_export_live_view), null otherwise.  The plan kernels and
// the rebuild's last block keep it odd from before the first cell the sweep or the rebuild changes to after the last;
// no kernel is added, and with seq null nothing new runs.
void launch_evict(const TableDev& t, uint32_t low_water, uint32_t target_free, uint32_t keep, uint32_t* ev, uint64_t* rb_keys,
                  uint32_t* rb_rows, uint32_t* seq, cudaStream_t st);
void launch_index_stats(const TableDev& t, uint32_t* out, cudaStream_t st);
// host-memory tier (pb_tier.cu).  h: the HBM table, t: its tier (rows in mapped pinned host memory).
// The eviction check of a table with a tier: the HBM sweep's victims move into the tier (whose own sweep first drops its
// oldest entries to make room) instead of being dropped.  ev / rb_*: the HBM table's workspaces, tev / trb_*: the tier's,
// move_cells: `h.capacity` words.
void launch_evict_tier(const TableDev& h, const TableDev& t, const HyperDev& hy, const OptimDev& op, uint32_t low_water,
                       uint32_t target_free, uint32_t keep, uint32_t* ev, uint64_t* rb_keys, uint32_t* rb_rows, uint32_t* tev,
                       uint64_t* trb_keys, uint32_t* trb_rows, uint32_t* move_cells, cudaStream_t st,
                       uint32_t blocks = 0);  // blocks: grid of the scans and moves (0 = their usual multiple of the SMs)
void launch_tier_plan(const TableDev& h, const TableDev& t, const uint32_t* ev, uint32_t* tev, cudaStream_t st);
void launch_tier_move(const TableDev& h, const TableDev& t, const HyperDev& hy, const OptimDev& op, const uint32_t* ev,
                      uint32_t* tev, uint64_t* keys, uint32_t* rows, uint32_t* cells, cudaStream_t st, uint32_t blocks = 0);
// pb_tier_stage: restores of an upcoming request's signs (slot-prefixed), on `blocks` blocks; a moved row gets the current
// batch number, a sign that finds no free HBM row stays in the tier (counted as a skipped stage)
void launch_tier_stage(const TableDev& h, const TableDev& t, const HyperDev& hy, const OptimDev& op, const SlotsDev& sl,
                       const uint64_t* ids, uint32_t n, uint32_t blocks, cudaStream_t st);
// before a probe: every sign the HBM index lacks and the tier holds is moved into a free HBM row (flat ids, prefixed by
// slot when `prefix`; or the distinct items of a batch)
void launch_tier_restore(const TableDev& h, const TableDev& t, const HyperDev& hy, const OptimDev& op, const SlotsDev& sl,
                         bool prefix, const uint64_t* ids, uint32_t n, cudaStream_t st);
void launch_tier_restore_items(const TableDev& h, const TableDev& t, const HyperDev& hy, const OptimDev& op,
                               const BatchDev& b, cudaStream_t st);
// sharded training forward (PB_PHASE_SERVE): the signs the R requests of the step brought this owner (its receive area,
// each source's count), before k_owner_lookup probes them.  stage_blocks != 0: pb_tier_stage_sharded's SERVE, on that
// many blocks: the signs of a stage exchange's area, restored as pb_tier_stage restores (age 0, skips counted as such)
void launch_tier_restore_recv(const TableDev& h, const TableDev& t, const HyperDev& hy, const OptimDev& op,
                              const XchgDev& x, cudaStream_t st, uint32_t stage_blocks = 0);
// pb_tier_stage_sharded's SEND (pb_shard.cu): every id slot-prefixed as k_tier_stage does, sent once per warp to its
// owner's stage area (farmhash64 % R); sent[q] counts the signs for owner q (zeroed by the caller; over cap: x.err[0])
void launch_stage_route(const SlotsDev& sl, const uint64_t* ids, uint32_t n, const XchgDev& x, uint32_t* sent,
                        cudaStream_t st);
// Reads in place (no move): signs the HBM probe missed (occ_cell = none) that the tier holds.
//   pb_get_rows: whole entries (len = entry length) + found;  inference pb_lookup: embeddings (len = dim), and the
//   HBM table's CTR_MISS gives back the misses it counted for them (miss_ctr = that counter)
void launch_tier_get(const TableDev& h, const TableDev& t, const uint64_t* signs, const uint32_t* occ_cell, uint32_t n,
                     uint32_t len, float* entries, uint8_t* found, uint32_t* miss_ctr, cudaStream_t st);
// inference pb_forward: items the HBM probe missed get target = h.capacity + tier row (launch_gather_items reads it)
void launch_tier_find_items(const TableDev& h, const TableDev& t, const BatchDev& b, cudaStream_t st);
// inference pb_forward_raw: distinct signs the HBM probe missed are filled into the f16 table from the tier
void launch_tier_raw_fill(const TableDev& h, const TableDev& t, const SlotsDev& sl, const uint64_t* ids, uint32_t n,
                          const uint32_t* occ_cell, const RawWork& w, void* table_f16, cudaStream_t st);
// pb_update: where[i] = the tier cell of every sign the HBM probe missed and the tier holds (else none); the HBM table's
// CTR_GRAD_MISS gives back the miss its update will count for it
void launch_tier_where(const TableDev& h, const TableDev& t, const uint64_t* signs, const uint32_t* occ_cell, uint32_t n,
                       uint32_t* where, cudaStream_t st);
// pb_set_rows: entries the HBM table had no row for are stored in the tier
void launch_tier_set(const TableDev& h, const TableDev& t, const HyperDev& hy, const OptimDev& op, const uint64_t* signs,
                     const uint32_t* occ_cell, uint32_t n, const float* entries, cudaStream_t st);
void launch_rebuild(const TableDev& t, uint32_t* ev, uint64_t* keys, uint32_t* rows, cudaStream_t st, uint32_t blocks = 0,
                    uint32_t* seq = nullptr);
// A growable table's index doubled (or more) in place: the live pairs of `from`'s normal cells are compacted, the
// N_SPECIAL reserved cells move from from.n_cells to to.n_cells, to's normal cells are filled with EMPTY and every pair
// is re-inserted with to's masks (CTR_USED = pairs).  `to` differs from `from` in n_cells and the masks only; the cells
// up to to.n_cells + N_SPECIAL are mapped.  Ordered like a rebuild: nothing that holds cell numbers runs beside it.
void launch_grow_index(const TableDev& from, const TableDev& to, uint32_t* ev, uint64_t* keys, uint32_t* rows,
                       cudaStream_t st);
// counters[CTR_ROWS] and counters[CTR_USED] copied to host-mapped `out` ([0], [1]), then out[2] = stamp: the host's
// bound on what a growable table's enqueued calls can admit reads them once the stamp is there
void launch_grow_readback(const uint32_t* counters, uint32_t* out, uint32_t stamp, cudaStream_t st);
// checkpoint images (pb_dump.cu).  The part of a sign in a background dump: splitmix64(sign) % n_parts, with
// splitmix64(x): z = x + 0x9E3779B97F4A7C15; z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9;
// z = (z ^ (z >> 27)) * 0x94D049BB133111EB; return z ^ (z >> 31)   (include/persia_b200.h, pb_table_dump_part)
__host__ __device__ __forceinline__ uint64_t dump_splitmix64(uint64_t x) {
  uint64_t z = x + 0x9E3779B97F4A7C15ULL;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
  return z ^ (z >> 31);
}
enum { DW_COUNT = 0, DW_NODES, DW_WORDS };
// a table's dump workspace (pb_table_dump_reserve): `max_items` entries of each array, the sort's temporary storage
struct DumpWs {
  uint64_t* key;    // collected: sign ^ 2^63
  uint64_t* key_s;  // (sorted keys: discarded)
  uint64_t* loc;    // collected: row | (1 = the tier's row) << 32; pb_dump_nodes: the located rows
  uint32_t *rec, *rec2, *rec_s;     // last-use request: collected, in sign order, (sorted: discarded)
  uint32_t *idx0, *idx1, *idx2;     // item numbers: identity, in sign order, in (request, sign) order
  uint32_t* words;  // DW_* counters
  void* sort_tmp;
  uint64_t sort_bytes;
  uint32_t max_items;
};
uint64_t dump_node_bytes(uint32_t entry_len);
uint64_t dump_sort_bytes(uint32_t max_items);
// h: the tier behind t (null: none)
cudaError_t launch_dump_part(const TableDev& t, const TableDev* h, uint32_t part, uint32_t n_parts, const DumpWs& w,
                             uint8_t* image, uint64_t max_bytes, unsigned long long* d_bytes, uint32_t* d_request,
                             cudaStream_t st);
// the part of a table that was never allocated: the empty list
cudaError_t launch_dump_empty(uint8_t* image, uint64_t max_bytes, unsigned long long* d_bytes, uint32_t* d_request,
                              cudaStream_t st);
cudaError_t launch_dump_nodes(const TableDev& t, const TableDev* h, const uint64_t* signs, uint32_t n_list, uint32_t lo,
                              uint32_t n, const DumpWs& w, uint8_t* out, cudaStream_t st);
// checkpoint loads (pb_load.cu): one list image or incremental-update packet, read in place (mapped pinned host
// memory), and its per-dim summary
constexpr uint32_t LOAD_DIMS = 32, LOAD_PAIRS = 64;  // distinct dims, distinct (dim, entry length) pairs of one image
constexpr uint32_t LOAD_NONE = 0xFF;                  // slot of a position not selected
constexpr uint32_t LOAD_NODE_HDR = 9;                 // bytes before an entry's `len`: a `.emb` node's next, prev, flag
enum { LOAD_FLAG_BAD = 0, LOAD_FLAG_FULL, LOAD_FLAGS };
struct LoadImg {
  const uint8_t* img;   // device address of the image's bytes (a window: its first node's; a packet: its first entry's
                        // when off is null)
  const uint64_t* off;  // byte offset of each list position's record; null: arithmetic offsets (pos * nb)
  uint64_t nb;          // arithmetic offsets: record bytes
  uint32_t hdr;         // bytes before each record's `len`: LOAD_NODE_HDR (a `.emb` node), 0 (a packet entry)
  uint32_t n;           // list positions
  uint32_t p_lo, p_hi;  // positions offered (the others are not selected)
  uint64_t node0, n_total, dim;  // writer-layout window (hdr != 0): the window's first node, the file's nodes, its dim
  uint32_t len;                  // arithmetic offsets: every record's entry length
  uint32_t R, rank;              // selection: farmhash64(sign) % R == rank
  uint8_t* slot;                 // per position: summary slot of its dim, LOAD_NONE = not selected
  unsigned long long* dims;      // LOAD_DIMS, KEY_EMPTY = unused
  unsigned long long* pairs;     // LOAD_PAIRS: slot << 32 | entry length, KEY_EMPTY = unused
  uint32_t* counts;              // LOAD_PAIRS: selected entries of each pair
  uint32_t* flags;               // LOAD_FLAGS
};
bool load_index_host(const uint8_t* image, uint64_t nbytes, std::vector<uint64_t>& pos_off, std::string& err);
bool packet_index_host(const uint8_t* packet, uint64_t nbytes, std::vector<uint64_t>& pos_off, std::string& err);
cudaError_t launch_load_select(const LoadImg& L, cudaStream_t st);
size_t load_list_bytes(uint32_t n);
cudaError_t launch_load_list(const LoadImg& L, uint32_t slot, void* tmp, size_t tmp_bytes, uint32_t* sel,
                             uint32_t* d_count, cudaStream_t st);
cudaError_t launch_load_gather(const LoadImg& L, const uint32_t* sel, uint32_t K, uint32_t lo, uint32_t n, int rev,
                               uint32_t len, uint64_t* signs, float* ent, cudaStream_t st);
uint64_t launch_count();
enum { FAM_PROBE = 0, FAM_DEDUP, FAM_GATHER, FAM_NAN, FAM_HOT, FAM_UPDATE, FAM_OTHER, FAM_WARM, FAM_WAIT, FAM_ROUTE, FAM_OWNER, FAM_COUNT };
bool profiling();  // a kernel family is being timed: the backward then runs its kernels one after another
void profile_enable(uint32_t family_mask);
void profile_read(double* ms, uint64_t* count, int n_families);

enum { MODE_FIND = 0, MODE_TRAIN = 1, MODE_SET = 2, MODE_MOVE = 3 };

}  // namespace pb
