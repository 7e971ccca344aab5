// pb_api.cu — the C ABI of libpersia_b200.so (include/persia_b200.h): object lifetime, argument checks,
// kernel sequencing.  No torch types, no allocation on the hot path after the first call of a given size.
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <random>
#include <string>
#include <utility>
#include <vector>

#include <unistd.h>

#include "pb_kernels.cuh"
#include "pb_own.cuh"

using namespace pb;

namespace {

struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(int dev) {
    cudaGetDevice(&prev);
    if (prev != dev) cudaSetDevice(dev);
    else prev = -1;
  }
  ~DeviceGuard() {
    if (prev >= 0) cudaSetDevice(prev);
  }
};

uint32_t next_pow2(uint64_t v) {
  uint64_t p = 1;
  while (p < v) p <<= 1;
  return (uint32_t)p;
}

// rand 0.8 UniformFloat::new: shrink the scale until the largest draw stays below `hi`
float uniform_scale(float lo, float hi) {
  float scale = hi - lo;
  uint32_t mb = (0xFFFFFFFFu >> 9) | 0x3f800000u;
  float max_rand;
  std::memcpy(&max_rand, &mb, 4);
  max_rand -= 1.0f;
  if (!(hi > lo)) return 0.0f;
  while (!(scale * max_rand + lo < hi)) {
    uint32_t b;
    std::memcpy(&b, &scale, 4);
    b -= 1;
    std::memcpy(&scale, &b, 4);
  }
  return scale;
}

// an event recorded on a caller's stream, and the stream capture it was recorded into (0 = none: a real record)
struct Mark {
  cudaEvent_t ev = nullptr;
  unsigned long long capture = 0;
  bool set = false;
};

// Grid of pb_tier_stage's kernels: they run beside the backward and the dense step of the batch before, so they take a
// fixed share of the GPU rather than the usual grids (8 blocks per SM for the index scans).  One block per SM: measured
// on an H100 with scripts/host_tier_bench.py (DESIGN.md §4 "Staging"), a step with the stage on 8, 16, 32, 64 and 132
// blocks took 6.49, 3.97, 2.93, 2.58 and 2.43 ms beside a 1.06 ms dense stand-in: the stage's eviction check moves
// ~45k entries out per step, and fewer blocks leave too few copies in flight to keep PCIe busy, so the stage outlasts
// the dense step and the backward and delays the next forward.
uint32_t g_stage_blocks = PB_NUM_SMS;

}  // namespace

struct pb_table {
  int device = 0;
  pb_table_cfg cfg{};
  OptimDev op{};
  bool has_op = false;
  HyperDev hy{};
  bool has_hy = false;
  TableDev d{};
  bool allocated = false;
  uint32_t* scratch = nullptr;  // index cells of a single-request call
  uint32_t scratch_cap = 0;
  // Adam: accumulated (beta1^t, beta2^t) per feature group, keyed by index prefix (optim.rs:99-131, 155-197)
  // (the pairs live on the device: a captured backward advances them on every replay)
  std::vector<uint64_t> adam_keys;  // position = pair number; pair PB_ADAM_KEYS-1 serves pb_update
  float* adam_dev = nullptr;
  // capacity policy (pb_table_set_eviction): 0 = refuse admissions when full
  uint32_t evict_every = 0, evict_low = 0, evict_target = 0, evict_keep = 2;
  uint32_t train_calls = 0;
  uint32_t* evict_ws = nullptr;
  uint64_t* rebuild_keys = nullptr;  // the index rebuild's compacted (sign, row) pairs, `capacity` each
  uint32_t* rebuild_rows = nullptr;
  uint32_t* stats_ws = nullptr;      // pb_table_index_stats
  uint32_t pending_batches = 0;  // training forwards whose backward has not been enqueued yet
  // host-memory tier (pb_tier.cu): `host` = this table's rows are mapped pinned host memory (pb_table_create_host);
  // `tier` = the host table attached behind this one, `tier_of` = the table this one is attached behind
  bool host = false;
  float* host_rows = nullptr;  // host address of d.rows
  // pb_table_create_host_shared: the host rows are a memfd mapping (`shared_fd`) that peer processes can map too
  bool shared = false;
  int shared_fd = -1;
  pb_table* tier = nullptr;
  pb_table* tier_of = nullptr;
  uint32_t* move_cells = nullptr;  // the eviction check's victim list (with rebuild_keys / rebuild_rows), `capacity` words
  // ordering of calls on several streams (TableCall): `index` after every call that probes or changes the index (or
  // moves entries between the table and its tier), `step` after every call that steps rows, advances Adam's beta
  // powers or marks the incremental set
  Mark index, step;
  // incremental updates (pb_table_enable_incremental): the set of signs stepped since the last take; cells == null: off
  IncDev inc{};
  unsigned long long* inc_host = nullptr;  // host address of inc.mirror
  // checkpoint images (pb_table_dump_reserve): one allocation holding every DumpWs array; null: none reserved
  DumpWs dump{};
  void* dump_mem = nullptr;
  // pb_table_export_view: peers read the index and rows in place from then on, so nothing may move cells or step rows
  // (writable); `seq` is the write-sequence word pb_set_rows keeps odd while it writes
  bool exported = false;
  uint32_t* seq = nullptr;
  // pb_table_export_live_view: peers read in place while the table keeps training; sweeps, rebuilds, pb_set_rows and
  // pb_table_clear keep `seq` odd while they move cells or reuse rows (one table, one export mode)
  bool live = false;
  // growable storage (pb_table_set_growth): the rows, row_tick, free-row stack, rebuild pairs and index cells each have
  // address space reserved for `capacity` rows (the index: for its largest size, max_cells), backed by memory from the
  // start up to `mapped` bytes (grow_for)
  bool grow = false;
  struct Region {
    char* base = nullptr;
    size_t mapped = 0;
  };
  enum { G_ROWS, G_TICK, G_FREE, G_RKEYS, G_RROWS, G_CELLS, G_COUNT };
  Region region[G_COUNT];
  uint32_t max_cells = 0;
  size_t gran = 0;  // every chunk's size is a multiple of it
  // the host's bound on the rows (CTR_ROWS) and used cells (CTR_USED) of every call enqueued: the last values read back
  // (base_*) plus every sign an admitting call issued since (issued - base_issued).  A read-back (k_grow_readback into
  // mapped pinned rb_host, stamped rb_stamp) is enqueued by an admitting call when none is outstanding and read by a
  // later one once its stamp is there; it covers the calls issued before it (rb_issued), which the index chain orders
  // before it
  uint64_t issued = 0, base_issued = 0, rb_issued = 0;
  uint32_t base_rows = 0, base_used = 0, rb_stamp = 0;
  bool rb_pending = false;
  uint32_t* rb_host = nullptr;  // [3]: rows, used cells, stamp
  uint32_t* rb_dev = nullptr;
  cudaStream_t grow_st = nullptr;  // growth asked for under stream capture runs here, outside the graph
  Owned own;  // every CUDA resource above
};

struct pb_ctx {
  // A training forward's batch, pending in the context until its backward: counted in its table's pending_batches, so
  // that eviction spares its rows.
  struct Pending {
    bool on = false;
    pb_table* table = nullptr;
    void hold(pb_table* t) {
      on = true;
      table = t;
      t->pending_batches++;
    }
    int check(const pb_table* t, const char* not_pending_msg, const char* other_table_msg) const {
      if (!on) return fail(PB_ERR_STATE, not_pending_msg);
      if (table != t) return fail(PB_ERR_INVALID, other_table_msg);
      return PB_OK;
    }
    void drop() {
      if (table && table->pending_batches) table->pending_batches--;
      on = false;
      table = nullptr;
    }
  };
  int device = 0;
  uint32_t max_occ = 0, max_out = 0;
  pb_slots_cfg slots{};
  bool has_slots = false;
  // forward -> backward state (the EW's post_forward_buffer entry, mod.rs:1087-1098): the batch's distinct signs,
  // where each lives, the occurrence lists and the work lists of the backward (pb_kernels.cuh BatchDev)
  BatchDev b{};
  size_t set_cells = 0;
  bool set_dirty = false;  // the scratch set still holds the last batch's cells
  uint32_t* occ_outrow = nullptr;
  uint32_t* row_off = nullptr;
  bool multi_id = false;
  uint32_t n_occ = 0, batch = 0;
  uint32_t* dev_tick = nullptr;  // request number of the pending forward (device side, CUDA-graph safe)
  uint32_t occ_off[PB_MAX_SLOTS + 1];
  Pending pending;  // a summation batch awaiting its backward
  // slots of one feature group take turns in the backward (mod.rs:720-822): round of every slot
  uint32_t n_rounds = 1;
  uint8_t round_of[PB_MAX_SLOTS];
  GroupLinks links;  // sharded path: previous / next slot of every slot's group (k_link_items)
  // backward workspace
  uint32_t* nan_tick = nullptr;
  float* vw_stage = nullptr;
  size_t vw_stage_floats = 0;
  float* hot_stage = nullptr;  // the hot items' sums, b.hot_cap x dim floats (allocated by the training pb_forward)
  size_t hot_stage_floats = 0;
  cudaStream_t side = nullptr;  // hot items run beside the main stream during pb_backward
  cudaStream_t side2 = nullptr;  // scratch-set clearing, then the warm items beside the cold ones
  cudaStream_t side3 = nullptr;  // the short hot items' sums beside everything else (one round, large batches)
  cudaEvent_t ev_fork = nullptr, ev_nan = nullptr, ev_join = nullptr, ev_join2 = nullptr;
  cudaEvent_t ev_short = nullptr;  // `side3` staged the short hot items' sums (k_step_hot on `side` waits for it)
  // raw slot (pb_forward_raw / pb_backward_raw): allocated on first use
  uint32_t* occ_cell = nullptr;
  RawWork raw{};
  bool raw_ready = false;
  Pending raw_pending;  // a raw batch awaiting its backward
  float* raw_stage = nullptr;
  size_t raw_stage_floats = 0;
  // sharded path, PB_PHASE_PREPARE: the batch deduplicated ahead of its SEND (PREP_SUM / PREP_RAW: which call's, with
  // its ids) and its distinct items per owner
  int prepared = 0;
  uint32_t prepared_n = 0, prepared_batch = 0;
  uint32_t* need = nullptr;  // [PB_MAX_RANKS]
  // pb_forward_remote / pb_forward_raw_remote: the rows read from their owners, one per distinct item (grow_stage)
  float* remote_stage = nullptr;
  size_t remote_stage_floats = 0;
  Owned own;  // every CUDA resource above
};
enum { PREP_NONE = 0, PREP_SUM = 1, PREP_RAW = 2 };

namespace {

// ---- growable storage (pb_table_set_growth) --------------------------------------------------------------------------
// bytes per row of each row-indexed region
size_t region_row_bytes(const pb_table* t, int r) {
  switch (r) {
    case pb_table::G_ROWS: return sizeof(float) * (size_t)t->d.stride;
    case pb_table::G_RKEYS: return sizeof(uint64_t);
    default: return sizeof(uint32_t);  // row_tick, free_rows, rebuild_rows
  }
}

// The chunks that back `rows` rows and `cells` index cells (+ N_SPECIAL), acquired into `o`; `mapped[r]` receives
// each region's new extent.  Nothing is enqueued.
int map_growth(pb_table* t, uint64_t rows, uint64_t cells, Owned& o, size_t mapped[pb_table::G_COUNT]) {
  for (int r = 0; r < pb_table::G_COUNT; ++r) {
    const size_t want = r == pb_table::G_CELLS ? sizeof(Cell) * ((size_t)cells + N_SPECIAL) : region_row_bytes(t, r) * rows;
    const size_t to = (want + t->gran - 1) / t->gran * t->gran;
    pb_table::Region& g = t->region[r];
    mapped[r] = g.mapped;
    if (to <= g.mapped) continue;
    if (int rc = o.chunk(g.base + g.mapped, to - g.mapped, t->device)) return rc;
    mapped[r] = to;
  }
  return PB_OK;
}

// largest extent of each region: `capacity` rows, the index at max_cells
size_t region_reserved(const pb_table* t, int r) {
  if (r == pb_table::G_CELLS) return sizeof(Cell) * ((size_t)t->max_cells + N_SPECIAL);
  return region_row_bytes(t, r) * t->d.capacity;
}

// A growable table's first allocation: every region reserved at its largest extent (rounded to the granularity), the
// first chunk of rows and the index they need backed, counters, the sweep's workspace, the read-back word and the stream
// of captured growth; the cells filled, row_tick zeroed.  The index starts at the size an eager table of `mapped`
// rows would have.
int acquire_growable(pb_table* t, Owned& o) {
  TableDev& d = t->d;
  t->max_cells = d.n_cells;
  if (!(t->gran = vmm_granularity(t->device))) return fail(PB_ERR_CUDA, "no virtual memory management on this device");
  int rc;
  for (int r = 0; r < pb_table::G_COUNT; ++r) {
    const size_t span = (region_reserved(t, r) + t->gran - 1) / t->gran * t->gran;
    t->region[r] = pb_table::Region{};
    if ((rc = o.reserve(t->region[r].base, span))) return rc;
  }
  uint64_t rows = t->gran / region_row_bytes(t, pb_table::G_ROWS);
  rows = rows < 1 ? 1 : rows > d.capacity ? d.capacity : rows;
  uint64_t want = rows + rows / 2;
  const uint32_t cells = next_pow2(want < 1024 ? 1024 : want);
  size_t mapped[pb_table::G_COUNT];
  if ((rc = map_growth(t, rows, cells, o, mapped)) || (rc = o.dev(d.counters, sizeof(uint32_t) * CTR_COUNT)) ||
      (rc = o.dev(t->evict_ws, sizeof(uint32_t) * EVICT_WS_WORDS)) ||
      (rc = o.mapped(t->rb_host, t->rb_dev, 3 * sizeof(uint32_t))) || (rc = o.stream(t->grow_st)))
    return rc;
  for (int r = 0; r < pb_table::G_COUNT; ++r) t->region[r].mapped = mapped[r];
  d.cells = reinterpret_cast<Cell*>(t->region[pb_table::G_CELLS].base);
  d.rows = reinterpret_cast<float*>(t->region[pb_table::G_ROWS].base);
  d.row_tick = reinterpret_cast<uint32_t*>(t->region[pb_table::G_TICK].base);
  d.free_rows = nullptr;  // (the gate: set once adopted)
  t->rebuild_keys = reinterpret_cast<uint64_t*>(t->region[pb_table::G_RKEYS].base);
  t->rebuild_rows = reinterpret_cast<uint32_t*>(t->region[pb_table::G_RROWS].base);
  d.mapped = (uint32_t)rows;
  d.n_cells = cells;
  d.cell_mask = cells - 1;
  d.bucket_mask = cells / BUCKET - 1;
  t->issued = t->base_issued = t->rb_issued = 0;
  t->base_rows = t->base_used = 0;
  t->rb_pending = false;
  t->rb_host[2] = t->rb_stamp;
  PB_CUDA(cudaMemset(d.row_tick, 0, sizeof(uint32_t) * rows));
  PB_CUDA(cudaMemset(d.counters, 0, sizeof(uint32_t) * CTR_COUNT));
  launch_fill_cells(d.cells, (uint64_t)d.n_cells + N_SPECIAL, 0);
  PB_CUDA(cudaDeviceSynchronize());
  return PB_OK;
}

// The table's index, rows, counters and row_tick, acquired into `o`: the caller adopts `o`, then sets `allocated`.
int acquire_storage(pb_table* t, Owned& o) {
  if (!t->has_op) return fail(PB_ERR_STATE, "optimizer not registered (OptimizerNotFoundError)");
  uint32_t dim = t->cfg.dim;
  uint32_t state = 0;
  switch (t->op.kind) {
    case PB_OPT_ADAGRAD: state = dim; break;
    case PB_OPT_ADAGRAD_VW: state = 1; break;
    case PB_OPT_ADAM: state = 2 * dim; break;
    default: state = 0;
  }
  TableDev& d = t->d;
  d.dim = dim;
  d.state_floats = state;
  d.stride = (dim + state + 3u) & ~3u;
  if (t->cfg.capacity >= 0xFFFFFFF0ull) return fail(PB_ERR_INVALID, "capacity must be < 2^32 - 16 rows per shard");
  d.capacity = (uint32_t)t->cfg.capacity;
  uint64_t want = (uint64_t)d.capacity + d.capacity / 2;
  if (want < 1024) want = 1024;
  if (want > (1ull << 31)) return fail(PB_ERR_INVALID, "capacity too large for a 2^31-cell index");
  d.n_cells = next_pow2(want);
  d.cell_mask = d.n_cells - 1;
  d.bucket_mask = d.n_cells / BUCKET - 1;
  const size_t rows_bytes = sizeof(float) * (size_t)d.capacity * d.stride;
  d.mapped = d.capacity;
  if (t->grow) return acquire_growable(t, o);
  int rc;
  if ((rc = o.dev(d.cells, sizeof(Cell) * ((size_t)d.n_cells + N_SPECIAL))) ||
      // a host table's rows are not write-combined: the host reads them back (checkpoints)
      (rc = t->shared ? o.shared(t->host_rows, d.rows, rows_bytes, -1, t->shared_fd)
            : t->host ? o.mapped(t->host_rows, d.rows, rows_bytes)
                      : o.dev(d.rows, rows_bytes)) ||
      (rc = o.dev(d.counters, sizeof(uint32_t) * CTR_COUNT)) || (rc = o.dev(d.row_tick, sizeof(uint32_t) * (size_t)d.capacity)))
    return rc;
  PB_CUDA(cudaMemset(d.row_tick, 0, sizeof(uint32_t) * (size_t)d.capacity));
  PB_CUDA(cudaMemset(d.counters, 0, sizeof(uint32_t) * CTR_COUNT));
  launch_fill_cells(d.cells, (uint64_t)d.n_cells + N_SPECIAL, 0);
  d.free_rows = nullptr;
  PB_CUDA(cudaDeviceSynchronize());
  return PB_OK;
}

int ensure_alloc(pb_table* t) {
  if (t->allocated) return PB_OK;
  Owned o;
  if (int rc = acquire_storage(t, o)) return rc;
  t->own.adopt(o);
  if (t->grow) t->d.free_rows = reinterpret_cast<uint32_t*>(t->region[pb_table::G_FREE].base);
  t->allocated = true;
  return PB_OK;
}

int ensure_scratch(pb_table* t, uint32_t n) {
  if (n <= t->scratch_cap) return PB_OK;
  t->own.release(t->scratch);
  t->scratch_cap = 0;
  uint32_t cap = next_pow2(n);
  if (int rc = t->own.dev(t->scratch, sizeof(uint32_t) * (size_t)cap)) return rc;
  t->scratch_cap = cap;
  return PB_OK;
}

// the free-row stack (into `free_rows`, the gate, once the rest is held), the sweep's workspace and the rebuild's
// pair buffer, acquired into `o`
int acquire_evict_ws(pb_table* t, Owned& o, uint32_t*& free_rows) {
  const size_t cap = t->d.capacity;
  int rc;
  if ((rc = o.dev(t->evict_ws, sizeof(uint32_t) * EVICT_WS_WORDS)) || (rc = o.dev(t->rebuild_keys, sizeof(uint64_t) * cap)) ||
      (rc = o.dev(t->rebuild_rows, sizeof(uint32_t) * cap)))
    return rc;
  return o.dev(free_rows, sizeof(uint32_t) * cap);
}

// allocated by the first sweep
int ensure_evict_ws(pb_table* t) {
  if (t->d.free_rows) return PB_OK;
  Owned o;
  if (int rc = acquire_evict_ws(t, o, t->d.free_rows)) return rc;
  t->own.adopt(o);
  return PB_OK;
}

int wait_for(const Mark& m, cudaStream_t st);

// A live-exported table with a host tier (a shared one: no other tier can be exported) holds its write-sequence word
// odd around every launch that moves an entry between the table and its tier or hands a row of either to another sign
// (the eviction check with its moves, sweeps and rebuilds; every restore): a reader that probed the HBM index before
// such a move and the tier after it would otherwise find the sign in neither table (pb_remote.cu).  Two one-thread
// launches (k_seq_begin, k_seq_end) around each; every other table launches nothing here.
// The two kernels step the word with a plain read and +1, not atomically, so windows on one word must never overlap:
// they are opened only by calls in the table's index chain (TableCall CALL_INDEX: training forwards, the sharded
// SERVE, pb_set_rows, pb_table_clear, and the stages, which wait for every earlier call and which every later one but
// a backward waits for), each on its call's stream, so every window is stream-ordered after the one before it.  The
// backward (step chain only, beside a stage or the next forward) opens none.  A call outside the index chain must not
// open one.
struct TierWindow {
  uint32_t* seq = nullptr;
  cudaStream_t st = nullptr;
  TierWindow(const pb_table* t, cudaStream_t s) : st(s) {
    if (t->live && t->tier) launch_seq_bump(seq = t->seq, true, st);
  }
  ~TierWindow() {
    if (seq) launch_seq_bump(seq, false, st);
  }
};

// The eviction check: release the least recently used rows when free storage runs low, and rebuild the index when its
// EMPTY cells run short.  blocks: grid of its scans (0 = the usual; pb_tier_stage's is small).
int evict_check(pb_table* t, cudaStream_t st, uint32_t blocks = 0) {
  int rc = ensure_evict_ws(t);
  if (rc) return rc;
  // `pending_batches` drops when a backward is enqueued, perhaps on another stream: the check first waits for every
  // enqueued step, so the rows it may release are those it would release were every call on one stream
  if ((rc = wait_for(t->step, st))) return rc;
  // rows of batches whose gradients are still to come are never released: a row used by a pending batch was
  // refreshed by its forward, i.e. at most `pending_batches` requests ago
  const uint32_t keep = t->evict_keep > t->pending_batches + 1 ? t->evict_keep : t->pending_batches + 1;
  if (t->tier) {  // the victims move into the tier
    pb_table* h = t->tier;
    TierWindow win(t, st);
    launch_evict_tier(t->d, h->d, t->hy, t->op, t->evict_low, t->evict_target, keep, t->evict_ws, t->rebuild_keys,
                      t->rebuild_rows, h->evict_ws, h->rebuild_keys, h->rebuild_rows, t->move_cells, st, blocks);
    return PB_OK;
  }
  launch_evict(t->d, t->evict_low, t->evict_target, keep, t->evict_ws, t->rebuild_keys, t->rebuild_rows,
               t->live ? t->seq : nullptr, st);
  return PB_OK;
}

// between two training requests: every `evict_every`-th one runs the check
int maybe_evict(pb_table* t, cudaStream_t st) {
  if (!t->evict_every || (++t->train_calls % t->evict_every)) return PB_OK;
  return evict_check(t, st);
}

// ---- event marks ---------------------------------------------------------------------------------------------------
// A Mark is recorded on the stream of one call, and later calls on other streams wait for it (TableCall, below).
// Waiting on a completed event costs nothing.
// Stream capture (CUDA 12.9): a capturing stream may wait only on an event recorded into the same capture (a fork/join
// inside the graph).  Waiting on an event recorded outside it is invalid without cudaEventWaitExternal, and that flag
// would make every replay wait on whatever the event's latest record is by then: not the dependency meant here.  So an
// event recorded outside the capture is queried instead: complete, there is nothing to wait for; still running, the
// call fails with PB_ERR_STATE rather than record a dependency it cannot keep.  The query runs under
// cudaThreadExchangeStreamCaptureMode(relaxed): a global-mode capture forbids it otherwise; querying an event recorded
// inside a capture stays forbidden, and is never done.  A mark recorded into another capture is part of that graph,
// whose launches the caller orders: nothing is waited for.

cudaError_t capture_id(cudaStream_t st, unsigned long long& id) {
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  id = 0;
  const cudaError_t e = cudaStreamGetCaptureInfo(st, &cs, &id);
  if (cs != cudaStreamCaptureStatusActive) id = 0;
  return e;
}

int record(Mark& m, cudaStream_t st) {
  PB_CUDA(capture_id(st, m.capture));
  PB_CUDA(cudaEventRecord(m.ev, st));
  m.set = true;
  return PB_OK;
}

// `st` waits for the work behind `m`
int wait_for(const Mark& m, cudaStream_t st) {
  if (!m.set) return PB_OK;
  unsigned long long cap = 0;
  PB_CUDA(capture_id(st, cap));
  if (m.capture) {  // recorded into a capture: a dependency inside that graph only
    if (m.capture == cap) PB_CUDA(cudaStreamWaitEvent(st, m.ev, 0));
    return PB_OK;
  }
  if (!cap) {
    PB_CUDA(cudaStreamWaitEvent(st, m.ev, 0));
    return PB_OK;
  }
  cudaStreamCaptureMode mode = cudaStreamCaptureModeRelaxed;
  PB_CUDA(cudaThreadExchangeStreamCaptureMode(&mode));
  const cudaError_t q = cudaEventQuery(m.ev);
  cudaThreadExchangeStreamCaptureMode(&mode);
  if (q == cudaSuccess) return PB_OK;
  if (q == cudaErrorNotReady)
    return fail(PB_ERR_STATE, "earlier work on this table issued outside this stream capture has not completed: "
                              "synchronise before capturing, or capture that work too");
  return fail(PB_ERR_CUDA, std::string("cudaEventQuery: ") + cudaGetErrorString(q));
}

// ---- ordering of calls on several streams ------------------------------------------------------------------------
// Batches of different contexts may be in flight on different streams (embedding_staleness > 1).  A call's work falls
// in two chains, each kept in the order the calls were issued, whatever their streams:
//   CALL_INDEX  index work: probes (training or not), admissions, eviction checks and rebuilds, row_tick, tier moves;
//   CALL_STEP   row steps, Adam's beta-power advance and the incremental set's marks.
// A call waits for the latest call of each chain it belongs to and becomes that chain's latest.  So two steps never
// overlap (no update is lost or torn; every row is stepped in issue order) and no probe runs beside a rebuild, while a
// backward (CALL_STEP only) still runs beside the next batch's forward (CALL_INDEX only): no backward kernel reads
// index cells, the free-row stack or row_tick.  A forward reads rows that a backward beside it may be stepping: a
// stale read, as staleness allows.  An eviction check also waits for the step chain (evict_check).  Calls that read
// or write entries or counters outside a batch (set/get rows, export, statistics, takes, clear) are in both chains.
// A stage (pb_tier_stage) waits for both chains and is in the index chain only, so it starts after every earlier call
// and every later call but a backward starts after it.
// Under stream capture the marks follow wait_for: within one capture they become edges of the graph; graphs captured
// separately are ordered by whoever launches them.
enum : unsigned { CALL_INDEX = 1, CALL_STEP = 2, CALL_ALL = 3 };

// One call on a table: begin() makes `st` wait for the latest call of every chain in `ch | after`; when the call
// returns it is recorded as the latest of the chains in `ch`.  A host tier's calls use its table's marks.
struct TableCall {
  pb_table* m = nullptr;
  cudaStream_t st = nullptr;
  unsigned chains = 0;
  int begin(pb_table* t, cudaStream_t s, unsigned ch, unsigned after = 0) {
    pb_table* o = t->tier_of ? t->tier_of : t;
    int rc;
    if (((ch | after) & CALL_INDEX) && (rc = wait_for(o->index, s))) return rc;
    if (((ch | after) & CALL_STEP) && (rc = wait_for(o->step, s))) return rc;
    m = o;
    st = s;
    chains = ch;
    return PB_OK;
  }
  ~TableCall() {
    if (!m) return;
    if (chains & CALL_INDEX) record(m->index, st);
    if (chains & CALL_STEP) record(m->step, st);
  }
};

// Before a call on a growable table launches anything that can admit up to `n` signs (a training forward or lookup,
// pb_set_rows, an owner's training SERVE), in the index chain: back every row the enqueued calls and this one can hand
// out, and grow the index so that the cells they can use stay within 2/3 of it.  Rows grow by at least 1/8 of what is
// mapped (a logarithmic number of mappings), the index by doubling.  A chunk that cannot be had fails the call with
// PB_ERR_CUDA before any kernel or copy is enqueued (the call's TableCall has made its stream wait for the table's
// earlier calls and records its mark: ordering only); the table stays as it was.  Under stream capture the whole capacity is
// backed (a replay never passes here), the work enqueued outside the graph and waited for.  Any other table: nothing.
int grow_for(pb_table* t, uint64_t n, cudaStream_t st) {
  if (!t->grow) return PB_OK;
  unsigned long long cap_id = 0;
  PB_CUDA(capture_id(st, cap_id));
  TableDev& d = t->d;
  if (cap_id && d.mapped == d.capacity && d.n_cells == t->max_cells) return PB_OK;
  if (t->rb_pending && reinterpret_cast<volatile uint32_t*>(t->rb_host)[2] == t->rb_stamp) {
    std::atomic_thread_fence(std::memory_order_acquire);
    t->base_rows = reinterpret_cast<volatile uint32_t*>(t->rb_host)[0];
    t->base_used = reinterpret_cast<volatile uint32_t*>(t->rb_host)[1];
    t->base_issued = t->rb_issued;
    t->rb_pending = false;
  }
  const uint64_t since = t->issued - t->base_issued + n;
  uint64_t rows = std::min<uint64_t>(d.capacity, t->base_rows + since);
  const uint64_t used = std::max<uint64_t>(rows, t->base_used + since);
  uint64_t cells = d.n_cells;
  while (cells < t->max_cells && 3 * used > 2 * cells) cells *= 2;
  if (cap_id) {
    rows = d.capacity;
    cells = t->max_cells;
  } else if (rows > d.mapped) {
    rows = std::min<uint64_t>(d.capacity, std::max<uint64_t>(rows, (uint64_t)d.mapped + d.mapped / 8));
  } else {
    rows = d.mapped;
  }
  if (rows > d.mapped || cells > d.n_cells) {
    // captured: relaxed mode lets this thread map memory and use an uncaptured stream meanwhile
    cudaStreamCaptureMode mode = cudaStreamCaptureModeRelaxed;
    if (cap_id) PB_CUDA(cudaThreadExchangeStreamCaptureMode(&mode));
    struct Restore {
      bool on;
      cudaStreamCaptureMode& m;
      ~Restore() {
        if (on) cudaThreadExchangeStreamCaptureMode(&m);
      }
    } restore{cap_id != 0, mode};
    const cudaStream_t ws = cap_id ? t->grow_st : st;
    Owned o;
    size_t mapped[pb_table::G_COUNT];
    if (int rc = map_growth(t, rows, cells, o, mapped)) return rc;
    t->own.adopt(o);
    for (int r = 0; r < pb_table::G_COUNT; ++r) t->region[r].mapped = mapped[r];
    if (rows > d.mapped)
      PB_CUDA(cudaMemsetAsync(d.row_tick + d.mapped, 0, sizeof(uint32_t) * (size_t)(rows - d.mapped), ws));
    d.mapped = (uint32_t)rows;
    if (cells > d.n_cells) {
      TableDev to = d;
      to.n_cells = (uint32_t)cells;
      to.cell_mask = cells - 1;
      to.bucket_mask = (uint32_t)(cells / BUCKET - 1);
      launch_grow_index(d, to, t->evict_ws, t->rebuild_keys, t->rebuild_rows, ws);
      d = to;
    }
    PB_CUDA(cudaGetLastError());
    if (cap_id) PB_CUDA(cudaStreamSynchronize(ws));
  }
  if (!cap_id && !t->rb_pending) {
    launch_grow_readback(d.counters, t->rb_dev, ++t->rb_stamp, st);
    t->rb_issued = t->issued;
    t->rb_pending = true;
  }
  t->issued += n;
  return PB_OK;
}

// a table's counter words (`n` of them at `src`), copied to the host under a call in both chains; synchronises `st`
template <typename W>
int read_counters(pb_table* t, const W* src, W* dst, size_t n, cudaStream_t st) {
  DeviceGuard g(t->device);
  TableCall call;
  if (int rc = call.begin(t, st, CALL_ALL)) return rc;
  PB_CUDA(cudaMemcpyAsync(dst, src, sizeof(W) * n, cudaMemcpyDeviceToHost, st));
  PB_CUDA(cudaStreamSynchronize(st));
  return PB_OK;
}

// a training request's signs the HBM table lacks and its tier holds are moved back into HBM rows before they are probed
void restore_ids(pb_table* t, bool prefix, const SlotsDev& sl, const uint64_t* ids, uint32_t n, cudaStream_t st) {
  if (!t->tier) return;
  TierWindow win(t, st);
  launch_tier_restore(t->d, t->tier->d, t->hy, t->op, sl, prefix, ids, n, st);
}

// Calls that move index cells or step rows: refused once peers read the table in place (pb_table_export_view).
int writable(const pb_table* t) {
  if (t->exported)
    return fail(PB_ERR_STATE, "the table was exported for remote reads (pb_table_export_view): it is read-only for the "
                              "rest of its life (pb_set_rows and pb_image_insert stay allowed)");
  return PB_OK;
}

int ready_for_training(pb_table* t) {
  if (t->tier_of) return fail(PB_ERR_STATE, "a host tier is not trained directly: use the table it is attached to");
  if (!t->has_op) return fail(PB_ERR_STATE, "optimizer not registered (OptimizerNotFoundError)");
  if (!t->has_hy) return fail(PB_ERR_STATE, "embedding server not configured (NotConfiguredError)");
  return PB_OK;
}

// pair number of a feature group (keyed by its index prefix); -1 when the table is out of pairs
int adam_index(pb_table* t, uint64_t prefix) {
  for (size_t i = 0; i < t->adam_keys.size(); ++i)
    if (t->adam_keys[i] == prefix) return (int)i;
  if (t->adam_keys.size() + 1 >= PB_ADAM_KEYS) return -1;
  t->adam_keys.push_back(prefix);
  return (int)t->adam_keys.size() - 1;
}

SlotsDev no_slots() {
  SlotsDev s;
  std::memset(&s, 0, sizeof(s));
  s.n_slots = 1;
  s.spacing = ~0ULL;
  s.spacing_bits = 64;
  return s;
}

int make_slots(const pb_slots_cfg& cfg, const uint32_t* h_occ_off, SlotsDev& s) {
  std::memset(&s, 0, sizeof(s));
  if (cfg.n_slots == 0 || cfg.n_slots > PB_MAX_SLOTS) return fail(PB_ERR_INVALID, "n_slots must be in 1..PB_MAX_SLOTS");
  s.n_slots = cfg.n_slots;
  s.spacing = cfg.prefix_bit > 0 ? ((1ULL << (64 - cfg.prefix_bit)) - 1) : ~0ULL;
  s.spacing_bits = 64 - cfg.prefix_bit;
  for (uint32_t i = 0; i < cfg.n_slots; ++i) {
    s.prefix[i] = cfg.prefix[i];
    s.sqrt_scaling[i] = cfg.sqrt_scaling[i];
    s.occ_off[i] = h_occ_off[i];
  }
  s.occ_off[cfg.n_slots] = h_occ_off[cfg.n_slots];
  s.uniform = cfg.n_slots ? (h_occ_off[cfg.n_slots] - h_occ_off[0]) / cfg.n_slots : 0;
  for (uint32_t i = 0; i <= cfg.n_slots && s.uniform; ++i)
    if (h_occ_off[i] != i * s.uniform) s.uniform = 0;
  return PB_OK;
}

// the slots of ids given as pb_add_prefix takes them: one prefix per slot, no sqrt scaling
int prefix_slots(const uint32_t* h_occ_off, const uint64_t* h_prefix, uint32_t n_slots, uint32_t prefix_bit,
                 SlotsDev& s) {
  if (n_slots == 0 || n_slots > PB_MAX_SLOTS) return fail(PB_ERR_INVALID, "n_slots must be in 1..PB_MAX_SLOTS");
  pb_slots_cfg cfg;
  std::memset(&cfg, 0, sizeof(cfg));
  cfg.n_slots = n_slots;
  cfg.prefix_bit = prefix_bit;
  for (uint32_t i = 0; i < n_slots; ++i) cfg.prefix[i] = h_prefix[i];
  return make_slots(cfg, h_occ_off, s);
}

// a raw context's one slot over n ids (its samples are ragged: never uniform)
int raw_slots(const pb_ctx* c, uint32_t n, SlotsDev& s) {
  const uint32_t occ_off[2] = {0, n};
  int rc = make_slots(c->slots, occ_off, s);
  s.uniform = 0;
  return rc;
}

int check_slot_offsets(const uint32_t* h_occ_off, uint32_t n_slots, uint32_t n) {
  if (h_occ_off[0] != 0 || h_occ_off[n_slots] != n) return fail(PB_ERR_INVALID, "slot offsets do not span the id array");
  for (uint32_t s = 0; s < n_slots; ++s)
    if (h_occ_off[s] > h_occ_off[s + 1]) return fail(PB_ERR_INVALID, "slot offsets must ascend");
  return PB_OK;
}

// gradient, output and update buffers are accessed with vector loads and stores of up to 16 bytes
bool misaligned(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) != 0; }
int check_grads_aligned(const void* const* h_grads, uint32_t n_slots) {
  for (uint32_t s = 0; s < n_slots; ++s)
    if (h_grads[s] && misaligned(h_grads[s])) return fail(PB_ERR_INVALID, "gradient pointers must be 16-byte aligned");
  return PB_OK;
}

// A loss scale is applied unless it is within f32::EPSILON of 1 (mod.rs:751); then its inverse must be finite.
int loss_scale(float sc, uint8_t& on, float& inv) {
  on = std::fabs(sc - 1.0f) > 1.1920929e-07f;
  inv = 1.0f / sc;
  if (on && !std::isfinite(inv)) return fail(PB_ERR_INVALID, "scale on gradient must be finite");
  return PB_OK;
}

// the per-slot gradient table of a summation backward (h_scale null: no loss scale)
int make_grads(const void* const* h_grads, const float* h_scale, uint32_t n_slots, GradsDev& gr) {
  std::memset(&gr, 0, sizeof(gr));
  for (uint32_t s = 0; s < n_slots; ++s) {
    gr.ptr[s] = h_grads[s];
    if (int rc = loss_scale(h_scale ? h_scale[s] : 1.0f, gr.do_scale[s], gr.inv_scale[s])) return rc;
  }
  return PB_OK;
}

// one beta-power step of Adam's pair k (one request of one feature group, optim.rs:155-197); returns the pair
const float* advance_adam_pair(pb_table* t, int k, cudaStream_t st) {
  AdamKeys keys{};
  keys.idx[0] = (uint8_t)k;
  keys.n = 1;
  launch_adam_advance(t->adam_dev, keys, t->op.b1, t->op.b2, st);
  return t->adam_dev + 2 * k;
}

// ---- what the local and sharded forms of the forwards and backwards share ------------------------------------------
int check_forward(pb_table* t, pb_ctx* c, const uint64_t* d_ids, uint32_t n_occ, const uint32_t* d_row_off,
                  const uint32_t* h_slot_occ_off, uint32_t batch, void* d_out_f16) {
  if (!t || !c || !h_slot_occ_off || !d_out_f16 || (n_occ && !d_ids)) return fail(PB_ERR_INVALID, "null argument");
  if (misaligned(d_out_f16)) return fail(PB_ERR_INVALID, "output pointer must be 16-byte aligned");
  if (!c->has_slots) return fail(PB_ERR_STATE, "pb_ctx_set_slots not called");
  if (t->device != c->device) return fail(PB_ERR_INVALID, "table and context live on different devices");
  if (batch > 65535) return fail(PB_ERR_BATCH, "batch size cannot be larger than 65535");
  const uint32_t S = c->slots.n_slots;
  const uint64_t n_out = (uint64_t)S * batch;
  if (n_occ > c->max_occ || n_out > c->max_out) return fail(PB_ERR_CAPACITY, "batch exceeds the context's capacity");
  if (!d_row_off && n_occ != n_out) return fail(PB_ERR_INVALID, "row offsets are required unless every sample has one id per slot");
  return check_slot_offsets(h_slot_occ_off, S, n_occ);
}

int check_raw_forward(pb_table* t, pb_ctx* c, const uint64_t* d_ids, uint32_t n_occ, const uint32_t* d_row_off,
                      uint32_t batch, uint32_t sample_fixed_size, void* d_table_f16, int64_t* d_index,
                      int64_t* d_non_empty, uint32_t* d_sample_id_num, uint32_t* d_counts) {
  if (!t || !c || !d_table_f16 || !d_index || !d_non_empty || !d_sample_id_num || !d_counts || (n_occ && !d_ids))
    return fail(PB_ERR_INVALID, "null argument");
  if (misaligned(d_table_f16)) return fail(PB_ERR_INVALID, "output pointer must be 16-byte aligned");
  if (!c->has_slots || c->slots.n_slots != 1) return fail(PB_ERR_STATE, "a raw context serves exactly one slot (pb_ctx_set_slots)");
  if (t->device != c->device) return fail(PB_ERR_INVALID, "table and context live on different devices");
  if (batch > 65535) return fail(PB_ERR_BATCH, "batch size cannot be larger than 65535");
  if (sample_fixed_size == 0) return fail(PB_ERR_INVALID, "sample_fixed_size must be positive");
  if (n_occ > c->max_occ || batch > c->max_out || (uint64_t)batch * sample_fixed_size > (1ull << 31))
    return fail(PB_ERR_CAPACITY, "batch exceeds the context's capacity");
  if (!d_row_off && n_occ != batch) return fail(PB_ERR_INVALID, "row offsets are required unless every sample has one id");
  return PB_OK;
}

int check_backward(pb_table* t, pb_ctx* c, const void* const* h_grads) {
  if (!t || !c || !h_grads) return fail(PB_ERR_INVALID, "null argument");
  if (int rc = writable(t)) return rc;
  int rc = c->pending.check(t, "no forward batch is pending in this context (backward_ref_id not found)",
                            "the pending batch was looked up in another table");
  if (rc || (rc = ready_for_training(t))) return rc;
  return check_grads_aligned(h_grads, c->slots.n_slots);
}

// (t and c not null: each caller checks them with its own arguments)
int check_raw_backward(pb_table* t, pb_ctx* c, const void* d_grad) {
  if (int rc = writable(t)) return rc;
  int rc = c->raw_pending.check(t, "no raw forward batch is pending in this context (backward_ref_id not found)",
                                "the pending raw batch was looked up in another table");
  if (rc) return rc;
  if (d_grad && misaligned(d_grad)) return fail(PB_ERR_INVALID, "gradient pointer must be 16-byte aligned");
  return ready_for_training(t);
}

// the context's copy of a batch's row offsets (n_rows + 1) and the output row of every id occurrence
int copy_row_off(pb_ctx* c, const uint32_t* d_row_off, uint32_t n_rows, cudaStream_t st) {
  PB_CUDA(cudaMemcpyAsync(c->row_off, d_row_off, 4 * ((size_t)n_rows + 1), cudaMemcpyDeviceToDevice, st));
  launch_expand_rows(c->row_off, n_rows, c->occ_outrow, st);
  return PB_OK;
}

// The context's previous batch goes (like an expired post_forward_buffer entry, mod.rs:991-1029), and with it any
// batch prepared and never sent.
void drop_batch(pb_ctx* c, cudaStream_t st) {
  // a batch whose gradients never came (or an inference request) leaves its cells in the scratch set: empty it first
  if (c->set_dirty) {
    launch_clear_items(c->b, st);
    c->set_dirty = false;
  }
  if (c->pending.on) launch_clear_hot_bits(c->b, st);  // its hot items' bitmaps were never consumed
  c->pending.drop();
  c->prepared = PREP_NONE;
}

// A summation forward's start: the context's previous batch goes, then the new batch's distinct items are found.
// `prepared`: PB_PHASE_PREPARE found them already (prepare_batch); only the table's part is left.
int begin_forward(pb_table* t, pb_ctx* c, const SlotsDev& sl, const uint64_t* d_ids, uint32_t n_occ, int training,
                  cudaStream_t st, bool prepared = false) {
  if (!prepared) drop_batch(c, st);
  if (training) {
    if (int rc = maybe_evict(t, st)) return rc;
  }
  if (prepared) {  // the request number only: the dedup's counters hold the prepared batch
    if (training) launch_begin_batch(t->d, c->dev_tick, nullptr, st, true);
    c->prepared = PREP_NONE;
    return PB_OK;
  }
  launch_begin_batch(t->d, training ? c->dev_tick : nullptr, c->b.cnt, st, training != 0);
  c->b.n = n_occ;
  launch_dedup(sl, c->b, d_ids, st);
  return PB_OK;
}

// PB_PHASE_PREPARE of a summation forward: begin_forward's dedup alone.  It reads no table state (k_dedup works in the
// context's scratch set), so the eviction check and the request number stay with SEND.  The set holds the batch from
// here on: a batch prepared and never sent is emptied by the context's next forward.
void prepare_batch(const pb_table* t, pb_ctx* c, const SlotsDev& sl, const uint64_t* d_ids, uint32_t n_occ,
                   uint32_t batch, cudaStream_t st) {
  drop_batch(c, st);
  launch_begin_batch(t->d, nullptr, c->b.cnt, st, false);  // (no bump: the table's counters are not touched)
  c->b.n = n_occ;
  launch_dedup(sl, c->b, d_ids, st);
  c->set_dirty = true;
  c->prepared = PREP_SUM;
  c->prepared_n = n_occ;
  c->prepared_batch = batch;
}

// A summation forward's end: a training batch stays in the context, pending, for its backward (its cells are emptied
// beside the backward, or by the next forward); an inference request's cells are emptied now.
int end_forward(pb_table* t, pb_ctx* c, const uint32_t* d_row_off, const uint32_t* h_slot_occ_off, uint32_t n_occ,
                uint32_t batch, int training, cudaStream_t st) {
  if (!training) {
    launch_clear_items(c->b, st);
    c->set_dirty = false;  // (a prepared batch marked it)
    return PB_OK;
  }
  const uint32_t S = c->slots.n_slots;
  c->n_occ = n_occ;
  c->batch = batch;
  c->multi_id = d_row_off != nullptr;
  std::memcpy(c->occ_off, h_slot_occ_off, sizeof(uint32_t) * (S + 1));
  if (d_row_off) {
    if (int rc = copy_row_off(c, d_row_off, S * batch, st)) return rc;
  }
  c->pending.hold(t);
  c->set_dirty = true;
  return PB_OK;
}

// a raw training forward's batch stays pending in the context, its rows spared by eviction, until its backward
void hold_raw_batch(pb_table* t, pb_ctx* c, uint32_t n_occ, uint32_t batch) {
  c->n_occ = n_occ;
  c->batch = batch;
  c->raw_pending.hold(t);
}

// what the reduces of a summation backward read of the context's pending batch
ReduceArgs reduce_args(const pb_ctx* c) {
  ReduceArgs a;
  std::memset(&a, 0, sizeof(a));
  a.b = c->b;
  a.b.n = c->n_occ;
  a.occ_outrow = c->multi_id ? c->occ_outrow : nullptr;
  a.row_off = c->multi_id ? c->row_off : nullptr;
  a.tick_ptr = c->dev_tick;
  a.nan_tick = c->nan_tick;
  a.batch = c->batch;
  return a;
}

// A summation backward's side streams: `side` and `side2` follow `st` from fork_side on, and again from fork_after_nan
// on (what comes after reads the NaN scan's marks); join_sides makes `st` wait for both.
int fork_side(pb_ctx* c, cudaStream_t st) {
  PB_CUDA(cudaEventRecord(c->ev_fork, st));
  PB_CUDA(cudaStreamWaitEvent(c->side, c->ev_fork, 0));
  PB_CUDA(cudaStreamWaitEvent(c->side2, c->ev_fork, 0));
  return PB_OK;
}

int fork_after_nan(pb_ctx* c, cudaStream_t st) {
  PB_CUDA(cudaEventRecord(c->ev_nan, st));
  PB_CUDA(cudaStreamWaitEvent(c->side, c->ev_nan, 0));
  PB_CUDA(cudaStreamWaitEvent(c->side2, c->ev_nan, 0));
  return PB_OK;
}

int join_sides(pb_ctx* c, cudaStream_t st) {
  PB_CUDA(cudaEventRecord(c->ev_join, c->side));
  PB_CUDA(cudaStreamWaitEvent(st, c->ev_join, 0));
  PB_CUDA(cudaEventRecord(c->ev_join2, c->side2));
  PB_CUDA(cudaStreamWaitEvent(st, c->ev_join2, 0));
  return PB_OK;
}

}  // namespace

extern "C" {

const char* pb_last_error(void) { return g_err.c_str(); }
int pb_version(void) { return 100; }
uint64_t pb_launch_count(void) { return launch_count(); }
int pb_hot_geometry(uint32_t dim, int is_f16, int ragged, uint32_t h_out[12]) {
  if (!h_out) return fail(PB_ERR_INVALID, "null argument");
  if (dim == 0 || dim > 4096) return fail(PB_ERR_INVALID, "dim must be in 1..4096");
  hot_geometry(dim, is_f16 != 0, ragged != 0, h_out);
  return PB_OK;
}
int pb_profile_enable(int family_mask) {
  profile_enable((uint32_t)family_mask);
  return PB_OK;
}
int pb_profile_read(double* h_ms, uint64_t* h_count, int n) {
  if (!h_ms || !h_count || n <= 0) return fail(PB_ERR_INVALID, "bad argument");
  PB_CUDA(cudaDeviceSynchronize());
  profile_read(h_ms, h_count, n < FAM_COUNT ? n : FAM_COUNT);
  for (int i = FAM_COUNT; i < n; ++i) {
    h_ms[i] = 0;
    h_count[i] = 0;
  }
  return PB_OK;
}

int pb_table_create(int device, const pb_table_cfg* cfg, pb_table** out) {
  if (!cfg || !out) return fail(PB_ERR_INVALID, "null argument");
  if (cfg->dim == 0 || cfg->dim > 4096) return fail(PB_ERR_INVALID, "dim must be in 1..4096");
  if (cfg->capacity == 0) return fail(PB_ERR_INVALID, "capacity must be > 0");
  int ndev = 0;
  PB_CUDA(cudaGetDeviceCount(&ndev));
  if (device < 0 || device >= ndev) return fail(PB_ERR_INVALID, "no such CUDA device");
  DeviceGuard g(device);
  std::unique_ptr<pb_table> t(new pb_table());
  t->device = device;
  t->cfg = *cfg;
  int rc;
  if ((rc = t->own.event(t->index.ev)) || (rc = t->own.event(t->step.ev))) return rc;
  *out = t.release();
  return PB_OK;
}

int pb_table_create_host(int device, const pb_table_cfg* cfg, pb_table** out) {
  int rc = pb_table_create(device, cfg, out);
  if (rc) return rc;
  (*out)->host = true;
  return PB_OK;
}

int pb_table_create_host_shared(int device, const pb_table_cfg* cfg, pb_table** out) {
  int rc = pb_table_create_host(device, cfg, out);
  if (rc) return rc;
  (*out)->shared = true;
  return PB_OK;
}

int pb_table_attach_tier(pb_table* t, pb_table* tier) {
  if (!t || !tier) return fail(PB_ERR_INVALID, "null argument");
  if (int rc = writable(t)) return rc;  // (an exported table can have no tier: peers could not read its host rows)
  if (t->live) return fail(PB_ERR_STATE, "a live-exported table cannot take a host tier: peers could not read its host rows");
  if (t->grow) return fail(PB_ERR_STATE, "a growable table cannot take a host tier");
  if (t->host || !tier->host) return fail(PB_ERR_INVALID, "the tier must be a host table (pb_table_create_host) behind an HBM table");
  if (t->tier || t->tier_of || tier->tier_of || tier->tier) return fail(PB_ERR_STATE, "one of the tables already has a tier or is one");
  if (t->device != tier->device) return fail(PB_ERR_INVALID, "the tables live on different devices");
  if (!t->has_op || !tier->has_op) return fail(PB_ERR_STATE, "register the optimizer of both tables before attaching the tier");
  if (t->cfg.dim != tier->cfg.dim || t->op.kind != tier->op.kind)
    return fail(PB_ERR_INVALID, "the tier must have the table's dim and optimizer (one entry layout)");
  DeviceGuard g(t->device);
  // both tables' storage and sweep workspace, and the victim list: committed together once all are held
  pb_table* tt[2] = {t, tier};
  Owned o[2];
  uint32_t* free_rows[2] = {t->d.free_rows, tier->d.free_rows};
  uint32_t* move_cells = nullptr;
  int rc = 0;
  for (int i = 0; i < 2 && !rc; ++i)
    if (!tt[i]->allocated) rc = acquire_storage(tt[i], o[i]);
  if (!rc && t->d.stride != tier->d.stride) rc = fail(PB_ERR_INVALID, "the tier's row stride differs from the table's");
  for (int i = 0; i < 2 && !rc; ++i)
    if (!free_rows[i]) rc = acquire_evict_ws(tt[i], o[i], free_rows[i]);
  if (rc || (rc = o[0].dev(move_cells, sizeof(uint32_t) * (size_t)t->d.capacity))) return rc;
  for (int i = 0; i < 2; ++i) {
    tt[i]->own.adopt(o[i]);
    tt[i]->allocated = true;
    tt[i]->d.free_rows = free_rows[i];
  }
  t->move_cells = move_cells;
  t->tier = tier;
  tier->tier_of = t;
  return PB_OK;
}

int pb_tier_stats(pb_table* t, uint64_t h_out[5], void* stream) {
  if (!t || !h_out) return fail(PB_ERR_INVALID, "null argument");
  for (int i = 0; i < 5; ++i) h_out[i] = 0;
  if (!t->tier) return PB_OK;
  uint32_t c[CTR_COUNT];
  if (int rc = read_counters(t, t->tier->d.counters, c, CTR_COUNT, (cudaStream_t)stream)) return rc;
  h_out[0] = c[CTR_ADMIT] - c[CTR_EVICT] - c[CTR_TIER_IN];
  h_out[1] = c[CTR_TIER_OUT];
  h_out[2] = c[CTR_TIER_IN];
  h_out[3] = (uint64_t)c[CTR_EVICT] + c[CTR_TIER_LOST];
  h_out[4] = c[CTR_TIER_REFUSED];
  return PB_OK;
}

int pb_tier_stage(pb_table* t, const uint64_t* d_ids, uint32_t n, const uint32_t* h_slot_occ_off, const uint64_t* h_prefix,
                  uint32_t n_slots, uint32_t prefix_bit, void* stream) {
  if (!t || (n && !d_ids) || !h_slot_occ_off || !h_prefix) return fail(PB_ERR_INVALID, "null argument");
  if (t->tier_of) return fail(PB_ERR_STATE, "a host tier is not staged directly: use the table it is attached to");
  if (n_slots == 0 || n_slots > PB_MAX_SLOTS) return fail(PB_ERR_INVALID, "n_slots must be in 1..PB_MAX_SLOTS");
  if (prefix_bit == 0 || prefix_bit > 63) return fail(PB_ERR_INVALID, "feature_index_prefix_bit must be in 1..63");
  int rc = check_slot_offsets(h_slot_occ_off, n_slots, n);
  if (rc || (rc = writable(t))) return rc;  // (its eviction check)
  if (!t->tier) return PB_OK;  // nothing to move
  if ((rc = ready_for_training(t))) return rc;
  SlotsDev sl;
  if ((rc = prefix_slots(h_slot_occ_off, h_prefix, n_slots, prefix_bit, sl))) return rc;
  DeviceGuard g(t->device);
  cudaStream_t st = (cudaStream_t)stream;
  // After both chains, in the index chain only: every earlier call on the table first (enqueued backwards included),
  // and every later call but the backwards after this stage.  Why it may run beside a backward: no backward kernel
  // reads index cells, the free-row stack or row_tick (the only index read outside the forward path is k_raw_table's,
  // in the raw forward, which waits), and a backward writes only the rows of its own batch, which are never victims
  // here (keep > pending_batches) nor restore targets (those come off the free stack).  Counters it shares with a
  // backward are updated atomically.
  TableCall call;
  if ((rc = call.begin(t, st, CALL_INDEX, CALL_STEP))) return rc;
  // the check the request would run (not counted in train_calls, so the request's own stays where it was: after a
  // stage it usually finds enough free rows and does nothing); keep covers the batches pending now
  if (t->evict_every && (rc = evict_check(t, st, g_stage_blocks))) return rc;
  TierWindow win(t, st);
  launch_tier_stage(t->d, t->tier->d, t->hy, t->op, sl, d_ids, n, g_stage_blocks, st);
  PB_CUDA(cudaGetLastError());
  return PB_OK;
}

int pb_tier_stage_stats(pb_table* t, uint64_t h_out[2], void* stream) {
  if (!t || !h_out) return fail(PB_ERR_INVALID, "null argument");
  h_out[0] = h_out[1] = 0;
  if (!t->tier) return PB_OK;
  uint32_t c[CTR_COUNT];
  if (int rc = read_counters(t, t->tier->d.counters, c, CTR_COUNT, (cudaStream_t)stream)) return rc;
  h_out[0] = c[CTR_STAGE_IN];
  h_out[1] = c[CTR_STAGE_SKIP];
  return PB_OK;
}

int pb_table_enable_incremental(pb_table* t, uint64_t capacity) {
  if (!t) return fail(PB_ERR_INVALID, "null argument");
  if (t->host) return fail(PB_ERR_STATE, "a host tier has no set of its own: enable it on the table the tier is attached to");
  if (capacity >= (1ull << 30)) return fail(PB_ERR_INVALID, "capacity must be < 2^30 signs");
  DeviceGuard g(t->device);
  PB_CUDA(cudaDeviceSynchronize());  // enqueued marks may still use the old set
  t->own.release(t->inc.cells);
  t->own.release(t->inc.ctr);
  t->own.release(t->inc_host);
  t->inc = IncDev{};
  if (!capacity) return PB_OK;
  IncDev s{};
  s.capacity = capacity;
  s.n_cells = next_pow2(2 * capacity < 1024 ? 1024 : 2 * capacity);
  s.bucket_mask = s.n_cells / BUCKET - 1;
  Owned o;
  unsigned long long* host = nullptr;
  int rc;
  if ((rc = o.dev(s.cells, sizeof(Cell) * ((size_t)s.n_cells + N_SPECIAL))) ||
      (rc = o.dev(s.ctr, sizeof(unsigned long long) * INC_WORDS)) || (rc = o.mapped(host, s.mirror, sizeof(unsigned long long))))
    return rc;
  *host = 0;
  launch_inc_fill(s, 0);
  PB_CUDA(cudaDeviceSynchronize());
  t->own.adopt(o);
  t->inc = s;
  t->inc_host = host;
  return PB_OK;
}

int pb_inc_take(pb_table* t, uint64_t* d_signs, uint32_t max_n, uint32_t* d_count, void* stream) {
  if (!t || !d_count || (max_n && !d_signs)) return fail(PB_ERR_INVALID, "null argument");
  if (!t->inc.cells) return fail(PB_ERR_STATE, "incremental updates are not enabled on this table");
  DeviceGuard g(t->device);
  cudaStream_t st = (cudaStream_t)stream;
  TableCall call;
  if (int rc = call.begin(t, st, CALL_ALL)) return rc;
  launch_inc_take(t->inc, d_signs, max_n, d_count, st);
  PB_CUDA(cudaGetLastError());
  return PB_OK;
}

int pb_inc_stats(pb_table* t, uint64_t h_out[4], void* stream) {
  if (!t || !h_out) return fail(PB_ERR_INVALID, "null argument");
  for (int i = 0; i < 4; ++i) h_out[i] = 0;
  if (!t->inc.cells) return PB_OK;
  unsigned long long c[INC_WORDS];
  if (int rc = read_counters(t, t->inc.ctr, c, INC_WORDS, (cudaStream_t)stream)) return rc;
  h_out[0] = c[INC_HELD];
  h_out[1] = c[INC_INSERTED];
  h_out[2] = c[INC_DROPPED];
  h_out[3] = c[INC_TAKEN];
  return PB_OK;
}

int pb_inc_held(pb_table* t, uint64_t* h_out) {
  if (!t || !h_out) return fail(PB_ERR_INVALID, "null argument");
  *h_out = t->inc_host ? *reinterpret_cast<volatile unsigned long long*>(t->inc_host) : 0;
  return PB_OK;
}

int pb_table_destroy(pb_table* t) {
  if (!t) return PB_OK;
  DeviceGuard g(t->device);
  if (t->tier) t->tier->tier_of = nullptr;
  if (t->tier_of) t->tier_of->tier = nullptr;
  if (t->allocated || t->inc.cells || t->dump_mem) cudaDeviceSynchronize();  // (enqueued work may still use them)
  delete t;
  return PB_OK;
}

int pb_table_set_optimizer(pb_table* t, const pb_optim_cfg* c) {
  if (!t || !c) return fail(PB_ERR_INVALID, "null argument");
  if (c->kind < PB_OPT_SGD || c->kind > PB_OPT_ADAM) return fail(PB_ERR_INVALID, "unknown optimizer kind");
  if (t->allocated && c->kind != t->op.kind)
    return fail(PB_ERR_STATE, "optimizer kind cannot change once rows are resident (row layout is fixed)");
  int rc;
  t->op.kind = c->kind;
  t->op.lr = c->lr;
  t->op.wd = c->wd;
  t->op.mom = c->g_square_momentum;
  t->op.init_acc = c->initialization;
  t->op.eps = c->eps;
  t->op.b1 = c->beta1;
  t->op.b2 = c->beta2;
  if (!t->has_op && c->kind == PB_OPT_ADAM) {  // AdamPowerOfBetas starts at (beta1, beta2) for every feature group (optim.rs:118-124)
    DeviceGuard g(t->device);
    t->adam_keys.clear();
    Owned o;
    float* pairs = t->adam_dev;
    if (!pairs && (rc = o.dev(pairs, sizeof(float) * 2 * PB_ADAM_KEYS))) return rc;
    launch_adam_fill(pairs, c->beta1, c->beta2, 0);
    PB_CUDA(cudaDeviceSynchronize());
    t->own.adopt(o);
    t->adam_dev = pairs;
  }
  t->has_op = true;
  return PB_OK;
}

int pb_table_set_rsqrt(pb_table* t, int mode) {
  if (!t) return fail(PB_ERR_INVALID, "null argument");
  if (mode != PB_RSQRT_EXACT && mode != PB_RSQRT_INTEL) return fail(PB_ERR_INVALID, "unknown rsqrt mode");
  t->op.rsqrt = mode;
  return PB_OK;
}

int pb_table_configure(pb_table* t, const pb_hyper_cfg* c) {
  if (!t || !c) return fail(PB_ERR_INVALID, "null argument");
  t->hy.lo = c->init_lower;
  t->hy.scale = uniform_scale(c->init_lower, c->init_upper);
  t->hy.admit_p = c->admit_probability;
  t->hy.enable_wb = c->enable_weight_bound;
  t->hy.wb = c->weight_bound;
  t->has_hy = true;
  return PB_OK;
}

int pb_table_set_eviction(pb_table* t, uint32_t check_every, uint64_t low_water, uint64_t target_free, uint32_t keep_batches) {
  if (!t) return fail(PB_ERR_INVALID, "null argument");
  if (check_every && (target_free < low_water || target_free > t->cfg.capacity))
    return fail(PB_ERR_INVALID, "need low_water <= target_free <= capacity");
  t->evict_every = check_every;
  t->evict_low = (uint32_t)low_water;
  t->evict_target = (uint32_t)target_free;
  t->evict_keep = keep_batches;
  return PB_OK;
}

int pb_table_entry_len(pb_table* t, uint32_t* h_out) {
  if (!t || !h_out) return fail(PB_ERR_INVALID, "null argument");
  if (!t->has_op) return fail(PB_ERR_STATE, "optimizer not registered");
  uint32_t dim = t->cfg.dim;
  *h_out = dim + (t->op.kind == PB_OPT_ADAGRAD ? dim : t->op.kind == PB_OPT_ADAGRAD_VW ? 1 : t->op.kind == PB_OPT_ADAM ? 2 * dim : 0);
  return PB_OK;
}

int pb_table_counters(pb_table* t, uint64_t h_out[5], void* stream) {
  if (!t || !h_out) return fail(PB_ERR_INVALID, "null argument");
  h_out[0] = h_out[1] = h_out[2] = h_out[3] = h_out[4] = 0;
  if (!t->allocated) return PB_OK;
  uint32_t c[CTR_COUNT];
  if (int rc = read_counters(t, t->d.counters, c, CTR_COUNT, (cudaStream_t)stream)) return rc;
  h_out[0] = c[CTR_ADMIT] - c[CTR_EVICT] - c[CTR_TIER_IN];  // resident rows (a tier's restored rows left it)
  h_out[1] = c[CTR_MISS];
  h_out[2] = c[CTR_GRAD_MISS];
  h_out[3] = c[CTR_FULL];
  h_out[4] = c[CTR_ERR];
  return PB_OK;
}

int pb_table_index_stats(pb_table* t, uint64_t h_out[3], void* stream) {
  if (!t || !h_out) return fail(PB_ERR_INVALID, "null argument");
  h_out[0] = h_out[1] = h_out[2] = 0;
  if (!t->allocated) return PB_OK;
  DeviceGuard g(t->device);
  cudaStream_t st = (cudaStream_t)stream;
  TableCall call;
  int rc;
  if ((rc = call.begin(t, st, CALL_ALL))) return rc;
  if (!t->stats_ws && (rc = t->own.dev(t->stats_ws, 3 * sizeof(uint32_t)))) return rc;
  launch_index_stats(t->d, t->stats_ws, st);
  uint32_t c[3];
  PB_CUDA(cudaMemcpyAsync(c, t->stats_ws, sizeof(c), cudaMemcpyDeviceToHost, st));
  PB_CUDA(cudaStreamSynchronize(st));
  for (int i = 0; i < 3; ++i) h_out[i] = c[i];
  return PB_OK;
}

int pb_table_set_growth(pb_table* t, int on) {
  if (!t) return fail(PB_ERR_INVALID, "null argument");
  if (t->host) return fail(PB_ERR_STATE, "a host table's storage cannot grow");
  if (t->allocated) return fail(PB_ERR_STATE, "growth must be chosen before the table's first allocation");
  t->grow = on != 0;
  return PB_OK;
}

int pb_table_storage_stats(pb_table* t, uint64_t h_out[4], void* stream) {
  if (!t || !h_out) return fail(PB_ERR_INVALID, "null argument");
  h_out[0] = t->cfg.capacity;
  h_out[1] = h_out[2] = h_out[3] = 0;
  if (!t->allocated) return PB_OK;
  uint32_t c[CTR_COUNT];
  if (int rc = read_counters(t, t->d.counters, c, CTR_COUNT, (cudaStream_t)stream)) return rc;
  h_out[1] = t->d.mapped;
  h_out[2] = t->d.n_cells;
  h_out[3] = c[CTR_UNMAPPED];
  return PB_OK;
}

int pb_table_size(pb_table* t, uint64_t* h_out, void* stream) {
  if (!t || !h_out) return fail(PB_ERR_INVALID, "null argument");
  uint64_t c[5];
  int rc = pb_table_counters(t, c, stream);
  if (rc) return rc;
  *h_out = c[0];
  return PB_OK;
}

int pb_table_clear(pb_table* t, void* stream) {
  if (!t) return fail(PB_ERR_INVALID, "null argument");
  if (int rc = writable(t)) return rc;
  if (!t->allocated) return PB_OK;
  DeviceGuard g(t->device);
  cudaStream_t st = (cudaStream_t)stream;
  TableCall call;
  if (int rc = call.begin(t, st, CALL_ALL)) return rc;
  // peers reading in place wait until every cell of the table and of its tier is EMPTY again
  if (t->live) launch_seq_bump(t->seq, true, st);
  launch_fill_cells(t->d.cells, (uint64_t)t->d.n_cells + N_SPECIAL, st);
  PB_CUDA(cudaMemsetAsync(t->d.counters, 0, sizeof(uint32_t) * CTR_COUNT, st));
  PB_CUDA(cudaMemsetAsync(t->d.row_tick, 0, sizeof(uint32_t) * (size_t)t->d.mapped, st));
  const int rc = t->tier ? pb_table_clear(t->tier, stream) : PB_OK;
  if (t->live) launch_seq_bump(t->seq, false, st);
  return rc;
}

int pb_lookup(pb_table* t, const uint64_t* d_signs, uint32_t n, int training, float* d_out, void* stream) {
  if (!t || (n && (!d_signs || !d_out))) return fail(PB_ERR_INVALID, "null argument");
  if (training) {
    int rc = writable(t);
    if (rc || (rc = ready_for_training(t))) return rc;
  } else if (!t->has_op) {  // nothing can be resident yet: zeros
    DeviceGuard g(t->device);
    PB_CUDA(cudaMemsetAsync(d_out, 0, sizeof(float) * (size_t)n * t->cfg.dim, (cudaStream_t)stream));
    return PB_OK;
  }
  DeviceGuard g(t->device);
  cudaStream_t st = (cudaStream_t)stream;
  TableCall call;
  if (int rc = call.begin(t, st, CALL_INDEX)) return rc;
  int rc = ensure_alloc(t);
  if (rc) return rc;
  if ((rc = ensure_scratch(t, n))) return rc;
  if (training && (rc = grow_for(t, n, st))) return rc;
  SlotsDev sl = no_slots();
  if (training) {
    if ((rc = maybe_evict(t, st))) return rc;
    launch_begin_batch(t->d, nullptr, nullptr, st);
    restore_ids(t, false, sl, d_signs, n, st);
    launch_probe(MODE_TRAIN, false, t->d, t->hy, t->op, sl, d_signs, n, t->scratch, st);
  } else {
    launch_probe(MODE_FIND, false, t->d, t->hy, t->op, sl, d_signs, n, t->scratch, st);
  }
  launch_gather(t->d, t->scratch, n, d_out, st);
  if (!training && t->tier)  // inference moves nothing: a tier-held sign is read where it is
    launch_tier_get(t->d, t->tier->d, d_signs, t->scratch, n, t->d.dim, d_out, nullptr, t->d.counters + CTR_MISS, st);
  PB_CUDA(cudaGetLastError());
  return PB_OK;
}

int pb_update(pb_table* t, const uint64_t* d_signs, const float* d_grads, uint32_t n, void* stream) {
  if (!t || (n && (!d_signs || !d_grads))) return fail(PB_ERR_INVALID, "null argument");
  if (n && misaligned(d_grads)) return fail(PB_ERR_INVALID, "gradient pointer must be 16-byte aligned");
  int rc = writable(t);
  if (rc || (rc = ready_for_training(t))) return rc;
  DeviceGuard g(t->device);
  cudaStream_t st = (cudaStream_t)stream;
  TableCall call;
  if ((rc = call.begin(t, st, CALL_ALL))) return rc;
  if ((rc = ensure_alloc(t))) return rc;
  if ((rc = ensure_scratch(t, n))) return rc;
  SlotsDev sl = no_slots();
  launch_probe(MODE_FIND, false, t->d, t->hy, t->op, sl, d_signs, n, t->scratch, st);
  if (t->tier) {  // a tier-held sign's row is stepped where it is (no HBM row is needed)
    if ((rc = ensure_scratch(t->tier, n))) return rc;
    launch_tier_where(t->d, t->tier->d, d_signs, t->scratch, n, t->tier->scratch, st);
  }
  // get_batch_level_state: one power step per request
  const float* pair = t->op.kind == PB_OPT_ADAM ? advance_adam_pair(t, PB_ADAM_KEYS - 1, st) : nullptr;
  launch_update_direct(t->d, t->op, t->hy, t->scratch, d_grads, n, pair, st);
  if (t->tier) launch_update_direct(t->tier->d, t->op, t->hy, t->tier->scratch, d_grads, n, pair, st);
  if (t->inc.cells && n)  // the signs just stepped, in HBM or in the tier
    launch_inc_mark_signs(t->inc, t->d, d_signs, t->scratch, n, t->tier ? t->tier->d : t->d,
                          t->tier ? t->tier->scratch : nullptr, st);
  PB_CUDA(cudaGetLastError());
  return PB_OK;
}

int pb_set_rows(pb_table* t, const uint64_t* d_signs, const float* d_entries, uint32_t n, void* stream) {
  if (!t || (n && (!d_signs || !d_entries))) return fail(PB_ERR_INVALID, "null argument");
  if (!t->has_op) return fail(PB_ERR_STATE, "optimizer not registered: entry length unknown");
  DeviceGuard g(t->device);
  cudaStream_t st = (cudaStream_t)stream;
  TableCall call;
  if (int rc = call.begin(t, st, CALL_ALL)) return rc;
  int rc = ensure_alloc(t);
  if (rc) return rc;
  if ((rc = ensure_scratch(t, n)) || (rc = grow_for(t, n, st))) return rc;
  SlotsDev sl = no_slots();
  // an exported table, frozen or live: peers reading it in place see the write-sequence word odd from before the first
  // cell it may claim (or, with a tier, the first entry it moves back) to after the last entry it writes (pb_remote.cu),
  // and read those items again
  const bool bracket = t->exported || t->live;
  if (bracket) launch_seq_bump(t->seq, true, st);
  // with a tier: a tier-held sign is first moved back (it then lives in one table), and an entry the HBM table has no
  // row for goes to the tier
  if (t->tier) launch_tier_restore(t->d, t->tier->d, t->hy, t->op, sl, false, d_signs, n, st);
  launch_probe(MODE_SET, false, t->d, t->hy, t->op, sl, d_signs, n, t->scratch, st);
  launch_copy_entries(true, t->d, t->scratch, n, const_cast<float*>(d_entries), nullptr, st);
  if (t->tier) launch_tier_set(t->d, t->tier->d, t->hy, t->op, d_signs, t->scratch, n, d_entries, st);
  if (bracket) launch_seq_bump(t->seq, false, st);
  PB_CUDA(cudaGetLastError());
  return PB_OK;
}

int pb_get_rows(pb_table* t, const uint64_t* d_signs, uint32_t n, float* d_entries, uint8_t* d_found, void* stream) {
  if (!t || (n && (!d_signs || !d_entries))) return fail(PB_ERR_INVALID, "null argument");
  if (!t->has_op) return fail(PB_ERR_STATE, "optimizer not registered: entry length unknown");
  DeviceGuard g(t->device);
  cudaStream_t st = (cudaStream_t)stream;
  TableCall call;
  if (int rc = call.begin(t, st, CALL_ALL)) return rc;
  int rc = ensure_alloc(t);
  if (rc) return rc;
  if ((rc = ensure_scratch(t, n))) return rc;
  SlotsDev sl = no_slots();
  launch_probe(MODE_FIND, false, t->d, t->hy, t->op, sl, d_signs, n, t->scratch, st);
  launch_copy_entries(false, t->d, t->scratch, n, d_entries, d_found, st);
  if (t->tier)  // read in place
    launch_tier_get(t->d, t->tier->d, d_signs, t->scratch, n, t->d.dim + t->d.state_floats, d_entries, d_found, nullptr, st);
  PB_CUDA(cudaGetLastError());
  return PB_OK;
}

int pb_table_export_signs(pb_table* t, uint64_t* d_signs, uint32_t* d_recency, uint32_t max_n, uint32_t* d_count,
                          void* stream) {
  if (!t || !d_count || (max_n && (!d_signs || !d_recency))) return fail(PB_ERR_INVALID, "null argument");
  DeviceGuard g(t->device);
  cudaStream_t st = (cudaStream_t)stream;
  TableCall call;
  if (int rc = call.begin(t, st, CALL_ALL)) return rc;
  if (!t->allocated) {
    PB_CUDA(cudaMemsetAsync(d_count, 0, sizeof(uint32_t), st));
    return PB_OK;
  }
  launch_export_signs(t->d, d_signs, d_recency, max_n, d_count, st);
  PB_CUDA(cudaGetLastError());
  return PB_OK;
}

namespace {

uint64_t dump_items(pb_table* t, uint64_t max_bytes) {
  uint32_t len = 0;
  pb_table_entry_len(t, &len);
  const uint64_t nb = dump_node_bytes(len);
  return max_bytes > 28 ? (max_bytes - 28) / nb : 0;
}

// a dump call on `t`: the table a tier is attached to, with a workspace of at least `items` entries
int dump_ready(pb_table* t, uint64_t items) {
  if (t->tier_of) return fail(PB_ERR_INVALID, "dump the table the tier is attached to");
  if (!t->dump_mem) return fail(PB_ERR_STATE, "no dump workspace: call pb_table_dump_reserve first");
  if (items > t->dump.max_items)
    return fail(PB_ERR_INVALID, "the dump workspace holds " + std::to_string(t->dump.max_items) + " entries, the call needs " +
                                    std::to_string(items) + ": reserve a larger one");
  return PB_OK;
}

}  // namespace

int pb_table_dump_reserve(pb_table* t, uint64_t max_bytes) {
  if (!t) return fail(PB_ERR_INVALID, "null argument");
  if (t->tier_of) return fail(PB_ERR_INVALID, "dump the table the tier is attached to");
  if (!t->has_op) return fail(PB_ERR_STATE, "optimizer not registered: entry length unknown");
  DeviceGuard g(t->device);
  uint64_t items = dump_items(t, max_bytes);
  if (items < 1) items = 1;
  if (items >= (1ull << 31)) return fail(PB_ERR_INVALID, "a dump image holds fewer than 2^31 entries");
  PB_CUDA(cudaDeviceSynchronize());  // a part issued on the old workspace may still run
  t->own.release(t->dump_mem);
  t->dump = DumpWs{};
  const uint32_t m = (uint32_t)items;
  auto r = [](uint64_t b) { return (b + 255) & ~255ull; };
  const uint64_t sort_bytes = dump_sort_bytes(m);
  const uint64_t sz8 = r(8ull * m), sz4 = r(4ull * m);
  if (int rc = t->own.dev(t->dump_mem, 3 * sz8 + 6 * sz4 + 256 + r(sort_bytes))) return rc;
  char* p = static_cast<char*>(t->dump_mem);
  DumpWs& w = t->dump;
  w.key = reinterpret_cast<uint64_t*>(p), p += sz8;
  w.key_s = reinterpret_cast<uint64_t*>(p), p += sz8;
  w.loc = reinterpret_cast<uint64_t*>(p), p += sz8;
  uint32_t** u32s[6] = {&w.rec, &w.rec2, &w.rec_s, &w.idx0, &w.idx1, &w.idx2};
  for (uint32_t** q : u32s) *q = reinterpret_cast<uint32_t*>(p), p += sz4;
  w.words = reinterpret_cast<uint32_t*>(p), p += 256;
  w.sort_tmp = p;
  w.sort_bytes = sort_bytes;
  w.max_items = m;
  return PB_OK;
}

int pb_table_dump_release(pb_table* t) {
  if (!t) return fail(PB_ERR_INVALID, "null argument");
  if (!t->dump_mem) return PB_OK;
  DeviceGuard g(t->device);
  PB_CUDA(cudaDeviceSynchronize());
  t->own.release(t->dump_mem);
  t->dump = DumpWs{};
  return PB_OK;
}

int pb_table_dump_part(pb_table* t, uint32_t part, uint32_t n_parts, void* d_image, uint64_t max_bytes,
                       uint64_t* d_bytes, uint32_t* d_request, void* stream) {
  if (!t || !d_bytes || !d_request || (max_bytes && !d_image)) return fail(PB_ERR_INVALID, "null argument");
  if (n_parts == 0 || part >= n_parts) return fail(PB_ERR_INVALID, "part must be in 0..n_parts-1");
  if (misaligned(d_image)) return fail(PB_ERR_INVALID, "image pointer must be 16-byte aligned");
  if (!t->has_op) return fail(PB_ERR_STATE, "optimizer not registered: entry length unknown");
  int rc = dump_ready(t, dump_items(t, max_bytes));
  if (rc) return rc;
  DeviceGuard g(t->device);
  cudaStream_t st = (cudaStream_t)stream;
  TableCall call;
  if ((rc = call.begin(t, st, CALL_ALL))) return rc;
  if (!t->allocated) {  // nothing was ever stored (no allocation here: the caller may hold the table's lock)
    PB_CUDA(launch_dump_empty(static_cast<uint8_t*>(d_image), max_bytes, reinterpret_cast<unsigned long long*>(d_bytes),
                              d_request, st));
    return PB_OK;
  }
  const TableDev* h = t->tier && t->tier->allocated ? &t->tier->d : nullptr;
  PB_CUDA(launch_dump_part(t->d, h, part, n_parts, t->dump, static_cast<uint8_t*>(d_image), max_bytes,
                           reinterpret_cast<unsigned long long*>(d_bytes), d_request, st));
  return PB_OK;
}

int pb_dump_nodes(pb_table* t, const uint64_t* d_signs, uint32_t n_list, uint32_t lo, uint32_t n, void* d_out,
                  void* stream) {
  if (!t || (n && (!d_signs || !d_out))) return fail(PB_ERR_INVALID, "null argument");
  if ((uint64_t)lo + n > n_list) return fail(PB_ERR_INVALID, "nodes [lo, lo + n) must lie in the list");
  if (misaligned(d_out)) return fail(PB_ERR_INVALID, "output pointer must be 16-byte aligned");
  if (!t->has_op) return fail(PB_ERR_STATE, "optimizer not registered: entry length unknown");
  int rc = dump_ready(t, n);
  if (rc) return rc;
  DeviceGuard g(t->device);
  cudaStream_t st = (cudaStream_t)stream;
  TableCall call;
  if ((rc = call.begin(t, st, CALL_ALL))) return rc;
  if ((rc = ensure_alloc(t))) return rc;
  const TableDev* h = t->tier && t->tier->allocated ? &t->tier->d : nullptr;
  PB_CUDA(launch_dump_nodes(t->d, h, d_signs, n_list, lo, n, t->dump, static_cast<uint8_t*>(d_out), st));
  return PB_OK;
}

// ---- checkpoint loads (pb_load.cu) ----------------------------------------------------------------------------------
struct pb_image {
  int device = 0;
  uint32_t max_chunk = 0;
  LoadImg L{};           // the image indexed last
  bool indexed = false;
  void* sum_mem = nullptr;  // dims, pairs, counts, flags of L
  uint64_t* off = nullptr;  // per position (whole images)
  uint8_t* slot = nullptr;
  uint32_t* sel = nullptr;  // the selected positions of one dim, in list order
  uint32_t* d_count = nullptr;
  uint32_t pos_cap = 0;
  void* tmp = nullptr;
  size_t tmp_bytes = 0;
  int sel_slot = -1;        // the dim slot `sel` holds
  uint64_t* st_signs = nullptr;  // aligned staging of one insert
  float* st_ent = nullptr;
  uint64_t st_entries = 0, st_floats = 0;
  std::vector<uint64_t> host_off;
  cudaStream_t st = nullptr;  // the stream of the latest call: workspace is allocated and freed in its order
  unsigned long long h_dims[LOAD_DIMS], h_pairs[LOAD_PAIRS];
  uint32_t h_counts[LOAD_PAIRS], h_flags[LOAD_FLAGS];
  Owned own;  // the workspace
};

namespace {

// The workspace is stream-ordered (Owned::async, released on the load's stream): a load beside training never waits
// for the device as a whole, and a buffer is released only after the inserts issued before that read it.
// The summary, on first use.
int image_ready(pb_image* im, cudaStream_t st) {
  im->st = st;
  if (im->sum_mem) return PB_OK;
  const size_t sum_bytes = sizeof(unsigned long long) * (LOAD_DIMS + LOAD_PAIRS) + sizeof(uint32_t) * (LOAD_PAIRS + LOAD_FLAGS);
  Owned o;
  int rc;  // (sum_mem, the gate, last)
  if ((rc = o.async(im->d_count, sizeof(uint32_t), st)) || (rc = o.async(im->sum_mem, sum_bytes + 16, st))) return rc;
  im->own.adopt(o);
  LoadImg& L = im->L;
  L.dims = static_cast<unsigned long long*>(im->sum_mem);
  L.pairs = L.dims + LOAD_DIMS;
  L.counts = reinterpret_cast<uint32_t*>(L.pairs + LOAD_PAIRS);
  L.flags = L.counts + LOAD_PAIRS;
  return PB_OK;
}

// workspace for n positions (grown, never shrunk while the load runs)
int image_room(pb_image* im, uint32_t n, cudaStream_t st) {
  int rc = image_ready(im, st);
  if (rc) return rc;
  if (n <= im->pos_cap && im->pos_cap) return PB_OK;
  im->own.release(im->off, st), im->own.release(im->slot, st), im->own.release(im->sel, st), im->own.release(im->tmp, st);
  im->pos_cap = 0;
  const uint32_t cap = n ? n : 1;
  const size_t tmp_bytes = load_list_bytes(cap);
  Owned o;
  uint64_t* off;
  uint8_t* slot;
  uint32_t* sel;
  void* tmp;
  if ((rc = o.async(off, sizeof(uint64_t) * cap, st)) || (rc = o.async(slot, cap, st)) ||
      (rc = o.async(sel, sizeof(uint32_t) * cap, st)) || (rc = o.async(tmp, tmp_bytes ? tmp_bytes : 16, st)))
    return rc;
  im->own.adopt(o);
  im->off = off, im->slot = slot, im->sel = sel, im->tmp = tmp, im->tmp_bytes = tmp_bytes;
  im->pos_cap = cap;
  return PB_OK;
}

// the selection of im->L (positions set up by the caller), its flags and summary read back; one host synchronisation
int image_select(pb_image* im, cudaStream_t st) {
  LoadImg& L = im->L;
  L.slot = im->slot;
  PB_CUDA(cudaMemsetAsync(L.dims, 0xFF, sizeof(unsigned long long) * (LOAD_DIMS + LOAD_PAIRS), st));
  PB_CUDA(cudaMemsetAsync(L.counts, 0, sizeof(uint32_t) * (LOAD_PAIRS + LOAD_FLAGS), st));
  PB_CUDA(launch_load_select(L, st));
  PB_CUDA(cudaMemcpyAsync(im->h_dims, L.dims, sizeof(im->h_dims), cudaMemcpyDeviceToHost, st));
  PB_CUDA(cudaMemcpyAsync(im->h_pairs, L.pairs, sizeof(im->h_pairs), cudaMemcpyDeviceToHost, st));
  PB_CUDA(cudaMemcpyAsync(im->h_counts, L.counts, sizeof(im->h_counts), cudaMemcpyDeviceToHost, st));
  PB_CUDA(cudaMemcpyAsync(im->h_flags, L.flags, sizeof(im->h_flags), cudaMemcpyDeviceToHost, st));
  PB_CUDA(cudaStreamSynchronize(st));
  im->sel_slot = -1;
  im->indexed = true;
  return PB_OK;
}

// the per-dim summary of the selection image_select made, and staging for its largest insert
int image_summary(pb_image* im, uint64_t* h_summary, uint32_t max_rows, uint32_t* h_rows, cudaStream_t st) {
  if (im->h_flags[LOAD_FLAG_FULL])
    return fail(PB_ERR_INVALID, "a checkpoint file holds more than " + std::to_string(LOAD_DIMS) + " dims or " +
                                    std::to_string(LOAD_PAIRS) + " (dim, entry length) pairs");
  // rows (dim, entry length, entries), and staging for the largest insert they allow
  uint32_t rows = 0;
  uint64_t most = 0, widest = 0;
  for (uint32_t j = 0; j < LOAD_PAIRS; ++j) {
    if (im->h_pairs[j] == KEY_EMPTY) continue;
    if (rows >= max_rows) return fail(PB_ERR_CAPACITY, "summary rows: pass room for " + std::to_string(LOAD_PAIRS));
    const uint64_t len = im->h_pairs[j] & 0xFFFFFFFFu;
    h_summary[3 * rows] = im->h_dims[im->h_pairs[j] >> 32];
    h_summary[3 * rows + 1] = len;
    h_summary[3 * rows + 2] = im->h_counts[j];
    ++rows;
    most = most > im->h_counts[j] ? most : im->h_counts[j];
    widest = widest > len ? widest : len;
  }
  *h_rows = rows;
  const uint64_t ent = most < im->max_chunk ? most : im->max_chunk;
  if (ent > im->st_entries || ent * widest > im->st_floats) {
    im->own.release(im->st_signs, st), im->own.release(im->st_ent, st);
    im->st_entries = 0, im->st_floats = 0;
    Owned o;
    uint64_t* signs;
    float* ent_rows;
    int rc;
    if ((rc = o.async(signs, sizeof(uint64_t) * ent, st)) || (rc = o.async(ent_rows, sizeof(float) * ent * widest, st))) return rc;
    im->own.adopt(o);
    im->st_signs = signs, im->st_ent = ent_rows, im->st_entries = ent, im->st_floats = ent * widest;
  }
  return PB_OK;
}

int image_device_ptr(const void* h, const uint8_t** d) {
  void* p = nullptr;
  PB_CUDA(cudaHostGetDevicePointer(&p, const_cast<void*>(h), 0));
  *d = static_cast<const uint8_t*>(p);
  return PB_OK;
}

}  // namespace

int pb_image_create(int device, uint32_t max_chunk, pb_image** out) {
  if (!out || !max_chunk) return fail(PB_ERR_INVALID, "null argument or zero max_chunk");
  pb_image* im = new pb_image();
  im->device = device;
  im->max_chunk = max_chunk;
  *out = im;
  return PB_OK;
}

int pb_image_destroy(pb_image* im) {
  if (!im) return PB_OK;
  DeviceGuard g(im->device);
  im->own.release_all(im->st);  // (after the inserts in flight on the load's stream)
  cudaStreamSynchronize(im->st);
  delete im;
  return PB_OK;
}

int pb_host_alloc(uint64_t bytes, void** out) {
  if (!out) return fail(PB_ERR_INVALID, "null argument");
  *out = nullptr;
  PB_CUDA(cudaHostAlloc(out, bytes ? bytes : 1, cudaHostAllocMapped | cudaHostAllocPortable));
  return PB_OK;
}

int pb_host_free(void* p) {
  if (p) PB_CUDA(cudaFreeHost(p));
  return PB_OK;
}

int pb_image_index(pb_image* im, const void* h_image, uint64_t nbytes, uint32_t p_lo, uint32_t p_hi, uint32_t R,
                   uint32_t rank, uint64_t* h_summary, uint32_t max_rows, uint32_t* h_rows, void* stream) {
  if (!im || !h_image || !h_summary || !h_rows) return fail(PB_ERR_INVALID, "null argument");
  if (R == 0 || rank >= R) return fail(PB_ERR_INVALID, "rank must be in 0..R-1");
  DeviceGuard g(im->device);
  cudaStream_t st = (cudaStream_t)stream;
  im->indexed = false;
  std::string err;
  try {
    if (!load_index_host(static_cast<const uint8_t*>(h_image), nbytes, im->host_off, err)) return fail(PB_ERR_FORMAT, err);
  } catch (const std::bad_alloc&) {
    return fail(PB_ERR_CAPACITY, "host memory for the node offsets of a " + std::to_string(nbytes) + "-byte image");
  }
  const uint32_t n = (uint32_t)im->host_off.size();
  int rc = image_room(im, n, st);
  if (rc) return rc;
  LoadImg& L = im->L;
  if ((rc = image_device_ptr(h_image, &L.img))) return rc;
  if (n) PB_CUDA(cudaMemcpyAsync(im->off, im->host_off.data(), sizeof(uint64_t) * n, cudaMemcpyHostToDevice, st));
  L.off = im->off;
  L.nb = 0, L.hdr = LOAD_NODE_HDR, L.n = n, L.p_lo = p_lo, L.p_hi = p_hi < n ? p_hi : n;
  L.node0 = 0, L.n_total = n, L.dim = 0, L.len = 0, L.R = R, L.rank = rank;
  if ((rc = image_select(im, st))) return rc;
  return image_summary(im, h_summary, max_rows, h_rows, st);
}

int pb_image_window(pb_image* im, const void* h_window, uint64_t node0, uint32_t n, uint64_t n_total, uint32_t entry_len,
                    uint64_t dim, uint32_t R, uint32_t rank, uint64_t* h_summary, uint32_t max_rows, uint32_t* h_rows,
                    int* h_writer, void* stream) {
  if (!im || !h_window || !h_summary || !h_rows || !h_writer) return fail(PB_ERR_INVALID, "null argument");
  if (R == 0 || rank >= R) return fail(PB_ERR_INVALID, "rank must be in 0..R-1");
  if (node0 + n > n_total || n_total >= (1ull << 32)) return fail(PB_ERR_INVALID, "nodes [node0, node0 + n) must lie in the file");
  DeviceGuard g(im->device);
  cudaStream_t st = (cudaStream_t)stream;
  im->indexed = false;
  int rc = image_room(im, n, st);
  if (rc) return rc;
  LoadImg& L = im->L;
  if ((rc = image_device_ptr(h_window, &L.img))) return rc;
  L.off = nullptr;
  L.nb = dump_node_bytes(entry_len), L.hdr = LOAD_NODE_HDR, L.n = n, L.p_lo = 0, L.p_hi = n;
  L.node0 = node0, L.n_total = n_total, L.dim = dim, L.len = entry_len, L.R = R, L.rank = rank;
  if ((rc = image_select(im, st)) || (rc = image_summary(im, h_summary, max_rows, h_rows, st))) return rc;
  *h_writer = im->h_flags[LOAD_FLAG_BAD] ? 0 : 1;
  if (!*h_writer) im->indexed = false;
  return PB_OK;
}

int pb_image_packet(pb_image* im, const void* h_packet, uint64_t nbytes, uint32_t R, uint32_t rank,
                    uint64_t* h_summary, uint32_t max_rows, uint32_t* h_rows, uint64_t* h_timestamp, void* stream) {
  if (!im || !h_packet || !h_summary || !h_rows || !h_timestamp) return fail(PB_ERR_INVALID, "null argument");
  if (R == 0 || rank >= R) return fail(PB_ERR_INVALID, "rank must be in 0..R-1");
  DeviceGuard g(im->device);
  cudaStream_t st = (cudaStream_t)stream;
  im->indexed = false;
  const uint8_t* b = static_cast<const uint8_t*>(h_packet);
  if (nbytes < 12) return fail(PB_ERR_FORMAT, "ValueError: truncated packet");
  uint32_t count, len0;
  std::memcpy(&count, b, 4);
  std::memcpy(&len0, b + 4, 4);
  LoadImg& L = im->L;
  const uint8_t* d_packet = nullptr;
  int rc = image_device_ptr(h_packet, &d_packet);
  if (rc) return rc;
  L.hdr = 0, L.node0 = 0, L.dim = 0, L.R = R, L.rank = rank;
  // uniform: the size of `count` entries of the first one's length (every packet this project writes with one dim)
  const uint64_t nb = 20 + 4ull * len0;  // (entries of 2^31 bytes or more are errors: packet_index_host)
  bool arithmetic = count && nb <= INT32_MAX && (nbytes - 12) % nb == 0 && (nbytes - 12) / nb == count;
  if (arithmetic) {
    if ((rc = image_room(im, count, st))) return rc;
    L.img = d_packet + 4, L.off = nullptr, L.nb = nb, L.len = len0;
    L.n = count, L.p_lo = 0, L.p_hi = count, L.n_total = count;
    if ((rc = image_select(im, st))) return rc;
    arithmetic = !im->h_flags[LOAD_FLAG_BAD];  // an entry of another length: the host walk finds out what it is
  }
  if (!arithmetic) {
    im->indexed = false;
    std::string err;
    try {
      if (!packet_index_host(b, nbytes, im->host_off, err)) return fail(PB_ERR_FORMAT, err);
    } catch (const std::bad_alloc&) {
      return fail(PB_ERR_CAPACITY, "host memory for the entry offsets of a " + std::to_string(nbytes) + "-byte packet");
    }
    const uint32_t n = (uint32_t)im->host_off.size();
    if ((rc = image_room(im, n, st))) return rc;
    if (n) PB_CUDA(cudaMemcpyAsync(im->off, im->host_off.data(), sizeof(uint64_t) * n, cudaMemcpyHostToDevice, st));
    L.img = d_packet, L.off = im->off, L.nb = 0, L.len = 0;
    L.n = n, L.p_lo = 0, L.p_hi = n, L.n_total = n;
    if ((rc = image_select(im, st))) return rc;
  }
  if (im->h_flags[LOAD_FLAG_FULL]) {
    im->indexed = false;
    return fail(PB_ERR_CAPACITY, "an incremental-update packet holds more than " + std::to_string(LOAD_DIMS) +
                                     " dims or " + std::to_string(LOAD_PAIRS) + " (dim, entry length) pairs");
  }
  if ((rc = image_summary(im, h_summary, max_rows, h_rows, st))) return rc;
  std::memcpy(h_timestamp, b + nbytes - 8, 8);
  return PB_OK;
}

int pb_image_insert(pb_image* im, pb_table* t, uint64_t dim, uint32_t lo, uint32_t hi, int newest_first, void* stream) {
  if (!im || !t) return fail(PB_ERR_INVALID, "null argument");
  if (!im->indexed) return fail(PB_ERR_STATE, "no image indexed: call pb_image_index, pb_image_window or pb_image_packet first");
  if (!t->has_op) return fail(PB_ERR_STATE, "optimizer not registered: entry length unknown");
  uint32_t len = 0;
  pb_table_entry_len(t, &len);
  int j = -1;
  for (uint32_t k = 0; k < LOAD_DIMS; ++k)
    if (im->h_dims[k] == dim) j = (int)k;
  uint64_t K = 0;
  for (uint32_t k = 0; j >= 0 && k < LOAD_PAIRS; ++k) {
    if (im->h_pairs[k] == KEY_EMPTY || (int)(im->h_pairs[k] >> 32) != j) continue;
    if ((im->h_pairs[k] & 0xFFFFFFFFu) != len)
      return fail(PB_ERR_INVALID, "the image's dim-" + std::to_string(dim) + " entries are not of the table's length");
    K += im->h_counts[k];
  }
  if (lo > hi || hi > K) return fail(PB_ERR_INVALID, "entries [lo, hi) must lie in the image's entries of `dim`");
  const uint32_t n = hi - lo;
  if (n > im->st_entries) return fail(PB_ERR_INVALID, "at most max_chunk entries per insert");
  if (!n) return PB_OK;
  DeviceGuard g(im->device);
  cudaStream_t st = (cudaStream_t)stream;
  if (im->sel_slot != j) {
    PB_CUDA(launch_load_list(im->L, (uint32_t)j, im->tmp, im->tmp_bytes, im->sel, im->d_count, st));
    im->sel_slot = j;
  }
  PB_CUDA(launch_load_gather(im->L, im->sel, (uint32_t)K, lo, n, newest_first, len, im->st_signs, im->st_ent, st));
  return pb_set_rows(t, im->st_signs, im->st_ent, n, stream);
}

int pb_add_prefix(const uint64_t* d_ids, uint32_t n, const uint32_t* h_slot_occ_off, const uint64_t* h_prefix,
                  uint32_t n_slots, uint32_t prefix_bit, uint64_t* d_out, void* stream) {
  if (n && (!d_ids || !d_out)) return fail(PB_ERR_INVALID, "null argument");
  if (!h_slot_occ_off || !h_prefix) return fail(PB_ERR_INVALID, "null argument");
  SlotsDev sl;
  int rc = prefix_slots(h_slot_occ_off, h_prefix, n_slots, prefix_bit, sl);
  if (rc) return rc;
  launch_add_prefix(sl, d_ids, n, d_out, (cudaStream_t)stream);
  PB_CUDA(cudaGetLastError());
  return PB_OK;
}

int pb_shard_of(const uint64_t* d_signs, uint32_t n, uint32_t R, uint32_t* d_shard, void* stream) {
  if (n && (!d_signs || !d_shard)) return fail(PB_ERR_INVALID, "null argument");
  if (R == 0) return fail(PB_ERR_INVALID, "replica size must be > 0");
  launch_shard_of(d_signs, n, R, d_shard, nullptr, (cudaStream_t)stream);
  PB_CUDA(cudaGetLastError());
  return PB_OK;
}

int pb_farmhash64(const uint64_t* d_in, uint32_t n, uint64_t* d_out, void* stream) {
  if (n && (!d_in || !d_out)) return fail(PB_ERR_INVALID, "null argument");
  launch_shard_of(d_in, n, 1, nullptr, d_out, (cudaStream_t)stream);
  PB_CUDA(cudaGetLastError());
  return PB_OK;
}

int pb_hash_stack(const uint64_t* d_ids, uint32_t n, uint32_t rounds, uint64_t embedding_size, uint64_t* d_out, void* stream) {
  if (n && (!d_ids || !d_out)) return fail(PB_ERR_INVALID, "null argument");
  if (rounds == 0 || embedding_size == 0) return fail(PB_ERR_INVALID, "hash_stack_rounds and embedding_size must be > 0");
  launch_hash_stack(d_ids, n, rounds, embedding_size, d_out, (cudaStream_t)stream);
  PB_CUDA(cudaGetLastError());
  return PB_OK;
}

uint64_t pb_partition_workspace(uint32_t n) { return partition_workspace_bytes(n); }

int pb_partition_by_shard(const uint64_t* d_signs, uint32_t n, uint32_t R, uint32_t* d_perm, uint32_t* d_counts,
                          void* d_work, uint64_t work_bytes, void* stream) {
  if ((n && (!d_signs || !d_perm)) || !d_counts || !d_work) return fail(PB_ERR_INVALID, "null argument");
  if (R == 0 || R > 256) return fail(PB_ERR_INVALID, "replica size must be in 1..256");
  if (work_bytes < pb_partition_workspace(n)) return fail(PB_ERR_CAPACITY, "workspace smaller than pb_partition_workspace(n)");
  launch_partition_by_shard(d_signs, n, R, d_perm, d_counts, (uint32_t*)d_work, (cudaStream_t)stream);
  PB_CUDA(cudaGetLastError());
  return PB_OK;
}

int pb_ctx_create(int device, uint32_t max_occurrences, uint32_t max_out_rows, pb_ctx** out) {
  if (!out || max_occurrences == 0 || max_out_rows == 0) return fail(PB_ERR_INVALID, "bad argument");
  if (max_occurrences > (1u << 24)) return fail(PB_ERR_INVALID, "at most 2^24 id occurrences per batch");
  DeviceGuard g(device);
  std::unique_ptr<pb_ctx> c(new pb_ctx());
  c->device = device;
  c->max_occ = max_occurrences;
  c->max_out = max_out_rows;
  std::memset(c->round_of, 0, sizeof(c->round_of));
  const size_t n = max_occurrences;
  c->set_cells = 2 * n + 2 * PB_MAX_SLOTS;  // region of slot s: 2*n_s + 1 cells and the reserved one
  c->b.giant_cap = n / PB_GIANT_MIN + 1;
  c->b.hot_cap = n / (PB_WARM_MAX + 1) + 1 + c->b.giant_cap;
  c->b.hot_words = (uint32_t)(n < 4096 ? 4096 : n);  // 32 bits of pool per id occurrence the context can hold
  Owned& o = c->own;
  int rc;
  if ((rc = o.dev(c->b.set, sizeof(DCell) * c->set_cells)) || (rc = o.dev(c->b.occ_set, 4 * n)) ||
      (rc = o.dev(c->b.item_cell, 4 * n)) || (rc = o.dev(c->b.seg_occ, 4 * n)) || (rc = o.dev(c->b.cold, 8 * n)) ||
      (rc = o.dev(c->b.warm, 16 * (n / 2 + 1))) || (rc = o.dev(c->b.hot, 16 * (size_t)c->b.hot_cap)) ||
      (rc = o.dev(c->b.hot_bits, 4 * (size_t)c->b.hot_words)) || (rc = o.dev(c->b.cnt, 4 * BC_COUNT)) ||
      (rc = o.dev(c->occ_cell, 4 * n)) || (rc = o.dev(c->occ_outrow, 4 * n)) ||
      (rc = o.dev(c->row_off, 4 * ((size_t)max_out_rows + 1))) || (rc = o.dev(c->nan_tick, 4 * PB_MAX_SLOTS)) ||
      (rc = o.dev(c->dev_tick, 4)) || (rc = o.dev(c->need, 4 * PB_MAX_RANKS)))
    return rc;
  PB_CUDA(cudaMemset(c->need, 0, 4 * PB_MAX_RANKS));
  PB_CUDA(cudaMemset(c->nan_tick, 0, 4 * PB_MAX_SLOTS));
  PB_CUDA(cudaMemset(c->dev_tick, 0, 4));
  PB_CUDA(cudaMemset(c->b.cnt, 0, 4 * BC_COUNT));
  PB_CUDA(cudaMemset(c->b.hot_bits, 0, 4 * (size_t)c->b.hot_words));
  launch_fill_set(c->b.set, c->set_cells, 0);
  PB_CUDA(cudaDeviceSynchronize());
  if ((rc = o.stream(c->side)) || (rc = o.stream(c->side2)) || (rc = o.stream(c->side3)) || (rc = o.event(c->ev_join2)) ||
      (rc = o.event(c->ev_fork)) || (rc = o.event(c->ev_nan)) || (rc = o.event(c->ev_join)) || (rc = o.event(c->ev_short)))
    return rc;
  *out = c.release();
  return PB_OK;
}

int pb_ctx_destroy(pb_ctx* c) {
  if (!c) return PB_OK;
  DeviceGuard g(c->device);
  cudaDeviceSynchronize();
  c->pending.drop();
  c->raw_pending.drop();
  delete c;
  return PB_OK;
}

int pb_ctx_set_slots(pb_ctx* c, const pb_slots_cfg* cfg) {
  if (!c || !cfg) return fail(PB_ERR_INVALID, "null argument");
  if (cfg->n_slots == 0 || cfg->n_slots > PB_MAX_SLOTS) return fail(PB_ERR_INVALID, "n_slots must be in 1..PB_MAX_SLOTS");
  if (cfg->prefix_bit == 0 || cfg->prefix_bit > 63)  // parse_embedding_config asserts > 0 (config lib.rs:624-627)
    return fail(PB_ERR_INVALID, "feature_index_prefix_bit must be in 1..63");
  c->slots = *cfg;
  c->has_slots = true;
  // two slots with the same prefix share a key space (one feature group): a sign may sit in both, and the reference
  // steps it once per slot, in slot order (mod.rs:720-822).  Slot s runs in round = number of earlier slots of its group.
  c->n_rounds = 1;
  std::memset(&c->links, 0xFF, sizeof(c->links));
  for (uint32_t i = 0; i < cfg->n_slots; ++i) {
    uint32_t r = 0;
    for (uint32_t k = 0; k < i; ++k)
      if (cfg->prefix[i] == cfg->prefix[k]) {
        ++r;
        c->links.prev[i] = (uint8_t)k;  // (the nearest earlier slot of the group is the last one found)
      }
    if (c->links.prev[i] != 0xFF) c->links.next[c->links.prev[i]] = (uint8_t)i;
    c->round_of[i] = (uint8_t)r;
    if (r + 1 > c->n_rounds) c->n_rounds = r + 1;
  }
  return PB_OK;
}

int pb_ctx_batch_stats(pb_ctx* c, uint32_t h_out[6], void* stream) {
  if (!c || !h_out) return fail(PB_ERR_INVALID, "null argument");
  DeviceGuard g(c->device);
  uint32_t w[BC_PEER];
  PB_CUDA(cudaMemcpyAsync(w, c->b.cnt, sizeof(w), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  PB_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
  h_out[0] = w[BC_ITEMS];
  h_out[1] = w[BC_COLD];
  h_out[2] = w[BC_WARM];
  h_out[3] = w[BC_HOT] + w[BC_HUGE] + w[BC_GIANT];
  h_out[4] = w[BC_SEG];
  h_out[5] = c->n_occ;
  return PB_OK;
}

// A backward's staging buffer `buf` of `floats` floats, held by `own`, grown to hold `need`.  The training forward grows
// it, so the backward that follows neither synchronises nor allocates (and can be captured without a warm-up call).  The first
// allocation neither synchronises nor enqueues anything, so that a context's first forward can be captured too: the
// thread's capture mode is relaxed around it (cudaMalloc is refused under a global-mode capture otherwise).  Growing
// synchronises the stream and frees the old buffer: a forward captured with a larger need than any call before it fails
// its capture, and a graph captured earlier must not be replayed after a larger call ran eagerly (warm up with the
// largest batch, as for vw_stage).
static int grow_stage(Owned& own, float*& buf, size_t& floats, size_t need, cudaStream_t st) {
  if (need <= floats) return PB_OK;
  if (buf) {  // the old buffer may still be read by enqueued work
    PB_CUDA(cudaStreamSynchronize(st));
    own.release(buf);
    floats = 0;
  }
  cudaStreamCaptureMode mode = cudaStreamCaptureModeRelaxed;
  PB_CUDA(cudaThreadExchangeStreamCaptureMode(&mode));
  const int rc = own.dev(buf, sizeof(float) * need);
  cudaThreadExchangeStreamCaptureMode(&mode);  // the caller's mode again
  if (rc) return rc;
  floats = need;
  return PB_OK;
}

int pb_forward(pb_table* t, pb_ctx* c, const uint64_t* d_ids, uint32_t n_occ, const uint32_t* d_row_off,
               const uint32_t* h_slot_occ_off, uint32_t batch, int training, void* d_out_f16, void* stream) {
  int rc = check_forward(t, c, d_ids, n_occ, d_row_off, h_slot_occ_off, batch, d_out_f16);
  if (rc) return rc;
  const uint64_t n_out = (uint64_t)c->slots.n_slots * batch;
  if (training) {
    if ((rc = writable(t)) || (rc = ready_for_training(t))) return rc;
  } else if (!t->has_op) {
    DeviceGuard g(t->device);
    PB_CUDA(cudaMemsetAsync(d_out_f16, 0, 2 * n_out * t->cfg.dim, (cudaStream_t)stream));
    return PB_OK;
  }
  DeviceGuard g(t->device);
  cudaStream_t st = (cudaStream_t)stream;
  TableCall call;
  if ((rc = call.begin(t, st, CALL_INDEX))) return rc;
  if ((rc = ensure_alloc(t)) || (training && (rc = grow_for(t, n_occ, st)))) return rc;
  // pb_backward's staging of the hot items' sums, hot_cap x dim floats (a wider table grows it)
  if (training && (rc = grow_stage(c->own, c->hot_stage, c->hot_stage_floats, (size_t)c->b.hot_cap * t->d.dim, st))) return rc;
  SlotsDev sl;
  if ((rc = make_slots(c->slots, h_slot_occ_off, sl))) return rc;
  if ((rc = begin_forward(t, c, sl, d_ids, n_occ, training, st))) return rc;
  // a training batch moves its tier-held signs into HBM rows (each distinct sign once); inference reads them in place
  if (t->tier && training) {
    TierWindow win(t, st);
    launch_tier_restore_items(t->d, t->tier->d, t->hy, t->op, c->b, st);
  }
  launch_probe_items(training != 0, t->d, t->hy, t->op, sl, c->b, st);
  if (t->tier && !training) {
    launch_tier_find_items(t->d, t->tier->d, c->b, st);
    launch_gather_items(t->d, sl, c->b, d_row_off, (uint32_t)n_out, batch, false, d_out_f16, st, t->tier->d.rows,
                        t->tier->d.capacity);
  } else {
    launch_gather_items(t->d, sl, c->b, d_row_off, (uint32_t)n_out, batch, training != 0, d_out_f16, st);
  }
  if ((rc = end_forward(t, c, d_row_off, h_slot_occ_off, n_occ, batch, training, st))) return rc;
  PB_CUDA(cudaGetLastError());
  return PB_OK;
}

int pb_backward(pb_table* t, pb_ctx* c, const void* const* h_grads, int is_f16, const float* h_scale,
                int32_t* d_slot_status, void* stream) {
  int rc = check_backward(t, c, h_grads);
  if (rc) return rc;
  uint32_t S = c->slots.n_slots;
  DeviceGuard g(t->device);
  cudaStream_t st = (cudaStream_t)stream;
  TableCall call;  // in the step chain only: runs beside the next forward and a pb_tier_stage (see there)
  if ((rc = call.begin(t, st, CALL_STEP))) return rc;
  SlotsDev sl;
  if ((rc = make_slots(c->slots, c->occ_off, sl))) return rc;
  GradsDev gr;
  if ((rc = make_grads(h_grads, h_scale, S, gr))) return rc;
  AdamKeys adam_keys{};
  if (t->op.kind == PB_OPT_ADAM) {  // get_batch_level_state: one power step per request and feature group
    AdamKeys keys{};
    for (uint32_t s = 0; s < S; ++s) {
      if (!h_grads[s]) continue;
      const int k = adam_index(t, c->slots.prefix[s]);
      if (k < 0) return fail(PB_ERR_CAPACITY, "more feature groups than Adam beta-power pairs");
      gr.pow_idx[s] = (uint8_t)k;
      bool done = false;
      for (uint32_t i = 0; i < keys.n; ++i) done |= keys.idx[i] == (uint8_t)k;
      if (!done) keys.idx[keys.n++] = (uint8_t)k;
    }
    gr.adam_pow = t->adam_dev;
    adam_keys = keys;  // advanced below, once the NaN marks of this request are known
  }
  float* vw = nullptr;
  if (t->op.kind == PB_OPT_ADAGRAD_VW) {
    if ((rc = grow_stage(c->own, c->vw_stage, c->vw_stage_floats, (size_t)c->n_occ * t->d.dim, st))) return rc;
    vw = c->vw_stage;
  }
  if ((size_t)c->b.hot_cap * t->d.dim > c->hot_stage_floats)
    return fail(PB_ERR_STATE, "pb_backward: the pending batch did not come from a training pb_forward of this table");
  ReduceArgs a = reduce_args(c);
  a.vw_stage = vw;
  a.hot_stage = c->hot_stage;
  a.short_max = hot_short_max(c->batch);
  auto set_round = [&](uint32_t r) {
    a.round = r;
    std::memset(a.round_mask, 0, sizeof(a.round_mask));
    for (uint32_t s = 0; s < S; ++s)
      if (c->round_of[s] == r) a.round_mask[s >> 5] |= 1u << (s & 31);
  };
  // One round (no shared feature groups, the usual case): the hot items' sums need no NaN mark, so their reduces — the
  // longest kernel of the step on `side`, and at large batches the light one for the short items on `side3` — start at
  // once, beside the NaN scan; once the marks and the short sums are known the hot rows are stepped on `side`,
  // and the cold and warm items are reduced and stepped on `st` and `side2`.  Several rounds (the items of a round are
  // distinct rows, whatever their list), or a kernel family being timed: everything on `st`, round after round.
  const bool beside = c->n_rounds == 1 && !profiling();
  if ((rc = fork_side(c, st))) return rc;
  if (beside) {
    set_round(0);
    launch_reduce_hot(t->d, sl, gr, is_f16 != 0, a, c->side);
    if (a.short_max) {
      PB_CUDA(cudaStreamWaitEvent(c->side3, c->ev_fork, 0));
      launch_reduce_hot_short(t->d, sl, gr, is_f16 != 0, a, c->side3);
      PB_CUDA(cudaEventRecord(c->ev_short, c->side3));
      PB_CUDA(cudaStreamWaitEvent(c->side, c->ev_short, 0));  // (joins `side3` back; the reduce queued before does not wait)
    }
  }
  const bool mark = t->inc.cells != nullptr;  // the mark reads the scratch set and empties it after the steps
  if (c->set_dirty && !mark) {
    launch_clear_items(c->b, c->side2);
    c->set_dirty = false;
  }
  uint32_t elems = c->batch * t->d.dim;
  launch_nan_scan(gr, S, elems, is_f16 != 0, c->dev_tick, c->nan_tick, d_slot_status, st);
  if (adam_keys.n) launch_adam_advance(t->adam_dev, adam_keys, t->op.b1, t->op.b2, st, &gr, S, c->dev_tick, c->nan_tick);
  if ((rc = fork_after_nan(c, st))) return rc;
  for (uint32_t r = 0; r < c->n_rounds; ++r) {
    set_round(r);
    if (!beside) {
      launch_reduce_hot(t->d, sl, gr, is_f16 != 0, a, st);
      launch_reduce_hot_short(t->d, sl, gr, is_f16 != 0, a, st);
    }
    launch_step_hot(t->d, t->op, t->hy, sl, gr, a, beside ? c->side : st);
    launch_reduce_items(t->d, t->op, t->hy, sl, gr, is_f16 != 0, a, st, beside ? c->side2 : st, false);
  }
  if ((rc = join_sides(c, st))) return rc;
  if (mark) {  // every round has stepped: the applied items that had a row
    IncSlots on{};
    for (uint32_t s = 0; s < S; ++s)
      if (h_grads[s]) on.applied[s >> 5] |= 1u << (s & 31);
    BatchDev b = c->b;
    b.n = c->n_occ;
    launch_inc_mark_items(t->inc, b, sl, on, c->dev_tick, c->nan_tick, c->set_dirty, st);
    c->set_dirty = false;
  }
  c->pending.drop();
  PB_CUDA(cudaGetLastError());
  return PB_OK;
}

// ---- the sharded path: R GPUs of one box -------------------------------------------------------------
struct pb_xchg {
  int device = 0;
  uint32_t dim = 0;
  XchgDev d{};
  uint32_t* mem = nullptr;  // epoch | waited | own_cnt | err | own_row | uwin
  UCell* ucell = nullptr;   // rows of the step's requests (owner side)
  uint64_t* akeys = nullptr;  // Adam: the table's feature-group prefixes on the device
  uint32_t* apresent = nullptr;
  float* apow = nullptr;
  size_t akeys_uploaded = 0;
  bool u_dirty = false;     // a training lookup filled ucell and its update has not run (abandoned batch)
  // a stage exchange (pb_xchg_create_stage): ctrl and sign areas only, dim 0 (so check_exchange refuses it); `sent`:
  // [PB_MAX_RANKS] signs of this rank's stage per owner (in `mem`, after the phase words)
  bool stage = false;
  uint32_t* sent = nullptr;
  Owned own;  // mem, ucell, akeys, apresent, apow
};

namespace {
uint64_t round256(uint64_t v) { return (v + 255u) & ~(uint64_t)255u; }
void xchg_layout(uint32_t R, uint32_t cap, uint32_t dim, int rows_f32, uint64_t off[6]) {
  off[0] = round256((uint64_t)XC_WORDS * PB_MAX_RANKS * 4);                        // sign
  off[1] = off[0] + round256((uint64_t)R * cap * 8);                               // row
  off[2] = off[1] + round256((uint64_t)R * cap * dim * (rows_f32 ? 4 : 2));        // grad
  off[3] = off[2] + round256((uint64_t)R * cap * dim * 4);                         // gok
  off[4] = off[3] + round256((uint64_t)R * cap * 4);                               // chain
  off[5] = off[4] + round256((uint64_t)R * cap * 4);                               // end
}

// a stage exchange's area: ctrl, then the R x cap signs sent to this rank (off[0] sign, off[1] end)
void xchg_stage_layout(uint32_t R, uint32_t cap, uint64_t off[2]) {
  off[0] = round256((uint64_t)XC_WORDS * PB_MAX_RANKS * 4);
  off[1] = off[0] + round256((uint64_t)R * cap * 8);
}

// the rows this rank's receive area holds, returned by the owners (the requester's FINISH reads them)
const void* received_rows(const pb_xchg* x) {
  return reinterpret_cast<const void*>(x->d.base[x->d.rank] + x->d.off_row);
}

// The phases a sharded call runs (PB_PHASE_*; 0 = all).  Each phase ends by signalling a flag of the exchange that a
// later phase of every peer waits for: a call that runs every phase waits for its peers' flags in the signal's launch
// (post); a phase-split call signals only, and its next phase starts by waiting (await).  wait_peers = false: the
// reader waits for each peer itself (the vectorwise Adagrad owner, owner_backward).  PB_PHASE_PREPARE signals nothing
// and is not part of that choice.
struct Phases {
  int mask;
  explicit Phases(int phases) : mask(phases ? phases : PB_PHASE_ALL) {}
  bool has(int phase) const { return (mask & phase) != 0; }
  bool exchanges() const { return (mask & PB_PHASE_ALL) != 0; }  // any phase beyond PREPARE
  bool all() const { return (mask & PB_PHASE_ALL) == PB_PHASE_ALL; }
  void post(const pb_xchg* x, int flag, const uint32_t* counts, cudaStream_t st, bool wait_peers = true) const {
    if (all() && wait_peers) launch_signal_wait(x->d, flag, counts, st);
    else launch_signal(x->d, flag, counts, st);
  }
  void await(const pb_xchg* x, int flag, cudaStream_t st) const {
    if (!all()) launch_wait(x->d, flag, -1, st);
  }
};

// A SEND after a PREPARE must bring the batch that was prepared (`kind` PREP_SUM or PREP_RAW): refused before anything
// is enqueued otherwise.
int check_prepared(const pb_ctx* c, const Phases& ph, int kind, uint32_t n_occ, uint32_t batch) {
  if (ph.has(PB_PHASE_PREPARE) || !ph.has(PB_PHASE_SEND) || c->prepared != kind) return PB_OK;
  if (c->prepared_n != n_occ || c->prepared_batch != batch)
    return fail(PB_ERR_STATE, "PB_PHASE_SEND after PB_PHASE_PREPARE must pass the prepared batch");
  return PB_OK;
}

// What a sharded call needs of its exchange: the table's device and dim, and f32 rows where `need_f32_rows` (refused
// with `f32_message`).  A backward passes its context, whose device it has not checked yet; a forward passes none
// (check_forward has checked it).
int check_exchange(const pb_table* t, const pb_ctx* c, const pb_xchg* x, bool need_f32_rows, const char* f32_message) {
  if (c && (t->device != c->device || t->device != x->device))
    return fail(PB_ERR_INVALID, "table, context and exchange live on different devices");
  if (t->device != x->device) return fail(PB_ERR_INVALID, "table and exchange live on different devices");
  if (x->dim != t->cfg.dim) return fail(PB_ERR_INVALID, "the exchange was sized for another embedding dim");
  if (need_f32_rows && !x->d.row_f32) return fail(PB_ERR_INVALID, f32_message);
  return PB_OK;
}

// The owner's part of a sharded forward (PB_PHASE_SERVE), shared by the summation and the raw calls: the rows of the
// signs sent to this shard, into the requesters' areas.  With a host tier, as on one GPU: a training request's tier-held
// signs move into HBM rows first (a sign that finds no free row stays in the tier, counted, and reads zeros), so the
// backward, the eviction check and the incremental marks see only HBM rows; an inference request reads them in place.
void serve_lookup(pb_table* t, pb_xchg* x, int training, const Phases& ph, cudaStream_t st) {
  ph.await(x, XC_FLAG_SIGN, st);
  if (training && x->u_dirty) launch_uclear(x->d, st);  // a training batch whose gradients never came left its rows noted
  if (training && t->tier) {
    TierWindow win(t, st);
    launch_tier_restore_recv(t->d, t->tier->d, t->hy, t->op, x->d, st);
  }
  launch_owner_lookup(training != 0, t->d, t->tier ? &t->tier->d : nullptr, t->hy, t->op, x->d, st);
  if (training) x->u_dirty = true;
  ph.post(x, XC_FLAG_ROW, nullptr, st);
}

// A growable owner's training SERVE admits up to R x cap signs (the R requests' receive areas): its table grows first
// (grow_for), and the call joins the table's index chain, which the read-back that bounds its growth relies on.  Every
// other sharded call orders nothing here, as before.
int owner_grow(pb_table* t, pb_xchg* x, int training, const Phases& ph, TableCall& call, cudaStream_t st) {
  if (!t->grow || !training || !ph.has(PB_PHASE_SERVE)) return PB_OK;
  if (int rc = call.begin(t, st, CALL_INDEX)) return rc;
  return grow_for(t, (uint64_t)x->d.R * x->d.cap, st);
}

// The owner's part of a sharded backward (PB_PHASE_SERVE), shared by the summation and the raw calls: the step's R
// gradient requests, every row stepped once per request in rank order.  prefix[n_prefix]: the feature groups of the
// slots the exchange serves (Adam beta powers).
int owner_backward(pb_table* t, pb_xchg* x, const uint64_t* prefix, uint32_t n_prefix, uint64_t spacing,
                   const Phases& ph, cudaStream_t st) {
  if (t->op.kind == PB_OPT_ADAGRAD_VW) {  // (needs the whole gradient's dot per step) one request after another
    for (uint32_t src = 0; src < x->d.R; ++src) {
      launch_wait(x->d, XC_FLAG_GRAD, (int)src, st);
      launch_owner_update(t->d, t->op, t->hy, x->d, src, st);
    }
    launch_uclear(x->d, st);
  } else {  // owner: the R requests in one launch, every row stepped in rank order
    ph.await(x, XC_FLAG_GRAD, st);
    if (t->op.kind == PB_OPT_ADAM) {  // every request advances the beta powers of the feature groups it holds here
      for (uint32_t s = 0; s < n_prefix; ++s)
        if (adam_index(t, prefix[s]) < 0) return fail(PB_ERR_CAPACITY, "more feature groups than Adam beta-power pairs");
      if (x->akeys_uploaded != t->adam_keys.size()) {  // (first steps only: not inside a graph capture)
        PB_CUDA(cudaStreamSynchronize(st));
        PB_CUDA(cudaMemcpy(x->akeys, t->adam_keys.data(), sizeof(uint64_t) * t->adam_keys.size(), cudaMemcpyHostToDevice));
        x->akeys_uploaded = t->adam_keys.size();
      }
      x->d.n_akeys = (uint32_t)t->adam_keys.size();
      x->d.amask = ~spacing;
      launch_owner_adam(x->d, t->adam_dev, t->op.b1, t->op.b2, st);
    }
    launch_owner_update_all(t->d, t->op, t->hy, x->d, st);
  }
  if (t->inc.cells) launch_inc_mark_owner(t->inc, x->d, t->d.capacity, st);  // the entries just stepped
  x->u_dirty = false;
  return PB_OK;
}
}  // namespace

uint64_t pb_xchg_bytes(uint32_t R, uint32_t cap, uint32_t dim, int rows_f32) {
  if (R == 0 || R > PB_MAX_RANKS || cap == 0 || dim == 0) return 0;
  uint64_t off[6];
  xchg_layout(R, cap, dim, rows_f32, off);
  return off[5];
}

int pb_xchg_create(int device, uint32_t R, uint32_t rank, uint32_t cap, uint32_t dim, int rows_f32,
                   const uint64_t* h_peer_base, pb_xchg** out) {
  if (!out || !h_peer_base || R == 0 || R > PB_MAX_RANKS || rank >= R || cap == 0 || dim == 0)
    return fail(PB_ERR_INVALID, "bad argument");
  if ((uint64_t)R * cap >= 0xFFFFFFF0ull) return fail(PB_ERR_INVALID, "R * cap must stay below 2^32 - 16");
  if (cap >= CHAIN_END) return fail(PB_ERR_INVALID, "cap must stay below 2^31 - 1");
  for (uint32_t q = 0; q < R; ++q)
    if (!h_peer_base[q] || (h_peer_base[q] & 255u)) return fail(PB_ERR_INVALID, "receive areas must be mapped and 256-byte aligned");
  DeviceGuard g(device);
  std::unique_ptr<pb_xchg> x(new pb_xchg());
  x->device = device;
  x->dim = dim;
  uint64_t off[6];
  xchg_layout(R, cap, dim, rows_f32, off);
  XchgDev& d = x->d;
  std::memset(&d, 0, sizeof(d));
  for (uint32_t q = 0; q < R; ++q) d.base[q] = h_peer_base[q];
  d.off_sign = off[0];
  d.off_row = off[1];
  d.off_grad = off[2];
  d.off_gok = off[3];
  d.off_chain = off[4];
  d.R = R;
  d.rank = rank;
  d.cap = cap;
  d.row_f32 = rows_f32 ? 1 : 0;
  const size_t words = XC_WORDS + (size_t)XC_WORDS * PB_MAX_RANKS + PB_MAX_RANKS + 4 + 3 * (size_t)R * cap + 1;
  uint32_t ucells = 1024;
  while ((size_t)ucells < 2 * (size_t)R * cap) ucells <<= 1;
  const size_t apresent_bytes = sizeof(uint32_t) * PB_MAX_RANKS * (PB_ADAM_KEYS / 32);
  int rc;
  if ((rc = x->own.dev(x->mem, 4 * words)) || (rc = x->own.dev(x->ucell, sizeof(UCell) * (size_t)ucells)) ||
      (rc = x->own.dev(x->akeys, sizeof(uint64_t) * PB_ADAM_KEYS)) || (rc = x->own.dev(x->apresent, apresent_bytes)) ||
      (rc = x->own.dev(x->apow, sizeof(float) * 2 * PB_MAX_RANKS * PB_ADAM_KEYS)))
    return rc;
  PB_CUDA(cudaMemset(x->mem, 0, 4 * words));
  PB_CUDA(cudaMemset(x->apresent, 0, apresent_bytes));
  d.epoch = x->mem;
  d.waited = d.epoch + XC_WORDS;
  d.own_cnt = d.waited + (size_t)XC_WORDS * PB_MAX_RANKS;
  d.err = d.own_cnt + PB_MAX_RANKS;
  d.own_row = d.err + 4;
  d.uwin = d.own_row + (size_t)R * cap;
  d.own_link = d.uwin + (size_t)R * cap;
  d.chained = d.own_link + (size_t)R * cap;
  d.ucell = x->ucell;
  d.ucells = ucells;
  d.akeys = x->akeys;
  d.apresent = x->apresent;
  d.apow = x->apow;
  launch_uclear(d, nullptr);
  PB_CUDA(cudaDeviceSynchronize());
  *out = x.release();
  return PB_OK;
}

int pb_xchg_destroy(pb_xchg* x) {
  if (!x) return PB_OK;
  DeviceGuard g(x->device);
  cudaDeviceSynchronize();
  delete x;
  return PB_OK;
}

uint64_t pb_xchg_stage_bytes(uint32_t R, uint32_t cap) {
  if (R == 0 || R > PB_MAX_RANKS || cap == 0 || (uint64_t)R * cap >= 0xFFFFFFF0ull) return 0;
  uint64_t off[2];
  xchg_stage_layout(R, cap, off);
  return off[1];
}

int pb_xchg_create_stage(int device, uint32_t R, uint32_t rank, uint32_t cap, const uint64_t* h_peer_base, pb_xchg** out) {
  if (!out || !h_peer_base || R == 0 || R > PB_MAX_RANKS || rank >= R || cap == 0)
    return fail(PB_ERR_INVALID, "bad argument");
  if ((uint64_t)R * cap >= 0xFFFFFFF0ull) return fail(PB_ERR_INVALID, "R * cap must stay below 2^32 - 16");
  for (uint32_t q = 0; q < R; ++q)
    if (!h_peer_base[q] || (h_peer_base[q] & 255u)) return fail(PB_ERR_INVALID, "stage areas must be mapped and 256-byte aligned");
  DeviceGuard g(device);
  std::unique_ptr<pb_xchg> x(new pb_xchg());
  x->device = device;
  x->stage = true;  // dim 0: no row, gradient or chain area, no ucell set, no Adam arrays
  uint64_t off[2];
  xchg_stage_layout(R, cap, off);
  XchgDev& d = x->d;
  std::memset(&d, 0, sizeof(d));
  for (uint32_t q = 0; q < R; ++q) d.base[q] = h_peer_base[q];
  d.off_sign = off[0];
  d.off_row = d.off_grad = d.off_gok = d.off_chain = off[1];
  d.R = R;
  d.rank = rank;
  d.cap = cap;
  const size_t words = XC_WORDS + (size_t)XC_WORDS * PB_MAX_RANKS + PB_MAX_RANKS + 4;  // epoch | waited | sent | err
  if (int rc = x->own.dev(x->mem, 4 * words)) return rc;
  PB_CUDA(cudaMemset(x->mem, 0, 4 * words));
  PB_CUDA(cudaDeviceSynchronize());
  d.epoch = x->mem;
  d.waited = d.epoch + XC_WORDS;
  x->sent = d.waited + (size_t)XC_WORDS * PB_MAX_RANKS;
  d.err = x->sent + PB_MAX_RANKS;
  *out = x.release();
  return PB_OK;
}

int pb_tier_stage_sharded(pb_table* t, pb_xchg* xs, const uint64_t* d_ids, uint32_t n, const uint32_t* h_slot_occ_off,
                          const uint64_t* h_prefix, uint32_t n_slots, uint32_t prefix_bit, void* stream, int phases) {
  if (!t || !xs || (n && !d_ids) || !h_slot_occ_off || !h_prefix) return fail(PB_ERR_INVALID, "null argument");
  if (!xs->stage)
    return fail(PB_ERR_INVALID, "a batch exchange carries no stage: create a stage exchange (pb_xchg_create_stage)");
  if (phases & ~(PB_PHASE_SEND | PB_PHASE_SERVE))
    return fail(PB_ERR_INVALID, "a stage has the phases PB_PHASE_SEND and PB_PHASE_SERVE only");
  if (t->tier_of) return fail(PB_ERR_STATE, "a host tier is not staged directly: use the table it is attached to");
  if (n_slots == 0 || n_slots > PB_MAX_SLOTS) return fail(PB_ERR_INVALID, "n_slots must be in 1..PB_MAX_SLOTS");
  if (prefix_bit == 0 || prefix_bit > 63) return fail(PB_ERR_INVALID, "feature_index_prefix_bit must be in 1..63");
  if (t->device != xs->device) return fail(PB_ERR_INVALID, "table and exchange live on different devices");
  int rc = check_slot_offsets(h_slot_occ_off, n_slots, n);
  if (rc || (rc = writable(t))) return rc;  // (its eviction check)
  if (t->tier && (rc = ready_for_training(t))) return rc;
  SlotsDev sl;
  if ((rc = prefix_slots(h_slot_occ_off, h_prefix, n_slots, prefix_bit, sl))) return rc;
  DeviceGuard g(t->device);
  cudaStream_t st = (cudaStream_t)stream;
  // a stage has no FINISH: SEND and SERVE together are the whole call (one process per GPU: one signal-and-wait launch)
  const int mask = phases ? phases : PB_PHASE_SEND | PB_PHASE_SERVE;
  const Phases ph(mask == (PB_PHASE_SEND | PB_PHASE_SERVE) ? PB_PHASE_ALL : mask);
  if (ph.has(PB_PHASE_SEND)) {  // requester: the next batch's signs -> their owners' stage areas
    PB_CUDA(cudaMemsetAsync(xs->sent, 0, 4 * PB_MAX_RANKS, st));
    launch_stage_route(sl, d_ids, n, xs->d, xs->sent, st);
    ph.post(xs, XC_FLAG_SIGN, xs->sent, st);
  }
  if (ph.has(PB_PHASE_SERVE)) {  // owner: the check the next request would run, then the received signs' restores
    ph.await(xs, XC_FLAG_SIGN, st);
    if (t->tier) {
      // Outside the table's chains, like every sharded call (the caller orders it; see include/persia_b200.h).  Not
      // counted in train_calls; keep covers the batches pending now.  Beside a sharded backward: no owner-side backward
      // kernel reads index cells, the free-row stack or row_tick, and the rows they step are never victims here (keep >
      // pending_batches) nor restore targets (those come off the free stack).
      if (t->evict_every && (rc = evict_check(t, st, g_stage_blocks))) return rc;
      TierWindow win(t, st);
      launch_tier_restore_recv(t->d, t->tier->d, t->hy, t->op, xs->d, st, g_stage_blocks);
    }
  }
  PB_CUDA(cudaGetLastError());
  return PB_OK;
}

int pb_xchg_need(pb_xchg* x, pb_ctx* c, uint32_t h_out[1], void* stream) {
  if (!x || !c || !h_out) return fail(PB_ERR_INVALID, "null argument");
  if (x->device != c->device) return fail(PB_ERR_INVALID, "context and exchange live on different devices");
  if (c->prepared == PREP_NONE) return fail(PB_ERR_STATE, "no batch of this context is prepared (PB_PHASE_PREPARE)");
  DeviceGuard g(x->device);
  uint32_t n[PB_MAX_RANKS];
  PB_CUDA(cudaMemcpyAsync(n, c->need, 4 * (size_t)x->d.R, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  PB_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
  uint32_t most = 0;
  for (uint32_t q = 0; q < x->d.R; ++q) most = n[q] > most ? n[q] : most;
  h_out[0] = most;
  return PB_OK;
}

int pb_xchg_status(pb_xchg* x, uint32_t h_out[2], void* stream) {
  if (!x || !h_out) return fail(PB_ERR_INVALID, "null argument");
  DeviceGuard g(x->device);
  PB_CUDA(cudaMemcpyAsync(h_out, x->d.err, 8, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  PB_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
  return PB_OK;
}

int pb_forward_sharded(pb_table* t, pb_ctx* c, pb_xchg* x, const uint64_t* d_ids, uint32_t n_occ, const uint32_t* d_row_off,
                       const uint32_t* h_slot_occ_off, uint32_t batch, int training, void* d_out_f16, void* stream,
                       int phases) {
  const Phases ph(phases);
  if (!x) return fail(PB_ERR_INVALID, "null argument");
  int rc = check_forward(t, c, d_ids, n_occ, d_row_off, h_slot_occ_off, batch, d_out_f16);
  // (a PREPARE alone may meet a ragged batch on an f16 exchange: finding that out is what it is for)
  if (rc || (rc = check_exchange(t, nullptr, x, d_row_off != nullptr && ph.exchanges(),
                                 "ragged layouts need an exchange created with f32 rows")) ||
      (rc = check_prepared(c, ph, PREP_SUM, n_occ, batch)) || (training && (rc = writable(t))))
    return rc;
  const uint64_t n_out = (uint64_t)c->slots.n_slots * batch;
  // every rank serves lookups whether or not its own batch trains: the shard must be usable (a collective call)
  if ((rc = ready_for_training(t))) return rc;
  DeviceGuard g(t->device);
  cudaStream_t st = (cudaStream_t)stream;
  if (ph.exchanges() && (rc = ensure_alloc(t))) return rc;
  TableCall call;
  if ((rc = owner_grow(t, x, training, ph, call, st))) return rc;
  SlotsDev sl;
  if ((rc = make_slots(c->slots, h_slot_occ_off, sl))) return rc;
  if (ph.has(PB_PHASE_PREPARE)) {  // requester, local: the dedup and its items per owner
    prepare_batch(t, c, sl, d_ids, n_occ, batch, st);
    PB_CUDA(cudaMemsetAsync(c->need, 0, 4 * PB_MAX_RANKS, st));
    launch_count_owners(false, c->b, c->raw, n_occ, x->d.R, c->need, st);
  }
  if (ph.has(PB_PHASE_SEND)) {
    if ((rc = begin_forward(t, c, sl, d_ids, n_occ, training, st, c->prepared == PREP_SUM))) return rc;
    launch_route_items(training != 0, sl, c->b, x->d, st);               // requester: signs -> owners' areas
    if (training && c->n_rounds > 1) launch_link_items(sl, c->b, x->d, c->links, st);  // a sign's entries, slot order
    ph.post(x, XC_FLAG_SIGN, c->b.cnt + BC_PEER, st);
  }
  if (ph.has(PB_PHASE_SERVE)) serve_lookup(t, x, training, ph, st);
  if (ph.has(PB_PHASE_FINISH)) {
    ph.await(x, XC_FLAG_ROW, st);
    launch_expand_items(t->d, sl, c->b, received_rows(x), x->d.row_f32 != 0, d_row_off, (uint32_t)n_out, batch,
                        training != 0, d_out_f16, st);
    if ((rc = end_forward(t, c, d_row_off, h_slot_occ_off, n_occ, batch, training, st))) return rc;
  }
  PB_CUDA(cudaGetLastError());
  return PB_OK;
}

int pb_backward_sharded(pb_table* t, pb_ctx* c, pb_xchg* x, const void* const* h_grads, int is_f16, const float* h_scale,
                        int32_t* d_slot_status, void* stream, int phases) {
  const Phases ph(phases);
  if (!x) return fail(PB_ERR_INVALID, "null argument");
  if (ph.has(PB_PHASE_PREPARE)) return fail(PB_ERR_INVALID, "PB_PHASE_PREPARE is a phase of the sharded forwards");
  int rc = check_backward(t, c, h_grads);
  if (rc || (rc = check_exchange(t, c, x, false, nullptr))) return rc;
  uint32_t S = c->slots.n_slots;
  DeviceGuard g(t->device);
  cudaStream_t st = (cudaStream_t)stream;
  SlotsDev sl;
  if ((rc = make_slots(c->slots, c->occ_off, sl))) return rc;
  GradsDev gr;
  if ((rc = make_grads(h_grads, h_scale, S, gr))) return rc;
  if (ph.has(PB_PHASE_SEND)) {
    if ((rc = fork_side(c, st))) return rc;
    if (c->set_dirty) {
      launch_clear_items(c->b, c->side);
      c->set_dirty = false;
    }
    launch_nan_scan(gr, S, c->batch * t->d.dim, is_f16 != 0, c->dev_tick, c->nan_tick, d_slot_status, st);  // per slot, on the requester (mod.rs:731-746)
    if ((rc = fork_after_nan(c, st))) return rc;
    ReduceArgs a = reduce_args(c);
    for (uint32_t s = 0; s < S; ++s) a.round_mask[s >> 5] |= 1u << (s & 31);
    a.x = x->d;
    // requester: gradients -> owners' areas
    launch_reduce_hot(t->d, sl, gr, is_f16 != 0, a, profiling() ? st : c->side, true);
    launch_reduce_items(t->d, t->op, t->hy, sl, gr, is_f16 != 0, a, st, profiling() ? st : c->side2, true);
    if ((rc = join_sides(c, st))) return rc;
    ph.post(x, XC_FLAG_GRAD, nullptr, st, t->op.kind != PB_OPT_ADAGRAD_VW);
  }
  if (ph.has(PB_PHASE_SERVE)) {
    if ((rc = owner_backward(t, x, c->slots.prefix, S, sl.spacing, ph, st))) return rc;
    c->pending.drop();
  }
  PB_CUDA(cudaGetLastError());
  return PB_OK;
}

// ---- raw slots ------------------------------------------------------------------------------------
static int ensure_raw(pb_ctx* c) {
  if (c->raw_ready) return PB_OK;
  RawWork w = c->raw;
  size_t n = c->max_occ;
  size_t m = n > c->max_out ? n : c->max_out;
  uint32_t cells = next_pow2(2 * (uint64_t)n < 1024 ? 1024 : 2 * (uint64_t)n);
  w.set_mask = cells - 1;
  Owned o;
  int rc;
  if ((rc = o.dev(w.set, sizeof(RawCell) * ((size_t)cells + 1))) || (rc = o.dev(w.occ_set, 4 * n)) ||
      (rc = o.dev(w.flag, 4 * m)) || (rc = o.dev(w.rank, 4 * m)) ||
      (rc = o.dev(w.tiles, 4 * (size_t)raw_scan_tiles((uint32_t)m))) || (rc = o.dev(w.distinct_cell, 4 * n)) ||
      (rc = o.dev(w.counts, 8)) || (rc = o.dev(w.target, 4 * n)) || (rc = o.dev(w.peer, 4 * PB_MAX_RANKS)))
    return rc;
  PB_CUDA(cudaMemset(w.counts, 0, 8));
  c->own.adopt(o);
  c->raw = w;
  c->raw_ready = true;
  return PB_OK;
}

// pb_backward_raw's f32 staging buffer: one row per distinct sign of the batch, so n_occ x dim floats bound it.  Sized
// by the batch, not by max_occ: a context made at twice a batch's ids (persia_core) would otherwise ask for twice the
// staging, 64 GB at 2^24 occurrences and dim 1024.  It grows when a larger batch or dim comes.
static int ensure_raw_stage(pb_ctx* c, uint32_t n_occ, uint32_t dim, cudaStream_t st) {
  return grow_stage(c->own, c->raw_stage, c->raw_stage_floats, (size_t)(n_occ ? n_occ : 1) * dim, st);
}

int pb_forward_raw(pb_table* t, pb_ctx* c, const uint64_t* d_ids, uint32_t n_occ, const uint32_t* d_row_off,
                   uint32_t batch, uint32_t sample_fixed_size, int training, void* d_table_f16, int64_t* d_index,
                   int64_t* d_non_empty, uint32_t* d_sample_id_num, uint32_t* d_counts, void* stream) {
  int rc = check_raw_forward(t, c, d_ids, n_occ, d_row_off, batch, sample_fixed_size, d_table_f16, d_index, d_non_empty,
                             d_sample_id_num, d_counts);
  if (rc) return rc;
  if (training) {
    if ((rc = writable(t)) || (rc = ready_for_training(t))) return rc;
  } else if (!t->has_op) {
    return fail(PB_ERR_STATE, "optimizer not registered (OptimizerNotFoundError)");
  }
  DeviceGuard g(t->device);
  cudaStream_t st = (cudaStream_t)stream;
  TableCall call;
  if ((rc = call.begin(t, st, CALL_INDEX))) return rc;
  if ((rc = ensure_alloc(t))) return rc;
  if ((rc = ensure_raw(c))) return rc;
  if (training && ((rc = ensure_raw_stage(c, n_occ, t->d.dim, st)) || (rc = grow_for(t, n_occ, st)))) return rc;
  SlotsDev sl;
  if ((rc = raw_slots(c, n_occ, sl))) return rc;
  c->raw_pending.drop();  // the numbering below replaces the pending batch's
  c->prepared = PREP_NONE;
  if (training) {
    if ((rc = maybe_evict(t, st))) return rc;
    launch_begin_batch(t->d, c->dev_tick, nullptr, st);
    restore_ids(t, true, sl, d_ids, n_occ, st);
    launch_probe(MODE_TRAIN, true, t->d, t->hy, t->op, sl, d_ids, n_occ, c->occ_cell, st);
  } else {
    launch_probe(MODE_FIND, true, t->d, t->hy, t->op, sl, d_ids, n_occ, c->occ_cell, st);
  }
  if (d_row_off && (rc = copy_row_off(c, d_row_off, batch, st))) return rc;
  launch_raw_forward(t->d, sl, d_ids, n_occ, d_row_off ? c->row_off : nullptr, d_row_off ? c->occ_outrow : nullptr,
                     batch, sample_fixed_size, c->occ_cell, c->raw, d_table_f16, (long long*)d_index,
                     (long long*)d_non_empty, d_sample_id_num, st);
  if (!training && t->tier)  // inference moves nothing: tier-held signs are read where they are
    launch_tier_raw_fill(t->d, t->tier->d, sl, d_ids, n_occ, c->occ_cell, c->raw, d_table_f16, st);
  PB_CUDA(cudaMemcpyAsync(d_counts, c->raw.counts, 8, cudaMemcpyDeviceToDevice, st));
  if (training) hold_raw_batch(t, c, n_occ, batch);
  PB_CUDA(cudaGetLastError());
  return PB_OK;
}

int pb_backward_raw(pb_table* t, pb_ctx* c, const void* d_grad, int is_f16, float scale, int32_t* d_status,
                    void* stream) {
  if (!t || !c) return fail(PB_ERR_INVALID, "null argument");
  int rc = check_raw_backward(t, c, d_grad);
  if (rc) return rc;
  DeviceGuard g(t->device);
  cudaStream_t st = (cudaStream_t)stream;
  TableCall call;  // in the step chain only: runs beside the next forward and a pb_tier_stage (see there)
  if ((rc = call.begin(t, st, CALL_STEP))) return rc;
  c->raw_pending.drop();  // enqueued below: the sweep of the next training call runs after these gradients
  GradsDev gr;
  std::memset(&gr, 0, sizeof(gr));
  gr.ptr[0] = d_grad;
  if (!d_grad) {  // add_skipped_gradient
    if (d_status) launch_slot_status(gr, 1, c->dev_tick, c->nan_tick, d_status, st);
    return PB_OK;
  }
  uint8_t do_scale;
  float inv;
  if ((rc = loss_scale(scale, do_scale, inv))) return rc;
  const float* pair = nullptr;
  if (t->op.kind == PB_OPT_ADAM) {  // one power step per request and feature group
    const int k = adam_index(t, c->slots.prefix[0]);
    if (k < 0) return fail(PB_ERR_CAPACITY, "more feature groups than Adam beta-power pairs");
    pair = advance_adam_pair(t, k, st);
  }
  const uint32_t dim = t->d.dim;
  launch_raw_nan(d_grad, is_f16 != 0, c->raw.counts, dim, c->dev_tick, c->nan_tick, st);
  if (d_status) launch_slot_status(gr, 1, c->dev_tick, c->nan_tick, d_status, st);
  // Always staged, f32 without a loss scale included: the EW adds each row into zeros (mod.rs:780-798), which turns a -0
  // gradient into +0.  pb_update takes its gradients as given, like the PS (PS mod.rs:359-427), so the step does not.
  // The pending training forward allocated the buffer for this table's dim; only another table's larger dim allocates.
  if ((rc = ensure_raw_stage(c, c->n_occ, dim, st))) return rc;
  launch_raw_stage(d_grad, is_f16 != 0, c->raw.counts, dim, inv, do_scale != 0, c->raw_stage, st);
  launch_update_direct(t->d, t->op, t->hy, c->raw.target, c->raw_stage, c->n_occ, pair, st, c->raw.counts,
                       c->dev_tick, c->nan_tick, true);
  if (t->inc.cells && c->n_occ) launch_inc_mark_raw(t->inc, c->raw, c->n_occ, c->dev_tick, c->nan_tick, st);
  PB_CUDA(cudaGetLastError());
  return PB_OK;
}

int pb_forward_raw_sharded(pb_table* t, pb_ctx* c, pb_xchg* x, const uint64_t* d_ids, uint32_t n_occ,
                           const uint32_t* d_row_off, uint32_t batch, uint32_t sample_fixed_size, int training,
                           void* d_table_f16, int64_t* d_index, int64_t* d_non_empty, uint32_t* d_sample_id_num,
                           uint32_t* d_counts, void* stream, int phases) {
  const Phases ph(phases);
  if (!x) return fail(PB_ERR_INVALID, "null argument");
  int rc = check_raw_forward(t, c, d_ids, n_occ, d_row_off, batch, sample_fixed_size, d_table_f16, d_index, d_non_empty,
                             d_sample_id_num, d_counts);
  if (rc || (rc = check_exchange(t, nullptr, x, ph.exchanges(),
                                 "raw slots need an exchange created with f32 rows (the requester rounds them)")) ||
      (rc = check_prepared(c, ph, PREP_RAW, n_occ, batch)) || (training && (rc = writable(t))))
    return rc;
  // every rank serves lookups whether or not its own batch trains: the shard must be usable (a collective call)
  if ((rc = ready_for_training(t))) return rc;
  DeviceGuard g(t->device);
  cudaStream_t st = (cudaStream_t)stream;
  if (ph.exchanges() && (rc = ensure_alloc(t))) return rc;
  TableCall call;
  if ((rc = owner_grow(t, x, training, ph, call, st)) || (rc = ensure_raw(c))) return rc;
  SlotsDev sl;
  if ((rc = raw_slots(c, n_occ, sl))) return rc;
  // the slot's distinct signs numbered, index / non_empty / sample_id_num written: no table state is read
  auto number = [&]() -> int {
    if (d_row_off && (rc = copy_row_off(c, d_row_off, batch, st))) return rc;
    launch_raw_number(sl, d_ids, n_occ, d_row_off ? c->row_off : nullptr, d_row_off ? c->occ_outrow : nullptr, batch,
                      sample_fixed_size, nullptr, c->raw, (long long*)d_index, (long long*)d_non_empty, d_sample_id_num,
                      st);
    PB_CUDA(cudaMemcpyAsync(d_counts, c->raw.counts, 8, cudaMemcpyDeviceToDevice, st));
    return PB_OK;
  };
  if (ph.has(PB_PHASE_PREPARE)) {  // requester, local: the numbering and its distinct signs per owner
    c->raw_pending.drop();  // the numbering below replaces the pending batch's
    if ((rc = number())) return rc;
    PB_CUDA(cudaMemsetAsync(c->need, 0, 4 * PB_MAX_RANKS, st));
    launch_count_owners(true, c->b, c->raw, n_occ, x->d.R, c->need, st);
    c->prepared = PREP_RAW;
    c->prepared_n = n_occ;
    c->prepared_batch = batch;
  }
  if (ph.has(PB_PHASE_SEND)) {
    const bool prepared = c->prepared == PREP_RAW;
    c->prepared = PREP_NONE;
    if (!prepared) c->raw_pending.drop();
    if (training) {
      if ((rc = maybe_evict(t, st))) return rc;
      launch_begin_batch(t->d, c->dev_tick, nullptr, st);
    }
    if (!prepared && (rc = number())) return rc;
    PB_CUDA(cudaMemsetAsync(c->raw.peer, 0, 4 * PB_MAX_RANKS, st));
    launch_raw_route(c->raw, n_occ, x->d, st);  // requester: distinct signs -> owners' areas
    ph.post(x, XC_FLAG_SIGN, c->raw.peer, st);
  }
  if (ph.has(PB_PHASE_SERVE)) serve_lookup(t, x, training, ph, st);
  if (ph.has(PB_PHASE_FINISH)) {
    ph.await(x, XC_FLAG_ROW, st);
    launch_raw_fill(c->raw, n_occ, t->d.dim, static_cast<const float*>(received_rows(x)), d_table_f16, st);  // rows in -> table
    if (training) hold_raw_batch(t, c, n_occ, batch);
  }
  PB_CUDA(cudaGetLastError());
  return PB_OK;
}

int pb_backward_raw_sharded(pb_table* t, pb_ctx* c, pb_xchg* x, const void* d_grad, int is_f16, float scale,
                            int32_t* d_status, void* stream, int phases) {
  const Phases ph(phases);
  if (!t || !c || !x) return fail(PB_ERR_INVALID, "null argument");
  if (ph.has(PB_PHASE_PREPARE)) return fail(PB_ERR_INVALID, "PB_PHASE_PREPARE is a phase of the sharded forwards");
  if (!c->has_slots || c->slots.n_slots != 1) return fail(PB_ERR_STATE, "a raw context serves exactly one slot (pb_ctx_set_slots)");
  int rc = check_exchange(t, c, x, false, nullptr);
  if (rc || (rc = check_raw_backward(t, c, d_grad))) return rc;
  uint8_t do_scale = 0;  // (add_skipped_gradient: the send reads no gradient, nor its scale)
  float inv = 1.0f;
  if (d_grad && (rc = loss_scale(scale, do_scale, inv))) return rc;
  DeviceGuard g(t->device);
  cudaStream_t st = (cudaStream_t)stream;
  const uint32_t dim = t->d.dim;
  if (ph.has(PB_PHASE_SEND)) {  // the NaN rule, add_skipped_gradient, the clamp and 1/scale: on the requester
    GradsDev gr;
    std::memset(&gr, 0, sizeof(gr));
    gr.ptr[0] = d_grad;
    if (d_grad) launch_raw_nan(d_grad, is_f16 != 0, c->raw.counts, dim, c->dev_tick, c->nan_tick, st);
    if (d_status) launch_slot_status(gr, 1, c->dev_tick, c->nan_tick, d_status, st);
    launch_raw_send(d_grad, is_f16 != 0, c->raw, c->n_occ, dim, inv, do_scale != 0, c->dev_tick, c->nan_tick, x->d, st);
    ph.post(x, XC_FLAG_GRAD, nullptr, st, t->op.kind != PB_OPT_ADAGRAD_VW);
  }
  if (ph.has(PB_PHASE_SERVE)) {
    SlotsDev sl;
    if ((rc = raw_slots(c, c->n_occ, sl))) return rc;
    if ((rc = owner_backward(t, x, c->slots.prefix, 1, sl.spacing, ph, st))) return rc;
    c->raw_pending.drop();
  }
  PB_CUDA(cudaGetLastError());
  return PB_OK;
}

// ---- inference on R GPUs one rank at a time: views of the owners' tables --------------------------------------------
namespace {
// The bytes pb_table_export_view writes: what a peer needs to read the table in place.
constexpr uint32_t VIEW_MAGIC = 0x57564250u;  // "PBVW"
constexpr uint32_t VIEW_VERSION = 1;
constexpr uint32_t VIEW_VERSION_TIERED = 2;  // the same layout, of a table with a shared tier: opened with its tier blob
enum { VA_CELLS = 0, VA_ROWS, VA_COUNTERS, VA_SEQ, VA_COUNT };  // the allocations a reader touches
struct ViewBlob {
  uint32_t magic, version;
  uint64_t pid;                                // the exporting process ...
  uint64_t nonce;                              // ... and its random number (pids repeat across PID namespaces)
  int32_t device;                              // its device ordinal, in the exporting process
  uint32_t ipc;                                // 1: the handles below are valid
  uint64_t ptr[VA_COUNT];                      // device pointers in the exporting process
  cudaIpcMemHandle_t handle[VA_COUNT];         // the same allocations for other processes
  uint32_t dim, stride, state_floats, n_cells, capacity, pad;
};
// The bytes pb_table_export_tier_view writes: the shared tier behind a table exported with version 2.
constexpr uint32_t TIER_MAGIC = 0x54564250u;  // "PBVT"
constexpr uint32_t TIER_VERSION = 1;
struct TierBlob {
  uint32_t magic, version;
  uint64_t pid, nonce;             // the exporting process (as ViewBlob)
  int32_t device;                  // its device ordinal, in the exporting process
  uint32_t ipc;                    // 1: `handle` is valid
  uint64_t cells, rows;            // device pointers of the tier's index cells and (mapped) rows, in the exporter
  cudaIpcMemHandle_t handle;       // the index cells for other processes
  int32_t fd;                      // the memfd of the rows in the exporting process (/proc/<pid>/fd/<fd>) ...
  uint32_t pad0;
  uint64_t bytes;                  // ... and its size: capacity x stride floats
  uint32_t n_cells, capacity, stride, dim;
};
// A random number drawn once per process: a blob is this process's own only when both its pid and this number match.
uint64_t process_nonce() {
  static const uint64_t n = [] {
    std::random_device rd;
    uint64_t v = ((uint64_t)rd() << 32) ^ rd();
    return v ? v : 1;
  }();
  return n;
}
}  // namespace

struct pb_view {
  int device = 0;
  TableDev d{};
  TableDev tier{};  // the owner's shared host tier (pb_view_open_tiered); cells null: none
  uint32_t* seq = nullptr;
  Owned own;  // the IPC mappings of another process's table, and the mapping of its tier's rows
};

namespace {
// The owners' tables of a remote read as this GPU reaches them: views[q] for q != rank, `own` itself for `rank`.
// tiers[q]: owner q's shared host tier (cells null: none)
int remote_views(pb_table* own, pb_view* const* views, uint32_t R, uint32_t rank, RemoteDev& rv, TableDev* tiers) {
  if (R == 0 || R > PB_MAX_RANKS || rank >= R) return fail(PB_ERR_INVALID, "need 1 <= R <= 16 and rank < R");
  if (R > 1 && !views) return fail(PB_ERR_INVALID, "null argument");
  if ((own->tier && !own->tier->shared) || own->host || own->tier_of)
    return fail(PB_ERR_STATE, "a table with a host tier serves one GPU only (no remote reads)");
  if (!own->has_op) return fail(PB_ERR_STATE, "optimizer not registered (OptimizerNotFoundError)");
  std::memset(&rv, 0, sizeof(rv));
  std::memset(tiers, 0, sizeof(TableDev) * PB_MAX_RANKS);
  rv.R = R;
  for (uint32_t q = 0; q < R; ++q) {
    if (q == rank) continue;
    const pb_view* v = views[q];
    if (!v) return fail(PB_ERR_INVALID, "every owner but this rank needs a view (views[q] null)");
    if (v->device != own->device) return fail(PB_ERR_INVALID, "a view was opened on another device than the table's");
    if (v->d.dim != own->cfg.dim) return fail(PB_ERR_INVALID, "a view's table holds another embedding dim");
    rv.t[q] = v->d;
    rv.seq[q] = v->seq;
    tiers[q] = v->tier;
  }
  return PB_OK;
}

// The start of a remote call, after its argument checks: `own` allocated and in its index chain, this rank's entry of
// `rv`, and the staging of `floats` floats.
int begin_remote(pb_table* own, pb_ctx* c, RemoteDev& rv, TableDev* tiers, uint32_t rank, size_t floats, TableCall& call,
                 cudaStream_t st) {
  if (int rc = call.begin(own, st, CALL_INDEX)) return rc;
  if (int rc = ensure_alloc(own)) return rc;
  rv.t[rank] = own->d;
  rv.seq[rank] = own->seq;  // (null unless exported; a live table's training calls need not be ordered with this one)
  if (own->tier) tiers[rank] = own->tier->d;
  return grow_stage(c->own, c->remote_stage, c->remote_stage_floats, floats ? floats : 1, st);
}

// the owners' tiers for launch_remote_lookup: null when no owner has one (the untiered kernels)
const TableDev* any_tier(const TableDev* tiers, uint32_t R) {
  for (uint32_t q = 0; q < R; ++q)
    if (tiers[q].cells) return tiers;
  return nullptr;
}
}  // namespace

uint64_t pb_table_view_bytes(void) { return sizeof(ViewBlob); }

namespace {
// pb_table_export_view (live = false) and pb_table_export_live_view (live = true): one blob layout, one reader
int export_blob(pb_table* t, void* h_blob, bool live) {
  if (!t || !h_blob) return fail(PB_ERR_INVALID, "null argument");
  if (live ? t->exported : t->live)
    return fail(PB_ERR_STATE, live ? "the table was exported frozen (pb_table_export_view): one table, one export mode"
                                   : "the table was exported live (pb_table_export_live_view): one table, one export mode");
  if (t->host || t->tier_of)
    return fail(PB_ERR_STATE, "a host tier cannot be exported: its rows are pinned host memory no peer process can map");
  if (t->tier && !t->tier->shared)
    return fail(PB_ERR_STATE, "a table with a host tier cannot be exported: peers could not read its tier's rows");
  if (t->grow)
    return fail(PB_ERR_STATE, "a growable table cannot be exported: its storage is mapped in chunks no export describes");
  DeviceGuard g(t->device);
  if (int rc = ensure_alloc(t)) return rc;
  if (!t->seq) {
    Owned o;
    uint32_t* seq;
    if (int rc = o.dev(seq, sizeof(uint32_t))) return rc;
    PB_CUDA(cudaMemset(seq, 0, sizeof(uint32_t)));
    PB_CUDA(cudaDeviceSynchronize());
    t->own.adopt(o);
    t->seq = seq;
  }
  ViewBlob b;
  std::memset(&b, 0, sizeof(b));
  b.magic = VIEW_MAGIC;
  b.version = t->tier ? VIEW_VERSION_TIERED : VIEW_VERSION;
  b.pid = (uint64_t)getpid();
  b.nonce = process_nonce();
  b.device = t->device;
  void* p[VA_COUNT] = {t->d.cells, t->d.rows, t->d.counters, t->seq};
  b.ipc = 1;
  for (int i = 0; i < VA_COUNT; ++i) {
    b.ptr[i] = reinterpret_cast<uint64_t>(p[i]);
    if (b.ipc && cudaIpcGetMemHandle(&b.handle[i], p[i]) != cudaSuccess) b.ipc = 0;  // same-process views still work
  }
  if (!b.ipc) {
    cudaGetLastError();  // (the failed handle request is not this call's error)
    std::memset(b.handle, 0, sizeof(b.handle));
  }
  b.dim = t->d.dim;
  b.stride = t->d.stride;
  b.state_floats = t->d.state_floats;
  b.n_cells = t->d.n_cells;
  b.capacity = t->d.capacity;
  std::memcpy(h_blob, &b, sizeof(b));
  if (live) t->live = true;
  else t->exported = true;
  return PB_OK;
}
}  // namespace

int pb_table_export_view(pb_table* t, void* h_blob) { return export_blob(t, h_blob, false); }

int pb_table_export_live_view(pb_table* t, void* h_blob) { return export_blob(t, h_blob, true); }

uint64_t pb_tier_view_bytes(void) { return sizeof(TierBlob); }

int pb_table_export_tier_view(pb_table* t, void* h_blob) {
  if (!t || !h_blob) return fail(PB_ERR_INVALID, "null argument");
  if (t->host || t->tier_of)
    return fail(PB_ERR_STATE, "a host tier cannot be exported: its rows are pinned host memory no peer process can map");
  if (!t->tier) return fail(PB_ERR_STATE, "the table has no host tier");
  if (!t->tier->shared)
    return fail(PB_ERR_STATE, "a table with a host tier cannot be exported: peers could not read its tier's rows");
  if (!t->exported && !t->live)
    return fail(PB_ERR_STATE, "export the table first (pb_table_export_view or pb_table_export_live_view)");
  const pb_table* h = t->tier;
  TierBlob b;
  std::memset(&b, 0, sizeof(b));
  b.magic = TIER_MAGIC;
  b.version = TIER_VERSION;
  b.pid = (uint64_t)getpid();
  b.nonce = process_nonce();
  b.device = t->device;
  b.cells = reinterpret_cast<uint64_t>(h->d.cells);
  b.rows = reinterpret_cast<uint64_t>(h->d.rows);
  DeviceGuard g(t->device);
  b.ipc = cudaIpcGetMemHandle(&b.handle, h->d.cells) == cudaSuccess ? 1u : 0u;
  if (!b.ipc) {
    cudaGetLastError();  // (same-process views still work)
    std::memset(&b.handle, 0, sizeof(b.handle));
  }
  b.fd = h->shared_fd;
  b.bytes = sizeof(float) * (uint64_t)h->d.capacity * h->d.stride;
  b.n_cells = h->d.n_cells;
  b.capacity = h->d.capacity;
  b.stride = h->d.stride;
  b.dim = h->d.dim;
  std::memcpy(h_blob, &b, sizeof(b));
  return PB_OK;
}

namespace {
// pb_view_open (tb = null) and pb_view_open_tiered: the table's view and, with tb, its shared tier
int open_view(int device, const void* h_blob, const void* h_tier_blob, pb_view** out) {
  ViewBlob b;
  std::memcpy(&b, h_blob, sizeof(b));
  if (b.magic != VIEW_MAGIC || (b.version != VIEW_VERSION && b.version != VIEW_VERSION_TIERED))
    return fail(PB_ERR_INVALID, "not a table view (pb_table_export_view)");
  if (!b.n_cells || (b.n_cells & (b.n_cells - 1)) || !b.dim || b.stride < b.dim)
    return fail(PB_ERR_INVALID, "the view's table geometry is malformed");
  TierBlob tb;
  if (h_tier_blob) {
    std::memcpy(&tb, h_tier_blob, sizeof(tb));
    if (tb.magic != TIER_MAGIC || tb.version != TIER_VERSION)
      return fail(PB_ERR_INVALID, "not a tier view (pb_table_export_tier_view)");
    if (!tb.n_cells || (tb.n_cells & (tb.n_cells - 1)) || tb.dim != b.dim || tb.stride != b.stride ||
        tb.bytes != sizeof(float) * (uint64_t)tb.capacity * tb.stride)
      return fail(PB_ERR_INVALID, "the tier view's geometry is malformed or not its table's");
    if (tb.pid != b.pid || tb.nonce != b.nonce || tb.device != b.device)
      return fail(PB_ERR_INVALID, "the tier view comes from another table's export");
    if (b.version != VIEW_VERSION_TIERED)
      return fail(PB_ERR_INVALID, "the table has no shared host tier: open it with pb_view_open");
  } else if (b.version == VIEW_VERSION_TIERED) {
    // (a reader that ignored the tier would read zeros for every tier-held sign)
    return fail(PB_ERR_STATE, "the table has a shared host tier: open it with pb_view_open_tiered and its tier view "
                              "(pb_table_export_tier_view)");
  }
  DeviceGuard g(device);
  std::unique_ptr<pb_view> v(new pb_view());
  v->device = device;
  void* p[VA_COUNT];
  void* tp[2] = {nullptr, nullptr};  // the tier's cells and rows
  if (b.pid == (uint64_t)getpid() && b.nonce == process_nonce()) {  // CUDA IPC cannot open a handle in its own process: the pointers are valid here
    for (int i = 0; i < VA_COUNT; ++i) p[i] = reinterpret_cast<void*>(b.ptr[i]);
    if (h_tier_blob) {
      tp[0] = reinterpret_cast<void*>(tb.cells);
      tp[1] = reinterpret_cast<void*>(tb.rows);
    }
    if (b.device != device) {
      const cudaError_t e = cudaDeviceEnablePeerAccess(b.device, 0);
      if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled)
        return fail(PB_ERR_CUDA, std::string("cudaDeviceEnablePeerAccess: ") + cudaGetErrorString(e));
      cudaGetLastError();
    }
  } else {
    if (!b.ipc || (h_tier_blob && !tb.ipc))
      return fail(PB_ERR_STATE, "the exporting process could not make CUDA IPC handles for this table");
    for (int i = 0; i < VA_COUNT; ++i)
      if (int rc = v->own.ipc(p[i], b.handle[i])) return rc;
    if (h_tier_blob) {
      if (int rc = v->own.ipc(tp[0], tb.handle)) return rc;
      // the tier's rows: the exporter's memfd, reached through /proc (one user, one PID namespace, a dumpable owner)
      // read-only where the device can register read-only host memory: a reader never writes the owner's rows
      int ro = 0;
      if (cudaDeviceGetAttribute(&ro, cudaDevAttrHostRegisterReadOnlySupported, device) != cudaSuccess) {
        cudaGetLastError();
        ro = 0;
      }
      const std::string path = "/proc/" + std::to_string(tb.pid) + "/fd/" + std::to_string(tb.fd);
      const int fd = open(path.c_str(), (ro ? O_RDONLY : O_RDWR) | O_CLOEXEC);
      if (fd < 0)
        return fail(PB_ERR_STATE, "cannot open the exporting process's shared tier (" + path + ": " + strerror(errno) +
                                      "): its ranks must run as one user in one PID namespace, and it must be dumpable");
      float *h = nullptr, *dr = nullptr;
      int kept = -1;
      if (int rc = v->own.shared(h, dr, tb.bytes, fd, kept, ro != 0)) return rc;
      tp[1] = dr;
    }
  }
  TableDev& d = v->d;
  d.cells = static_cast<Cell*>(p[VA_CELLS]);
  d.rows = static_cast<float*>(p[VA_ROWS]);
  d.counters = static_cast<uint32_t*>(p[VA_COUNTERS]);
  d.n_cells = b.n_cells;
  d.cell_mask = b.n_cells - 1;
  d.bucket_mask = b.n_cells / BUCKET - 1;
  d.capacity = b.capacity;
  d.mapped = b.capacity;
  d.dim = b.dim;
  d.stride = b.stride;
  d.state_floats = b.state_floats;
  if (h_tier_blob) {  // (a find touches only cells and rows)
    TableDev& h = v->tier;
    h.cells = static_cast<Cell*>(tp[0]);
    h.rows = static_cast<float*>(tp[1]);
    h.n_cells = tb.n_cells;
    h.cell_mask = tb.n_cells - 1;
    h.bucket_mask = tb.n_cells / BUCKET - 1;
    h.capacity = tb.capacity;
    h.mapped = tb.capacity;
    h.dim = tb.dim;
    h.stride = tb.stride;
    h.state_floats = b.state_floats;
  }
  v->seq = static_cast<uint32_t*>(p[VA_SEQ]);
  *out = v.release();
  return PB_OK;
}
}  // namespace

int pb_view_open(int device, const void* h_blob, pb_view** out) {
  if (!h_blob || !out) return fail(PB_ERR_INVALID, "null argument");
  return open_view(device, h_blob, nullptr, out);
}

int pb_view_open_tiered(int device, const void* h_blob, const void* h_tier_blob, pb_view** out) {
  if (!h_blob || !h_tier_blob || !out) return fail(PB_ERR_INVALID, "null argument");
  return open_view(device, h_blob, h_tier_blob, out);
}

int pb_view_close(pb_view* v) {
  if (!v) return PB_OK;
  DeviceGuard g(v->device);
  cudaDeviceSynchronize();  // (remote reads through it may still run)
  delete v;
  return PB_OK;
}

int pb_forward_remote(pb_table* own, pb_view* const* views, uint32_t R, uint32_t rank, pb_ctx* c, const uint64_t* d_ids,
                      uint32_t n_occ, const uint32_t* d_row_off, const uint32_t* h_slot_occ_off, uint32_t batch,
                      void* d_out_f16, void* stream) {
  int rc = check_forward(own, c, d_ids, n_occ, d_row_off, h_slot_occ_off, batch, d_out_f16);
  RemoteDev rv;
  TableDev tiers[PB_MAX_RANKS];
  if (rc || (rc = remote_views(own, views, R, rank, rv, tiers))) return rc;
  const uint64_t n_out = (uint64_t)c->slots.n_slots * batch;
  const bool row_f32 = d_row_off != nullptr;  // ragged layouts pool f32 rows, as on an exchange of f32 rows
  DeviceGuard g(own->device);
  cudaStream_t st = (cudaStream_t)stream;
  TableCall call;
  const size_t elems = (size_t)n_occ * own->cfg.dim;  // at most one row per id occurrence
  if ((rc = begin_remote(own, c, rv, tiers, rank, row_f32 ? elems : (elems + 1) / 2, call, st))) return rc;
  SlotsDev sl;
  if ((rc = make_slots(c->slots, h_slot_occ_off, sl))) return rc;
  if ((rc = begin_forward(own, c, sl, d_ids, n_occ, 0, st))) return rc;  // the dedup (an inference request)
  launch_remote_lookup(false, row_f32, rv, any_tier(tiers, R), c->b, c->raw, n_occ, c->remote_stage, own->d.dim,
                       own->d.counters + CTR_ERR, st);
  launch_expand_items(own->d, sl, c->b, c->remote_stage, row_f32, d_row_off, (uint32_t)n_out, batch, false, d_out_f16, st);
  if ((rc = end_forward(own, c, d_row_off, h_slot_occ_off, n_occ, batch, 0, st))) return rc;
  PB_CUDA(cudaGetLastError());
  return PB_OK;
}

int pb_forward_raw_remote(pb_table* own, pb_view* const* views, uint32_t R, uint32_t rank, pb_ctx* c,
                          const uint64_t* d_ids, uint32_t n_occ, const uint32_t* d_row_off, uint32_t batch,
                          uint32_t sample_fixed_size, void* d_table_f16, int64_t* d_index, int64_t* d_non_empty,
                          uint32_t* d_sample_id_num, uint32_t* d_counts, void* stream) {
  int rc = check_raw_forward(own, c, d_ids, n_occ, d_row_off, batch, sample_fixed_size, d_table_f16, d_index, d_non_empty,
                             d_sample_id_num, d_counts);
  RemoteDev rv;
  TableDev tiers[PB_MAX_RANKS];
  if (rc || (rc = remote_views(own, views, R, rank, rv, tiers))) return rc;
  DeviceGuard g(own->device);
  cudaStream_t st = (cudaStream_t)stream;
  TableCall call;
  if ((rc = begin_remote(own, c, rv, tiers, rank, (size_t)n_occ * own->cfg.dim, call, st))) return rc;
  if ((rc = ensure_raw(c))) return rc;
  SlotsDev sl;
  if ((rc = raw_slots(c, n_occ, sl))) return rc;
  c->raw_pending.drop();  // the numbering below replaces the pending batch's
  c->prepared = PREP_NONE;
  if (d_row_off && (rc = copy_row_off(c, d_row_off, batch, st))) return rc;
  launch_raw_number(sl, d_ids, n_occ, d_row_off ? c->row_off : nullptr, d_row_off ? c->occ_outrow : nullptr, batch,
                    sample_fixed_size, nullptr, c->raw, (long long*)d_index, (long long*)d_non_empty, d_sample_id_num, st);
  PB_CUDA(cudaMemcpyAsync(d_counts, c->raw.counts, 8, cudaMemcpyDeviceToDevice, st));
  launch_remote_lookup(true, true, rv, any_tier(tiers, R), c->b, c->raw, n_occ, c->remote_stage, own->d.dim,
                       own->d.counters + CTR_ERR, st);
  launch_raw_fill(c->raw, n_occ, own->d.dim, c->remote_stage, d_table_f16, st);  // row u + 1 = f16(row), rounded once
  PB_CUDA(cudaGetLastError());
  return PB_OK;
}

}  // extern "C"

// debugging aid (not in include/persia_b200.h): device buffer of 4 u64 per hot item that k_reduce_hot stamps
namespace pb { void set_hot_trace(unsigned long long* p); }
extern "C" void pb_debug_hot_trace(void* d_buf) { pb::set_hot_trace(reinterpret_cast<unsigned long long*>(d_buf)); }
// measuring aid (not in include/persia_b200.h): pb_tier_stage's grid (scripts/host_tier_bench.py --stage-blocks)
extern "C" void pb_debug_stage_blocks(uint32_t blocks) { g_stage_blocks = blocks ? blocks : PB_NUM_SMS; }
// measuring aid (not in include/persia_b200.h): an exported table's write-sequence word, read after the device is idle
// (scripts/live_remote_bench.py: how many owner write windows a reader's requests overlapped)
extern "C" int pb_debug_table_seq(pb_table* t, uint32_t* h_out) {
  if (!t || !h_out) return fail(PB_ERR_INVALID, "null argument");
  if (!t->seq) return fail(PB_ERR_STATE, "the table was not exported");
  DeviceGuard g(t->device);
  PB_CUDA(cudaMemcpy(h_out, t->seq, sizeof(uint32_t), cudaMemcpyDeviceToHost));
  return PB_OK;
}
// testing aids (not in include/persia_b200.h): the resources every live object holds, [count, device + host bytes];
// and a refusal: the (n+1)-th acquisition from now fails as if CUDA had refused it, before any CUDA call (-1: none)
extern "C" int pb_debug_owned(uint64_t h_out[2]) {
  if (!h_out) return fail(PB_ERR_INVALID, "null argument");
  h_out[0] = g_owned_count.load();
  h_out[1] = g_owned_bytes.load();
  return PB_OK;
}
extern "C" void pb_debug_refuse_after(int64_t n) { g_refuse_after = n < 0 ? -1 : n; }
