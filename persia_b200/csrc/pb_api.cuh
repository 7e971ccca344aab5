// pb_api.cuh — what the C ABI's files share (private to pb_api.cu, pb_api_ckpt.cu, pb_api_batch.cu,
// pb_api_shard.cu and pb_api_view.cu): the table and context objects, the ordering of calls on a table, and the helpers
// more than one of those files calls.  A helper only one of them calls stays in that file.
#pragma once
#include <cstdint>
#include <vector>

#include "pb_kernels.cuh"
#include "pb_own.cuh"

using namespace pb;  // every ABI file uses the kernels' and pb_own.cuh's names unqualified

namespace pb {

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

// an event recorded on a caller's stream, and the stream capture it was recorded into (0 = none: a real record)
struct Mark {
  cudaEvent_t ev = nullptr;
  unsigned long long capture = 0;
  bool set = false;
};

uint32_t next_pow2(uint64_t v);

// grid of pb_tier_stage's and pb_tier_stage_sharded's kernels (pb_api.cu)
extern uint32_t g_stage_blocks;

}  // namespace pb

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
    size_t span = 0;  // reserved
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
  // exportable growth (pb_table_set_growth(t, 2)): every chunk is created exportable, and the chunks of the two regions
  // a reader touches (rows, cells) are listed in mapping order.  Each reader registered in another process
  // (pb_table_add_reader) is a connected socket and the number of listed chunks it has been sent (send_chunks)
  // (each chunk's descriptor is exported once, when it is mapped, and kept open for the table's life)
  bool grow_share = false;
  struct Chunk {
    uint32_t region;  // G_ROWS or G_CELLS
    size_t off, bytes;
    int fd;
  };
  struct Reader {
    int sock;
    size_t sent;
  };
  struct Readers {
    std::vector<Chunk> chunks;
    std::vector<Reader> r;
    bool defer = false;  // pb_debug_defer_sends: nothing is sent until it is cleared
    ~Readers();
  } readers;
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
  // ... and, when an owner is an exportable growable table in another process, the count of items its read found in
  // rows or cells this process has not mapped yet, and its pinned copy
  uint32_t* stale = nullptr;
  uint32_t* stale_host = nullptr;
  Owned own;  // every CUDA resource above
};
enum { PREP_NONE = 0, PREP_SUM = 1, PREP_RAW = 2 };

namespace pb {

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

// `m` recorded on `st`, and `st` made to wait for the work behind `m` (pb_api.cu, "event marks")
int record(Mark& m, cudaStream_t st);
int wait_for(const Mark& m, cudaStream_t st);

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

// ---- pb_api.cu ---------------------------------------------------------------------------------------------------
int ensure_alloc(pb_table* t);
int evict_check(pb_table* t, cudaStream_t st, uint32_t blocks = 0);
int maybe_evict(pb_table* t, cudaStream_t st);
int grow_for(pb_table* t, uint64_t n, cudaStream_t st);

// ---- pb_api_view.cu ----------------------------------------------------------------------------------------------
// an exportable growable table: every listed chunk its registered readers have not been sent yet, sent without
// blocking (a send that would block is kept for the next call)
void send_chunks(pb_table* t);
void restore_ids(pb_table* t, bool prefix, const SlotsDev& sl, const uint64_t* ids, uint32_t n, cudaStream_t st);
int writable(const pb_table* t);
int ready_for_training(pb_table* t);
int adam_index(pb_table* t, uint64_t prefix);
int make_slots(const pb_slots_cfg& cfg, const uint32_t* h_occ_off, SlotsDev& s);
int prefix_slots(const uint32_t* h_occ_off, const uint64_t* h_prefix, uint32_t n_slots, uint32_t prefix_bit,
                 SlotsDev& s);
int raw_slots(const pb_ctx* c, uint32_t n, SlotsDev& s);
int check_slot_offsets(const uint32_t* h_occ_off, uint32_t n_slots, uint32_t n);
bool misaligned(const void* p);
const float* advance_adam_pair(pb_table* t, int k, cudaStream_t st);

// ---- pb_api_batch.cu ---------------------------------------------------------------------------------------------
int loss_scale(float sc, uint8_t& on, float& inv);
int make_grads(const void* const* h_grads, const float* h_scale, uint32_t n_slots, GradsDev& gr);
int check_forward(pb_table* t, pb_ctx* c, const uint64_t* d_ids, uint32_t n_occ, const uint32_t* d_row_off,
                  const uint32_t* h_slot_occ_off, uint32_t batch, void* d_out_f16);
int check_raw_forward(pb_table* t, pb_ctx* c, const uint64_t* d_ids, uint32_t n_occ, const uint32_t* d_row_off,
                      uint32_t batch, uint32_t sample_fixed_size, void* d_table_f16, int64_t* d_index,
                      int64_t* d_non_empty, uint32_t* d_sample_id_num, uint32_t* d_counts);
int check_backward(pb_table* t, pb_ctx* c, const void* const* h_grads);
int check_raw_backward(pb_table* t, pb_ctx* c, const void* d_grad);
int begin_forward(pb_table* t, pb_ctx* c, const SlotsDev& sl, const uint64_t* d_ids, uint32_t n_occ, int training,
                  cudaStream_t st, bool prepared = false);
void prepare_batch(const pb_table* t, pb_ctx* c, const SlotsDev& sl, const uint64_t* d_ids, uint32_t n_occ,
                   uint32_t batch, cudaStream_t st);
int end_forward(pb_table* t, pb_ctx* c, const uint32_t* d_row_off, const uint32_t* h_slot_occ_off, uint32_t n_occ,
                uint32_t batch, int training, cudaStream_t st);
void hold_raw_batch(pb_table* t, pb_ctx* c, uint32_t n_occ, uint32_t batch);
ReduceArgs reduce_args(const pb_ctx* c);
int fork_side(pb_ctx* c, cudaStream_t st);
int fork_after_nan(pb_ctx* c, cudaStream_t st);
int join_sides(pb_ctx* c, cudaStream_t st);
int grow_stage(Owned& own, float*& buf, size_t& floats, size_t need, cudaStream_t st);
int ensure_raw(pb_ctx* c);
int number_raw(pb_ctx* c, const SlotsDev& sl, const uint64_t* d_ids, uint32_t n_occ, const uint32_t* d_row_off,
               uint32_t batch, uint32_t sample_fixed_size, int64_t* d_index, int64_t* d_non_empty,
               uint32_t* d_sample_id_num, uint32_t* d_counts, cudaStream_t st);

}  // namespace pb
