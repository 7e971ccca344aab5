// pb_api.cu — the C ABI of libpersia_b200.so (include/persia_b200.h): object lifetime, argument checks,
// kernel sequencing.  No torch types, no allocation on the hot path after the first call of a given size.
// This file: tables (lifetime, configuration, storage and growth, eviction, host tiers, incremental sets, statistics),
// the ordering of calls on a table, the id-level calls, the hash utilities and the debugging aids.  Checkpoints are in
// pb_api_ckpt.cu, batch contexts and their forwards and backwards in pb_api_batch.cu, the sharded calls in
// pb_api_shard.cu, table views and remote reads in pb_api_view.cu; pb_api.cuh holds what they share.
#include <algorithm>
#include <atomic>
#include <cstring>
#include <memory>
#include <string>

#include "pb_api.cuh"

namespace pb {

uint32_t next_pow2(uint64_t v) {
  uint64_t p = 1;
  while (p < v) p <<= 1;
  return (uint32_t)p;
}

// rand 0.8 UniformFloat::new: shrink the scale until the largest draw stays below `hi`
static float uniform_scale(float lo, float hi) {
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

// Grid of pb_tier_stage's kernels: they run beside the backward and the dense step of the batch before, so they take a
// fixed share of the GPU rather than the usual grids (8 blocks per SM for the index scans).  One block per SM: measured
// on an H100 with scripts/host_tier_bench.py (DESIGN.md §4 "Staging"), a step with the stage on 8, 16, 32, 64 and 132
// blocks took 6.49, 3.97, 2.93, 2.58 and 2.43 ms beside a 1.06 ms dense stand-in: the stage's eviction check moves
// ~45k entries out per step, and fewer blocks leave too few copies in flight to keep PCIe busy, so the stage outlasts
// the dense step and the backward and delays the next forward.
uint32_t g_stage_blocks = PB_NUM_SMS;

// ---- growable storage (pb_table_set_growth) --------------------------------------------------------------------------
// bytes per row of each row-indexed region
static size_t region_row_bytes(const pb_table* t, int r) {
  switch (r) {
    case pb_table::G_ROWS: return sizeof(float) * (size_t)t->d.stride;
    case pb_table::G_RKEYS: return sizeof(uint64_t);
    default: return sizeof(uint32_t);  // row_tick, free_rows, rebuild_rows
  }
}

// The chunks that back `rows` rows and `cells` index cells (+ N_SPECIAL), acquired into `o`; `mapped[r]` receives
// each region's new extent, and `rec` the new chunks of the rows and the cells (exportable growth: what readers are
// sent).  Nothing is enqueued.
static int map_growth(pb_table* t, uint64_t rows, uint64_t cells, Owned& o, size_t mapped[pb_table::G_COUNT],
                      std::vector<pb_table::Chunk>& rec) {
  for (int r = 0; r < pb_table::G_COUNT; ++r) {
    const size_t want = r == pb_table::G_CELLS ? sizeof(Cell) * ((size_t)cells + N_SPECIAL) : region_row_bytes(t, r) * rows;
    const size_t to = (want + t->gran - 1) / t->gran * t->gran;
    pb_table::Region& g = t->region[r];
    mapped[r] = g.mapped;
    if (to <= g.mapped) continue;
    unsigned long long h = 0;
    if (int rc = o.chunk(g.base + g.mapped, to - g.mapped, t->device, t->grow_share, &h)) return rc;
    if (t->grow_share && (r == pb_table::G_ROWS || r == pb_table::G_CELLS)) {
      int fd = -1;
      if (CUresult e = vmm().export_fd(&fd, (CUmemGenericAllocationHandle)h, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0))
        return fail(PB_ERR_CUDA, "cuMemExportToShareableHandle: CUresult " + std::to_string((int)e));
      rec.push_back({(uint32_t)r, g.mapped, to - g.mapped, fd});
    }
    mapped[r] = to;
  }
  return PB_OK;
}

// largest extent of each region: `capacity` rows, the index at max_cells
static size_t region_reserved(const pb_table* t, int r) {
  if (r == pb_table::G_CELLS) return sizeof(Cell) * ((size_t)t->max_cells + N_SPECIAL);
  return region_row_bytes(t, r) * t->d.capacity;
}

// A growable table's first allocation: every region reserved at its largest extent (rounded to the granularity), the
// first chunk of rows and the index they need backed, counters, the sweep's workspace, the read-back word and the stream
// of captured growth; the cells filled, row_tick zeroed.  The index starts at the size an eager table of `mapped`
// rows would have.
static int acquire_growable(pb_table* t, Owned& o) {
  TableDev& d = t->d;
  t->max_cells = d.n_cells;
  if (!(t->gran = vmm_granularity(t->device))) return fail(PB_ERR_CUDA, "no virtual memory management on this device");
  int rc;
  for (int r = 0; r < pb_table::G_COUNT; ++r) {
    const size_t span = (region_reserved(t, r) + t->gran - 1) / t->gran * t->gran;
    t->region[r] = pb_table::Region{};
    if ((rc = o.reserve(t->region[r].base, span))) return rc;
    t->region[r].span = span;
  }
  uint64_t rows = t->gran / region_row_bytes(t, pb_table::G_ROWS);
  rows = rows < 1 ? 1 : rows > d.capacity ? d.capacity : rows;
  uint64_t want = rows + rows / 2;
  const uint32_t cells = next_pow2(want < 1024 ? 1024 : want);
  size_t mapped[pb_table::G_COUNT];
  std::vector<pb_table::Chunk> rec;
  if ((rc = map_growth(t, rows, cells, o, mapped, rec)) || (rc = o.dev(d.counters, sizeof(uint32_t) * CTR_COUNT)) ||
      (rc = o.dev(t->evict_ws, sizeof(uint32_t) * EVICT_WS_WORDS)) ||
      (rc = o.mapped(t->rb_host, t->rb_dev, 3 * sizeof(uint32_t))) || (rc = o.stream(t->grow_st))) {
    for (const pb_table::Chunk& c : rec) close(c.fd);
    return rc;
  }
  t->readers.chunks = rec;
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
static int acquire_storage(pb_table* t, Owned& o) {
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

static int ensure_scratch(pb_table* t, uint32_t n) {
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
static int acquire_evict_ws(pb_table* t, Owned& o, uint32_t*& free_rows) {
  const size_t cap = t->d.capacity;
  int rc;
  if ((rc = o.dev(t->evict_ws, sizeof(uint32_t) * EVICT_WS_WORDS)) || (rc = o.dev(t->rebuild_keys, sizeof(uint64_t) * cap)) ||
      (rc = o.dev(t->rebuild_rows, sizeof(uint32_t) * cap)))
    return rc;
  return o.dev(free_rows, sizeof(uint32_t) * cap);
}

// allocated by the first sweep
static int ensure_evict_ws(pb_table* t) {
  if (t->d.free_rows) return PB_OK;
  Owned o;
  if (int rc = acquire_evict_ws(t, o, t->d.free_rows)) return rc;
  t->own.adopt(o);
  return PB_OK;
}


// The eviction check: release the least recently used rows when free storage runs low, and rebuild the index when its
// EMPTY cells run short.  blocks: grid of its scans (0 = the usual; pb_tier_stage's is small).
int evict_check(pb_table* t, cudaStream_t st, uint32_t blocks) {
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

static cudaError_t capture_id(cudaStream_t st, unsigned long long& id) {
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


// Before a call on a growable table launches anything that can admit up to `n` signs (a training forward or lookup,
// pb_set_rows, an owner's training SERVE), in the index chain: back every row the enqueued calls and this one can hand
// out, and grow the index so that the cells they can use stay within 2/3 of it.  Rows grow by at least 1/8 of what is
// mapped (a logarithmic number of mappings), the index by doubling.  A chunk that cannot be had fails the call with
// PB_ERR_CUDA before any kernel or copy is enqueued (the call's TableCall has made its stream wait for the table's
// earlier calls and records its mark: ordering only); the table stays as it was.  Under stream capture the whole capacity is
// backed (a replay never passes here), the work enqueued outside the graph and waited for.  Any other table: nothing.
int grow_for(pb_table* t, uint64_t n, cudaStream_t st) {
  if (!t->grow) return PB_OK;
  if (t->grow_share) send_chunks(t);  // (sends an earlier call had to keep)
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
    std::vector<pb_table::Chunk> rec;
    if (int rc = map_growth(t, rows, cells, o, mapped, rec)) {
      for (const pb_table::Chunk& c : rec) close(c.fd);
      return rc;
    }
    t->own.adopt(o);
    for (int r = 0; r < pb_table::G_COUNT; ++r) t->region[r].mapped = mapped[r];
    // readers in other processes get the new chunks before any kernel that can use them is enqueued
    if (!rec.empty()) {
      t->readers.chunks.insert(t->readers.chunks.end(), rec.begin(), rec.end());
      send_chunks(t);
    }
    if (rows > d.mapped)
      PB_CUDA(cudaMemsetAsync(d.row_tick + d.mapped, 0, sizeof(uint32_t) * (size_t)(rows - d.mapped), ws));
    d.mapped = (uint32_t)rows;
    if (cells > d.n_cells) {
      TableDev to = d;
      to.n_cells = (uint32_t)cells;
      to.cell_mask = cells - 1;
      to.bucket_mask = (uint32_t)(cells / BUCKET - 1);
      // an exported table (exportable growth: live or frozen) holds its write-sequence word odd while every cell
      // moves, and publishes the new cell count to its readers before it is even again (pb_remote.cu)
      if (t->seq) launch_seq_bump(t->seq, true, ws);
      launch_grow_index(d, to, t->evict_ws, t->rebuild_keys, t->rebuild_rows, ws);
      if (t->seq) launch_seq_bump(t->seq, false, ws, to.n_cells);
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
static int read_counters(pb_table* t, const W* src, W* dst, size_t n, cudaStream_t st) {
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

static SlotsDev no_slots() {
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

// one beta-power step of Adam's pair k (one request of one feature group, optim.rs:155-197); returns the pair
const float* advance_adam_pair(pb_table* t, int k, cudaStream_t st) {
  AdamKeys keys{};
  keys.idx[0] = (uint8_t)k;
  keys.n = 1;
  launch_adam_advance(t->adam_dev, keys, t->op.b1, t->op.b2, st);
  return t->adam_dev + 2 * k;
}

}  // namespace pb

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
  if (on < 0 || on > 2) return fail(PB_ERR_INVALID, "growth mode must be 0, 1 or 2");
  if (t->host) return fail(PB_ERR_STATE, "a host table's storage cannot grow");
  if (t->allocated) return fail(PB_ERR_STATE, "growth must be chosen before the table's first allocation");
  if (on == 2 && !vmm_fd_supported(t->device))
    return fail(PB_ERR_STATE, "exportable growth needs device memory that can be shared as POSIX file descriptors, "
                              "and this device or driver does not report CU_DEVICE_ATTRIBUTE_HANDLE_TYPE_POSIX_FILE_"
                              "DESCRIPTOR_SUPPORTED (or lacks cuMemExportToShareableHandle)");
  t->grow = on != 0;
  t->grow_share = on == 2;
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
// testing aid (not in include/persia_b200.h): an exportable growable table keeps every chunk it would send its readers
// while `on` is set; clearing it sends them.  So a reader meets rows or cells it has not mapped yet, deterministically
extern "C" int pb_debug_defer_sends(pb_table* t, int on) {
  if (!t) return fail(PB_ERR_INVALID, "null argument");
  t->readers.defer = on != 0;
  if (!on) send_chunks(t);
  return PB_OK;
}
