// pb_api_view.cu — the C ABI's reads of other ranks' tables: export blobs, views of an owner's table (and its shared
// host tier) opened in another process, and the remote forwards that read the owners' shards in place over NVLink.
#include <cerrno>
#include <cstring>
#include <memory>
#include <random>
#include <string>

#include <unistd.h>

#include "pb_api.cuh"

extern "C" {

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
  if ((rc = number_raw(c, sl, d_ids, n_occ, d_row_off, batch, sample_fixed_size, d_index, d_non_empty, d_sample_id_num,
                       d_counts, st)))
    return rc;
  launch_remote_lookup(true, true, rv, any_tier(tiers, R), c->b, c->raw, n_occ, c->remote_stage, own->d.dim,
                       own->d.counters + CTR_ERR, st);
  launch_raw_fill(c->raw, n_occ, own->d.dim, c->remote_stage, d_table_f16, st);  // row u + 1 = f16(row), rounded once
  PB_CUDA(cudaGetLastError());
  return PB_OK;
}

}  // extern "C"
