// pb_api_view.cu — the C ABI's reads of other ranks' tables: export blobs, views of an owner's table (and its shared
// host tier) opened in another process, and the remote forwards that read the owners' shards in place over NVLink.
#include <atomic>
#include <cerrno>
#include <chrono>
#include <cstring>
#include <memory>
#include <random>
#include <string>
#include <thread>

#include <sys/socket.h>
#include <sys/un.h>
#include <unistd.h>

#include "pb_api.cuh"

extern "C" {

// ---- inference on R GPUs one rank at a time: views of the owners' tables --------------------------------------------
namespace {
// The bytes pb_table_export_view writes: what a peer needs to read the table in place.
constexpr uint32_t VIEW_MAGIC = 0x57564250u;  // "PBVW"
constexpr uint32_t VIEW_VERSION = 1;
constexpr uint32_t VIEW_VERSION_TIERED = 2;  // the same layout, of a table with a shared tier: opened with its tier blob
// The same layout, of a table with exportable growth (pb_table_set_growth(t, 2)).  Its cells and rows are VMM
// reservations backed chunk by chunk, which no IPC handle describes: their handle slots hold each reservation's span
// (GrowSpan) instead, `pad` holds the largest index's cell count, and the reader receives the chunks themselves over
// a socket (pb_table_add_reader).  The write-sequence word's allocation holds a second word: the index's cell count.
constexpr uint32_t VIEW_VERSION_GROW = 3;
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
struct GrowSpan {  // version 3, in handle[VA_CELLS] and handle[VA_ROWS]
  uint64_t span;   // bytes of address space the owner reserved for the region
  uint64_t gran;   // every chunk's offset and size are multiples of it
};
static_assert(sizeof(GrowSpan) <= sizeof(cudaIpcMemHandle_t), "a span fits a handle's slot");
// One message of chunks (exportable growth): up to CHUNKS_PER_MSG entries, their descriptors in SCM_RIGHTS, in order
constexpr uint32_t CHUNKS_PER_MSG = 32;
struct ChunkMsg {
  uint32_t n, pad;
  struct {
    uint32_t region, pad;  // 0: rows, 1: cells
    uint64_t off, bytes;
  } e[CHUNKS_PER_MSG];
};
std::atomic<uint64_t> g_stale_retries{0};  // pb_debug_stale_retries
// how long a remote read waits for an owner's chunk that its stale items need, before it fails
#ifndef PB_STALE_WAIT_MS
#define PB_STALE_WAIT_MS 20000
#endif
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
  // exportable growth (version 3): the owner's published cell count (seq + 1), and what this process has mapped of
  // the owner's rows and cell slots (~0: all of them, a view in the owner's process).  Another process's view reserves
  // the owner's spans (base[], span[]), listens on an abstract socket (`addr`, pb_view_address) and maps each chunk
  // the owner sends over the connection it accepts there (drain)
  bool grow = false;
  const uint32_t* geo = nullptr;
  uint32_t mapped_rows = 0, mapped_cells = 0;
  char* base[2] = {nullptr, nullptr};  // rows, cells
  size_t span[2] = {0, 0}, mapped[2] = {0, 0};
  int listen_fd = -1, conn_fd = -1;
  std::string addr;
  Owned own;  // the IPC mappings of another process's table, and the mapping of its tier's rows (or its chunks)
  ~pb_view() {
    if (conn_fd >= 0) close(conn_fd);
    if (listen_fd >= 0) close(listen_fd);
  }
};

pb_table::Readers::~Readers() {
  for (const pb_table::Reader& x : r) close(x.sock);
  for (const pb_table::Chunk& c : chunks) close(c.fd);
}

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

// Every chunk that has arrived on a view of another process's growable table, imported and mapped read-only at its
// offset: nothing is waited for.  A chunk that does not follow its region's last one, or runs past its span, is a
// broken stream: PB_ERR_STATE.
int drain(pb_view* v) {
  if (v->listen_fd < 0) return PB_OK;
  if (v->conn_fd < 0) {
    v->conn_fd = accept4(v->listen_fd, nullptr, nullptr, SOCK_NONBLOCK | SOCK_CLOEXEC);
    if (v->conn_fd < 0) {
      if (errno == EAGAIN || errno == EWOULDBLOCK) return PB_OK;  // (the owner has not registered this reader yet)
      return fail(PB_ERR_STATE, std::string("accept4 on a view's socket: ") + strerror(errno));
    }
  }
  int rc = PB_OK;
  for (;;) {
    ChunkMsg m;
    char ctl[CMSG_SPACE(sizeof(int) * CHUNKS_PER_MSG)];
    iovec io{&m, sizeof(m)};
    msghdr h{};
    h.msg_iov = &io;
    h.msg_iovlen = 1;
    h.msg_control = ctl;
    h.msg_controllen = sizeof(ctl);
    const ssize_t got = recvmsg(v->conn_fd, &h, MSG_DONTWAIT | MSG_CMSG_CLOEXEC);
    if (got < 0 && (errno == EAGAIN || errno == EWOULDBLOCK)) break;
    if (got < 0) return fail(PB_ERR_STATE, std::string("recvmsg on a view's socket: ") + strerror(errno));
    if (got == 0) break;  // (the owner closed: nothing more will come)
    int fds[CHUNKS_PER_MSG];
    uint32_t n_fd = 0;
    for (cmsghdr* c = CMSG_FIRSTHDR(&h); c; c = CMSG_NXTHDR(&h, c))
      if (c->cmsg_level == SOL_SOCKET && c->cmsg_type == SCM_RIGHTS)
        for (size_t i = 0; i < (c->cmsg_len - CMSG_LEN(0)) / sizeof(int) && n_fd < CHUNKS_PER_MSG; ++i)
          std::memcpy(&fds[n_fd++], CMSG_DATA(c) + i * sizeof(int), sizeof(int));
    const bool whole = (size_t)got == sizeof(m) && !(h.msg_flags & (MSG_CTRUNC | MSG_TRUNC)) && m.n == n_fd &&
                       m.n <= CHUNKS_PER_MSG;
    for (uint32_t i = 0; i < n_fd; ++i) {  // every descriptor is consumed: imported, or closed
      const uint32_t g = whole ? m.e[i].region : 2u;
      if (rc || g > 1 || m.e[i].off != v->mapped[g] || m.e[i].bytes > v->span[g] - m.e[i].off) {
        close(fds[i]);
        if (!rc) rc = fail(PB_ERR_STATE, "a view's chunk stream is broken (a chunk out of order, or a malformed message)");
        continue;
      }
      if ((rc = v->own.import_chunk(v->base[g] + m.e[i].off, m.e[i].bytes, fds[i], v->device))) continue;
      v->mapped[g] += m.e[i].bytes;
    }
    if (rc) return rc;
    if (!whole) return fail(PB_ERR_STATE, "a view's chunk stream is broken (a chunk out of order, or a malformed message)");
  }
  const uint64_t rows = v->mapped[0] / (sizeof(float) * (uint64_t)v->d.stride);
  v->mapped_rows = (uint32_t)(rows < v->d.capacity ? rows : v->d.capacity);
  v->mapped_cells = (uint32_t)(v->mapped[1] / sizeof(Cell));
  return PB_OK;
}

// The owners' growth for launch_remote_lookup (`any` false: no owner grows, and the kernels without the stale check
// run).  `check` true: some owner is another process's, whose items can be stale (a view in the owner's process maps
// everything the owner does).
void grow_views(pb_view* const* views, uint32_t R, uint32_t rank, RemoteGrowDev& g, bool& any, bool& check) {
  std::memset(&g, 0, sizeof(g));
  any = check = false;
  for (uint32_t q = 0; q < R; ++q) {
    g.rows[q] = g.cells[q] = ~0u;  // (an owner without geo: its table as the call has it, never stale)
    const pb_view* v = q == rank ? nullptr : views[q];
    if (!v || !v->grow) continue;
    g.geo[q] = v->geo;
    g.rows[q] = v->mapped_rows;
    g.cells[q] = v->mapped_cells;
    any = true;
    check = check || v->listen_fd >= 0;
  }
}

// The remote read of a call: launch_remote_lookup, and where an owner in another process grows, the stale items read
// again until none is left.  That needs the count of stale items on the host: one copy and a synchronisation of `st`
// per call.  Each round first imports every chunk that has arrived; a round that finds nothing new waits (polling the
// views' sockets) up to PB_STALE_WAIT_MS for one, then fails with PB_ERR_STATE (the staging is then not read).
int remote_lookup(bool raw, bool row_f32, const RemoteDev& rv, const TableDev* tiers, pb_view* const* views, uint32_t R,
                  uint32_t rank, pb_ctx* c, uint32_t n_occ, uint32_t dim, uint32_t* err, cudaStream_t st) {
  RemoteGrowDev g;
  bool any = false, check = false;
  for (uint32_t q = 0; q < R; ++q)
    if (q != rank && views[q] && views[q]->grow)
      if (int rc = drain(views[q])) return rc;
  grow_views(views, R, rank, g, any, check);
  if (any && tiers)
    return fail(PB_ERR_STATE, "owners with exportable growth and owners with shared tiers cannot be read in one call");
  if (!any) {
    launch_remote_lookup(raw, row_f32, rv, tiers, nullptr, c->b, c->raw, n_occ, c->remote_stage, dim, err, st);
    return PB_OK;
  }
  if (!c->stale) {
    Owned o;
    uint32_t *s = nullptr, *h = nullptr, *hd = nullptr;
    if (int rc = o.dev(s, sizeof(uint32_t))) return rc;
    if (int rc = o.mapped(h, hd, sizeof(uint32_t))) return rc;
    c->own.adopt(o);
    c->stale = s;
    c->stale_host = h;
  }
  g.stale = c->stale;
  if (check) {  // (the stale count is read on the host: no stream capture can hold that)
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    PB_CUDA(cudaStreamIsCapturing(st, &cs));
    if (cs != cudaStreamCaptureStatusNone)
      return fail(PB_ERR_STATE, "a remote read of a growable table in another process synchronises its stream on the "
                                "host (its stale check) and cannot be captured in a CUDA graph");
  }
  const auto deadline = std::chrono::steady_clock::now() + std::chrono::milliseconds(PB_STALE_WAIT_MS);
  for (uint32_t round = 0;; ++round) {
    g.only_stale = round > 0;
    if (check) PB_CUDA(cudaMemsetAsync(c->stale, 0, sizeof(uint32_t), st));
    launch_remote_lookup(raw, row_f32, rv, nullptr, &g, c->b, c->raw, n_occ, c->remote_stage, dim, err, st);
    if (!check) return PB_OK;
    PB_CUDA(cudaMemcpyAsync(c->stale_host, c->stale, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    PB_CUDA(cudaStreamSynchronize(st));
    if (*reinterpret_cast<volatile uint32_t*>(c->stale_host) == 0) return PB_OK;
    g_stale_retries += 1;
    for (;;) {  // until some chunk has arrived
      RemoteGrowDev was = g;
      for (uint32_t q = 0; q < R; ++q)
        if (q != rank && views[q] && views[q]->grow)
          if (int rc = drain(views[q])) return rc;
      grow_views(views, R, rank, g, any, check);
      if (std::memcmp(was.rows, g.rows, sizeof(g.rows)) || std::memcmp(was.cells, g.cells, sizeof(g.cells))) break;
      if (std::chrono::steady_clock::now() > deadline)
        return fail(PB_ERR_STATE, "a remote read found rows or index cells of a growing owner that this process has "
                                  "not mapped, and the owner's chunks did not arrive within " +
                                      std::to_string(PB_STALE_WAIT_MS) + " ms");
      std::this_thread::sleep_for(std::chrono::microseconds(200));
    }
    g.stale = c->stale;
  }
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
  if (t->grow && !t->grow_share)
    return fail(PB_ERR_STATE, "a growable table cannot be exported: its storage is mapped in chunks no export describes");
  DeviceGuard g(t->device);
  if (int rc = ensure_alloc(t)) return rc;
  if (!t->seq) {  // the word and, after it, the index's cell count (read by views of an exportable growable table)
    Owned o;
    uint32_t* seq;
    if (int rc = o.dev(seq, 2 * sizeof(uint32_t))) return rc;
    PB_CUDA(cudaDeviceSynchronize());  // (every doubling enqueued so far is done: the count below is the index's)
    const uint32_t init[2] = {0, t->d.n_cells};
    PB_CUDA(cudaMemcpy(seq, init, sizeof(init), cudaMemcpyHostToDevice));
    t->own.adopt(o);
    t->seq = seq;
  }
  ViewBlob b;
  std::memset(&b, 0, sizeof(b));
  b.magic = VIEW_MAGIC;
  b.version = t->tier ? VIEW_VERSION_TIERED : t->grow ? VIEW_VERSION_GROW : VIEW_VERSION;
  b.pid = (uint64_t)getpid();
  b.nonce = process_nonce();
  b.device = t->device;
  void* p[VA_COUNT] = {t->d.cells, t->d.rows, t->d.counters, t->seq};
  b.ipc = 1;
  for (int i = 0; i < VA_COUNT; ++i) {
    b.ptr[i] = reinterpret_cast<uint64_t>(p[i]);
    if (t->grow && (i == VA_CELLS || i == VA_ROWS)) continue;  // (their spans, below)
    if (b.ipc && cudaIpcGetMemHandle(&b.handle[i], p[i]) != cudaSuccess) b.ipc = 0;  // same-process views still work
  }
  if (!b.ipc) {
    cudaGetLastError();  // (the failed handle request is not this call's error)
    std::memset(b.handle, 0, sizeof(b.handle));
  }
  if (t->grow) {
    const GrowSpan cells{t->region[pb_table::G_CELLS].span, t->gran}, rows{t->region[pb_table::G_ROWS].span, t->gran};
    std::memcpy(&b.handle[VA_CELLS], &cells, sizeof(cells));
    std::memcpy(&b.handle[VA_ROWS], &rows, sizeof(rows));
    b.pad = t->max_cells;
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
  if (b.magic != VIEW_MAGIC || (b.version != VIEW_VERSION && b.version != VIEW_VERSION_TIERED && b.version != VIEW_VERSION_GROW))
    return fail(PB_ERR_INVALID, "not a table view (pb_table_export_view)");
  if (!b.n_cells || (b.n_cells & (b.n_cells - 1)) || !b.dim || b.stride < b.dim)
    return fail(PB_ERR_INVALID, "the view's table geometry is malformed");
  const bool grow = b.version == VIEW_VERSION_GROW;
  GrowSpan gs[2] = {};  // rows, cells
  if (grow) {
    std::memcpy(&gs[0], &b.handle[VA_ROWS], sizeof(GrowSpan));
    std::memcpy(&gs[1], &b.handle[VA_CELLS], sizeof(GrowSpan));
    if (h_tier_blob) return fail(PB_ERR_INVALID, "a growable table has no shared host tier: open it with pb_view_open");
    if (b.pad < b.n_cells || (b.pad & (b.pad - 1)) || !gs[0].gran || gs[0].span % gs[0].gran || gs[1].span % gs[0].gran ||
        gs[0].span < sizeof(float) * (uint64_t)b.stride * b.capacity ||
        gs[1].span < sizeof(Cell) * ((uint64_t)b.pad + N_SPECIAL))
      return fail(PB_ERR_INVALID, "the view's growable table geometry is malformed");
  }
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
      if (!grow || (i != VA_CELLS && i != VA_ROWS))
        if (int rc = v->own.ipc(p[i], b.handle[i])) return rc;
    if (grow) {  // the owner's spans, reserved here, and the socket its chunks arrive on
      for (int g = 0; g < 2; ++g) {
        if (int rc = v->own.reserve(v->base[g], gs[g].span)) return rc;
        v->span[g] = gs[g].span;
      }
      p[VA_ROWS] = v->base[0];
      p[VA_CELLS] = v->base[1];
      static std::atomic<uint64_t> serial{0};
      v->addr = "persia_b200.view." + std::to_string(getpid()) + "." + std::to_string(process_nonce()) + "." +
                std::to_string(serial++);
      sockaddr_un sa{};
      sa.sun_family = AF_UNIX;
      std::memcpy(sa.sun_path + 1, v->addr.data(), v->addr.size());  // abstract: no file, gone with the socket
      const socklen_t len = (socklen_t)(offsetof(sockaddr_un, sun_path) + 1 + v->addr.size());
      v->listen_fd = socket(AF_UNIX, SOCK_SEQPACKET | SOCK_NONBLOCK | SOCK_CLOEXEC, 0);
      if (v->listen_fd < 0 || bind(v->listen_fd, reinterpret_cast<sockaddr*>(&sa), len) != 0 || listen(v->listen_fd, 4) != 0)
        return fail(PB_ERR_STATE, std::string("cannot listen on a view's socket: ") + strerror(errno));
    }
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
  if (grow) {
    v->grow = true;
    v->geo = v->seq + 1;
    if (v->listen_fd < 0) v->mapped_rows = v->mapped_cells = ~0u;  // (the owner's own mappings)
  }
  *out = v.release();
  return PB_OK;
}
}  // namespace

int pb_view_address(const pb_view* v, char* h_out, uint64_t cap) {
  if (!v || !h_out || !cap) return fail(PB_ERR_INVALID, "null argument");
  if (v->addr.size() + 1 > cap) return fail(PB_ERR_INVALID, "the address does not fit");
  std::memcpy(h_out, v->addr.c_str(), v->addr.size() + 1);
  return PB_OK;
}

int pb_table_add_reader(pb_table* t, const char* addr) {
  if (!t || !addr) return fail(PB_ERR_INVALID, "null argument");
  if (!t->grow_share) return fail(PB_ERR_STATE, "only a table with exportable growth (pb_table_set_growth(t, 2)) has readers");
  if (!t->exported && !t->live) return fail(PB_ERR_STATE, "export the table first (pb_table_export_view or pb_table_export_live_view)");
  const size_t n = std::strlen(addr);
  if (!n) return PB_OK;  // a view in this process: it maps what the table maps
  sockaddr_un sa{};
  if (n + 1 > sizeof(sa.sun_path)) return fail(PB_ERR_INVALID, "not a view's address (pb_view_address)");
  sa.sun_family = AF_UNIX;
  std::memcpy(sa.sun_path + 1, addr, n);
  const int fd = socket(AF_UNIX, SOCK_SEQPACKET | SOCK_CLOEXEC, 0);
  if (fd < 0 || connect(fd, reinterpret_cast<sockaddr*>(&sa), (socklen_t)(offsetof(sockaddr_un, sun_path) + 1 + n)) != 0) {
    const std::string why = strerror(errno);
    if (fd >= 0) close(fd);
    return fail(PB_ERR_STATE, "cannot reach the reader's view (" + why + "): open the view before registering it, on "
                              "this host, in this network namespace");
  }
  t->readers.r.push_back({fd, 0});
  send_chunks(t);  // every chunk mapped so far
  return PB_OK;
}

uint64_t pb_debug_stale_retries(void) { return g_stale_retries.load(); }

}  // extern "C"

namespace pb {
void send_chunks(pb_table* t) {
  if (t->readers.defer) return;
  const std::vector<pb_table::Chunk>& chunks = t->readers.chunks;
  for (size_t k = 0; k < t->readers.r.size();) {
    pb_table::Reader& x = t->readers.r[k];
    bool gone = false;
    while (x.sent < chunks.size()) {
      ChunkMsg m;
      std::memset(&m, 0, sizeof(m));
      int fds[CHUNKS_PER_MSG];
      for (size_t i = x.sent; i < chunks.size() && m.n < CHUNKS_PER_MSG; ++i) {
        fds[m.n] = chunks[i].fd;
        m.e[m.n].region = chunks[i].region == pb_table::G_ROWS ? 0u : 1u;
        m.e[m.n].off = chunks[i].off;
        m.e[m.n].bytes = chunks[i].bytes;
        m.n++;
      }
      char ctl[CMSG_SPACE(sizeof(int) * CHUNKS_PER_MSG)];
      std::memset(ctl, 0, sizeof(ctl));
      iovec io{&m, sizeof(m)};
      msghdr h{};
      h.msg_iov = &io;
      h.msg_iovlen = 1;
      h.msg_control = ctl;
      h.msg_controllen = CMSG_SPACE(sizeof(int) * m.n);
      cmsghdr* c = CMSG_FIRSTHDR(&h);
      c->cmsg_level = SOL_SOCKET;
      c->cmsg_type = SCM_RIGHTS;
      c->cmsg_len = CMSG_LEN(sizeof(int) * m.n);
      std::memcpy(CMSG_DATA(c), fds, sizeof(int) * m.n);
      const ssize_t sent = sendmsg(x.sock, &h, MSG_DONTWAIT | MSG_NOSIGNAL);  // (the message holds its own references)
      const int e = errno;
      if (sent == (ssize_t)sizeof(m)) {
        x.sent += m.n;
        continue;
      }
      // Only a connection the reader has closed (its view is gone) drops it.  Every other failure keeps the chunks for
      // a later call: a full socket (EAGAIN), and limits that pass, such as ETOOMANYREFS (this user's descriptors in
      // flight over RLIMIT_NOFILE until readers receive them), ENOBUFS or ENOMEM.
      if (sent < 0 && (e == EPIPE || e == ECONNRESET || e == ECONNREFUSED)) gone = true;
      break;
    }
    if (gone) {
      close(x.sock);
      t->readers.r.erase(t->readers.r.begin() + k);
    } else {
      ++k;
    }
  }
}
}  // namespace pb

extern "C" {

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
  if ((rc = remote_lookup(false, row_f32, rv, any_tier(tiers, R), views, R, rank, c, n_occ, own->d.dim,
                          own->d.counters + CTR_ERR, st)))
    return rc;
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
  if ((rc = remote_lookup(true, true, rv, any_tier(tiers, R), views, R, rank, c, n_occ, own->d.dim,
                          own->d.counters + CTR_ERR, st)))
    return rc;
  launch_raw_fill(c->raw, n_occ, own->d.dim, c->remote_stage, d_table_f16, st);  // row u + 1 = f16(row), rounded once
  PB_CUDA(cudaGetLastError());
  return PB_OK;
}

}  // extern "C"
