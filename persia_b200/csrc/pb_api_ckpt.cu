// pb_api_ckpt.cu — the C ABI's checkpoint calls: dump workspaces, parts and nodes (pb_dump.cu), and the images and
// incremental-update packets that loads index and insert (pb_load.cu).
#include <cstring>
#include <new>
#include <string>
#include <vector>

#include "pb_api.cuh"

extern "C" {

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

}  // extern "C"
