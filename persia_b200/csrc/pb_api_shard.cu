// pb_api_shard.cu — the C ABI's sharded path, R GPUs of one box: exchanges, the sharded stage of host-tier moves, and
// the summation and raw forwards and backwards in phases (PB_PHASE_*) over an exchange.
#include <cstring>
#include <memory>
#include <string>

#include "pb_api.cuh"

extern "C" {

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

// The arguments both kinds of exchange check: `chains`, a batch exchange's cap must leave room for its chain links;
// `areas` names the peers' areas in the message.
int check_xchg(uint32_t R, uint32_t rank, uint32_t cap, const uint64_t* h_peer_base, pb_xchg** out, bool chains,
               const char* areas) {
  if (!out || !h_peer_base || R == 0 || R > PB_MAX_RANKS || rank >= R || cap == 0)
    return fail(PB_ERR_INVALID, "bad argument");
  if ((uint64_t)R * cap >= 0xFFFFFFF0ull) return fail(PB_ERR_INVALID, "R * cap must stay below 2^32 - 16");
  if (chains && cap >= CHAIN_END) return fail(PB_ERR_INVALID, "cap must stay below 2^31 - 1");
  for (uint32_t q = 0; q < R; ++q)
    if (!h_peer_base[q] || (h_peer_base[q] & 255u))
      return fail(PB_ERR_INVALID, std::string(areas) + " must be mapped and 256-byte aligned");
  return PB_OK;
}

// Both kinds of exchange start their words with epoch | waited | a count per rank | err (4 words).
constexpr size_t XC_CTRL_WORDS = XC_WORDS + (size_t)XC_WORDS * PB_MAX_RANKS + PB_MAX_RANKS + 4;

// `d` zeroed, then the peers' areas (signs at `off_sign`), R, rank, cap and the control words at `mem` set; returns
// the per-rank counts
uint32_t* init_xchg(XchgDev& d, uint32_t R, uint32_t rank, uint32_t cap, const uint64_t* h_peer_base, uint64_t off_sign,
                    uint32_t* mem) {
  std::memset(&d, 0, sizeof(d));
  for (uint32_t q = 0; q < R; ++q) d.base[q] = h_peer_base[q];
  d.off_sign = off_sign;
  d.R = R;
  d.rank = rank;
  d.cap = cap;
  d.epoch = mem;
  d.waited = d.epoch + XC_WORDS;
  uint32_t* counts = d.waited + (size_t)XC_WORDS * PB_MAX_RANKS;
  d.err = counts + PB_MAX_RANKS;
  return counts;
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
  if (dim == 0) return fail(PB_ERR_INVALID, "bad argument");
  if (int rc = check_xchg(R, rank, cap, h_peer_base, out, true, "receive areas")) return rc;
  DeviceGuard g(device);
  std::unique_ptr<pb_xchg> x(new pb_xchg());
  x->device = device;
  x->dim = dim;
  uint64_t off[6];
  xchg_layout(R, cap, dim, rows_f32, off);
  const size_t words = XC_CTRL_WORDS + 3 * (size_t)R * cap + 1;
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
  XchgDev& d = x->d;
  d.own_cnt = init_xchg(d, R, rank, cap, h_peer_base, off[0], x->mem);
  d.off_row = off[1];
  d.off_grad = off[2];
  d.off_gok = off[3];
  d.off_chain = off[4];
  d.row_f32 = rows_f32 ? 1 : 0;
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
  if (int rc = check_xchg(R, rank, cap, h_peer_base, out, false, "stage areas")) return rc;
  DeviceGuard g(device);
  std::unique_ptr<pb_xchg> x(new pb_xchg());
  x->device = device;
  x->stage = true;  // dim 0: no row, gradient or chain area, no ucell set, no Adam arrays
  uint64_t off[2];
  xchg_stage_layout(R, cap, off);
  if (int rc = x->own.dev(x->mem, 4 * XC_CTRL_WORDS)) return rc;  // the control words alone, `sent` as the counts
  PB_CUDA(cudaMemset(x->mem, 0, 4 * XC_CTRL_WORDS));
  PB_CUDA(cudaDeviceSynchronize());
  XchgDev& d = x->d;
  x->sent = init_xchg(d, R, rank, cap, h_peer_base, off[0], x->mem);
  d.off_row = d.off_grad = d.off_gok = d.off_chain = off[1];
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
  if (ph.has(PB_PHASE_PREPARE)) {  // requester, local: the numbering and its distinct signs per owner
    c->raw_pending.drop();  // the numbering below replaces the pending batch's
    if ((rc = number_raw(c, sl, d_ids, n_occ, d_row_off, batch, sample_fixed_size, d_index, d_non_empty, d_sample_id_num,
                         d_counts, st)))
      return rc;
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
    if (!prepared && (rc = number_raw(c, sl, d_ids, n_occ, d_row_off, batch, sample_fixed_size, d_index, d_non_empty,
                                      d_sample_id_num, d_counts, st)))
      return rc;
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

}  // extern "C"
