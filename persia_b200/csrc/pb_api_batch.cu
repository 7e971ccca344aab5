// pb_api_batch.cu — the C ABI's batch contexts and the calls that run a batch on one GPU: pb_forward / pb_backward
// (summation slots) and pb_forward_raw / pb_backward_raw (a raw slot), with the checks and steps that their sharded
// (pb_api_shard.cu) and remote (pb_api_view.cu) forms share.
#include <cmath>
#include <cstring>
#include <memory>

#include "pb_api.cuh"

namespace pb {

// ---- what the local and sharded forms of the forwards and backwards share ------------------------------------------
static int check_grads_aligned(const void* const* h_grads, uint32_t n_slots) {
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
static int copy_row_off(pb_ctx* c, const uint32_t* d_row_off, uint32_t n_rows, cudaStream_t st) {
  PB_CUDA(cudaMemcpyAsync(c->row_off, d_row_off, 4 * ((size_t)n_rows + 1), cudaMemcpyDeviceToDevice, st));
  launch_expand_rows(c->row_off, n_rows, c->occ_outrow, st);
  return PB_OK;
}

// The context's previous batch goes (like an expired post_forward_buffer entry, mod.rs:991-1029), and with it any
// batch prepared and never sent.
static void drop_batch(pb_ctx* c, cudaStream_t st) {
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
                  cudaStream_t st, bool prepared) {
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

// A backward's staging buffer `buf` of `floats` floats, held by `own`, grown to hold `need`.  The training forward grows
// it, so the backward that follows neither synchronises nor allocates (and can be captured without a warm-up call).  The first
// allocation neither synchronises nor enqueues anything, so that a context's first forward can be captured too: the
// thread's capture mode is relaxed around it (cudaMalloc is refused under a global-mode capture otherwise).  Growing
// synchronises the stream and frees the old buffer: a forward captured with a larger need than any call before it fails
// its capture, and a graph captured earlier must not be replayed after a larger call ran eagerly (warm up with the
// largest batch, as for vw_stage).
int grow_stage(Owned& own, float*& buf, size_t& floats, size_t need, cudaStream_t st) {
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

// ---- raw slots ------------------------------------------------------------------------------------
int ensure_raw(pb_ctx* c) {
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

// A raw slot's numbering, for the calls whose rows come from elsewhere (the sharded and remote raw forwards): the
// slot's distinct signs numbered, index / non_empty / sample_id_num written and the counts copied out.  No table state
// is read.
int number_raw(pb_ctx* c, const SlotsDev& sl, const uint64_t* d_ids, uint32_t n_occ, const uint32_t* d_row_off,
               uint32_t batch, uint32_t sample_fixed_size, int64_t* d_index, int64_t* d_non_empty,
               uint32_t* d_sample_id_num, uint32_t* d_counts, cudaStream_t st) {
  if (d_row_off) {
    if (int rc = copy_row_off(c, d_row_off, batch, st)) return rc;
  }
  launch_raw_number(sl, d_ids, n_occ, d_row_off ? c->row_off : nullptr, d_row_off ? c->occ_outrow : nullptr, batch,
                    sample_fixed_size, nullptr, c->raw, (long long*)d_index, (long long*)d_non_empty, d_sample_id_num, st);
  PB_CUDA(cudaMemcpyAsync(d_counts, c->raw.counts, 8, cudaMemcpyDeviceToDevice, st));
  return PB_OK;
}

}  // namespace pb

extern "C" {

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

}  // extern "C"
