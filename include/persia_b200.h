/* persia_b200.h — C ABI of libpersia_b200.so: PERSIA's sparse-embedding hot path on H100 (sm_90a).
 *
 * The reference (PersiaML/PERSIA @ ff754b8) has no FFI for this path: its NN-worker engine
 * (rust/persia-core) talks to an embedding worker and R parameter servers over HTTP.  These entry
 * points are what a Rust `extern "C"` block in persia-core (or the C++/Python host side shipped in
 * this repo) binds instead of those RPC clients; each one names the reference interface it replaces.
 * Plain pointers and sizes only; every call is ordered on the given CUDA stream (passed as void*,
 * i.e. a cudaStream_t), never synchronises the device unless its comment says so, and returns 0 or a
 * negative pb_status; pb_last_error() gives the message for the calling thread.
 *
 * Conventions: `d_` = device pointer, `h_` = host pointer.  Gradient, output and update buffers (the gradients of
 * pb_backward, pb_backward_sharded, pb_backward_raw(_sharded) and pb_update; d_out_f16 of pb_forward and
 * pb_forward_sharded; d_table_f16 of pb_forward_raw(_sharded)) must be 16-byte aligned: the kernels access them with vector loads and stores.  A
 * call given a pointer that is not returns PB_ERR_INVALID before it enqueues anything.  (A contiguous tensor view at
 * a storage offset, e.g. one slot of an [S, B, dim] tensor when B * dim * 2 is not a multiple of 16, can break the
 * rule; the Python wrappers pass a copy of such views.)  A "sign" is a prefixed u64 feature id
 * (embedding_worker_service/mod.rs:402-429).  One pb_table is one parameter-server shard resident in
 * one GPU's HBM, fixed embedding dim (the host side keeps one table per distinct dim).
 */
#ifndef PERSIA_B200_H_
#define PERSIA_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PB_MAX_SLOTS 128

typedef enum {
  PB_OK = 0,
  PB_ERR_INVALID = -1,   /* bad argument */
  PB_ERR_CUDA = -2,      /* CUDA runtime error (message in pb_last_error) */
  PB_ERR_STATE = -3,     /* optimizer / hyper-parameters not configured (reference: OptimizerNotFoundError, NotConfiguredError) */
  PB_ERR_CAPACITY = -4,  /* workspace too small for this batch */
  PB_ERR_BATCH = -5      /* batch size > 65535 (persia-common/src/lib.rs:49-51 panics) */
} pb_status;

typedef enum { PB_OPT_SGD = 0, PB_OPT_ADAGRAD = 1, PB_OPT_ADAGRAD_VW = 2, PB_OPT_ADAM = 3 } pb_optim_kind;

typedef struct pb_table pb_table; /* one shard: hash index + row store, owned by the library */
typedef struct pb_ctx pb_ctx;     /* per-batch device context: what the EW keeps in post_forward_buffer */

/* EmbeddingParameterServerConfig.capacity (persia-embedding-config/src/lib.rs:389-468) + slot dim. */
typedef struct {
  uint32_t dim;
  uint64_t capacity; /* max resident rows of this shard */
} pb_table_cfg;

/* OptimizerConfig (persia-common/src/optim.rs:11-41). */
typedef struct {
  int kind; /* pb_optim_kind */
  float lr, wd, g_square_momentum, initialization, eps, beta1, beta2;
} pb_optim_cfg;

/* PersiaEmbeddingModelHyperparameters: configure_embedding_parameter_servers (persia-core/src/nats.rs:355-384
 * -> embedding_parameter_service/mod.rs:440-451). */
typedef struct {
  float init_lower, init_upper, admit_probability;
  int enable_weight_bound;
  float weight_bound;
} pb_hyper_cfg;

const char* pb_last_error(void);
int pb_version(void);

/* ---- table lifetime / configuration ------------------------------------------------------------ */
/* PersiaEmbeddingHolder::get (persia-embedding-holder/src/lib.rs:36-71). Allocation is deferred to the
 * first use, once the optimizer (hence the per-row state size, optim.rs:84) is known. */
int pb_table_create(int device, const pb_table_cfg* cfg, pb_table** out);
int pb_table_destroy(pb_table* t);
/* register_optimizer (embedding_parameter_service/mod.rs:429-438). Must precede the first insert. */
int pb_table_set_optimizer(pb_table* t, const pb_optim_cfg* cfg);
/* configure (embedding_parameter_service/mod.rs:440-451). */
int pb_table_configure(pb_table* t, const pb_hyper_cfg* cfg);
/* num_total_signs (persia-embedding-holder/src/lib.rs:73-79); synchronises `stream`. */
int pb_table_size(pb_table* t, uint64_t* h_out, void* stream);
/* clear (persia-embedding-holder/src/lib.rs:95-97). */
int pb_table_clear(pb_table* t, void* stream);
/* Capacity policy.  The reference's EvictionMap drops the least recently used entry on every insert beyond capacity
 * (persia-embedding-holder/src/eviction_map.rs:76-97).  Here recency is the batch number of a row's last training
 * lookup and eviction is a sweep: every `check_every` training requests, if fewer than `low_water` rows are free,
 * the oldest rows are released until `target_free` are (rows touched in the last `keep_batches` batches are never
 * released: gradients may still be in flight for them).  check_every == 0 (default): no eviction, admissions beyond
 * capacity are refused and counted. */
int pb_table_set_eviction(pb_table* t, uint32_t check_every, uint64_t low_water, uint64_t target_free, uint32_t keep_batches);
/* floats per resident row: dim + optimizer state (emb_entry.rs:17-25 `inner`). */
int pb_table_entry_len(pb_table* t, uint32_t* h_out);
/* Host-DRAM tier (BASELINE.json configs[4]: the embedding holder's DRAM behind a GPU-resident working set): release the
 * least recently used rows until `want_free` rows are free, like the capacity sweep (rows touched by the last
 * max(keep_batches, pending batches + 1) requests stay), but WRITE EVERY VICTIM OUT first: its sign to d_signs[k] and its
 * whole entry (embedding ++ optimizer state, pb_entry_len floats) to d_entries[k].  Victims beyond max_n stay resident;
 * *d_count = victims found (<= max_n were released).  The caller keeps the pairs (persia_b200/tier.py) and brings a sign
 * back with pb_set_rows before its next lookup.  Enqueued on `stream`. */
int pb_table_spill(pb_table* t, uint64_t want_free, uint32_t keep_batches, uint64_t* d_signs, float* d_entries, uint32_t max_n,
                   uint32_t* d_count, void* stream);
/* counters since creation / clear: [0] resident rows (admitted - evicted), [1] distinct signs of a request that missed
 * (infer) or were not admitted (index_miss_count), [2] gradient ids not found (gradient_id_miss_count), [3] admissions
 * refused because the shard is full, [4] in-kernel waits that gave up (must stay 0: a non-zero value voids the batch
 * that raised it).  Synchronises `stream`. */
int pb_table_counters(pb_table* t, uint64_t h_out[5], void* stream);

/* ---- single-request entry points (the PS RPCs) ------------------------------------------------- */
/* lookup_mixed -> batched_lookup (embedding_parameter_service/mod.rs:162-262, 344-357).
 * d_signs[n] -> d_out[n*dim] f32.  training!=0: hit refreshes recency, miss admits + initialises;
 * training==0: read-only, zeros on miss. */
int pb_lookup(pb_table* t, const uint64_t* d_signs, uint32_t n, int training, float* d_out, void* stream);
/* update_gradient_mixed (embedding_parameter_service/mod.rs:359-427): one optimizer step per sign in
 * request order, d_grads[n*dim] f32; absent signs are counted and skipped.  Signs must be distinct
 * within one call (the EW sends each sign once per slot; see pb_backward for the batched form). */
int pb_update(pb_table* t, const uint64_t* d_signs, const float* d_grads, uint32_t n, void* stream);
/* set_embedding (embedding_parameter_service/mod.rs:287-306; persia-core/src/lib.rs:433-449):
 * d_entries[n*entry_len] = emb ++ optimizer state. */
int pb_set_rows(pb_table* t, const uint64_t* d_signs, const float* d_entries, uint32_t n, void* stream);
/* debug read-back of full entries (zeros + found=0 when absent); does not touch recency. */
int pb_get_rows(pb_table* t, const uint64_t* d_signs, uint32_t n, float* d_entries, uint8_t* d_found, void* stream);

/* Checkpoint support (persia-model-manager/src/lib.rs:242-257 dumps every internal shard's LRU list): the signs
 * resident in the table and, per sign, the training-request number it was last used in (ascending = the
 * reference's list order, oldest first, up to ties inside a request).  At most max_n pairs are written, in no
 * particular order; *d_count receives the number of resident signs (call with max_n = 0 to size the buffers).
 * Entries are then read with pb_get_rows and restored with pb_set_rows. */
int pb_table_export_signs(pb_table* t, uint64_t* d_signs, uint32_t* d_recency, uint32_t max_n, uint32_t* d_count,
                          void* stream);

/* ---- id preprocessing (the EW's lookup_batched_all_slots_preprocess) --------------------------- */
/* indices_add_prefix (embedding_worker_service/mod.rs:402-429): out[i] = ids[i] % spacing + prefix of
 * the slot owning occurrence i; h_slot_occ_off[n_slots+1] are the slot boundaries in the flat id array. */
int pb_add_prefix(const uint64_t* d_ids, uint32_t n, const uint32_t* h_slot_occ_off, const uint64_t* h_prefix,
                  uint32_t n_slots, uint32_t prefix_bit, uint64_t* d_out, void* stream);
/* sign_to_shard_modulo (embedding_worker_service/mod.rs:341-345): farmhash64(sign LE bytes) % R. */
int pb_shard_of(const uint64_t* d_signs, uint32_t n, uint32_t R, uint32_t* d_shard, void* stream);
/* indices_to_hashstack_indices (embedding_worker_service/mod.rs:347-400): every id becomes `rounds` keys,
 * d_out[i * rounds + r] = farmhash64^(r+1)(id_i) % embedding_size + r * embedding_size (a sample's ids stay together:
 * sample_num_signs grows by `rounds`, :393-397; the caller scales its row offsets).  The regrouping per hashed key
 * is the forward's per-batch dedup. */
int pb_hash_stack(const uint64_t* d_ids, uint32_t n, uint32_t rounds, uint64_t embedding_size, uint64_t* d_out, void* stream);
/* farmhash64 of each 8-byte little-endian value (hash-stack building block, :364). */
int pb_farmhash64(const uint64_t* d_in, uint32_t n, uint64_t* d_out, void* stream);
/* indices_to_sharded_indices (embedding_worker_service/mod.rs:454-479) as a stable partition:
 * d_perm[n] lists input positions grouped by shard (input order kept inside a shard),
 * d_counts[R] the group sizes.  d_work: pb_partition_workspace(n) bytes. */
int pb_partition_by_shard(const uint64_t* d_signs, uint32_t n, uint32_t R, uint32_t* d_perm, uint32_t* d_counts,
                          void* d_work, uint64_t work_bytes, void* stream);
uint64_t pb_partition_workspace(uint32_t n);

/* ---- batched path: forward_batched_direct / update_gradient_batched ---------------------------- */
/* Slot semantics of one batch stream (persia-embedding-config/src/lib.rs:528-550). */
typedef struct {
  uint32_t n_slots;
  uint32_t prefix_bit;               /* feature_index_prefix_bit */
  uint64_t prefix[PB_MAX_SLOTS];     /* SlotConfig.index_prefix (0 = none) */
  uint8_t sqrt_scaling[PB_MAX_SLOTS];
} pb_slots_cfg;

int pb_ctx_create(int device, uint32_t max_occurrences, uint32_t max_out_rows, pb_ctx** out);
int pb_ctx_destroy(pb_ctx* c);
int pb_ctx_set_slots(pb_ctx* c, const pb_slots_cfg* cfg);
/* The last training batch seen by the context, as the reference's batch_unique_indices_rate gauge reports it
 * (embedding_worker_service/mod.rs:664-673): [0] distinct (slot, sign) pairs, of which [1] occur once, [2] 2..32 times,
 * [3] more often; [4] occurrences held by the repeated ones; [5] id occurrences.  Synchronises `stream`. */
int pb_ctx_batch_stats(pb_ctx* c, uint32_t h_out[6], void* stream);

/* EmbeddingWorker::forward_batched_direct for summation slots
 * (embedding_worker_service/mod.rs:1076-1107 -> :874-942 -> PS :162-262 -> :486-629).
 * d_ids: flat raw ids, slot-major then sample-major; d_row_off[n_slots*batch+1] CSR offsets, or NULL
 * when every sample holds exactly one id per slot (then n_occ == n_slots*batch).
 * h_slot_occ_off[n_slots+1]: slot boundaries in d_ids.  d_out: n_slots*batch rows of `dim` f16
 * (slot s, sample b at row s*batch+b).  training!=0 keeps the deduplicated ids in `c` for pb_backward.
 * Inside: FeatureBatch::new (persia-common/src/lib.rs:45-82) as a device-side per-slot dedup, then the lookup over the
 * distinct signs only, then pooling.  Capturable in a CUDA graph on its own. */
int pb_forward(pb_table* t, pb_ctx* c, const uint64_t* d_ids, uint32_t n_occ, const uint32_t* d_row_off,
               const uint32_t* h_slot_occ_off, uint32_t batch, int training, void* d_out_f16, void* stream);

/* EmbeddingWorker::update_gradient_batched (embedding_worker_service/mod.rs:1109-1129 -> :703-872 ->
 * PS :359-427).  h_grads[s]: device pointer to slot s's [batch, dim] gradient (GradientBatch::add_gradient,
 * persia-core/src/backward.rs:86-105), NULL = add_skipped_gradient; is_f16 as there; h_scale[s] the loss
 * scale.  A slot whose gradient holds a NaN is skipped whole (:731-746); d_slot_status[n_slots] (optional)
 * receives 0 applied / 1 skipped / 2 NaN.  The gradients of a sign are summed in the reference's order (ascending
 * sample) whatever its multiplicity, so updated rows are bit-identical to the reference's f32 arithmetic.  Part of the
 * work runs on a stream owned by the context and is joined before the call returns control of `stream`'s order
 * (capturable in a CUDA graph on its own). */
int pb_backward(pb_table* t, pb_ctx* c, const void* const* h_grads, int is_f16, const float* h_scale,
                int32_t* d_slot_status, void* stream);

/* Raw (embedding_summation: false) slot of one batch — FeatureRawEmbeddingBatch,
 * embedding_worker_service/mod.rs:498-512, :540-545, :593-623 and the index list of persia-core forward.rs:336-347.
 * The context serves ONE slot (pb_ctx_set_slots with n_slots == 1; its prefix applies).  d_ids: the slot's flat
 * ids, sample-major; d_row_off[batch+1] CSR offsets or NULL when every sample holds one id.  Outputs (device):
 *   d_table_f16   [(U+1), dim] f16, row 0 zeros, row u+1 = embedding of distinct sign u; capacity n_occ+1 rows
 *   d_index       [batch * sample_fixed_size] i64, 0 = padding, else u+1
 *   d_non_empty   ascending positions of d_index that hold an id; capacity batch * sample_fixed_size
 *   d_sample_id_num [batch] = min(ids of the sample, sample_fixed_size)
 *   d_counts      [2] = {U, number of entries of d_non_empty}
 * Distinct signs are numbered by first occurrence (the reference: hashbrown iteration order, unpinned).  A raw slot
 * with hash-stack (mod.rs:503-507, :581-590) is not supported. */
int pb_forward_raw(pb_table* t, pb_ctx* c, const uint64_t* d_ids, uint32_t n_occ, const uint32_t* d_row_off,
                   uint32_t batch, uint32_t sample_fixed_size, int training, void* d_table_f16, int64_t* d_index,
                   int64_t* d_non_empty, uint32_t* d_sample_id_num, uint32_t* d_counts, void* stream);
/* Raw arm of update_all_batched_gradients (mod.rs:731-755, :790-798) + update_gradient_mixed: d_grad is the
 * [U, dim] gradient of the distinct-sign table without its row 0 (persia/ctx.py:970-980 passes f32), NULL =
 * add_skipped_gradient.  *d_status: 0 applied, 1 skipped, 2 dropped for NaN. */
int pb_backward_raw(pb_table* t, pb_ctx* c, const void* d_grad, int is_f16, float scale, int32_t* d_status,
                    void* stream);

/* ---- the same two calls over the R GPUs of one box ------------------------------------------------------------------
 * Every rank is the embedding worker of its own batches and parameter server `rank` (rows with
 * farmhash64(sign) % R == rank, sign_to_shard_modulo, embedding_worker_service/mod.rs:341-345).  The EW's fan-out
 * (one lookup_mixed / update_gradient_mixed per server, mod.rs:886-919, :835-859) is done by the kernels themselves:
 * the distinct signs of the batch (mod.rs:454-479 shards the deduplicated signs), the returned rows and the reduced
 * gradients are stored straight into the receiver's area over NVLink peer mappings, ordered by flag words in that
 * area.  No NCCL and no host on the data path; a step is capturable in a CUDA graph.
 *
 * A rank's batch is one request per owner, as with R data-parallel NN workers in the reference; an owner serves the
 * forward requests of a step together and applies the R gradient requests one after another in rank order (the
 * reference applies them in arrival order).  Both calls are collective: every rank of the box calls them once per
 * step.  A rank's receive area is pb_xchg_bytes() bytes of zero-initialised device memory that all ranks can store
 * to (CUDA peer access / symmetric memory); h_peer_base[q] is rank q's area as mapped in this process, 256-byte
 * aligned; cap = slots per (source, owner) pair, i.e. the most distinct signs one rank may request of one owner in one
 * batch; rows_f32 != 0 returns f32 rows (needed for ragged layouts, which pool on the requester; f16 otherwise). */
typedef struct pb_xchg pb_xchg;
uint64_t pb_xchg_bytes(uint32_t R, uint32_t cap, uint32_t dim, int rows_f32);
int pb_xchg_create(int device, uint32_t R, uint32_t rank, uint32_t cap, uint32_t dim, int rows_f32,
                   const uint64_t* h_peer_base, pb_xchg** out);
int pb_xchg_destroy(pb_xchg* x);
/* h_out[0] != 0: a batch needed more than cap slots for one pair (its excess signs read as zeros and took no
 * gradient: re-run it with a larger cap); h_out[1] != 0: a wait for a peer gave up.  Synchronises `stream`. */
int pb_xchg_status(pb_xchg* x, uint32_t h_out[2], void* stream);
/* `phases`: the call enqueues these parts of the exchange (0 = PB_PHASE_ALL, the normal call).  One process per GPU
 * always passes 0.  Splitting exists for hosts that drive several ranks of one GPU from one thread (tests: R virtual
 * ranks sharing a device): enqueue SEND for every rank, then SERVE for every rank, then FINISH for every rank, with
 * the same arguments each time — no rank then waits on a flag whose raising has not been enqueued yet. */
#define PB_PHASE_SEND 1   /* requester: forward dedup + signs out; backward NaN rule + reduce + gradients out */
#define PB_PHASE_SERVE 2  /* owner: forward lookups + rows out; backward optimizer steps */
#define PB_PHASE_FINISH 4 /* requester, forward only: rows in -> output */
#define PB_PHASE_ALL 7
/* forward_batched_direct over R shards: arguments as pb_forward (raw slots: pb_forward_raw_sharded below).  Slots that
 * share a feature group (equal prefixes) are supported: a sign held by several of them is one entry per slot of the
 * request, and the owner steps a row rank by rank, each rank's entries in slot order, as the reference does. */
int pb_forward_sharded(pb_table* t, pb_ctx* c, pb_xchg* x, const uint64_t* d_ids, uint32_t n_occ, const uint32_t* d_row_off,
                       const uint32_t* h_slot_occ_off, uint32_t batch, int training, void* d_out_f16, void* stream,
                       int phases);
/* update_gradient_batched over R shards: arguments as pb_backward.  The NaN rule is applied per slot on the requesting
 * rank, before anything is sent (mod.rs:731-746). */
int pb_backward_sharded(pb_table* t, pb_ctx* c, pb_xchg* x, const void* const* h_grads, int is_f16, const float* h_scale,
                        int32_t* d_slot_status, void* stream, int phases);
/* A raw (embedding_summation: false) slot over R shards: arguments and outputs as pb_forward_raw / pb_backward_raw, plus
 * the exchange and `phases`.  Each call is one request per owner (the slot's distinct signs, sharded by
 * farmhash64(sign) % R); the owner serves and applies them like the summation calls' (R requests, rank order).
 *   - The exchange must be created with rows_f32 != 0, and its dim must be the table's.  The owner returns f32 rows and
 *     the requester rounds them once: table row u+1 is f16(row) bit for bit, so a -0 element stays -0 (an f16 exchange
 *     would give f16(0 + row)).  Signs over `cap` read as zeros, take no gradient and raise pb_xchg_status' h_out[0].
 *   - The context serves one slot; the exchange serves this slot only (one exchange per raw slot and rank).  Its rows
 *     may live in the same pb_table as the summation slots of that dim.
 *   - Backward: d_grad is the [U, dim] gradient (U = d_counts[0] of the forward), NULL = add_skipped_gradient.  The NaN
 *     rule (the whole request is dropped), the f16 +-inf clamp and 1/scale are applied on the requesting rank before
 *     anything is sent; *d_status as pb_backward_raw.  Without a pending raw training forward: PB_ERR_STATE.
 *   - Both are collective, also for an empty batch (U = 0): every rank calls them once per step, and every rank must
 *     issue the step's collective calls (raw and summation, over all exchanges) in the same order — a rank waiting on
 *     one exchange blocks its stream while a peer may be waiting on another.
 * U stays on the device: no host sync and no allocation after the first call of a context, so a step is capturable. */
int pb_forward_raw_sharded(pb_table* t, pb_ctx* c, pb_xchg* x, const uint64_t* d_ids, uint32_t n_occ,
                           const uint32_t* d_row_off, uint32_t batch, uint32_t sample_fixed_size, int training,
                           void* d_table_f16, int64_t* d_index, int64_t* d_non_empty, uint32_t* d_sample_id_num,
                           uint32_t* d_counts, void* stream, int phases);
int pb_backward_raw_sharded(pb_table* t, pb_ctx* c, pb_xchg* x, const void* d_grad, int is_f16, float scale,
                            int32_t* d_status, void* stream, int phases);

/* Number of kernels the library has launched on behalf of the caller since load (bench bookkeeping). */
uint64_t pb_launch_count(void);
/* Bench instrumentation: launches of the kernel families selected by the bit mask are bracketed by CUDA events on
 * their stream (0 = off).  pb_profile_read synchronises the device and returns summed milliseconds and launch
 * counts per family: 0 probe/admit, 1 dedup, 2 gather+pool, 3 NaN scan, 4 reduce+update of hot signs (> 32 occurrences),
 * 5 update of the signs that occur once, 6 other, 7 reduce+update of the signs of 2..32 occurrences; sharded path: 8 waits
 * for peers' flags, 9 route + signals, 10 the owner's update (its lookup counts as 0, the expand as 2). */
#define PB_PROFILE_FAMILIES 11
int pb_profile_enable(int family_mask);
int pb_profile_read(double* h_ms, uint64_t* h_count, int n_families);

#ifdef __cplusplus
}
#endif
#endif /* PERSIA_B200_H_ */
