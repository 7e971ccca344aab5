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
 * Conventions: `d_` = device pointer, `h_` = host pointer.  A create or call that returns an error leaves nothing
 * allocated by it, but for what the steps it completed before the error acquired (a context's first-use buffers, say),
 * which the object keeps and its next call uses instead of acquiring them again.  Gradient, output and update buffers (the gradients of
 * pb_backward, pb_backward_sharded, pb_backward_raw(_sharded) and pb_update; d_out_f16 of pb_forward and
 * pb_forward_sharded; d_table_f16 of pb_forward_raw(_sharded)) must be 16-byte aligned: the kernels access them with vector loads and stores.  A
 * call given a pointer that is not returns PB_ERR_INVALID before it enqueues anything.  (A contiguous tensor view at
 * a storage offset, e.g. one slot of an [S, B, dim] tensor when B * dim * 2 is not a multiple of 16, can break the
 * rule; the Python wrappers pass a copy of such views.)  A "sign" is a prefixed u64 feature id
 * (embedding_worker_service/mod.rs:402-429).  One pb_table is one parameter-server shard resident in
 * one GPU's HBM, fixed embedding dim (the host side keeps one table per distinct dim).
 *
 * Several streams on one table (batches in flight, embedding_staleness > 1: one pb_ctx and one stream per batch).
 * The library orders the calls on one table, whatever their streams, in the order they are issued, in two chains:
 *   - steps: pb_backward, pb_backward_raw and pb_update (the row steps, Adam's beta-power advance and the incremental
 *     set's marks).  Two steps never overlap, so no gradient is lost and no entry torn, and every row is stepped in
 *     issue order, as the reference's entry locks step it in some serial order.
 *   - index work: the training and inference forms of pb_forward, pb_forward_raw and pb_lookup (probes, admissions,
 *     eviction checks, index rebuilds, tier restores), plus pb_update.
 *   A backward is in the step chain only, so it runs beside the next batch's forward: a forward may read rows a backward
 *   on another stream is stepping (the staleness embedding_staleness allows).  An eviction check also waits for every
 *   step issued before it, so it never releases a row whose gradients are still to be applied.  pb_set_rows,
 *   pb_get_rows, pb_table_export_signs, pb_table_clear, the statistics calls, pb_inc_take, pb_table_dump_part and
 *   pb_dump_nodes are in both chains.
 *   pb_tier_stage waits for both chains and is in the index chain only.
 * Waiting costs a stream-wait on an event per call; a wait on work already complete costs nothing on the device.
 * Calls on one table must still be issued from one host thread at a time (the persia_core groups hold a lock), and a
 * pb_ctx holds one batch at a time.  Under CUDA stream capture the ordering becomes edges of the graph when the calls
 * are captured into one graph (contexts forked onto side streams of one capture); graphs captured separately cannot be
 * ordered by the library (a capture waits only on events of the same capture): whoever launches them orders them, e.g.
 * replays on one stream, or events between replays that touch one table.  A call captured while earlier work on the
 * table issued outside the capture is still running fails with PB_ERR_STATE (synchronise before capturing).  The
 * sharded calls (pb_*_sharded) are not in these chains: their caller orders them.
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
  PB_ERR_BATCH = -5,     /* batch size > 65535 (persia-common/src/lib.rs:49-51 panics) */
  PB_ERR_FORMAT = -6     /* malformed checkpoint image or packet; pb_last_error() = "ExceptionType: message"
                            (pb_image_index, pb_image_packet) */
} pb_status;

typedef enum { PB_OPT_SGD = 0, PB_OPT_ADAGRAD = 1, PB_OPT_ADAGRAD_VW = 2, PB_OPT_ADAM = 3 } pb_optim_kind;

/* What Adagrad's fused lanes (elements < 8 * floor(dim / 8)) take for 1 / sqrt(s + eps); the tail is exact either way.
 * EXACT: the correctly rounded value.  INTEL: _mm256_rsqrt_ps as Intel CPUs compute it (a 2 x 1024-entry table), which
 * reproduces the reference's Adagrad steps bit for bit as run on an Intel CPU. */
typedef enum { PB_RSQRT_EXACT = 0, PB_RSQRT_INTEL = 1 } pb_rsqrt_mode;

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
/* Adagrad's rsqrt mode (pb_rsqrt_mode; PB_RSQRT_EXACT until set).  Like pb_table_set_optimizer, it is read when work is
 * enqueued: it applies to every row step enqueued after the call, and a captured graph keeps the mode it was captured
 * with.  Any optimizer kind accepts it; only the Adagrad kinds read it.  Rows of an attached host-memory tier are stepped
 * with the mode of the table they are attached to. */
int pb_table_set_rsqrt(pb_table* t, int mode);
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
/* counters since creation / clear: [0] resident rows (admitted - evicted), [1] distinct signs of a request that missed
 * (infer) or were not admitted (index_miss_count), [2] gradient ids not found (gradient_id_miss_count), [3] admissions
 * refused because the shard is full, [4] in-kernel waits that gave up (must stay 0: a non-zero value voids the batch
 * that raised it).  Synchronises `stream`. */
int pb_table_counters(pb_table* t, uint64_t h_out[5], void* stream);
/* ---- host-memory tier: a table larger than HBM, on one GPU or behind each of R ------------------------------------
 * The reference's parameter server keeps every entry in host DRAM, bounded by `capacity`.  A tier is a second table
 * whose rows (embedding ++ optimizer state) live in mapped pinned host memory (cudaHostAllocMapped | Portable, not
 * write-combined); its index cells, row recency, free-row stack and counters live in HBM like any table's.  So HBM
 * bounds the tier too, at 44-68 B of HBM per host row: 16 B index cells, n_cells = next_pow2(1.5 x rows) (24-48 B per
 * row), plus row recency 4, free-row stack 4 and the rebuild's pairs 12.  That is about 1.2e8-1.8e8 host rows per 8 GB.
 * (The HBM table itself adds 4 B per HBM row for the move's victim list.)
 *
 * Attached behind an HBM table (same dim and optimizer kind: one entry layout), the tier is never trained directly; the
 * kernels only move or read whole entries, stream-ordered, without host synchronisation (a step stays capturable in a
 * CUDA graph):
 *   - out: every eviction check of the HBM table (pb_table_set_eviction) moves its victims into the tier instead of
 *     dropping them.  The tier first drops its own oldest entries until it can hold them (counted as dropped: the
 *     reference's LRU bound on the whole table), then each victim is written to a tier row and published there before
 *     its HBM cell is released.  Rows of pending batches (raw ones included) are never victims.
 *   - restore: training requests — pb_forward (over the batch's distinct signs), pb_forward_raw, pb_lookup — and
 *     pb_set_rows first move every tier-held sign of the request back into a free HBM row (a pending batch holds HBM rows).
 *   - in place: inference requests (training == 0) of pb_forward, pb_forward_raw and pb_lookup read tier-held signs where
 *     they are and move nothing, so an inference pass of any size returns every value; pb_update steps a tier-held row
 *     where it is; pb_get_rows reads the tier in place; pb_set_rows stores the entries the HBM table has no row for in
 *     the tier (entries neither table has a row for are counted as dropped).
 * Invariants: a sign lives in at most one of the two tables.  A tier-held sign is never re-initialised: if a training
 * request finds no free HBM row for it (e.g. pending batches protect every row) its restore is refused and counted, it
 * reads as zeros and its gradient counts as a gradient miss (as an admission refused for capacity does), and its tier
 * entry stays as it was.  A moved entry keeps its recency, and the tier ages rows by the HBM table's training-request
 * number: the union evicts least recently used first, and pb_table_export_signs of both tables merges into the
 * reference's list order.
 * pb_table_clear of the table clears its tier too.  Destroy the table before its tier.  The sharded calls serve a
 * table with a tier on its owner rank by the same rules (see the R-GPU calls below).  A table whose tier came from
 * pb_table_create_host cannot be exported; one whose tier came from pb_table_create_host_shared can (below).
 *
 * Staging (pb_tier_stage): the ids of batch i+1 are known while batch i trains, and moving an entry never changes its
 * value, so the moves of request i+1 can run one batch ahead, on a stream of their own, beside batch i's dense step and
 * backward.  The library orders a stage through the two chains above: it starts after every earlier call on the table
 * (pending backwards included, whatever their streams), and every later call on the table or its tier except
 * pb_backward and pb_backward_raw (in the step chain alone, they run beside it) starts after it.  In a CUDA graph, a
 * stage and the calls after it work when they are captured into one graph, the stage on a stream forked from the
 * capturing one; a call captured after a stage issued outside the capture that has not completed fails with
 * PB_ERR_STATE (synchronise before capturing). */
int pb_table_create_host(int device, const pb_table_cfg* cfg, pb_table** out);
/* A host tier whose rows another process can map: pb_table_create_host in every way but where the host rows come
 * from.  They are an anonymous memfd (memfd_create; no named /dev/shm file, whose mount is often 64 MB in containers),
 * ftruncate'd and mapped MAP_SHARED | MAP_POPULATE, then registered with cudaHostRegister(Mapped | Portable): not
 * write-combined, like pb_table_create_host's.  A table with such a tier can be exported (pb_table_export_view,
 * pb_table_export_live_view, then pb_table_export_tier_view), and its peers read the tier in place.  The memory is
 * shmem: it is charged to the owning process's memory cgroup, and every peer that opens the tier pins it once more. */
int pb_table_create_host_shared(int device, const pb_table_cfg* cfg, pb_table** out);
/* Both tables need their optimizer registered; checks dim, optimizer kind and row stride. */
int pb_table_attach_tier(pb_table* t, pb_table* tier);
/* The tier behind `t` (zeros without one): [0] entries it holds, [1] entries moved out of HBM into it, [2] entries
 * restored into HBM, [3] entries dropped: by its own sweep, or because neither table had a row for them (an eviction
 * victim or a pb_set_rows entry), [4] training restores refused for want of a free HBM row.  Synchronises `stream`. */
int pb_tier_stats(pb_table* t, uint64_t h_out[5], void* stream);
/* Moves the host-tier traffic of an upcoming training request off its critical path: the eviction check that request
 * would run (victims out to the tier), then every sign of d_ids the HBM table lacks and its tier holds back into a
 * free HBM row.  Values never change; only where entries live.  No tier: does nothing.
 * d_ids, h_slot_occ_off, h_prefix, n_slots and prefix_bit as pb_add_prefix: raw slot ids (hash-stacked where a slot
 * hash-stacks), prefixed here by slot (prefix 0 = taken as they are).  The check runs whenever the table has an
 * eviction policy, gated on low water as always, with keep = max(keep_batches, pending batches + 1); it does not count
 * as one of the request's every-`check_every` calls.  A staged row gets the current batch number (age 0: any check
 * before the request keeps it).  A sign that finds no free HBM row stays in the tier for the request's own restore.
 * Never admits a sign, never refreshes an HBM-resident one.  Runs on a fixed, small grid (it shares the GPU). */
int pb_tier_stage(pb_table* t, const uint64_t* d_ids, uint32_t n, const uint32_t* h_slot_occ_off,
                  const uint64_t* h_prefix, uint32_t n_slots, uint32_t prefix_bit, void* stream);
/* [0] signs moved into HBM by stages (also counted in pb_tier_stats[2]), [1] stage restores skipped for want of a
 * free HBM row (left to the request's own restore; NOT counted in pb_tier_stats[4]).  Since creation / clear; zeros
 * without a tier.  Synchronises `stream`. */
int pb_tier_stage_stats(pb_table* t, uint64_t h_out[2], void* stream);
/* ---- incremental updates: the signs stepped since the last take ---------------------------------------------------
 * The reference's parameter server hands every sign update_gradient_mixed stepped to its incremental-update manager,
 * which dumps the entries of the signs it collected once there are more than incremental_buffer_size of them
 * (embedding_parameter_service/mod.rs:366-424, persia-incremental-update-manager/src/lib.rs:251-312).  Here the set of
 * such signs lives on the device and the training calls fill it, after the optimizer step they report and on the same
 * stream (a captured step stays one graph):
 *   - pb_backward: every distinct (slot, sign) item of the batch whose slot was applied (d_slot_status 0) and that had a
 *     row (a gradient miss is not marked), once per call whatever the feature groups;
 *   - pb_backward_raw: the slot's distinct signs that had a row, if the request was applied;
 *   - pb_update: the signs it found, in HBM or in the host tier (a tier-held row is stepped in place and marked too);
 *   - pb_backward_sharded / pb_backward_raw_sharded: on the owner (PB_PHASE_SERVE), every received entry whose gradient
 *     was applied and that had a row.  Nothing is marked on the requesting side.
 * Lookups, admissions, pb_set_rows, tier moves and stages mark nothing.  A sign is held once however often it is marked.
 * A set that holds `capacity` signs drops further new signs and counts them (as the reference's full channel does,
 * mod.rs:415-423): a mark never blocks and never fails a step.  The set is keyed by sign, so a move between a table and
 * its tier never touches it; a tier has no set of its own.  A table that never enables one launches no extra kernel. */
/* Allocates the set (an open-addressing set of next_pow2(2 x capacity) cells of 16 B, counters in HBM, the held count
 * mirrored into one word of mapped pinned host memory), emptying any set the table had; capacity 0 frees it.
 * Synchronises the device. */
int pb_table_enable_incremental(pb_table* t, uint64_t capacity);
/* If the set holds at most max_n signs, writes them to d_signs (in no particular order) and empties the set, in one pass;
 * otherwise writes nothing and leaves the set as it is.  Either way *d_count = the signs held (max_n = 0 sizes the
 * buffer, as pb_table_export_signs).  Ordered after every mark issued before it and before every mark issued after it,
 * whatever their streams (the step chain, top of this file); the sharded owners' marks are ordered by the caller. */
int pb_inc_take(pb_table* t, uint64_t* d_signs, uint32_t max_n, uint32_t* d_count, void* stream);
/* [0] signs held, [1] signs inserted, [2] signs dropped because the set was full, [3] signs taken; since the set was
 * enabled.  Zeros without a set.  Synchronises `stream`. */
int pb_inc_stats(pb_table* t, uint64_t h_out[4], void* stream);
/* The held count as the last completed mark or take left it, read from host memory without synchronising: it may lag
 * the stream by the calls still in flight.  0 without a set. */
int pb_inc_held(pb_table* t, uint64_t* h_out);
/* Diagnostic: the state of the hash index's n_cells normal cells (the three cells reserved for the marker-valued signs
 * are not counted): [0] live (a resident sign), [1] tombstones (an evicted sign), [2] EMPTY.  An admission needs an
 * EMPTY cell on its probe path; every eviction check rebuilds the index (tombstones dropped) once fewer than 1/8 of the
 * cells are EMPTY.  Synchronises `stream`. */
int pb_table_index_stats(pb_table* t, uint64_t h_out[3], void* stream);
/* ---- growable storage: `capacity` bounds a table instead of reserving it ----------------------------------------
 * pb_table_set_growth(t, 1), before the table's first allocation (after it: PB_ERR_STATE; a host table refuses it with
 * PB_ERR_STATE), makes the table's storage grow with its entries.  Device address space is reserved for `capacity` rows
 * (rows, row recency, free-row stack, the rebuild's pairs) and for the largest index (next_pow2(1.5 x capacity) cells
 * + 3) through the driver's virtual memory calls; physical HBM backs it in chunks of the allocation granularity as
 * admissions reach it.  Before a call that can admit signs launches anything (training pb_forward, pb_forward_raw and
 * pb_lookup, pb_set_rows and so pb_image_insert, an owner's training PB_PHASE_SERVE: at most R x cap signs), the host
 * backs every row that call and the calls still in flight could hand out, by a bound it keeps without waiting for the
 * device (the last row count read back, plus the signs of every call issued since), growing by at least 1/8 of what is
 * mapped.  When the cells those rows and the used cells could take pass 2/3 of the index, the index is doubled in the
 * table's index chain: its live entries are re-inserted as an eviction check's rebuild does.  Rows never move, so
 * pending batches survive growth.  Results are bit for bit those of the same table without growth; the allocator never
 * hands out a row that is not backed (pb_table_storage_stats [3] counts such refusals and stays 0).  A chunk that
 * cannot be had fails the call with PB_ERR_CUDA before it launches any kernel or copy (only the event wait and record
 * that order it among the table's calls reach its stream); the table stays valid and a later call can grow it.  Eviction still works against `capacity`: running out of HBM never evicts.  A call enqueued under stream
 * capture first backs the whole capacity (a replay never passes through the host's bound).  A table of mode 1 cannot
 * be exported (pb_table_export_view, pb_table_export_live_view); no growable table can take a host tier
 * (pb_table_attach_tier): PB_ERR_STATE.  pb_debug_owned counts the bytes backed, not those reserved.  Memory is not
 * given back before the table is destroyed (pb_table_clear and eviction keep it).
 * Mode 2, exportable growth: as mode 1, but every chunk is created exportable as a POSIX file descriptor, and the
 * table can be exported, frozen or live (below: "Exportable growth").  Where the device does not report
 * CU_DEVICE_ATTRIBUTE_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR_SUPPORTED, or the driver lacks cuMemExportToShareableHandle /
 * cuMemImportFromShareableHandle, mode 2 is refused with PB_ERR_STATE and a message that says so.  `on`: 0 (off), 1 or
 * 2; anything else PB_ERR_INVALID. */
int pb_table_set_growth(pb_table* t, int on);
/* [0] rows reserved (capacity), [1] rows backed by memory (= capacity on a table without growth), [2] index cells,
 * [3] admissions refused because their row was not backed (must stay 0).  Before the first allocation [1..3] are 0.
 * Synchronises `stream`. */
int pb_table_storage_stats(pb_table* t, uint64_t h_out[4], void* stream);

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

/* ---- checkpoint images on the device ---------------------------------------------------------------------------------
 * The reference's parameter server dumps each internal shard's entries under that shard's read lock on a thread pool
 * while training goes on (persia-model-manager/src/lib.rs:286-343).  These calls write the bytes of such a file, the
 * speedy encoding of an ArrayLinkedList<HashMapEmbeddingEntry> (persia_b200/checkpoint.py), on the device:
 *   header = count u64 | first u32 | last u32 | free u32 (0) | end u32 (0) | n_nodes u32            (28 bytes)
 *   node i = next u32 (i + 2, 0 for the last) | prev u32 (i) | flag u8 (1) | len u32 | f32 x len | dim u64 | sign u64
 * (29 + 4 len bytes, len = embedding ++ optimizer state).  Entries are read in HBM or, through a host tier, in place in
 * its mapped host rows.  A host tier is dumped with the table it is attached to (calls on the tier itself are refused).
 * Both calls are in both chains (top of this file), like pb_get_rows: calls issued before them finish first, calls
 * issued after them start after them.  The sharded calls are outside the chains: on R GPUs the caller orders a dump
 * call against them (e.g. by issuing it on the stream its sharded calls use).
 *
 * The workspace (collection, sort and locations; about 60 B per entry plus the sort's temporary storage) is allocated
 * by pb_table_dump_reserve for images of up to max_bytes, replacing any earlier one, and freed by
 * pb_table_dump_release (or pb_table_destroy).  Both synchronise the device, touch nothing but the workspace and may
 * run on another host thread than the table's other calls (not beside a dump call on the same table). */
int pb_table_dump_reserve(pb_table* t, uint64_t max_bytes);
int pb_table_dump_release(pb_table* t);
/* One part of a background dump: the entries (HBM and tier, the three marker-valued signs included) whose sign has
 * part(sign) == part, where part(sign) = splitmix64(sign) % n_parts and
 *   splitmix64(x): z = x + 0x9E3779B97F4A7C15; z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9;
 *                  z = (z ^ (z >> 27)) * 0x94D049BB133111EB; return z ^ (z >> 31).
 * They are taken as they are at this call's point in the table's order and listed oldest first: last-use request
 * number ascending, ties by sign compared as an int64 (pb_table_export_signs' order).  Writes the part's whole image
 * (header and nodes) to d_image (16-byte aligned) and its size to *d_bytes; an image larger than max_bytes is not
 * written, only *d_bytes is set (as pb_inc_take does).  *d_request = the table's training-request number at that point.
 * No host synchronisation and no allocation: the entry count stays on the device (a table that was never allocated
 * gives the empty list without allocating it).  Needs a workspace reserved for max_bytes or more (else PB_ERR_INVALID). */
int pb_table_dump_part(pb_table* t, uint32_t part, uint32_t n_parts, void* d_image, uint64_t max_bytes,
                       uint64_t* d_bytes, uint32_t* d_request, void* stream);
/* The synchronous dump's slices: nodes [lo, lo + n) of a list of the n_list signs d_signs (the list order the caller
 * chose, e.g. pb_table_export_signs' sorted), without the header, to d_out (16-byte aligned; n * (29 + 4 len) bytes).
 * A sign no table holds gets zeros.  Needs a workspace reserved for n entries or more. */
int pb_dump_nodes(pb_table* t, const uint64_t* d_signs, uint32_t n_list, uint32_t lo, uint32_t n, void* d_out,
                  void* stream);

/* ---- checkpoint loads on the device ----------------------------------------------------------------------------------
 * The reference's server loads every `.emb` of its shard directory, one job per file, each decoded whole
 * (read_to_end_speedy) and inserted in list order (persia-model-manager/src/lib.rs:259-273, 375-425;
 * embedding_parameter_service/mod.rs:460-466); a re-sharding load keeps the entries with
 * farmhash64(sign) % R == rank (embedding_worker_service/mod.rs:1197-1259).  A pb_image indexes one list image (or a
 * window of whole nodes of one) that lies in pinned host memory (cudaHostAlloc, or any pinned buffer under unified
 * addressing): the kernels read it in place.  pb_image_insert then gathers selected entries into aligned staging and
 * stores them with pb_set_rows (so in both chains, HBM first, then the tier).  The image must stay unchanged until
 * the inserts that read it have run (e.g. an event recorded after them).
 *
 * Workspace (about 13 B per list position, the staging of max_chunk entries, and the host pass's 13 B per node) is
 * allocated by the index calls as they need it, in the order of their stream (cudaMallocAsync), and freed by
 * pb_image_destroy, which synchronises that stream only. */
typedef struct pb_image pb_image;
int pb_image_create(int device, uint32_t max_chunk, pb_image** out);
int pb_image_destroy(pb_image* im);
/* A whole image of any layout (free nodes, nodes out of list order, mixed entry lengths): node offsets, links and
 * list order from one sequential pass over it on the host, with checkpoint.decode_list's checks in its order
 * (PB_ERR_FORMAT with the first failure).  Then, on the device, the entries at list positions [p_lo, p_hi) with
 * farmhash64(sign) % R == rank are selected and counted per (dim, entry length): h_summary gets *h_rows rows
 * (dim, entry length, selected entries), at most max_rows (64 always suffice).  Synchronises `stream` once. */
int pb_image_index(pb_image* im, const void* h_image, uint64_t nbytes, uint32_t p_lo, uint32_t p_hi, uint32_t R,
                   uint32_t rank, uint64_t* h_summary, uint32_t max_rows, uint32_t* h_rows, void* stream);
/* A window of the writer layout (every file this library's dumps write): nodes [node0, node0 + n) of a file of n_total
 * nodes of entry_len floats, the window's bytes starting at its first node.  Each node's header is checked on the
 * device: next = i + 2 (0 for the last), flag 1, entry_len and dim.  *h_writer = 0 when one is not so (nothing of the
 * window may then be inserted: index the whole file instead); else the selection and summary as pb_image_index's.
 * Synchronises `stream` once. */
int pb_image_window(pb_image* im, const void* h_window, uint64_t node0, uint32_t n, uint64_t n_total, uint32_t entry_len,
                    uint64_t dim, uint32_t R, uint32_t rank, uint64_t* h_summary, uint32_t max_rows, uint32_t* h_rows,
                    int* h_writer, void* stream);
/* One incremental-update packet (persia_b200/incremental.py): count u32 | entry x count | unix seconds u64, each entry
 * len u32 | f32 x len | dim u64 | sign u64, lying in pinned host memory (as pb_image_index's image).  Its list positions
 * are the packet's entry order.  Checks, and their first failure, are decode_packet's: PB_ERR_FORMAT with
 * pb_last_error() = "ValueError: truncated packet" / "...: truncated packet: entry" / "...: packet length does not
 * match its entries".  Then the selection (farmhash64(sign) % R == rank) and the per-(dim, entry length) summary as
 * pb_image_index; *h_timestamp = the packet's timestamp.  Synchronises `stream` once; touches no table.  A well-formed
 * packet of more than 32 dims or 64 (dim, entry length) pairs gives PB_ERR_CAPACITY (nothing of it may be inserted).
 * A packet whose size is that of `count` entries of its first entry's length (every packet this library's flushes
 * write for one dim) is read at arithmetic offsets, each entry's `len` checked on the device; any other packet, or one
 * that fails that check, takes one sequential host pass over its length fields (and then twice the synchronisation). */
int pb_image_packet(pb_image* im, const void* h_packet, uint64_t nbytes, uint32_t R, uint32_t rank,
                    uint64_t* h_summary, uint32_t max_rows, uint32_t* h_rows, uint64_t* h_timestamp, void* stream);
/* set_embedding of the indexed image's selected dim-`dim` entries [lo, hi) (counted in list order, or from the end of
 * the list when newest_first, and offered in that order) into `t`, whose entry length they must have; hi - lo at most
 * max_chunk.  No host synchronisation. */
int pb_image_insert(pb_image* im, pb_table* t, uint64_t dim, uint32_t lo, uint32_t hi, int newest_first, void* stream);
/* Pinned host memory, mapped into every device's address space (cudaHostAlloc mapped | portable), for images; freed
 * by pb_host_free, not kept by any caching allocator once the load ends. */
int pb_host_alloc(uint64_t bytes, void** out);
int pb_host_free(void* p);

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

/* A context holds up to 2^24 id occurrences.  It allocates about 105 bytes per occurrence of max_occurrences and 4 per
 * output row when created (1.8 GB at 2^24), then, on first use, max_occurrences / 33 x dim f32 of hot-sign staging (a
 * training pb_forward) or 52 to 84 bytes per occurrence of raw scratch (pb_forward_raw).  A training pb_forward_raw
 * also keeps n_occ x dim f32 of gradient staging, sized by its batch and grown when a larger batch or dim comes; growing
 * synchronises the stream and frees the old buffer, so a raw step is capturable (and its graph replayable) only after a
 * batch at least as large has run on the context. */
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
 * batch; rows_f32 != 0 returns f32 rows (needed for ragged layouts, which pool on the requester; f16 otherwise).
 *
 * A shard may have a host tier (pb_table_attach_tier): R GPUs then hold R x (HBM + tier) entries.  Its owner serves the
 * requests it receives as one GPU serves its own (PB_PHASE_SERVE of the summation and raw forwards alike): a training
 * request's tier-held signs are first moved into free HBM rows (a sign that finds none stays in the tier, reads zeros,
 * takes no gradient and counts in pb_tier_stats[4]); an inference request (training == 0) reads them in place and moves
 * nothing.  The eviction check in each rank's SEND moves its own shard's victims into its tier, and the backwards step
 * only HBM rows: the rows of pending requests are never victims.  Nothing else changes: no host synchronisation, and a
 * step stays capturable.  A requester cannot tell a tiered owner from an untiered one. */
typedef struct pb_xchg pb_xchg;
uint64_t pb_xchg_bytes(uint32_t R, uint32_t cap, uint32_t dim, int rows_f32);
int pb_xchg_create(int device, uint32_t R, uint32_t rank, uint32_t cap, uint32_t dim, int rows_f32,
                   const uint64_t* h_peer_base, pb_xchg** out);
/* Replacing an exchange (e.g. by one of a larger cap, or with f32 rows): an exchange keeps nothing across steps but its
 * phase epochs, which live in it and in its area, and a cache of the table's feature-group prefixes; the Adam beta powers,
 * the rows and the incremental set live in the pb_table.  So the ranks may destroy their exchanges and create new ones
 * (zero-initialised areas) collectively, at a step boundary — after the last step that used the old ones has completed
 * on every rank and before any rank calls the next — and the table, its Adam powers and its incremental set are
 * unaffected.  A context's prepared batch (PB_PHASE_PREPARE) survives the replacement. */
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
/* Forwards only, never part of phases = 0: requester, local work only — the forward's per-slot dedup (summation call)
 * or the slot's distinct-sign numbering (raw call), then the batch's distinct (slot, sign) items per owner
 * farmhash64(sign) % R, for pb_xchg_need.  Raises no flag, stores into no peer's area and reads or writes no table
 * state (no eviction check, no request number, no probe); the context's previous batch goes, as in SEND.  A ragged
 * batch may be prepared on an f16 exchange.  A later call with PB_PHASE_SEND on the same context and the same ids
 * reuses the prepared work and then runs SEND's table part as always: eviction check, request number, route, link,
 * signal (a different n_occ or batch: PB_ERR_STATE).  Between the two the caller may replace the exchange (see
 * pb_xchg_destroy) so that its cap covers pb_xchg_need; that is how a step is sized from its own batch. */
#define PB_PHASE_PREPARE 8
/* h_out[0] = the most items the context's prepared batch sends to one owner (what cap must hold).  Synchronises
 * `stream`.  PB_ERR_STATE without a prepared batch (its SEND consumes it). */
int pb_xchg_need(pb_xchg* x, pb_ctx* c, uint32_t h_out[1], void* stream);
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

/* ---- staging on R GPUs: the next batch's host-tier moves one step early --------------------------------------------
 * pb_tier_stage on R GPUs.  A rank's next batch asks for signs that its owners hold, so its stage needs those signs at
 * the owners a step early.  A stage exchange carries them: an exchange with a ctrl and a sign part only (no rows,
 * gradients or chain words; no owner-side set or Adam arrays).  Its area is pb_xchg_stage_bytes(R, cap) bytes of
 * zero-initialised device memory that all ranks can store to, mapped as for pb_xchg_create:
 *   [0, 512)          ctrl: XC_WORDS (5) x 16 u32 flag and count words (as a batch exchange's)
 *   [512, 512 + S)    sign: R x cap u64, the signs each source stages here, by source; S = R x cap x 8 rounded up to 256
 * pb_xchg_stage_bytes returns 0 for R = 0, R > 16, cap = 0 or R x cap >= 2^32 - 16.  cap: the most signs one rank sends
 * one owner in one stage.  pb_xchg_destroy frees a stage exchange and pb_xchg_status reads it: h_out[0] != 0 when a
 * stage had more than cap signs for one owner (the excess was not sent; the forward restores it as unstaged), h_out[1]
 * as for a batch exchange.  The sharded forwards and backwards refuse a stage exchange (PB_ERR_INVALID), and
 * pb_tier_stage_sharded refuses a batch exchange (PB_ERR_INVALID).
 *
 * pb_tier_stage_sharded: arguments as pb_tier_stage (raw slot ids, slot offsets, per-slot prefixes, 0 = taken as they
 * are) plus the stage exchange and `phases`: PB_PHASE_SEND, PB_PHASE_SERVE or both (0 = both; PB_PHASE_FINISH and
 * PB_PHASE_PREPARE are refused, PB_ERR_INVALID).  Virtual ranks of one GPU enqueue SEND for every rank, then SERVE.
 *   SEND (requester)  every id slot-prefixed, its owner farmhash64 % R, duplicates inside a warp dropped, the sign
 *                     stored into the owner's stage area; then the flag.
 *   SERVE (owner)     waits for the R flags; with a host tier, runs the eviction check pb_tier_stage runs (not counted
 *                     as one of the every-`check_every` calls; keep = max(keep_batches, pending batches + 1); victims
 *                     out to the tier), then moves every received sign the HBM table lacks and its tier holds into a
 *                     free HBM row, stamped with the current batch number.  Never admits a sign.  A sign that finds no
 *                     free row is counted as a skipped stage and left to the forward.  Counters: pb_tier_stage_stats of
 *                     the owner's table.  An owner without a tier waits for and consumes the flags and moves nothing.
 * Values never change, only where entries live, and a sign the stage did not move is restored by the forward exactly
 * as unstaged: a staged run equals the unstaged one bit for bit.
 * Rules: the call is collective, like the other sharded calls, and outside the table's chains: the caller orders it.
 *   - A rank's stage starts after its previous training forward (every phase) has completed, and its next sharded
 *     forward on the table starts after the stage has completed.  Refused on a host tier (PB_ERR_STATE) and on a table
 *     exported for remote reads (pb_table_export_view: PB_ERR_STATE).
 *   - It may run beside the sharded backwards, summation and raw alike, on another stream: no owner-side backward kernel
 *     (k_owner_update_all, k_owner_update, the raw owner path, which is the same, and the Adam beta-power advance)
 *     reads index cells, the free-row stack or row_tick.  They step only the rows their forward found, by the row
 *     numbers it stored; those rows are never victims (their age is below keep) nor restore targets (those come off
 *     the free stack), and the incremental marks read the exchange, not the index.
 *   - A stage area is never rewritten while its owner still reads the previous stage: rank r's stage i+1 starts after
 *     r's forward i, which waited for every owner's SERVE of forward i, and each owner's forward i started after its
 *     own stage i had completed.  One area per rank therefore suffices.
 *   - No host synchronisation: a step with a stage, the stage forked onto a side stream, is capturable in one graph. */
uint64_t pb_xchg_stage_bytes(uint32_t R, uint32_t cap);
int pb_xchg_create_stage(int device, uint32_t R, uint32_t rank, uint32_t cap, const uint64_t* h_peer_base, pb_xchg** out);
int pb_tier_stage_sharded(pb_table* t, pb_xchg* xs, const uint64_t* d_ids, uint32_t n, const uint32_t* h_slot_occ_off,
                          const uint64_t* h_prefix, uint32_t n_slots, uint32_t prefix_bit, void* stream, int phases);

/* ---- inference on R GPUs one rank at a time: reading the owners' shards in place --------------------------------------
 * The reference's Infer handlers each call get_embedding_from_bytes on their own requests, and the embedding servers
 * answer each request alone (persia/ctx.py:1077-1135, embedding_parameter_service/mod.rs:162-262).  The sharded calls
 * above are collective instead: every rank must call them in the same step.  For inference the requesting GPU does the
 * owner's part itself: it probes each owner's index and reads its rows through a peer mapping (CUDA IPC or, in one
 * process, the pointers themselves).  No flag, no collective, no kernel on the owner: one rank serves its request
 * while its peers are idle.
 *
 * Read-only rule: from pb_table_export_view on, for the rest of its life, the table refuses with PB_ERR_STATE, before
 * enqueuing anything, every call that moves index cells or steps rows: training forms of pb_forward, pb_forward_raw,
 * pb_lookup and the sharded forwards; pb_backward, pb_backward_raw and the sharded backwards; pb_update; pb_table_clear;
 * pb_tier_stage (an eviction check) and pb_table_attach_tier.  pb_set_rows and pb_image_insert stay allowed (an Infer
 * job applies checkpoint loads and incremental packets with them), as do inference forwards, reads, statistics and
 * dumps.  The owner cannot know when a peer closes its view, so there is no way back: export a table only to serve it.
 * Consistency rule: the exported table keeps a write-sequence word in its HBM.  pb_set_rows raises it to odd before its
 * writes and back to even after them (one-thread kernels with system-scope fences, on the call's stream).  A remote
 * read checks each owner's word before and after it probes and copies an item, and reads the item again while the
 * word is odd or if it changed (a row still being published counts the same).  So a returned row is an entry as it
 * was before an insert or after it, never a mix, as the reference's entry lock gives.  A read that is still waiting
 * after the sharded calls' wait budget gives up and counts in the reader's pb_table_counters[4].
 * Ownership rule: the owner outlives every view of its table (destroy views first; a view of a destroyed table reads
 * freed memory).  A tier cannot be exported on its own, nor a table with a tier from pb_table_create_host (no peer can
 * reach its rows).  A table with a shared tier (pb_table_create_host_shared) can: see "Shared tiers" below. */
/* Bytes of a view blob (fixed: the exporting pid and a random number drawn once per process, the device pointers and CUDA IPC handles of the index cells, rows,
 * counters and write-sequence word, and the table's geometry). */
uint64_t pb_table_view_bytes(void);
/* Writes t's view blob to h_blob (pb_table_view_bytes() bytes) and makes t read-only (above).  Allocates the table if
 * needed (so the optimizer must be registered) and synchronises the device the first time. */
int pb_table_export_view(pb_table* t, void* h_blob);
/* The live export: the same blob, opened by pb_view_open and read by pb_forward_remote / pb_forward_raw_remote as they
 * are, but t stays writable: training forwards and backwards, pb_update, eviction checks, pb_set_rows, pb_table_clear,
 * dumps and loads all run.  So a training job serves its forwards that do not train one rank at a time.
 * Live consistency rule: the write-sequence word is odd from before the first cell to after the last row each of these
 * changes: a capacity sweep (tombstones cells, frees rows the next admission gives to another sign), an index rebuild
 * (cells go EMPTY and are re-inserted), pb_table_clear and pb_set_rows.  The sweep and the rebuild move it inside the
 * eviction check's own kernels (no launch is added; a captured step stays one graph with no host sync).  So a read never
 * returns another sign's row, and a sign resident before and after the read is never a false miss.  The word does not
 * cover an admission (the index publishes a row only once it is initialised; a reader waits on an unpublished one) nor
 * an optimizer step on a resident row: a read beside a step returns, per element, the value before or after that step,
 * the stale read a forward beside a backward on one GPU may give too.  A read that waits out the budget counts in
 * the reader's pb_table_counters[4] and reads zeros.  A table is exported one way only (the other call: PB_ERR_STATE);
 * the host-tier refusals and the ownership rule are the frozen export's, and a live table refuses pb_table_attach_tier. */
int pb_table_export_live_view(pb_table* t, void* h_blob);
typedef struct pb_view pb_view;
/* A view of an exported table for reads issued on `device`.  A blob of another process: each handle is opened with
 * cudaIpcOpenMemHandle(cudaIpcMemLazyEnablePeerAccess); of this process: its pointers are used as they are (peer access
 * is enabled when the table lives on another device); a blob is this process's own when both its pid and its random number
 * are this process's (pids alone repeat across PID namespaces).  pb_view_close synchronises `device` and closes the handles. */
int pb_view_open(int device, const void* h_blob, pb_view** out);
int pb_view_close(pb_view* v);
/* ---- Shared tiers: reading a tiered owner in place ------------------------------------------------------------------
 * A table with a tier from pb_table_create_host_shared exports, frozen or live, a view blob of the same size and layout
 * marked as tiered (version 2), which pb_view_open refuses (PB_ERR_STATE): a reader that ignored the tier would read
 * zeros for every tier-held sign.  The tier's part is a second fixed-size blob, pb_table_export_tier_view's, written
 * after the table's export: the exporting pid and random number, the device pointer and CUDA IPC handle of the tier's
 * index cells, the memfd number and byte size of its rows, and its geometry (n_cells, capacity, stride).
 * pb_view_open_tiered opens both: from this process it uses the pointers as they are; from another it opens the cells'
 * handle, then /proc/<pid>/fd/<fd>, checks the size with fstat, maps it MAP_SHARED and registers it mapped (read-only,
 * PROT_READ and cudaHostRegisterReadOnly, where the device supports it: a reader never writes the owner's rows).  Where that
 * open fails (ranks in other PID namespaces or of other users, an owner that is not dumpable) it returns PB_ERR_STATE
 * and says why.  pb_forward_remote and pb_forward_raw_remote then probe an owner's tier where its HBM index misses and
 * read the hit from the host row (a kernel of its own, launched only when some owner has a tier): outputs stay bit for
 * bit the sharded inference forwards', and only a sign neither table holds counts as a miss, on its owner.  `own` may
 * have a shared tier too.
 * Consistency: one write-sequence word covers a table and its tier.  Frozen: pb_set_rows (so pb_image_insert) holds it
 * odd from before its restores to after its tier inserts.  Live: pb_table_clear holds it odd across the tier's clear
 * too, and every launch that moves an entry between the two tables or hands a row of either to another sign runs
 * inside a window of two added one-thread launches (k_seq_begin before it, k_seq_end after it): each eviction check
 * (threshold, the tier's drop sweep, the move, both rebuilds); each restore (pb_forward, pb_forward_raw and pb_lookup
 * training requests; an owner's SERVE of a training pb_forward_sharded / pb_forward_raw_sharded); pb_tier_stage's
 * restores and pb_tier_stage_sharded's SERVE restores, each beside the window of the eviction check it runs.  So a
 * live tiered training step adds 2 launches per restore it makes and 2 per eviction check it runs, and nothing else;
 * untiered tables, tables with a private tier and tables not exported launch what they launched before.  Optimizer
 * steps on tier-held rows stay outside the word: a read beside one sees each element before or after it, as for HBM
 * rows. */
/* Bytes of a tier blob (fixed). */
uint64_t pb_tier_view_bytes(void);
/* Writes the tier blob of t's shared tier (pb_tier_view_bytes() bytes).  t must have been exported (either way) first;
 * a table without a tier, or with a tier from pb_table_create_host, and a tier itself: PB_ERR_STATE. */
int pb_table_export_tier_view(pb_table* t, void* h_blob);
/* pb_view_open for a tiered view blob and its tier blob (above).  Blobs of different exports: PB_ERR_INVALID. */
int pb_view_open_tiered(int device, const void* h_blob, const void* h_tier_blob, pb_view** out);
/* ---- Exportable growth: reading a growing owner in place -----------------------------------------------------------
 * A table of growth mode 2 exports, frozen or live, a view blob of the same size and layout marked version 3: the
 * handle slots of its cells and rows hold the spans the owner reserved for them instead (no IPC handle describes a
 * reservation backed chunk by chunk), and its write-sequence word has a second word after it, the index's current cell
 * count.  pb_view_open opens it.  From the owner's process the view uses the owner's pointers.  From another it opens
 * the counters and the word through CUDA IPC, reserves the same spans in its own address space, and listens on an
 * abstract-namespace AF_UNIX socket (pb_view_address).  The owner registers that address (pb_table_add_reader) and
 * sends over it, with SCM_RIGHTS, the descriptor, region, offset and size of every chunk of its rows and cells mapped so
 * far, then of each new one, right after mapping it and before any kernel that can use it is enqueued.  Sends never
 * block: one that would is kept and retried by the table's next call that can grow it.  A reader imports each chunk
 * and maps it read-only (where the driver allows; else read-write) at the same offset of its reservation, at the start
 * of every remote call; each descriptor is closed once imported, and pb_view_close unmaps and releases them all.
 * Geometry: an index doubling moves every cell, so the exported table holds its write-sequence word odd around each
 * doubling (in both export modes) and publishes the new cell count before the word is even again.  A remote read reads
 * the count inside its window and probes with it.  It never touches an address its process has not mapped: an item
 * whose owner's count (and 3 reserved cells) pass the cells mapped here, or whose row is at or above the rows mapped
 * here, is stale, not read.  The call then copies the count of stale items to the host (one synchronisation of its
 * stream per call, only when some owner is another process's growable table), imports what has arrived and reads the
 * stale items again, waiting for a missing chunk for up to 20 s; still stale then, it fails with PB_ERR_STATE, and no
 * output is written.  That synchronisation rules out stream capture: such a call under capture fails with
 * PB_ERR_STATE before it launches anything (views in the owner's process and eager owners capture as before).  A kept
 * send is retried only by the owner's next call that can grow the table (a training forward, an owner's SERVE,
 * pb_set_rows, pb_image_insert): an owner that makes no such call again (a frozen Infer owner done loading) leaves a
 * kept chunk unsent, and a reader that needs it fails after the wait.  Outputs are bit for bit those of the same reads
 * of eager owners.  Owners with exportable growth
 * and owners with shared tiers cannot be read in one call (PB_ERR_STATE). */
/* The abstract socket name (without its leading NUL) a view of another process's growable table listens on, as a
 * string in h_out (cap bytes); "" for every other view (nothing to register). */
int pb_view_address(const pb_view* v, char* h_out, uint64_t cap);
/* Registers a reader of t (a table of growth mode 2, exported either way) by its view's address (pb_view_address) and
 * sends it every chunk mapped so far; "" does nothing.  The view must be open (else PB_ERR_STATE, and why).  A reader
 * whose view has closed is dropped at the next send. */
int pb_table_add_reader(pb_table* t, const char* addr);
/* The inference form (training == 0) of pb_forward_sharded, served by this rank alone: arguments as pb_forward, plus
 * views[R] (owner q's table; views[rank] may be NULL: `own`, this rank's table, is probed directly), R and rank.  The
 * batch's distinct (slot, sign) items are read from their owners farmhash64(sign) % R into staging the context owns
 * (n_occ x dim f32 at most, grown like pb_forward_raw's staging: a call is capturable in a CUDA graph, and no host sync
 * or allocation happens, once a batch at least as large ran on the context), then pooled by the sharded path's own
 * kernels.  Outputs are bit for bit pb_forward_sharded(training = 0)'s on the same tables and batch; a sign no owner
 * holds reads as zeros and counts as a lookup miss on its owner (pb_table_counters[1], a system-scope atomic through the
 * view).  `own` is in its own index chain; the owners' calls are ordered only by the consistency rule. */
int pb_forward_remote(pb_table* own, pb_view* const* views, uint32_t R, uint32_t rank, pb_ctx* c, const uint64_t* d_ids,
                      uint32_t n_occ, const uint32_t* d_row_off, const uint32_t* h_slot_occ_off, uint32_t batch,
                      void* d_out_f16, void* stream);
/* The same for a raw slot: arguments and outputs as pb_forward_raw plus views, R and rank; bit for bit
 * pb_forward_raw_sharded(training = 0)'s: row u+1 is f16(row), rounded once. */
int pb_forward_raw_remote(pb_table* own, pb_view* const* views, uint32_t R, uint32_t rank, pb_ctx* c,
                          const uint64_t* d_ids, uint32_t n_occ, const uint32_t* d_row_off, uint32_t batch,
                          uint32_t sample_fixed_size, void* d_table_f16, int64_t* d_index, int64_t* d_non_empty,
                          uint32_t* d_sample_id_num, uint32_t* d_counts, void* stream);

/* Number of kernels the library has launched on behalf of the caller since load (bench bookkeeping). */
uint64_t pb_launch_count(void);
/* Diagnostic: the geometry the backward gives its reduce of hot signs (> 32 occurrences) for rows of `dim` columns
 * (1..4096), f16 or f32 gradients, and a batch with several ids per sample in some slot (ragged) or one id per sample
 * in every slot.  Host-only, no device needed.  h_out: [0] EPL columns per chain lane, [1] CH chain warps, [2] PW
 * producer warps, [3] 16-byte producer loads (else element by element), [4] log2 of the 16-byte vectors per row when
 * that is a power of two (else 32), [5] the producers' lean loop, [6] R1 rows per producer part, [7] R rows per ring
 * slot, [8] S ring slots, [9] columns per pass, [10] floats per ring row, [11] column passes. */
int pb_hot_geometry(uint32_t dim, int is_f16, int ragged, uint32_t h_out[12]);
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
