// pb_remote.cu — inference on R GPUs one rank at a time (pb_forward_remote / pb_forward_raw_remote).
//
// Reference: an Infer job's handlers each call get_embedding_from_bytes on their own requests (persia/ctx.py:1077-1135),
// and the embedding servers answer each lookup_mixed alone (embedding_parameter_service/mod.rs:162-262, 344-357).  The
// collective path (pb_shard.cu) needs every rank in the same step.  Inference is read-only, and each owner's index and
// rows are one NVLink hop away, so here the requester does the owner's part itself:
//   k_remote_lookup  (requester) every distinct item of the batch: owner = farmhash64(sign) % R, a MODE_FIND probe of
//                    that owner's index through the view (pb_probe.cuh), the row read through the peer mapping and
//                    written, converted as k_owner_lookup converts it, to the context's staging at the item's number
// then the collective path's own pooling (k_expand_copy / k_expand_pool, or k_raw_fill for a raw slot) reads the
// staging.  No flag, no peer kernel, no collective.
//
// Consistency with writes: the owner keeps a write-sequence word, odd while an insert runs (pb_set_rows on an exported
// table) and, on a table exported live that keeps training, while a capacity sweep, an index rebuild (pb_index.cu) or a
// clear runs.  A lane group reads it before its probe and copy and again after them; while it is odd, or if it
// changed, the item is read again.  A returned row is therefore the entry before an insert or after it, never a mix.
// A row still ROW_PENDING in the index is an insert in flight: the word has moved, so it is read again as well.
//
// An owner with a shared host tier (pb_table_create_host_shared, pb_view_open_tiered): k_remote_lookup<TIER> probes the
// tier's index (HBM, through the view) where the owner's HBM probe misses, and reads a hit from the tier's host row (the
// owner's memfd, mapped into this process and registered with CUDA).  One word covers the table and its tier: the owner
// holds it odd around every launch that moves an entry between the two or hands a row of either to another sign
// (pb_api.cuh, TierWindow), so a reader never finds a moving sign in neither table, and a tier-held row read between two
// equal even words is that sign's whole row.  The loads between the two reads of the word are the same for both tables:
// the word is read with ld.acquire.sys (no later load of this thread is performed before it), the index and row loads
// are plain weak ld.global.cg (whether the row sits in peer HBM over NVLink or in host memory over PCIe: the PTX memory
// model orders by address, not by where the address lives), and fence.acq_rel.sys orders every one of them before the
// second ld.acquire.sys.  The owner's side is the converse: its k_seq_begin store is followed by fence.sc.sys
// (__threadfence_system) before the kernels that write cells or rows, and k_seq_end puts one between them and its store.
// At .sys scope those fences and the reader's acquire/fence pair synchronise, whichever GPU or PCIe path carries the
// data: a reader that reads the same even word twice read no row written inside a window.
//
// An owner with exportable growth (pb_table_set_growth(t, 2)): its rows and cells are chunks this process maps as they
// arrive (pb_api_view.cu), and its index doubles under the readers.  k_remote_lookup<GROW> reads the owner's cell
// count from the word after its sequence word, inside the same window (the owner publishes it inside the window that
// holds the doubling), and probes with that geometry.  It touches no address this process has not mapped: an item is
// stale, not read, when that count and the reserved cells pass the cells mapped here, or when the row found is at or
// above the rows mapped here.  The caller imports what has arrived and reads the stale items again.
#include "pb_device.cuh"
#include "pb_probe.cuh"

#include <type_traits>

namespace pb {

#ifndef PB_WAIT_SPINS
#define PB_WAIT_SPINS (1u << 25)  // (pb_shard.cu's wait budget)
#endif

__device__ __forceinline__ uint32_t seq_acquire(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// the loads of a probe and copy complete before the word is read again (the seqlock reader's read barrier)
__device__ __forceinline__ void fence_acq_rel_sys() { asm volatile("fence.acq_rel.sys;" ::: "memory"); }

__device__ __forceinline__ const RemoteDev& remote_of(const RemoteDev& a) { return a; }
__device__ __forceinline__ const RemoteDev& remote_of(const RemoteTierDev& a) { return a.rv; }
__device__ __forceinline__ const RemoteDev& remote_of(const RemoteGrowDev& a) { return a.rv; }
template <bool TIER, bool GROW>
using RemoteArg = typename std::conditional<TIER, RemoteTierDev,
                                            typename std::conditional<GROW, RemoteGrowDev, RemoteDev>::type>::type;

// One lane group (BUCKET lanes) per distinct item; the grid strides over the items.  Must be called by whole warps.
// TIER: a miss in the owner's HBM index is probed again in the owner's host tier (a.tier[owner]; cells null: it has none).
// GROW (never with TIER: a growable table has no tier): the owners' geometry and this process's mapped extents
// (RemoteGrowDev).
template <bool RAW, bool ROW_F32, bool TIER, bool GROW>
__global__ void __launch_bounds__(256, PB_PROBE_BLOCKS) k_remote_lookup(RemoteArg<TIER, GROW> a, BatchDev b, RawWork w,
                                                                         void* __restrict__ stage, uint32_t dim,
                                                                         uint32_t* __restrict__ err) {
  static_assert(!(TIER && GROW), "a growable table has no host tier");
  const RemoteDev& rv = remote_of(a);
  const uint32_t sub = threadIdx.x % BUCKET;
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t gshift = lane & ~(BUCKET - 1);
  const uint32_t groups = gridDim.x * (blockDim.x / BUCKET);
  const uint32_t n_items = RAW ? w.counts[0] : b.cnt[BC_ITEMS];
  const uint32_t warp_first = ((blockIdx.x * blockDim.x + threadIdx.x) / 32) * (32 / BUCKET);
  const HyperDev hy{};  // (a find neither admits nor initialises)
  const OptimDev op{};
  for (uint32_t j0 = warp_first; j0 < n_items; j0 += groups) {  // uniform per warp
    const uint32_t u = j0 + lane / BUCKET;
    bool valid = u < n_items;
    uint64_t sign = 0;
    uint32_t cell = 0;
    if (valid) {
      if (RAW) {
        sign = w.set[w.distinct_cell[u]].key;  // (as k_raw_route reads it)
      } else {
        cell = b.item_cell[u];  // (as k_route_items reads it)
        const uint4 lo = *reinterpret_cast<const uint4*>(&b.set[cell]);
        const uint4 hi = *(reinterpret_cast<const uint4*>(&b.set[cell]) + 1);
        sign = (hi.w >> 31) ? KEY_EMPTY : ((uint64_t)lo.x | ((uint64_t)lo.y << 32));
      }
      if constexpr (GROW) {
        if (a.only_stale) valid = (RAW ? w.target[u] : b.set[cell].target) == ROW_STALE;
      }
    }
    const uint32_t owner = valid ? (uint32_t)(farmhash64_u64(sign) % rv.R) : 0u;  // sign_to_shard_modulo, mod.rs:341-345
    const TableDev& t = rv.t[owner];
    const uint32_t* seq = rv.seq[owner];
    TableDev tg;  // GROW: the owner's table at the geometry it published
    if constexpr (GROW) tg = t;
    bool todo = valid;
    uint32_t spins = 0;
    while (__any_sync(0xffffffffu, todo)) {
      // every lane reads the word with acquire semantics itself, so that its own probe and row loads are ordered after
      // that read; the group acts on its first lane's value, and each lane checks its own read against it below
      uint32_t s0 = 0;
      if (todo && seq) s0 = seq_acquire(seq);
      const uint32_t s0_lead = __shfl_sync(0xffffffffu, s0, gshift);
      const bool go = todo && !(s0_lead & 1u);  // odd: an insert is running on the owner
      bool stale = false;
      if constexpr (GROW) {
        // the cell count the owner published, read after the word (ordered by its acquire); the group probes with
        // its first lane's, and a doubling between the two reads of the word shows as a changed word
        const uint32_t* geo = a.geo[owner];
        uint32_t nc = 0;
        if (go && geo) nc = *reinterpret_cast<const volatile uint32_t*>(geo);
        nc = __shfl_sync(0xffffffffu, nc, gshift);
        if (geo) {
          stale = (uint64_t)nc + N_SPECIAL > a.cells[owner] || nc < BUCKET || (nc & (nc - 1));
          if (!stale) {
            tg.n_cells = nc;
            tg.cell_mask = nc - 1;
            tg.bucket_mask = nc / BUCKET - 1;
          }
        }
      }
      const ProbeOut r = probe_group<MODE_FIND>(GROW ? tg : t, hy, op, sign, go && !stale, 0u, sub, gshift);
      if constexpr (GROW) stale = stale || (a.geo[owner] && r.row < t.capacity && r.row >= a.rows[owner]);
      // k_owner_lookup_tier's choice: the HBM row, else the tier row, else zeros
      const float* src = t.rows;
      uint32_t src_row = r.row, src_cap = t.capacity, src_stride = t.stride;
      if constexpr (TIER) {
        const TableDev& h = a.tier[owner];
        const ProbeOut tr = probe_group<MODE_FIND>(h, hy, op, sign, go && r.row >= t.capacity && h.cells, 0u, sub, gshift);
        if (r.row >= t.capacity && h.cells) {
          src = h.rows;
          src_row = tr.row;
          src_cap = h.capacity;
          src_stride = h.stride;
        }
      }
      const bool have = src_row < src_cap;
      if (go && !stale) {
        // k_owner_lookup's conversion: f16(0 + row) for one-id layouts, the f32 row for ragged ones (zeros on a miss)
        const float* row = src + (size_t)(have ? src_row : 0u) * src_stride;
        if (dim % 4 == 0) {
          for (uint32_t e = sub * 4; e < dim; e += BUCKET * 4) {
            const float4 v = have ? __ldcg(reinterpret_cast<const float4*>(row + e)) : make_float4(0.f, 0.f, 0.f, 0.f);
            if (ROW_F32) {
              *reinterpret_cast<float4*>(static_cast<float*>(stage) + (size_t)u * dim + e) = v;
            } else {
              __half2 a2 = __floats2half2_rn(__fadd_rn(0.0f, v.x), __fadd_rn(0.0f, v.y));
              __half2 c = __floats2half2_rn(__fadd_rn(0.0f, v.z), __fadd_rn(0.0f, v.w));
              uint2 pk;
              pk.x = *reinterpret_cast<uint32_t*>(&a2);
              pk.y = *reinterpret_cast<uint32_t*>(&c);
              *reinterpret_cast<uint2*>(static_cast<__half*>(stage) + (size_t)u * dim + e) = pk;
            }
          }
        } else {
          for (uint32_t e = sub; e < dim; e += BUCKET) {
            const float v = have ? __ldcg(row + e) : 0.0f;
            if (ROW_F32) static_cast<float*>(stage)[(size_t)u * dim + e] = v;
            else static_cast<__half*>(stage)[(size_t)u * dim + e] = __float2half_rn(__fadd_rn(0.0f, v));
          }
        }
      }
      // every lane's loads of the probe and the copy complete before that lane reads the word again
      uint32_t s1 = s0;
      if (go && seq) {
        fence_acq_rel_sys();
        s1 = seq_acquire(seq);
      }
      const uint32_t same = __ballot_sync(0xffffffffu, !go || (s0 == s0_lead && s1 == s0_lead));
      if (go && ((same >> gshift) & 0xFFu) == 0xFFu) {  // the item read whole by every lane, between two inserts
        if (sub == 0) {
          if (stale) {  // (GROW: read again once this process has mapped more of the owner's chunks)
            if constexpr (GROW) atomicAdd(a.stale, 1u);
          } else if (!have) {
            atomicAdd_system(&t.counters[CTR_MISS], 1u);  // counted on its owner, as there
          }
          const uint32_t to = stale ? ROW_STALE : u;
          if (RAW) w.target[u] = to;
          else b.set[cell].target = to;
        }
        todo = false;
      } else if (todo && ++spins > PB_WAIT_SPINS) {  // the owner never finished its insert: give up, and say so
        if (sub == 0) {
          atomicAdd(err, 1u);
          if (RAW) w.target[u] = ROW_NONE;  // (the item reads as zeros: its staging slot may hold a torn row)
          else b.set[cell].target = ROW_NONE;
        }
        todo = false;
      }
    }
  }
}

void launch_remote_lookup(bool raw, bool row_f32, const RemoteDev& rv, const TableDev* tiers, const RemoteGrowDev* grow,
                          const BatchDev& b, const RawWork& w, uint32_t n, void* stage, uint32_t dim, uint32_t* err,
                          cudaStream_t st) {
  if (!n) return;
  const uint32_t full = cdiv((uint64_t)n * BUCKET, 256);  // worst case: every id a distinct item
  const uint32_t grid = full < PB_NUM_SMS * PB_PROBE_BLOCKS ? full : PB_NUM_SMS * PB_PROBE_BLOCKS;
#define PB_R(RW, F32, TR, GR, A) \
  PB_LAUNCH_F(FAM_PROBE, (k_remote_lookup<RW, F32, TR, GR>), grid, 256, 0, st, A, b, w, stage, dim, err)
  if (tiers) {
    RemoteTierDev a;
    a.rv = rv;
    for (uint32_t q = 0; q < PB_MAX_RANKS; ++q) a.tier[q] = tiers[q];
    if (raw) PB_R(true, true, true, false, a);
    else if (row_f32) PB_R(false, true, true, false, a);
    else PB_R(false, false, true, false, a);
  } else if (grow) {
    RemoteGrowDev a = *grow;
    a.rv = rv;
    if (raw) PB_R(true, true, false, true, a);
    else if (row_f32) PB_R(false, true, false, true, a);
    else PB_R(false, false, false, true, a);
  } else {
    if (raw) PB_R(true, true, false, false, rv);
    else if (row_f32) PB_R(false, true, false, false, rv);
    else PB_R(false, false, false, false, rv);
  }
#undef PB_R
}

// the owner's side of the sequence word: one thread, on the table's stream, around the writes of a pb_set_rows
__global__ void k_seq_begin(uint32_t* seq) {
  *reinterpret_cast<volatile uint32_t*>(seq) = *seq + 1u;  // odd: readers wait
  __threadfence_system();  // ... before any entry of the insert is written
}
__global__ void k_seq_end(uint32_t* seq) {
  __threadfence_system();  // every entry written before
  *reinterpret_cast<volatile uint32_t*>(seq) = *seq + 1u;  // even again
}
// the end of an index doubling's window (exportable growth): the new cell count, then the word even again
__global__ void k_seq_end_cells(uint32_t* seq, uint32_t cells) {
  __threadfence_system();  // every cell written before
  reinterpret_cast<volatile uint32_t*>(seq)[1] = cells;
  __threadfence_system();
  *reinterpret_cast<volatile uint32_t*>(seq) = *seq + 1u;
}
void launch_seq_bump(uint32_t* seq, bool begin, cudaStream_t st, uint32_t cells) {
  if (begin) PB_LAUNCH(k_seq_begin, 1, 1, 0, st, seq);
  else if (cells) PB_LAUNCH(k_seq_end_cells, 1, 1, 0, st, seq, cells);
  else PB_LAUNCH(k_seq_end, 1, 1, 0, st, seq);
}

}  // namespace pb
