// pb_shard.cu — the embedding worker's fan-out over the R GPUs of one box (SURVEY.md §8e), fused with the compute
// on both sides of it.
//
// Reference: the EW shards a batch's DISTINCT signs by farmhash64(sign) % R (indices_to_sharded_indices,
// embedding_worker_service/mod.rs:454-479), issues one lookup_mixed per parameter server (:886-919), puts the rows
// back in batch order (:486-629); in backward it reduces the gradients per distinct sign and issues one
// update_gradient_mixed per server (:786-857), which applies them (embedding_parameter_service/mod.rs:359-427).
// Here every rank is the EW of its own batches and PS `rank`; a "request" is what one rank sends one owner.  The
// requests of the R data-parallel trainers reach an owner as R separate requests — exactly the reference's picture
// with R NN workers — and are served in rank order, so a sign looked up by several ranks takes one optimizer step
// per requesting rank, as it does there (deterministically ordered here).
//
// There is no separate exchange step: the kernel that produces data writes it where its consumer lives.
//   k_route_items    (requester) owner of every distinct sign, sign stored straight into the owner's receive area
//   k_link_items     (requester, slots sharing a feature group only) a sign's entries of one request linked in slot order
//   k_owner_lookup   (owner) find / admit / initialise, row gathered, converted and stored straight into the
//                    requester's receive area
//   k_expand_items   (requester) received rows -> output rows in batch order (+ pooling for ragged layouts)
//   k_reduce_items / k_reduce_hot <SEND>  (requester, pb_reduce.cu) reduced gradient stored into the owner's area
//   k_owner_update   (owner) one request at a time, in rank order: optimizer step on the resident rows
// Ordering between ranks is by flag words in the receiver's area (one per phase and source, written after a
// system-scope fence); k_wait spins on them in ONE block so that the box — or, in tests, the other virtual ranks
// sharing a GPU — keeps running.  Phase counters live on the device: a whole step is CUDA-graph capturable.
#include "pb_batch.cuh"
#include "pb_optim.cuh"
#include "pb_probe.cuh"

namespace pb {

constexpr uint32_t UWIN_MISS = 0xFFFFFFFDu;  // uwin: the sign has no storage (its gradient counts as a miss)

__device__ __forceinline__ uint32_t* x_ctrl(const XchgDev& x, uint32_t q) { return reinterpret_cast<uint32_t*>(x.base[q]); }
__device__ __forceinline__ uint64_t* x_sign(const XchgDev& x, uint32_t q) {
  return reinterpret_cast<uint64_t*>(x.base[q] + x.off_sign);
}
__device__ __forceinline__ unsigned char* x_row(const XchgDev& x, uint32_t q) {
  return reinterpret_cast<unsigned char*>(x.base[q] + x.off_row);
}
__device__ __forceinline__ uint32_t* x_chain(const XchgDev& x, uint32_t q) {
  return reinterpret_cast<uint32_t*>(x.base[q] + x.off_chain);
}

// ------------------------------------------------------------------------------------------------
// requester, forward: A3 over the distinct signs.  One thread per item; segment slots are handed out per owner
// with one atomic per warp and owner (__match_any_sync).  Mirrors k_probe_items' bookkeeping: the item's target
// (owner * cap + slot) replaces the row, and the backward's work lists are filled by multiplicity.
// ------------------------------------------------------------------------------------------------
template <bool TRAIN>
__global__ void __launch_bounds__(256) k_route_items(SlotsDev sl, BatchDev b, XchgDev x) {
  const uint32_t n_items = b.cnt[BC_ITEMS];
  if (blockIdx.x * blockDim.x >= n_items) return;  // whole block (the grid is sized for the worst case)
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t u = blockIdx.x * blockDim.x + threadIdx.x;
  const bool valid = u < n_items;
  uint32_t cell = 0, cnt = 0, first = 0, owner = 0xFFFFFFFFu;
  uint64_t sign = 0;
  if (valid) {
    cell = b.item_cell[u];
    const uint4 lo = *reinterpret_cast<const uint4*>(&b.set[cell]);
    const uint4 hi = *(reinterpret_cast<const uint4*>(&b.set[cell]) + 1);
    sign = (hi.w >> 31) ? KEY_EMPTY : ((uint64_t)lo.x | ((uint64_t)lo.y << 32));
    cnt = TRAIN ? lo.z : 0u;
    first = hi.z;
    owner = (uint32_t)(farmhash64_u64(sign) % x.R);  // sign_to_shard_modulo, mod.rs:341-345
  }
  // a slot in the owner's segment: counted per block in shared memory, one global atomic per block and owner
  __shared__ uint32_t s_n[PB_MAX_RANKS], s_g[PB_MAX_RANKS];
  if (threadIdx.x < PB_MAX_RANKS) s_n[threadIdx.x] = 0;
  __syncthreads();
  const uint32_t peers = __match_any_sync(0xffffffffu, owner);
  const uint32_t leader = __ffs(peers) - 1;
  uint32_t k = 0;
  if (valid && lane == leader) k = atomicAdd(&s_n[owner], (uint32_t)__popc(peers));
  k = __shfl_sync(0xffffffffu, k, leader) + __popc(peers & ((1u << lane) - 1u));
  __syncthreads();
  if (threadIdx.x < x.R && s_n[threadIdx.x]) s_g[threadIdx.x] = atomicAdd(&b.cnt[BC_PEER + threadIdx.x], s_n[threadIdx.x]);
  __syncthreads();
  uint32_t target = ROW_NONE;
  if (valid) {
    k += s_g[owner];
    if (k < x.cap) {
      target = owner * x.cap + k;
      x_sign(x, owner)[(size_t)x.rank * x.cap + k] = sign;  // over NVLink when owner != rank
    } else {
      x.err[0] = 1u;  // the pair needs more than cap slots: the caller re-runs the batch with a larger cap
    }
  }
  uint32_t slot = 0, hot_nwords = 0;
  if (valid && cnt > PB_WARM_MAX) {
    slot = slot_of_occ(sl, first);
    hot_nwords = (sl.occ_off[slot + 1] - sl.occ_off[slot] + 31u) / 32u;
  }
  const ItemSlots is = block_item_slots(b, valid, cnt, hot_nwords);
  if (valid) {
    *(reinterpret_cast<uint2*>(&b.set[cell]) + 2) = make_uint2(target, is.base);  // target, base
    if (is.cls == 1) b.cold[is.pos] = make_uint2(target, first);
    else if (is.cls == 2) b.warm[is.pos] = make_uint4(target, is.base, cnt, 0u);
    else if (is.cls == 3) b.hot[is.pos] = make_uint4(target, is.base, cnt, slot);
  }
}

// ------------------------------------------------------------------------------------------------
// requester, pb_tier_stage_sharded's SEND: the next batch's ids, slot-prefixed as k_tier_stage prefixes them, each sent
// to its owner's stage area.  One thread per id; a sign that several lanes of a warp hold is sent once (the owner's
// restore is idempotent, so duplicates across warps only cost slots).  Slots per owner as in k_route_items: counted per
// block in shared memory, one global atomic per block and owner.  A sign over `cap` is not sent (x.err[0]): its
// forward restores it as it would unstaged.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_stage_route(SlotsDev sl, const uint64_t* __restrict__ ids, uint32_t n, XchgDev x,
                                                     uint32_t* __restrict__ sent) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  bool valid = i < n;
  uint64_t sign = 0;
  if (valid) {
    sign = ids[i];
    const uint64_t p = sl.prefix[slot_of_occ(sl, i)];
    if (p) sign = mod_mersenne(sign, sl.spacing_bits) + p;
  }
  const uint32_t live = __ballot_sync(0xffffffffu, valid);
  const uint32_t same = __match_any_sync(0xffffffffu, (unsigned long long)sign) & live;
  valid = valid && (uint32_t)(__ffs(same) - 1) == lane;  // the warp's first lane of the sign sends it
  const uint32_t owner = valid ? (uint32_t)(farmhash64_u64(sign) % x.R) : 0xFFFFFFFFu;  // sign_to_shard_modulo
  __shared__ uint32_t s_n[PB_MAX_RANKS], s_g[PB_MAX_RANKS];
  if (threadIdx.x < PB_MAX_RANKS) s_n[threadIdx.x] = 0;
  __syncthreads();
  const uint32_t peers = __match_any_sync(0xffffffffu, owner);
  const uint32_t leader = __ffs(peers) - 1;
  uint32_t k = 0;
  if (valid && lane == leader) k = atomicAdd(&s_n[owner], (uint32_t)__popc(peers));
  k = __shfl_sync(0xffffffffu, k, leader) + __popc(peers & ((1u << lane) - 1u));
  __syncthreads();
  if (threadIdx.x < x.R && s_n[threadIdx.x]) s_g[threadIdx.x] = atomicAdd(&sent[threadIdx.x], s_n[threadIdx.x]);
  __syncthreads();
  if (!valid) return;
  k += s_g[owner];
  if (k < x.cap) x_sign(x, owner)[(size_t)x.rank * x.cap + k] = sign;  // over NVLink when owner != rank
  else x.err[0] = 1u;
}

void launch_stage_route(const SlotsDev& sl, const uint64_t* ids, uint32_t n, const XchgDev& x, uint32_t* sent,
                        cudaStream_t st) {
  if (n) PB_LAUNCH_F(FAM_ROUTE, k_stage_route, cdiv(n, 256), 256, 0, st, sl, ids, n, x, sent);
}

// ------------------------------------------------------------------------------------------------
// requester, PB_PHASE_PREPARE: how many of the batch's distinct items go to each owner — what `cap` must cover — read
// from the context alone (the dedup's set, or the raw numbering's), before anything is sent.  Counted per block in
// shared memory, one global atomic per block and owner.
// ------------------------------------------------------------------------------------------------
template <bool RAW>
__global__ void __launch_bounds__(256) k_count_owners(BatchDev b, RawWork w, uint32_t R, uint32_t* __restrict__ need) {
  __shared__ uint32_t s_n[PB_MAX_RANKS];
  if (threadIdx.x < PB_MAX_RANKS) s_n[threadIdx.x] = 0;
  __syncthreads();
  const uint32_t n_items = RAW ? w.counts[0] : b.cnt[BC_ITEMS];
  for (uint32_t u = blockIdx.x * blockDim.x + threadIdx.x; u < n_items; u += gridDim.x * blockDim.x) {
    uint64_t sign;
    if (RAW) {
      sign = w.set[w.distinct_cell[u]].key;  // (as k_raw_route reads it)
    } else {
      const uint32_t cell = b.item_cell[u];  // (as k_route_items reads it)
      const uint4 lo = *reinterpret_cast<const uint4*>(&b.set[cell]);
      const uint4 hi = *(reinterpret_cast<const uint4*>(&b.set[cell]) + 1);
      sign = (hi.w >> 31) ? KEY_EMPTY : ((uint64_t)lo.x | ((uint64_t)lo.y << 32));
    }
    atomicAdd(&s_n[(uint32_t)(farmhash64_u64(sign) % R)], 1u);  // sign_to_shard_modulo, mod.rs:341-345
  }
  __syncthreads();
  if (threadIdx.x < R && s_n[threadIdx.x]) atomicAdd(&need[threadIdx.x], s_n[threadIdx.x]);
}

void launch_count_owners(bool raw, const BatchDev& b, const RawWork& w, uint32_t n, uint32_t R, uint32_t* need,
                         cudaStream_t st) {
  if (!n) return;
  const uint32_t full = cdiv(n, 256);  // worst case U = N; the blocks stride over the items
  const uint32_t grid = full < PB_NUM_SMS * 4u ? full : PB_NUM_SMS * 4u;
  if (raw) PB_LAUNCH_F(FAM_ROUTE, k_count_owners<true>, grid, 256, 0, st, b, w, R, need);
  else PB_LAUNCH_F(FAM_ROUTE, k_count_owners<false>, grid, 256, 0, st, b, w, R, need);
}

// ------------------------------------------------------------------------------------------------
// requester, forward, slots sharing a feature group (launched only then): a sign that several slots of one group hold
// is one entry per slot in its owner's request, and the reference steps them one after another in slot order
// (mod.rs:703-872).  Every routed item looks for its sign in the regions of the other slots of its group, nearest
// first, and writes its entry's chain word: CHAIN_CONT if an earlier slot holds the sign (the owner steps it after
// that one), and the entry of the next later slot that does (or CHAIN_END).  Items over cap take no part.  Block 0
// also marks this request as carrying chain words: the owner compares ctrl[XC_CHAIN] with the SIGN flag about to be
// raised, so a mark left from an earlier step never counts.
// ------------------------------------------------------------------------------------------------
// target of `sign` in the scratch-set region of `slot` (k_dedup's probe sequence), ROW_NONE if absent or over cap
__device__ __forceinline__ uint32_t find_in_slot(const SlotsDev& sl, const BatchDev& b, uint32_t slot, uint64_t sign) {
  uint32_t size;
  const uint32_t off = set_region(sl, slot, size);
  if (sign == KEY_EMPTY) {  // the reserved cell: key 0 when the slot holds the sign
    const DCell& c = b.set[off + size];
    return c.key != KEY_EMPTY ? c.target : ROW_NONE;
  }
  uint32_t idx = off + __umulhi((uint32_t)(mix64(sign) >> 32), size);
  for (;;) {  // the region has more cells than the slot has ids: ends on an empty cell
    const uint64_t k = b.set[idx].key;
    if (k == sign) return b.set[idx].target;
    if (k == KEY_EMPTY) return ROW_NONE;
    idx = (idx + 1 == off + size) ? off : idx + 1;
  }
}

__global__ void __launch_bounds__(256) k_link_items(SlotsDev sl, BatchDev b, XchgDev x, GroupLinks gl) {
  if (blockIdx.x == 0 && threadIdx.x < x.R) x_ctrl(x, threadIdx.x)[XC_CHAIN * PB_MAX_RANKS + x.rank] = x.epoch[XC_FLAG_SIGN] + 1u;
  const uint32_t n_items = b.cnt[BC_ITEMS];
  for (uint32_t u = blockIdx.x * blockDim.x + threadIdx.x; u < n_items; u += gridDim.x * blockDim.x) {
    const uint32_t cell = b.item_cell[u];
    const uint4 lo = *reinterpret_cast<const uint4*>(&b.set[cell]);
    const uint4 hi = *(reinterpret_cast<const uint4*>(&b.set[cell]) + 1);  // target, base, first, item
    const uint32_t target = hi.x;
    if (target == ROW_NONE) continue;
    const uint64_t sign = (hi.w >> 31) ? KEY_EMPTY : ((uint64_t)lo.x | ((uint64_t)lo.y << 32));
    const uint32_t slot = slot_of_occ(sl, hi.z);
    uint32_t word = CHAIN_END;
    for (uint32_t s = gl.prev[slot]; s != 0xFFu; s = gl.prev[s])
      if (find_in_slot(sl, b, s, sign) != ROW_NONE) {
        word |= CHAIN_CONT;
        break;
      }
    for (uint32_t s = gl.next[slot]; s != 0xFFu; s = gl.next[s]) {
      const uint32_t t2 = find_in_slot(sl, b, s, sign);
      if (t2 != ROW_NONE) {
        word = (word & CHAIN_CONT) | (t2 % x.cap);  // (same sign, same owner)
        break;
      }
    }
    x_chain(x, target / x.cap)[(size_t)x.rank * x.cap + target % x.cap] = word;  // over NVLink when the owner is a peer
  }
}

// ------------------------------------------------------------------------------------------------
// flags.  signal: this rank finished writing phase `phase` into every peer's area -> bump the device-side phase
// counter, publish (optionally) the per-owner counts, fence, write the flag word [phase][rank] of every peer.
// wait: spin (bounded) until source `src` (or every source) has signalled the phase this rank is about to consume.
// ------------------------------------------------------------------------------------------------
#ifndef PB_WAIT_SPINS
#define PB_WAIT_SPINS (1u << 25)
#endif
__device__ __forceinline__ void signal_phase(const XchgDev& x, int phase, const uint32_t* __restrict__ counts) {
  __shared__ uint32_t e_s;
  if (threadIdx.x == 0) {
    e_s = x.epoch[phase] + 1;
    x.epoch[phase] = e_s;
  }
  __syncthreads();
  const uint32_t q = threadIdx.x;
  if (q < x.R) {
    uint32_t* ctrl = x_ctrl(x, q);
    if (counts) ctrl[XC_COUNT * PB_MAX_RANKS + x.rank] = counts[q] < x.cap ? counts[q] : x.cap;
    __threadfence_system();  // everything this GPU stored into the peer's area before is visible before the flag
    *reinterpret_cast<volatile uint32_t*>(&ctrl[phase * PB_MAX_RANKS + x.rank]) = e_s;
  }
}
__device__ __forceinline__ void wait_phase(const XchgDev& x, int phase, int src) {
  const uint32_t q = threadIdx.x;
  if (q >= x.R || (src >= 0 && q != (uint32_t)src)) return;
  uint32_t* w = &x.waited[phase * PB_MAX_RANKS + q];
  const uint32_t e = *w + 1;
  *w = e;
  volatile uint32_t* flag = reinterpret_cast<volatile uint32_t*>(&x_ctrl(x, x.rank)[phase * PB_MAX_RANKS + q]);
  uint32_t spins = 0;
  while ((int32_t)(*flag - e) < 0) {
    if (++spins > PB_WAIT_SPINS) {  // a peer is not coming: give up instead of hanging the GPU, and say so
      x.err[1] = 1u;
      break;
    }
  }
  __threadfence_system();
}
__global__ void k_signal(XchgDev x, int phase, const uint32_t* __restrict__ counts) { signal_phase(x, phase, counts); }
__global__ void k_wait(XchgDev x, int phase, int src) { wait_phase(x, phase, src); }
// one process per GPU: a phase's signal is directly followed by the wait for the peers' — one launch
__global__ void k_signal_wait(XchgDev x, int phase, const uint32_t* __restrict__ counts) {
  signal_phase(x, phase, counts);
  wait_phase(x, phase, -1);
}

// ------------------------------------------------------------------------------------------------
// owner, forward: lookup_mixed of R requests at once (PS mod.rs:162-262, 344-357).  Eight lanes per received sign
// probe the index (pb_probe.cuh: find / refresh / admit + initialise), then the same eight lanes read the row and
// store it, converted, into the requester's area.  f16 rows serve one-id-per-sample layouts (the EW's result is
// f16(0 + row) there, bit for bit); f32 rows serve ragged layouts, which pool on the requester.
// ------------------------------------------------------------------------------------------------
// TIER (inference, MODE_FIND, on a table with a host tier `tier`): a sign the HBM index lacks is probed in the tier and
// read from its mapped host row where it is, converted as an HBM row is; only a sign neither table holds is a miss.
// Training requests never take this path: their tier-held signs were moved into HBM rows first (k_tier_restore_recv).
template <int MODE, bool ROW_F32, bool TIER>
__device__ __forceinline__ void owner_lookup(const TableDev& t, const TableDev& tier, const HyperDev& hy, const OptimDev& op,
                                             const XchgDev& x) {
  const uint32_t tick = t.counters[CTR_TICK];
  const uint32_t sub = threadIdx.x % BUCKET;
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t gshift = lane & ~(BUCKET - 1);
  const uint32_t groups = gridDim.x * (blockDim.x / BUCKET);
  const uint32_t total = x.R * x.cap;
  const uint32_t* ctrl = x_ctrl(x, x.rank);
  const uint32_t warp_first = ((blockIdx.x * blockDim.x + threadIdx.x) / 32) * (32 / BUCKET);
  if (blockIdx.x == 0 && threadIdx.x < x.R) x.own_cnt[threadIdx.x] = ctrl[XC_COUNT * PB_MAX_RANKS + threadIdx.x];
  uint32_t chained = 0;  // sources whose request carries chain words (k_link_items)
  if (MODE == MODE_TRAIN) {
    __shared__ uint32_t s_chained;
    if (threadIdx.x == 0) s_chained = 0u;
    __syncthreads();
    if (threadIdx.x < x.R) {
      const uint32_t f = ctrl[XC_FLAG_SIGN * PB_MAX_RANKS + threadIdx.x];
      if (f != 0u && ctrl[XC_CHAIN * PB_MAX_RANKS + threadIdx.x] == f) atomicOr(&s_chained, 1u << threadIdx.x);
    }
    __syncthreads();
    chained = s_chained;
    if (blockIdx.x == 0 && threadIdx.x == 0) *x.chained = chained;
  }
  for (uint32_t j0 = warp_first; j0 < total; j0 += groups) {  // uniform per warp
    const uint32_t j = j0 + lane / BUCKET;
    const uint32_t src = j / x.cap, k = j % x.cap;
    const bool valid = j < total && k < ctrl[XC_COUNT * PB_MAX_RANKS + src];
    if (!__any_sync(0xffffffffu, valid)) continue;
    uint64_t sign = 0;
    if (valid && sub == 0) sign = x_sign(x, x.rank)[j];
    sign = __shfl_sync(0xffffffffu, sign, gshift);
    const ProbeOut r = probe_group<MODE>(t, hy, op, sign, valid, tick, sub, gshift);
    uint32_t trow = ROW_NONE;  // TIER: the sign's tier row
    if (TIER) trow = probe_group<MODE_FIND>(tier, HyperDev{}, OptimDev{}, sign, valid && r.row == ROW_NONE, 0u, sub, gshift).row;
    // a row admitted just now was initialised by this very group (fenced before its number was published); rows are
    // read through L2 below, never from a stale L1 line
    if (!valid) continue;
    if (sub == 0) {
      x.own_row[j] = r.row;
      if (r.row == ROW_NONE && (!TIER || trow == ROW_NONE)) atomicAdd(&t.counters[CTR_MISS], 1u);
      if (MODE == MODE_TRAIN) {
        // the backward steps every row ONCE for all the requests that hold it (in rank order): note who asked.  A
        // chained request notes the head of each sign's chain; the other entries are reached through the links.
        uint32_t won = ROW_NONE, link = CHAIN_END;
        if ((chained >> src) & 1u) {
          link = x_chain(x, x.rank)[j];
          x.own_link[j] = link;  // (the area's word may be overwritten by the source's next request before the backward)
        }
        if (r.row < t.capacity && !(link & CHAIN_CONT)) {
          uint32_t idx = (r.row * 0x9E3779B1u) & (x.ucells - 1u);
          for (;;) {
            const uint32_t old = atomicCAS(&x.ucell[idx].row, ROW_NONE, r.row);
            if (old == ROW_NONE) won = idx;
            if (old == ROW_NONE || old == r.row) break;
            idx = (idx + 1u) & (x.ucells - 1u);
          }
          atomicOr(&x.ucell[idx].mask, 1u << src);
          x.ucell[idx].k[src] = k;
        }
        x.uwin[j] = r.row < t.capacity ? won : UWIN_MISS;
      }
    }
    const float* row = (!TIER || r.row < t.capacity) ? t.rows + (size_t)(r.row < t.capacity ? r.row : 0u) * t.stride
                                                     : tier.rows + (size_t)(trow < tier.capacity ? trow : 0u) * tier.stride;
    const bool have = r.row < t.capacity || (TIER && trow < tier.capacity);
    const size_t slot = (size_t)x.rank * x.cap + k;  // this owner's segment in the requester's area
    if (ROW_F32) {
      float* dst = reinterpret_cast<float*>(x_row(x, src)) + slot * t.dim;
      if (t.dim % 4 == 0) {
        for (uint32_t e = sub * 4; e < t.dim; e += BUCKET * 4) {
          float4 v = have ? __ldcg(reinterpret_cast<const float4*>(row + e)) : make_float4(0.f, 0.f, 0.f, 0.f);
          *reinterpret_cast<float4*>(dst + e) = v;
        }
      } else {
        for (uint32_t e = sub; e < t.dim; e += BUCKET) dst[e] = have ? __ldcg(row + e) : 0.0f;
      }
    } else {
      __half* dst = reinterpret_cast<__half*>(x_row(x, src)) + slot * t.dim;
      if (t.dim % 8 == 0) {
        // a lane converts 8 consecutive floats into one 16-byte store: the group's stores are 128 contiguous bytes —
        // whole NVLink write packets when the requester is a peer; two such chunks (four loads) in flight per lane
        for (uint32_t e0 = sub * 8; e0 < t.dim; e0 += BUCKET * 8 * 2) {
          float4 v[2][2];
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            const uint32_t e = e0 + (uint32_t)u * BUCKET * 8;
            const bool in = have && e < t.dim;
            v[u][0] = in ? __ldcg(reinterpret_cast<const float4*>(row + e)) : make_float4(0.f, 0.f, 0.f, 0.f);
            v[u][1] = in ? __ldcg(reinterpret_cast<const float4*>(row + e + 4)) : make_float4(0.f, 0.f, 0.f, 0.f);
          }
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            const uint32_t e = e0 + (uint32_t)u * BUCKET * 8;
            if (e >= t.dim) break;
            // the EW adds the row into a zeroed f32 row, then converts (mod.rs:555-561, persia-common lib.rs:157-161)
            __half2 h0 = __floats2half2_rn(__fadd_rn(0.0f, v[u][0].x), __fadd_rn(0.0f, v[u][0].y));
            __half2 h1 = __floats2half2_rn(__fadd_rn(0.0f, v[u][0].z), __fadd_rn(0.0f, v[u][0].w));
            __half2 h2 = __floats2half2_rn(__fadd_rn(0.0f, v[u][1].x), __fadd_rn(0.0f, v[u][1].y));
            __half2 h3 = __floats2half2_rn(__fadd_rn(0.0f, v[u][1].z), __fadd_rn(0.0f, v[u][1].w));
            uint4 pk;
            pk.x = *reinterpret_cast<uint32_t*>(&h0);
            pk.y = *reinterpret_cast<uint32_t*>(&h1);
            pk.z = *reinterpret_cast<uint32_t*>(&h2);
            pk.w = *reinterpret_cast<uint32_t*>(&h3);
            *reinterpret_cast<uint4*>(dst + e) = pk;
          }
        }
      } else if (t.dim % 4 == 0) {
        for (uint32_t e = sub * 4; e < t.dim; e += BUCKET * 4) {
          float4 v = have ? __ldcg(reinterpret_cast<const float4*>(row + e)) : make_float4(0.f, 0.f, 0.f, 0.f);
          __half2 a = __floats2half2_rn(__fadd_rn(0.0f, v.x), __fadd_rn(0.0f, v.y));
          __half2 c = __floats2half2_rn(__fadd_rn(0.0f, v.z), __fadd_rn(0.0f, v.w));
          uint2 pk;
          pk.x = *reinterpret_cast<uint32_t*>(&a);
          pk.y = *reinterpret_cast<uint32_t*>(&c);
          *reinterpret_cast<uint2*>(dst + e) = pk;
        }
      } else {
        for (uint32_t e = sub; e < t.dim; e += BUCKET) dst[e] = __float2half_rn(__fadd_rn(0.0f, have ? __ldcg(row + e) : 0.0f));
      }
    }
  }
}

template <int MODE, bool ROW_F32>
__global__ void __launch_bounds__(256, PB_PROBE_BLOCKS) k_owner_lookup(TableDev t, HyperDev hy, OptimDev op, XchgDev x) {
  owner_lookup<MODE, ROW_F32, false>(t, t, hy, op, x);
}

template <bool ROW_F32>
__global__ void __launch_bounds__(256, PB_PROBE_BLOCKS) k_owner_lookup_tier(TableDev t, TableDev tier, HyperDev hy,
                                                                            OptimDev op, XchgDev x) {
  owner_lookup<MODE_FIND, ROW_F32, true>(t, tier, hy, op, x);
}

// ------------------------------------------------------------------------------------------------
// requester, forward: received rows -> batch order (lookup_batched_all_slots_postprocess, mod.rs:486-629).
// One-id layouts: a pure copy of the f16 row.  Ragged layouts: f32 rows summed in sample order, sqrt scaling, RNE.
// TRAIN: files every occurrence of a repeated sign into the sign's list, like k_gather_items.
// `rows`: the rows an item's set cell `target` indexes — this rank's receive area (target = owner * cap + slot), or the
// context's staging of a remote read (pb_remote.cu, target = the item's number).
// ------------------------------------------------------------------------------------------------
template <bool TRAIN>
__global__ void __launch_bounds__(256) k_expand_copy(uint32_t dim, SlotsDev sl, BatchDev b, const void* __restrict__ rows,
                                                     uint32_t n_out, __half* __restrict__ out, uint32_t lanes) {
  // `lanes` lanes per output row, 16 bytes per lane and step
  if (TRAIN) {  // one occurrence per thread first (the grid has at least n_out threads), one atomic per warp and sign
    const uint32_t gt = blockIdx.x * blockDim.x + threadIdx.x;
    if ((gt & ~31u) < n_out) file_occurrences_warp(b, sl, gt, gt < n_out);
  }
  const uint32_t g = (blockIdx.x * blockDim.x + threadIdx.x) / lanes;
  const uint32_t l = threadIdx.x % lanes;
  if (g >= n_out) return;
  const uint32_t cell = b.occ_set[g];
  const uint32_t target = (reinterpret_cast<const uint4*>(&b.set[cell]) + 1)->x;
  const uint32_t words = dim / 8;  // 16-byte words per f16 row (dim % 8 == 0 on this path)
  const uint4* src = reinterpret_cast<const uint4*>(rows) + (size_t)(target == ROW_NONE ? 0u : target) * words;
  uint4* dst = reinterpret_cast<uint4*>(out) + (size_t)g * words;
  for (uint32_t w = l; w < words; w += lanes) dst[w] = target == ROW_NONE ? make_uint4(0u, 0u, 0u, 0u) : src[w];
}

template <bool TRAIN, bool ROW_F32>
__global__ void __launch_bounds__(256) k_expand_pool(uint32_t dim, SlotsDev sl, BatchDev b, const void* __restrict__ rows,
                                                     const uint32_t* __restrict__ row_off, uint32_t n_out, uint32_t batch,
                                                     __half* __restrict__ out, uint32_t G) {
  const uint32_t gid = (blockIdx.x * blockDim.x + threadIdx.x) / G;
  const uint32_t lane = threadIdx.x % G;
  if (gid >= n_out) return;
  const uint32_t beg = row_off ? row_off[gid] : gid, end = row_off ? row_off[gid + 1] : gid + 1;
  float scale = 1.0f;
  if (row_off && batch && sl.sqrt_scaling[gid / batch]) {
    uint32_t cnt = end - beg;
    scale = __fdiv_rn(1.0f, __fsqrt_rn((float)(cnt > 1 ? cnt : 1)));
  }
  if (TRAIN && lane == 0) {
    for (uint32_t j = beg; j < end; ++j) {
      const uint32_t cell = b.occ_set[j];
      file_occurrence(b, sl, cell, occ_ref(b, cell), j);
    }
  }
  if (!ROW_F32 && end - beg == 1) {  // one id: the owner already rounded 0 + row to f16 (a copy keeps the sign of a -0)
    const uint32_t target = b.set[b.occ_set[beg]].target;
    const __half* src = reinterpret_cast<const __half*>(rows) + (size_t)(target == ROW_NONE ? 0u : target) * dim;
    for (uint32_t e = lane; e < dim; e += G) out[(size_t)gid * dim + e] = target == ROW_NONE ? __float2half_rn(0.0f) : src[e];
    return;
  }
  for (uint32_t e = lane; e < dim; e += G) {
    float acc = 0.0f;
    for (uint32_t j = beg; j < end; ++j) {
      const uint32_t target = b.set[b.occ_set[j]].target;
      if (target == ROW_NONE) continue;
      float v;
      if (ROW_F32) v = reinterpret_cast<const float*>(rows)[(size_t)target * dim + e];
      else v = __half2float(reinterpret_cast<const __half*>(rows)[(size_t)target * dim + e]);
      acc = __fadd_rn(acc, v);
    }
    out[(size_t)gid * dim + e] = __float2half_rn(__fmul_rn(acc, scale));
  }
}

// ------------------------------------------------------------------------------------------------
// owner, backward, Adam: get_batch_level_state per request (optim.rs:151-197).  A request advances the accumulated
// (beta1^t, beta2^t) of every feature group that occurs among the signs it applies on THIS parameter server, once,
// and all its signs of the group use the advanced pair.  k_owner_adam_present finds the groups per request (block-level
// bit sets: a few global atomics per block), k_owner_adam_pows walks the requests in rank order.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t adam_key_of(const XchgDev& x, uint64_t sign) {
  const uint64_t m = sign & x.amask;
  for (uint32_t g = 0; g < x.n_akeys; ++g)
    if (x.akeys[g] == m) return g;
  return PB_ADAM_KEYS - 1u;  // (a group the table has never seen in a forward: cannot hold rows)
}
// request src's (beta1^t, beta2^t) of feature group akey
__device__ __forceinline__ const float* owner_adam_pair(const XchgDev& x, uint32_t src, uint32_t akey) {
  return x.apow + ((size_t)src * PB_ADAM_KEYS + akey) * 2u;
}
__global__ void __launch_bounds__(256) k_owner_adam_present(XchgDev x) {
  __shared__ uint32_t bits[PB_MAX_RANKS][PB_ADAM_KEYS / 32];
  for (uint32_t i = threadIdx.x; i < PB_MAX_RANKS * (PB_ADAM_KEYS / 32); i += blockDim.x) (&bits[0][0])[i] = 0u;
  __syncthreads();
  const uint32_t total = x.R * x.cap;
  const uint32_t* gok = reinterpret_cast<const uint32_t*>(x.base[x.rank] + x.off_gok);
  for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < total; j += gridDim.x * blockDim.x) {
    const uint32_t src = j / x.cap, k = j % x.cap;
    if (k >= x.own_cnt[src] || gok[j] == 0u) continue;
    const uint32_t g = adam_key_of(x, x_sign(x, x.rank)[j]);
    atomicOr(&bits[src][g >> 5], 1u << (g & 31u));
  }
  __syncthreads();
  for (uint32_t i = threadIdx.x; i < x.R * (PB_ADAM_KEYS / 32); i += blockDim.x) {
    const uint32_t v = (&bits[0][0])[(i / (PB_ADAM_KEYS / 32)) * (PB_ADAM_KEYS / 32) + i % (PB_ADAM_KEYS / 32)];
    if (v) atomicOr(&x.apresent[i], v);
  }
}
__global__ void k_owner_adam_pows(XchgDev x, float* table_pow, float b1, float b2) {
  const uint32_t g = threadIdx.x;
  if (g >= PB_ADAM_KEYS) return;
  float p1 = table_pow[2 * g], p2 = table_pow[2 * g + 1];
  for (uint32_t s = 0; s < x.R; ++s) {
    uint32_t* w = &x.apresent[s * (PB_ADAM_KEYS / 32) + (g >> 5)];
    if ((*w >> (g & 31u)) & 1u) {
      p1 = __fmul_rn(p1, b1);
      p2 = __fmul_rn(p2, b2);
    }
    x.apow[(s * PB_ADAM_KEYS + g) * 2] = p1;
    x.apow[(s * PB_ADAM_KEYS + g) * 2 + 1] = p2;
  }
  table_pow[2 * g] = p1;
  table_pow[2 * g + 1] = p2;
  __syncthreads();
  for (uint32_t i = threadIdx.x; i < x.R * (PB_ADAM_KEYS / 32); i += blockDim.x) x.apresent[i] = 0u;  // for the next step
}
void launch_owner_adam(const XchgDev& x, float* table_pow, float b1, float b2, cudaStream_t st) {
  const uint32_t full = cdiv((uint64_t)x.R * x.cap, 256);
  PB_LAUNCH(k_owner_adam_present, full < PB_NUM_SMS * 2u ? full : PB_NUM_SMS * 2u, 256, 0, st, x);
  PB_LAUNCH(k_owner_adam_pows, 1, PB_ADAM_KEYS, 0, st, x, table_pow, b1, b2);
}

// ------------------------------------------------------------------------------------------------
// owner, backward: update_gradient_mixed of the step's R requests (PS mod.rs:359-427) in ONE launch.  The reference
// serves the requests one after another; a row that several requests hold is stepped once per request, in the order
// the requests arrive — here: rank order.  A lane group takes a row (through the request that opened its cell in the
// forward), keeps it in registers and applies the holders' gradients in rank order, each a full optimizer step on the
// result of the previous one: the same arithmetic as R sequential passes, one read and one write of the row.
// The rule is ONE holder, and that holder is the opener itself: its row number, apply word and gradient are all at the
// request's own index, so the row, the gradient and the cell's holder mask are fetched together, two dependent memory
// round trips per row in all.  Signs without storage are counted (gradient_id_miss_count).  The cell goes back to empty.
// ------------------------------------------------------------------------------------------------
template <int VEC, int CPL, int KIND, bool INTEL = false>
__global__ void __launch_bounds__(256, CPL == 1 ? 3 : 2) k_owner_update_all(TableDev t, OptimDev op, HyperDev hy, XchgDev x, uint32_t G) {
  // G lanes per row, CPL chunks of VEC floats per lane (G * CPL * VEC == dim): few lanes per row keep the per-row
  // bookkeeping off most of the warp, and a lane has CPL independent loads in flight
  __shared__ uint32_t s_cnt[PB_MAX_RANKS], s_chained;
  if (threadIdx.x < PB_MAX_RANKS) s_cnt[threadIdx.x] = threadIdx.x < x.R ? x.own_cnt[threadIdx.x] : 0u;
  if (threadIdx.x == 0) s_chained = *x.chained;
  __syncthreads();
  const uint32_t wl = threadIdx.x & 31u, lane = wl % G, gi = wl / G, n_g = 32u / G;
  const uint32_t gmask = group_mask(G);
  const uint32_t total = x.R * x.cap;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = (gridDim.x * blockDim.x) >> 5;
  const float* grads = reinterpret_cast<const float*>(x.base[x.rank] + x.off_grad);
  const uint32_t* gok = reinterpret_cast<const uint32_t*>(x.base[x.rank] + x.off_gok);
  constexpr uint32_t J = 8;  // requests looked at per warp and round: their rows are stepped by the warp's lane groups
  for (uint32_t j0 = warp * J; j0 < total; j0 += n_warps * J) {
    // ---- lanes 0..J-1: did request j open a row's cell; its row and apply word (three independent loads)
    uint32_t w = ROW_NONE, crow = 0, cok = 0;
    if (wl < J) {
      const uint32_t j = j0 + wl;
      if (j < total && j % x.cap < s_cnt[j / x.cap]) {
        w = x.uwin[j];
        crow = x.own_row[j];
        cok = gok[j];
        if (w == UWIN_MISS) {
          if (cok != 0u) atomicAdd(&t.counters[CTR_GRAD_MISS], 1u);  // gradient_id_miss_count (PS mod.rs:401-403)
          w = ROW_NONE;
        }
      }
    }
    uint32_t winners = __ballot_sync(0xffffffffu, w != ROW_NONE);
    // ---- the lane groups take the rows, n_g at a time
    while (winners) {
      const uint32_t mine = __fns(winners, 0, gi + 1);  // this group's row of the round (0xFFFFFFFF: none left)
      for (uint32_t q = 0; q < n_g && winners; ++q) winners &= winners - 1u;
      const uint32_t bl = mine < 32u ? mine : 0u;
      const uint32_t idx = __shfl_sync(0xffffffffu, w, bl), row = __shfl_sync(0xffffffffu, crow, bl);
      const uint32_t ok1 = __shfl_sync(0xffffffffu, cok, bl);
      if (mine >= 32u) continue;
      const uint32_t j = j0 + mine, me = j / x.cap;
      UCell* cell = x.ucell + idx;
      float* prow = t.rows + (size_t)row * t.stride;
      uint32_t akey = 0;
      if (op.kind == PB_OPT_ADAM) akey = adam_key_of(x, x_sign(x, x.rank)[j]);  // the row's feature group
      // the step of request s's gradient
      auto ctx = [&](uint32_t s) { return step_ctx(op, 0.0f, owner_adam_pair(x, s, akey)); };
      // the holder mask, the row and the opener's gradient: one round trip
      const uint32_t mask = cell->mask;
      RowElems<KIND, VEC, INTEL> rc[CPL];
      float g1[CPL][VEC];
#pragma unroll
      for (int u = 0; u < CPL; ++u) {
        const uint32_t e = ((uint32_t)u * G + lane) * VEC;
        rc[u].load(prow, e, t, op);
        load_vec<VEC>(grads + (size_t)j * t.dim + e, g1[u]);
      }
      const uint32_t chained = mask & s_chained;  // holders whose request may hold the row more than once
      if (mask == (1u << me) && !chained) {  // the opener is the only holder, with one entry (the rule)
        if (ok1) {
          const StepCtx sc = ctx(me);
#pragma unroll
          for (int u = 0; u < CPL; ++u) {
            const uint32_t e = ((uint32_t)u * G + lane) * VEC;
            rc[u].step(e, g1[u], t, op, hy, sc);
            rc[u].store(prow, e, t, op);
          }
        }
      } else if (chained) {
        // slots sharing a feature group: every holder in rank order, and within its request the sign's entries in
        // slot order — the head (the cell's index), then the chain; a skipped entry is passed over, the walk goes on
        for (uint32_t m = mask; m; m &= m - 1u) {
          const uint32_t s = (uint32_t)__ffs(m) - 1u;
          uint32_t k = cell->k[s];
          for (uint32_t d = 0; d < PB_MAX_SLOTS; ++d) {  // (a chain holds at most one entry per slot)
            const uint32_t at = s * x.cap + k;
            if (gok[at]) {
              float g[CPL][VEC];
#pragma unroll
              for (int u = 0; u < CPL; ++u) load_vec<VEC>(grads + (size_t)at * t.dim + ((uint32_t)u * G + lane) * VEC, g[u]);
              const StepCtx sc = ctx(s);
#pragma unroll
              for (int u = 0; u < CPL; ++u) rc[u].step(((uint32_t)u * G + lane) * VEC, g[u], t, op, hy, sc);
            }
            if (!((chained >> s) & 1u)) break;
            k = x.own_link[at] & CHAIN_END;
            if (k >= s_cnt[s]) break;  // CHAIN_END
          }
        }
#pragma unroll
        for (int u = 0; u < CPL; ++u) rc[u].store(prow, ((uint32_t)u * G + lane) * VEC, t, op);
      } else {
        for (uint32_t m = mask; m;) {  // holders in rank order, two at a time: index, apply word, gradient — each stage
          uint32_t at[2], ok[2];       // issued for both before the next
          float g[2][CPL][VEC];
          int n = 0;
          uint32_t src[2];
          for (; n < 2 && m; ++n, m &= m - 1u) src[n] = (uint32_t)__ffs(m) - 1u;
#pragma unroll
          for (int v = 0; v < 2; ++v)
            if (v < n) at[v] = src[v] * x.cap + cell->k[src[v]];
#pragma unroll
          for (int v = 0; v < 2; ++v)
            if (v < n) ok[v] = gok[at[v]];  // 0: that requester skipped the slot (NaN gradient or add_skipped_gradient)
#pragma unroll
          for (int v = 0; v < 2; ++v)
            if (v < n && ok[v]) {
#pragma unroll
              for (int u = 0; u < CPL; ++u) load_vec<VEC>(grads + (size_t)at[v] * t.dim + ((uint32_t)u * G + lane) * VEC, g[v][u]);
            }
#pragma unroll
          for (int v = 0; v < 2; ++v)
            if (v < n && ok[v]) {
              const StepCtx sc = ctx(src[v]);
#pragma unroll
              for (int u = 0; u < CPL; ++u) rc[u].step(((uint32_t)u * G + lane) * VEC, g[v][u], t, op, hy, sc);
            }
        }
#pragma unroll
        for (int u = 0; u < CPL; ++u) rc[u].store(prow, ((uint32_t)u * G + lane) * VEC, t, op);
      }
      __syncwarp(gmask);
      if (lane == 0) {  // every lane of the group has read the cell: it goes back to empty
        cell->row = ROW_NONE;
        cell->mask = 0u;
      }
    }
  }
}

__global__ void k_uclear(XchgDev x) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < x.ucells; i += gridDim.x * blockDim.x) {
    x.ucell[i].row = ROW_NONE;
    x.ucell[i].mask = 0u;
  }
}

// ------------------------------------------------------------------------------------------------
// owner, backward: update_gradient_mixed of ONE request (PS mod.rs:359-427): one optimizer step per received
// (sign, gradient) whose apply word is set; signs without storage are counted (gradient_id_miss_count).  The
// requests of a step are served one launch after another, in rank order.
// ------------------------------------------------------------------------------------------------
template <int VEC, bool INTEL = false>
__global__ void __launch_bounds__(256) k_owner_update(TableDev t, OptimDev op, HyperDev hy, XchgDev x, uint32_t src,
                                                      uint32_t G) {
  const uint32_t lane = threadIdx.x % G, gmask = group_mask(G);
  const uint32_t n = x.own_cnt[src];
  const uint32_t nvec = t.dim / VEC;
  const uint32_t n_groups = gridDim.x * (blockDim.x / G);
  const float* grads = reinterpret_cast<const float*>(x.base[x.rank] + x.off_grad) + (size_t)src * x.cap * t.dim;
  const uint32_t* gok = reinterpret_cast<const uint32_t*>(x.base[x.rank] + x.off_gok) + (size_t)src * x.cap;
  const uint32_t* own_row = x.own_row + (size_t)src * x.cap;
  if ((*x.chained >> src) & 1u) {
    // slots sharing a feature group: a lane group takes a chain's head and steps the sign's entries one after another in
    // slot order (so no two groups hold one row); the entries after the head only count their misses here
    const uint32_t* link = x.own_link + (size_t)src * x.cap;
    for (uint32_t k0 = blockIdx.x * (blockDim.x / G) + threadIdx.x / G; k0 < n; k0 += n_groups) {
      const uint32_t row = own_row[k0];
      if (row_missing(row, t, lane, gok[k0] != 0u) || (link[k0] & CHAIN_CONT)) continue;
      float* prow = t.rows + (size_t)row * t.stride;
      // this request's (beta1^t, beta2^t) of the row's feature group
      const uint32_t akey = op.kind == PB_OPT_ADAM ? adam_key_of(x, x_sign(x, x.rank)[(size_t)src * x.cap + k0]) : 0u;
      StepCtx sc = step_ctx(op, 0.0f, owner_adam_pair(x, src, akey));
      uint32_t k = k0;
      for (uint32_t d = 0; d < PB_MAX_SLOTS; ++d) {  // (a chain holds at most one entry per slot)
        if (gok[k] != 0u) {
          const float* g0 = grads + (size_t)k * t.dim;
          sc.vw_state = op.kind == PB_OPT_ADAGRAD_VW ? prow[t.dim] : 0.0f;
          step_row<-1, VEC, INTEL>(prow, t, op, hy, sc, lane, G, [&](uint32_t e0, float (&g)[VEC]) { load_vec<VEC>(g0 + e0, g); });
          if (op.kind == PB_OPT_ADAGRAD_VW) vw_state_step(prow, g0, t, op, sc, lane, gmask);
        }
        k = link[k] & CHAIN_END;
        if (k >= n) break;  // CHAIN_END
      }
    }
    return;
  }
  for (uint32_t k0 = (blockIdx.x * (blockDim.x / G) + threadIdx.x / G) * 2; k0 < n; k0 += n_groups * 2) {
    // two requests' worth of loads in flight per lane group
    float* prow[2];
    const float* g0[2];
    bool act[2];
    StepCtx sc[2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const uint32_t k = k0 + u;
      act[u] = k < n && gok[k < n ? k : 0] != 0u;
      uint32_t row = act[u] ? own_row[k] : ROW_NONE;
      if (act[u] && row_missing(row, t, lane, true)) act[u] = false;
      prow[u] = t.rows + (size_t)(act[u] ? row : 0u) * t.stride;
      g0[u] = grads + (size_t)(act[u] ? k : 0u) * t.dim;
      // this request's (beta1^t, beta2^t) of the row's feature group
      const uint32_t akey = act[u] && op.kind == PB_OPT_ADAM ? adam_key_of(x, x_sign(x, x.rank)[(size_t)src * x.cap + k]) : 0u;
      sc[u] = step_ctx(op, (act[u] && op.kind == PB_OPT_ADAGRAD_VW) ? prow[u][t.dim] : 0.0f, owner_adam_pair(x, src, akey));
    }
    for (uint32_t c = lane; c < nvec; c += G) {
      RowElems<-1, VEC, INTEL> rc[2];
      float g[2][VEC];
#pragma unroll
      for (int u = 0; u < 2; ++u)
        if (act[u]) {
          rc[u].load(prow[u], c * VEC, t, op);
          load_vec<VEC>(g0[u] + c * VEC, g[u]);
        }
#pragma unroll
      for (int u = 0; u < 2; ++u)
        if (act[u]) {
          rc[u].step(c * VEC, g[u], t, op, hy, sc[u]);
          rc[u].store(prow[u], c * VEC, t, op);
        }
    }
    if (op.kind == PB_OPT_ADAGRAD_VW) {
#pragma unroll
      for (int u = 0; u < 2; ++u)
        if (act[u]) vw_state_step(prow[u], g0[u], t, op, sc[u], lane, gmask);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// raw slot over R shards (pb_forward_raw_sharded / pb_backward_raw_sharded).  The requester numbers the slot's distinct
// signs like pb_forward_raw (pb_raw.cu), then every distinct sign is one entry of its owner's request:
//   k_raw_route  sign -> owner's area; target[u] = owner * cap + slot, kept for the fill and the backward
//   k_raw_fill   received f32 row -> table row u + 1, rounded once (f16(row): a -0 stays -0); row 0 and misses zeros
//                (rows: the receive area, or a remote read's staging, pb_remote.cu; target[u] indexes it either way)
//   k_raw_send   the [U, dim] gradient, +-inf clamped and unscaled, -> owner's gradient area with its apply word
// The owner's side is the summation path's: k_owner_lookup, then k_owner_update_all / k_owner_update.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_raw_route(RawWork w, XchgDev x) {
  const uint32_t n_items = w.counts[0];
  if (blockIdx.x * blockDim.x >= n_items) return;  // whole block (the grid is sized for the worst case)
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t u = blockIdx.x * blockDim.x + threadIdx.x;
  const bool valid = u < n_items;
  uint32_t owner = 0xFFFFFFFFu;
  uint64_t sign = 0;
  if (valid) {
    sign = w.set[w.distinct_cell[u]].key;  // (the sign 2^64-1 has the set's extra cell, whose key stays 2^64-1)
    owner = (uint32_t)(farmhash64_u64(sign) % x.R);  // sign_to_shard_modulo, mod.rs:341-345
  }
  __shared__ uint32_t s_n[PB_MAX_RANKS], s_g[PB_MAX_RANKS];
  if (threadIdx.x < PB_MAX_RANKS) s_n[threadIdx.x] = 0;
  __syncthreads();
  const uint32_t peers = __match_any_sync(0xffffffffu, owner);
  const uint32_t leader = __ffs(peers) - 1;
  uint32_t k = 0;
  if (valid && lane == leader) k = atomicAdd(&s_n[owner], (uint32_t)__popc(peers));
  k = __shfl_sync(0xffffffffu, k, leader) + __popc(peers & ((1u << lane) - 1u));
  __syncthreads();
  if (threadIdx.x < x.R && s_n[threadIdx.x]) s_g[threadIdx.x] = atomicAdd(&w.peer[threadIdx.x], s_n[threadIdx.x]);
  __syncthreads();
  if (!valid) return;
  k += s_g[owner];
  uint32_t target = ROW_NONE;
  if (k < x.cap) {
    target = owner * x.cap + k;
    x_sign(x, owner)[(size_t)x.rank * x.cap + k] = sign;  // over NVLink when owner != rank
  } else {
    x.err[0] = 1u;  // the pair needs more than cap slots: the caller re-runs the batch with a larger cap
  }
  w.target[u] = target;
}

__global__ void __launch_bounds__(256) k_raw_fill(const uint32_t* __restrict__ counts, const uint32_t* __restrict__ target,
                                                  uint32_t dim, const float* __restrict__ rows, __half* __restrict__ out,
                                                  uint32_t G) {
  const uint32_t r = (blockIdx.x * blockDim.x + threadIdx.x) / G;  // table row
  const uint32_t lane = threadIdx.x % G;
  if (r > counts[0]) return;
  const uint32_t tg = r ? target[r - 1] : ROW_NONE;
  const float* src = rows + (size_t)(tg == ROW_NONE ? 0u : tg) * dim;
  __half* o = out + (size_t)r * dim;
  for (uint32_t e = lane; e < dim; e += G) o[e] = __float2half_rn(tg == ROW_NONE ? 0.0f : src[e]);  // ndarray_f32_to_f16: RNE
}

template <bool F16>
__global__ void __launch_bounds__(256) k_raw_send(const void* __restrict__ grad, const uint32_t* __restrict__ counts,
                                                  const uint32_t* __restrict__ target, uint32_t dim, float inv_scale,
                                                  int do_scale, const uint32_t* __restrict__ tick,
                                                  const uint32_t* __restrict__ nan_tick, XchgDev x, uint32_t G) {
  const uint32_t U = counts[0];
  // add_skipped_gradient, or a NaN anywhere in the gradient (mod.rs:731-746): the whole request is dropped
  const bool drop = grad == nullptr || nan_tick[0] == *tick;
  const uint32_t lane = threadIdx.x % G;
  const uint32_t n_groups = gridDim.x * (blockDim.x / G);
  for (uint32_t u = (blockIdx.x * blockDim.x + threadIdx.x) / G; u < U; u += n_groups) {
    const uint32_t tg = target[u];
    if (tg == ROW_NONE) continue;  // over cap: the sign was never looked up
    const uint32_t owner = tg / x.cap;
    const size_t j = (size_t)x.rank * x.cap + tg % x.cap;  // this request's entry in the owner's area
    if (!drop) {
      float* dst = reinterpret_cast<float*>(x.base[owner] + x.off_grad) + j * dim;
      for (uint32_t e = lane; e < dim; e += G) {
        const size_t i = (size_t)u * dim + e;
        float v;
        if (F16) {  // f16 -> f32 with +-inf -> +-65504 (persia-common lib.rs:163-180)
          v = __half2float(reinterpret_cast<const __half*>(grad)[i]);
          if (v == INFINITY) v = 65504.0f;
          else if (v == -INFINITY) v = -65504.0f;
        } else {
          v = reinterpret_cast<const float*>(grad)[i];
        }
        // x 1/scale_factor (mod.rs:751-755), rounded, then added into a zeroed row (mod.rs:780-798), so -0 -> +0.
        // Not one fma: a negative product that underflows rounds to -0, and only the separate add makes it +0.
        dst[e] = __fadd_rn(do_scale ? __fmul_rn(v, inv_scale) : v, 0.0f);
      }
    }
    if (lane == 0) reinterpret_cast<uint32_t*>(x.base[owner] + x.off_gok)[j] = drop ? 0u : 1u;
  }
}

static uint32_t lanes_for(uint32_t dim) {
  uint32_t G = 1;
  while (G < dim && G < 32) G <<= 1;
  return G;
}

void launch_raw_route(const RawWork& w, uint32_t n, const XchgDev& x, cudaStream_t st) {
  if (!n) return;
  PB_LAUNCH_F(FAM_ROUTE, k_raw_route, cdiv(n, 256), 256, 0, st, w, x);
}

void launch_raw_fill(const RawWork& w, uint32_t n, uint32_t dim, const float* rows, void* table_f16, cudaStream_t st) {
  const uint32_t G = lanes_for(dim);
  PB_LAUNCH_F(FAM_GATHER, k_raw_fill, cdiv((uint64_t)(n + 1) * G, 256), 256, 0, st, w.counts, w.target, dim, rows,
              reinterpret_cast<__half*>(table_f16), G);
}

void launch_raw_send(const void* grad, bool f16, const RawWork& w, uint32_t n, uint32_t dim, float inv_scale,
                     bool do_scale, const uint32_t* tick, const uint32_t* nan_tick, const XchgDev& x, cudaStream_t st) {
  if (!n) return;
  const uint32_t G = lanes_for(dim);
  const uint32_t full = cdiv((uint64_t)n * G, 256);
  const uint32_t grid = full < PB_NUM_SMS * 4u ? full : PB_NUM_SMS * 4u;
  if (f16) PB_LAUNCH_F(FAM_ROUTE, k_raw_send<true>, grid, 256, 0, st, grad, w.counts, w.target, dim, inv_scale, do_scale ? 1 : 0, tick, nan_tick, x, G);
  else PB_LAUNCH_F(FAM_ROUTE, k_raw_send<false>, grid, 256, 0, st, grad, w.counts, w.target, dim, inv_scale, do_scale ? 1 : 0, tick, nan_tick, x, G);
}

// ------------------------------------------------------------------------------------------------
// launchers (host)
// ------------------------------------------------------------------------------------------------
void launch_route_items(bool training, const SlotsDev& sl, const BatchDev& b, const XchgDev& x, cudaStream_t st) {
  if (!b.n) return;
  const uint32_t grid = cdiv(b.n, 256);  // worst case U = N; blocks past the item count return at once
  if (training) PB_LAUNCH_F(FAM_ROUTE, (k_route_items<true>), grid, 256, 0, st, sl, b, x);
  else PB_LAUNCH_F(FAM_ROUTE, (k_route_items<false>), grid, 256, 0, st, sl, b, x);
}

void launch_link_items(const SlotsDev& sl, const BatchDev& b, const XchgDev& x, const GroupLinks& gl, cudaStream_t st) {
  if (!b.n) return;
  const uint32_t full = cdiv(b.n, 256);  // worst case U = N; the blocks stride over the items
  PB_LAUNCH_F(FAM_ROUTE, k_link_items, full < PB_NUM_SMS * 4u ? full : PB_NUM_SMS * 4u, 256, 0, st, sl, b, x, gl);
}

void launch_signal(const XchgDev& x, int phase, const uint32_t* counts, cudaStream_t st) {
  PB_LAUNCH_F(FAM_ROUTE, k_signal, 1, 32, 0, st, x, phase, counts);
}

void launch_signal_wait(const XchgDev& x, int phase, const uint32_t* counts, cudaStream_t st) {
  PB_LAUNCH_F(FAM_WAIT, k_signal_wait, 1, 32, 0, st, x, phase, counts);
}
void launch_wait(const XchgDev& x, int phase, int src, cudaStream_t st) {
  PB_LAUNCH_F(FAM_WAIT, k_wait, 1, 32, 0, st, x, phase, src);
}

void launch_owner_lookup(bool training, const TableDev& t, const TableDev* tier, const HyperDev& hy, const OptimDev& op,
                         const XchgDev& x, cudaStream_t st) {
  const uint32_t full = cdiv((uint64_t)x.R * x.cap * BUCKET, 256);
  const uint32_t grid = full < PB_NUM_SMS * PB_PROBE_BLOCKS ? full : PB_NUM_SMS * PB_PROBE_BLOCKS;
  if (tier && !training) {  // inference reads tier-held signs in place
    if (x.row_f32) PB_LAUNCH_F(FAM_PROBE, k_owner_lookup_tier<true>, grid, 256, 0, st, t, *tier, hy, op, x);
    else PB_LAUNCH_F(FAM_PROBE, k_owner_lookup_tier<false>, grid, 256, 0, st, t, *tier, hy, op, x);
  } else if (training) {
    if (x.row_f32) PB_LAUNCH_F(FAM_PROBE, (k_owner_lookup<MODE_TRAIN, true>), grid, 256, 0, st, t, hy, op, x);
    else PB_LAUNCH_F(FAM_PROBE, (k_owner_lookup<MODE_TRAIN, false>), grid, 256, 0, st, t, hy, op, x);
  } else {
    if (x.row_f32) PB_LAUNCH_F(FAM_PROBE, (k_owner_lookup<MODE_FIND, true>), grid, 256, 0, st, t, hy, op, x);
    else PB_LAUNCH_F(FAM_PROBE, (k_owner_lookup<MODE_FIND, false>), grid, 256, 0, st, t, hy, op, x);
  }
}

void launch_expand_items(const TableDev& t, const SlotsDev& sl, const BatchDev& b, const void* rows, bool row_f32,
                         const uint32_t* row_off, uint32_t n_out, uint32_t batch, bool training, void* out_f16,
                         cudaStream_t st) {
  if (!n_out) return;
  __half* out = reinterpret_cast<__half*>(out_f16);
  if (!row_off && !row_f32 && t.dim % 8 == 0) {
    uint32_t words = t.dim / 8, lanes = 1;
    while (lanes < words && lanes < 32) lanes <<= 1;
    uint32_t grid = cdiv((uint64_t)n_out * lanes, 256);
    if (grid < cdiv(n_out, 256)) grid = cdiv(n_out, 256);
    if (training) PB_LAUNCH_F(FAM_GATHER, (k_expand_copy<true>), grid, 256, 0, st, t.dim, sl, b, rows, n_out, out, lanes);
    else PB_LAUNCH_F(FAM_GATHER, (k_expand_copy<false>), grid, 256, 0, st, t.dim, sl, b, rows, n_out, out, lanes);
    return;
  }
  uint32_t G = 1;
  while (G < t.dim && G < 32) G <<= 1;
  const uint32_t grid = cdiv((uint64_t)n_out * G, 256);
#define PB_E(TR, F32) PB_LAUNCH_F(FAM_GATHER, (k_expand_pool<TR, F32>), grid, 256, 0, st, t.dim, sl, b, rows, row_off, n_out, batch, out, G)
  if (training) {
    if (row_f32) PB_E(true, true);
    else PB_E(true, false);
  } else {
    if (row_f32) PB_E(false, true);
    else PB_E(false, false);
  }
#undef PB_E
}

void launch_uclear(const XchgDev& x, cudaStream_t st) { PB_LAUNCH(k_uclear, PB_NUM_SMS * 4, 256, 0, st, x); }

void launch_owner_update(const TableDev& t, const OptimDev& op, const HyperDev& hy, const XchgDev& x, uint32_t src,
                         cudaStream_t st);

template <int VEC, int CPL>
static void owner_update_all_kind(const TableDev& t, const OptimDev& op, const HyperDev& hy, const XchgDev& x, uint32_t G,
                                  uint32_t grid, cudaStream_t st) {
  const bool intel = op.rsqrt == PB_RSQRT_INTEL;
  if (op.kind == PB_OPT_SGD) PB_LAUNCH_F(FAM_OWNER, (k_owner_update_all<VEC, CPL, PB_OPT_SGD>), grid, 256, 0, st, t, op, hy, x, G);
  else if (op.kind == PB_OPT_ADAGRAD && intel) PB_LAUNCH_F(FAM_OWNER, (k_owner_update_all<VEC, CPL, PB_OPT_ADAGRAD, true>), grid, 256, 0, st, t, op, hy, x, G);
  else if (op.kind == PB_OPT_ADAGRAD) PB_LAUNCH_F(FAM_OWNER, (k_owner_update_all<VEC, CPL, PB_OPT_ADAGRAD>), grid, 256, 0, st, t, op, hy, x, G);
  else if (op.kind == PB_OPT_ADAGRAD_VW && intel) PB_LAUNCH_F(FAM_OWNER, (k_owner_update_all<VEC, CPL, -1, true>), grid, 256, 0, st, t, op, hy, x, G);
  else PB_LAUNCH_F(FAM_OWNER, (k_owner_update_all<VEC, CPL, -1>), grid, 256, 0, st, t, op, hy, x, G);
}

void launch_owner_update_all(const TableDev& t, const OptimDev& op, const HyperDev& hy, const XchgDev& x, cudaStream_t st) {
  int vec, Gi;
  vec_group(t.dim, vec, Gi);  // Gi lanes cover a row with one chunk each (a power of two <= 32)
  const uint32_t full = cdiv((uint64_t)x.R * x.cap * 4u, 256);  // a warp per eight requests
  const uint32_t grid = full < PB_NUM_SMS * 6u ? full : PB_NUM_SMS * 6u;
  const uint32_t nvec = t.dim / (uint32_t)vec;
  const bool exact = (uint32_t)Gi == nvec;  // (rows longer than 32 chunks keep one chunk per lane and stride)
  if (vec == 4 && exact) owner_update_all_kind<4, 1>(t, op, hy, x, (uint32_t)Gi, grid, st);
  else if (vec == 1 && exact) owner_update_all_kind<1, 1>(t, op, hy, x, (uint32_t)Gi, grid, st);
  else {  // long or odd rows: one request after another with the striding kernel
    for (uint32_t src = 0; src < x.R; ++src) launch_owner_update(t, op, hy, x, src, st);
    launch_uclear(x, st);
  }
}

void launch_owner_update(const TableDev& t, const OptimDev& op, const HyperDev& hy, const XchgDev& x, uint32_t src,
                         cudaStream_t st) {
  int vec, Gi;
  vec_group(t.dim, vec, Gi);
  const uint32_t G = (uint32_t)Gi;
  const uint32_t full = cdiv((uint64_t)cdiv(x.cap, 2) * G, 256);
  const uint32_t grid = full < PB_NUM_SMS * 6u ? full : PB_NUM_SMS * 6u;
  if (op.rsqrt == PB_RSQRT_INTEL) {
    if (vec == 4) PB_LAUNCH_F(FAM_UPDATE, (k_owner_update<4, true>), grid, 256, 0, st, t, op, hy, x, src, G);
    else PB_LAUNCH_F(FAM_UPDATE, (k_owner_update<1, true>), grid, 256, 0, st, t, op, hy, x, src, G);
  } else {
    if (vec == 4) PB_LAUNCH_F(FAM_UPDATE, (k_owner_update<4>), grid, 256, 0, st, t, op, hy, x, src, G);
    else PB_LAUNCH_F(FAM_UPDATE, (k_owner_update<1>), grid, 256, 0, st, t, op, hy, x, src, G);
  }
}

}  // namespace pb
