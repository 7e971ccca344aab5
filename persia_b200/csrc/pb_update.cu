// pb_update.cu — the NaN rule of the backward (A8), pb_update's direct optimizer step and Adam's batch-level state.
// The batched reduce + step is pb_reduce.cu.  SURVEY.md §8a.
#include "pb_optim.cuh"

namespace pb {

// ------------------------------------------------------------------------------------------------
// A8 (NaN rule): a slot whose gradient holds any NaN is skipped whole (mod.rs:731-746).
// grid.y = slot.  status[s] = tick when a NaN was seen (no reset needed between batches).
// ------------------------------------------------------------------------------------------------
template <bool F16>
__global__ void __launch_bounds__(256) k_nan_scan(GradsDev gr, uint32_t elems_per_slot,
                                                  const uint32_t* __restrict__ tick_ptr,
                                                  uint32_t* __restrict__ nan_tick) {
  uint32_t s = blockIdx.y;
  const void* base = gr.ptr[s];
  if (!base) return;
  bool bad = false;
  uint32_t stride = gridDim.x * blockDim.x;
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (F16) {
    // 8 halves per 16 B load; every slot tensor is at least 16 B aligned (torch allocations are 512 B)
    const uint4* p = reinterpret_cast<const uint4*>(base);
    uint32_t nv = elems_per_slot / 8;
    for (uint32_t j = i; j < nv; j += stride) {
      uint4 v = p[j];
      uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        uint32_t lo = w[k] & 0x7fffu, hi = (w[k] >> 16) & 0x7fffu;
        bad |= (lo > 0x7c00u) | (hi > 0x7c00u);
      }
    }
    const uint16_t* q = reinterpret_cast<const uint16_t*>(base);
    for (uint32_t j = nv * 8 + i; j < elems_per_slot; j += stride) bad |= (q[j] & 0x7fffu) > 0x7c00u;
  } else {
    const float* p = reinterpret_cast<const float*>(base);
    for (uint32_t j = i; j < elems_per_slot; j += stride) bad |= isnan(p[j]);
  }
  if (__any_sync(0xffffffffu, bad) && (threadIdx.x & 31) == 0) nan_tick[s] = *tick_ptr;
}

__global__ void k_slot_status(GradsDev gr, uint32_t n_slots, const uint32_t* __restrict__ tick_ptr,
                              const uint32_t* __restrict__ nan_tick, int32_t* __restrict__ status) {
  uint32_t s = threadIdx.x;
  const uint32_t tick = *tick_ptr;
  if (s < n_slots) status[s] = !gr.ptr[s] ? 1 : (nan_tick[s] == tick ? 2 : 0);
}

// pb_update: distinct signs with explicit f32 gradients (update_gradient_mixed, PS mod.rs:359-427).
template <int VEC, int G>
__global__ void __launch_bounds__(256) k_update_direct(TableDev t, OptimDev op, HyperDev hy,
                                                       const uint32_t* __restrict__ occ_cell,
                                                       const float* __restrict__ grads, uint32_t n,
                                                       const float* __restrict__ adam_pair,
                                                       const uint32_t* __restrict__ n_ptr,
                                                       const uint32_t* __restrict__ tick_ptr,
                                                       const uint32_t* __restrict__ nan_tick) {
  uint32_t gid = (blockIdx.x * blockDim.x + threadIdx.x) / G;
  uint32_t lane = threadIdx.x % G;
  if (n_ptr) n = *n_ptr;
  if (gid >= n) return;
  if (nan_tick && nan_tick[0] == *tick_ptr) return;  // NaN rule: the whole gradient is dropped
  uint32_t h = occ_cell[gid];
  uint32_t row = (h < t.n_cells + N_SPECIAL) ? t.cells[h].row : ROW_NONE;
  if (row >= t.capacity) {
    if (lane == 0) atomicAdd(&t.counters[CTR_GRAD_MISS], 1u);
    return;
  }
  float* prow = t.rows + (size_t)row * t.stride;
  const uint32_t nvec = t.dim / VEC;
  StepCtx sc;
  sc.vw_state = (op.kind == PB_OPT_ADAGRAD_VW) ? prow[t.dim] : 0.0f;
  sc.r1 = sc.r2 = 0.0f;
  if (op.kind == PB_OPT_ADAM) {
    sc.r1 = __fdiv_rn(1.0f, __fsub_rn(1.0f, adam_pair[0]));
    sc.r2 = __fdiv_rn(1.0f, __fsub_rn(1.0f, adam_pair[1]));
  }
  const float* g0 = grads + (size_t)gid * t.dim;
  for (uint32_t c = lane; c < nvec; c += G) {
    float g[VEC];
    load_vec<VEC>(g0 + c * VEC, g);
    RowElems<-1, VEC> rc;
    rc.load(prow, c * VEC, t, op);
    rc.step(c * VEC, g, t, op, hy, sc);
    rc.store(prow, c * VEC, t, op);
  }
  if (op.kind == PB_OPT_ADAGRAD_VW && lane == 0) {
    float gs = __fdiv_rn(vw_dot(g0, t.dim), (float)t.dim);
    prow[t.dim] = __fadd_rn(__fmul_rn(sc.vw_state, op.mom), gs);
  }
}

// ------------------------------------------------------------------------------------------------
// launchers (host)
// ------------------------------------------------------------------------------------------------
void launch_nan_scan(const GradsDev& gr, uint32_t n_slots, uint32_t elems_per_slot, bool f16, const uint32_t* tick,
                     uint32_t* nan_tick, int32_t* status, cudaStream_t st) {
  uint32_t per = f16 ? elems_per_slot / 8 : elems_per_slot;
  uint32_t gx = cdiv(per ? per : 1, 256 * 4);
  if (gx > PB_NUM_SMS * 4) gx = PB_NUM_SMS * 4;
  dim3 grid(gx, n_slots);
  if (f16) PB_LAUNCH_F(FAM_NAN, k_nan_scan<true>, grid, 256, 0, st, gr, elems_per_slot, tick, nan_tick);
  else PB_LAUNCH_F(FAM_NAN, k_nan_scan<false>, grid, 256, 0, st, gr, elems_per_slot, tick, nan_tick);
  if (status) PB_LAUNCH(k_slot_status, 1, PB_MAX_SLOTS, 0, st, gr, n_slots, tick, nan_tick, status);
}

// Adam's batch-level state (optim.rs:99-131, 155-197): one (beta1^t, beta2^t) pair per feature group, kept on the
// device so that a captured backward advances it on every replay.
__global__ void k_adam_fill(float* pow, float b1, float b2) {
  uint32_t i = threadIdx.x;
  if (i < PB_ADAM_KEYS) {
    pow[2 * i] = b1;
    pow[2 * i + 1] = b2;
  }
}
// gr / tick / nan_tick (optional): a feature group advances only if one of its slots is applied by this request — a slot
// skipped for a NaN gradient sends nothing to the parameter server (mod.rs:731-746), so it cannot advance the powers
__global__ void k_adam_advance(float* pow, AdamKeys keys, float b1, float b2, GradsDev gr, uint32_t n_slots,
                               const uint32_t* __restrict__ tick, const uint32_t* __restrict__ nan_tick) {
  uint32_t i = threadIdx.x;
  if (i < keys.n) {
    bool applied = nan_tick == nullptr;
    if (!applied) {
      const uint32_t now = *tick;
      for (uint32_t s = 0; s < n_slots; ++s) applied |= gr.ptr[s] && gr.pow_idx[s] == keys.idx[i] && nan_tick[s] != now;
    }
    if (applied) {
      float* p = pow + 2u * keys.idx[i];
      p[0] = __fmul_rn(p[0], b1);
      p[1] = __fmul_rn(p[1], b2);
    }
  }
}
void launch_adam_fill(float* pow, float b1, float b2, cudaStream_t st) { PB_LAUNCH(k_adam_fill, 1, PB_ADAM_KEYS, 0, st, pow, b1, b2); }
void launch_adam_advance(float* pow, const AdamKeys& keys, float b1, float b2, cudaStream_t st, const GradsDev* gr,
                         uint32_t n_slots, const uint32_t* tick, const uint32_t* nan_tick) {
  GradsDev none{};
  if (keys.n) PB_LAUNCH(k_adam_advance, 1, PB_MAX_SLOTS, 0, st, pow, keys, b1, b2, gr ? *gr : none, n_slots, tick, gr ? nan_tick : nullptr);
}

void launch_slot_status(const GradsDev& gr, uint32_t n_slots, const uint32_t* tick, const uint32_t* nan_tick,
                        int32_t* status, cudaStream_t st) {
  PB_LAUNCH(k_slot_status, 1, PB_MAX_SLOTS, 0, st, gr, n_slots, tick, nan_tick, status);
}

void launch_update_direct(const TableDev& t, const OptimDev& op, const HyperDev& hy, const uint32_t* occ_cell,
                          const float* grads, uint32_t n, const float* adam_pair, cudaStream_t st,
                          const uint32_t* n_ptr, const uint32_t* tick, const uint32_t* nan_tick) {
  if (!n) return;
  int vec, G;
  vec_group(t.dim, vec, G);
  uint32_t grid = cdiv((uint64_t)n * G, 256);
#define PB_U(V, GG)                                                                                          \
  if (vec == V && G == GG)                                                                                   \
    PB_LAUNCH_F(FAM_UPDATE, (k_update_direct<V, GG>), grid, 256, 0, st, t, op, hy, occ_cell, grads, n, adam_pair, n_ptr, \
                tick, nan_tick);
  PB_U(4, 1) PB_U(4, 2) PB_U(4, 4) PB_U(4, 8) PB_U(4, 16) PB_U(4, 32)
  PB_U(1, 1) PB_U(1, 2) PB_U(1, 4) PB_U(1, 8) PB_U(1, 16) PB_U(1, 32)
#undef PB_U
}

}  // namespace pb
