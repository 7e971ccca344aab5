// pb_update.cu — the NaN rule of the backward (A8), pb_update's direct optimizer step and Adam's batch-level state.
// The batched reduce + step is pb_reduce.cu.  SURVEY.md §8a.
#include "pb_optim.cuh"

namespace pb {

// ------------------------------------------------------------------------------------------------
// A8 (NaN rule): a slot whose gradient holds any NaN is skipped whole (mod.rs:731-746).
// grid.y = slot.  status[s] = tick when a NaN was seen (no reset needed between batches).
// The scan runs beside k_reduce_hot, which holds most of every SM's registers and shared memory, so only a few of its
// warps fit on an SM: each thread has NAN_LOADS independent 16-byte loads in flight before it tests any, and the
// register cap (__launch_bounds__ below: <= 32 per thread) lets two 256-thread blocks sit beside a hot block of up to
// 192 registers per thread.  (A 24-register cap would serialise the loads two by two.)
// ------------------------------------------------------------------------------------------------
constexpr uint32_t NAN_LOADS = 4;
constexpr uint32_t NAN_TRIPS = 4;  // loop trips per thread the grid is sized for (up to 4 blocks per SM and slot)

template <bool F16>
__device__ __forceinline__ bool nan_bits(uint32_t w) {
  if (F16) return ((w & 0x7fffu) > 0x7c00u) | (((w >> 16) & 0x7fffu) > 0x7c00u);
  return (w & 0x7fffffffu) > 0x7f800000u;
}

template <bool F16>
__global__ void __launch_bounds__(256, 8) k_nan_scan(GradsDev gr, uint32_t elems_per_slot,
                                                      const uint32_t* __restrict__ tick_ptr,
                                                      uint32_t* __restrict__ nan_tick) {
  const uint32_t s = blockIdx.y;
  const void* base = gr.ptr[s];
  if (!base) return;
  bool bad = false;
  const uint32_t stride = gridDim.x * blockDim.x;
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  // 8 halves or 4 floats per 16-byte load; the ABI refuses gradient pointers that are not 16-byte aligned
  constexpr uint32_t EV = F16 ? 8u : 4u;
  const uint4* p = reinterpret_cast<const uint4*>(base);
  const uint32_t nv = elems_per_slot / EV;
  for (uint32_t j = i; j < nv; j += NAN_LOADS * stride) {
    uint4 v[NAN_LOADS];
#pragma unroll
    for (uint32_t u = 0; u < NAN_LOADS; ++u) v[u] = j + u * stride < nv ? p[j + u * stride] : make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
    for (uint32_t u = 0; u < NAN_LOADS; ++u)
      bad |= nan_bits<F16>(v[u].x) | nan_bits<F16>(v[u].y) | nan_bits<F16>(v[u].z) | nan_bits<F16>(v[u].w);
  }
  for (uint32_t j = nv * EV + i; j < elems_per_slot; j += stride) {
    bad |= F16 ? nan_bits<true>(reinterpret_cast<const uint16_t*>(base)[j])
               : nan_bits<false>(reinterpret_cast<const uint32_t*>(base)[j]);
  }
  if (__any_sync(0xffffffffu, bad) && (threadIdx.x & 31) == 0) nan_tick[s] = *tick_ptr;
}

__global__ void k_slot_status(GradsDev gr, uint32_t n_slots, const uint32_t* __restrict__ tick_ptr,
                              const uint32_t* __restrict__ nan_tick, int32_t* __restrict__ status) {
  uint32_t s = threadIdx.x;
  const uint32_t tick = *tick_ptr;
  if (s < n_slots) status[s] = !gr.ptr[s] ? 1 : (nan_tick[s] == tick ? 2 : 0);
}

// pb_update: distinct signs with explicit f32 gradients (update_gradient_mixed, PS mod.rs:359-427); the raw backward
// (by_row: the rows its forward found).
template <int VEC, int G, bool INTEL = false>
__global__ void __launch_bounds__(256) k_update_direct(TableDev t, OptimDev op, HyperDev hy, int by_row,
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
  uint32_t row = by_row ? h : (h < t.n_cells + N_SPECIAL) ? t.cells[h].row : ROW_NONE;
  if (row_missing(row, t, lane, true)) return;
  float* prow = t.rows + (size_t)row * t.stride;
  const StepCtx sc = step_ctx(op, op.kind == PB_OPT_ADAGRAD_VW ? prow[t.dim] : 0.0f, adam_pair);
  const float* g0 = grads + (size_t)gid * t.dim;
  step_row<-1, VEC, INTEL>(prow, t, op, hy, sc, lane, G, [&](uint32_t e0, float (&g)[VEC]) { load_vec<VEC>(g0 + e0, g); });
  if (op.kind == PB_OPT_ADAGRAD_VW) vw_state_step(prow, g0, t, op, sc, lane, group_mask(G));
}

// ------------------------------------------------------------------------------------------------
// launchers (host)
// ------------------------------------------------------------------------------------------------
void launch_nan_scan(const GradsDev& gr, uint32_t n_slots, uint32_t elems_per_slot, bool f16, const uint32_t* tick,
                     uint32_t* nan_tick, int32_t* status, cudaStream_t st) {
  const uint32_t per = elems_per_slot / (f16 ? 8u : 4u);  // 16-byte loads per slot
  uint32_t gx = cdiv(per ? per : 1, 256 * NAN_LOADS * NAN_TRIPS);
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

void launch_update_direct(const TableDev& t, const OptimDev& op, const HyperDev& hy, const uint32_t* where,
                          const float* grads, uint32_t n, const float* adam_pair, cudaStream_t st,
                          const uint32_t* n_ptr, const uint32_t* tick, const uint32_t* nan_tick, bool by_row) {
  if (!n) return;
  int vec, G;
  vec_group(t.dim, vec, G);
  uint32_t grid = cdiv((uint64_t)n * G, 256);
  const bool intel = op.rsqrt == PB_RSQRT_INTEL;
#define PB_U(V, GG)                                                                                                 \
  if (vec == V && G == GG) {                                                                                        \
    if (intel)                                                                                                      \
      PB_LAUNCH_F(FAM_UPDATE, (k_update_direct<V, GG, true>), grid, 256, 0, st, t, op, hy, by_row ? 1 : 0, where,   \
                  grads, n, adam_pair, n_ptr, tick, nan_tick);                                                      \
    else                                                                                                            \
      PB_LAUNCH_F(FAM_UPDATE, (k_update_direct<V, GG>), grid, 256, 0, st, t, op, hy, by_row ? 1 : 0, where, grads, n, \
                  adam_pair, n_ptr, tick, nan_tick);                                                                \
  }
  PB_U(4, 1) PB_U(4, 2) PB_U(4, 4) PB_U(4, 8) PB_U(4, 16) PB_U(4, 32)
  PB_U(1, 1) PB_U(1, 2) PB_U(1, 4) PB_U(1, 8) PB_U(1, 16) PB_U(1, 32)
#undef PB_U
}

}  // namespace pb
