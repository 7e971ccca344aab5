// pb_raw.cu — raw (embedding_summation = false) slots.
//
// Reference: FeatureRawEmbeddingBatch, embedding_worker_service/mod.rs:498-512 (table of distinct signs, row 0
// = zeros), :540-545 (row idx+1 = the sign's embedding), :593-623 (index / sample_id_num), persia-core
// forward.rs:336-347 (non_empty_index) and the raw arm of update_all_batched_gradients, mod.rs:790-798 (the
// gradient of distinct sign u is row u of the [U, dim] gradient tensor; no reduction).
//
// The reference numbers distinct signs in hashbrown iteration order (unpinned, random per process); here the
// number of a sign is the rank of its first occurrence in the flat id array, which is what oracle/ uses too.
// Distinct signs are found in a per-batch scratch set (independent of the table: signs without storage still
// get a number and read as zeros, like a lookup miss in the reference).
#include <cuda_fp16.h>

#include "pb_device.cuh"

namespace pb {

namespace {

constexpr uint32_t SCAN_THREADS = 256;
constexpr uint32_t SCAN_ITEMS = 4;
constexpr uint32_t SCAN_TILE = SCAN_THREADS * SCAN_ITEMS;

__device__ __forceinline__ uint32_t warp_incl_scan(uint32_t v) {
  const uint32_t lane = threadIdx.x & 31;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    uint32_t o = __shfl_up_sync(0xffffffffu, v, d);
    if (lane >= (uint32_t)d) v += o;
  }
  return v;
}

// exclusive scan of one value per thread across the block; *total = block sum
__device__ uint32_t block_excl_scan(uint32_t v, uint32_t* total) {
  __shared__ uint32_t warp_sum[32];
  const uint32_t lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  uint32_t inc = warp_incl_scan(v);
  if (lane == 31) warp_sum[w] = inc;
  __syncthreads();
  if (w == 0) {
    uint32_t s = lane < nw ? warp_sum[lane] : 0;
    uint32_t si = warp_incl_scan(s);
    warp_sum[lane] = si - s;
    if (lane == 31) *total = si;  // lane 31 holds the block total
  }
  __syncthreads();
  uint32_t r = inc - v + warp_sum[w];
  __syncthreads();
  return r;
}

__global__ void __launch_bounds__(SCAN_THREADS) k_scan_tiles(const uint32_t* __restrict__ in, uint32_t n,
                                                             uint32_t* __restrict__ tiles) {
  __shared__ uint32_t tot;
  uint32_t base = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_ITEMS;
  uint32_t s = 0;
#pragma unroll
  for (uint32_t k = 0; k < SCAN_ITEMS; ++k)
    if (base + k < n) s += in[base + k];
  block_excl_scan(s, &tot);
  if (threadIdx.x == 0) tiles[blockIdx.x] = tot;
}

// one block: exclusive scan of the tile sums in place, grand total to *total
__global__ void __launch_bounds__(1024) k_scan_spine(uint32_t* __restrict__ tiles, uint32_t n_tiles,
                                                     uint32_t* __restrict__ total) {
  __shared__ uint32_t tot;
  uint32_t carry = 0;
  for (uint32_t b = 0; b < n_tiles; b += blockDim.x) {
    uint32_t i = b + threadIdx.x;
    uint32_t v = i < n_tiles ? tiles[i] : 0;
    uint32_t e = block_excl_scan(v, &tot);
    if (i < n_tiles) tiles[i] = carry + e;
    carry += tot;
    __syncthreads();
  }
  if (threadIdx.x == 0) *total = carry;
}

__global__ void __launch_bounds__(SCAN_THREADS) k_scan_apply(const uint32_t* __restrict__ in, uint32_t n,
                                                             const uint32_t* __restrict__ tiles,
                                                             uint32_t* __restrict__ out) {
  __shared__ uint32_t tot;
  uint32_t base = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_ITEMS;
  uint32_t v[SCAN_ITEMS], s = 0;
#pragma unroll
  for (uint32_t k = 0; k < SCAN_ITEMS; ++k) {
    v[k] = base + k < n ? in[base + k] : 0;
    s += v[k];
  }
  uint32_t e = block_excl_scan(s, &tot) + tiles[blockIdx.x];
#pragma unroll
  for (uint32_t k = 0; k < SCAN_ITEMS; ++k) {
    if (base + k < n) out[base + k] = e;
    e += v[k];
  }
}

void exclusive_scan(const uint32_t* in, uint32_t* out, uint32_t n, uint32_t* tiles, uint32_t* total, cudaStream_t st) {
  uint32_t nt = cdiv(n ? n : 1, SCAN_TILE);
  PB_LAUNCH(k_scan_tiles, nt, SCAN_THREADS, 0, st, in, n, tiles);
  PB_LAUNCH(k_scan_spine, 1, 1024, 0, st, tiles, nt, total);
  PB_LAUNCH(k_scan_apply, nt, SCAN_THREADS, 0, st, in, n, tiles, out);
}

// ---- distinct signs of the batch ----------------------------------------------------------------
// Scratch set cell: {sign, first occurrence, rank}.  Cleared to 0xFF bytes (key == KEY_EMPTY, first == ~0).
// The sign that equals KEY_EMPTY owns the extra cell at index n_set.
__global__ void __launch_bounds__(256) k_raw_insert(SlotsDev sl, const uint64_t* __restrict__ ids, uint32_t n,
                                                    RawCell* __restrict__ set, uint32_t set_mask,
                                                    uint32_t* __restrict__ occ_set) {
  uint32_t i = blockIdx.x * 256 + threadIdx.x;
  if (i >= n) return;
  uint64_t sign = ids[i];
  const uint64_t p = sl.prefix[0];
  if (p) sign = mod_mersenne(sign, sl.spacing_bits) + p;  // indices_add_prefix, mod.rs:402-429
  uint32_t h;
  if (sign == KEY_EMPTY) {
    h = set_mask + 1;
  } else {
    h = (uint32_t)mix64(sign) & set_mask;
    for (;;) {  // the set holds 2x the occurrences: always terminates on an empty cell
      unsigned long long k = atomicCAS(reinterpret_cast<unsigned long long*>(&set[h].key), KEY_EMPTY, sign);
      if (k == KEY_EMPTY || k == sign) break;
      h = (h + 1) & set_mask;
    }
  }
  atomicMin(&set[h].first, i);
  occ_set[i] = h;
}

__global__ void __launch_bounds__(256) k_raw_flag(const RawCell* __restrict__ set, const uint32_t* __restrict__ occ_set,
                                                  uint32_t n, uint32_t* __restrict__ flag) {
  uint32_t i = blockIdx.x * 256 + threadIdx.x;
  if (i < n) flag[i] = set[occ_set[i]].first == i ? 1u : 0u;
}

// first occurrences publish their sign's number and remember, per distinct sign, its index cell for the backward
// (occ_cell given: the local table's probe) or its cell of the scratch set (occ_cell null: the sharded path, whose
// route kernel reads the sign from there)
__global__ void __launch_bounds__(256) k_raw_assign(RawCell* __restrict__ set, const uint32_t* __restrict__ occ_set,
                                                    const uint32_t* __restrict__ flag,
                                                    const uint32_t* __restrict__ rank,
                                                    const uint32_t* __restrict__ occ_cell, uint32_t n,
                                                    uint32_t* __restrict__ distinct_cell) {
  uint32_t i = blockIdx.x * 256 + threadIdx.x;
  if (i >= n || !flag[i]) return;
  set[occ_set[i]].rank = rank[i];
  distinct_cell[rank[i]] = occ_cell ? occ_cell[i] : occ_set[i];
}

// mod.rs:593-620: index[b * fixed + col] = number + 1 for col < fixed (0 = padding).  The reference's
// `sample_id_num[b] < fixed` guard never fires before every col < fixed of the sample is placed, so the
// result does not depend on the order signs are visited in.
__global__ void __launch_bounds__(256) k_raw_index(const RawCell* __restrict__ set, const uint32_t* __restrict__ occ_set,
                                                   const uint32_t* __restrict__ occ_sample,
                                                   const uint32_t* __restrict__ row_off, uint32_t n, uint32_t fixed,
                                                   long long* __restrict__ index) {
  uint32_t i = blockIdx.x * 256 + threadIdx.x;
  if (i >= n) return;
  uint32_t b = occ_sample ? occ_sample[i] : i;
  uint32_t col = occ_sample ? i - row_off[b] : 0;
  if (col < fixed) index[(size_t)b * fixed + col] = (long long)set[occ_set[i]].rank + 1;
}

__global__ void __launch_bounds__(256) k_raw_sample_num(const uint32_t* __restrict__ row_off, uint32_t batch,
                                                        uint32_t fixed, uint32_t* __restrict__ sample_id_num) {
  uint32_t b = blockIdx.x * 256 + threadIdx.x;
  if (b >= batch) return;
  uint32_t len = row_off ? row_off[b + 1] - row_off[b] : 1;
  sample_id_num[b] = len < fixed ? len : fixed;
}

// forward.rs:336-347: ascending positions of index that hold an id
__global__ void __launch_bounds__(256) k_raw_non_empty(const uint32_t* __restrict__ sample_id_num,
                                                       const uint32_t* __restrict__ off, uint32_t batch,
                                                       uint32_t fixed, long long* __restrict__ non_empty) {
  uint32_t b = blockIdx.x * 256 + threadIdx.x;
  if (b >= batch) return;
  uint32_t m = sample_id_num[b], o = off[b];
  for (uint32_t j = 0; j < m; ++j) non_empty[o + j] = (long long)b * fixed + j;
}

// table row d + 1 = f16(embedding of distinct sign d); zeros when the sign has no storage (lookup miss).  The row
// itself goes to distinct_row[d] for the backward: a cell may move (index rebuild) before the gradients come, a row
// held by a pending batch does not
template <int VEC, int G>
__global__ void __launch_bounds__(256) k_raw_table(TableDev t, const uint32_t* __restrict__ distinct_cell,
                                                   const uint32_t* __restrict__ n_distinct, __half* __restrict__ out,
                                                   uint32_t* __restrict__ distinct_row) {
  const uint32_t d = (blockIdx.x * 256 + threadIdx.x) / G;
  const uint32_t lane = threadIdx.x % G;
  if (d == 0 && blockIdx.x == 0)  // row 0: padding target of index == 0
    for (uint32_t e = lane; e < t.dim; e += G) out[e] = __float2half_rn(0.0f);
  if (d >= *n_distinct) return;
  const uint32_t h = distinct_cell[d];
  const uint32_t row = (h < t.n_cells + N_SPECIAL) ? t.cells[h].row : ROW_NONE;
  if (lane == 0) distinct_row[d] = row < t.capacity ? row : ROW_NONE;
  __half* o = out + (size_t)(d + 1) * t.dim;
  const float* prow = t.rows + (size_t)(row < t.capacity ? row : 0) * t.stride;
  for (uint32_t c = lane; c < t.dim / VEC; c += G) {
    float v[VEC];
    if (row < t.capacity) load_vec<VEC>(prow + c * VEC, v);
    else
#pragma unroll
      for (int k = 0; k < VEC; ++k) v[k] = 0.0f;
#pragma unroll
    for (int k = 0; k < VEC; ++k) o[c * VEC + k] = __float2half_rn(v[k]);  // ndarray_f32_to_f16: RNE
  }
}

// ---- backward ------------------------------------------------------------------------------------
// mod.rs:731-746 on the [U, dim] gradient; U lives on the device
template <bool F16>
__global__ void __launch_bounds__(256) k_raw_nan(const void* __restrict__ grad, const uint32_t* __restrict__ n_distinct,
                                                 uint32_t dim, const uint32_t* __restrict__ tick_ptr,
                                                 uint32_t* __restrict__ nan_tick) {
  const size_t total = (size_t)(*n_distinct) * dim;
  bool bad = false;
  for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (size_t)gridDim.x * 256) {
    if (F16) {
      unsigned short h = reinterpret_cast<const unsigned short*>(grad)[i];
      bad |= ((h & 0x7c00u) == 0x7c00u) && (h & 0x03ffu);
    } else {
      float f = reinterpret_cast<const float*>(grad)[i];
      bad |= f != f;
    }
  }
  if (__any_sync(0xffffffffu, bad) && (threadIdx.x & 31) == 0) nan_tick[0] = *tick_ptr;
}

// f16 -> f32 with +-inf -> +-65504 (persia-common lib.rs:163-180), then x 1/scale_factor (mod.rs:751-755), then
// added into a zeroed row as the EW builds sign_gradients (mod.rs:780-798): a -0 gradient reaches the step as +0
template <bool F16>
__global__ void __launch_bounds__(256) k_raw_stage(const void* __restrict__ grad, const uint32_t* __restrict__ n_distinct,
                                                   uint32_t dim, float inv_scale, int do_scale,
                                                   float* __restrict__ out) {
  const size_t total = (size_t)(*n_distinct) * dim;
  for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (size_t)gridDim.x * 256) {
    float v;
    if (F16) {
      v = __half2float(reinterpret_cast<const __half*>(grad)[i]);
      if (v == INFINITY) v = 65504.0f;
      else if (v == -INFINITY) v = -65504.0f;
    } else {
      v = reinterpret_cast<const float*>(grad)[i];
    }
    // rounded product first, then + 0: a negative product that underflows is -0 and only the add makes it +0
    out[i] = __fadd_rn(do_scale ? __fmul_rn(v, inv_scale) : v, 0.0f);
  }
}

}  // namespace

uint32_t raw_scan_tiles(uint32_t n) { return cdiv(n ? n : 1, SCAN_TILE) + 1; }

void launch_raw_number(const SlotsDev& sl, const uint64_t* ids, uint32_t n, const uint32_t* row_off,
                       const uint32_t* occ_sample, uint32_t batch, uint32_t fixed, const uint32_t* occ_cell,
                       const RawWork& w, long long* index, long long* non_empty, uint32_t* sample_id_num,
                       cudaStream_t st) {
  cudaMemsetAsync(w.set, 0xFF, sizeof(RawCell) * ((size_t)w.set_mask + 2), st);
  cudaMemsetAsync(index, 0, sizeof(long long) * (size_t)batch * fixed, st);
  if (n) {
    const uint32_t g = cdiv(n, 256);
    PB_LAUNCH(k_raw_insert, g, 256, 0, st, sl, ids, n, w.set, w.set_mask, w.occ_set);
    PB_LAUNCH(k_raw_flag, g, 256, 0, st, w.set, w.occ_set, n, w.flag);
  }
  exclusive_scan(w.flag, w.rank, n, w.tiles, w.counts, st);  // counts[0] = distinct signs
  if (n) {
    const uint32_t g = cdiv(n, 256);
    PB_LAUNCH(k_raw_assign, g, 256, 0, st, w.set, w.occ_set, w.flag, w.rank, occ_cell, n, w.distinct_cell);
    PB_LAUNCH(k_raw_index, g, 256, 0, st, w.set, w.occ_set, occ_sample, row_off, n, fixed, index);
  }
  if (batch) {
    PB_LAUNCH(k_raw_sample_num, cdiv(batch, 256), 256, 0, st, row_off, batch, fixed, sample_id_num);
    exclusive_scan(sample_id_num, w.flag, batch, w.tiles, w.counts + 1, st);  // counts[1] = ids placed in index
    PB_LAUNCH(k_raw_non_empty, cdiv(batch, 256), 256, 0, st, sample_id_num, w.flag, batch, fixed, non_empty);
  } else {
    cudaMemsetAsync(w.counts + 1, 0, 4, st);
  }
}

void launch_raw_forward(const TableDev& t, const SlotsDev& sl, const uint64_t* ids, uint32_t n,
                        const uint32_t* row_off, const uint32_t* occ_sample, uint32_t batch, uint32_t fixed,
                        const uint32_t* occ_cell, const RawWork& w, void* table_f16, long long* index,
                        long long* non_empty, uint32_t* sample_id_num, cudaStream_t st) {
  launch_raw_number(sl, ids, n, row_off, occ_sample, batch, fixed, occ_cell, w, index, non_empty, sample_id_num, st);
  int vec, G;
  vec_group(t.dim, vec, G);
  const uint32_t grid = cdiv((uint64_t)(n ? n : 1) * G, 256);
#define PB_T(V, GG) \
  if (vec == V && G == GG) PB_LAUNCH((k_raw_table<V, GG>), grid, 256, 0, st, t, w.distinct_cell, w.counts, (__half*)table_f16, w.target);
  PB_T(4, 1) PB_T(4, 2) PB_T(4, 4) PB_T(4, 8) PB_T(4, 16) PB_T(4, 32)
  PB_T(1, 1) PB_T(1, 2) PB_T(1, 4) PB_T(1, 8) PB_T(1, 16) PB_T(1, 32)
#undef PB_T
}

void launch_raw_nan(const void* grad, bool f16, const uint32_t* n_distinct, uint32_t dim, const uint32_t* tick,
                    uint32_t* nan_tick, cudaStream_t st) {
  if (f16) PB_LAUNCH_F(FAM_NAN, k_raw_nan<true>, PB_NUM_SMS * 2, 256, 0, st, grad, n_distinct, dim, tick, nan_tick);
  else PB_LAUNCH_F(FAM_NAN, k_raw_nan<false>, PB_NUM_SMS * 2, 256, 0, st, grad, n_distinct, dim, tick, nan_tick);
}

void launch_raw_stage(const void* grad, bool f16, const uint32_t* n_distinct, uint32_t dim, float inv_scale,
                      bool do_scale, float* out, cudaStream_t st) {
  if (f16) PB_LAUNCH(k_raw_stage<true>, PB_NUM_SMS * 4, 256, 0, st, grad, n_distinct, dim, inv_scale, do_scale ? 1 : 0, out);
  else PB_LAUNCH(k_raw_stage<false>, PB_NUM_SMS * 4, 256, 0, st, grad, n_distinct, dim, inv_scale, do_scale ? 1 : 0, out);
}

}  // namespace pb
