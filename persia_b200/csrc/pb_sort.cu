// pb_sort.cu — stable LSD radix partition of a batch's signs by shard (SURVEY.md §8a row A3).
//
// "Warp-radix partition": ranks inside a warp come from __match_any_sync, across warps from per-warp digit
// counters in shared memory, across blocks from a block-major digit histogram that every scatter block folds
// itself (no separate scan kernel).  A scatter pass also builds the histogram of the next pass with global
// REDs on each element's destination tile, so a k-pass sort is 1 + k launches.  Digits are 9 bits.
//
// Use: pb_partition_by_shard: key = farmhash64(sign) % R, one pass (indices_to_sharded_indices, mod.rs:454-479).
// (Round 1 also grouped the backward's occurrences with it; the batched path now dedups first, pb_dedup.cu.)
#include "pb_group.cuh"

namespace pb {

template <typename SRC>
__global__ void __launch_bounds__(RS_THREADS) k_radix_hist(SRC src, uint32_t n, uint32_t tile,
                                                           uint32_t* __restrict__ keys_out, uint32_t* __restrict__ hist,
                                                           uint32_t* __restrict__ z1, uint32_t* __restrict__ z2,
                                                           uint32_t* __restrict__ z3, uint32_t* __restrict__ zero4) {
  radix_hist_body(blockIdx.x, src, n, tile, keys_out, hist, z1, z2, z3, zero4);
}
template <typename VALOP>
__global__ void __launch_bounds__(RS_THREADS) k_radix_scatter(const uint32_t* __restrict__ keys_in,
                                                              const uint32_t* __restrict__ vals_in,
                                                              uint32_t* __restrict__ keys_out,
                                                              uint32_t* __restrict__ vals_out, uint32_t n, uint32_t shift,
                                                              uint32_t tile, VALOP vop, const uint32_t* __restrict__ hist,
                                                              uint32_t* __restrict__ hist_next) {
  radix_scatter_body(blockIdx.x, gridDim.x, keys_in, vals_in, keys_out, vals_out, n, shift, tile, vop, hist, hist_next);
}

// per-shard group sizes of a single-pass partition: column sums of the block-major histogram
__global__ void k_counts_from_hist(const uint32_t* __restrict__ hist, uint32_t n_blocks, uint32_t R,
                                   uint32_t* __restrict__ counts) {
  uint32_t d = threadIdx.x;
  if (d >= R) return;
  uint32_t t = 0;
  for (uint32_t c = 0; c * RS_COARSE < n_blocks; ++c) t += hist[c * RS_BINS + d];  // coarse rows hold the column sums
  counts[d] = t;
}

// ------------------------------------------------------------------------------------------------
// launchers (host)
// ------------------------------------------------------------------------------------------------
uint32_t radix_tile(uint32_t n) {
  // tiles are multiples of the 512-key sub-tile; at most 256 of them so that folding the block-major
  // histogram inside every scatter block stays cheap
  uint32_t tile = RS_SUB;
  while (cdiv(n, tile) > RS_MAX_TILES) tile += RS_SUB;
  return tile;
}
uint32_t radix_hist_words() { return (uint32_t)(RS_COARSE_ROWS + RS_MAX_TILES) * RS_BINS; }  // one pass's region
uint32_t radix_hist_zero_words(uint32_t n) {  // what must be zero before the histogram pass of an n-key sort
  return (uint32_t)(RS_COARSE_ROWS + cdiv(n ? n : 1, radix_tile(n ? n : 1))) * RS_BINS;
}

void launch_zero_words(uint32_t* p, uint32_t n_words, cudaStream_t st);

__global__ void k_zero_words(uint32_t* p, uint32_t n) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) p[i] = 0;
}
void launch_zero_words(uint32_t* p, uint32_t n_words, cudaStream_t st) {
  if (n_words) PB_LAUNCH(k_zero_words, cdiv(n_words, 1024) < PB_NUM_SMS ? cdiv(n_words, 1024) : PB_NUM_SMS, 256, 0, st, p, n_words);
}

// d_work layout: [one pass's histogram region][n materialised shard ids]
uint64_t partition_workspace_bytes(uint32_t n) { return ((uint64_t)radix_hist_words() + n) * sizeof(uint32_t); }

void launch_partition_by_shard(const uint64_t* signs, uint32_t n, uint32_t R, uint32_t* perm, uint32_t* counts,
                               uint32_t* work, cudaStream_t st) {
  uint32_t tile = radix_tile(n ? n : 1), nb = cdiv(n ? n : 1, tile);
  uint32_t* hist = work;
  uint32_t* keys = work + radix_hist_words();
  SrcShard src{signs, R};
  launch_zero_words(hist, radix_hist_zero_words(n), st);
  if (n)
    PB_LAUNCH((k_radix_hist<SrcShard>), cdiv(n, RH_KEYS), RS_THREADS, 0, st, src, n, tile, keys, hist, (uint32_t*)nullptr,
              (uint32_t*)nullptr, (uint32_t*)nullptr, (uint32_t*)nullptr);
  PB_LAUNCH(k_counts_from_hist, 1, 256, 0, st, hist, nb, R, counts);
  if (n)
    PB_LAUNCH((k_radix_scatter<ValIdentity>), nb, RS_THREADS, 0, st, keys, (const uint32_t*)nullptr, (uint32_t*)nullptr,
              perm, n, 0u, tile, ValIdentity(), hist, (uint32_t*)nullptr);
}

}  // namespace pb
