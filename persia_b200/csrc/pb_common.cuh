// pb_common.cuh — shared device helpers for libpersia_b200 (sm_90a only).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "persia_b200.h"

namespace pb {

constexpr uint64_t KEY_EMPTY = ~0ULL;          // hash-index cell holds no key
constexpr uint64_t KEY_TOMB = ~0ULL - 2;       // cell whose sign was evicted: probing continues past it, admissions reuse it
constexpr uint32_t N_SPECIAL = 3;              // signs >= KEY_TOMB collide with the markers: each has a reserved cell
constexpr uint32_t ROW_PENDING = 0xFFFFFFFFu;  // key claimed, row not yet published (never visible across kernels)
constexpr uint32_t ROW_NONE = 0xFFFFFFFEu;     // key present but no storage (shard was full when it was admitted)
constexpr uint32_t BUCKET = 8;                 // cells per bucket
constexpr uint64_t PB_NULL_SIGN = 0xFFFFFFFFFFFFFFFEULL;  // padding of a framed shard exchange (owner-mode contexts only)
constexpr uint32_t PB_NUM_SMS = 132;           // SMs of an H100 SXM: grid-stride kernels launch a small multiple of it

// One cell of the index: 16 B.  Cells are grouped in buckets of BUCKET = 8 (one 128 B line): a sign's home
// bucket is mix64(sign) & bucket_mask; a lookup reads whole buckets with 8 lanes, so the probe length is
// counted in lines (almost always one), not cells.
struct __align__(16) Cell {
  unsigned long long key;
  uint32_t row;
  uint32_t aux;   // reserved (recency lives in TableDev::row_tick)
};

// One cell of a batch's scratch set (pb_dedup.cu): the device-side FeatureBatch::new (persia-common/src/lib.rs:45-82).
// The set is split into one region per slot (the reference builds one hashmap per slot), so a sign carried by two
// slots of one feature group is two entries, as there.  32 B = one sector per access.
struct __align__(32) DCell {
  unsigned long long key;  // the (prefixed) sign; KEY_EMPTY = free
  uint32_t count;          // occurrences of the sign in this slot of this batch
  uint32_t cursor;         // next free entry of the sign's occurrence list (count > 1)
  uint32_t target;         // where the sign lives: table row (single GPU) or owner slot (sharded); ROW_NONE = nowhere
  uint32_t base;           // first entry of the occurrence list in BatchDev::seg_occ (count > 1)
  uint32_t first;          // the occurrence that inserted the sign: its only one when count == 1
  uint32_t item;           // number of the distinct sign in this batch (insertion order)
};

// farmhash 1.1.5 hash64 of an 8-byte LE value (FarmHash HashLen0to16, 8..16 branch).
// Reference call sites: embedding_worker_service/mod.rs:341-345, :364.  Bit-exact.
__host__ __device__ __forceinline__ uint64_t farmhash64_u64(uint64_t x) {
  const uint64_t k2 = 0x9ae16a3b2f90404fULL;
  const uint64_t mul = k2 + 16;
  uint64_t a = x + k2;
  uint64_t b = x;
  uint64_t c = ((b >> 37) | (b << 27)) * mul + a;
  uint64_t d = (((a >> 25) | (a << 39)) + b) * mul;
  uint64_t h = (c ^ d) * mul;
  h ^= (h >> 47);
  uint64_t g = (d ^ h) * mul;
  g ^= (g >> 47);
  return g * mul;
}

// placement hash inside a shard (independent of the shard-selection hash above)
__host__ __device__ __forceinline__ uint64_t mix64(uint64_t k) {
  k ^= k >> 33;
  k *= 0xff51afd7ed558ccdULL;
  k ^= k >> 33;
  k *= 0xc4ceb9fe1a85ec53ULL;
  k ^= k >> 33;
  return k;
}

struct TableDev {
  Cell* cells;         // n_cells + N_SPECIAL entries; the last ones are reserved for the signs that equal a marker
  float* rows;         // capacity * stride floats: emb(dim) ++ optimizer state ++ pad
  uint32_t* counters;  // see CTR_* below
  uint32_t* free_rows;   // stack of rows released by eviction (CTR_FREE entries)
  uint32_t* row_tick;    // per row: batch number of its last training lookup (get_refresh, eviction_map.rs:48-60)
  uint64_t cell_mask;    // n_cells - 1
  uint32_t bucket_mask;  // n_cells / BUCKET - 1
  uint32_t n_cells;
  uint32_t capacity;
  uint32_t dim, stride, state_floats;
};

enum {
  CTR_ROWS = 0,      // bump allocator of row storage
  CTR_FREE = 1,      // rows on the free stack
  CTR_TICK = 2,      // batch number: bumped on the device by every training request (CUDA-graph safe)
  CTR_MISS = 3,      // infer misses / refused admissions
  CTR_GRAD_MISS = 4, // gradient ids not found
  CTR_FULL = 5,      // admissions refused for lack of capacity
  CTR_ADMIT = 6,     // rows admitted
  CTR_EVICT = 7,     // rows evicted
  CTR_ERR = 8,       // an in-kernel wait gave up (mbarrier / peer flag): results of that batch are void
  CTR_COUNT = 16
};

struct OptimDev {
  int kind;
  float lr, wd, mom, init_acc, eps, b1, b2;
};

struct HyperDev {
  float lo, scale;  // init = u01 * scale + lo (scale from rand's UniformFloat::new loop)
  float admit_p;
  int enable_wb;
  float wb;
};

}  // namespace pb
