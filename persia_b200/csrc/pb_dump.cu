// pb_dump.cu — checkpoint images on the device: the reference's `.emb` list encoding (persia_b200/checkpoint.py) of a
// table's entries, for the background dump (pb_table_dump_part: one part of the table, collected, ordered and encoded
// at one point of the table's call order) and the synchronous dump (pb_dump_nodes: a slice of a list whose order the
// caller gives).
//
// Image of a list of n entries (speedy, little endian):
//   count u64 | first u32 | last u32 | free u32 | end u32 | n_nodes u32              (28 bytes)
//   node i = next u32 | prev u32 | flag u8 | len u32 | f32 x len | dim u64 | sign u64  (29 + 4 len bytes)
// with next = i + 2 (0 for the last node), prev = i, flag = 1.  A node is not 4-byte aligned in the image, so each
// block lays out a run of whole nodes in shared memory byte by byte and stores the run with aligned 16-byte stores
// (byte stores only at the run's two ends, which it shares with the neighbouring runs).
#include <cub/device/device_radix_sort.cuh>

#include "pb_probe.cuh"

namespace pb {

namespace {

constexpr uint64_t SIGN_BIT = 1ULL << 63;  // sign ^ SIGN_BIT orders as u64 the way the sign orders as an int64
constexpr uint32_t HEAD_BYTES = 28;
constexpr uint32_t ENC_SMEM = 24576;       // shared bytes one block's run of nodes aims for
constexpr uint32_t ENC_THREADS = 256;

__device__ __forceinline__ uint32_t part_of(uint64_t sign, uint32_t n_parts) {
  return (uint32_t)(dump_splitmix64(sign) % n_parts);
}

// the live cells of `t` whose sign falls in `part`: key = sign ^ SIGN_BIT, rec = last-use request, loc = row | which << 32
__global__ void __launch_bounds__(256) k_dump_collect(TableDev t, uint64_t which, uint32_t part, uint32_t n_parts,
                                                      DumpWs w) {
  const uint64_t n = (uint64_t)t.n_cells + N_SPECIAL;
  const uint32_t lane = threadIdx.x & 31;
  for (uint64_t base = (uint64_t)blockIdx.x * blockDim.x; base < n; base += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t i = base + threadIdx.x;
    bool take = false;
    uint64_t sign = 0;
    uint32_t row = 0;
    if (i < n) {
      const Cell c = t.cells[i];
      if (cell_live(t, i, c)) {
        sign = cell_sign(t, i, c);
        row = c.row;
        take = part_of(sign, n_parts) == part;
      }
    }
    const uint32_t m = __ballot_sync(0xffffffffu, take);
    if (!m) continue;
    const int leader = __ffs(m) - 1;
    uint32_t k0 = 0;
    if ((int)lane == leader) k0 = atomicAdd(&w.words[DW_COUNT], (uint32_t)__popc(m));
    k0 = __shfl_sync(0xffffffffu, k0, leader);
    if (!take) continue;
    const uint32_t k = k0 + __popc(m & ((1u << lane) - 1u));
    if (k < w.max_items) {
      w.key[k] = sign ^ SIGN_BIT;
      w.rec[k] = t.row_tick[row];
      w.loc[k] = (which << 32) | row;
    }
  }
}

// item numbers for the first sort; the slots past the collected items get maximal keys, so they sort last (the sort
// is stable and they follow every collected item) and the item count never leaves the device
__global__ void __launch_bounds__(256) k_dump_pad(DumpWs w) {
  const uint32_t count = min(w.words[DW_COUNT], w.max_items);
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < w.max_items; i += gridDim.x * blockDim.x) {
    w.idx0[i] = i;
    if (i >= count) {
      w.key[i] = ~0ULL;
      w.rec[i] = ~0u;
    }
  }
}

__global__ void __launch_bounds__(256) k_dump_gather_rec(DumpWs w) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < w.max_items; i += gridDim.x * blockDim.x)
    w.rec2[i] = w.rec[w.idx1[i]];
}

// size of the part's image, the request number, the list header; DW_NODES = nodes to encode (0: the image does not fit)
__global__ void k_dump_finish(TableDev t, DumpWs w, uint8_t* __restrict__ image, uint64_t max_bytes,
                              unsigned long long* __restrict__ d_bytes, uint32_t* __restrict__ d_request) {
  const uint32_t n = w.words[DW_COUNT];
  const uint64_t bytes = HEAD_BYTES + (uint64_t)n * (29u + 4u * (t.dim + t.state_floats));
  *d_bytes = bytes;
  *d_request = t.counters[CTR_TICK];
  const bool fits = bytes <= max_bytes;
  w.words[DW_NODES] = fits ? n : 0u;
  if (!fits) return;
  const uint32_t head[5] = {n ? 1u : 0u, n, 0u, 0u, n};
  const uint64_t cnt = n;
  for (int b = 0; b < 8; ++b) image[b] = (uint8_t)(cnt >> (8 * b));
  for (int f = 0; f < 5; ++f)
    for (int b = 0; b < 4; ++b) image[8 + 4 * f + b] = (uint8_t)(head[f] >> (8 * b));
}

// a table that has never been allocated holds nothing: the empty list's header (all zeros)
__global__ void k_dump_empty(uint8_t* __restrict__ image, uint64_t max_bytes, unsigned long long* __restrict__ d_bytes,
                             uint32_t* __restrict__ d_request) {
  *d_bytes = HEAD_BYTES;
  *d_request = 0;
  if (max_bytes >= HEAD_BYTES)
    for (uint32_t b = 0; b < HEAD_BYTES; ++b) image[b] = 0;
}

// every sign's location: its HBM row, else its tier row (which = 1), else ~0 (not resident)
__global__ void __launch_bounds__(256) k_dump_locate(TableDev t, TableDev h, int has_tier,
                                                     const uint64_t* __restrict__ signs, uint32_t n,
                                                     uint64_t* __restrict__ loc) {
  const uint64_t i = ((uint64_t)blockIdx.x * 256 + threadIdx.x) / BUCKET;
  const uint32_t sub = threadIdx.x % BUCKET;
  const uint32_t gshift = (threadIdx.x & 31) & ~(BUCKET - 1);
  const bool valid = i < n;
  const uint64_t sign = valid ? signs[i] : 0ULL;
  const ProbeOut r = probe_group<MODE_FIND>(t, HyperDev{}, OptimDev{}, sign, valid, 0u, sub, gshift);
  const bool in_hbm = r.row < t.capacity;
  const bool look = valid && !in_hbm && has_tier;
  const ProbeOut q = probe_group<MODE_FIND>(h, HyperDev{}, OptimDev{}, sign, look, 0u, sub, gshift);  // (h = t: no tier)
  if (!valid || sub != 0) return;
  loc[i] = in_hbm ? (uint64_t)r.row : (look && q.row < h.capacity) ? ((1ULL << 32) | q.row) : ~0ULL;
}

// what the encoder writes: nodes [0, n) of a run that is nodes [lo, lo + n) of a list of n_list entries
struct EncSrc {
  const uint32_t* order;   // node -> item (null: node i is item i)
  const uint64_t* sign;    // per item, xor `flip`
  uint64_t flip;
  const uint64_t* loc;     // per item (see k_dump_locate)
  const uint32_t* n_dev;   // nodes to encode, on the device (then n_list = n); null: n_host, list_host
  uint32_t n_host;
  uint64_t list_host, lo;
};

__global__ void __launch_bounds__(ENC_THREADS) k_dump_encode(TableDev t, TableDev h, EncSrc s, uint8_t* __restrict__ out,
                                                             uint64_t off0, uint32_t K) {
  extern __shared__ uint4 sbuf[];
  uint8_t* sb = reinterpret_cast<uint8_t*>(sbuf);
  const uint32_t L = t.dim + t.state_floats;
  const uint64_t NB = 29u + 4ull * L;
  const uint64_t n = s.n_dev ? *s.n_dev : s.n_host;
  const uint64_t n_list = s.n_dev ? n : s.list_host;
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  const uint32_t nv = (L + 3) / 4;
  for (uint64_t i0 = (uint64_t)blockIdx.x * K; i0 < n; i0 += (uint64_t)gridDim.x * K) {
    const uint64_t i1 = min(i0 + K, n);
    const uint64_t start = off0 + i0 * NB, end = off0 + i1 * NB, a0 = start & ~15ULL;
    for (uint64_t i = i0 + warp; i < i1; i += nw) {
      const uint32_t j = s.order ? s.order[i] : (uint32_t)i;
      const uint64_t sign = s.sign[j] ^ s.flip, loc = s.loc[j];
      const float* src = loc == ~0ULL ? nullptr : ((loc >> 32) ? h.rows : t.rows) + (size_t)(uint32_t)loc * t.stride;
      uint8_t* p = sb + (off0 + i * NB - a0);
      const uint64_t g = s.lo + i;
      if (lane < 13) {
        const uint32_t next = g + 1 < n_list ? (uint32_t)(g + 2) : 0u;
        const uint32_t v = lane < 4 ? next : lane < 8 ? (uint32_t)g : lane == 8 ? 1u : L;
        const uint32_t b = lane < 8 ? lane & 3 : lane == 8 ? 0 : lane - 9;
        p[lane] = (uint8_t)(v >> (8 * b));
      } else if (lane < 29) {
        const uint32_t b = lane - 13;
        const uint64_t v = b < 8 ? (uint64_t)t.dim : sign;
        p[13 + 4 * L + b] = (uint8_t)(v >> (8 * (b & 7)));
      }
      for (uint32_t v = lane; v < nv; v += 32) {
        const float4 x = src ? *reinterpret_cast<const float4*>(src + 4 * v) : make_float4(0.f, 0.f, 0.f, 0.f);
        const uint32_t e[4] = {__float_as_uint(x.x), __float_as_uint(x.y), __float_as_uint(x.z), __float_as_uint(x.w)};
#pragma unroll
        for (uint32_t q = 0; q < 4; ++q) {
          if (4 * v + q >= L) break;
          uint8_t* d = p + 13 + 4 * (4 * v + q);
          d[0] = (uint8_t)e[q];
          d[1] = (uint8_t)(e[q] >> 8);
          d[2] = (uint8_t)(e[q] >> 16);
          d[3] = (uint8_t)(e[q] >> 24);
        }
      }
    }
    __syncthreads();
    const uint64_t chunks = (end - a0 + 15) / 16;
    for (uint64_t c = threadIdx.x; c < chunks; c += blockDim.x) {
      const uint64_t ga = a0 + 16 * c;
      if (ga >= start && ga + 16 <= end) {
        *reinterpret_cast<uint4*>(out + ga) = sbuf[c];
      } else {
        for (uint32_t b = 0; b < 16; ++b)
          if (ga + b >= start && ga + b < end) out[ga + b] = sb[16 * c + b];
      }
    }
    __syncthreads();
  }
}

// nodes per block run and its shared bytes (the run's bytes, plus up to 15 in front for alignment, rounded up to 16)
void enc_geometry(uint32_t L, uint32_t& K, uint32_t& smem) {
  const uint32_t nb = 29u + 4u * L;
  K = ENC_SMEM / nb;
  if (K < 1) K = 1;
  if (K > 512) K = 512;
  smem = (K * nb + 31u) & ~15u;
}

cudaError_t launch_encode(const TableDev& t, const TableDev& h, const EncSrc& s, uint8_t* out, uint64_t off0,
                          uint32_t grid, cudaStream_t st) {
  uint32_t K, smem;
  enc_geometry(t.dim + t.state_floats, K, smem);
  if (smem > 48 * 1024) {
    const cudaError_t e = cudaFuncSetAttribute(k_dump_encode, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  PB_LAUNCH(k_dump_encode, grid, ENC_THREADS, smem, st, t, h, s, out, off0, K);
  return cudaGetLastError();
}

}  // namespace

uint64_t dump_node_bytes(uint32_t entry_len) { return 29u + 4ull * entry_len; }

uint64_t dump_sort_bytes(uint32_t max_items) {
  size_t a = 0, b = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, a, (const uint64_t*)nullptr, (uint64_t*)nullptr, (const uint32_t*)nullptr,
                                  (uint32_t*)nullptr, (int)max_items);
  cub::DeviceRadixSort::SortPairs(nullptr, b, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const uint32_t*)nullptr,
                                  (uint32_t*)nullptr, (int)max_items);
  return a > b ? a : b;
}

cudaError_t launch_dump_empty(uint8_t* image, uint64_t max_bytes, unsigned long long* d_bytes, uint32_t* d_request,
                              cudaStream_t st) {
  PB_LAUNCH(k_dump_empty, 1, 1, 0, st, image, max_bytes, d_bytes, d_request);
  return cudaGetLastError();
}

cudaError_t launch_dump_part(const TableDev& t, const TableDev* h, uint32_t part, uint32_t n_parts, const DumpWs& w,
                             uint8_t* image, uint64_t max_bytes, unsigned long long* d_bytes, uint32_t* d_request,
                             cudaStream_t st) {
  cudaError_t e = cudaMemsetAsync(w.words, 0, sizeof(uint32_t) * DW_WORDS, st);
  if (e != cudaSuccess) return e;
  // collect: the index scans of both tables (PB_NUM_SMS * 8 blocks, as the other whole-index scans)
  PB_LAUNCH(k_dump_collect, PB_NUM_SMS * 8, 256, 0, st, t, 0ULL, part, n_parts, w);
  if (h) PB_LAUNCH(k_dump_collect, PB_NUM_SMS * 8, 256, 0, st, *h, 1ULL, part, n_parts, w);
  // order: by sign (as an int64), then stably by last-use request: (request, sign) ascending
  const uint32_t grid = cdiv(w.max_items, 256) < PB_NUM_SMS * 4 ? cdiv(w.max_items, 256) : PB_NUM_SMS * 4;
  PB_LAUNCH(k_dump_pad, grid, 256, 0, st, w);
  size_t tb = w.sort_bytes;
  e = cub::DeviceRadixSort::SortPairs(w.sort_tmp, tb, w.key, w.key_s, w.idx0, w.idx1, (int)w.max_items, 0, 64, st);
  if (e != cudaSuccess) return e;
  PB_LAUNCH(k_dump_gather_rec, grid, 256, 0, st, w);
  tb = w.sort_bytes;
  e = cub::DeviceRadixSort::SortPairs(w.sort_tmp, tb, w.rec2, w.rec_s, w.idx1, w.idx2, (int)w.max_items, 0, 32, st);
  if (e != cudaSuccess) return e;
  PB_LAUNCH(k_dump_finish, 1, 1, 0, st, t, w, image, max_bytes, d_bytes, d_request);
  // encode (the node count stays on the device: a fixed grid strides over the runs)
  EncSrc s{w.idx2, w.key, SIGN_BIT, w.loc, w.words + DW_NODES, 0u, 0ULL, 0ULL};
  return launch_encode(t, h ? *h : t, s, image, HEAD_BYTES, PB_NUM_SMS * 4, st);
}

cudaError_t launch_dump_nodes(const TableDev& t, const TableDev* h, const uint64_t* signs, uint32_t n_list, uint32_t lo,
                              uint32_t n, const DumpWs& w, uint8_t* out, cudaStream_t st) {
  if (!n) return cudaSuccess;
  PB_LAUNCH(k_dump_locate, cdiv((uint64_t)n * BUCKET, 256), 256, 0, st, t, h ? *h : t, h ? 1 : 0, signs + lo, n, w.loc);
  uint32_t K, smem;
  enc_geometry(t.dim + t.state_floats, K, smem);
  const uint32_t runs = cdiv(n, K);
  EncSrc s{nullptr, signs + lo, 0ULL, w.loc, nullptr, n, (uint64_t)n_list, (uint64_t)lo};
  return launch_encode(t, h ? *h : t, s, out, 0, runs < PB_NUM_SMS * 4 ? runs : PB_NUM_SMS * 4, st);
}

}  // namespace pb
