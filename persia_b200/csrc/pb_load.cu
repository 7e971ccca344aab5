// pb_load.cu — checkpoint loads on the device: the entries of a `.emb` list image (persia_b200/checkpoint.py, the
// layout in pb_dump.cu's header) selected, gathered out of their unaligned nodes and handed to pb_set_rows.
//
// The image is read in place, in mapped pinned host memory, as the host tier's rows are read.  Two cases:
//   writer layout  (every file this project writes: every node live, one entry length, next = i + 2): a window of whole
//                  nodes at a time; node offsets are arithmetic, list position = node index, and every node's header
//                  is checked on the device (k_load_select) before anything of the window is inserted;
//   any other      (the reference's files: nodes out of list order, free nodes, mixed entry lengths): the whole image,
//                  whose node offsets, links and list order come from one sequential pass on the host
//                  (load_index_host: 13 bytes read per node and a walk over a 4-byte array), with exactly the checks,
//                  and the first failure, of checkpoint.decode_list.
// An incremental-update packet (persia_b200/incremental.py) holds the same entries without a node header (LoadImg.hdr
// = 0), in packet order from byte 4.  When its size says every entry has the first one's length, offsets are arithmetic
// and k_load_select checks each entry's `len` on the device; any other packet takes one host pass over its length
// fields (packet_index_host, with incremental.decode_packet's checks and first failure).
// Selection (farmhash64(sign) % R == rank, the re-sharding load) and the per-dim counts run on the device.
#include <thrust/iterator/counting_iterator.h>

#include <cub/device/device_select.cuh>
#include <cstring>
#include <string>
#include <vector>

#include "pb_device.cuh"

namespace pb {

namespace {

__device__ __forceinline__ uint32_t ld_u32(const uint8_t* p) {
  return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}

__device__ __forceinline__ uint64_t ld_u64(const uint8_t* p) { return (uint64_t)ld_u32(p) | ((uint64_t)ld_u32(p + 4) << 32); }

__device__ __forceinline__ const uint8_t* node_at(const LoadImg& L, uint32_t pos) {
  return L.img + (L.off ? L.off[pos] : (uint64_t)pos * L.nb);
}

// the summary slot of `dim` (inserted on first sight); LOAD_NONE when the table of dims is full
__device__ uint32_t dim_slot(const LoadImg& L, uint64_t dim) {
  for (uint32_t j = 0; j < LOAD_DIMS; ++j) {
    unsigned long long cur = *(volatile unsigned long long*)&L.dims[j];
    if (cur == KEY_EMPTY) cur = atomicCAS(&L.dims[j], KEY_EMPTY, (unsigned long long)dim);
    if (cur == KEY_EMPTY || cur == dim) return j;
  }
  return LOAD_NONE;
}

__device__ bool count_pair(const LoadImg& L, uint32_t slot, uint32_t len) {
  const unsigned long long key = ((unsigned long long)slot << 32) | len;
  for (uint32_t j = 0; j < LOAD_PAIRS; ++j) {
    unsigned long long cur = *(volatile unsigned long long*)&L.pairs[j];
    if (cur == KEY_EMPTY) cur = atomicCAS(&L.pairs[j], KEY_EMPTY, key);
    if (cur == KEY_EMPTY || cur == key) {
      atomicAdd(&L.counts[j], 1u);
      return true;
    }
  }
  return false;
}

// per list position: the checks of arithmetic offsets (every record of the one entry length; a writer-layout window's
// node headers too), the selection, the dim's summary slot
__global__ void __launch_bounds__(256) k_load_select(LoadImg L) {
  for (uint32_t pos = blockIdx.x * blockDim.x + threadIdx.x; pos < L.n; pos += gridDim.x * blockDim.x) {
    const uint8_t* p = node_at(L, pos);
    const uint32_t len = ld_u32(p + L.hdr);
    uint8_t slot = LOAD_NONE;
    if (!L.off) {  // of the one entry length; a window's node also node0 + pos of n_total, live, of the window's dim
      const uint64_t g = L.node0 + pos;
      const uint32_t next = g + 1 < L.n_total ? (uint32_t)(g + 2) : 0u;
      if (len != L.len || (L.hdr && (ld_u32(p) != next || p[8] != 1 || ld_u64(p + L.hdr + 4 + 4ull * L.len) != L.dim))) {
        atomicOr(&L.flags[LOAD_FLAG_BAD], 1u);
        L.slot[pos] = LOAD_NONE;
        continue;
      }
    }
    const uint8_t* q = p + L.hdr + 4 + 4ull * len;
    const uint64_t dim = ld_u64(q), sign = ld_u64(q + 8);
    const bool keep = pos >= L.p_lo && pos < L.p_hi && (L.R <= 1 || farmhash64_u64(sign) % L.R == L.rank);
    if (keep) {
      const uint32_t j = dim_slot(L, dim);
      if (j == LOAD_NONE || !count_pair(L, j, len)) atomicOr(&L.flags[LOAD_FLAG_FULL], 1u);
      else slot = (uint8_t)j;
    }
    L.slot[pos] = slot;
  }
}

// one warp per entry: kept entries [lo, lo + n) of one dim (counted from the end when rev) into aligned staging
__global__ void __launch_bounds__(256) k_load_gather(LoadImg L, const uint32_t* __restrict__ sel, uint32_t K,
                                                     uint32_t lo, uint32_t n, int rev, uint32_t len,
                                                     uint64_t* __restrict__ signs, float* __restrict__ ent) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t warps = gridDim.x * (blockDim.x >> 5);
  for (uint32_t e = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; e < n; e += warps) {
    const uint32_t r = rev ? K - 1 - (lo + e) : lo + e;
    const uint8_t* p = node_at(L, sel[r]);
    // the entry's floats start after its `len`, at any byte alignment: aligned words, shifted into place
    const uint8_t* f = p + L.hdr + 4;
    const uint32_t a = (uint32_t)((uintptr_t)f & 3u);
    const uint32_t* w = reinterpret_cast<const uint32_t*>(f - a);
    float* out = ent + (size_t)e * len;
    for (uint32_t k = lane; k < len; k += 32) {
      const uint32_t v = a ? __funnelshift_r(w[k], w[k + 1], 8 * a) : w[k];  // (w[k + 1] stays inside the record)
      out[k] = __uint_as_float(v);
    }
    if (lane == 0) signs[e] = ld_u64(f + 4ull * len + 8);
  }
}

struct InSlot {
  const uint8_t* slot;
  uint8_t j;
  __device__ __forceinline__ bool operator()(uint32_t i) const { return slot[i] == j; }
};

uint32_t grid_for(uint64_t threads) {
  const uint32_t g = cdiv(threads, 256);
  return g < PB_NUM_SMS * 8 ? (g ? g : 1) : PB_NUM_SMS * 8;
}

}  // namespace

size_t load_list_bytes(uint32_t n) {
  size_t b = 0;
  cub::DeviceSelect::If(nullptr, b, thrust::counting_iterator<uint32_t>(0), (uint32_t*)nullptr, (uint32_t*)nullptr,
                        (int)n, InSlot{nullptr, 0});
  return b;
}

cudaError_t launch_load_select(const LoadImg& L, cudaStream_t st) {
  if (!L.n) return cudaSuccess;
  PB_LAUNCH(k_load_select, grid_for(L.n), 256, 0, st, L);
  return cudaGetLastError();
}

cudaError_t launch_load_list(const LoadImg& L, uint32_t slot, void* tmp, size_t tmp_bytes, uint32_t* sel,
                             uint32_t* d_count, cudaStream_t st) {
  size_t b = tmp_bytes;
  return cub::DeviceSelect::If(tmp, b, thrust::counting_iterator<uint32_t>(0), sel, d_count, (int)L.n,
                               InSlot{L.slot, (uint8_t)slot}, st);
}

cudaError_t launch_load_gather(const LoadImg& L, const uint32_t* sel, uint32_t K, uint32_t lo, uint32_t n, int rev,
                               uint32_t len, uint64_t* signs, float* ent, cudaStream_t st) {
  if (!n) return cudaSuccess;
  PB_LAUNCH(k_load_gather, grid_for(32ull * n), 256, 0, st, L, sel, K, lo, n, rev, len, signs, ent);
  return cudaGetLastError();
}

// checkpoint.decode_list's checks over a whole image, in its order; "Type: message" of the first failure in err
bool load_index_host(const uint8_t* b, uint64_t nbytes, std::vector<uint64_t>& pos_off, std::string& err) {
  auto u32 = [b](uint64_t o) {
    uint32_t v;
    std::memcpy(&v, b + o, 4);
    return v;
  };
  if (nbytes < 28) return err = "ValueError: truncated checkpoint: header", false;
  uint64_t count;
  std::memcpy(&count, b, 8);
  const uint32_t first = u32(8), n_nodes = u32(24);
  // grown node by node: every node takes at least 9 bytes, so they never outgrow the image whatever n_nodes says
  const uint64_t most = (nbytes - 28) / 9;
  std::vector<uint64_t> off;
  std::vector<uint32_t> nxt;
  std::vector<uint8_t> live;
  off.reserve(n_nodes < most ? n_nodes : most);
  nxt.reserve(off.capacity());
  live.reserve(off.capacity());
  uint64_t o = 28, n_live = 0;
  for (uint32_t i = 0; i < n_nodes; ++i) {
    if (nbytes < o + 9) return err = "ValueError: truncated checkpoint: node", false;
    off.push_back(o);
    nxt.push_back(u32(o));
    live.push_back(0);
    const uint8_t flag = b[o + 8];
    o += 9;
    if (flag) {
      // (numpy's own errors where fewer than the 4 bytes of `len` remain: an empty view has no element 0, a short
      // one is not a whole u32)
      if (nbytes == o) return err = "IndexError: index 0 is out of bounds for axis 0 with size 0", false;
      if (nbytes < o + 4) return err = "ValueError: buffer size must be a multiple of element size", false;
      const uint64_t L = u32(o);
      if (nbytes < o + 4 + 4 * L + 16) return err = "ValueError: truncated checkpoint: entry", false;
      o += 20 + 4 * L;
      live.back() = 1;
      ++n_live;
    }
  }
  if (o != nbytes) return err = "ValueError: trailing bytes after the node array", false;
  if (n_live != count)
    return err = "ValueError: checkpoint says " + std::to_string(count) + " entries, " + std::to_string(n_live) +
                 " nodes hold one", false;
  // the walk from `first` along `next` (checkpoint._walk); count <= n_nodes here
  pos_off.resize(count);
  uint64_t cur = first;
  bool unused = false;
  for (uint64_t k = 0; k < count; ++k) {
    if (cur == 0 || cur > n_nodes) return err = "ValueError: broken list: it ends before `count` entries", false;
    pos_off[k] = off[cur - 1];
    unused |= !live[cur - 1];
    cur = nxt[cur - 1];
  }
  if (cur != 0) return err = "ValueError: broken list: it continues past `count` entries", false;
  if (unused) return err = "ValueError: the list runs through an unused node", false;
  return true;
}

// incremental.decode_packet's checks over a whole packet, in its order (its runs of one length fail exactly where their
// first entry that does not fit with the timestamp after it would); the byte offset of each entry in pos_off
bool packet_index_host(const uint8_t* b, uint64_t nbytes, std::vector<uint64_t>& pos_off, std::string& err) {
  if (nbytes < 12) return err = "ValueError: truncated packet", false;
  uint32_t count;
  std::memcpy(&count, b, 4);
  // grown entry by entry: every entry takes at least 20 bytes, so they never outgrow the packet whatever count says
  pos_off.clear();
  pos_off.reserve(count < nbytes / 20 ? count : nbytes / 20);
  uint64_t o = 4;
  for (uint32_t k = 0; k < count; ++k) {
    if (nbytes < o + 4) return err = "ValueError: truncated packet: entry", false;
    uint32_t L;
    std::memcpy(&L, b + o, 4);
    // (numpy's own errors for an entry dtype beyond a C int; one of 2^31 bytes or more has a negative itemsize there,
    // so no run of it fits)
    if (L > INT32_MAX) return err = "ValueError: invalid shape in fixed-type tuple: dimension does not fit into a C int.", false;
    if (4ull * L > INT32_MAX)
      return err = "ValueError: invalid shape in fixed-type tuple: dtype size in bytes must fit into a C int.", false;
    if (20 + 4ull * L > INT32_MAX || nbytes < o + 28 + 4ull * L) return err = "ValueError: truncated packet: entry", false;
    pos_off.push_back(o);
    o += 20 + 4ull * L;
  }
  if (o + 8 != nbytes) return err = "ValueError: packet length does not match its entries", false;
  return true;
}

}  // namespace pb
