// pb_device.cuh — device helpers and the launch macro shared by the kernel translation units (internal).
#pragma once
#include "pb_kernels.cuh"

namespace pb {

__device__ __forceinline__ uint32_t slot_of_occ(const SlotsDev& s, uint32_t occ) {
  if (s.uniform) return occ / s.uniform;
  // slot boundaries are ascending; n_slots <= 128 -> <= 7 steps over kernel-parameter memory
  uint32_t lo = 0, hi = s.n_slots;
  while (hi - lo > 1) {
    uint32_t mid = (lo + hi) >> 1;
    if (occ >= s.occ_off[mid]) lo = mid; else hi = mid;
  }
  return lo;
}

// x % (2^w - 1) without a 64-bit division (feature_spacing = 2^(64-prefix_bit) - 1, mod.rs:403-407):
// 2^w == 1 (mod 2^w - 1), so the w-bit digits of x can simply be added.
__device__ __forceinline__ uint64_t mod_mersenne(uint64_t x, uint32_t w) {
  const uint64_t m = (w >= 64) ? ~0ULL : ((1ULL << w) - 1ULL);
  if (w >= 64) return x == m ? 0 : x;  // spacing = u64::MAX when no prefix bits
  uint64_t r = x;
  while (r > m) r = (r & m) + (r >> w);
  return r == m ? 0 : r;
}

template <int VEC>
__device__ __forceinline__ void load_vec(const float* p, float (&v)[VEC]) {
  if (VEC == 4) {
    float4 x = *reinterpret_cast<const float4*>(p);
    v[0] = x.x; v[1] = x.y; v[2] = x.z; v[3] = x.w;
  } else {
    v[0] = p[0];
  }
}
template <int VEC>
__device__ __forceinline__ void store_vec(float* p, const float (&v)[VEC]) {
  if (VEC == 4) *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  else p[0] = v[0];
}

// the lanes of this thread's group of G lanes (G a power of two <= 32) within its warp
__device__ __forceinline__ uint32_t group_mask(uint32_t G) {
  const uint32_t wl = threadIdx.x & 31u;
  return (G == 32) ? 0xffffffffu : (((1u << G) - 1u) << (wl / G * G));
}

// lanes per row and floats per lane for a given embedding dim
static inline void vec_group(uint32_t dim, int& vec, int& G) {
  vec = (dim % 4 == 0) ? 4 : 1;
  uint32_t nvec = dim / vec;
  G = 1;
  while ((uint32_t)G < nvec && G < 32) G <<= 1;
}

static inline uint32_t cdiv(uint64_t a, uint32_t b) { return (uint32_t)((a + b - 1) / b); }

bool profiling();  // a kernel family is being timed: the backward then runs its kernels one after another
void prof_begin(int family, cudaStream_t st);
void prof_end(cudaStream_t st);
void count_launch();

#define PB_LAUNCH_F(family, kernel, grid, block, smem, stream, ...)     \
  do {                                                                  \
    prof_begin((family), (stream));                                     \
    kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__);         \
    prof_end((stream));                                                 \
    count_launch();                                                     \
  } while (0)
#define PB_LAUNCH(kernel, grid, block, smem, stream, ...) PB_LAUNCH_F(FAM_OTHER, kernel, grid, block, smem, stream, __VA_ARGS__)

}  // namespace pb
