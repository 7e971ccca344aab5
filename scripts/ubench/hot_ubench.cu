// micro-benchmarks behind k_reduce_hot's design: what one warp sustains for each pipeline role, alone and beside
// warps parked on an mbarrier.  nvcc -O3 -gencode arch=compute_90a,code=sm_90a hot_ubench.cu -o hot_ubench
#include <cuda_fp16.h>
#include <cstdio>
#include <cstdlib>
#include <cstdint>
#include <vector>

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try(uint32_t bar, uint32_t parity) {
  uint32_t done;
  asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
               : "=r"(done) : "r"(bar), "r"(parity) : "memory");
  return done;
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  while (!mbar_try(bar, parity)) {}
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
               "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ __half2 clamp_h2(__half2 v) {
  const __half2 lim = __floats2half2_rn(65504.0f, 65504.0f);
  return __hmin2(__hmax2(v, __hneg2(lim)), lim);
}

// raw: 4 KB of f16 (32 rows x 64) -> dst: 8 KB f32
__device__ __forceinline__ void convert(float* dst, const unsigned char* raw, uint32_t lane) {
  uint4 x[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) x[j] = *reinterpret_cast<const uint4*>(raw + (size_t)(j * 32 + lane) * 16u);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const __half2* h = reinterpret_cast<const __half2*>(&x[j]);
    float y[8];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float2 z = __half22float2(clamp_h2(h[q]));
      y[2 * q] = z.x; y[2 * q + 1] = z.y;
    }
    float4* o = reinterpret_cast<float4*>(dst + (size_t)(j * 32 + lane) * 8u);
    o[0] = make_float4(y[0], y[1], y[2], y[3]);
    o[1] = make_float4(y[4], y[5], y[6], y[7]);
  }
}

// 32 rows of 64 floats: lanes 0..15 own 4 columns each
__device__ __forceinline__ void chain32(float (&acc)[4], const float* rp) {
  float4 va[4], vb[4], vc[4];
#define LD(V, GI) _Pragma("unroll") for (int u = 0; u < 4; ++u) V[u] = *reinterpret_cast<const float4*>(rp + ((GI) * 4 + u) * 64);
#define AD(V) _Pragma("unroll") for (int u = 0; u < 4; ++u) { acc[0] = __fadd_rn(acc[0], V[u].x); acc[1] = __fadd_rn(acc[1], V[u].y); acc[2] = __fadd_rn(acc[2], V[u].z); acc[3] = __fadd_rn(acc[3], V[u].w); }
  LD(va, 0) LD(vb, 1)
  LD(vc, 2) AD(va) LD(va, 3) AD(vb) LD(vb, 4) AD(vc) LD(vc, 5) AD(va) LD(va, 6) AD(vb) LD(vb, 7) AD(vc) AD(va) AD(vb)
#undef LD
#undef AD
}

// mode 0: converter alone.  1: converter + 6 warps parked on a barrier.  2: chain alone.  3: chain + parked warps.
// 4: pipeline without loads: 6 converters + chain with full/empty barriers.  5: loader alone, `runs` copies per round.
// 6: full pipeline: loader + converters + chain.
__global__ void __launch_bounds__(256, 2) k_bench(int mode, int n_chunks, int runs, const __half* g, float* out, long long* cyc) {
  extern __shared__ __align__(128) unsigned char smem[];
  __shared__ __align__(8) uint64_t bars[64];
  float* ring = reinterpret_cast<float*>(smem);                 // 4 x 8 KB
  unsigned char* raw = smem + 4 * 8192;                         // 10 x 4 KB
  const uint32_t tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const uint32_t full0 = smem_u32(bars), empty0 = smem_u32(bars + 8), rfull0 = smem_u32(bars + 16), rempty0 = smem_u32(bars + 32);
  const uint32_t park = smem_u32(bars + 48);
  if (tid == 0) {
    for (int s = 0; s < 8; ++s) { mbar_init(full0 + 8 * s, 32); mbar_init(empty0 + 8 * s, 32); }
    for (int s = 0; s < 16; ++s) { mbar_init(rfull0 + 8 * s, 1); mbar_init(rempty0 + 8 * s, 32); }
    mbar_init(park, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (uint32_t i = tid; i < (4 * 8192 + 10 * 4096) / 4; i += 256) reinterpret_cast<uint32_t*>(smem)[i] = 0x3c003c00u;  // halves 1.0 / some float
  __syncthreads();
  const long long t0 = clock64();
  float acc[4] = {0, 0, 0, 0};
  if (mode == 0 || mode == 1) {
    if (warp == 1) {
      for (int c = 0; c < n_chunks; ++c) convert(ring + (c & 3) * 2048, raw + (c % 10) * 4096, lane);
      __syncwarp();
      if (lane == 0) { cyc[blockIdx.x] = clock64() - t0; mbar_arrive(park); }
    } else if (mode == 1 && warp >= 2) {
      mbar_wait(park, 0);
    }
  } else if (mode == 2 || mode == 3) {
    if (warp == 0) {
      for (int c = 0; c < n_chunks; ++c) if (lane < 16) chain32(acc, ring + (c & 3) * 2048 + lane * 4);
      __syncwarp();
      if (lane == 0) { cyc[blockIdx.x] = clock64() - t0; mbar_arrive(park); }
    } else if (mode == 3 && warp >= 2) {
      mbar_wait(park, 0);
    }
  } else if (mode == 4) {
    if (warp == 0) {
      for (int c = 0; c < n_chunks; ++c) {
        const uint32_t st = c & 3, par = (c >> 2) & 1;
        mbar_wait(full0 + 8 * st, par);
        if (lane < 16) chain32(acc, ring + st * 2048 + lane * 4);
        mbar_arrive(empty0 + 8 * st);
      }
      if (lane == 0) cyc[blockIdx.x] = clock64() - t0;
    } else if (warp >= 2) {
      for (int c = 0; c < n_chunks; ++c) {
        if (c % 6 != (int)warp - 2) continue;
        const uint32_t st = c & 3, par = (c >> 2) & 1;
        mbar_wait(empty0 + 8 * st, par ^ 1);
        convert(ring + st * 2048, raw + (c % 10) * 4096, lane);
        mbar_arrive(full0 + 8 * st);
      }
    }
  } else if (mode == 5 || mode == 6) {
    const unsigned char* gb = reinterpret_cast<const unsigned char*>(g) + (size_t)blockIdx.x * 4096 * 128;
    if (warp == 1) {  // loader: 32 rows of 128 B per round, `runs` copies of 32/runs rows each
      const uint32_t rows_per = 32 / runs;
      for (int c = 0; c < n_chunks; ++c) {
        const uint32_t rs = c % 10, rpar = (c / 10) & 1;
        mbar_wait(rempty0 + 8 * rs, rpar ^ 1);
        if (lane == 0) mbar_expect_tx(rfull0 + 8 * rs, 4096);
        __syncwarp();
        if (lane < (uint32_t)runs) {
          // scattered sources: run r of round c starts at row ((c * 37 + r * 101) % 4000)
          const uint32_t srow = (uint32_t)(c * 37 + lane * 101) % 4000u;
          bulk_g2s(smem_u32(raw + rs * 4096 + lane * rows_per * 128), gb + (size_t)srow * 128, rows_per * 128, rfull0 + 8 * rs);
        }
      }
      if (mode == 5) {  // drain: consume everything so that the waits above make progress
      }
      if (lane == 0 && mode == 5) cyc[blockIdx.x] = clock64() - t0;
    }
    if (mode == 5 && warp == 2) {  // a trivial consumer frees the raw slots
      for (int c = 0; c < n_chunks; ++c) {
        const uint32_t rs = c % 10, rpar = (c / 10) & 1;
        mbar_wait(rfull0 + 8 * rs, rpar);
        mbar_arrive(rempty0 + 8 * rs);
      }
    }
    if (mode == 6) {
      if (warp == 0) {
        for (int c = 0; c < n_chunks; ++c) {
          const uint32_t st = c & 3, par = (c >> 2) & 1;
          mbar_wait(full0 + 8 * st, par);
          if (lane < 16) chain32(acc, ring + st * 2048 + lane * 4);
          mbar_arrive(empty0 + 8 * st);
        }
        if (lane == 0) cyc[blockIdx.x] = clock64() - t0;
      } else if (warp >= 2) {
        for (int c = 0; c < n_chunks; ++c) {
          if (c % 6 != (int)warp - 2) continue;
          const uint32_t st = c & 3, par = (c >> 2) & 1, rs = c % 10, rpar = (c / 10) & 1;
          mbar_wait(rfull0 + 8 * rs, rpar);
          mbar_wait(empty0 + 8 * st, par ^ 1);
          convert(ring + st * 2048, raw + rs * 4096, lane);
          mbar_arrive(full0 + 8 * st);
          mbar_arrive(rempty0 + 8 * rs);
        }
      }
    }
  }
  if (lane < 16 && warp == 0) out[blockIdx.x * 64 + lane * 4] = acc[0] + acc[1] + acc[2] + acc[3];
}


// ---- lean direct producer: chunk of 32 rows x 64 halves; lane's vector j is row j*4 + lane/8, vector lane%8
__device__ __forceinline__ void produce_lean(float* dst, const unsigned char* gbase, const uint16_t* sorted, uint32_t k0, uint32_t lane) {
  uint4 x[8];
  const uint32_t c16 = (lane & 7u) * 16u, r0 = lane >> 3;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const uint32_t row = sorted[k0 + j * 4 + r0];
    x[j] = __ldg(reinterpret_cast<const uint4*>(gbase + (size_t)row * 128u + c16));
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const __half2* h = reinterpret_cast<const __half2*>(&x[j]);
    float y[8];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float2 z = __half22float2(clamp_h2(h[q]));
      y[2 * q] = z.x; y[2 * q + 1] = z.y;
    }
    float4* o = reinterpret_cast<float4*>(dst + (size_t)(j * 4 + r0) * 64u + (lane & 7u) * 8u);
    o[0] = make_float4(y[0], y[1], y[2], y[3]);
    o[1] = make_float4(y[4], y[5], y[6], y[7]);
  }
}
// 32 rows of 64 floats: 32 lanes own 2 columns each
__device__ __forceinline__ void chain32_e2(float (&acc)[2], const float* rp) {
  float2 va[4], vb[4], vc[4];
#define LD(V, GI) _Pragma("unroll") for (int u = 0; u < 4; ++u) V[u] = *reinterpret_cast<const float2*>(rp + ((GI) * 4 + u) * 64);
#define AD(V) _Pragma("unroll") for (int u = 0; u < 4; ++u) { acc[0] = __fadd_rn(acc[0], V[u].x); acc[1] = __fadd_rn(acc[1], V[u].y); }
  LD(va, 0) LD(vb, 1)
  LD(vc, 2) AD(va) LD(va, 3) AD(vb) LD(vb, 4) AD(vc) LD(vc, 5) AD(va) LD(va, 6) AD(vb) LD(vb, 7) AD(vc) AD(va) AD(vb)
#undef LD
#undef AD
}
// all 32 rows loaded first (64 registers), then the adds
__device__ __forceinline__ void chain32_e2_all(float (&acc)[2], const float* rp) {
  float2 v[32];
#pragma unroll
  for (int u = 0; u < 32; ++u) v[u] = *reinterpret_cast<const float2*>(rp + u * 64);
#pragma unroll
  for (int u = 0; u < 32; ++u) { acc[0] = __fadd_rn(acc[0], v[u].x); acc[1] = __fadd_rn(acc[1], v[u].y); }
}

template <int NT>
__global__ void __launch_bounds__(NT, 1) k_bench2(int mode, int n_chunks, const __half* g, float* out, long long* cyc) {
  extern __shared__ __align__(128) unsigned char smem[];
  __shared__ __align__(8) uint64_t bars[64];
  __shared__ uint16_t sorted[4096];
  float* ring = reinterpret_cast<float*>(smem);  // 8 x 8 KB
  const uint32_t tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const uint32_t full0 = smem_u32(bars), empty0 = smem_u32(bars + 8);
  constexpr uint32_t PW = NT / 32 - 1;
  if (tid == 0) {
    for (int s = 0; s < 8; ++s) { mbar_init(full0 + 8 * s, 32); mbar_init(empty0 + 8 * s, 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (uint32_t i = tid; i < 8 * 8192 / 4; i += NT) reinterpret_cast<uint32_t*>(smem)[i] = 0x3f800000u;
  for (uint32_t i = tid; i < 4096; i += NT) sorted[i] = (uint16_t)((i * 2 + (i * 7) % 2) % 4096);  // ascending-ish scattered rows
  __syncthreads();
  const unsigned char* gb = reinterpret_cast<const unsigned char*>(g) + (size_t)blockIdx.x * 4096 * 128;
  const long long t0 = clock64();
  float acc[2] = {0, 0};
  if (mode == 7 || mode == 11) {
    if (warp == 0) {
      for (int c = 0; c < n_chunks; ++c) { if (mode == 7) chain32_e2(acc, ring + (c & 7) * 2048 + lane * 2); else chain32_e2_all(acc, ring + (c & 7) * 2048 + lane * 2); }
      __syncwarp();
      if (lane == 0) cyc[blockIdx.x] = clock64() - t0;
    }
  } else if (mode == 8) {
    if (warp == 1) {
      for (int c = 0; c < n_chunks; ++c) produce_lean(ring + (c & 7) * 2048, gb, sorted, (c * 32) % 4096, lane);
      __syncwarp();
      if (lane == 0) cyc[blockIdx.x] = clock64() - t0;
    }
  } else if (mode == 9) {
    if (warp == 0) {
      for (int c = 0; c < n_chunks; ++c) {
        const uint32_t st = c & 7, par = (c >> 3) & 1;
        mbar_wait(full0 + 8 * st, par);
        chain32_e2(acc, ring + st * 2048 + lane * 2);
        mbar_arrive(empty0 + 8 * st);
      }
      if (lane == 0) cyc[blockIdx.x] = clock64() - t0;
    } else {
      for (int c = 0; c < n_chunks; ++c) {
        if (c % PW != warp - 1) continue;
        const uint32_t st = c & 7, par = (c >> 3) & 1;
        mbar_wait(empty0 + 8 * st, par ^ 1);
        produce_lean(ring + st * 2048, gb, sorted, (c * 32) % 4096, lane);
        mbar_arrive(full0 + 8 * st);
      }
    }
  }
  if (warp == 0) out[blockIdx.x * 64 + lane * 2] = acc[0] + acc[1];
}

// the product kernel's chain loop shape: runtime stride, runtime group count, three groups in flight
__device__ __forceinline__ void chain_rt(float (&acc)[2], const float* rp, uint32_t stride, uint32_t nv) {
  const uint32_t G = (nv + 3u) >> 2;
  float2 va[4], vb[4], vc[4];
#define LD(V, GI) _Pragma("unroll") for (int u = 0; u < 4; ++u) V[u] = *reinterpret_cast<const float2*>(rp + (size_t)((GI) * 4u + u) * stride);
#define AD(V) _Pragma("unroll") for (int u = 0; u < 4; ++u) { acc[0] = __fadd_rn(acc[0], V[u].x); acc[1] = __fadd_rn(acc[1], V[u].y); }
  LD(va, 0)
  if (G > 1) { LD(vb, 1) }
  for (uint32_t gi = 0;;) {
    if (gi + 2 < G) { LD(vc, gi + 2) }
    AD(va)
    if (++gi >= G) break;
    if (gi + 2 < G) { LD(va, gi + 2) }
    AD(vb)
    if (++gi >= G) break;
    if (gi + 2 < G) { LD(vb, gi + 2) }
    AD(vc)
    if (++gi >= G) break;
  }
#undef LD
#undef AD
}
__global__ void __launch_bounds__(256, 2) k_bench3(int mode, int n_chunks, uint32_t stride, uint32_t nv, const __half* g, float* out, long long* cyc) {
  extern __shared__ __align__(128) unsigned char smem[];
  __shared__ __align__(8) uint64_t bars[64];
  __shared__ uint16_t sorted[4096];
  float* ring = reinterpret_cast<float*>(smem);  // 8 x 8 KB
  const uint32_t tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const uint32_t full0 = smem_u32(bars), empty0 = smem_u32(bars + 8);
  if (tid == 0) {
    for (int s = 0; s < 8; ++s) { mbar_init(full0 + 8 * s, 32); mbar_init(empty0 + 8 * s, 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (uint32_t i = tid; i < 8 * 8192 / 4; i += 256) reinterpret_cast<uint32_t*>(smem)[i] = 0x3f800000u;
  for (uint32_t i = tid; i < 4096; i += 256) sorted[i] = (uint16_t)((i * 2 + (i * 7) % 2) % 4096);
  __syncthreads();
  const unsigned char* gb = reinterpret_cast<const unsigned char*>(g) + (size_t)(blockIdx.x % 296) * 4096 * 128;
  const long long t0 = clock64();
  float acc[2] = {0, 0};
  if (mode == 12) {
    if (warp == 0) {
      for (int c = 0; c < n_chunks; ++c) chain_rt(acc, ring + (c & 7) * 2048 + lane * 2, stride, nv);
      __syncwarp();
      if (lane == 0) cyc[blockIdx.x] = clock64() - t0;
    }
  } else {  // 13: pipeline with the product's chain; 7 lean producers
    if (warp == 0) {
      for (int c = 0; c < n_chunks; ++c) {
        const uint32_t st = c & 7, par = (c >> 3) & 1;
        mbar_wait(full0 + 8 * st, par);
        chain_rt(acc, ring + st * 2048 + lane * 2, stride, nv);
        mbar_arrive(empty0 + 8 * st);
      }
      if (lane == 0) cyc[blockIdx.x] = clock64() - t0;
    } else {
      for (int c = 0; c < n_chunks; ++c) {
        if (c % 7 != (int)warp - 1) continue;
        const uint32_t st = c & 7, par = (c >> 3) & 1;
        mbar_wait(empty0 + 8 * st, par ^ 1);
        produce_lean(ring + st * 2048, gb, sorted, (c * 32) % 4096, lane);
        mbar_arrive(full0 + 8 * st);
      }
    }
  }
  if (warp == 0) out[(blockIdx.x % 296) * 64 + lane * 2] = acc[0] + acc[1];
}

int main(int argc, char** argv) {
  setvbuf(stdout, NULL, _IONBF, 0);
  const int only = argc > 1 ? atoi(argv[1]) : -1;
  const int grid = 296, n_chunks = 64;
  __half* g;
  float* out;
  long long* cyc;
  cudaMalloc(&g, (size_t)grid * 4096 * 128);
  cudaMemset(g, 0, (size_t)grid * 4096 * 128);
  cudaMalloc(&out, grid * 64 * 4);
  cudaMalloc(&cyc, grid * 8);
  const size_t smem = 4 * 8192 + 10 * 4096;
  cudaFuncSetAttribute(k_bench, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  const char* names[] = {"converter alone", "converter + 6 parked warps", "chain alone", "chain + 6 parked warps",
                         "pipeline, no loads (6 converters + chain)", "loader alone", "loader + converters + chain"};
  for (int g_blocks : {1, 296}) {
    for (int mode = 0; mode <= 6; ++mode) {
      if (only >= 0 && mode != only) continue;
      for (int runs : {32, 8, 1}) {
        if (mode < 5 && runs != 32) continue;
        std::vector<long long> h(grid);
        for (int rep = 0; rep < 3; ++rep) {
          cudaMemset(cyc, 0, grid * 8);
          k_bench<<<g_blocks, 256, smem>>>(mode, n_chunks, runs, g, out, cyc);
          cudaError_t e = cudaDeviceSynchronize();
          if (e != cudaSuccess) { printf("error %s\n", cudaGetErrorString(e)); return 1; }
        }
        cudaMemcpy(h.data(), cyc, grid * 8, cudaMemcpyDeviceToHost);
        long long mx = 0, sum = 0;
        for (int b = 0; b < g_blocks; ++b) { mx = h[b] > mx ? h[b] : mx; sum += h[b]; }
        printf("blocks %3d  %-44s runs/round %2d : %7.1f cycles/chunk avg, %7.1f max  (%.1f /row)\n", g_blocks, names[mode], runs,
               (double)sum / g_blocks / n_chunks, (double)mx / n_chunks, (double)sum / g_blocks / n_chunks / 32);
      }
    }
  }
  const char* names2[] = {"chain 32 lanes x 2 cols", "lean direct producer alone", "direct pipeline (producers + chain x2cols)", "", "chain x2cols, 32 rows loaded at once"};
  const size_t smem2 = 8 * 8192;
  cudaFuncSetAttribute(k_bench2<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem2);
  cudaFuncSetAttribute(k_bench2<512>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem2);
  cudaFuncSetAttribute(k_bench2<1024>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem2);
  for (int g_blocks : {1, 132}) {
    for (int mode : {7, 11, 8, 9}) {
      if (only >= 0 && mode != only) continue;
      for (int nt : {256, 512, 1024}) {
        if (mode != 9 && nt != 256) continue;
        std::vector<long long> h(grid);
        for (int rep = 0; rep < 3; ++rep) {
          cudaMemset(cyc, 0, grid * 8);
          if (nt == 256) k_bench2<256><<<g_blocks, 256, smem2>>>(mode, 128, g, out, cyc);
          else if (nt == 512) k_bench2<512><<<g_blocks, 512, smem2>>>(mode, 128, g, out, cyc);
          else k_bench2<1024><<<g_blocks, 1024, smem2>>>(mode, 128, g, out, cyc);
          cudaError_t e = cudaDeviceSynchronize();
          if (e != cudaSuccess) { printf("error %s\n", cudaGetErrorString(e)); return 1; }
        }
        cudaMemcpy(h.data(), cyc, grid * 8, cudaMemcpyDeviceToHost);
        long long mx = 0, sum = 0;
        for (int b = 0; b < g_blocks; ++b) { mx = h[b] > mx ? h[b] : mx; sum += h[b]; }
        printf("blocks %3d  %-44s threads %4d : %7.1f cycles/chunk avg, %7.1f max  (%.1f /row)\n", g_blocks, names2[mode - 7], nt,
               (double)sum / g_blocks / 128, (double)mx / 128, (double)sum / g_blocks / 128 / 32);
      }
    }
  }
  cudaFuncSetAttribute(k_bench3, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem2);
  for (int g_blocks : {1, 132, 264}) {
    for (int mode : {12, 13}) {
      if (only >= 0 && mode != only) continue;
      std::vector<long long> h(grid);
      for (int rep = 0; rep < 3; ++rep) {
        cudaMemset(cyc, 0, grid * 8);
        k_bench3<<<g_blocks, 256, smem2>>>(mode, 128, 64, 32, g, out, cyc);
        cudaError_t e = cudaDeviceSynchronize();
        if (e != cudaSuccess) { printf("error %s\n", cudaGetErrorString(e)); return 1; }
      }
      cudaMemcpy(h.data(), cyc, grid * 8, cudaMemcpyDeviceToHost);
      long long mx = 0, sum = 0;
      for (int b = 0; b < g_blocks; ++b) { mx = h[b] > mx ? h[b] : mx; sum += h[b]; }
      printf("blocks %3d  %-44s : %7.1f cycles/chunk avg, %7.1f max  (%.1f /row)\n", g_blocks,
             mode == 12 ? "product chain loop alone" : "pipeline: 7 lean producers + product chain", (double)sum / g_blocks / 128,
             (double)mx / 128, (double)sum / g_blocks / 128 / 32);
    }
  }
  return 0;
}
