// pb_optim.cuh — the optimizer step on resident rows (internal; SURVEY.md §8a row A9).
// persia-simd/src/lib.rs, persia-common/src/optim.rs:227-307.
// The reference runs 8-wide AVX2 FMAs on elements [0, 8*floor(len/8)) and an UNFUSED scalar tail after that; both
// forms are reproduced per element (the library is compiled with --fmad=false) so that SGD is bit-exact.  Adagrad's
// fused lanes take _mm256_rsqrt_ps(s + eps) there, its tail exact 1/sqrt.  A table's rsqrt mode (pb_table_set_rsqrt)
// picks what the fused lanes take here: PB_RSQRT_EXACT (default) exact 1/sqrt, as the tail, so that the step differs
// from the reference by the approximation's error (<= 1.5 * 2^-12 relative); PB_RSQRT_INTEL rsqrt_intel, the
// instruction as Intel CPUs compute it, so that the step is the reference's bit for bit as run on an Intel CPU (AMD's
// approximation differs in the low bits and is not reproduced).  The mode is a template argument of every kernel that
// steps rows, dispatched at launch: the exact instantiations are the code that runs without the mode.
#pragma once
#include "pb_device.cuh"
#include "pb_rsqrt_table.cuh"

namespace pb {

__device__ __forceinline__ float bound(float w, const HyperDev& hy) {
  return hy.enable_wb ? fminf(fmaxf(w, -hy.wb), hy.wb) : w;
}

__device__ __forceinline__ void sgd_elem(float& w, float g, bool fused, const OptimDev& op) {
  if (fused) {
    float dg = __fmaf_rn(op.wd, w, g);
    w = __fmaf_rn(-op.lr, dg, w);
  } else {
    float dg = __fadd_rn(g, __fmul_rn(w, op.wd));
    w = __fsub_rn(w, __fmul_rn(op.lr, dg));
  }
}

// RSQRTPS as Intel CPUs compute it: for x = 2^k * 1.m, p = k & 1, the entry at (p, top 10 bits of m) with its exponent
// lowered by (k - p) / 2; zeros and denormals give a signed infinity, +inf +0, a negative input the default NaN and a
// NaN itself, quieted.  The table (scripts/gen_rsqrt_table.py) was read from the instruction, and this model matches
// it on all 2^32 inputs.  Read through L1: neighbouring lanes take different entries, which constant memory would
// serialize.
__device__ __forceinline__ float rsqrt_intel(float x) {
  const uint32_t u = __float_as_uint(x);
  if (u - 0x00800000u < 0x7f000000u) {  // positive normal
    const int k = (int)(u >> 23) - 127, p = k & 1;
    const uint32_t t = __ldg(&kRsqrtIntel[(p << 10) | ((u >> 13) & 1023u)]);
    return __uint_as_float((uint32_t)((int)t - ((k - p) >> 1) * (1 << 23)));
  }
  const uint32_t e = (u >> 23) & 0xffu, neg = u >> 31;
  if (e == 0xffu) return __uint_as_float((u & 0x7fffffu) ? (u | 0x400000u) : (neg ? 0xffc00000u : 0u));
  if (e == 0u) return __uint_as_float(neg ? 0xff800000u : 0x7f800000u);
  return __uint_as_float(0xffc00000u);  // negative normal or -inf
}

template <bool INTEL>
__device__ __forceinline__ void adagrad_elem(float& w, float& s, float g, bool fused, const OptimDev& op) {
  float sq = __fmul_rn(g, g);
  const float x = __fadd_rn(s, op.eps);
  float r = (INTEL && fused) ? rsqrt_intel(x) : __fdiv_rn(1.0f, __fsqrt_rn(x));
  float scaled = __fmul_rn(g, r);
  if (fused) {
    w = __fmaf_rn(-op.lr, scaled, w);
    s = __fmaf_rn(s, op.mom, sq);
  } else {
    w = __fadd_rn(__fmul_rn(-op.lr, scaled), w);
    s = __fadd_rn(__fmul_rn(s, op.mom), sq);
  }
}

// adam_avx2 (persia-simd/src/lib.rs:147-228); r1/r2 = 1/(1 - accumulated beta powers of the feature group).
__device__ __forceinline__ void adam_elem(float& w, float& m, float& v, float g, bool fused, const OptimDev& op,
                                          float r1, float r2) {
  float omb1 = __fsub_rn(1.0f, op.b1), omb2 = __fsub_rn(1.0f, op.b2);
  float um, uv;
  if (fused) {
    um = __fmaf_rn(op.b1, m, __fmul_rn(omb1, g));
    uv = __fmaf_rn(op.b2, v, __fmul_rn(omb2, __fmul_rn(g, g)));
  } else {
    um = __fadd_rn(__fmul_rn(op.b1, m), __fmul_rn(omb1, g));
    uv = __fadd_rn(__fmul_rn(op.b2, v), __fmul_rn(__fmul_rn(omb2, g), g));
  }
  float mc = __fmul_rn(um, r1), vc = __fmul_rn(uv, r2);
  float descent = __fdiv_rn(mc, __fadd_rn(op.eps, __fsqrt_rn(vc)));
  w = fused ? __fmaf_rn(-op.lr, descent, w) : __fsub_rn(w, __fmul_rn(op.lr, descent));
  m = um;
  v = uv;
}

// what a step needs besides the row and the gradient
struct StepCtx {
  float vw_state;  // Adagrad vectorwise: the OLD scalar state (lib.rs:81-121)
  float r1, r2;    // Adam bias corrections
};

// N consecutive elements of a resident row starting at element e0: load (issued early so that it overlaps the
// gradient fetch), optimizer step + weight bound given the reduced gradient, store.  KIND < 0: decided at run time.
// INTEL: Adagrad's fused lanes take rsqrt_intel (the table's rsqrt mode is PB_RSQRT_INTEL).
template <int KIND, int N, bool INTEL = false>
struct RowElems {
  static constexpr bool kRuntime = KIND < 0;
  static constexpr bool kS1 = kRuntime || KIND == PB_OPT_ADAGRAD || KIND == PB_OPT_ADAM;
  static constexpr bool kS2 = kRuntime || KIND == PB_OPT_ADAM;
  float w[N], s1[kS1 ? N : 1], s2[kS2 ? N : 1];

  __device__ __forceinline__ int kind(const OptimDev& op) const { return kRuntime ? op.kind : KIND; }
  template <int M>
  static __device__ __forceinline__ void ld(const float* p, float (&v)[M]) {
    if (M % 4 == 0) {
#pragma unroll
      for (int q = 0; q < M / 4; ++q) {
        float4 x = *reinterpret_cast<const float4*>(p + 4 * q);
        v[4 * q] = x.x; v[4 * q + 1] = x.y; v[4 * q + 2] = x.z; v[4 * q + 3] = x.w;
      }
    } else if (M % 2 == 0) {
#pragma unroll
      for (int q = 0; q < M / 2; ++q) {
        float2 x = *reinterpret_cast<const float2*>(p + 2 * q);
        v[2 * q] = x.x; v[2 * q + 1] = x.y;
      }
    } else {
#pragma unroll
      for (int q = 0; q < M; ++q) v[q] = p[q];
    }
  }
  template <int M>
  static __device__ __forceinline__ void st(float* p, const float (&v)[M]) {
    if (M % 4 == 0) {
#pragma unroll
      for (int q = 0; q < M / 4; ++q) *reinterpret_cast<float4*>(p + 4 * q) = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
    } else if (M % 2 == 0) {
#pragma unroll
      for (int q = 0; q < M / 2; ++q) *reinterpret_cast<float2*>(p + 2 * q) = make_float2(v[2 * q], v[2 * q + 1]);
    } else {
#pragma unroll
      for (int q = 0; q < M; ++q) p[q] = v[q];
    }
  }
  __device__ __forceinline__ void load(const float* row, uint32_t e0, const TableDev& t, const OptimDev& op) {
    ld<N>(row + e0, w);
    const int k = kind(op);
    if constexpr (kS1) {
      if (k == PB_OPT_ADAGRAD || k == PB_OPT_ADAM) ld<N>(row + t.dim + e0, s1);
    }
    if constexpr (kS2) {
      if (k == PB_OPT_ADAM) ld<N>(row + 2 * t.dim + e0, s2);
    }
  }
  __device__ __forceinline__ void step(uint32_t e0, const float (&g)[N], const TableDev& t, const OptimDev& op,
                                       const HyperDev& hy, const StepCtx& sc) {
    const uint32_t fused_end = (t.dim / 8) * 8;
    const int k = kind(op);
    if (k == PB_OPT_SGD) {
#pragma unroll
      for (int q = 0; q < N; ++q) {
        sgd_elem(w[q], g[q], e0 + q < fused_end, op);
        w[q] = bound(w[q], hy);
      }
    } else if (k == PB_OPT_ADAGRAD) {
#pragma unroll
      for (int q = 0; q < N; ++q) {
        adagrad_elem<INTEL>(w[q], s1[kS1 ? q : 0], g[q], e0 + q < fused_end, op);
        w[q] = bound(w[q], hy);
      }
    } else if (k == PB_OPT_ADAGRAD_VW) {  // emb step with the OLD scalar state (lib.rs:81-121)
      const float x = __fadd_rn(sc.vw_state, op.eps);
      const float r = __fdiv_rn(1.0f, __fsqrt_rn(x));
      const float rf = INTEL ? rsqrt_intel(x) : r;  // the fused lanes' factor
#pragma unroll
      for (int q = 0; q < N; ++q) {
        const bool fused = e0 + q < fused_end;
        float scaled = __fmul_rn(g[q], fused ? rf : r);
        w[q] = fused ? __fmaf_rn(-op.lr, scaled, w[q]) : __fadd_rn(__fmul_rn(-op.lr, scaled), w[q]);
        w[q] = bound(w[q], hy);
      }
    } else {  // Adam
#pragma unroll
      for (int q = 0; q < N; ++q) {
        adam_elem(w[q], s1[kS1 ? q : 0], s2[kS2 ? q : 0], g[q], e0 + q < fused_end, op, sc.r1, sc.r2);
        w[q] = bound(w[q], hy);
      }
    }
  }
  __device__ __forceinline__ void store(float* row, uint32_t e0, const TableDev& t, const OptimDev& op) const {
    st<N>(row + e0, w);
    const int k = kind(op);
    if constexpr (kS1) {
      if (k == PB_OPT_ADAGRAD || k == PB_OPT_ADAM) st<N>(row + t.dim + e0, s1);
    }
    if constexpr (kS2) {
      if (k == PB_OPT_ADAM) st<N>(row + 2 * t.dim + e0, s2);
    }
  }
};

// pair: the (beta1^t, beta2^t) of the row's feature group, read only when the optimizer is Adam
__device__ __forceinline__ StepCtx step_ctx(const OptimDev& op, float vw_state, const float* pair) {
  StepCtx sc;
  sc.vw_state = vw_state;
  sc.r1 = sc.r2 = 0.0f;
  if (op.kind == PB_OPT_ADAM) {
    sc.r1 = __fdiv_rn(1.0f, __fsub_rn(1.0f, pair[0]));
    sc.r2 = __fdiv_rn(1.0f, __fsub_rn(1.0f, pair[1]));
  }
  return sc;
}
__device__ __forceinline__ StepCtx step_ctx(const float* row, const TableDev& t, const OptimDev& op, const GradsDev& gr,
                                            uint32_t slot) {
  return step_ctx(op, op.kind == PB_OPT_ADAGRAD_VW ? row[t.dim] : 0.0f, gr.adam_pow + 2u * gr.pow_idx[slot]);
}

// a sign without a row in the table; lane 0 counts it when `count` (gradient_id_miss_count, PS mod.rs:401-403)
__device__ __forceinline__ bool row_missing(uint32_t row, const TableDev& t, uint32_t lane, bool count) {
  if (row < t.capacity) return false;
  if (lane == 0 && count) atomicAdd(&t.counters[CTR_GRAD_MISS], 1u);
  return true;
}

// one optimizer step on the lane's columns of a resident row, VEC at a time (lane < G lanes per row): the row's
// elements are loaded first, so that they are in flight while grad(e0, g) fills g with the gradient of columns
// [e0, e0 + VEC)
template <int KIND, int VEC, bool INTEL = false, typename GRAD>
__device__ __forceinline__ void step_row(float* prow, const TableDev& t, const OptimDev& op, const HyperDev& hy,
                                         const StepCtx& sc, uint32_t lane, uint32_t G, GRAD grad) {
  const uint32_t nvec = t.dim / VEC;
  for (uint32_t c = lane; c < nvec; c += G) {
    RowElems<KIND, VEC, INTEL> rc;
    float g[VEC];
    rc.load(prow, c * VEC, t, op);
    grad(c * VEC, g);
    rc.step(c * VEC, g, t, op, hy, sc);
    rc.store(prow, c * VEC, t, op);
  }
}

// ndarray 0.15 unrolled_dot order (8 partial sums, pairwise fold, scalar tail), serial per row: one lane calls it on
// the reduced gradient in memory
static __device__ float vw_dot(const float* g, uint32_t n) {
  float p[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  uint32_t i = 0;
  for (; i + 8 <= n; i += 8)
#pragma unroll
    for (int k = 0; k < 8; ++k) p[k] = __fadd_rn(p[k], __fmul_rn(g[i + k], g[i + k]));
  float sum = 0.0f;
  sum = __fadd_rn(sum, __fadd_rn(p[0], p[4]));
  sum = __fadd_rn(sum, __fadd_rn(p[1], p[5]));
  sum = __fadd_rn(sum, __fadd_rn(p[2], p[6]));
  sum = __fadd_rn(sum, __fadd_rn(p[3], p[7]));
  for (; i < n; ++i) sum = __fadd_rn(sum, __fmul_rn(g[i], g[i]));
  return sum;
}

// Adagrad vectorwise, after the group (gmask) stepped the row with the old state sc.vw_state and g, the reduced
// gradient, is in memory: state = state*mom + dot(g,g)/dim (optim.rs:280-283)
__device__ __forceinline__ void vw_state_step(float* prow, const float* g, const TableDev& t, const OptimDev& op,
                                              const StepCtx& sc, uint32_t lane, uint32_t gmask) {
  __syncwarp(gmask);  // every lane of the group has read the old state, and g is visible to lane 0
  if (lane == 0) prow[t.dim] = __fadd_rn(__fmul_rn(sc.vw_state, op.mom), __fdiv_rn(vw_dot(g, t.dim), (float)t.dim));
  __syncwarp(gmask);  // the new state is written before any lane of the group reads it again
}

// one gradient value as the EW prepares it before summing: f16 -> f32 with +-inf clamped to +-65504
// (persia-common lib.rs:163-180), x 1/scale_factor (mod.rs:751-755), x 1/sqrt(n ids of the sample) (mod.rs:757-768)
struct GradPrep {
  float inv_scale, sqrt_f;
  bool do_scale, do_sqrt;
  __device__ __forceinline__ float operator()(float v) const {
    if (do_scale) v = __fmul_rn(v, inv_scale);
    if (do_sqrt) v = __fmul_rn(v, sqrt_f);
    return v;
  }
};
__device__ __forceinline__ float clamp_f16(float v) { return fminf(fmaxf(v, -65504.0f), 65504.0f); }

}  // namespace pb
