// The CPU oracle (oracle/persia_oracle.cpp) with _mm256_rsqrt_ps computed from the committed RSQRTPS table
// (tests/golden/intel_rsqrtps_table.json) instead of by the host's instruction, so that its Adagrad steps are the
// reference's as run on an Intel CPU whatever CPU runs the checker (AMD's RSQRTPS differs in the low bits).  The oracle's
// own modes stay: set_rsqrt_exact(False) then means the table, set_rsqrt_exact(True) exact 1/sqrt.  Built by
// tests/rsqrt_oracle.py, which also loads the table (po_set_rsqrt_table) before any step.
#include <immintrin.h>

#include <cstdint>
#include <cstring>

static uint32_t g_rsqrt_table[2048];

// the model scripts/gen_rsqrt_table.py checked against the instruction on all 2^32 inputs (pb_optim.cuh rsqrt_intel)
static inline uint32_t rsqrt_table_bits(uint32_t u) {
  const uint32_t e = (u >> 23) & 0xffu, m = u & 0x7fffffu, neg = u >> 31;
  if (e == 0xffu) return m ? (u | 0x400000u) : (neg ? 0xffc00000u : 0u);
  if (e == 0u) return neg ? 0xff800000u : 0x7f800000u;
  if (neg) return 0xffc00000u;
  const int k = (int)e - 127, p = k & 1;
  return (uint32_t)((int32_t)g_rsqrt_table[(p << 10) | (m >> 13)] - ((k - p) / 2) * (1 << 23));
}

static inline __m256 rsqrt_table_ps(__m256 v) {
  uint32_t a[8];
  _mm256_storeu_ps(reinterpret_cast<float*>(a), v);
  for (int q = 0; q < 8; ++q) a[q] = rsqrt_table_bits(a[q]);
  return _mm256_loadu_ps(reinterpret_cast<const float*>(a));
}

extern "C" {
void po_set_rsqrt_table(const uint32_t* entries) { std::memcpy(g_rsqrt_table, entries, sizeof(g_rsqrt_table)); }

// out[i] = the table model of x[i] (bit patterns)
void po_rsqrt_table_many(const uint32_t* x, uint64_t n, uint32_t* out) {
  for (uint64_t i = 0; i < n; ++i) out[i] = rsqrt_table_bits(x[i]);
}

// out[i] = this host's RSQRTPS of x[i] (bit patterns)
void po_rsqrt_intrinsic_many(const uint32_t* x, uint64_t n, uint32_t* out) {
  uint64_t i = 0;
  for (; i + 8 <= n; i += 8)
    _mm256_storeu_ps(reinterpret_cast<float*>(out + i), _mm256_rsqrt_ps(_mm256_loadu_ps(reinterpret_cast<const float*>(x + i))));
  for (; i < n; ++i) {
    float f;
    std::memcpy(&f, x + i, 4);
    f = _mm_cvtss_f32(_mm_rsqrt_ss(_mm_set_ss(f)));
    std::memcpy(out + i, &f, 4);
  }
}

// mismatching inputs between the model and this host's RSQRTPS over the bit patterns [lo, hi)
uint64_t po_rsqrt_table_mismatches(uint64_t lo, uint64_t hi) {
  uint64_t bad = 0;
  for (uint64_t x0 = lo; x0 < hi; x0 += 8) {
    uint32_t in[8], out[8];
    for (int q = 0; q < 8; ++q) in[q] = (uint32_t)(x0 + q);
    _mm256_storeu_ps(reinterpret_cast<float*>(out), _mm256_rsqrt_ps(_mm256_loadu_ps(reinterpret_cast<const float*>(in))));
    for (int q = 0; q < 8 && x0 + q < hi; ++q) bad += out[q] != rsqrt_table_bits(in[q]);
  }
  return bad;
}
}

// every use of the instruction in the oracle takes the table from here on
#define _mm256_rsqrt_ps rsqrt_table_ps
#include "../oracle/persia_oracle.cpp"
