// rsqrt_table_probe.c — reads the 2 x 1024 entries behind the x86 RSQRTPS instruction, and checks that those entries
// reproduce the instruction on every positive normal float (gen_rsqrt_table.py compiles and runs it; gcc -O2 -mavx).
//
// The model: for x = 2^k * 1.m (k = exponent - 127), p = k & 1, the result is the entry at (p, top 10 bits of m),
// read as rsqrtps(2^p * 1.m[top 10]), with its exponent lowered by (k - p) / 2.  Zeros and denormals give a signed
// infinity, +inf gives +0, a negative input gives the default NaN (0xffc00000) and a NaN comes back quieted.
//
// Output (stdout): "cpu <brand string>", then 2048 lines "<index> <entry bits, hex>", then "mismatches <n>" after
// comparing all 2^32 bit patterns.  Exit status 2 when the CPU is not a GenuineIntel part with AVX.
#include <cpuid.h>
#include <immintrin.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

static float as_f(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
static uint32_t as_u(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }

static uint32_t model(uint32_t x, const uint32_t* T) {
  const uint32_t e = (x >> 23) & 0xffu, m = x & 0x7fffffu, neg = x >> 31;
  if (e == 0xffu) return m ? (x | 0x400000u) : (neg ? 0xffc00000u : 0u);
  if (e == 0u) return neg ? 0xff800000u : 0x7f800000u;
  if (neg) return 0xffc00000u;
  const int k = (int)e - 127, p = k & 1;
  return (uint32_t)((int32_t)T[(p << 10) | (m >> 13)] - ((k - p) / 2) * (1 << 23));
}

int main(void) {
  unsigned a, b, c, d;
  char vendor[13] = {0};
  __get_cpuid(0, &a, &b, &c, &d);
  memcpy(vendor, &b, 4); memcpy(vendor + 4, &d, 4); memcpy(vendor + 8, &c, 4);
  __get_cpuid(1, &a, &b, &c, &d);
  if (strcmp(vendor, "GenuineIntel") != 0 || !(c & bit_AVX)) {
    fprintf(stderr, "need a GenuineIntel CPU with AVX (found %s, avx=%d)\n", vendor, !!(c & bit_AVX));
    return 2;
  }
  char brand[49] = {0};
  for (unsigned i = 0; i < 3; ++i) __get_cpuid(0x80000002u + i, (unsigned*)(brand + 16 * i), (unsigned*)(brand + 16 * i + 4),
                                              (unsigned*)(brand + 16 * i + 8), (unsigned*)(brand + 16 * i + 12));
  printf("cpu %s\n", brand);
  uint32_t T[2048];
  for (uint32_t i = 0; i < 2048; ++i) {
    const uint32_t p = i >> 10, x = ((127u + p) << 23) | ((i & 1023u) << 13);
    T[i] = as_u(_mm_cvtss_f32(_mm_rsqrt_ss(_mm_set_ss(as_f(x)))));
    printf("%u %08x\n", i, T[i]);
  }
  unsigned long long bad = 0;
  for (uint64_t x0 = 0; x0 < (1ull << 32); x0 += 8) {
    uint32_t in[8], out[8];
    for (int q = 0; q < 8; ++q) in[q] = (uint32_t)x0 + q;
    _mm256_storeu_ps((float*)out, _mm256_rsqrt_ps(_mm256_loadu_ps((const float*)in)));
    for (int q = 0; q < 8; ++q) bad += out[q] != model(in[q], T);
  }
  printf("mismatches %llu\n", bad);
  return 0;
}
