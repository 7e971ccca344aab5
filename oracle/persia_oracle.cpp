// persia_oracle.cpp — CPU restatement of PERSIA's sparse-embedding hot path.
//
// TEST INFRASTRUCTURE ONLY.  Nothing in the product path (persia_b200/) may
// import, link or call this file; only tests/, __graft_entry__.smoke() and the
// cpu_baseline / --impl reference legs of bench.py use it, as the checker and
// as the timed CPU baseline.
//
// The reference (PersiaML/PERSIA @ ff754b8) is Rust, which this project does
// not build, so this is a C++17 restatement, function by
// function, of the files cited below (paths relative to the reference root).
// It is pinned against every golden vector the reference's own unit tests hold
// for this path (tests/test_oracle_golden.py):
//   * farmhash64 chain + modulo  — embedding_worker_service/mod.rs:1570-1613
//   * prefix arithmetic          — embedding_worker_service/mod.rs:1615-1660
//   * Adagrad (elementwise)      — persia-common/src/optim.rs:362-408
//   * Adagrad (vectorwise)       — persia-common/src/optim.rs:410-445
//   * LRU / capacity semantics   — persia-embedding-holder/src/eviction_map.rs:113-148
// PARITY UNPINNED for: the initial value of a newly admitted row (the reference
// draws it from rand 0.8.4 SmallRng + rand_distr Uniform, third-party code that
// is absent from the tree and asserted by no reference test; po_init_row below
// restates the published algorithm from memory), the ahash-selected internal
// lock shard, and hashbrown's iteration order (replaced by first-occurrence
// order, see FeatureBatch below).
//
// Build: g++ -O2 -std=c++17 -mavx2 -mfma -mf16c -ffp-contract=off -fPIC -shared
//        (-ffp-contract=off matters: Rust never contracts a*b+c into an FMA.)

#include <immintrin.h>
#include <malloc.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

namespace {

// ---------------------------------------------------------------------------
// farmhash 1.1.5 hash64 on an 8-byte little-endian input.
// Third-party (rust/Cargo.lock "farmhash 1.1.5"); published FarmHash
// HashLen0to16, 8..16-byte branch.  Call sites:
//   embedding_worker_service/mod.rs:341-345 (sign_to_shard_modulo), :364 (hash stack)
// ---------------------------------------------------------------------------
inline uint64_t rotr64(uint64_t v, int s) { return (v >> s) | (v << (64 - s)); }

inline uint64_t farmhash64_u64(uint64_t x) {
  const uint64_t k2 = 0x9ae16a3b2f90404fULL;
  const uint64_t mul = k2 + 16;  // k2 + len*2, len = 8
  uint64_t a = x + k2;
  uint64_t b = x;
  uint64_t c = rotr64(b, 37) * mul + a;
  uint64_t d = (rotr64(a, 25) + b) * mul;
  uint64_t h = (c ^ d) * mul;
  h ^= (h >> 47);
  uint64_t g = (d ^ h) * mul;
  g ^= (g >> 47);
  return g * mul;
}

// ---------------------------------------------------------------------------
// f32 <-> f16.  half 1.8.2 from_f32_slice / to_f32_vec are IEEE-754
// round-to-nearest-even conversions (persia-common/src/lib.rs:157-180).
// ---------------------------------------------------------------------------
inline uint16_t f32_to_f16(float f) {
  return (uint16_t)_cvtss_sh(f, _MM_FROUND_TO_NEAREST_INT | _MM_FROUND_NO_EXC);
}
inline float f16_to_f32(uint16_t h) { return _cvtsh_ss(h); }

// ---------------------------------------------------------------------------
// persia-simd/src/lib.rs — the reference's only "kernels".
// 8-wide AVX2 body + scalar tail, exactly as there (the tail is NOT fused).
// rsqrt mode: 0 = _mm256_rsqrt_ps (what the reference runs; reproduces its
// golden vectors on an Intel host), 1 = exact 1/sqrt in every lane (the GPU
// comparison target; the reference's own tail lanes already use this form).
// ---------------------------------------------------------------------------
int g_rsqrt_exact = 0;

inline __m256 rsqrt8(__m256 v) {
  if (!g_rsqrt_exact) return _mm256_rsqrt_ps(v);
  return _mm256_div_ps(_mm256_set1_ps(1.0f), _mm256_sqrt_ps(v));
}

// persia-simd/src/lib.rs:4-18
void add_assign(float* a, const float* b, size_t n) {
  size_t end = (n / 8) * 8;
  for (size_t i = 0; i < end; i += 8)
    _mm256_storeu_ps(a + i, _mm256_add_ps(_mm256_loadu_ps(a + i), _mm256_loadu_ps(b + i)));
  for (size_t i = end; i < n; ++i) a[i] += b[i];
}

// persia-simd/src/lib.rs:21-77
void decayed_adagrad(float* acc, float* emb, const float* g, size_t n, float mom, float lr, float eps) {
  size_t end = (n / 8) * 8;
  for (size_t i = 0; i < end; i += 8) {
    __m256 s = _mm256_loadu_ps(acc + i), w = _mm256_loadu_ps(emb + i), gv = _mm256_loadu_ps(g + i);
    __m256 sq = _mm256_mul_ps(gv, gv);
    __m256 scaled = _mm256_mul_ps(gv, rsqrt8(_mm256_add_ps(s, _mm256_set1_ps(eps))));
    _mm256_storeu_ps(emb + i, _mm256_fnmadd_ps(_mm256_set1_ps(lr), scaled, w));
    _mm256_storeu_ps(acc + i, _mm256_fmadd_ps(s, _mm256_set1_ps(mom), sq));
  }
  for (size_t i = end; i < n; ++i) {
    float s = acc[i], w = emb[i], gv = g[i];
    float sq = gv * gv;
    float scaled = gv * (1.0f / std::sqrt(s + eps));
    emb[i] = -lr * scaled + w;
    acc[i] = s * mom + sq;
  }
}

// persia-simd/src/lib.rs:81-121
void decayed_adagrad_vectorwise(float acc, float* emb, const float* g, size_t n, float lr, float eps) {
  size_t end = (n / 8) * 8;
  __m256 s = _mm256_set1_ps(acc);
  for (size_t i = 0; i < end; i += 8) {
    __m256 w = _mm256_loadu_ps(emb + i), gv = _mm256_loadu_ps(g + i);
    __m256 scaled = _mm256_mul_ps(gv, rsqrt8(_mm256_add_ps(s, _mm256_set1_ps(eps))));
    _mm256_storeu_ps(emb + i, _mm256_fnmadd_ps(_mm256_set1_ps(lr), scaled, w));
  }
  for (size_t i = end; i < n; ++i) {
    float scaled = g[i] * (1.0f / std::sqrt(acc + eps));
    emb[i] = -lr * scaled + emb[i];
  }
}

// persia-simd/src/lib.rs:124-144
void decayed_sgd(float* emb, const float* g, size_t n, float wd, float lr) {
  size_t end = (n / 8) * 8;
  for (size_t i = 0; i < end; i += 8) {
    __m256 gv = _mm256_loadu_ps(g + i), w = _mm256_loadu_ps(emb + i);
    __m256 dg = _mm256_fmadd_ps(_mm256_set1_ps(wd), w, gv);
    _mm256_storeu_ps(emb + i, _mm256_fnmadd_ps(_mm256_set1_ps(lr), dg, w));
  }
  for (size_t i = end; i < n; ++i) {
    float dg = g[i] + emb[i] * wd;
    emb[i] = emb[i] - lr * dg;
  }
}

// persia-simd/src/lib.rs:147-228
void adam(float* m, float* v, float b1p, float b2p, float* emb, const float* g, size_t n, float lr,
          float b1, float b2, float eps) {
  size_t end = (n / 8) * 8;
  float r1 = 1.0f / (1.0f - b1p), r2 = 1.0f / (1.0f - b2p);
  float omb1 = 1.0f - b1, omb2 = 1.0f - b2;
  for (size_t i = 0; i < end; i += 8) {
    __m256 gv = _mm256_loadu_ps(g + i), w = _mm256_loadu_ps(emb + i);
    __m256 vv = _mm256_loadu_ps(v + i), mv = _mm256_loadu_ps(m + i);
    __m256 um = _mm256_fmadd_ps(_mm256_set1_ps(b1), mv, _mm256_mul_ps(_mm256_set1_ps(omb1), gv));
    __m256 uv = _mm256_fmadd_ps(_mm256_set1_ps(b2), vv,
                                _mm256_mul_ps(_mm256_set1_ps(omb2), _mm256_mul_ps(gv, gv)));
    __m256 mc = _mm256_mul_ps(um, _mm256_set1_ps(r1));
    __m256 vc = _mm256_mul_ps(uv, _mm256_set1_ps(r2));
    __m256 descent = _mm256_div_ps(mc, _mm256_add_ps(_mm256_set1_ps(eps), _mm256_sqrt_ps(vc)));
    _mm256_storeu_ps(m + i, um);
    _mm256_storeu_ps(v + i, uv);
    _mm256_storeu_ps(emb + i, _mm256_fnmadd_ps(_mm256_set1_ps(lr), descent, w));
  }
  for (size_t i = end; i < n; ++i) {
    float um = b1 * m[i] + omb1 * g[i];
    float uv = b2 * v[i] + omb2 * g[i] * g[i];
    float mc = um * r1, vc = uv * r2;
    float descent = mc / (eps + std::sqrt(vc));
    float w = emb[i] - lr * descent;
    m[i] = um;
    v[i] = uv;
    emb[i] = w;
  }
}

// persia-simd/src/lib.rs:231-251
void weight_bound(float* emb, size_t n, float b) {
  size_t end = (n / 8) * 8;
  for (size_t i = 0; i < end; i += 8) {
    __m256 w = _mm256_loadu_ps(emb + i);
    _mm256_storeu_ps(emb + i, _mm256_min_ps(_mm256_max_ps(w, _mm256_set1_ps(-b)), _mm256_set1_ps(b)));
  }
  for (size_t i = end; i < n; ++i) emb[i] = std::fmin(std::fmax(emb[i], -b), b);
}

// ndarray 0.15.3 numeric_util::unrolled_dot (third-party; pinned by the
// vectorwise golden vector).  Eight partial sums, no FMA.
float unrolled_dot(const float* x, const float* y, size_t n) {
  float p[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  size_t i = 0;
  for (; i + 8 <= n; i += 8)
    for (int k = 0; k < 8; ++k) p[k] = p[k] + x[i + k] * y[i + k];
  float sum = 0.0f;
  sum = sum + (p[0] + p[4]);
  sum = sum + (p[1] + p[5]);
  sum = sum + (p[2] + p[6]);
  sum = sum + (p[3] + p[7]);
  for (; i < n; ++i) sum = sum + x[i] * y[i];
  return sum;
}

// ---------------------------------------------------------------------------
// persia-common/src/optim.rs:66-307 — Optimizable
// ---------------------------------------------------------------------------
struct OptimCfg {
  int kind = -1;  // 0 SGD, 1 Adagrad, 2 Adagrad vectorwise-shared, 3 Adam
  float lr = 0, wd = 0, mom = 1, init_acc = 0, eps = 0, b1 = 0, b2 = 0;
};

inline size_t require_space(const OptimCfg& o, size_t dim) {  // optim.rs:84,141,252
  switch (o.kind) {
    case 1: return dim;
    case 2: return 1;
    case 3: return 2 * dim;
    default: return 0;
  }
}
inline void state_initialization(const OptimCfg& o, float* entry, size_t dim) {  // optim.rs:299-302
  if (o.kind == 1 || o.kind == 2) {
    size_t s = require_space(o, dim);
    for (size_t i = 0; i < s; ++i) entry[dim + i] = o.init_acc;
  }
}
// optim.rs:199-221 (Adam), :229-239 (SGD), :260-296 (Adagrad)
inline void optim_update(const OptimCfg& o, float* entry, size_t entry_len, const float* g, size_t dim,
                         float b1p, float b2p) {
  switch (o.kind) {
    case 0: decayed_sgd(entry, g, entry_len, o.wd, o.lr); break;  // whole entry; SGD keeps no state
    case 1: decayed_adagrad(entry + dim, entry, g, dim, o.mom, o.lr, o.eps); break;
    case 2: {
      float* s = entry + dim;
      decayed_adagrad_vectorwise(*s, entry, g, dim, o.lr, o.eps);
      float gs = unrolled_dot(g, g, dim) / (float)dim;
      *s = *s * o.mom + gs;
      break;
    }
    case 3: adam(entry + dim, entry + 2 * dim, b1p, b2p, entry, g, dim, o.lr, o.b1, o.b2, o.eps); break;
    default: break;
  }
}

// ---------------------------------------------------------------------------
// New-row initialisation: emb_entry.rs:28-68 (BoundedUniform arm).
// PARITY UNPINNED — restated from the published sources of rand_core 0.6
// (seed_from_u64 default: PCG32 expansion), rand 0.8.4 SmallRng (64-bit:
// Xoshiro256++, next_u32 = upper half of next_u64) and rand 0.8 UniformFloat.
// ---------------------------------------------------------------------------
struct Xoshiro256pp {
  uint64_t s[4];
  explicit Xoshiro256pp(uint64_t seed) {
    uint64_t state = seed;
    uint32_t w[8];
    for (int i = 0; i < 8; ++i) {
      state = state * 6364136223846793005ULL + 11634580027462260723ULL;
      uint32_t xs = (uint32_t)(((state >> 18) ^ state) >> 27);
      uint32_t rot = (uint32_t)(state >> 59);
      w[i] = (xs >> rot) | (xs << ((32 - rot) & 31));
    }
    for (int i = 0; i < 4; ++i) s[i] = (uint64_t)w[2 * i] | ((uint64_t)w[2 * i + 1] << 32);
  }
  uint64_t next() {
    auto rotl = [](uint64_t x, int k) { return (x << k) | (x >> (64 - k)); };
    uint64_t r = rotl(s[0] + s[3], 23) + s[0];
    uint64_t t = s[1] << 17;
    s[2] ^= s[0];
    s[3] ^= s[1];
    s[1] ^= s[2];
    s[0] ^= s[3];
    s[2] ^= t;
    s[3] = rotl(s[3], 45);
    return r;
  }
};

inline float uniform_scale(float lo, float hi) {
  float scale = hi - lo;
  uint32_t mb = (0xFFFFFFFFu >> 9) | 0x3f800000u;
  float max_rand;
  std::memcpy(&max_rand, &mb, 4);
  max_rand -= 1.0f;
  while (!(scale * max_rand + lo < hi)) {
    uint32_t b;
    std::memcpy(&b, &scale, 4);
    b -= 1;
    std::memcpy(&scale, &b, 4);
  }
  return scale;
}

void init_row(uint64_t seed, size_t dim, float lo, float hi, float* out) {
  Xoshiro256pp rng(seed);
  float scale = uniform_scale(lo, hi);
  for (size_t i = 0; i < dim; ++i) {
    uint32_t r = (uint32_t)(rng.next() >> 32);
    uint32_t bits = (r >> 9) | 0x3f800000u;
    float v12;
    std::memcpy(&v12, &bits, 4);
    float v01 = v12 - 1.0f;
    out[i] = v01 * scale + lo;
  }
}

// ---------------------------------------------------------------------------
// Flat open-addressing map u64 -> u32 (stand-in for hashbrown 0.11; only its
// set semantics are observable).
// ---------------------------------------------------------------------------
struct FlatMap {
  std::vector<uint64_t> keys;
  std::vector<uint32_t> vals;
  std::vector<uint8_t> used;
  size_t mask = 0, count = 0;
  explicit FlatMap(size_t cap_hint = 16) { rehash(cap_hint * 2); }
  static uint64_t mix(uint64_t k) {
    k ^= k >> 33;
    k *= 0xff51afd7ed558ccdULL;
    k ^= k >> 33;
    k *= 0xc4ceb9fe1a85ec53ULL;
    k ^= k >> 33;
    return k;
  }
  void rehash(size_t want) {
    size_t n = 16;
    while (n < want) n <<= 1;
    std::vector<uint64_t> ok;
    std::vector<uint32_t> ov;
    std::vector<uint8_t> ou;
    ok.swap(keys);
    ov.swap(vals);
    ou.swap(used);
    keys.assign(n, 0);
    vals.assign(n, 0);
    used.assign(n, 0);
    mask = n - 1;
    count = 0;
    for (size_t i = 0; i < ok.size(); ++i)
      if (ou[i]) *slot(ok[i], true) = ov[i];
  }
  // find (insert=false: nullptr when absent) or find-or-insert (value left as is / 0)
  uint32_t* slot(uint64_t k, bool insert) {
    size_t i = mix(k) & mask;
    while (used[i]) {
      if (keys[i] == k) return &vals[i];
      i = (i + 1) & mask;
    }
    if (!insert) return nullptr;
    if ((count + 1) * 2 > mask + 1) {
      rehash((mask + 1) * 2);
      return slot(k, true);
    }
    used[i] = 1;
    keys[i] = k;
    vals[i] = 0;
    ++count;
    return &vals[i];
  }
  bool erase(uint64_t k) {
    size_t i = mix(k) & mask;
    while (used[i]) {
      if (keys[i] == k) break;
      i = (i + 1) & mask;
    }
    if (!used[i]) return false;
    // backward-shift deletion
    size_t j = i;
    for (;;) {
      j = (j + 1) & mask;
      if (!used[j]) break;
      size_t h = mix(keys[j]) & mask;
      bool between = (i <= j) ? (i < h && h <= j) : (i < h || h <= j);
      if (!between) {
        keys[i] = keys[j];
        vals[i] = vals[j];
        i = j;
      }
    }
    used[i] = 0;
    --count;
    return true;
  }
  void clear() {
    std::fill(used.begin(), used.end(), 0);
    count = 0;
  }
};

// ---------------------------------------------------------------------------
// persia-embedding-holder/src/emb_entry.rs:17-25 + eviction_map.rs:11-111
// EvictionMap = hash map (key -> node index) + LRU linked list held in an
// array (array_linked_list.rs; only its list semantics matter here).
// ---------------------------------------------------------------------------
struct Entry {
  std::vector<float> inner;  // emb(dim) ++ optimizer state
  size_t dim = 0;
  uint64_t sign = 0;
};

struct EvictionMap {
  struct Node {
    uint32_t prev, next;
    bool live;
    Entry e;
  };
  static constexpr uint32_t NIL = 0xFFFFFFFFu;
  FlatMap map;
  std::vector<Node> nodes;
  std::vector<uint32_t> free_nodes;
  uint32_t head = NIL, tail = NIL;
  size_t len = 0, capacity;
  explicit EvictionMap(size_t cap) : map(1024), capacity(cap) {}

  uint32_t push_back(Entry&& e) {
    uint32_t idx;
    if (!free_nodes.empty()) {
      idx = free_nodes.back();
      free_nodes.pop_back();
    } else {
      idx = (uint32_t)nodes.size();
      nodes.emplace_back();
    }
    Node& n = nodes[idx];
    n.e = std::move(e);
    n.live = true;
    n.prev = tail;
    n.next = NIL;
    if (tail != NIL) nodes[tail].next = idx; else head = idx;
    tail = idx;
    ++len;
    return idx;
  }
  Entry unlink(uint32_t idx) {
    Node& n = nodes[idx];
    if (n.prev != NIL) nodes[n.prev].next = n.next; else head = n.next;
    if (n.next != NIL) nodes[n.next].prev = n.prev; else tail = n.prev;
    n.live = false;
    free_nodes.push_back(idx);
    --len;
    return std::move(n.e);
  }
  Entry* get(uint64_t k) {  // :34-46 get / get_mut
    uint32_t* p = map.slot(k, false);
    return p ? &nodes[*p].e : nullptr;
  }
  Entry* get_refresh(uint64_t k) {  // :48-60 — move to the LRU tail
    uint32_t* p = map.slot(k, false);
    if (!p) return nullptr;
    Entry e = unlink(*p);
    uint32_t ni = push_back(std::move(e));
    *map.slot(k, false) = ni;
    return &nodes[ni].e;
  }
  void insert(uint64_t k, Entry&& e) {  // :76-97
    uint32_t* p = map.slot(k, false);
    if (p) (void)unlink(*p);
    uint32_t ni = push_back(std::move(e));
    *map.slot(k, true) = ni;
    if (len > capacity && head != NIL) {
      Entry ev = unlink(head);
      map.erase(ev.sign);
    }
  }
  void clear() {
    map.clear();
    nodes.clear();
    free_nodes.clear();
    head = tail = NIL;
    len = 0;
  }
};

// ---------------------------------------------------------------------------
// One embedding-parameter-server replica ("PS"):
//   persia-embedding-holder/src/lib.rs:27-101 + sharded.rs:10-27 (lock-striped
//   internal shards) and embedding_parameter_service/mod.rs:162-262, 287-306,
//   359-427, 429-451.
// ---------------------------------------------------------------------------
struct Hyper {  // PersiaEmbeddingModelHyperparameters (configure, mod.rs:440-451)
  float lo = -0.01f, hi = 0.01f, admit_p = 1.0f, wb = 10.0f;
  int enable_wb = 1;
};

struct ParamServer {
  std::vector<std::unique_ptr<EvictionMap>> shards;
  std::vector<std::unique_ptr<std::mutex>> locks;
  OptimCfg optim;
  Hyper hyper;
  bool configured = false;
  int faithful_miss = 1;  // see update(): the reference does not advance the gradient cursor on a miss
  std::atomic<uint64_t> index_miss{0}, grad_miss{0};
  uint64_t admit_rng = 0x9E3779B97F4A7C15ULL;  // reference: unseeded thread_rng (unpinned); only used when admit_p < 1
  // Adam: accumulated beta powers per feature group (optim.rs:99-131); key = sign & prefix mask
  uint32_t prefix_bit = 8;
  std::vector<std::pair<uint64_t, std::pair<float, float>>> accum_betas;
  std::mutex adam_lock;

  ParamServer(size_t capacity, size_t n_internal) {
    if (n_internal == 0) n_internal = 1;
    size_t per = capacity / n_internal;  // holder lib.rs:42-43
    for (size_t i = 0; i < n_internal; ++i) {
      shards.emplace_back(new EvictionMap(per));
      locks.emplace_back(new std::mutex());
    }
  }
  // sharded.rs:10-18 uses ahash 0.7 (unpinned, affects only which LRU list evicts)
  size_t shard_of(uint64_t sign) const { return FlatMap::mix(sign ^ 0x51afd7ed558ccd00ULL) % shards.size(); }

  bool admit() {
    if (hyper.admit_p >= 1.0f) return true;
    admit_rng ^= admit_rng << 13;
    admit_rng ^= admit_rng >> 7;
    admit_rng ^= admit_rng << 17;
    float u = (float)((admit_rng >> 40) * (1.0 / 16777216.0));
    return u < hyper.admit_p;
  }

  Entry make_entry(uint64_t sign, size_t dim) {  // emb_entry.rs:28-68
    Entry e;
    e.dim = dim;
    e.sign = sign;
    e.inner.assign(dim + require_space(optim, dim), 0.0f);
    init_row(sign, dim, hyper.lo, hyper.hi, e.inner.data());
    return e;
  }

  // mod.rs:162-262.  Returns 0, or -1 when training without optimizer/config.
  int lookup(const uint64_t* signs, const uint32_t* dims, size_t n, int training, float* out) {
    if (training && (optim.kind < 0 || !configured)) return -1;
    uint64_t miss = 0;
    for (size_t i = 0; i < n; ++i) {
      uint64_t sign = signs[i];
      size_t dim = dims[i];
      size_t si = shard_of(sign);
      std::lock_guard<std::mutex> g(*locks[si]);
      EvictionMap& m = *shards[si];
      if (training) {
        Entry* e = m.get_refresh(sign);
        if (!e) {
          if (admit()) {
            Entry ne = make_entry(sign, dim);
            state_initialization(optim, ne.inner.data(), dim);
            std::memcpy(out, ne.inner.data(), dim * 4);
            m.insert(sign, std::move(ne));
            ++miss;
          } else {
            std::memset(out, 0, dim * 4);
          }
        } else if (e->dim != dim) {
          Entry ne = make_entry(sign, dim);  // NB: the reference skips state_initialization here (mod.rs:216-226)
          std::memcpy(out, ne.inner.data(), dim * 4);
          m.insert(sign, std::move(ne));
        } else {
          std::memcpy(out, e->inner.data(), dim * 4);
        }
      } else {
        Entry* e = m.get(sign);
        if (e && e->dim == dim) {
          std::memcpy(out, e->inner.data(), dim * 4);
        } else {
          std::memset(out, 0, dim * 4);
          if (!e) ++miss;
        }
      }
      out += dim;
    }
    index_miss += miss;
    return 0;
  }

  // mod.rs:359-427.  `grads` is the concatenation of per-sign gradients.
  // Faithful quirk: when a sign is absent the reference does NOT consume its
  // gradient slice (the split happens inside `if let Some(entry)`), so every
  // later sign in the request reads a shifted slice.  faithful_miss=0 skips
  // the slice instead (what the GPU path does; needs `dims`).
  int update(const uint64_t* signs, const uint32_t* dims, size_t n, const float* grads, size_t n_grad_floats) {
    if (optim.kind < 0 || !configured) return -1;
    const float* cur = grads;
    const float* end = grads + n_grad_floats;
    uint64_t miss = 0;
    // Adam batch-level state (optim.rs:155-197): the first sign of every feature group seen in this request
    // advances that group's accumulated (beta1^t, beta2^t); every sign of the group then uses the advanced pair.
    std::vector<float> b1p(n, 0.0f), b2p(n, 0.0f);
    if (optim.kind == 3) {
      std::lock_guard<std::mutex> g(adam_lock);
      const uint64_t mask = ~((1ULL << (64 - prefix_bit)) - 1ULL);
      std::vector<std::pair<uint64_t, std::pair<float, float>>> stepped;
      for (size_t i = 0; i < n; ++i) {
        uint64_t m = signs[i] & mask;
        bool done = false;
        for (auto& st : stepped)
          if (st.first == m) {
            b1p[i] = st.second.first;
            b2p[i] = st.second.second;
            done = true;
            break;
          }
        if (done) continue;
        std::pair<float, float>* acc = nullptr;
        for (auto& a : accum_betas)
          if (a.first == m) acc = &a.second;
        if (!acc) {  // Adam::new seeds every feature group with (beta1, beta2) (optim.rs:104-131)
          accum_betas.push_back({m, {optim.b1, optim.b2}});
          acc = &accum_betas.back().second;
        }
        acc->first = acc->first * optim.b1;
        acc->second = acc->second * optim.b2;
        b1p[i] = acc->first;
        b2p[i] = acc->second;
        stepped.push_back({m, *acc});
      }
    }
    for (size_t i = 0; i < n; ++i) {
      uint64_t sign = signs[i];
      size_t si = shard_of(sign);
      std::lock_guard<std::mutex> g(*locks[si]);
      Entry* e = shards[si]->get(sign);
      if (e) {
        size_t d = e->dim;
        if (cur + d > end) return -2;  // the reference would panic in split_at
        optim_update(optim, e->inner.data(), e->inner.size(), cur, d, b1p[i], b2p[i]);
        if (hyper.enable_wb) weight_bound(e->inner.data(), d, hyper.wb);
        cur += d;
      } else {
        ++miss;
        if (!faithful_miss && dims) cur += dims[i];
      }
    }
    grad_miss += miss;
    return 0;
  }

  void set_entry(uint64_t sign, const float* inner, size_t dim, size_t inner_len) {  // mod.rs:287-306
    Entry e;
    e.dim = dim;
    e.sign = sign;
    e.inner.assign(inner, inner + inner_len);
    size_t si = shard_of(sign);
    std::lock_guard<std::mutex> g(*locks[si]);
    shards[si]->insert(sign, std::move(e));
  }
  size_t len() const {
    size_t t = 0;
    for (auto& s : shards) t += s->len;
    return t;
  }
};

// ---------------------------------------------------------------------------
// Slot semantics: persia-embedding-config/src/lib.rs:528-650.
// ---------------------------------------------------------------------------
struct Slot {
  uint32_t dim = 0;
  int summation = 1, sqrt_scaling = 0;
  uint32_t sample_fixed_size = 10;
  uint32_t hs_rounds = 0;
  uint64_t hs_size = 0;
  uint64_t prefix = 0;
};

// ---------------------------------------------------------------------------
// persia-common/src/lib.rs:45-82 FeatureBatch::new — per-slot dedup.
// hashbrown's iteration order (which defines index_batch order) is random per
// process in the reference; here uniques are numbered in FIRST-OCCURRENCE
// order.  Occurrence lists keep (sample, col) in push order, as there.
// ---------------------------------------------------------------------------
struct FeatureBatch {
  std::vector<uint64_t> signs;       // index_batch[i].sign
  std::vector<uint32_t> seg_off;     // CSR into occ_* per unique
  std::vector<uint16_t> occ_sample;  // in_which_batch_samples.0
  std::vector<uint16_t> occ_col;     // in_which_batch_samples.1
  std::vector<uint32_t> sample_num_signs;
  uint32_t batch_size = 0;
};

int feature_batch_new(const uint64_t* ids, const uint32_t* row_off, uint32_t B, FeatureBatch& fb) {
  if (B > 65535) return -1;  // lib.rs:49-51 panics
  fb = FeatureBatch();
  fb.batch_size = B;
  fb.sample_num_signs.resize(B);
  uint32_t n = row_off[B] - row_off[0];
  FlatMap m(n + 1);
  std::vector<uint32_t> uid(n);
  std::vector<uint32_t> cnt;
  uint32_t k = 0;
  for (uint32_t b = 0; b < B; ++b) {
    fb.sample_num_signs[b] = row_off[b + 1] - row_off[b];
    for (uint32_t j = row_off[b]; j < row_off[b + 1]; ++j, ++k) {
      size_t before = m.count;
      uint32_t* p = m.slot(ids[j], true);
      if (m.count != before) {
        *p = (uint32_t)fb.signs.size();
        fb.signs.push_back(ids[j]);
        cnt.push_back(0);
      }
      uid[k] = *p;
      ++cnt[*p];
    }
  }
  size_t U = fb.signs.size();
  fb.seg_off.assign(U + 1, 0);
  for (size_t u = 0; u < U; ++u) fb.seg_off[u + 1] = fb.seg_off[u] + cnt[u];
  fb.occ_sample.resize(n);
  fb.occ_col.resize(n);
  std::vector<uint32_t> cur(fb.seg_off.begin(), fb.seg_off.end() - 1);
  k = 0;
  for (uint32_t b = 0; b < B; ++b)
    for (uint32_t j = row_off[b]; j < row_off[b + 1]; ++j, ++k) {
      uint32_t pos = cur[uid[k]]++;
      fb.occ_sample[pos] = (uint16_t)b;
      fb.occ_col[pos] = (uint16_t)(j - row_off[b]);
    }
  return 0;
}

// embedding_worker_service/mod.rs:347-400 — hash stack (regroups occurrences per hashed key).
// Within a round, keys are emitted in first-occurrence order (reference: hashmap order).
void hashstack(FeatureBatch& fb, const Slot& s) {
  if (s.hs_rounds == 0) return;
  FeatureBatch out;
  out.batch_size = fb.batch_size;
  size_t U = fb.signs.size();
  std::vector<uint64_t> h(fb.signs);
  std::vector<std::vector<uint32_t>> groups;  // per new key: list of old uniques
  for (uint32_t r = 0; r < s.hs_rounds; ++r) {
    FlatMap m(U + 1);
    size_t base = out.signs.size();
    for (size_t u = 0; u < U; ++u) {
      h[u] = farmhash64_u64(h[u]);
      uint64_t key = h[u] % s.hs_size + (uint64_t)r * s.hs_size;
      size_t before = m.count;
      uint32_t* p = m.slot(key, true);
      if (m.count != before) {
        *p = (uint32_t)(out.signs.size() - base);
        out.signs.push_back(key);
        groups.emplace_back();
      }
      groups[base + *p].push_back((uint32_t)u);
    }
  }
  out.seg_off.push_back(0);
  for (size_t k = 0; k < out.signs.size(); ++k) {
    for (uint32_t u : groups[k])
      for (uint32_t j = fb.seg_off[u]; j < fb.seg_off[u + 1]; ++j) {
        out.occ_sample.push_back(fb.occ_sample[j]);
        out.occ_col.push_back(fb.occ_col[j]);
      }
    out.seg_off.push_back((uint32_t)out.occ_sample.size());
  }
  out.sample_num_signs = fb.sample_num_signs;
  for (auto& x : out.sample_num_signs) x *= s.hs_rounds;
  fb = std::move(out);
}

// embedding_worker_service/mod.rs:402-429
inline uint64_t feature_spacing(uint32_t prefix_bit) {
  return prefix_bit > 0 ? ((1ULL << (64 - prefix_bit)) - 1) : ~0ULL;
}
void add_prefix(FeatureBatch& fb, const Slot& s, uint32_t prefix_bit) {
  if (s.prefix == 0) return;
  uint64_t sp = feature_spacing(prefix_bit);
  for (auto& x : fb.signs) x = x % sp + s.prefix;
}

// ---------------------------------------------------------------------------
// The embedding worker ("EW") with its R parameter servers, in process.
// ---------------------------------------------------------------------------
struct Worker {
  std::vector<Slot> slots;
  uint32_t prefix_bit = 8;
  std::vector<std::unique_ptr<ParamServer>> ps;

  struct Ctx {  // post_forward_buffer entry (mod.rs:639, 1087-1098)
    std::vector<FeatureBatch> fbs;
  };

  // mod.rs:448-484 + 874-942 + 486-629 (summation slots; raw slots: forward_raw below)
  // ids: flat, slot-major; row_off: S*B+1 offsets; out: per slot [B,dim] f16, concatenated.
  int forward(const uint64_t* ids, const uint32_t* row_off, uint32_t B, int training, uint16_t* out, Ctx* keep) {
    size_t S = slots.size(), R = ps.size();
    std::vector<FeatureBatch> fbs(S);
    for (size_t s = 0; s < S; ++s) {
      const uint32_t* ro = row_off + s * B;
      if (feature_batch_new(ids, ro, B, fbs[s]) != 0) return -1;
      hashstack(fbs[s], slots[s]);
      add_prefix(fbs[s], slots[s], prefix_bit);
    }
    // indices_to_sharded_indices (mod.rs:454-479): (slot, index_batch) order per shard
    struct SW { uint64_t sign; uint32_t sign_idx, slot, dim; };
    std::vector<std::vector<SW>> sharded(R);
    for (size_t s = 0; s < S; ++s)
      for (size_t u = 0; u < fbs[s].signs.size(); ++u) {
        uint64_t sign = fbs[s].signs[u];
        sharded[farmhash64_u64(sign) % R].push_back({sign, (uint32_t)u, (uint32_t)s, slots[s].dim});
      }
    // per-slot f32 accumulators
    std::vector<std::vector<float>> acc(S);
    for (size_t s = 0; s < S; ++s) acc[s].assign((size_t)B * slots[s].dim, 0.0f);
    std::vector<uint64_t> sg;
    std::vector<uint32_t> dm;
    std::vector<float> rows;
    for (size_t r = 0; r < R; ++r) {
      size_t n = sharded[r].size();
      sg.resize(n);
      dm.resize(n);
      size_t tot = 0;
      for (size_t i = 0; i < n; ++i) {
        sg[i] = sharded[r][i].sign;
        dm[i] = sharded[r][i].dim;
        tot += dm[i];
      }
      rows.resize(tot);
      if (ps[r]->lookup(sg.data(), dm.data(), n, training, rows.data()) != 0) return -2;
      const float* p = rows.data();
      for (size_t i = 0; i < n; ++i) {  // postprocess, summation arm (mod.rs:547-561)
        const SW& w = sharded[r][i];
        const FeatureBatch& fb = fbs[w.slot];
        for (uint32_t j = fb.seg_off[w.sign_idx]; j < fb.seg_off[w.sign_idx + 1]; ++j)
          add_assign(acc[w.slot].data() + (size_t)fb.occ_sample[j] * w.dim, p, w.dim);
        p += w.dim;
      }
    }
    uint16_t* o = out;
    for (size_t s = 0; s < S; ++s) {
      uint32_t dim = slots[s].dim;
      if (slots[s].sqrt_scaling) {  // mod.rs:571-579
        for (uint32_t b = 0; b < B; ++b) {
          uint32_t c = fbs[s].sample_num_signs[b];
          float f = 1.0f / std::sqrt((float)std::max<uint32_t>(c, 1));
          for (uint32_t d = 0; d < dim; ++d) acc[s][(size_t)b * dim + d] *= f;
        }
      }
      for (size_t i = 0; i < (size_t)B * dim; ++i) o[i] = f32_to_f16(acc[s][i]);
      o += (size_t)B * dim;
    }
    if (keep) keep->fbs = std::move(fbs);
    return 0;
  }

  // mod.rs:703-872.  grads: per slot [B,dim], f16 or f32 (is_f16), concatenated; skip[s]!=0 = Skipped.
  // slot_status (optional, S ints): 0 applied, 1 skipped by caller, 2 skipped for NaN.
  int backward(const Ctx& ctx, const void* grads, int is_f16, const float* scale, const int* skip, int* slot_status) {
    size_t S = slots.size(), R = ps.size();
    std::vector<std::vector<uint64_t>> sh_signs(R);
    std::vector<std::vector<uint32_t>> sh_dims(R);
    std::vector<std::vector<float>> sh_grads(R);
    const uint8_t* gp = (const uint8_t*)grads;
    std::vector<float> g32, sg;
    for (size_t s = 0; s < S; ++s) {
      const FeatureBatch& fb = ctx.fbs[s];
      uint32_t dim = slots[s].dim, B = fb.batch_size;
      size_t n = (size_t)B * dim;
      const uint8_t* mine = gp;
      gp += n * (is_f16 ? 2 : 4);
      if (slot_status) slot_status[s] = 0;
      if (skip && skip[s]) {
        if (slot_status) slot_status[s] = 1;
        continue;
      }
      g32.resize(n);
      bool nan = false;
      if (is_f16) {
        const uint16_t* h = (const uint16_t*)mine;
        for (size_t i = 0; i < n; ++i) {
          if ((h[i] & 0x7c00) == 0x7c00 && (h[i] & 0x03ff)) { nan = true; break; }
        }
        if (!nan)
          for (size_t i = 0; i < n; ++i) {  // persia-common lib.rs:163-180: ±inf -> ±65504
            float v = f16_to_f32(h[i]);
            if (v == INFINITY) v = 65504.0f; else if (v == -INFINITY) v = -65504.0f;
            g32[i] = v;
          }
      } else {
        const float* f = (const float*)mine;
        for (size_t i = 0; i < n; ++i) if (std::isnan(f[i])) { nan = true; break; }
        if (!nan) std::memcpy(g32.data(), f, n * 4);
      }
      if (nan) {  // mod.rs:731-746 — the whole slot is skipped
        if (slot_status) slot_status[s] = 2;
        continue;
      }
      float sc = scale ? scale[s] : 1.0f;
      if (std::fabs(sc - 1.0f) > 1.1920929e-07f) {  // mod.rs:751-755: multiply by the reciprocal
        float r = 1.0f / sc;
        for (size_t i = 0; i < n; ++i) g32[i] *= r;
      }
      if (slots[s].sqrt_scaling) {  // mod.rs:757-778 (no max(.,1) here, unlike forward)
        for (uint32_t b = 0; b < B; ++b) {
          float f = 1.0f / std::sqrt((float)fb.sample_num_signs[b]);
          for (uint32_t d = 0; d < dim; ++d) g32[(size_t)b * dim + d] *= f;
        }
      }
      size_t U = fb.signs.size();
      sg.assign(U * dim, 0.0f);
      for (size_t u = 0; u < U; ++u)  // mod.rs:786-812, summation arm
        for (uint32_t j = fb.seg_off[u]; j < fb.seg_off[u + 1]; ++j)
          add_assign(sg.data() + u * dim, g32.data() + (size_t)fb.occ_sample[j] * dim, dim);
      for (size_t u = 0; u < U; ++u) {  // mod.rs:813-821
        size_t r = farmhash64_u64(fb.signs[u]) % R;
        sh_signs[r].push_back(fb.signs[u]);
        sh_dims[r].push_back(dim);
        sh_grads[r].insert(sh_grads[r].end(), sg.begin() + u * dim, sg.begin() + (u + 1) * dim);
      }
    }
    for (size_t r = 0; r < R; ++r)
      if (ps[r]->update(sh_signs[r].data(), sh_dims[r].data(), sh_signs[r].size(), sh_grads[r].data(),
                        sh_grads[r].size()) != 0)
        return -2;
    return 0;
  }

  // ---- raw (embedding_summation = false) slot, one slot per request -------------------------------
  // mod.rs:498-512 (table of distinct signs + zero row 0), :540-545 (row idx+1 = embedding), :593-623
  // (index / sample_id_num).  Hash-stack on a raw slot (:503-507, :581-590) is not restated.
  // table: (U+1)*dim f16 (caller sizes it for n_occ+1 rows); index: B*fixed; returns U via *n_distinct.
  int forward_raw(uint32_t slot, const uint64_t* ids, const uint32_t* row_off, uint32_t B, int training,
                  uint16_t* table, int64_t* index, uint32_t* sample_id_num, uint32_t* n_distinct, Ctx* keep) {
    const Slot& sc = slots[slot];
    if (sc.hs_rounds) return -3;
    size_t R = ps.size();
    FeatureBatch fb;
    if (feature_batch_new(ids, row_off, B, fb) != 0) return -1;
    add_prefix(fb, sc, prefix_bit);
    const uint32_t dim = sc.dim, fixed = sc.sample_fixed_size;
    size_t U = fb.signs.size();
    std::vector<float> res((U + 1) * dim, 0.0f);
    std::vector<std::vector<uint32_t>> sharded(R);
    for (size_t u = 0; u < U; ++u) sharded[farmhash64_u64(fb.signs[u]) % R].push_back((uint32_t)u);
    std::vector<uint64_t> sg;
    std::vector<uint32_t> dm;
    std::vector<float> rows;
    for (size_t r = 0; r < R; ++r) {
      size_t n = sharded[r].size();
      sg.resize(n);
      dm.assign(n, dim);
      for (size_t i = 0; i < n; ++i) sg[i] = fb.signs[sharded[r][i]];
      rows.resize(n * dim);
      if (ps[r]->lookup(sg.data(), dm.data(), n, training, rows.data()) != 0) return -2;
      for (size_t i = 0; i < n; ++i)  // sign2idx[sign] + 1 (mod.rs:540-545); sign2idx = index_batch position
        std::memcpy(res.data() + ((size_t)sharded[r][i] + 1) * dim, rows.data() + i * dim, dim * 4);
    }
    for (size_t i = 0; i < (U + 1) * dim; ++i) table[i] = f32_to_f16(res[i]);
    std::fill(index, index + (size_t)B * fixed, (int64_t)0);
    std::fill(sample_id_num, sample_id_num + B, 0u);
    for (size_t u = 0; u < U; ++u)  // mod.rs:601-616
      for (uint32_t j = fb.seg_off[u]; j < fb.seg_off[u + 1]; ++j) {
        uint32_t b = fb.occ_sample[j], col = fb.occ_col[j];
        if (sample_id_num[b] < fixed && col < fixed) {
          index[(size_t)b * fixed + col] = (int64_t)u + 1;
          sample_id_num[b] += 1;
        }
      }
    *n_distinct = (uint32_t)U;
    if (keep) {
      keep->fbs.clear();
      keep->fbs.push_back(std::move(fb));
    }
    return 0;
  }

  // raw arm of update_all_batched_gradients (mod.rs:731-755, :790-798): grads [U, dim]
  int backward_raw(uint32_t slot, const Ctx& ctx, const void* grads, int is_f16, float scale, int skip, int* status) {
    size_t R = ps.size();
    const FeatureBatch& fb = ctx.fbs[0];
    const uint32_t dim = slots[slot].dim;
    size_t U = fb.signs.size(), n = U * dim;
    if (status) *status = 0;
    if (skip) {
      if (status) *status = 1;
      return 0;
    }
    std::vector<float> g32(n);
    bool nan = false;
    if (is_f16) {
      const uint16_t* h = (const uint16_t*)grads;
      for (size_t i = 0; i < n; ++i)
        if ((h[i] & 0x7c00) == 0x7c00 && (h[i] & 0x03ff)) { nan = true; break; }
      if (!nan)
        for (size_t i = 0; i < n; ++i) {
          float v = f16_to_f32(h[i]);
          if (v == INFINITY) v = 65504.0f; else if (v == -INFINITY) v = -65504.0f;
          g32[i] = v;
        }
    } else {
      const float* f = (const float*)grads;
      for (size_t i = 0; i < n; ++i) if (std::isnan(f[i])) { nan = true; break; }
      if (!nan) std::memcpy(g32.data(), f, n * 4);
    }
    if (nan) {
      if (status) *status = 2;
      return 0;
    }
    if (std::fabs(scale - 1.0f) > 1.1920929e-07f) {
      float r = 1.0f / scale;
      for (size_t i = 0; i < n; ++i) g32[i] *= r;
    }
    // sqrt_scaling only scales a raw slot's gradient when hash-stack is on (mod.rs:769-776)
    std::vector<std::vector<uint64_t>> sh_signs(R);
    std::vector<std::vector<uint32_t>> sh_dims(R);
    std::vector<std::vector<float>> sh_grads(R);
    for (size_t u = 0; u < U; ++u) {  // hashed2index_batch_idx[sign] == u (mod.rs:790-798), then :813-821
      size_t r = farmhash64_u64(fb.signs[u]) % R;
      sh_signs[r].push_back(fb.signs[u]);
      sh_dims[r].push_back(dim);
      sh_grads[r].insert(sh_grads[r].end(), g32.begin() + u * dim, g32.begin() + (u + 1) * dim);
    }
    for (size_t r = 0; r < R; ++r)
      if (ps[r]->update(sh_signs[r].data(), sh_dims[r].data(), sh_signs[r].size(), sh_grads[r].data(),
                        sh_grads[r].size()) != 0)
        return -2;
    return 0;
  }
};

}  // namespace

// ===========================================================================
// C API (ctypes)
// ===========================================================================
extern "C" {

uint64_t po_farmhash64(uint64_t x) { return farmhash64_u64(x); }
void po_farmhash64_many(const uint64_t* x, uint64_t n, uint64_t* out) {
  for (uint64_t i = 0; i < n; ++i) out[i] = farmhash64_u64(x[i]);
}
void po_shard_of(const uint64_t* signs, uint64_t n, uint64_t R, uint32_t* out) {  // sign_to_shard_modulo
  for (uint64_t i = 0; i < n; ++i) out[i] = (uint32_t)(farmhash64_u64(signs[i]) % R);
}
void po_add_prefix(uint64_t* signs, uint64_t n, uint32_t prefix_bit, uint64_t prefix) {
  if (prefix == 0) return;
  uint64_t sp = feature_spacing(prefix_bit);
  for (uint64_t i = 0; i < n; ++i) signs[i] = signs[i] % sp + prefix;
}
// parse_embedding_config prefix rule (persia-embedding-config/src/lib.rs:630-647)
uint64_t po_index_prefix(uint32_t feature_group_index, uint32_t prefix_bit) {
  return ((uint64_t)feature_group_index + 1) << (64 - prefix_bit);
}
void po_set_rsqrt_exact(int exact) { g_rsqrt_exact = exact; }
void po_init_row(uint64_t sign, uint32_t dim, float lo, float hi, float* out) { init_row(sign, dim, lo, hi, out); }
void po_f32_to_f16(const float* in, uint64_t n, uint16_t* out) { for (uint64_t i = 0; i < n; ++i) out[i] = f32_to_f16(in[i]); }
void po_add_assign(float* a, const float* b, uint64_t n) { add_assign(a, b, n); }
void po_weight_bound(float* e, uint64_t n, float b) { weight_bound(e, n, b); }

// Optimizable on a bare entry (the shape of optim.rs's own execute_test, :338-360)
uint32_t po_optim_require_space(int kind, uint32_t dim) {
  OptimCfg o;
  o.kind = kind;
  return (uint32_t)require_space(o, dim);
}
void po_optim_state_init(int kind, float init_acc, float* entry, uint32_t dim) {
  OptimCfg o;
  o.kind = kind;
  o.init_acc = init_acc;
  state_initialization(o, entry, dim);
}
void po_optim_update(int kind, float lr, float wd, float mom, float eps, float b1, float b2, float b1p, float b2p,
                     float* entry, uint32_t entry_len, const float* grad, uint32_t dim) {
  OptimCfg o;
  o.kind = kind; o.lr = lr; o.wd = wd; o.mom = mom; o.eps = eps; o.b1 = b1; o.b2 = b2;
  optim_update(o, entry, entry_len, grad, dim, b1p, b2p);
}

// ---- EvictionMap (for the LRU golden test) ----
void* po_evmap_new(uint64_t cap) { return new EvictionMap(cap); }
void po_evmap_free(void* m) { delete (EvictionMap*)m; }
void po_evmap_insert(void* m, uint64_t k) {
  Entry e;
  e.sign = k;
  ((EvictionMap*)m)->insert(k, std::move(e));
}
int po_evmap_get_refresh(void* m, uint64_t k) { return ((EvictionMap*)m)->get_refresh(k) != nullptr; }
uint64_t po_evmap_len(void* m) { return ((EvictionMap*)m)->len; }

// ---- FeatureBatch dedup ----
void* po_fb_new(const uint64_t* ids, const uint32_t* row_off, uint32_t B) {
  auto* fb = new FeatureBatch();
  if (feature_batch_new(ids, row_off, B, *fb) != 0) {
    delete fb;
    return nullptr;
  }
  return fb;
}
void po_fb_free(void* p) { delete (FeatureBatch*)p; }
void po_fb_hashstack(void* p, uint32_t rounds, uint64_t size) {
  Slot s;
  s.hs_rounds = rounds;
  s.hs_size = size;
  hashstack(*(FeatureBatch*)p, s);
}
void po_fb_add_prefix(void* p, uint32_t prefix_bit, uint64_t prefix) {
  Slot s;
  s.prefix = prefix;
  add_prefix(*(FeatureBatch*)p, s, prefix_bit);
}
uint32_t po_fb_num_unique(void* p) { return (uint32_t)((FeatureBatch*)p)->signs.size(); }
uint32_t po_fb_num_occ(void* p) { return (uint32_t)((FeatureBatch*)p)->occ_sample.size(); }
void po_fb_export(void* p, uint64_t* signs, uint32_t* seg_off, uint16_t* occ_sample, uint16_t* occ_col,
                  uint32_t* sample_num_signs) {
  auto* fb = (FeatureBatch*)p;
  std::copy(fb->signs.begin(), fb->signs.end(), signs);
  std::copy(fb->seg_off.begin(), fb->seg_off.end(), seg_off);
  std::copy(fb->occ_sample.begin(), fb->occ_sample.end(), occ_sample);
  std::copy(fb->occ_col.begin(), fb->occ_col.end(), occ_col);
  std::copy(fb->sample_num_signs.begin(), fb->sample_num_signs.end(), sample_num_signs);
}

// ---- Worker + parameter servers ----
void* po_worker_new(uint32_t n_slots, uint32_t n_ps, uint64_t capacity_per_ps, uint32_t n_internal_shards,
                    uint32_t prefix_bit) {
  auto* w = new Worker();
  w->slots.resize(n_slots);
  w->prefix_bit = prefix_bit;
  for (uint32_t r = 0; r < n_ps; ++r) {
    w->ps.emplace_back(new ParamServer(capacity_per_ps, n_internal_shards));
    w->ps.back()->prefix_bit = prefix_bit;
  }
  return w;
}
void po_worker_free(void* w) { delete (Worker*)w; }
void po_worker_set_slot(void* w, uint32_t s, uint32_t dim, int summation, int sqrt_scaling, uint32_t sample_fixed_size,
                        uint32_t hs_rounds, uint64_t hs_size, uint64_t prefix) {
  Slot& sl = ((Worker*)w)->slots[s];
  sl.dim = dim; sl.summation = summation; sl.sqrt_scaling = sqrt_scaling; sl.sample_fixed_size = sample_fixed_size;
  sl.hs_rounds = hs_rounds; sl.hs_size = hs_size; sl.prefix = prefix;
}
// configure_embedding_parameter_servers (persia-core nats.rs:355-384 -> PS configure)
void po_worker_configure(void* w, float lo, float hi, float admit_p, int enable_wb, float wb) {
  for (auto& p : ((Worker*)w)->ps) {
    p->hyper.lo = lo; p->hyper.hi = hi; p->hyper.admit_p = admit_p; p->hyper.enable_wb = enable_wb; p->hyper.wb = wb;
    p->configured = true;
  }
}
// register_optimizer (PS mod.rs:429-438)
void po_worker_set_optimizer(void* w, int kind, float lr, float wd, float mom, float init_acc, float eps, float b1,
                             float b2) {
  for (auto& p : ((Worker*)w)->ps) {
    p->optim.kind = kind; p->optim.lr = lr; p->optim.wd = wd; p->optim.mom = mom; p->optim.init_acc = init_acc;
    p->optim.eps = eps; p->optim.b1 = b1; p->optim.b2 = b2;
  }
}
void po_worker_set_faithful_miss(void* w, int on) { for (auto& p : ((Worker*)w)->ps) p->faithful_miss = on; }
// set_embedding: routed by farmhash64 % R like the EW does (mod.rs:1150-1259)
void po_worker_set_embedding(void* w, const uint64_t* signs, uint64_t n, const float* entries, uint32_t dim,
                             uint32_t entry_len) {
  auto* W = (Worker*)w;
  for (uint64_t i = 0; i < n; ++i)
    W->ps[farmhash64_u64(signs[i]) % W->ps.size()]->set_entry(signs[i], entries + i * entry_len, dim, entry_len);
}
// read back entries (0 if absent); does not touch LRU order
int po_worker_get_entry(void* w, uint64_t sign, float* out, uint32_t max_len) {
  auto* W = (Worker*)w;
  ParamServer& p = *W->ps[farmhash64_u64(sign) % W->ps.size()];
  size_t si = p.shard_of(sign);
  std::lock_guard<std::mutex> g(*p.locks[si]);
  Entry* e = p.shards[si]->get(sign);
  if (!e) return 0;
  size_t n = std::min<size_t>(e->inner.size(), max_len);
  std::memcpy(out, e->inner.data(), n * 4);
  return (int)e->inner.size();
}
uint64_t po_worker_ps_len(void* w, uint32_t r) { return ((Worker*)w)->ps[r]->len(); }
uint64_t po_worker_grad_miss(void* w) {
  uint64_t t = 0;
  for (auto& p : ((Worker*)w)->ps) t += p->grad_miss.load();
  return t;
}
// direct PS request (lookup_mixed / update_gradient_mixed) on replica r
int po_ps_lookup(void* w, uint32_t r, const uint64_t* signs, const uint32_t* dims, uint64_t n, int training, float* out) {
  return ((Worker*)w)->ps[r]->lookup(signs, dims, n, training, out);
}
int po_ps_update(void* w, uint32_t r, const uint64_t* signs, const uint32_t* dims, uint64_t n, const float* grads,
                 uint64_t n_floats) {
  return ((Worker*)w)->ps[r]->update(signs, dims, n, grads, n_floats);
}

void* po_ctx_new() { return new Worker::Ctx(); }
void po_ctx_free(void* c) { delete (Worker::Ctx*)c; }
uint32_t po_ctx_num_unique(void* c, uint32_t slot) { return (uint32_t)((Worker::Ctx*)c)->fbs[slot].signs.size(); }
void po_ctx_signs(void* c, uint32_t slot, uint64_t* out) {
  auto& v = ((Worker::Ctx*)c)->fbs[slot].signs;
  std::copy(v.begin(), v.end(), out);
}

int po_worker_forward(void* w, const uint64_t* ids, const uint32_t* row_off, uint32_t B, int training, uint16_t* out,
                      void* ctx) {
  return ((Worker*)w)->forward(ids, row_off, B, training, out, (Worker::Ctx*)ctx);
}
int po_worker_backward(void* w, void* ctx, const void* grads, int is_f16, const float* scale, const int* skip,
                       int* slot_status) {
  return ((Worker*)w)->backward(*(Worker::Ctx*)ctx, grads, is_f16, scale, skip, slot_status);
}
int po_worker_forward_raw(void* w, uint32_t slot, const uint64_t* ids, const uint32_t* row_off, uint32_t B, int training,
                          uint16_t* table, int64_t* index, uint32_t* sample_id_num, uint32_t* n_distinct, void* ctx) {
  return ((Worker*)w)->forward_raw(slot, ids, row_off, B, training, table, index, sample_id_num, n_distinct,
                                   (Worker::Ctx*)ctx);
}
int po_worker_backward_raw(void* w, uint32_t slot, void* ctx, const void* grads, int is_f16, float scale, int skip,
                           int* status) {
  return ((Worker*)w)->backward_raw(slot, *(Worker::Ctx*)ctx, grads, is_f16, scale, skip, status);
}

// ---- timed CPU baseline ----
// T threads, each running forward+backward over its own pre-built batches against the shared
// parameter servers (the reference keeps several batches in flight: 10 forward / 8 backward
// workers, persia/data.py:233, persia/ctx.py:759).  ids: n_batches batches of the same shape.
// Returns wall seconds.
double po_worker_bench(void* w, const uint64_t* ids, const uint32_t* row_off, uint32_t B, uint64_t ids_per_batch,
                       uint32_t n_batches, const uint16_t* grads_f16, uint32_t n_threads) {
  auto* W = (Worker*)w;
  // keep the per-request arrays in the heap instead of fresh mmaps (page-fault storms would handicap the baseline)
  static bool tuned = (mallopt(M_MMAP_THRESHOLD, 32 << 20), mallopt(M_TRIM_THRESHOLD, 1 << 30), true);
  (void)tuned;
  size_t out_elems = 0;
  for (auto& s : W->slots) out_elems += (size_t)B * s.dim;
  std::atomic<uint32_t> next{0};
  auto t0 = std::chrono::steady_clock::now();
  std::vector<std::thread> th;
  for (uint32_t t = 0; t < n_threads; ++t)
    th.emplace_back([&]() {
      std::vector<uint16_t> out(out_elems);
      Worker::Ctx ctx;
      for (;;) {
        uint32_t b = next.fetch_add(1);
        if (b >= n_batches) break;
        W->forward(ids + (size_t)b * ids_per_batch, row_off, B, 1, out.data(), &ctx);
        W->backward(ctx, grads_f16, 1, nullptr, nullptr, nullptr);
      }
    });
  for (auto& x : th) x.join();
  return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}

}  // extern "C"
