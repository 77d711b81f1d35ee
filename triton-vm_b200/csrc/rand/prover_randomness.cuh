// The prover's randomness from its 32-byte seed (reference stark.rs:192, 293-328, 1316-1322; master_table.rs:423-434,
// 630-662, 1006-1025), as data-parallel stages over an executor `Ex`.
//
// Every array the prover draws comes from its own `StdRng::from_seed(offset_rng_seed(seed, k))` stream: main column i
// (k = i < 379, h B-field elements), aux column i (k = 379 + i, h X-field elements; the reference derives it as
// offset(offset(seed, 379), i), which is the same 256-bit little-endian sum), the batch-randomizer column 90 (k = 470, n
// X-field elements) and the quotient-segment randomizer (k = 471, (h + 1) * 5 X-field elements).  StdRng is ChaCha12 with
// a 64-bit block counter; a u64 is two consecutive keystream words, low first; a B-field element is rand's single-sample
// "Canon" widening multiply over the range [0, p - 1] (oracle/rand_compat.py restates all of it).
//
// Canon's method takes x * p for a u64 x.  If lo(x p) > 2^32 - 1 it takes a second u64 x2 and adds the carry of
// lo(x p) + hi(x2 p): two u64 per sample.  Otherwise (probability 2^-32) the sample is SHORT: one u64.  After a short
// sample every later sample of the stream starts one u64 earlier than 2j, so the stages are:
//   1. keystream: one body per (stream, 64-byte block), 2 * count u64 per stream (the most a stream can consume); the body
//      also appends every position whose u64 WOULD make a short sample to a compact flag list (almost always empty);
//   2. walk: one body per stream follows its flags in position order and records which samples really are short (a
//      flagged position is a sample start only if it has the parity the earlier shorts left);
//   3. sample: one body per output element; sample j starts at 2j - (number of short samples before j).
// Positions are exact in every case; nothing assumes a stride of 2.
//
// Executor interface (as in fill/main_fill.cuh):
//     u64 *alloc(size_t words)            memory of the executor's space, released with the executor
//     void launch(size_t count, F body)   body(i) for every i < count
//     u64 read_word(const u64 *p)         one word back to the host (synchronises)
// The library instantiates the stages with the CUDA executor of prover_randomness.cu; tests/host/prover_randomness_host.cu
// instantiates the same text with a sequential host executor (test infrastructure, not part of the library).
#pragma once
#include <cstddef>
#include <cstdint>
#include "../field.cuh"

namespace tvm {
namespace prand {

#define TVM_RAND_BODY [=] __host__ __device__

enum : unsigned { NUM_MAIN = 379, NUM_AUX = 91, STREAM_RCOL = NUM_MAIN + NUM_AUX, STREAM_QUOT = NUM_MAIN + NUM_AUX + 1,
                  NUM_STREAMS = NUM_MAIN + NUM_AUX + 2, STDRNG_ROUNDS = 12 };

struct Seed { uint32_t w[8]; };   // 32 seed bytes as little-endian words (rand_chacha's key)

TVM_HD uint32_t rotl32(uint32_t x, unsigned n) {
#ifdef __CUDA_ARCH__
  return __funnelshift_l(x, x, n);
#else
  return (x << n) | (x >> (32 - n));
#endif
}

// One ChaCha block: constants, key = 8 LE words, 64-bit block counter in words 12-13, stream id 0 in words 14-15.
TVM_HD void chacha_block(const Seed &key, uint64_t counter, unsigned rounds, uint32_t out[16]) {
  const uint32_t s[16] = {0x61707865u, 0x3320646eu, 0x79622d32u, 0x6b206574u, key.w[0], key.w[1], key.w[2], key.w[3],
                          key.w[4], key.w[5], key.w[6], key.w[7], (uint32_t)counter, (uint32_t)(counter >> 32), 0u, 0u};
  uint32_t w[16];
#pragma unroll
  for (int i = 0; i < 16; i++) w[i] = s[i];
#define TVM_CHACHA_QR(a, b, c, d)                                  \
  w[a] += w[b]; w[d] = rotl32(w[d] ^ w[a], 16);                    \
  w[c] += w[d]; w[b] = rotl32(w[b] ^ w[c], 12);                    \
  w[a] += w[b]; w[d] = rotl32(w[d] ^ w[a], 8);                     \
  w[c] += w[d]; w[b] = rotl32(w[b] ^ w[c], 7);
  for (unsigned r = 0; r < rounds; r += 2) {
    TVM_CHACHA_QR(0, 4, 8, 12) TVM_CHACHA_QR(1, 5, 9, 13) TVM_CHACHA_QR(2, 6, 10, 14) TVM_CHACHA_QR(3, 7, 11, 15)
    TVM_CHACHA_QR(0, 5, 10, 15) TVM_CHACHA_QR(1, 6, 11, 12) TVM_CHACHA_QR(2, 7, 8, 13) TVM_CHACHA_QR(3, 4, 9, 14)
  }
#undef TVM_CHACHA_QR
#pragma unroll
  for (int i = 0; i < 16; i++) out[i] = w[i] + s[i];
}

// master_table.rs:630-662 `offset_rng_seed`: the seed plus `offset` as 256-bit little-endian integers (mod 2^256)
TVM_HD Seed offset_seed(const Seed &seed, uint64_t offset) {
  Seed r;
  uint64_t carry = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    const uint64_t add = i == 0 ? (uint32_t)offset : (i == 1 ? offset >> 32 : 0);
    const uint64_t s = (uint64_t)seed.w[i] + add + carry;
    r.w[i] = (uint32_t)s;
    carry = s >> 32;
  }
  return r;
}

TVM_HD u64 mul_p_hi(u64 x) { return (u64)(((unsigned __int128)x * P) >> 64); }
TVM_HD u64 mul_p_lo(u64 x) { return x * P; }
// a sample starting at this u64 consumes only it (Canon: lo(x p) <= 2^32 - 1 = (-p) mod 2^64, no second draw)
TVM_HD bool is_short(u64 x) { return mul_p_lo(x) <= 0xFFFFFFFFull; }
// Canon's single sample of [0, p - 1], reduced like BFieldElement::new; `x2` is read only if the sample is not short
TVM_HD u64 canon_sample(u64 x, const u64 *x2) {
  u64 r = mul_p_hi(x);
  const u64 lo = mul_p_lo(x);
  if (lo > 0xFFFFFFFFull) {
    const u64 hi2 = mul_p_hi(*x2);
    if (lo + hi2 < lo) r++;
  }
  return r >= P ? r - P : r;
}

// ---- layout: up to four groups of equally long streams, outputs concatenated in group order --------------------------
struct Group {
  u64 streams;      // streams in the group
  u64 count;        // B-field samples per stream (an X-field element is 3 consecutive samples)
  u64 seed_offset;  // offset_rng_seed offset of the group's first stream
  u64 blocks;       // 64-byte keystream blocks per stream: ceil(2 count / 8)
  u64 block0;       // first block of the group in the keystream buffer (a stream's u64 k is at 8 * its first block + k)
  u64 out0;         // first output word of the group
  u64 stream0;      // global index of the group's first stream
};
struct Layout {
  Group g[4];
  unsigned ngroups;
  u64 total_blocks, total_out, total_streams;
};

inline void layout_add(Layout &L, u64 streams, u64 count, u64 seed_offset) {
  Group &g = L.g[L.ngroups++];
  g.streams = streams; g.count = count; g.seed_offset = seed_offset;
  g.blocks = (2 * count + 7) / 8;
  g.block0 = L.total_blocks; g.out0 = L.total_out; g.stream0 = L.total_streams;
  L.total_blocks += streams * g.blocks; L.total_out += streams * count; L.total_streams += streams;
}
// the prover's four arrays (reference_prover.randomness): main [379][h], aux [91][h][3], column 90 [n][3], quotient [nq][3]
inline Layout prover_layout(u64 n, u64 h, u64 nq) {
  Layout L{};
  layout_add(L, NUM_MAIN, h, 0);
  layout_add(L, NUM_AUX, 3 * h, NUM_MAIN);
  layout_add(L, 1, 3 * n, STREAM_RCOL);
  layout_add(L, 1, 3 * nq, STREAM_QUOT);
  return L;
}
inline Layout single_stream_layout(u64 count) {   // one stream of `count` samples drawn from the seed itself
  Layout L{};
  layout_add(L, 1, count, 0);
  return L;
}

struct Where { unsigned g; u64 s; u64 k; };   // group, stream within it, index within the stream
TVM_HD Where by_block(const Layout &L, u64 b) {
  for (unsigned g = 0; g + 1 < L.ngroups; g++)
    if (b < L.g[g + 1].block0) { const u64 r = b - L.g[g].block0; return {g, r / L.g[g].blocks, r % L.g[g].blocks}; }
  const Group &G = L.g[L.ngroups - 1];
  const u64 r = b - G.block0;
  return {L.ngroups - 1, r / G.blocks, r % G.blocks};
}
TVM_HD Where by_output(const Layout &L, u64 i) {
  for (unsigned g = 0; g + 1 < L.ngroups; g++)
    if (i < L.g[g + 1].out0) { const u64 r = i - L.g[g].out0; return {g, r / L.g[g].count, r % L.g[g].count}; }
  const Group &G = L.g[L.ngroups - 1];
  const u64 r = i - G.out0;
  return {L.ngroups - 1, r / G.count, r % G.count};
}
TVM_HD Where by_stream(const Layout &L, u64 gs) {
  for (unsigned g = 0; g + 1 < L.ngroups; g++)
    if (gs < L.g[g + 1].stream0) return {g, gs - L.g[g].stream0, 0};
  return {L.ngroups - 1, gs - L.g[L.ngroups - 1].stream0, 0};
}

TVM_HD u64 fetch_add(u64 *p, u64 v) {
#ifdef __CUDA_ARCH__
  return atomicAdd((unsigned long long *)p, (unsigned long long)v);
#else
  const u64 o = *p;   // the host executor runs bodies sequentially
  *p += v;
  return o;
#endif
}

// Flag list: flags[0] = number of flagged positions (may exceed `cap`), then `cap` pairs (global stream, position).
TVM_HD void flag_if_short(u64 *flags, u64 cap, u64 stream, u64 k, u64 x) {
  if (!is_short(x)) return;
  const u64 slot = fetch_add(flags, 1);
  if (slot < cap) { flags[1 + 2 * slot] = stream; flags[2 + 2 * slot] = k; }
}

// ---- stages ----------------------------------------------------------------------------------------------------------
// 1. keystream of every stream (`ks`: 8 * L.total_blocks words) and its flags
template <class Ex>
void keystream(Ex &ex, const Layout &L, const Seed &seed, u64 *ks, u64 *flags, u64 cap) {
  ex.launch(L.total_blocks, TVM_RAND_BODY(size_t b) {
    const Where w = by_block(L, b);
    const Group &G = L.g[w.g];
    uint32_t o[16];
    chacha_block(offset_seed(seed, G.seed_offset + w.s), w.k, STDRNG_ROUNDS, o);
    const u64 limit = 2 * G.count;   // u64 beyond it pad the last block and are never read
#pragma unroll
    for (int t = 0; t < 8; t++) {
      const u64 x = (u64)o[2 * t] | ((u64)o[2 * t + 1] << 32);
      ks[8 * b + t] = x;
      if (8 * w.k + t < limit) flag_if_short(flags, cap, G.stream0 + w.s, 8 * w.k + t, x);
    }
  });
}

// 1'. flags of a given keystream (flag capacity exceeded in stage 1, or a keystream supplied by a test)
template <class Ex>
void flag_keystream(Ex &ex, const Layout &L, const u64 *ks, u64 *flags, u64 cap) {
  ex.launch(8 * L.total_blocks, TVM_RAND_BODY(size_t i) {
    const Where w = by_block(L, i / 8);
    const Group &G = L.g[w.g];
    const u64 k = 8 * w.k + i % 8;
    if (k < 2 * G.count) flag_if_short(flags, cap, G.stream0 + w.s, k, ks[i]);
  });
}

// 2. per stream: the short samples in increasing order -> shorts[tab[2s] ..][tab[2s + 1]]
template <class Ex>
void walk(Ex &ex, const Layout &L, const u64 *flags, u64 *shorts, u64 *tab) {
  ex.launch(L.total_streams, TVM_RAND_BODY(size_t gs) {
    const u64 nf = flags[0];
    const Group &G = L.g[by_stream(L, gs).g];
    u64 off = 0;
    for (u64 f = 0; f < nf; f++) off += flags[1 + 2 * f] < gs;
    u64 len = 0, last = 0;
    bool any = false;
    for (;;) {   // next flagged position of this stream (the list is unordered and almost always empty)
      u64 pos = ~(u64)0;
      for (u64 f = 0; f < nf; f++) {
        const u64 k = flags[2 + 2 * f];
        if (flags[1 + 2 * f] == gs && (!any || k > last) && k < pos) pos = k;
      }
      if (pos == ~(u64)0) break;
      any = true;
      last = pos;
      if ((pos + len) & 1) continue;   // sample j starts at 2j - len: an odd sum is the second u64 of a sample
      const u64 j = (pos + len) / 2;
      if (j >= G.count) break;
      shorts[off + len++] = j;
    }
    tab[2 * gs] = off;
    tab[2 * gs + 1] = len;
  });
}

// 3. every sample, canonical, into out[L.total_out]
template <class Ex>
void sample(Ex &ex, const Layout &L, const u64 *ks, const u64 *shorts, const u64 *tab, u64 *out) {
  ex.launch(L.total_out, TVM_RAND_BODY(size_t i) {
    const Where w = by_output(L, i);
    const Group &G = L.g[w.g];
    const u64 gs = G.stream0 + w.s, j = w.k;
    const u64 *sh = shorts + tab[2 * gs];
    u64 lo = 0, hi = tab[2 * gs + 1];   // number of short samples before j
    while (lo < hi) {
      const u64 mid = (lo + hi) / 2;
      if (sh[mid] < j) lo = mid + 1; else hi = mid;
    }
    const u64 *x = ks + 8 * (G.block0 + w.s * G.blocks) + 2 * j - lo;
    out[i] = canon_sample(x[0], x + 1);
  });
}

// flags -> short-sample table -> samples; `flags` holds the result of stage 1 with capacity `cap`
template <class Ex>
void finish(Ex &ex, const Layout &L, const u64 *ks, u64 *flags, u64 cap, u64 *out) {
  u64 nf = ex.read_word(flags);
  if (nf > cap) {                      // more flags than room (never seen at 2^-32 per position, but exact regardless)
    cap = nf;
    flags = ex.alloc(1 + 2 * cap);
    ex.launch(1, TVM_RAND_BODY(size_t) { flags[0] = 0; });
    flag_keystream(ex, L, ks, flags, cap);
    nf = ex.read_word(flags);
  }
  u64 *shorts = ex.alloc(nf ? nf : 1), *tab = ex.alloc(2 * L.total_streams);
  walk(ex, L, flags, shorts, tab);
  sample(ex, L, ks, shorts, tab, out);
}

static constexpr u64 FLAG_CAPACITY = 1024;

// every stream of `L` from `seed` -> out[L.total_out], canonical
template <class Ex>
void generate(Ex &ex, const Layout &L, const Seed &seed, u64 *out) {
  u64 *ks = ex.alloc(8 * L.total_blocks), *flags = ex.alloc(1 + 2 * FLAG_CAPACITY);
  ex.launch(1, TVM_RAND_BODY(size_t) { flags[0] = 0; });
  keystream(ex, L, seed, ks, flags, FLAG_CAPACITY);
  finish(ex, L, ks, flags, FLAG_CAPACITY, out);
}

}  // namespace prand
}  // namespace tvm
