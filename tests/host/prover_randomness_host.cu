// TEST INFRASTRUCTURE — not part of the library.
// The sampler stages of triton-vm_b200/csrc/rand/prover_randomness.cuh instantiated with a sequential host executor, so that
// `pytest -m "not gpu"` can check them (ChaCha12, offset_rng_seed, Canon's sampling, the short-sample walk) against the
// oracle on a machine without a GPU, plus the multi-threaded search of tests/golden/make_short_draw_seed.py.  The library
// (csrc/prover_randomness.cu) instantiates the same header with the CUDA executor only; nothing here is linked into it.
// Build: nvcc -O3 -std=c++17 --extended-lambda -shared -Xcompiler -fPIC tests/host/prover_randomness_host.cu -o tests/host/_build/libprover_randomness_host.so
#include <atomic>
#include <cstring>
#include <memory>
#include <thread>
#include <vector>
#include "../../triton-vm_b200/csrc/rand/prover_randomness.cuh"

using namespace tvm;

namespace {

struct HostExec {
  std::vector<std::unique_ptr<u64[]>> mem;
  size_t launches = 0;
  u64 *alloc(size_t words) {
    mem.emplace_back(new u64[words ? words : 1]);
    std::memset(mem.back().get(), 0xA5, (words ? words : 1) * 8);   // uninitialised reads show up as garbage
    return mem.back().get();
  }
  template <class F>
  void launch(size_t count, F f) {
    launches++;
    for (size_t i = 0; i < count; i++) f(i);
  }
  u64 read_word(const u64 *p) { return *p; }
};

prand::Seed seed_of(const uint8_t *b) {
  prand::Seed s;
  for (int i = 0; i < 8; i++) s.w[i] = (uint32_t)b[4 * i] | ((uint32_t)b[4 * i + 1] << 8) | ((uint32_t)b[4 * i + 2] << 16) | ((uint32_t)b[4 * i + 3] << 24);
  return s;
}

}  // namespace

extern "C" {

void prand_host_chacha_block(const uint32_t key[8], uint64_t counter, unsigned rounds, uint32_t out[16]) {
  prand::Seed k;
  for (int i = 0; i < 8; i++) k.w[i] = key[i];
  prand::chacha_block(k, counter, rounds, out);
}

void prand_host_offset_seed(const uint8_t seed[32], uint64_t offset, uint8_t out[32]) {
  const prand::Seed r = prand::offset_seed(seed_of(seed), offset);
  for (int i = 0; i < 32; i++) out[i] = (uint8_t)(r.w[i / 4] >> (8 * (i % 4)));
}

// `count` B-field draws of StdRng::from_seed(seed); stats (optional) [2]: flagged positions, short samples
int prand_host_stream(const uint8_t seed[32], uint64_t count, uint64_t *out, uint64_t *stats) {
  HostExec ex;
  const prand::Layout L = prand::single_stream_layout(count);
  u64 *ks = ex.alloc(8 * L.total_blocks), *flags = ex.alloc(1 + 2 * prand::FLAG_CAPACITY);
  flags[0] = 0;
  prand::keystream(ex, L, seed_of(seed), ks, flags, prand::FLAG_CAPACITY);
  const u64 nf = flags[0];
  prand::finish(ex, L, ks, flags, prand::FLAG_CAPACITY, out);
  if (stats) {
    stats[0] = nf;
    stats[1] = 0;
    for (u64 j = 0, k = 0; j < count; j++) {   // sequential walk, as StdRng consumes the stream
      const bool s = prand::is_short(ks[k]);
      stats[1] += s;
      k += s ? 1 : 2;
    }
  }
  return 0;
}

// `count` samples of a given u64 stream words[2 * count] (the first `count` of them that Canon reads);
// `cap` = flag capacity (a small one exercises the overflow path)
int prand_host_words(const uint64_t *words, uint64_t count, uint64_t cap, uint64_t *out) {
  HostExec ex;
  const prand::Layout L = prand::single_stream_layout(count);
  u64 *ks = ex.alloc(8 * L.total_blocks), *flags = ex.alloc(1 + 2 * cap);
  for (u64 k = 0; k < 8 * L.total_blocks; k++) ks[k] = k < 2 * count ? words[k] : 0;
  flags[0] = 0;
  prand::flag_keystream(ex, L, ks, flags, cap);
  prand::finish(ex, L, ks, flags, cap, out);
  return 0;
}

// the prover's four arrays, concatenated: main [379][h], aux [91][h][3], column 90 [n][3], quotient [nq][3]
int prand_host_randomness(const uint8_t seed[32], uint64_t n, uint64_t h, uint64_t nq, uint64_t *out) {
  HostExec ex;
  prand::generate(ex, prand::prover_layout(n, h, nq), seed_of(seed), out);
  return 0;
}

// Searches seeds `prefix[0..24) ++ le64(i)`, first <= i < first + count, on `threads` threads, for one whose StdRng stream
// has a short sample among its first `samples`; returns 1 and the smallest such i and its sample index, else 0.
int prand_host_search(const uint8_t prefix[24], uint64_t first, uint64_t count, unsigned samples, unsigned threads, uint64_t *found_i,
                      uint64_t *found_sample) {
  std::atomic<uint64_t> best{~(uint64_t)0};
  std::vector<uint64_t> best_sample(threads ? threads : 1, 0), best_i(threads ? threads : 1, ~(uint64_t)0);
  const unsigned T = threads ? threads : 1;
  auto work = [&](unsigned t) {
    uint8_t bytes[32];
    std::memcpy(bytes, prefix, 24);
    for (uint64_t i = first + t; i < first + count; i += T) {
      if (i > best.load(std::memory_order_relaxed)) return;
      for (int b = 0; b < 8; b++) bytes[24 + b] = (uint8_t)(i >> (8 * b));
      const prand::Seed s = seed_of(bytes);
      uint32_t blk[16];
      uint64_t have = ~(uint64_t)0;   // block held in blk
      uint64_t pos = 0;
      for (unsigned j = 0; j < samples; j++) {
        if (pos / 8 != have) { have = pos / 8; prand::chacha_block(s, have, prand::STDRNG_ROUNDS, blk); }
        const unsigned o = 2 * (pos % 8);
        const u64 x = (u64)blk[o] | ((u64)blk[o + 1] << 32);
        if (prand::is_short(x)) {
          best_i[t] = i; best_sample[t] = j;
          uint64_t cur = best.load();
          while (i < cur && !best.compare_exchange_weak(cur, i)) {}
          return;
        }
        pos += 2;
      }
    }
  };
  std::vector<std::thread> pool;
  for (unsigned t = 0; t < T; t++) pool.emplace_back(work, t);
  for (auto &th : pool) th.join();
  const uint64_t b = best.load();
  if (b == ~(uint64_t)0) return 0;
  for (unsigned t = 0; t < T; t++)
    if (best_i[t] == b) { *found_i = b; *found_sample = best_sample[t]; }
  return 1;
}

}  // extern "C"
