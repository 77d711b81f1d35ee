// TEST INFRASTRUCTURE — not part of the library.
// The AIR checker's generated chunk bodies (triton-vm_b200/csrc/air_check_gen/air_check_bodies.cuh) run by a sequential host
// recorder, so that `pytest -m "not gpu"` can compare them with the oracle's check on a machine without a GPU.  The library
// (csrc/air_check.cu) runs the same bodies in its CUDA kernels only; nothing here is linked into libtvm_b200.so.
// Build: nvcc -O1 -std=c++17 --expt-relaxed-constexpr -shared -Xcompiler -fPIC tests/host/air_check_host.cu -o tests/host/_build/libair_check_host.so
#include <cstdint>
#include <vector>
#include "../../triton-vm_b200/csrc/air_check_gen/air_check_bodies.cuh"

using namespace tvm;

namespace {
typedef void (*HostBody)(const u64 *, const u64 *, const u64 *, const u64 *, const AirCheckStrides, const u64 *, AirCheckHostRecorder &);
struct Chunk {
  HostBody body;
  int category;
};
#define TVM_AIR_CHECK_TU(tu)
#define TVM_AIR_CHECK_CHUNK(body, cat, first, count) \
  void host_##body(const u64 *mc, const u64 *mn, const u64 *ac, const u64 *an, const AirCheckStrides a, const u64 *ch, AirCheckHostRecorder &r) { \
    body(mc, mn, ac, an, a, ch, r);                                                                                                                 \
  }
#include "../../triton-vm_b200/csrc/air_check_gen/air_check_meta.inc"
#undef TVM_AIR_CHECK_CHUNK
#define TVM_AIR_CHECK_CHUNK(body, cat, first, count) {host_##body, cat},
const Chunk CHUNKS[] = {
#include "../../triton-vm_b200/csrc/air_check_gen/air_check_meta.inc"
};
}  // namespace

extern "C" {

// main [379][n], aux [91][n][3], challenges [63][3], all canonical; counts / first / last [604] as tvm_air_check returns them
void air_check_host(const uint64_t *main, const uint64_t *aux, size_t n, const uint64_t *challenges, uint64_t *counts, uint64_t *first,
                    uint64_t *last) {
  std::vector<u64> m(379 * n), x(270 * n), ch(189);
  for (size_t i = 0; i < m.size(); i++) m[i] = to_mont(main[i]);
  for (size_t q = 0; q < 90; q++)
    for (size_t r = 0; r < n; r++)
      for (size_t d = 0; d < 3; d++) x[(3 * q + d) * n + r] = to_mont(aux[(q * n + r) * 3 + d]);
  for (size_t i = 0; i < 189; i++) ch[i] = to_mont(challenges[i]);
  for (size_t j = 0; j < 604; j++) { counts[j] = 0; first[j] = UINT64_MAX; last[j] = UINT64_MAX; }
  const AirCheckStrides st{n, n};
  for (const Chunk &c : CHUNKS) {
    const size_t lo = c.category == 3 ? n - 1 : 0;
    const size_t hi = c.category == 0 ? 1 : c.category == 2 ? n - 1 : n;
    for (size_t r = lo; r < hi; r++) {
      AirCheckHostRecorder rec{counts, first, last, r};
      const size_t nx = r + 1 < n ? r + 1 : r;
      c.body(m.data() + r, m.data() + nx, x.data() + r, x.data() + nx, st, ch.data(), rec);
    }
  }
}

}  // extern "C"
