// TEST INFRASTRUCTURE — not part of the library.
// The hash-trace expansion of triton-vm_b200/csrc/fill/hash_trace.cuh instantiated with a sequential host executor, so that
// `pytest -m "not gpu"` can check it against the oracle's three hash traces on a machine without a GPU.  The library itself
// (csrc/main_fill.cu) instantiates the same header with the CUDA executor only; nothing here is linked into libtvm_b200.so.
// Build: nvcc -O2 -std=c++17 --extended-lambda --expt-relaxed-constexpr -shared -Xcompiler -fPIC tests/host/hash_trace_host.cu -o tests/host/_build/libhash_trace_host.so
#include <cstring>
#include <vector>
#include "../../triton-vm_b200/csrc/fill/hash_trace.cuh"
#include "../../triton-vm_b200/csrc/tip5_constants.inc"

using namespace tvm;

namespace {
struct HostExec {
  template <class F>
  void launch(size_t count, F f) {
    for (size_t i = 0; i < count; i++) f(i);
  }
};
}  // namespace

extern "C" {

// states [count][16] canonical permutation inputs in execution order; section[k] 0 = program hash, 1 = sponge, 2 = hash;
// ci[k] the record's instruction; single_row[k] != 0 for a `sponge_init` row.  rows_out [3]: the sections' row counts (pass
// NULL outputs first to size them); out_*: [rows][67] canonical
void hash_trace_host_expand(const uint64_t *states, const uint32_t *section, const uint32_t *ci, const uint32_t *single_row, size_t count,
                            uint64_t *rows_out, uint64_t *out_program_hash, uint64_t *out_sponge, uint64_t *out_hash) {
  std::vector<u64> mont(16 * count), meta(count);
  uint64_t rows[3] = {0, 0, 0};
  for (size_t k = 0; k < count; k++) {
    for (int j = 0; j < 16; j++) mont[16 * k + j] = to_mont(states[16 * k + j]);
    meta[k] = hash_trace::meta_encode(rows[section[k]], ci[k], section[k], single_row[k] != 0);
    rows[section[k]] += single_row[k] ? 1 : 6;
  }
  std::memcpy(rows_out, rows, sizeof rows);
  if (!out_program_hash || !out_sponge || !out_hash) return;
  static const u64 rc_mont[80] = {TVM_TIP5_RC_MONT};
  static const unsigned char lut[256] = {TVM_TIP5_LUT};
  const std::vector<u64> k = hash_trace::constants(rc_mont, lut);
  HostExec ex;
  hash_trace::expand(ex, mont.data(), meta.data(), count, k.data(), out_program_hash, out_sponge, out_hash);
}

}  // extern "C"
