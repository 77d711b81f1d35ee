// The three Hash-table traces of the AlgebraicExecutionTrace (aet.rs:67-76: program hash, sponge, hash) expanded from the
// permutation inputs the VM records (csrc/vm.cu), as one data-parallel stage over an executor `Ex` (the interface of
// fill/main_fill.cuh; only `launch` is used).  Each record is the 16-word state a Tip5 permutation starts from; the stage
// recomputes its five rounds and writes one row per state it passes through (Tip5::trace: before round 0 .. after round 4),
// or the single zero-state row of a `sponge_init` record, in `tvm_aet`'s row layout: hash.rs:60-70 `trace_row_to_table_row`
// plus CI (aet.rs:203-205, 264-297), Mode left 0.
//
// The library instantiates it with the CUDA executor of main_fill.cu (one thread per permutation); tests/host/
// hash_trace_host.cu instantiates the same text with a sequential host executor.
#pragma once
#include <cstddef>
#include <vector>
#include "../tip5.cuh"
#include "main_fill.cuh"

namespace tvm {
namespace hash_trace {

// one u64 of metadata per record: the row it starts at in its section's array, its CI, its section, single-row flag
enum : unsigned { SECTION_PROGRAM_HASH = 0, SECTION_SPONGE = 1, SECTION_HASH = 2 };
static constexpr unsigned META_ROW_BITS = 48;
TVM_HD u64 meta_encode(u64 row, unsigned ci, unsigned section, bool single_row) {
  return row | ((u64)ci << META_ROW_BITS) | ((u64)section << 56) | ((u64)single_row << 58);
}
TVM_HD u64 meta_row(u64 m) { return m & ((1ULL << META_ROW_BITS) - 1); }
TVM_HD unsigned meta_ci(u64 m) { return (unsigned)(m >> META_ROW_BITS) & 0xFF; }
TVM_HD unsigned meta_section(u64 m) { return (unsigned)(m >> 56) & 3; }
TVM_HD bool meta_single_row(u64 m) { return (m >> 58) & 1; }

// HashMainColumn order (triton-air/src/table/hash.rs; airgen/columns.py prints the same names)
enum : unsigned {
  H_MODE = 0, H_CI = 1, H_ROUND = 2, H_LK_IN = 3, H_LK_OUT = 19, H_STATE4 = 35, H_INV = 47, H_CONST = 51, H_WIDTH = 67,
  // constant block: round constants (Montgomery), round constants (canonical), the 8-bit lookup table
  K_RC_MONT = 0, K_RC_CANON = 80, K_LUT = 160, K_WORDS = 160 + 256
};

inline std::vector<u64> constants(const u64 *rc_mont, const unsigned char *lut) {
  std::vector<u64> k(K_WORDS);
  for (unsigned i = 0; i < 80; i++) { k[K_RC_MONT + i] = rc_mont[i]; k[K_RC_CANON + i] = from_mont(rc_mont[i]); }
  for (unsigned i = 0; i < 256; i++) k[K_LUT + i] = lut[i];
  return k;
}

struct Lut { const u64 *t; TVM_HD unsigned operator()(unsigned i) const { return (unsigned)t[i]; } };
struct Rc { const u64 *t; TVM_HD u64 operator()(int i) const { return t[i]; } };

// one row of the trace: `s` the Montgomery state after `rnd` rounds (hash.rs:60-70)
TVM_HD void write_row(u64 *row, const u64 (&s)[16], unsigned rnd, unsigned ci, const u64 *k) {
  row[H_MODE] = 0;
  row[H_CI] = ci;
  row[H_ROUND] = rnd;
  for (unsigned e = 0; e < 4; e++) {
    const u64 x = s[e];                              // 16-bit limbs of the Montgomery representation (hash.rs:30-33)
    for (unsigned l = 0; l < 4; l++) {
      const unsigned limb = (unsigned)(x >> (16 * l)) & 0xFFFF, col = 4 * e + 3 - l;   // columns run Highest .. Lowest
      row[H_LK_IN + col] = limb;
      row[H_LK_OUT + col] = (k[K_LUT + (limb >> 8)] << 8) | k[K_LUT + (limb & 0xFF)];  // cascade.rs:29-35
    }
    row[H_INV + e] = fill::inv_or_zero_canon(0xFFFFFFFFULL - (x >> 32));   // inverse_or_zero_of_highest_2_limbs
  }
  for (unsigned e = 4; e < 16; e++) row[H_STATE4 + e - 4] = from_mont(s[e]);
  for (unsigned j = 0; j < 16; j++) row[H_CONST + j] = rnd < TIP5_ROUNDS ? k[K_RC_CANON + 16 * rnd + j] : 0;
}

// states [count][16] Montgomery, meta [count]; out_*: [rows][67] canonical, the sections' arrays
template <class Ex>
void expand(Ex &ex, const u64 *states, const u64 *meta, size_t count, const u64 *k, u64 *out_program_hash, u64 *out_sponge,
            u64 *out_hash) {
  ex.launch(count, TVM_FILL_BODY(size_t i) {
    u64 s[16];
    for (int j = 0; j < 16; j++) s[j] = states[16 * i + j];
    const u64 m = meta[i];
    const unsigned section = meta_section(m), ci = meta_ci(m);
    u64 *row = (section == SECTION_PROGRAM_HASH ? out_program_hash : section == SECTION_SPONGE ? out_sponge : out_hash) +
               meta_row(m) * H_WIDTH;
    if (meta_single_row(m)) {
      write_row(row, s, 0, ci, k);
      return;
    }
    for (unsigned rnd = 0; rnd <= TIP5_ROUNDS; rnd++) {
      write_row(row + rnd * H_WIDTH, s, rnd, ci, k);
      if (rnd < TIP5_ROUNDS) tip5_round_generic(s, (int)rnd, Lut{k + K_LUT}, Rc{k + K_RC_MONT});
    }
  });
}

}  // namespace hash_trace
}  // namespace tvm
