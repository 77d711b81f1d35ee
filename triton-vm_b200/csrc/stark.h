// Prover-level declarations shared by prover.cu, stark_kernels.cu and the C ABI.
#pragma once
#include <cstring>
#include <string>
#include <vector>
#include "ctx.h"

namespace tvm {

static constexpr int NUM_QUOTIENT_SEGMENTS = 4;              // stark.rs:66 (= air::TARGET_DEGREE)
static constexpr int NUM_RANDOMIZED_QUOTIENT_SEGMENTS = 5;   // stark.rs:75

struct StarkParams {          // stark.rs:113-145 (proven regime)
  unsigned security_level;
  unsigned log2_expansion;
  unsigned ldt_choice;        // 0 = heuristic (stark.rs:1942-1957), 1 = FRI, 2 = STIR
  unsigned soundness;         // 0 = ProximityRegime::Proven (default), 1 = ::Conjectured
};
inline StarkParams stark_params(const tvm_params &p) {
  return StarkParams{p.security_level, p.log2_ldt_expansion_factor, p.ldt_choice, p.soundness};
}
static constexpr int STIR_MAX_ROUNDS = 16;
static constexpr unsigned STIR_LOG2_FOLDING_FACTOR = 2;      // stark.rs:2023
struct StirDerived {          // stir.rs:112-147
  size_t folding_factor;
  int num_rounds;
  size_t in_domain[STIR_MAX_ROUNDS], out_of_domain[STIR_MAX_ROUNDS];
  size_t final_num_in_domain_queries, final_degree;
};
struct FriDerived {           // FriParameters::try_into_fri + Fri::{max_degree, num_rounds, last_round_max_degree} (fri.rs:799-924)
  size_t domain_len;
  u64 domain_offset;          // canonical: BFieldElement::generator()
  size_t expansion_factor, max_degree, num_collinearity_checks, num_rounds, last_round_max_degree;
};
struct StarkDerived {
  size_t padded_height, num_trace_randomizers, randomized_trace_len, trace_len, quotient_len, ldt_len;
  u64 ldt_offset;  // canonical
  size_t num_quotient_randomizer_coefficients;
  int ldt;                    // 1 = FRI, 2 = STIR
  size_t num_first_round_queries;
  FriDerived fri;             // derived for the final domain whichever low-degree test runs (tvm_derive_domains reports it)
  StirDerived stir;
};
// the Reed-Solomon code's proximity parameter δ of the regime (low_degree_test/mod.rs:243-320)
double rs_proximity_parameter(unsigned log2_expansion, bool conjectured);
// TVM_OK or TVM_ERR_LDT_PARAMS; `error` (optional) receives the name of the LdtParameterError variant
int stir_derive(unsigned security_level, unsigned log2_folding_factor, unsigned log2_initial_expansion, unsigned log2_high_degree_bound,
                bool conjectured, StirDerived &out, const char **error = nullptr);
// TVM_OK or TVM_ERR_LDT_PARAMS; `error` (optional) receives the name of the LdtParameterError variant
int fri_derive(unsigned security_level, bool conjectured, unsigned log2_initial_expansion, unsigned log2_high_degree_bound, FriDerived &out,
               const char **error = nullptr);
int stark_derive(const StarkParams &sp, size_t padded_height, StarkDerived &d);

struct ClaimView {            // proof.rs:68-88, canonical words
  const u64 *program_digest;  // 5
  unsigned version;
  const u64 *input; size_t num_input;
  const u64 *output; size_t num_output;
};
inline ClaimView claim_view(const tvm_claim &c) { return {c.program_digest, c.version, c.input, c.num_input, c.output, c.num_output}; }
// proof.rs:68-88: a claim's words are field elements; NULL with a non-zero count or a word >= p is an argument error (a
// non-canonical word would otherwise alias the claim [x] with [x + p] in the transcript)
inline bool claim_ok(const tvm_claim *c) {
  if ((c->num_input && !c->input) || (c->num_output && !c->output)) return false;
  for (int i = 0; i < 5; i++) if (c->program_digest[i] >= P) return false;
  for (size_t i = 0; i < c->num_input; i++) if (c->input[i] >= P) return false;
  for (size_t i = 0; i < c->num_output; i++) if (c->output[i] >= P) return false;
  return true;
}
// `text` into the caller's failure buffer of `capacity` bytes, truncated and NUL-terminated (nothing without a buffer)
inline void set_failure(char *failure, size_t capacity, const char *text) {
  if (!failure || !capacity) return;
  const size_t n = strnlen(text, capacity - 1);
  memcpy(failure, text, n);
  failure[n] = 0;
}
// Challenges::new (challenges.rs:88-135): appends the 4 challenges derived from the claim and the lookup table to the 59
// sampled ones (Montgomery form), which gives the 63 in the order the AIR reads them
void challenges_derive(const ClaimView &claim, std::vector<xfe> &ch);
// Given the 63 challenges (canonical), provides aux_trace [91][n][3] and aux_rand [91][h][3] (canonical).
// The callee sets *aux_trace / *aux_rand to its own (ideally pinned) buffers, which must stay valid
// until prove returns (zero copy: the library reads them straight into the H2D transfer).
typedef int (*AuxCallback)(void *user, const u64 *challenges, u64 **aux_trace, u64 **aux_rand);

struct ProveTimings {
  std::vector<std::pair<std::string, float>> stages;   // device ms per stage, reference profiler labels
  bool low_memory = false;                             // the last prove() ran in low-memory (just-in-time LDE) mode
};

// Where a prove's witness comes from.  Every array is canonical, in host or device memory.
// Without an aux callback the table stages run on the device ("device-table mode", tvm_prove_tables): MasterMainTable::extend
// (master_table.rs:1006-1075) runs inside the prove on the resident main trace; optionally the 230 degree-lowering main
// columns (fill_derived_main_columns, substitutions.rs:128-161) are computed on the device too and never uploaded.
struct ProveInputs {
  const u64 *main_trace = nullptr;          // [379][n]; only columns 0..148 are read with fill_derived_main
  const tvm_aet *aet = nullptr;             // device-table mode: the nine tables' columns come from the AET (main_fill.cu), no main trace is read
  bool fill_derived_main = false;           // device-table mode: columns 149..378 of the main trace are computed, not read
  AuxCallback aux_cb = nullptr;             // the caller extends the table; nullptr = device-table mode
  void *aux_user = nullptr;
  const u64 *main_rand = nullptr;           // [379][h]
  const u64 *aux_rand = nullptr;            // device-table mode: [91][h][3] (the callback hands back its own)
  const u64 *randomizer_column = nullptr;   // device-table mode: [n][3] aux column 90 (master_table.rs:1019-1025); nullptr = zeros
  const u64 *quot_rand = nullptr;           // [nq][3]
  const struct ExternalTranscript *ext = nullptr;   // the caller keeps the Fiat-Shamir transcript (tvm_prove_transcript)
};

void stark_prove(Ctx &c, const StarkParams &sp, const ClaimView &claim, size_t padded_height, const ProveInputs &in,
                 std::vector<u64> &proof, ProveTimings *timings);

// ---- main_fill.cu: MasterMainTable::new + pad from the AET; d_table [>= 149][n] receives CANONICAL columns ----
void main_fill_run(Ctx &c, struct DevMem &mem, const tvm_aet &aet, size_t n, u64 *d_table, uint64_t *lengths9);
// the witness's main trace from the AET: d_main [379][n] Montgomery (the fill's scratch is released before it returns);
// lengths9 (optional, host) receives the nine tables' lengths
void main_table_on_device(Ctx &c, u64 *d_main, size_t n, const tvm_aet &aet, uint64_t *lengths9 = nullptr);
// MasterMainTable::extend on the device: d_main [379][n] and d_ch [63*3] Montgomery (device) -> d_aux planes [273][n]
// Montgomery.  The planes of column 90 receive randomizer_column ([n][3] canonical, host or device), or zeros without it.
// The scratch comes from `mem` and goes back to it before this returns.
void aux_extend_on_device(Ctx &c, struct DevMem &mem, const u64 *d_main, size_t n, const u64 *d_ch, const u64 *randomizer_column,
                          u64 *d_aux);
void bezout_run(Ctx &c, struct DevMem &mem, const u64 *d_roots_mont, size_t m, u64 *d_a, u64 *d_b);
// the three hash traces of an execution (fill/hash_trace.cuh) into device memory of `mem`: d_out[section] [rows][67] canonical
void hash_trace_run(Ctx &c, struct DevMem &mem, const tvm_execution &ex, u64 *d_out[3]);

// ---- air_check.cu: every AIR constraint on the rows where it must vanish (check_constraints_fn!, stark.rs:2899-3015) ----
// main [379][n] and aux [91][n][3] canonical, host or device memory -> Montgomery device copies in `mem`: main [379][n] and
// the aux planes [270][n] (column 90 is read by no constraint).  A word >= p is an ApiError naming its column and row.
void air_check_upload(Ctx &c, struct DevMem &mem, const u64 *main, const u64 *aux, size_t n, u64 **d_main, u64 **d_aux);
// d_main [379][n], d_aux planes [>= 270][n] (Montgomery, device); ch_mont the 63 challenges (host, Montgomery X-field).
// counts / first / last [604] (host): violating rows per constraint; first = last = UINT64_MAX when there are none.
void air_check_run(Ctx &c, struct DevMem &mem, const u64 *d_main, const u64 *d_aux, size_t n, const u64 *ch_mont, uint64_t *counts,
                   uint64_t *first, uint64_t *last, uint64_t *num_violated);

// ---- prover_randomness.cu: the prover's four randomness arrays from its 32-byte seed, CANONICAL, concatenated ----
struct ProverRandomnessLayout {   // word offsets into the concatenation, and its length
  size_t main, aux, randomizer_column, quot, total;   // [379][h], [91][h][3], [n][3], [nq][3]
};
ProverRandomnessLayout prover_randomness_layout(size_t n, size_t h, size_t nq);
void prover_randomness_run(Ctx &c, const uint8_t seed[32], size_t n, size_t h, size_t nq, u64 *d_out);

// ---- stark_kernels.cu ----
struct SegmentArgs {
  const u64 *quot; size_t quot_stride;
  const u64 *rnd; size_t rnd_stride; unsigned rnd_len;
  u64 *out; size_t out_stride;
  size_t seg_len;
  PowTab zeta4, off;
  u64 zeta_pow[4];
};
struct DeepArgs {
  const u64 *cw; size_t cw_stride;
  u64 *out; size_t out_stride;
  int log_n, log_r;                          // trace length 2^log_n, domain of 2^(log_n+log_r) points
  unsigned coset_first, coset_step, num_cosets;   // local coset y is domain coset coset_first + coset_step*y
  PowTab dom;
  u64 offset;
  xfe point[4], value[4], weight[4];
};
void shards_to_natural_run(Ctx &c, const u64 *in, u64 *out, size_t rank_stride, size_t plane_stride, size_t out_stride, int log_n, int log_r,
                           int log_w, int planes);
void shard_digests_to_natural_run(Ctx &c, const u64 *in, u64 *out, int log_n, int log_r, int log_w);
void coset_to_natural_run(Ctx &c, const u64 *in, u64 *out, size_t in_stride, size_t out_stride, int log_n, int log_r, int planes);
void deinterleave3_run(Ctx &c, const u64 *in, u64 *out, size_t len, size_t ncols);
void segment_chain_run(Ctx &c, const SegmentArgs &a);
void xpow_vector_run(Ctx &c, xfe base, u64 *out, size_t stride, size_t len);
void col_dot_run(Ctx &c, const u64 *cols, size_t col_stride, size_t ncols, size_t len, const u64 *xvec, size_t xvec_stride,
                 size_t xvec_set_stride, int nvec, u64 *out);
void weighted_colsum_run(Ctx &c, const u64 *cols, size_t col_stride, unsigned ncols, bool xfield, const u64 *d_w, size_t len, u64 *out,
                         size_t out_stride, bool accumulate);
void deep_run(Ctx &c, const DeepArgs &a);
void fri_leaves_run(Ctx &c, const u64 *cw, size_t stride, size_t n, u64 *leaves);
void fri_fold_run(Ctx &c, const u64 *in, size_t in_stride, size_t n, u64 offset_mont, xfe chal, u64 *out, size_t out_stride);
void gather_rows_run(Ctx &c, const u64 *table, size_t col_stride, unsigned ncols, const unsigned *d_idx, unsigned nidx, int log_n, int log_r,
                     u64 *d_out, int log_w = 0, unsigned rank = 0, unsigned coset_mem_stride = 1);
void gather_rows_scatter_run(Ctx &c, const u64 *table, size_t col_stride, unsigned ncols, const unsigned *d_kt, unsigned count, u64 *d_out);
void gather_digests_run(Ctx &c, const u64 *nodes, const unsigned *d_idx, unsigned nidx, u64 *d_out, int log_w = 0, unsigned rank = 0);
void scale_by_powers_run(Ctx &c, u64 *v, size_t stride, int planes, size_t len, PowTab tab);

}  // namespace tvm
