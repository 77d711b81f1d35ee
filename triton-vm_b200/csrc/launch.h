// Host-side launch interfaces shared between translation units.
#pragma once
#include "ctx.h"
#include "tip5.cuh"

namespace tvm {

struct ApiError {
  int code;
  std::string msg;
};

struct NttJob {
  const u64 *in;
  size_t in_cstride;
  u64 *out;
  size_t out_cstride;   // per (col*num_cosets + coset)
  u64 *tmp;             // ncols*num_cosets*n words, distinct from out
  int log_n;
  size_t ncols;
  bool inverse;
  // coset mode (forward only): evaluate on num_cosets cosets; pre table = w_{num_cosets * n}
  int num_cosets = 1;       // cosets evaluated by this job (a shard of the domain's cosets)
  int total_cosets = 0;     // r: the pre-scale table is w_{r n}; 0 = num_cosets
  unsigned coset_first = 0, coset_step = 1;   // job coset y is domain coset coset_first + coset_step*y
  bool coset_pre = false;
  unsigned fold_count = 0;
  // output post-processing
  u64 post_mul = MONT_ONE;
  bool has_post = false;
  PowTab post{};
  const u64 *rand = nullptr;
  unsigned rand_count = 0, rand_pad = 0;
};

void ntt_run(Ctx &c, const NttJob &job);
void lde_run(Ctx &c, const u64 *d_trace, const u64 *d_rand, unsigned num_rand, unsigned log2_trace,
             unsigned log2_cosets, u64 offset_mont, size_t ncols, u64 *d_coef, u64 *d_out, u64 *d_tmp);
void lde_interpolate_run(Ctx &c, const u64 *d_trace, const u64 *d_rand, unsigned num_rand, unsigned rand_pad, unsigned log2_trace,
                         u64 offset_mont, size_t ncols, u64 *d_coef, size_t coef_stride, u64 *d_tmp);
void lde_evaluate_run(Ctx &c, const u64 *d_coef, size_t coef_stride, unsigned fold_count, unsigned log2_trace, unsigned log2_cosets,
                      unsigned coset_first, unsigned coset_step, unsigned num_cosets, size_t ncols, u64 *d_out, u64 *d_tmp);
// ntt_tile.cu: the same contracts on the two-round tile kernels; false = size not covered, use the kernels of ntt.cu
bool lde_evaluate_tiles(Ctx &c, const u64 *d_coef, size_t coef_stride, unsigned fold_count, unsigned log_n, unsigned log_r,
                        unsigned coset_first, unsigned coset_step, unsigned num_cosets, size_t ncols, u64 *d_out, u64 *d_tmp);
bool lde_interpolate_tiles(Ctx &c, const u64 *d_trace, const u64 *d_rand, unsigned num_rand, unsigned rand_pad, unsigned log_n,
                           u64 offset_mont, size_t ncols, u64 *d_coef, size_t coef_stride, u64 *d_tmp);
// row i = coset + (k << log_r) of the nrows rows is read from table coset `coset * coset_mem_stride` ([col][coset][k])
void hash_rows_run(Ctx &c, const u64 *table, size_t col_stride, size_t nrows, unsigned ncols, int log_r, u64 *digests,
                   unsigned coset_mem_stride = 1);
void merkle_run(Ctx &c, u64 *nodes, size_t nleaves);
void tip5_arith_check_run(Ctx &c, const u64 *in, size_t n, u64 *out);   // fsqr and the MDS finishes, for tests
void merkle_run_sharded(Ctx &c, u64 *nodes, size_t nleaves, unsigned rank, unsigned world);
void xfe_leaves_run(Ctx &c, const u64 *cw, size_t stride, size_t n, u64 *leaves);
void to_mont_run(Ctx &c, u64 *d, size_t n);
void from_mont_run(Ctx &c, u64 *d, size_t n);
// the tables of air_quotient_run as polynomials: pre-scaled interpolant coefficients (lde_interpolate_run), column q at
// main + q*stride / aux + q*stride, of degree < n + num_rand
struct AirCoefs {
  const u64 *main, *aux;
  size_t stride;
  unsigned num_rand;
};
// evaluates on `num_cosets` of the 2^log_r cosets (domain coset coset_first + coset_step*y); the output holds only those
// cosets ([y][k]); the tables hold coset y at memory coset y*coset_mem_stride ([col][..][k]).  `coefs` (optional) lets it
// evaluate constraints on half of the domain (quotient.cu, the degree split)
void air_quotient_run(Ctx &c, const u64 *d_main, size_t main_stride, const u64 *d_aux, size_t aux_stride,
                      const u64 *d_challenges, const u64 *d_weights, unsigned log_n, unsigned log_r,
                      unsigned coset_first, unsigned coset_step, unsigned num_cosets, unsigned coset_mem_stride,
                      u64 offset_mont, u64 *d_out, size_t out_stride, const AirCoefs *coefs = nullptr);
// auxiliary-table extension (aux_extend.cu): d_main [379][n], d_ch [63*3], d_aux [273][n] planes, all Montgomery;
// the batch-randomizer planes (column 90) are the caller's.  d_scratch: aux_extend_scratch_words(n) words
size_t aux_extend_scratch_words(size_t n);
void aux_extend_run(Ctx &c, const u64 *d_main, size_t n, const u64 *d_ch, u64 *d_aux, u64 *d_scratch);
void interleave3_from_mont_run(Ctx &c, const u64 *in, u64 *out, size_t n, size_t ncols);
void main_derived_run(Ctx &c, u64 *d_main, size_t n);   // main columns 149..378 from 0..148, [379][n] Montgomery
int translate_exception(Ctx *c);

}  // namespace tvm
