// Stark::prove on one GPU: orchestration of the device kernels + host Fiat-Shamir transcript.
//
// Restates Prover::prove (triton-vm/src/stark.rs:331-719) step by step for the cached-LDE branch
// with either low-degree test (FRI: csrc/fri.cu; STIR: csrc/stir.cu) and
// the parameter derivation of stark.rs:1885-2089, fri.rs:799-924, low_degree_test/mod.rs:250-300.
// Trace generation stays with the caller (SURVEY.md §8(b)): the main trace and all randomizer
// coefficients are inputs; the auxiliary trace is requested through a callback once the
// challenges exist (stark.rs:374-380).
//
// Device layout: every table is column-major; LDE tables are additionally coset-major
// ([col][coset][k], evaluation-domain row i = coset + r*k).  X-field columns are stored as three
// planar B-field columns.  Interpolant coefficients are kept pre-scaled by offset^j.
#include <cmath>
#include <cstring>
#include <set>
#include "air.cuh"
#include "launch.h"
#include "stark.h"
#include "transcript.h"
#include <functional>
#include "prove_common.h"

namespace tvm {
#include "air_gen/air_meta.inc"

static size_t next_pow2(size_t x) {
  size_t p = 1;
  while (p < x) p <<= 1;
  return p;
}
static int ilog2(size_t x) {
  int l = 0;
  while (((size_t)1 << (l + 1)) <= x) l++;
  return l;
}

// ---- STIR round structure: StirParameters::try_into_stir (stir.rs:437-567), ProximityRegime::Proven.
// All f64 expressions keep the reference's operation order (mod.rs:250-300, stir.rs:633-869).
namespace {
double rs_rate(unsigned log2_exp) { return 1.0 / (double)(1u << log2_exp); }
double rs_q_ary_entropy(unsigned log2_exp) {                         // mod.rs:258-264
  const double rate = rs_rate(log2_exp);
  const double rate_log_rate = rate * -(double)log2_exp;
  const double one_m = (1.0 - rate) * std::log2(1.0 - rate);
  return rate - (rate_log_rate + one_m) / 191.99999999899228;         // ReedSolomonCode::LOG2_FIELD_SIZE
}
// `conj`: ProximityRegime::Conjectured instead of ::Proven (mod.rs:60-80, 243-287)
double rs_margin(unsigned log2_exp, bool conj) { return conj ? rs_q_ary_entropy(log2_exp) : std::sqrt(rs_rate(log2_exp)); }
double rs_slackness(unsigned log2_exp, bool conj) { return rs_margin(log2_exp, conj) / 20.0; }
}  // namespace
double rs_proximity_parameter(unsigned log2_exp, bool conj) { return 1.0 - rs_margin(log2_exp, conj) - rs_slackness(log2_exp, conj); }
namespace {
double rs_log2_list_size(unsigned log2_exp, bool conj, unsigned log2_poly_degree) {
  const double ls = conj ? std::pow(2.0, (double)log2_poly_degree) / (rs_q_ary_entropy(log2_exp) * rs_slackness(log2_exp, conj))
                         : 1.0 / (2.0 * std::sqrt(rs_rate(log2_exp)) * rs_slackness(log2_exp, conj));
  return std::log2(ls);
}
double log2_binomial_coefficient(unsigned long long a, unsigned long long b) {   // stir.rs:854-869 (Kahan-Babuska)
  double log2_binom = 0.0, compensation = 0.0;
  unsigned long long m = std::min(b, a - b);
  for (unsigned long long i = 0; i < m; i++) {
    double summand = std::log2((double)(a - i)) - std::log2((double)(i + 1));
    double corrected = summand - compensation;
    double next = log2_binom + corrected;
    compensation = (next - log2_binom) - corrected;
    log2_binom = next;
  }
  return log2_binom;
}
size_t stir_num_in_domain_queries(unsigned security, unsigned log2_domain_size, unsigned log2_exp, bool conj) {   // stir.rs:597-609
  double nq = -(double)security / std::log2(1.0 - rs_proximity_parameter(log2_exp, conj));
  unsigned long long uniques = (unsigned long long)std::ceil(nq);
  uniques = std::min(uniques, 1ULL << log2_domain_size);
  // num_total_in_domain_queries (stir.rs:758-776)
  unsigned long long k_minus_1 = uniques - 1;
  unsigned long long domain_len = 1ULL << log2_domain_size;
  unsigned long long l = std::min(k_minus_1, domain_len / 2);
  double log2_u_choose_l = log2_binomial_coefficient(domain_len, l);
  double log2_k_minus_1 = k_minus_1 ? std::max(std::log2((double)k_minus_1), 0.0) : 0.0;
  double total = ((double)security + log2_k_minus_1 + log2_u_choose_l) / ((double)log2_domain_size - log2_k_minus_1);
  return (size_t)std::ceil(total);
}
size_t stir_num_ood_queries(unsigned security, unsigned log2_poly_degree, unsigned log2_exp, bool conj) {          // stir.rs:831-842
  double n = ((double)security - 1.0 + 2.0 * rs_log2_list_size(log2_exp, conj, log2_poly_degree)) / (double)(192u - log2_poly_degree);
  return (size_t)std::ceil(n);
}
}  // namespace

int stir_derive(unsigned security, unsigned log2_ff, unsigned log2_initial_exp, unsigned log2_hdb, bool conj, StirDerived &out) {
  if (log2_ff < 2 || log2_initial_exp == 0 || log2_hdb < log2_ff || log2_hdb + log2_initial_exp > 32) return TVM_ERR_LDT_PARAMS;
  out = StirDerived{};
  out.folding_factor = (size_t)1 << log2_ff;
  size_t folded_poly_degree = (((size_t)1 << log2_hdb) - 1) / out.folding_factor;
  unsigned log2_exp = log2_initial_exp;
  unsigned log2_folded_domain_size = log2_hdb + log2_initial_exp - log2_ff;
  while (folded_poly_degree > out.folding_factor) {
    size_t in_domain = stir_num_in_domain_queries(security, log2_folded_domain_size, log2_exp, conj);
    unsigned log2_next_exp = log2_exp + log2_ff - 1;
    size_t ood = stir_num_ood_queries(security, (unsigned)ilog2(folded_poly_degree), log2_next_exp, conj);
    size_t next_deg = folded_poly_degree / out.folding_factor;
    if (in_domain + ood > next_deg) break;
    if (out.num_rounds >= STIR_MAX_ROUNDS) return TVM_ERR_LDT_PARAMS;
    out.in_domain[out.num_rounds] = in_domain; out.out_of_domain[out.num_rounds] = ood; out.num_rounds++;
    folded_poly_degree = next_deg;
    log2_exp = log2_next_exp;
    log2_folded_domain_size -= 1;
  }
  out.final_num_in_domain_queries = stir_num_in_domain_queries(security, log2_folded_domain_size, log2_exp, conj);
  out.final_degree = folded_poly_degree;
  return TVM_OK;
}

int stark_derive(const StarkParams &sp, size_t padded_height, StarkDerived &d) {
  if (sp.log2_expansion == 0 || sp.log2_expansion > 8 || sp.security_level == 0 || sp.ldt_choice > 2 || sp.soundness > 1) return TVM_ERR_LDT_PARAMS;
  const bool conj = sp.soundness == 1;
  padded_height = next_pow2(padded_height ? padded_height : 1);
  if (padded_height > ((size_t)1 << 31)) return TVM_ERR_DOMAIN;
  const int log2_ph = ilog2(padded_height);
  d = StarkDerived{};
  d.ldt = sp.ldt_choice ? (int)sp.ldt_choice : (log2_ph < (conj ? 17 : 16) ? 1 : 2);      // stark.rs:1942-1951
  const size_t expansion = (size_t)1 << sp.log2_expansion;
  size_t h = 0, nqr = 0, rtl = 0, ldt_len = 0;
  int hdb = log2_ph;
  for (;;) {                                                             // stark.rs:1972-2060
    hdb++;
    if (int rc = fri_derive(sp.security_level, conj, sp.log2_expansion, (unsigned)hdb, d.fri)) return rc;   // Stark::fri
    ldt_len = d.fri.domain_len;
    size_t first_round = d.fri.num_collinearity_checks;
    if (d.ldt == 2) {
      int rc = stir_derive(sp.security_level, STIR_LOG2_FOLDING_FACTOR, sp.log2_expansion, (unsigned)hdb, conj, d.stir);
      if (rc) return rc;
      first_round = d.stir.num_rounds ? d.stir.in_domain[0] : d.stir.final_num_in_domain_queries;   // stir.rs:878-883
    }
    d.num_first_round_queries = first_round;
    h = first_round + NUM_QUOTIENT_SEGMENTS * 3 * 2 + 1;                 // stark.rs:2083-2089
    nqr = (h + 1) * NUM_RANDOMIZED_QUOTIENT_SEGMENTS;                    // stark.rs:1894-1896
    rtl = next_pow2(std::max(std::max(padded_height + h, 2 * h + 1), nqr));   // stark.rs:1885-1890
    if (ldt_len >= rtl * expansion) break;
  }
  const long long interpolant_degree = (long long)rtl - 1;
  long long max_cd = 0;
  auto upd = [&](const unsigned char *degs, int n, long long zerofier_degree) {
    for (int i = 0; i < n; i++) max_cd = std::max(max_cd, interpolant_degree * degs[i] - zerofier_degree);
  };
  upd(AIR_DEGREES_INIT, AIR_NUM_INIT, 1);
  upd(AIR_DEGREES_CONS, AIR_NUM_CONS, (long long)padded_height);
  upd(AIR_DEGREES_TRAN, AIR_NUM_TRAN, (long long)padded_height - 1);
  upd(AIR_DEGREES_TERM, AIR_NUM_TERM, 1);
  const size_t max_degree = next_pow2((size_t)max_cd) - 1;              // stark.rs:1905-1916
  d.padded_height = padded_height;
  d.num_trace_randomizers = h;
  d.randomized_trace_len = rtl;
  d.trace_len = rtl / 2;
  d.quotient_len = next_pow2(max_degree);
  d.ldt_len = ldt_len;
  d.ldt_offset = d.fri.domain_offset;
  d.num_quotient_randomizer_coefficients = nqr;
  return TVM_OK;
}

namespace {

xfe eval_arg_terminal(const u64 *symbols_canon, size_t n, xfe challenge) {  // cross_table_argument.rs:60-73
  xfe acc = xone();
  for (size_t i = 0; i < n; i++) acc = xaddb(xmul(challenge, acc), to_mont(symbols_canon[i] % P));
  return acc;
}

// Shard of the evaluation domain owned by this rank: domain coset first + step*y for y < count
// (SURVEY.md 8(e)); world == 1 owns all r cosets.
struct Shard {
  unsigned first, step, count;
  int log_w;
};

// forward coset-LDE of pre-scaled coefficient columns onto this rank's cosets, in batches that fit d_tmp
void evaluate_cols(Ctx &c, const u64 *d_coef, size_t coef_stride, unsigned fold_count, size_t ncols, unsigned log_n, unsigned log_r,
                   const Shard &sh, u64 *d_lde, u64 *d_tmp, size_t tmp_cols) {
  const size_t n = (size_t)1 << log_n, n_loc = n * sh.count;
  for (size_t c0 = 0; c0 < ncols; c0 += tmp_cols) {
    size_t b = std::min(tmp_cols, ncols - c0);
    lde_evaluate_run(c, d_coef + c0 * coef_stride, coef_stride, fold_count, log_n, log_r, sh.first, sh.step, sh.count, b,
                     d_lde + c0 * n_loc, d_tmp);
  }
}

}  // namespace

void challenges_derive(const ClaimView &claim, std::vector<xfe> &ch) {
  u64 lut[256];
  for (int i = 0; i < 256; i++) lut[i] = TIP5_LOOKUP_HOST[i];
  xfe compressed_digest = eval_arg_terminal(claim.program_digest, 5, ch[0]);
  xfe input_terminal = eval_arg_terminal(claim.input, claim.num_input, ch[1]);
  xfe output_terminal = eval_arg_terminal(claim.output, claim.num_output, ch[2]);
  xfe lookup_terminal = eval_arg_terminal(lut, 256, ch[54]);
  ch.push_back(input_terminal); ch.push_back(output_terminal); ch.push_back(lookup_terminal); ch.push_back(compressed_digest);
}

void stark_prove(Ctx &c, const StarkParams &sp, const ClaimView &claim, size_t padded_height, const u64 *h_main_trace,
                 const u64 *h_main_rand, AuxCallback aux_cb, void *aux_user, const u64 *h_quot_rand, std::vector<u64> &proof,
                 ProveTimings *timings, const DeviceTables *dev_tables, const ExternalTranscript *ext) {
  StarkDerived d{};
  int rc = stark_derive(sp, padded_height, d);
  if (rc) throw ApiError{rc, "parameter derivation failed"};
  const size_t n = d.trace_len, N = d.ldt_len, Q = d.quotient_len, h = d.num_trace_randomizers;
  const unsigned log_n = (unsigned)ilog2(n), log_N = (unsigned)ilog2(N), log_r = log_N - log_n, log_Q = (unsigned)ilog2(Q);
  // The tables live on the LDT domain (r = 2 * expansion cosets of the trace domain); the quotient domain (always 8
  // cosets: AIR degree 4 on the randomized trace) is every (N/Q)-th coset of it (master_table.rs:769-779).
  if (Q != 8 * n) throw ApiError{TVM_ERR_UNSUPPORTED, "quotient domain != 8 x trace domain"};
  if (log_r > 6 || log_r < 2) throw ApiError{TVM_ERR_UNSUPPORTED, "expansion factors outside 2..32 are not supported"};
  // Evaluation domain of the tables = the larger of the two (master_table.rs:258-322): `re` cosets.  Commitments and
  // openings use every es-th coset (LDT domain), the AIR every qs-th (quotient domain); es = qs = 1 at expansion 4.
  const unsigned log_re = std::max(log_r, 3u);
  const unsigned es = (1u << log_re) >> log_r, qs = (1u << log_re) / 8;
  if ((qs != 1 || es != 1) && c.comm.world > 1) throw ApiError{TVM_ERR_UNSUPPORTED, "multi-GPU sharding needs expansion factor 4"};
  const u64 off = to_mont(d.ldt_offset);
  const size_t NM = TVM_NUM_MAIN_COLUMNS, NA = TVM_NUM_AUX_COLUMNS, NA3 = 3 * NA;
  const size_t tmp_cols = 16;
  // multi-GPU shard (tvm_ctx_set_comm): this rank owns r/W cosets = N/W rows, and 1/W of the columns
  // for the column-sharded interpolation
  const unsigned W = (unsigned)c.comm.world, rank = (unsigned)c.comm.rank;
  if (W > (1u << log_r)) throw ApiError{TVM_ERR_INVALID_ARG, "more ranks than cosets"};
  const Shard sh{rank, W, (1u << log_r) / W, ilog2(W)};      // LDT-domain cosets of this rank
  const Shard she{rank, W, (1u << log_re) / W, ilog2(W)};   // evaluation-domain cosets of this rank (tables)
  const size_t NL = n * sh.count;                       // rows of the LDT domain held by this rank
  const size_t NLe = n * she.count;                     // rows of the evaluation domain held by this rank
  const size_t hpad = std::min(n, (h + 63) & ~(size_t)63);
  const size_t cs = n + hpad;                           // stride of a table column's interpolant coefficients
  // Low-memory mode (the reference's just-in-time LDE, stark.rs:805-1006, master_table.rs:470-503, 557-606): the
  // extended main/aux tables are never stored; every use (row hashing, AIR, openings) re-evaluates one coset at a
  // time from the interpolant coefficients.  Chosen automatically when the cached tables would not fit.
  bool jit = c.low_memory_mode == 1;
  if (c.low_memory_mode == 0) {
    size_t free_b = 0, total_b = 0;
    TVM_CUDA(cudaMemGetInfo(&free_b, &total_b));
    size_t pooled = 0;
    for (auto &kv : c.pool_free) pooled += kv.first;
    const double need = 8.0 * ((double)(NM + NA3) * (NLe + cs) + 40.0 * N) * 1.15;
    jit = need > (double)(free_b + pooled);
  }
  if (timings) timings->low_memory = jit;
  struct StageEvents {           // destroyed on every exit path (an exception used to leak them)
    cudaEvent_t ev[20];
    int n = 0;
    ~StageEvents() { for (int i = 0; i < n; i++) cudaEventDestroy(ev[i]); }
  } se;
  cudaEvent_t *ev = se.ev;
  int &nev = se.n;
  auto mark = [&]() {
    if (!timings || nev >= 20) return;
    cudaEventCreate(&ev[nev]);
    cudaEventRecord(ev[nev], c.stream);
    nev++;
  };

  DevMem mem(c);
  ProofStream ps;
  ps.ext = ext;
  ps.alter_fiat_shamir_state_with(encode_claim(claim.program_digest, claim.version, claim.input, claim.num_input, claim.output,
                                               claim.num_output));
  ps.enqueue(ItemKind::Log2PaddedHeight, {(u64)ilog2(d.padded_height)});
  mark();  // 0

  // ---- main table: upload, LDE, row hashes, Merkle tree (stark.rs:359-374) -------------------------
  u64 *d_tmp = mem.words(std::max(tmp_cols * NLe, 3 * std::max(N, Q)));
  mark();  // (kept for the stage table: uploads are issued asynchronously below)
  cudaStream_t cs_copy = c.get_copy_stream();
  size_t nevt = 0;
  // Upload + interpolate + extend one table.  `xf` = 1: B-field columns [ncols][n]; 3: X-field columns in the ABI's
  // interleaved layout [ncols][n][3] (de-interleaved into 3 planar columns each).  The trace is uploaded in column
  // batches on the copy stream while the compute stream converts the batches that have landed to Montgomery form and
  // transforms them (source pointers may be host or device memory).  With W > 1 ranks each rank uploads and
  // interpolates only its block of columns; the coefficient blocks are then all-gathered and every rank evaluates
  // all columns on its own cosets.
  // Device-table mode (dev_tables): `upload_cols` < ncols columns are read from src_trace, `after_upload(d_in)` produces
  // the remaining ones in place on the device ([ncols][n] Montgomery) before they are transformed; `d_ready` = the whole
  // planar Montgomery trace already sits on the device (nothing but the randomizers is uploaded); `keep_in` receives the
  // Montgomery trace buffer instead of it being released.
  struct ExtendOpts {
    size_t upload_cols = (size_t)-1;
    std::function<void(u64 *)> after_upload;
    u64 *d_ready = nullptr;
    u64 **keep_in = nullptr;
  };
  auto extend_table = [&](const u64 *src_trace, const u64 *src_rand, size_t ncols, int xf, u64 *&d_coef, u64 *&d_lde,
                          const ExtendOpts &opt) {
    const size_t cpr = (ncols + W - 1) / W;             // columns per rank (the last block may be short)
    const size_t own0 = std::min(ncols, rank * cpr), own1 = std::min(ncols, own0 + cpr), nown = own1 - own0;
    const size_t bcols = ncols * xf;                    // B-field columns
    const size_t up_cols = std::min(nown, opt.upload_cols);
    d_coef = mem.words(cpr * W * xf * cs);
    d_lde = jit ? nullptr : mem.words(bcols * NLe);
    if (W > 1 && !opt.d_ready && (opt.keep_in || opt.after_upload)) {
      // Device-table mode on several ranks: every rank holds the WHOLE main trace (uploads the table columns or fills them
      // from the AET, computes the derived ones) because MasterMainTable::extend needs all of it; the interpolation is
      // still sharded by columns.
      if (xf != 1) throw ApiError{TVM_ERR_UNSUPPORTED, "device-table mode: base-field trace expected"};
      const size_t U = std::min(ncols, opt.upload_cols);
      u64 *d_in = mem.words(ncols * n + ncols * h), *d_rand_in = d_in + ncols * n;
      cudaEvent_t e0 = c.get_copy_event(nevt++), e1 = c.get_copy_event(nevt++);
      TVM_CUDA(cudaEventRecord(e0, c.stream));
      TVM_CUDA(cudaStreamWaitEvent(cs_copy, e0, 0));
      TVM_CUDA(cudaMemcpyAsync(d_rand_in, src_rand, ncols * h * 8, cudaMemcpyDefault, cs_copy));
      if (U) TVM_CUDA(cudaMemcpyAsync(d_in, src_trace, U * n * 8, cudaMemcpyDefault, cs_copy));
      TVM_CUDA(cudaEventRecord(e1, cs_copy));
      TVM_CUDA(cudaStreamWaitEvent(c.stream, e1, 0));
      to_mont_run(c, d_rand_in, ncols * h);
      if (U) to_mont_run(c, d_in, U * n);
      if (opt.after_upload) opt.after_upload(d_in);
      const size_t bstep = std::max<size_t>(1, tmp_cols);
      for (size_t c0 = 0; c0 < nown; c0 += bstep) {
        const size_t b = std::min(bstep, nown - c0), q0 = own0 + c0;
        lde_interpolate_run(c, d_in + q0 * n, d_rand_in + q0 * h, (unsigned)h, (unsigned)hpad, log_n, off, b, d_coef + q0 * cs, cs, d_tmp);
      }
      c.all_gather(d_coef, cpr * cs * 8);
      if (!jit) evaluate_cols(c, d_coef, cs, (unsigned)h, bcols, log_n, log_re, she, d_lde, d_tmp, tmp_cols);
      if (opt.keep_in) *opt.keep_in = d_in;
      else mem.release(d_in);
      return;
    }
    u64 *d_in = opt.d_ready ? mem.words(ncols * xf * h) : mem.words(std::max<size_t>(1, nown) * xf * n + ncols * xf * h);
    u64 *d_rand_in = opt.d_ready ? d_in : d_in + std::max<size_t>(1, nown) * xf * n;
    u64 *d_planar = opt.d_ready ? opt.d_ready : (xf == 3 ? mem.words(std::max<size_t>(1, nown) * 3 * n + ncols * 3 * h) : d_in);
    u64 *d_rand_planar = opt.d_ready ? (xf == 3 ? mem.words(ncols * 3 * h) : d_rand_in) : nullptr;
    u64 *d_rand = opt.d_ready ? d_rand_planar : (xf == 3 ? d_planar + std::max<size_t>(1, nown) * 3 * n : d_rand_in);
    {
      cudaEvent_t e = c.get_copy_event(nevt++);   // the pool may hand out blocks the compute stream still uses
      TVM_CUDA(cudaEventRecord(e, c.stream));
      TVM_CUDA(cudaStreamWaitEvent(cs_copy, e, 0));
    }
    TVM_CUDA(cudaMemcpyAsync(d_rand_in, src_rand, ncols * xf * h * 8, cudaMemcpyDefault, cs_copy));
    const size_t bstep = std::max<size_t>(1, tmp_cols / xf);   // columns per batch
    const size_t evt0 = nevt;
    // batches: [0, up_cols) uploaded, [up_cols, nown) produced on the device (a batch never straddles the boundary)
    std::vector<std::pair<size_t, size_t>> batches;
    for (size_t c0 = 0; c0 < up_cols; c0 += bstep) batches.push_back({c0, std::min(bstep, up_cols - c0)});
    const size_t nup = batches.size();
    for (size_t c0 = up_cols; c0 < nown; c0 += bstep) batches.push_back({c0, std::min(bstep, nown - c0)});
    if (!opt.d_ready)
      for (size_t bi = 0; bi < nup; bi++) {
        const size_t c0 = batches[bi].first, b = batches[bi].second;
        TVM_CUDA(cudaMemcpyAsync(d_in + c0 * xf * n, src_trace + (own0 + c0) * xf * n, b * xf * n * 8, cudaMemcpyDefault, cs_copy));
        TVM_CUDA(cudaEventRecord(c.get_copy_event(nevt++), cs_copy));
      }
    if (opt.d_ready || nup == 0) TVM_CUDA(cudaEventRecord(c.get_copy_event(nevt++), cs_copy));   // "randomizers landed"
    for (size_t bi = 0; bi < std::max<size_t>(1, batches.size()); bi++) {
      const bool uploaded = !opt.d_ready && bi < nup;
      if (uploaded || bi == 0) TVM_CUDA(cudaStreamWaitEvent(c.stream, c.get_copy_event(evt0 + (uploaded ? bi : 0)), 0));
      if (bi == 0) {
        to_mont_run(c, d_rand_in, ncols * xf * h);
        if (xf == 3) deinterleave3_run(c, d_rand_in, d_rand, h, ncols);
      }
      if (batches.empty()) break;
      if (bi == nup && !opt.d_ready && opt.after_upload) opt.after_upload(d_in);
      const size_t c0 = batches[bi].first, b = batches[bi].second;
      if (uploaded) {
        to_mont_run(c, d_in + c0 * xf * n, b * xf * n);
        if (xf == 3) deinterleave3_run(c, d_in + c0 * 3 * n, d_planar + c0 * 3 * n, n, b);
      }
      const size_t q0 = (own0 + c0) * xf;               // first B-field column of the batch
      // (a table that is already on the device is complete on every rank: this rank's block starts at column own0)
      lde_interpolate_run(c, d_planar + ((opt.d_ready ? own0 : 0) + c0) * xf * n, d_rand + q0 * h, (unsigned)h, (unsigned)hpad, log_n, off, b * xf,
                          d_coef + q0 * cs, cs, d_tmp);
      if (W == 1 && !jit) lde_evaluate_run(c, d_coef + q0 * cs, cs, (unsigned)h, log_n, log_re, she.first, she.step, she.count, b * xf,
                                           d_lde + q0 * NLe, d_tmp);
    }
    if (W > 1) {
      c.all_gather(d_coef, cpr * xf * cs * 8);
      if (!jit) evaluate_cols(c, d_coef, cs, (unsigned)h, bcols, log_n, log_re, she, d_lde, d_tmp, tmp_cols);
    }
    if (opt.d_ready) {
      if (xf == 3) mem.release(d_rand_planar);
      mem.release(d_in);
    } else {
      if (xf == 3) mem.release(d_planar);
      if (opt.keep_in) *opt.keep_in = d_in;
      else mem.release(d_in);
    }
  };
  // Row digests of this rank's rows -> leaves of the full tree (all-gathered across ranks), then the tree.
  // one local evaluation-domain coset y of a table, evaluated from its coefficients (low-memory mode): [ncols][n]
  auto evaluate_coset = [&](const u64 *d_coef, unsigned ncols, unsigned y, u64 *d_out) {
    const Shard one{she.first + she.step * y, she.step, 1, she.log_w};
    evaluate_cols(c, d_coef, cs, (unsigned)h, ncols, log_n, log_re, one, d_out, d_tmp, tmp_cols);
  };
  // d_lde: a table on the evaluation domain (main/aux, `d_coef` given: LDT rows are every es-th coset) or on the LDT
  // domain (quotient segments, d_coef == nullptr)
  auto commit_rows = [&](const u64 *d_lde, const u64 *d_coef, unsigned ncols, u64 *d_nodes) {
    const unsigned stride = d_coef ? es : 1;
    const size_t col_stride = d_coef ? NLe : NL;
    TVM_CUDA(cudaMemsetAsync(d_nodes, 0, 40, c.stream));
    if (!d_lde) {                                       // low-memory mode: hash coset by coset
      u64 *d_dig = mem.words(5 * N);                    // [rank][y][k][5], y = local LDT coset
      u64 *d_coset = mem.words((size_t)ncols * n);
      for (unsigned y = 0; y < she.count; y++) {
        if (y % stride) continue;                       // W == 1 whenever stride != 1: y is the evaluation coset itself
        evaluate_coset(d_coef, ncols, y, d_coset);
        hash_rows_run(c, d_coset, n, n, ncols, 0, d_dig + ((size_t)rank * NL + (size_t)(y / stride) * n) * 5);
      }
      mem.release(d_coset);
      c.all_gather(d_dig, NL * 40);
      shard_digests_to_natural_run(c, d_dig, d_nodes + 5 * N, (int)log_n, (int)log_r, sh.log_w);
      mem.release(d_dig);
    } else if (W == 1) {
      hash_rows_run(c, d_lde, col_stride, N, ncols, (int)log_r, d_nodes + 5 * N, stride);
    } else {
      u64 *d_dig = mem.words(5 * N);                    // [rank][y][k][5]
      hash_rows_run(c, d_lde, NL, NL, ncols, 0, d_dig + (size_t)rank * NL * 5);
      c.all_gather(d_dig, NL * 40);
      shard_digests_to_natural_run(c, d_dig, d_nodes + 5 * N, (int)log_n, (int)log_r, sh.log_w);
      mem.release(d_dig);
    }
    merkle_run_sharded(c, d_nodes, N, rank, W);
    std::vector<u64> root = d2h(c, d_nodes + 5, 5);
    for (auto &v : root) v = from_mont(v);
    ps.enqueue(ItemKind::MerkleRoot, root);
  };

  u64 *d_main_coef = nullptr, *d_main_lde = nullptr;
  u64 *d_main_trace = nullptr;          // device-table mode: the Montgomery main trace stays resident for the extension
  {
    ExtendOpts o;
    if (dev_tables) {
      o.keep_in = &d_main_trace;
      if (dev_tables->aet) {              // MasterMainTable::new + pad on the device, then the degree-lowering columns
        o.upload_cols = 0;
        o.after_upload = [&](u64 *d_in) {
          {
            DevMem fill_mem(c);             // the AET's device copy and the fill's scratch go back to the pool right after
            main_fill_run(c, fill_mem, *dev_tables->aet, n, d_in, nullptr);
          }
          to_mont_run(c, d_in, (size_t)TVM_NUM_MAIN_TABLE_COLUMNS * n);
          main_derived_run(c, d_in, n);
        };
      } else if (dev_tables->fill_derived_main) {
        o.upload_cols = TVM_NUM_MAIN_TABLE_COLUMNS;
        o.after_upload = [&](u64 *d_in) { main_derived_run(c, d_in, n); };
      }
    }
    extend_table(h_main_trace, h_main_rand, NM, 1, d_main_coef, d_main_lde, o);
  }
  mark();  // 1: main LDE
  u64 *d_main_nodes = mem.words(2 * N * 5);
  commit_rows(d_main_lde, d_main_coef, (unsigned)NM, d_main_nodes);
  mark();  // 2: main Merkle

  // ---- challenges (stark.rs:374-376, challenges.rs:88-135) -------------------------------------------
  std::vector<xfe> ch = ps.sample_scalars(59);
  challenges_derive(claim, ch);
  std::vector<u64> ch_canon, ch_mont;
  for (xfe x : ch) {
    push_xfe_canon(ch_canon, x);
    ch_mont.push_back(x.c0); ch_mont.push_back(x.c1); ch_mont.push_back(x.c2);
  }

  // ---- auxiliary table (stark.rs:380-392) ---------------------------------------------------------------
  u64 *d_aux_coef = nullptr, *d_aux_lde = nullptr;
  if (dev_tables) {
    // MasterMainTable::extend on the resident main trace (aux_extend.cu); the planes feed the interpolation directly
    u64 *d_aux_planes = mem.words(NA3 * n);
    u64 *d_misc = mem.words(3 * TVM_NUM_CHALLENGES + 3 * n + aux_extend_scratch_words(n));
    u64 *d_ch = d_misc, *d_rc = d_misc + 3 * TVM_NUM_CHALLENGES, *d_scratch = d_rc + 3 * n;
    TVM_CUDA(cudaMemcpyAsync(d_ch, ch_mont.data(), 3 * TVM_NUM_CHALLENGES * 8, cudaMemcpyHostToDevice, c.stream));
    u64 *d_rplanes = d_aux_planes + 3 * (NA - 1) * n;
    if (dev_tables->randomizer_column) {
      TVM_CUDA(cudaMemcpyAsync(d_rc, dev_tables->randomizer_column, 3 * n * 8, cudaMemcpyDefault, c.stream));
      to_mont_run(c, d_rc, 3 * n);
      deinterleave3_run(c, d_rc, d_rplanes, n, 1);
    } else {
      TVM_CUDA(cudaMemsetAsync(d_rplanes, 0, 3 * n * 8, c.stream));
    }
    aux_extend_run(c, d_main_trace, n, d_ch, d_aux_planes, d_scratch);
    TVM_CUDA(cudaStreamSynchronize(c.stream));          // ch_mont is host memory of this frame
    mem.release(d_misc);
    mem.release(d_main_trace);
    mark();  // extend (device)
    ExtendOpts o;
    o.d_ready = d_aux_planes;
    extend_table(nullptr, dev_tables->aux_rand, NA, 3, d_aux_coef, d_aux_lde, o);
    mem.release(d_aux_planes);
  } else {
    if (!aux_cb) throw ApiError{TVM_ERR_INVALID_ARG, "aux callback missing"};
    u64 *h_aux_trace = nullptr, *h_aux_rand = nullptr;   // the callee hands back pointers to its own buffers
    TVM_CUDA(cudaStreamSynchronize(c.stream));
    if (int crc = aux_cb(aux_user, ch_canon.data(), &h_aux_trace, &h_aux_rand)) throw ApiError{TVM_ERR_INVALID_ARG, "aux callback failed: " + std::to_string(crc)};
    if (!h_aux_trace || !h_aux_rand) throw ApiError{TVM_ERR_INVALID_ARG, "aux callback returned a null buffer"};
    mark();  // extend (caller)
    extend_table(h_aux_trace, h_aux_rand, NA, 3, d_aux_coef, d_aux_lde, ExtendOpts{});
  }
  mark();  // 4: aux LDE
  u64 *d_aux_nodes = mem.words(2 * N * 5);
  commit_rows(d_aux_lde, d_aux_coef, (unsigned)NA3, d_aux_nodes);
  mark();  // 5: aux Merkle

  // ---- quotient codeword (stark.rs:396-411, master_table.rs:1264-1363) ---------------------------------------
  xfe w0 = ps.sample_scalars(1)[0];
  std::vector<u64> consts(ch_mont);
  {
    xfe acc = xone();
    for (int i = 0; i < TVM_NUM_CONSTRAINTS; i++) {
      consts.push_back(acc.c0); consts.push_back(acc.c1); consts.push_back(acc.c2);
      acc = xmul(acc, w0);
    }
  }
  u64 *d_consts = mem.words(consts.size());
  TVM_CUDA(cudaMemcpyAsync(d_consts, consts.data(), consts.size() * 8, cudaMemcpyHostToDevice, c.stream));
  TVM_CUDA(cudaStreamSynchronize(c.stream));
  const size_t QL = Q / W;          // quotient-domain rows of this rank
  u64 *d_quot = mem.words(3 * Q);   // gather buffer [rank][3][QL]; this rank's rows go to its own block
  if (jit) {
    u64 *d_mc = mem.words(NM * n), *d_ac = mem.words(NA3 * n);
    for (unsigned y = 0; y < she.count; y++) {
      const unsigned coset = she.first + she.step * y;
      if (coset % qs) continue;                          // not a quotient-domain coset
      evaluate_coset(d_main_coef, (unsigned)NM, y, d_mc);
      evaluate_coset(d_aux_coef, (unsigned)NA3, y, d_ac);
      air_quotient_run(c, d_mc, n, d_ac, n, d_consts, d_consts + 3 * TVM_NUM_CHALLENGES, log_n, log_re, coset, she.step, 1, 1,
                       off, d_quot + (size_t)rank * 3 * QL + (size_t)(y / qs) * n, QL);
    }
    mem.release(d_mc); mem.release(d_ac);
  } else {
    // (the tables are low-degree extensions: with all cosets in one call the constraints of degree <= 2 run on half of them)
    air_quotient_run(c, d_main_lde, NLe, d_aux_lde, NLe, d_consts, d_consts + 3 * TVM_NUM_CHALLENGES, log_n, log_re, she.first, she.step * qs,
                     she.count / qs, qs, off, d_quot + (size_t)rank * 3 * QL, QL, true);
  }
  mark();  // 6: AIR quotient

  // interpolate (stark.rs:1224-1231): natural order, iNTT, (coset offset undone inside the segment kernel)
  c.all_gather(d_quot, 3 * QL * 8);
  u64 *d_qnat = mem.words(3 * Q);
  shards_to_natural_run(c, d_quot, d_qnat, 3 * QL, QL, Q, (int)log_n, (int)(log_Q - log_n), sh.log_w, 3);
  {
    NttJob inv{};
    inv.in = d_qnat; inv.in_cstride = Q; inv.out = d_quot; inv.out_cstride = Q; inv.tmp = d_tmp;
    inv.log_n = (int)log_Q; inv.ncols = 3; inv.inverse = true;
    ntt_run(c, inv);   // d_quot[d][j] = a_j * offset^j
  }
  // split into 4 segments + randomizer segment, randomize (stark.rs:1252-1263, 1302-1356)
  const size_t seg_len = Q / NUM_QUOTIENT_SEGMENTS;     // == 2n
  const size_t nqr = d.num_quotient_randomizer_coefficients;
  u64 *d_qr_in = mem.words(3 * nqr);
  u64 *d_qr = mem.words(3 * nqr);
  TVM_CUDA(cudaMemcpyAsync(d_qr_in, h_quot_rand, 3 * nqr * 8, cudaMemcpyDefault, c.stream));   // host, or device (seeded proves)
  to_mont_run(c, d_qr_in, 3 * nqr);
  deinterleave3_run(c, d_qr_in, d_qr, nqr, 1);
  u64 *d_seg_coef = mem.words(15 * seg_len);
  {
    // undo the coset offset: a_j = (a_j offset^j) * offset^-j
    scale_by_powers_run(c, d_quot, Q, 3, Q, c.get_pow_tab(finv(off), (int)log_Q));
    SegmentArgs sa{};
    sa.quot = d_quot; sa.quot_stride = Q;
    sa.rnd = d_qr; sa.rnd_stride = nqr; sa.rnd_len = (unsigned)nqr;
    sa.out = d_seg_coef; sa.out_stride = seg_len; sa.seg_len = seg_len;
    u64 zeta = to_mont(3);
    sa.zeta4 = c.get_pow_tab(fpow(zeta, NUM_QUOTIENT_SEGMENTS), ilog2(seg_len));
    sa.off = c.get_pow_tab(off, ilog2(seg_len));
    for (int i = 0; i < 4; i++) sa.zeta_pow[i] = fpow(zeta, (u64)i);
    segment_chain_run(c, sa);
  }
  u64 *d_seg_lde = mem.words(15 * NL);
  evaluate_cols(c, d_seg_coef, seg_len, (unsigned)n, 15, log_n, log_r, sh, d_seg_lde, d_tmp, tmp_cols);
  mark();  // 7: quotient LDE
  u64 *d_quot_nodes = mem.words(2 * N * 5);
  commit_rows(d_seg_lde, nullptr, 15, d_quot_nodes);
  mark();  // 8: quotient Merkle
  mem.release(d_qnat);

  // ---- out-of-domain rows (stark.rs:450-495) --------------------------------------------------------------------
  const xfe alpha = ps.sample_scalars(1)[0];
  const u64 omega = root_of_unity_mont(log_n);
  const xfe alpha_next = xmulb(alpha, omega);
  const u64 off_inv = finv(off);
  const size_t clen = 2 * n;
  u64 *d_pw = mem.words(4 * 3 * clen);   // 4 power vectors (alpha, omega*alpha, alpha^4, (zeta alpha)^4), each / offset
  const xfe alpha_pow = xpow(alpha, NUM_QUOTIENT_SEGMENTS);
  const xfe alpha_zeta_pow = xpow(xmulb(alpha, to_mont(3)), NUM_QUOTIENT_SEGMENTS);
  const xfe pts[4] = {alpha, alpha_next, alpha_pow, alpha_zeta_pow};
  for (int t = 0; t < 4; t++) xpow_vector_run(c, xmulb(pts[t], off_inv), d_pw + (size_t)t * 3 * clen, clen, clen);
  u64 *d_dots = mem.words((NM + NA3 + 15 + 9) * 2 * 3);
  const size_t used = n + h;   // table interpolants have n + h non-zero (pre-scaled) coefficients
  std::vector<u64> dots;
  if (W == 1) {
    col_dot_run(c, d_main_coef, cs, NM, used, d_pw, clen, 3 * clen, 2, d_dots);
    col_dot_run(c, d_aux_coef, cs, NA3, used, d_pw, clen, 3 * clen, 2, d_dots + NM * 6);
    col_dot_run(c, d_seg_coef, seg_len, 15, seg_len, d_pw + 2 * 3 * clen, clen, 3 * clen, 2, d_dots + (NM + NA3) * 6);
    dots = d2h(c, d_dots, (NM + NA3 + 15) * 6);
  } else {
    // every rank holds all coefficients; each evaluates its block of columns, the (tiny) results are all-gathered
    auto sharded_dots = [&](const u64 *d_coef, size_t ncols) {
      const size_t cpr = (ncols + W - 1) / W, own0 = std::min(ncols, rank * cpr), own1 = std::min(ncols, own0 + cpr);
      u64 *d_blk = mem.words(cpr * W * 6);
      col_dot_run(c, d_coef + own0 * cs, cs, own1 - own0, used, d_pw, clen, 3 * clen, 2, d_blk + rank * cpr * 6);
      c.all_gather(d_blk, cpr * 6 * 8);
      std::vector<u64> v = d2h(c, d_blk, ncols * 6);
      mem.release(d_blk);
      return v;
    };
    dots = sharded_dots(d_main_coef, NM);
    std::vector<u64> da = sharded_dots(d_aux_coef, NA3);
    dots.insert(dots.end(), da.begin(), da.end());
    col_dot_run(c, d_seg_coef, seg_len, 15, seg_len, d_pw + 2 * 3 * clen, clen, 3 * clen, 2, d_dots);
    std::vector<u64> dsg = d2h(c, d_dots, 15 * 6);
    dots.insert(dots.end(), dsg.begin(), dsg.end());
  }
  auto dot_at = [&](size_t col, int v) { const u64 *p = &dots[(col * 2 + v) * 3]; return xmake(p[0], p[1], p[2]); };
  for (int v = 0; v < 2; v++) {
    std::vector<u64> row;
    for (size_t q = 0; q < NM; q++) push_xfe_canon(row, dot_at(q, v));
    ps.enqueue(ItemKind::OutOfDomainMainRow, row);
    row.clear();
    for (size_t q = 0; q < NA; q++)
      push_xfe_canon(row, combine_planes(dot_at(NM + 3 * q, v), dot_at(NM + 3 * q + 1, v), dot_at(NM + 3 * q + 2, v)));
    ps.enqueue(ItemKind::OutOfDomainAuxRow, row);
  }
  xfe seg_at[5][2];
  for (int s = 0; s < 5; s++)
    for (int v = 0; v < 2; v++)
      seg_at[s][v] = combine_planes(dot_at(NM + NA3 + 3 * s, v), dot_at(NM + NA3 + 3 * s + 1, v), dot_at(NM + NA3 + 3 * s + 2, v));
  {
    std::vector<u64> row;
    for (int s = 0; s < 4; s++) push_xfe_canon(row, seg_at[s][0]);       // p: s_0..s_3 at alpha^4
    ps.enqueue(ItemKind::OutOfDomainQuotientSegments, row);
    row.clear();
    for (int s = 1; s < 5; s++) push_xfe_canon(row, seg_at[s][1]);       // r: s_1..s_4 at (zeta alpha)^4
    ps.enqueue(ItemKind::OutOfDomainQuotientSegments, row);
  }
  mark();  // 9: OOD rows

  // ---- combination codeword (stark.rs:498-639) ----------------------------------------------------------------------
  std::vector<xfe> cw3 = ps.sample_scalars(3);
  std::vector<u64> wts;   // [470 main&aux][5 p][5 r] X-field weights
  {
    xfe acc = xone();
    for (size_t i = 0; i < NM + NA; i++) { wts.push_back(acc.c0); wts.push_back(acc.c1); wts.push_back(acc.c2); acc = xmul(acc, cw3[0]); }
    xfe wq[5];
    acc = xone();
    for (int i = 0; i < 5; i++) { wq[i] = acc; acc = xmul(acc, cw3[1]); }
    for (int i = 0; i < 5; i++) { xfe w = i < 4 ? wq[i] : xzero(); wts.push_back(w.c0); wts.push_back(w.c1); wts.push_back(w.c2); }
    for (int i = 0; i < 5; i++) { xfe w = i > 0 ? wq[i] : xzero(); wts.push_back(w.c0); wts.push_back(w.c1); wts.push_back(w.c2); }
  }
  xfe w_deep[4];
  {
    xfe acc = xone();
    for (int i = 0; i < 4; i++) { w_deep[i] = acc; acc = xmul(acc, cw3[2]); }
  }
  u64 *d_wts = mem.words(wts.size());
  TVM_CUDA(cudaMemcpyAsync(d_wts, wts.data(), wts.size() * 8, cudaMemcpyHostToDevice, c.stream));
  TVM_CUDA(cudaStreamSynchronize(c.stream));
  u64 *d_cpr = mem.words(9 * clen);    // combination, p, r polynomials (pre-scaled), 3 planes each
  TVM_CUDA(cudaMemsetAsync(d_cpr, 0, 3 * clen * 8, c.stream));
  weighted_colsum_run(c, d_main_coef, cs, (unsigned)NM, false, d_wts, used, d_cpr, clen, false);
  weighted_colsum_run(c, d_aux_coef, cs, (unsigned)NA, true, d_wts + 3 * NM, used, d_cpr, clen, true);
  weighted_colsum_run(c, d_seg_coef, seg_len, 5, true, d_wts + 3 * (NM + NA), seg_len, d_cpr + 3 * clen, clen, false);
  weighted_colsum_run(c, d_seg_coef, seg_len, 5, true, d_wts + 3 * (NM + NA + 5), seg_len, d_cpr + 6 * clen, clen, false);
  // values at the out-of-domain points
  col_dot_run(c, d_cpr, clen, 3, clen, d_pw, clen, 3 * clen, 2, d_dots);                               // comb at alpha, omega*alpha
  col_dot_run(c, d_cpr + 3 * clen, clen, 6, clen, d_pw + 2 * 3 * clen, clen, 3 * clen, 2, d_dots + 18);  // p, r at alpha^4, (zeta alpha)^4
  std::vector<u64> dv = d2h(c, d_dots, 9 * 6);
  auto dvat = [&](size_t col, int v) { const u64 *p = &dv[(col * 2 + v) * 3]; return xmake(p[0], p[1], p[2]); };
  DeepArgs da{};
  da.value[0] = combine_planes(dvat(0, 0), dvat(1, 0), dvat(2, 0));
  da.value[1] = combine_planes(dvat(0, 1), dvat(1, 1), dvat(2, 1));
  da.value[2] = combine_planes(dvat(3, 0), dvat(4, 0), dvat(5, 0));
  da.value[3] = combine_planes(dvat(6, 1), dvat(7, 1), dvat(8, 1));
  u64 *d_cpr_lde = mem.words(9 * NL);
  evaluate_cols(c, d_cpr, clen, (unsigned)n, 9, log_n, log_r, sh, d_cpr_lde, d_tmp, tmp_cols);
  u64 *d_deep = mem.words(3 * N);   // gather buffer [rank][3][NL]
  u64 *d_fri = mem.words(3 * N);
  da.cw = d_cpr_lde; da.cw_stride = NL; da.out = d_deep + (size_t)rank * 3 * NL; da.out_stride = NL;
  da.log_n = (int)log_n; da.log_r = (int)log_r;
  da.coset_first = sh.first; da.coset_step = sh.step; da.num_cosets = sh.count;
  da.dom = c.get_pow_tab(root_of_unity_mont(log_N), (int)log_N);
  da.offset = off;
  for (int t = 0; t < 4; t++) { da.point[t] = pts[t]; da.weight[t] = w_deep[t]; }
  deep_run(c, da);
  c.all_gather(d_deep, 3 * NL * 8);
  shards_to_natural_run(c, d_deep, d_fri, 3 * NL, NL, N, (int)log_n, (int)log_r, sh.log_w, 3);
  mem.release(d_deep);
  mark();  // 10: linear combination + DEEP

  // ---- low-degree test of the combination codeword (stark.rs:641-646) -------------------------------------------------
  std::vector<uint32_t> a_indices;
  const size_t max_open = std::max<size_t>(d.num_first_round_queries, 1);
  unsigned *d_idx = (unsigned *)mem.words(max_open * 64 + 64);
  u64 *d_gather = mem.words(max_open * 400 + max_open * 5 * 40 + 64);
  if (d.ldt == 2) a_indices = stir_prove_run(c, mem, ps, d_fri, N, off, d.stir, d_tmp);
  else a_indices = fri_prove_run(c, mem, ps, d_fri, N, off, d.fri, d_tmp);
  const unsigned nq = (unsigned)a_indices.size();
  mark();  // 11: FRI

  // ---- zero-knowledge guard (stark.rs:648-663) -----------------------------------------------------------------------------
  if (alpha_pow.c1 == 0 && alpha_pow.c2 == 0) {
    u64 g = root_of_unity_mont(log_N);
    u64 second = fmul(alpha_pow.c0, fpow(to_mont(3), NUM_QUOTIENT_SEGMENTS));
    for (uint32_t i : a_indices) {
      u64 x = fmul(off, fpow(g, i));
      if (x == alpha_pow.c0 || x == second) throw ApiError{TVM_ERR_ZK_VIOLATION, "out-of-domain point collides with a revealed row"};
    }
  }

  // ---- open rows (stark.rs:665-716) ---------------------------------------------------------------------------------------------
  auto open_table = [&](const u64 *table, const u64 *d_coef, unsigned ncols, ItemKind kind, const u64 *nodes) {
    const unsigned stride = d_coef ? es : 1;            // main/aux tables live on the evaluation domain
    if (table) {
      TVM_CUDA(cudaMemcpyAsync(d_idx, a_indices.data(), nq * 4, cudaMemcpyHostToDevice, c.stream));
      gather_rows_run(c, table, d_coef ? NLe : NL, ncols, d_idx, nq, (int)log_n, (int)log_r, d_gather, sh.log_w, rank, stride);
    } else {
      // low-memory mode: re-evaluate the cosets that contain opened rows (master_table.rs:557-606)
      TVM_CUDA(cudaMemsetAsync(d_gather, 0, (size_t)nq * ncols * 8, c.stream));
      u64 *d_coset = mem.words((size_t)ncols * n);
      for (unsigned y = 0; y < she.count; y++) {
        const unsigned ecoset = she.first + she.step * y;
        if (ecoset % stride) continue;
        const unsigned coset = ecoset / stride;         // LDT-domain coset
        std::vector<unsigned> kt;                       // (k, t) pairs of the queries that fall into this coset
        for (unsigned t = 0; t < nq; t++)
          if ((a_indices[t] & ((1u << log_r) - 1)) == coset) { kt.push_back(a_indices[t] >> log_r); kt.push_back(t); }
        if (kt.empty()) continue;
        evaluate_coset(d_coef, ncols, y, d_coset);
        TVM_CUDA(cudaMemcpyAsync(d_idx, kt.data(), kt.size() * 4, cudaMemcpyHostToDevice, c.stream));
        gather_rows_scatter_run(c, d_coset, n, ncols, d_idx, (unsigned)(kt.size() / 2), d_gather);
        TVM_CUDA(cudaStreamSynchronize(c.stream));      // `kt` goes out of scope
      }
      mem.release(d_coset);
    }
    c.all_reduce_sum(d_gather, (size_t)nq * ncols);
    std::vector<u64> rows = d2h(c, d_gather, (size_t)nq * ncols);
    std::vector<u64> payload;
    payload.push_back(nq);
    payload.insert(payload.end(), rows.begin(), rows.end());
    ps.enqueue(kind, payload);
    std::vector<unsigned> an = auth_structure_node_indices(N, a_indices);
    std::vector<u64> auth;
    auth.push_back(an.size());
    if (!an.empty()) {
      TVM_CUDA(cudaMemcpyAsync(d_idx, an.data(), an.size() * 4, cudaMemcpyHostToDevice, c.stream));
      gather_digests_run(c, nodes, d_idx, (unsigned)an.size(), d_gather, sh.log_w, rank);
      c.all_reduce_sum(d_gather, an.size() * 5);
      std::vector<u64> dg = d2h(c, d_gather, an.size() * 5);
      auth.insert(auth.end(), dg.begin(), dg.end());
    }
    ps.enqueue(ItemKind::AuthenticationStructure, auth);
  };
  open_table(d_main_lde, d_main_coef, (unsigned)NM, ItemKind::MasterMainTableRows, d_main_nodes);
  open_table(d_aux_lde, d_aux_coef, (unsigned)NA3, ItemKind::MasterAuxTableRows, d_aux_nodes);
  open_table(d_seg_lde, nullptr, 15, ItemKind::QuotientSegmentsElements, d_quot_nodes);
  mark();  // 12: open

  proof = ps.encode();
  if (timings) {
    TVM_CUDA(cudaStreamSynchronize(c.stream));
    const char *names[] = {"setup", dev_tables && dev_tables->aet ? "table fill+derived columns+LDE(main)" : dev_tables && dev_tables->fill_derived_main ? "upload+derived columns+LDE(main)" : "upload+LDE(main)",
                           "Merkle(main)", dev_tables ? "extend(device)" : "extend(caller)", dev_tables ? "LDE(aux)" : "upload+LDE(aux)",
                           "Merkle(aux)", "quotient(AIR)", "quotient LDE", "Merkle(quot)", "OOD rows", "linear combination+DEEP",
                           "low-degree test", "open"};
    timings->stages.clear();
    for (int i = 1; i < nev; i++) {
      float ms = 0;
      cudaEventElapsedTime(&ms, ev[i - 1], ev[i]);
      timings->stages.push_back({names[i - 1], ms});
    }
  }
}

}  // namespace tvm
