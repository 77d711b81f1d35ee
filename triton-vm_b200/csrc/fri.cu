// FRI low-degree test, prover side, on a device-resident codeword; and its parameter derivation.
//
// Restates FriParameters::try_into_fri and Fri::{max_degree, num_rounds, last_round_max_degree}
// (triton-vm/src/low_degree_test/fri.rs:799-924) and Fri::prove (fri.rs:212-366, 754-772).  The
// folding, leaf digests, Merkle levels and the gathers of revealed leaves and authentication
// structures run on the device; the host keeps the Fiat-Shamir transcript: per round it reads the
// 5-word Merkle root and hands the folding challenge back.  Used by the whole prove (prover.cu)
// and by the stand-alone tvm_fri_prove (api.cu).
//
// Layout: X-field codewords are 3 planes, [3][len] packed.
#include <cmath>
#include "prove_common.h"
#include "transcript.h"

namespace tvm {
namespace {
int ilog2f(size_t x) { int l = 0; while (((size_t)1 << (l + 1)) <= x) l++; return l; }
}  // namespace

int fri_derive(unsigned security, bool conj, unsigned log2_exp, unsigned log2_hdb, FriDerived &out, const char **error) {
  auto reject = [&](const char *what) {
    if (error) *error = what;
    return TVM_ERR_LDT_PARAMS;
  };
  // fri.rs:800-809; ReedSolomonCode::rate (mod.rs:318-320) refuses every expansion factor of 2^32 or more
  if (log2_exp == 0) return reject("LdtParameterError: TooSmallInitialExpansionFactor");
  if (log2_exp >= 32) return reject("LdtParameterError: TooBigInitialExpansionFactor");
  // ArithmeticDomain::of_length needs a 2-power root of unity of the domain's order (fri.rs:815-829)
  if ((unsigned long long)log2_hdb + log2_exp > 32) return reject("LdtParameterError: InitialDomainTooBig");
  out = FriDerived{};
  out.domain_len = (size_t)1 << (log2_hdb + log2_exp);
  out.domain_offset = 7;                                                  // BFieldElement::generator(), fri.rs:829
  out.expansion_factor = (size_t)1 << log2_exp;
  // fri.rs:832-836 (same f64 operation order)
  out.num_collinearity_checks = (size_t)std::ceil(-(double)security / std::log2(1.0 - rs_proximity_parameter(log2_exp, conj)));
  out.max_degree = out.domain_len / out.expansion_factor - 1;             // fri.rs:872-874
  // fri.rs:907-920: skip the rounds whose Merkle verification would cost more than their arithmetic
  const int max_num_rounds = ilog2f(out.max_degree + 1);                  // max_degree + 1 is a power of two
  const int skip = (out.num_collinearity_checks ? ilog2f(out.num_collinearity_checks) : 0) + 1;
  out.num_rounds = max_num_rounds > skip ? (size_t)(max_num_rounds - skip) : 0;
  out.last_round_max_degree = out.max_degree >> out.num_rounds;          // fri.rs:922-924
  return TVM_OK;
}

std::vector<uint32_t> fri_prove_run(Ctx &c, DevMem &mem, ProofStream &ps, const u64 *d_codeword, size_t len, u64 offset_mont,
                                    const FriDerived &fd, u64 *d_tmp) {
  if (len != fd.domain_len) throw ApiError{TVM_ERR_INVALID_ARG, "FRI: codeword length differs from the domain length"};
  const size_t checks = fd.num_collinearity_checks;
  // index and gather buffers for one FriResponse: `checks` leaves, at most checks * height authentication nodes
  const size_t max_nodes = std::max<size_t>(1, checks) * (size_t)ilog2f(len);
  unsigned *d_idx = (unsigned *)mem.words((std::max(checks, max_nodes) + 1) / 2);
  u64 *d_gather = mem.words(std::max(3 * checks, 5 * max_nodes));

  // commit phase (fri.rs:212-253): round 0 is the input codeword, every further round folds the previous one
  struct Round { const u64 *cw; size_t len; u64 *nodes; };
  std::vector<Round> rounds;
  std::vector<u64 *> owned;   // folded codewords
  {
    const u64 *cur = d_codeword;
    size_t cur_len = len;
    u64 offset = offset_mont;
    for (size_t r = 0; r <= fd.num_rounds; r++) {
      if (r > 0) {
        const xfe chal = ps.sample_scalars(1)[0];
        u64 *nxt = mem.words(3 * (cur_len / 2));
        fri_fold_run(c, cur, cur_len, cur_len, offset, chal, nxt, cur_len / 2);
        owned.push_back(nxt);
        cur = nxt; cur_len /= 2; offset = fmul(offset, offset);
      }
      u64 *nodes = mem.words(2 * cur_len * 5);
      TVM_CUDA(cudaMemsetAsync(nodes, 0, 40, c.stream));
      fri_leaves_run(c, cur, cur_len, cur_len, nodes + 5 * cur_len);
      merkle_run(c, nodes, cur_len);
      std::vector<u64> root = d2h(c, nodes + 5, 5);
      for (auto &v : root) v = from_mont(v);
      ps.enqueue(ItemKind::MerkleRoot, root);
      rounds.push_back({cur, cur_len, nodes});
    }
  }
  {
    const Round &last = rounds.back();
    std::vector<u64> planes = d2h(c, last.cw, 3 * last.len);
    std::vector<u64> payload;
    payload.push_back(last.len);
    for (size_t i = 0; i < last.len; i++)
      for (int dd = 0; dd < 3; dd++) payload.push_back(from_mont(planes[dd * last.len + i]));
    ps.enqueue(ItemKind::FriCodeword, payload);
    // last polynomial: interpolant over the unit-offset domain of that length (fri.rs:261-268)
    u64 *d_lp = mem.words(3 * last.len);
    NttJob inv{};
    inv.in = last.cw; inv.in_cstride = last.len; inv.out = d_lp; inv.out_cstride = last.len; inv.tmp = d_tmp;
    inv.log_n = ilog2f(last.len); inv.ncols = 3; inv.inverse = true;
    ntt_run(c, inv);
    std::vector<u64> co = d2h(c, d_lp, 3 * last.len);
    mem.release(d_lp);
    size_t deg_plus_1 = last.len;
    while (deg_plus_1 > 0 && co[deg_plus_1 - 1] == 0 && co[last.len + deg_plus_1 - 1] == 0 && co[2 * last.len + deg_plus_1 - 1] == 0) deg_plus_1--;
    // Polynomial { coefficients } encodes like a one-field struct: the coefficient Vec's encoding (count, elements) behind
    // its own length — pinned by the reference's whole-proof digest (tests/test_golden.py, proof.rs:200-226)
    payload.clear();
    payload.push_back(1 + 3 * deg_plus_1);
    payload.push_back(deg_plus_1);
    for (size_t i = 0; i < deg_plus_1; i++)
      for (int dd = 0; dd < 3; dd++) payload.push_back(from_mont(co[dd * last.len + i]));
    ps.enqueue(ItemKind::Polynomial, payload);
  }

  // query phase (fri.rs:270-319): A indices in round 0, B indices (A + len/2) in every round that has a successor
  const std::vector<uint32_t> a_indices = ps.sample_indices((uint32_t)len, checks);
  auto reveal = [&](const Round &rd, const std::vector<uint32_t> &idx) {
    std::vector<u64> leaves, auth;
    if (!idx.empty()) {
      TVM_CUDA(cudaMemcpyAsync(d_idx, idx.data(), idx.size() * 4, cudaMemcpyHostToDevice, c.stream));
      gather_rows_run(c, rd.cw, rd.len, 3, d_idx, (unsigned)idx.size(), 0, -1, d_gather);
      leaves = d2h(c, d_gather, idx.size() * 3);
    }
    const std::vector<unsigned> nodes = auth_structure_node_indices(rd.len, idx);
    if (!nodes.empty()) {      // empty when every leaf is revealed (checks >= len)
      TVM_CUDA(cudaMemcpyAsync(d_idx, nodes.data(), nodes.size() * 4, cudaMemcpyHostToDevice, c.stream));
      gather_digests_run(c, rd.nodes, d_idx, (unsigned)nodes.size(), d_gather);
      auth = d2h(c, d_gather, nodes.size() * 5);
    }
    ps.enqueue(ItemKind::FriResponse, encode_fri_response(leaves, auth));
  };
  reveal(rounds[0], a_indices);
  for (size_t r = 0; r + 1 < rounds.size(); r++) {
    std::vector<uint32_t> b(a_indices.size());
    for (size_t i = 0; i < b.size(); i++) b[i] = (uint32_t)(((size_t)a_indices[i] + rounds[r].len / 2) % rounds[r].len);
    reveal(rounds[r], b);
  }
  ps.sample_scalars(1);   // the verifier's barycentric indeterminate (fri.rs:764-769)

  for (const Round &rd : rounds) mem.release(rd.nodes);
  for (u64 *p : owned) mem.release(p);
  mem.release(d_idx); mem.release(d_gather);
  return a_indices;
}

}  // namespace tvm
