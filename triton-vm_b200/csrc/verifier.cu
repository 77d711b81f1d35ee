// Stark::verify (triton-vm/src/stark.rs:1388-1763) — SURVEY.md 8(f).4.
//
// Host code on purpose: verifying ONE proof is a short, strictly sequential Fiat-Shamir replay — a few hundred Tip5
// permutations for the transcript, one evaluation of the 604 AIR constraints at a single out-of-domain point,
// num_first_round_queries (173 at Stark::default()) Merkle paths and row hashes, and the low-degree test's collinearity
// or fold checks on those few points.  That is milliseconds on one core and offers no data parallelism a GPU could use;
// the device only becomes interesting for batches of thousands of proofs.  Everything here follows the oracle's restated
// verifier (oracle/stark.py::verify, pinned through the reference's whole-proof digests) step for step and reuses the
// prover's host-side transcript (transcript.h), parameter derivation (stark_derive) and Tip5.
//
// Failures carry the name of the reference's error variant (VerificationError, error.rs:190-260; LdtVerificationError,
// low_degree_test/mod.rs).  No CUDA call is made: tvm_verify needs no context and no GPU.
#include <algorithm>
#include <atomic>
#include <map>
#include <thread>
#include <set>
#include <cstring>
#include "../../include/tvm_b200.h"
#include "prove_common.h"
#include "transcript.h"

namespace tvm {
namespace {

struct VerifyFailure {
  const char *what;
};
[[noreturn]] void fail(const char *what) { throw VerifyFailure{what}; }

constexpr size_t NM = TVM_NUM_MAIN_COLUMNS, NA = TVM_NUM_AUX_COLUMNS, NCH = TVM_NUM_CHALLENGES;
constexpr int NUM_DEEP_CODEWORD_COMPONENTS = 4;
constexpr u64 ZETA = 3;   // stark.rs:1801

// The generated evaluator is ~9 000 straight-line statements executed once per proof: keep the field operations out of line
// there, or the host compiler spends minutes inlining them.
__attribute__((noinline)) xfe air_xmul(xfe a, xfe b) { return xmul(a, b); }
__attribute__((noinline)) xfe air_xmulb(xfe a, u64 b) { return xmulb(a, b); }
__attribute__((noinline)) xfe air_xadd(xfe a, xfe b) { return xadd(a, b); }
__attribute__((noinline)) xfe air_xaddb(xfe a, u64 b) { return xaddb(a, b); }
__attribute__((noinline)) u64 air_fmul(u64 a, u64 b) { return fmul(a, b); }
__attribute__((noinline)) u64 air_fadd(u64 a, u64 b) { return fadd(a, b); }
#define xmul air_xmul
#define xmulb air_xmulb
#define xadd air_xadd
#define xaddb air_xaddb
#define fmul air_fmul
#define fadd air_fadd
#define AIR_VERIFY_FN static __attribute__((optimize("O0")))
#define AIR_VERIFY_ARGS const xfe *mc, const xfe *ac, const xfe *mn, const xfe *an, const xfe *ch
#define MC(col) mc[col]
#define MN(col) mn[col]
#define AC(col) ac[col]
#define AN(col) an[col]
#define CH(i) ch[i]
#include "air_gen/air_verify_gen.inc"
#undef MC
#undef MN
#undef AC
#undef AN
#undef CH
#undef xmul
#undef xmulb
#undef xadd
#undef xaddb
#undef fmul
#undef fadd

// ---- field helpers (Montgomery form throughout) ---------------------------------------------------------------------
inline xfe xm(const u64 *canon) { return xmake(to_mont(canon[0]), to_mont(canon[1]), to_mont(canon[2])); }
inline xfe xscale(xfe a, u64 b_mont) { return xmulb(a, b_mont); }
inline u64 fpow(u64 b_mont, u64 e) {
  u64 r = MONT_ONE;
  while (e) {
    if (e & 1) r = fmul(r, b_mont);
    b_mont = fmul(b_mont, b_mont);
    e >>= 1;
  }
  return r;
}
std::vector<xfe> xpows(xfe x, size_t n) {
  std::vector<xfe> out(n);
  xfe acc = xone();
  for (size_t i = 0; i < n; i++) {
    out[i] = acc;
    acc = xmul(acc, x);
  }
  return out;
}
inline unsigned ilog2z(size_t v) {
  unsigned r = 0;
  while ((size_t)1 << (r + 1) <= v) r++;
  return r;
}

// ---- proof decoding (proof_stream.rs:110-125, proof_item.rs:96-147; BFieldCodec as in transcript.h) -------------------
struct Item {
  int kind;
  std::vector<u64> encoding;   // the item's full encoding (what Fiat-Shamir absorbs), canonical
  size_t payload_at;           // first payload word inside `encoding`
  const u64 *payload() const { return encoding.data() + payload_at; }
  size_t payload_len() const { return encoding.size() - payload_at; }
};

struct Transcript {
  std::vector<Item> items;
  size_t index = 0;
  Sponge sponge;

  explicit Transcript(const u64 *w, size_t n) {
    for (size_t i = 0; i < n; i++)
      if (w[i] >= P) fail("ProofDecodingError: non-canonical field element");
    size_t pos = 0;
    auto one = [&]() -> u64 {
      if (pos >= n) fail("ProofDecodingError: SequenceTooShort");
      return w[pos++];
    };
    if (one() != n - 1) fail("ProofDecodingError: length prefix mismatch");
    const u64 count = one();
    if (count > n) fail("ProofDecodingError: item count");
    for (u64 k = 0; k < count; k++) {
      const u64 len = one();
      if (len == 0 || len > n - pos) fail("ProofDecodingError: SequenceTooShort");
      Item it;
      it.encoding.assign(w + pos, w + pos + len);
      pos += len;
      if (it.encoding[0] > 13) fail("ProofDecodingError: unknown item variant");
      it.kind = (int)it.encoding[0];
      if (item_payload_static((ItemKind)it.kind)) {
        it.payload_at = 1;
      } else {
        if (len < 2 || it.encoding[1] != len - 2) fail("ProofDecodingError: payload length prefix mismatch");
        it.payload_at = 2;
      }
      items.push_back(std::move(it));
    }
    if (pos != n) fail("ProofDecodingError: trailing words");
  }

  const Item &dequeue(ItemKind k, const char *unexpected) {
    if (index >= items.size()) fail("ProofStreamError: EmptyQueue");
    const Item &it = items[index++];
    if (it.kind != (int)k) fail(unexpected);
    if (item_in_fiat_shamir(k)) sponge.pad_and_absorb_all(it.encoding);
    return it;
  }
  // typed payloads -------------------------------------------------------------------------------------------------
  std::vector<u64> digest(const char *u = "UnexpectedItem: MerkleRoot") {
    const Item &it = dequeue(ItemKind::MerkleRoot, u);
    if (it.payload_len() != 5) fail("ProofDecodingError: MerkleRoot");
    std::vector<u64> d(5);
    for (int i = 0; i < 5; i++) d[i] = to_mont(it.payload()[i]);
    return d;
  }
  std::vector<xfe> fixed_xfes(ItemKind k, size_t count, const char *u) {
    const Item &it = dequeue(k, u);
    if (it.payload_len() != 3 * count) fail("ProofDecodingError: row length");
    std::vector<xfe> v(count);
    for (size_t i = 0; i < count; i++) v[i] = xm(it.payload() + 3 * i);
    return v;
  }
  static std::vector<xfe> vec_xfe(const u64 *p, size_t len) {   // Vec<XFE>: count, elements
    if (len < 1 || p[0] > len || len != 1 + 3 * p[0]) fail("ProofDecodingError: Vec<XFieldElement>");
    std::vector<xfe> v(p[0]);
    for (size_t i = 0; i < v.size(); i++) v[i] = xm(p + 1 + 3 * i);
    return v;
  }
  static std::vector<std::vector<u64>> vec_digest(const u64 *p, size_t len) {
    if (len < 1 || p[0] > len || len != 1 + 5 * p[0]) fail("ProofDecodingError: Vec<Digest>");
    std::vector<std::vector<u64>> v(p[0], std::vector<u64>(5));
    for (size_t i = 0; i < v.size(); i++)
      for (int d = 0; d < 5; d++) v[i][d] = to_mont(p[1 + 5 * i + d]);
    return v;
  }
  std::vector<xfe> xfe_vector(ItemKind k, const char *u) {
    const Item &it = dequeue(k, u);
    return vec_xfe(it.payload(), it.payload_len());
  }
  std::vector<xfe> polynomial() {   // one-field struct: length of the Vec encoding, then the Vec; no trailing zeros
    const Item &it = dequeue(ItemKind::Polynomial, "UnexpectedItem: Polynomial");
    if (it.payload_len() < 1 || it.payload()[0] != it.payload_len() - 1) fail("ProofDecodingError: Polynomial");
    std::vector<xfe> c = vec_xfe(it.payload() + 1, it.payload_len() - 1);
    if (!c.empty() && xis_zero(c.back())) fail("ProofDecodingError: TrailingZerosInPolynomialEncoding");
    return c;
  }
  std::vector<std::vector<u64>> auth_structure() {
    const Item &it = dequeue(ItemKind::AuthenticationStructure, "UnexpectedItem: AuthenticationStructure");
    return vec_digest(it.payload(), it.payload_len());
  }
  // rows of `width` words each: count, then count * width words (canonical, returned as such)
  std::vector<const u64 *> rows(ItemKind k, size_t width, const char *u) {
    const Item &it = dequeue(k, u);
    if (it.payload_len() < 1 || it.payload()[0] > it.payload_len() || it.payload_len() != 1 + width * it.payload()[0])
      fail("ProofDecodingError: table rows");
    std::vector<const u64 *> r(it.payload()[0]);
    for (size_t i = 0; i < r.size(); i++) r[i] = it.payload() + 1 + width * i;
    return r;
  }
  // struct { queried_leaves: Vec<XFE>, auth_structure: Vec<Digest> } — fields in reverse order, each length-prefixed
  void fri_response(std::vector<xfe> &leaves, std::vector<std::vector<u64>> &auth) {
    const Item &it = dequeue(ItemKind::FriResponse, "UnexpectedItem: FriResponse");
    const u64 *p = it.payload();
    size_t len = it.payload_len(), pos = 0;
    auto field = [&](size_t &at, size_t &flen) {
      if (pos >= len) fail("ProofDecodingError: FriResponse");
      flen = p[pos++];
      if (flen > len - pos) fail("ProofDecodingError: FriResponse");
      at = pos;
      pos += flen;
    };
    size_t a_at, a_len, l_at, l_len;
    field(a_at, a_len);
    field(l_at, l_len);
    if (pos != len) fail("ProofDecodingError: FriResponse");
    auth = vec_digest(p + a_at, a_len);
    leaves = vec_xfe(p + l_at, l_len);
  }
  // struct { queried_leafs: Vec<Vec<XFE>>, auth_structure }
  void stir_response(std::vector<std::vector<xfe>> &leafs, std::vector<std::vector<u64>> &auth) {
    const Item &it = dequeue(ItemKind::StirResponse, "UnexpectedItem: StirResponse");
    const u64 *p = it.payload();
    size_t len = it.payload_len(), pos = 0;
    auto take = [&]() -> u64 {
      if (pos >= len) fail("ProofDecodingError: StirResponse");
      return p[pos++];
    };
    const size_t a_len = take();
    if (a_len > len - pos) fail("ProofDecodingError: StirResponse");
    auth = vec_digest(p + pos, a_len);
    pos += a_len;
    const size_t l_len = take();
    if (l_len != len - pos) fail("ProofDecodingError: StirResponse");
    const size_t count = take();
    if (count > len) fail("ProofDecodingError: StirResponse");
    leafs.clear();
    for (size_t i = 0; i < count; i++) {
      const size_t inner = take();
      if (inner > len - pos) fail("ProofDecodingError: StirResponse");
      leafs.push_back(vec_xfe(p + pos, inner));
      pos += inner;
    }
    if (pos != len) fail("ProofDecodingError: StirResponse");
  }
};

// ---- Merkle inclusion of several leaves at once (twenty-first MerkleTreeInclusionProof::verify) ----------------------
bool verify_inclusion(const std::vector<u64> &root, unsigned height, const std::vector<uint32_t> &indices,
                      const std::vector<std::vector<u64>> &leafs, const std::vector<std::vector<u64>> &auth) {
  const size_t num_leafs = (size_t)1 << height;
  for (uint32_t i : indices)
    if (i >= num_leafs) return false;
  std::vector<unsigned> idx = auth_structure_node_indices(num_leafs, indices);
  if (idx.size() != auth.size() || indices.size() != leafs.size()) return false;
  std::map<size_t, std::vector<u64>> known;
  for (size_t i = 0; i < idx.size(); i++) known[idx[i]] = auth[i];
  std::set<size_t> frontier;
  for (size_t i = 0; i < indices.size(); i++) {
    const size_t node = indices[i] + num_leafs;
    auto it = known.find(node);
    if (it != known.end() && it->second != leafs[i]) return false;
    known[node] = leafs[i];
    frontier.insert(node);
  }
  if (frontier.empty()) return false;
  while (!(frontier.size() == 1 && *frontier.begin() == 1)) {
    std::set<size_t> next;
    for (size_t node : frontier) {
      if (node == 1) { next.insert(1); continue; }
      auto sib = known.find(node ^ 1);
      if (sib == known.end()) return false;
      const std::vector<u64> &self = known[node];
      std::vector<u64> h(5);
      if (node % 2 == 0) tip5_hash_pair_host(self.data(), sib->second.data(), h.data());
      else tip5_hash_pair_host(sib->second.data(), self.data(), h.data());
      const size_t parent = node / 2;
      auto pk = known.find(parent);
      if (pk != known.end() && pk->second != h) return false;
      known[parent] = h;
      next.insert(parent);
    }
    frontier.swap(next);
  }
  return known[1] == root;
}
std::vector<u64> xfe_leaf(xfe v) { return {v.c0, v.c1, v.c2, 0, 0}; }   // Digest::from(xfe), fri.rs:343-347
std::vector<u64> hash_row(const u64 *canon, size_t n) {
  std::vector<u64> m(n), d(5);
  for (size_t i = 0; i < n; i++) m[i] = to_mont(canon[i]);
  tip5_hash_varlen_host(m.data(), n, d.data());
  return d;
}

// ---- FRI verifier (fri.rs:393-735) -> first-round indices and the revealed first-round values ------------------------
xfe xpoly_eval(const std::vector<xfe> &c, xfe x) {
  xfe acc = xzero();
  for (size_t i = c.size(); i-- > 0;) acc = xadd(xmul(acc, x), c[i]);
  return acc;
}
xfe barycentric_evaluate(const std::vector<xfe> &codeword, xfe x) {   // unit-offset domain of the codeword's length
  const size_t n = codeword.size();
  const u64 g = root_of_unity_mont(ilog2z(n));
  xfe num = xzero(), den = xzero();
  u64 dpt = MONT_ONE;
  for (size_t i = 0; i < n; i++) {
    xfe w = xscale(xinv(xsubb(x, dpt)), dpt);
    num = xadd(num, xmul(w, codeword[i]));
    den = xadd(den, w);
    dpt = fmul(dpt, g);
  }
  return xmul(num, xinv(den));
}

struct LdtResult {
  std::vector<uint32_t> indices;
  std::vector<xfe> values;
};

LdtResult fri_verify(Transcript &ps, const FriDerived &d) {
  const size_t checks = d.num_collinearity_checks, num_rounds = d.num_rounds;
  struct Round { u64 offset; size_t len; std::vector<u64> root; xfe chal; std::vector<xfe> a, b; };
  std::vector<Round> rounds;
  u64 offset = to_mont(d.domain_offset);
  size_t length = d.domain_len;
  for (size_t j = 0; j <= num_rounds; j++) {
    Round r;
    r.offset = offset; r.len = length;
    r.root = ps.digest();
    r.chal = xzero();
    if (num_rounds > 0 && j + 1 <= num_rounds) r.chal = ps.sponge.sample_scalars(1)[0];
    rounds.push_back(r);
    offset = fmul(offset, offset);
    length /= 2;
  }
  std::vector<xfe> last_codeword = ps.xfe_vector(ItemKind::FriCodeword, "UnexpectedItem: FriCodeword");
  std::vector<xfe> last_poly = ps.polynomial();
  if (last_codeword.size() != rounds.back().len) fail("LdtVerificationError: LastCodewordMismatch");

  auto check = [&](size_t rnd, const std::vector<uint32_t> &idx, const std::vector<xfe> &leaves,
                   const std::vector<std::vector<u64>> &auth) {
    std::vector<std::vector<u64>> lf;
    for (xfe v : leaves) lf.push_back(xfe_leaf(v));
    if (!verify_inclusion(rounds[rnd].root, ilog2z(rounds[rnd].len), idx, lf, auth)) fail("LdtVerificationError: BadMerkleAuthenticationPath");
  };
  std::vector<uint32_t> a_indices;
  {
    // The first response is read, and its size checked, before the indices are sampled: responses are outside Fiat-Shamir
    // (proof_item.rs:140-145), so the order changes no outcome, and the number of indices drawn stays bounded by the proof.
    std::vector<xfe> leaves;
    std::vector<std::vector<u64>> auth;
    ps.fri_response(leaves, auth);
    if (leaves.size() != checks) fail("LdtVerificationError: IncorrectNumberOfRevealedLeaves");
    a_indices = ps.sponge.sample_indices((uint32_t)d.domain_len, checks);
    std::vector<uint32_t> idx;
    for (uint32_t a : a_indices) idx.push_back(a % (uint32_t)rounds[0].len);
    check(0, idx, leaves, auth);
    rounds[0].a = leaves;
  }
  for (size_t rnd = 0; rnd < num_rounds; rnd++) {
    const size_t n = rounds[rnd].len;
    std::vector<xfe> leaves;
    std::vector<std::vector<u64>> auth;
    ps.fri_response(leaves, auth);
    if (leaves.size() != checks) fail("LdtVerificationError: IncorrectNumberOfRevealedLeaves");
    std::vector<uint32_t> idx;
    for (uint32_t a : a_indices) idx.push_back((uint32_t)((a + n / 2) % n));
    check(rnd, idx, leaves, auth);
    rounds[rnd].b = leaves;
  }
  for (size_t rnd = 0; rnd < num_rounds; rnd++) {   // collinearity: line through (xa, ya), (xb, yb) at the folding challenge
    Round &r = rounds[rnd];
    const size_t n = r.len;
    const u64 g = root_of_unity_mont(ilog2z(n));
    std::vector<xfe> folded;
    for (size_t i = 0; i < a_indices.size(); i++) {
      const size_t ia = a_indices[i] % n, ib = (a_indices[i] + n / 2) % n;
      const u64 xa = fmul(r.offset, fpow(g, ia)), xb = fmul(r.offset, fpow(g, ib));
      const xfe ya = r.a[i], yb = r.b[i];
      const xfe slope = xscale(xsub(yb, ya), finv(fsub(xb, xa)));
      folded.push_back(xadd(ya, xmul(slope, xsubb(r.chal, xa))));
    }
    rounds[rnd + 1].a = folded;
  }
  {   // the last codeword's Merkle root
    size_t nl = last_codeword.size();
    std::vector<std::vector<u64>> level;
    for (xfe v : last_codeword) level.push_back(xfe_leaf(v));
    while (level.size() > 1) {
      std::vector<std::vector<u64>> up(level.size() / 2, std::vector<u64>(5));
      for (size_t i = 0; i < up.size(); i++) tip5_hash_pair_host(level[2 * i].data(), level[2 * i + 1].data(), up[i].data());
      level.swap(up);
    }
    if (nl == 0 || level[0] != rounds.back().root) fail("LdtVerificationError: BadMerkleRootForLastCodeword");
    for (size_t i = 0; i < a_indices.size(); i++)
      if (!xeq(last_codeword[a_indices[i] % nl], rounds.back().a[i])) fail("LdtVerificationError: LastCodewordMismatch");
  }
  if (!last_poly.empty() && last_poly.size() - 1 > d.last_round_max_degree) fail("LdtVerificationError: LastRoundPolynomialHasTooHighDegree");
  const xfe x = ps.sponge.sample_scalars(1)[0];
  if (!xeq(xpoly_eval(last_poly, x), barycentric_evaluate(last_codeword, x))) fail("LdtVerificationError: LastRoundPolynomialEvaluationMismatch");
  return {a_indices, rounds[0].a};
}

LdtResult stir_verify(Transcript &ps, const StarkDerived &d);   // below

// ---- Verifier::verify ---------------------------------------------------------------------------------------------------
void stark_verify(const StarkParams &sp, const ClaimView &claim, const u64 *proof, size_t proof_len, bool check_air) {
  Transcript ps(proof, proof_len);
  ps.sponge.pad_and_absorb_all(encode_claim(claim.program_digest, claim.version, claim.input, claim.num_input, claim.output, claim.num_output));
  const Item &lp = ps.dequeue(ItemKind::Log2PaddedHeight, "UnexpectedItem: Log2PaddedHeight");
  if (lp.payload_len() != 1) fail("ProofDecodingError: Log2PaddedHeight");
  if (lp.payload()[0] >= 32) fail("VerificationError: Log2PaddedHeightTooLarge");
  StarkDerived d;
  if (stark_derive(sp, (size_t)1 << lp.payload()[0], d) != 0) fail("VerificationError: LdtParameterError");
  const size_t N = d.ldt_len, n = d.trace_len;
  if (N == 0 || N > ((size_t)1 << 31)) fail("VerificationError: LdtParameterError");   // indices are sampled as u32 below N
  const unsigned height = ilog2z(N);

  const std::vector<u64> main_root = ps.digest();
  // challenges.rs:88-135: 59 sampled, 4 derived from the claim
  std::vector<xfe> ch = ps.sponge.sample_scalars(59);
  {
    auto terminal = [&](const u64 *symbols_canon, size_t count, xfe challenge) {   // EvalArg::compute_terminal
      xfe acc = xone();
      for (size_t i = 0; i < count; i++) acc = xaddb(xmul(challenge, acc), to_mont(symbols_canon[i]));
      return acc;
    };
    std::vector<u64> lookup(256);
    for (int i = 0; i < 256; i++) lookup[i] = TIP5_LOOKUP_HOST[i];
    const xfe compressed_digest = terminal(claim.program_digest, 5, ch[0]);
    const xfe input_terminal = terminal(claim.input, claim.num_input, ch[1]);
    const xfe output_terminal = terminal(claim.output, claim.num_output, ch[2]);
    const xfe lookup_terminal = terminal(lookup.data(), 256, ch[54]);
    ch.push_back(input_terminal); ch.push_back(output_terminal); ch.push_back(lookup_terminal); ch.push_back(compressed_digest);
  }
  const std::vector<u64> aux_root = ps.digest();
  const xfe w0 = ps.sponge.sample_scalars(1)[0];
  const std::vector<u64> quot_root = ps.digest();
  const u64 omega = root_of_unity_mont(ilog2z(n));
  const xfe alpha = ps.sponge.sample_scalars(1)[0];
  const xfe alpha_next = xscale(alpha, omega);
  const xfe alpha_zeta = xscale(alpha, to_mont(ZETA));
  const xfe alpha_pow = xpow(alpha, NUM_QUOTIENT_SEGMENTS), alpha_zeta_pow = xpow(alpha_zeta, NUM_QUOTIENT_SEGMENTS);
  const std::vector<xfe> ood_main = ps.fixed_xfes(ItemKind::OutOfDomainMainRow, NM, "UnexpectedItem: OutOfDomainMainRow");
  const std::vector<xfe> ood_aux = ps.fixed_xfes(ItemKind::OutOfDomainAuxRow, NA, "UnexpectedItem: OutOfDomainAuxRow");
  const std::vector<xfe> ood_main_next = ps.fixed_xfes(ItemKind::OutOfDomainMainRow, NM, "UnexpectedItem: OutOfDomainMainRow");
  const std::vector<xfe> ood_aux_next = ps.fixed_xfes(ItemKind::OutOfDomainAuxRow, NA, "UnexpectedItem: OutOfDomainAuxRow");
  const std::vector<xfe> ood_p = ps.fixed_xfes(ItemKind::OutOfDomainQuotientSegments, NUM_QUOTIENT_SEGMENTS, "UnexpectedItem: OutOfDomainQuotientSegments");
  const std::vector<xfe> ood_r = ps.fixed_xfes(ItemKind::OutOfDomainQuotientSegments, NUM_QUOTIENT_SEGMENTS, "UnexpectedItem: OutOfDomainQuotientSegments");

  if (check_air) {   // stark.rs:1469-1540
    const int total = AIR_VERIFY_NUM_CONSTRAINTS[0] + AIR_VERIFY_NUM_CONSTRAINTS[1] + AIR_VERIFY_NUM_CONSTRAINTS[2] + AIR_VERIFY_NUM_CONSTRAINTS[3];
    std::vector<xfe> weights = xpows(w0, total), vals(total);
    air_verify_init(ood_main.data(), ood_aux.data(), ood_main_next.data(), ood_aux_next.data(), ch.data(), vals.data());
    air_verify_cons(ood_main.data(), ood_aux.data(), ood_main_next.data(), ood_aux_next.data(), ch.data(), vals.data() + AIR_VERIFY_NUM_CONSTRAINTS[0]);
    air_verify_tran(ood_main.data(), ood_aux.data(), ood_main_next.data(), ood_aux_next.data(), ch.data(),
                    vals.data() + AIR_VERIFY_NUM_CONSTRAINTS[0] + AIR_VERIFY_NUM_CONSTRAINTS[1]);
    air_verify_term(ood_main.data(), ood_aux.data(), ood_main_next.data(), ood_aux_next.data(), ch.data(),
                    vals.data() + AIR_VERIFY_NUM_CONSTRAINTS[0] + AIR_VERIFY_NUM_CONSTRAINTS[1] + AIR_VERIFY_NUM_CONSTRAINTS[2]);
    const xfe zi = xinv(xsubb(alpha, MONT_ONE));
    const xfe zc = xinv(xsubb(xpow(alpha, n), MONT_ONE));
    const xfe except_last = xsubb(alpha, finv(omega));
    const xfe zinv[4] = {zi, zc, xmul(except_last, zc), xinv(except_last)};
    xfe sum = xzero();
    int k = 0;
    for (int cat = 0; cat < 4; cat++)
      for (int j = 0; j < AIR_VERIFY_NUM_CONSTRAINTS[cat]; j++, k++) sum = xadd(sum, xmul(weights[k], xmul(vals[k], zinv[cat])));
    xfe lhs = xzero();
    for (int i = 0; i < NUM_QUOTIENT_SEGMENTS; i++) lhs = xadd(lhs, xmul(xpow(alpha, i), ood_p[i]));
    for (int i = 0; i < NUM_QUOTIENT_SEGMENTS; i++) lhs = xadd(lhs, xmul(xpow(alpha_zeta, i), ood_r[i]));
    if (!xeq(sum, lhs)) fail("VerificationError: OutOfDomainQuotientValueMismatch");
  }

  const std::vector<xfe> w3 = ps.sponge.sample_scalars(3);
  const std::vector<xfe> w_main_aux = xpows(w3[0], NM + NA), w_quot = xpows(w3[1], NUM_RANDOMIZED_QUOTIENT_SEGMENTS),
                         w_deep = xpows(w3[2], NUM_DEEP_CODEWORD_COMPONENTS);
  auto lin_x = [&](const std::vector<xfe> &m, const std::vector<xfe> &a) {
    xfe acc = xzero();
    for (size_t i = 0; i < NM; i++) acc = xadd(acc, xmul(w_main_aux[i], m[i]));
    for (size_t i = 0; i < NA; i++) acc = xadd(acc, xmul(w_main_aux[NM + i], a[i]));
    return acc;
  };
  const xfe ood_curr_value = lin_x(ood_main, ood_aux), ood_next_value = lin_x(ood_main_next, ood_aux_next);
  xfe ood_p_value = xzero(), ood_r_value = xzero();
  for (int i = 0; i < NUM_QUOTIENT_SEGMENTS; i++) {
    ood_p_value = xadd(ood_p_value, xmul(ood_p[i], w_quot[i]));
    ood_r_value = xadd(ood_r_value, xmul(ood_r[i], w_quot[i + 1]));
  }

  LdtResult ldt = d.ldt == 2 ? stir_verify(ps, d) : fri_verify(ps, d.fri);
  const size_t q = d.num_first_round_queries;
  if (ldt.indices.size() != q || ldt.values.size() != q) fail("VerificationError: IncorrectNumberOfRowIndices");

  auto open = [&](ItemKind kind, size_t width, const std::vector<u64> &root, const char *unexpected, const char *count_error,
                  const char *auth_error) {
    std::vector<const u64 *> rows = ps.rows(kind, width, unexpected);
    std::vector<std::vector<u64>> auth = ps.auth_structure();
    if (rows.size() != q) fail(count_error);
    std::vector<std::vector<u64>> leafs;
    for (const u64 *r : rows) leafs.push_back(hash_row(r, width));
    if (!verify_inclusion(root, height, ldt.indices, leafs, auth)) fail(auth_error);
    return rows;
  };
  const auto main_rows = open(ItemKind::MasterMainTableRows, NM, main_root, "UnexpectedItem: MasterMainTableRows",
                              "VerificationError: IncorrectNumberOfMainTableRows", "VerificationError: MainCodewordAuthenticationFailure");
  const auto aux_rows = open(ItemKind::MasterAuxTableRows, 3 * NA, aux_root, "UnexpectedItem: MasterAuxTableRows",
                             "VerificationError: IncorrectNumberOfAuxTableRows", "VerificationError: AuxiliaryCodewordAuthenticationFailure");
  const auto quot_rows = open(ItemKind::QuotientSegmentsElements, 3 * NUM_RANDOMIZED_QUOTIENT_SEGMENTS, quot_root,
                              "UnexpectedItem: QuotientSegmentsElements", "VerificationError: IncorrectNumberOfQuotientSegmentElements",
                              "VerificationError: QuotientCodewordAuthenticationFailure");

  const u64 g = root_of_unity_mont(height), off = to_mont(d.ldt_offset);
  for (size_t k = 0; k < q; k++) {   // stark.rs:1673-1745
    const u64 x = fmul(off, fpow(g, ldt.indices[k]));
    xfe ma = xzero();
    for (size_t i = 0; i < NM; i++) ma = xadd(ma, xmulb(w_main_aux[i], to_mont(main_rows[k][i])));
    for (size_t i = 0; i < NA; i++) ma = xadd(ma, xmul(w_main_aux[NM + i], xm(aux_rows[k] + 3 * i)));
    xfe qe[NUM_RANDOMIZED_QUOTIENT_SEGMENTS];
    for (int i = 0; i < NUM_RANDOMIZED_QUOTIENT_SEGMENTS; i++) qe[i] = xm(quot_rows[k] + 3 * i);
    xfe shared = xzero();
    for (int i = 1; i + 1 < NUM_RANDOMIZED_QUOTIENT_SEGMENTS; i++) shared = xadd(shared, xmul(qe[i], w_quot[i]));
    const xfe for_p = xadd(xmul(w_quot[0], qe[0]), shared);
    const xfe for_r = xadd(xmul(w_quot[NUM_RANDOMIZED_QUOTIENT_SEGMENTS - 1], qe[NUM_RANDOMIZED_QUOTIENT_SEGMENTS - 1]), shared);
    auto deep = [&](xfe value, xfe point, xfe ood_value) { return xmul(xsub(value, ood_value), xinv(xsub(xlift(x), point))); };
    const xfe comps[4] = {deep(ma, alpha, ood_curr_value), deep(ma, alpha_next, ood_next_value), deep(for_p, alpha_pow, ood_p_value),
                          deep(for_r, alpha_zeta_pow, ood_r_value)};
    xfe acc = xzero();
    for (int i = 0; i < 4; i++) acc = xadd(acc, xmul(comps[i], w_deep[i]));
    if (!xeq(acc, ldt.values[k])) fail("VerificationError: CombinationCodewordMismatch");
  }
  if (ps.index != ps.items.size()) fail("VerificationError: SuperfluousProofItems");
}

// ---- STIR verifier (low_degree_test/stir.rs:995-1370; oracle/stir.py::verify) ---------------------------------------------
typedef std::vector<xfe> XPoly;   // little-endian coefficients
xfe peval(const XPoly &c, xfe x) { return xpoly_eval(c, x); }
XPoly zerofier(const std::vector<xfe> &points) {   // Polynomial::zerofier
  XPoly z{xone()};
  for (xfe p : points) {
    XPoly nz(z.size() + 1, xzero());
    for (size_t i = 0; i < z.size(); i++) {
      nz[i + 1] = xadd(nz[i + 1], z[i]);
      nz[i] = xsub(nz[i], xmul(z[i], p));
    }
    z.swap(nz);
  }
  return z;
}
XPoly interpolate(const std::vector<xfe> &xs, const std::vector<xfe> &ys) {   // Polynomial::interpolate, Lagrange form
  const XPoly z = zerofier(xs);
  XPoly out(xs.size(), xzero());
  for (size_t i = 0; i < xs.size(); i++) {
    XPoly q(z.size() - 1, xzero());   // z / (X - x_i) by synthetic division
    xfe acc = xzero();
    for (size_t k = z.size() - 1; k >= 1; k--) {
      acc = xadd(z[k], xmul(acc, xs[i]));
      q[k - 1] = acc;
    }
    const xfe scale = xmul(ys[i], xinv(peval(q, xs[i])));
    for (size_t k = 0; k < q.size(); k++) out[k] = xadd(out[k], xmul(scale, q[k]));
  }
  return out;
}
// value at x of the interpolant through (point_j, value_j), point_j = root * kth^j (Polynomial::fast_coset_interpolate + evaluate)
xfe coset_interpolate_evaluate(u64 root, u64 kth, const std::vector<xfe> &values, xfe x) {
  const size_t k = values.size();
  std::vector<u64> pts(k);
  u64 cur = root;
  for (size_t j = 0; j < k; j++) { pts[j] = cur; cur = fmul(cur, kth); }
  xfe acc = xzero();
  for (size_t j = 0; j < k; j++) {
    xfe num = xone();
    u64 den = MONT_ONE;
    for (size_t m = 0; m < k; m++) {
      if (m == j) continue;
      num = xmul(num, xsubb(x, pts[m]));
      den = fmul(den, fsub(pts[j], pts[m]));
    }
    acc = xadd(acc, xmul(values[j], xscale(num, finv(den))));
  }
  return acc;
}

struct StirQuery {
  uint32_t index, fidx;
  u64 point, root, kth;                 // Montgomery
  const std::vector<xfe> *values;       // the revealed stack: evaluations in the k-th roots of `point`
};

LdtResult stir_verify(Transcript &ps, const StarkDerived &d) {
  const StirDerived &sp = d.stir;
  const size_t ff = sp.folding_factor;
  u64 offset = to_mont(d.ldt_offset);
  size_t length = d.ldt_len;
  std::vector<u64> prev_root = ps.digest();
  LdtResult first;
  bool have_first = false, have_quotient = false;
  std::vector<xfe> quotient_set, quotient_answers;
  xfe dcr = xzero();
  std::vector<std::vector<xfe>> leafs;   // storage the queries point into

  auto extract = [&](size_t num_queries, std::vector<StirQuery> &queries, std::vector<std::vector<u64>> &auth, size_t &f_len) {
    std::vector<uint32_t> queried = ps.sponge.sample_indices((uint32_t)length, num_queries);
    ps.stir_response(leafs, auth);
    f_len = length / ff;
    const u64 f_off = fpow(offset, ff);
    std::vector<uint32_t> folded_idx;   // unique, first-occurrence order
    for (uint32_t i : queried) {
      const uint32_t fi = (uint32_t)(i % f_len);
      if (std::find(folded_idx.begin(), folded_idx.end(), fi) == folded_idx.end()) folded_idx.push_back(fi);
    }
    if (leafs.size() != folded_idx.size()) fail("LdtVerificationError: IncorrectNumberOfRevealedLeaves");
    for (const auto &l : leafs)
      if (l.size() != ff) fail("LdtVerificationError: IncorrectNumberOfRevealedLeaves");
    const u64 g = root_of_unity_mont(ilog2z(length)), gf = root_of_unity_mont(ilog2z(f_len));
    const u64 kth = fpow(g, f_len);
    queries.clear();
    for (uint32_t index : queried) {
      const uint32_t qi = (uint32_t)(index % f_len);
      const size_t slot = std::find(folded_idx.begin(), folded_idx.end(), qi) - folded_idx.begin();
      queries.push_back(StirQuery{index, qi, fmul(f_off, fpow(gf, qi)), fmul(offset, fpow(g, qi)), kth, &leafs[slot]});
    }
  };
  auto authenticate = [&](const std::vector<StirQuery> &queries, const std::vector<std::vector<u64>> &auth, size_t f_len,
                          const std::vector<u64> &root) {
    std::map<uint32_t, std::vector<u64>> indexed;   // ascending folded index
    for (const StirQuery &q : queries) {
      std::vector<u64> words;
      for (xfe v : *q.values) { words.push_back(v.c0); words.push_back(v.c1); words.push_back(v.c2); }
      std::vector<u64> dg(5);
      tip5_hash_varlen_host(words.data(), words.size(), dg.data());
      indexed[q.fidx] = dg;
    }
    std::vector<uint32_t> idx;
    std::vector<std::vector<u64>> lf;
    for (auto &kv : indexed) { idx.push_back(kv.first); lf.push_back(kv.second); }
    if (!verify_inclusion(root, ilog2z(f_len), idx, lf, auth)) fail("LdtVerificationError: BadMerkleAuthenticationPath");
  };
  auto answers = [&](const std::vector<StirQuery> &queries, xfe r) {
    std::vector<xfe> out;
    if (!have_quotient) {
      for (const StirQuery &q : queries) out.push_back(coset_interpolate_evaluate(q.root, q.kth, *q.values, r));
      return out;
    }
    const XPoly ans = interpolate(quotient_set, quotient_answers), zf = zerofier(quotient_set);
    const u64 degree_difference = quotient_set.size() + 1;
    for (const StirQuery &q : queries) {
      u64 cur = q.root;
      std::vector<xfe> evals;
      for (xfe ev : *q.values) {
        const xfe xc = xlift(cur);
        const xfe quot = xmul(xsub(ev, peval(ans, xc)), xinv(peval(zf, xc)));
        const xfe common = xscale(dcr, cur);
        xfe dcf;
        if (xeq(common, xone())) dcf = xlift(to_mont(degree_difference));
        else dcf = xmul(xsub(xone(), xpow(common, degree_difference)), xinv(xsub(xone(), common)));
        evals.push_back(xmul(dcf, quot));
        cur = fmul(cur, q.kth);
      }
      out.push_back(coset_interpolate_evaluate(q.root, q.kth, evals, r));
    }
    return out;
  };
  auto remember_first = [&](const std::vector<StirQuery> &queries, size_t f_len) {
    if (have_first) return;
    have_first = true;
    for (const StirQuery &q : queries) {
      first.indices.push_back(q.index);
      first.values.push_back((*q.values)[q.index / f_len]);
    }
  };

  for (int round = 0; round < sp.num_rounds; round++) {
    const xfe r = ps.sponge.sample_scalars(1)[0];
    const std::vector<u64> cur_root = ps.digest();
    const std::vector<xfe> ood_queries = ps.sponge.sample_scalars(sp.out_of_domain[round]);
    const std::vector<xfe> ood_answers = ps.xfe_vector(ItemKind::StirOutOfDomainValues, "UnexpectedItem: StirOutOfDomainValues");
    if (ood_answers.size() != ood_queries.size()) fail("LdtVerificationError: IncorrectNumberOfOutOfDomainValues");
    std::vector<StirQuery> queries;
    std::vector<std::vector<u64>> auth;
    size_t f_len;
    extract(sp.in_domain[round], queries, auth, f_len);
    authenticate(queries, auth, f_len, prev_root);
    remember_first(queries, f_len);
    const std::vector<xfe> ans = answers(queries, r);
    std::vector<xfe> qs, qa;   // de-duplicated by point, first occurrence wins
    auto add = [&](xfe pt, xfe a) {
      for (xfe s : qs)
        if (xeq(s, pt)) return;
      qs.push_back(pt);
      qa.push_back(a);
    };
    for (size_t i = 0; i < queries.size(); i++) add(xlift(queries[i].point), ans[i]);
    for (size_t i = 0; i < ood_queries.size(); i++) add(ood_queries[i], ood_answers[i]);
    dcr = ps.sponge.sample_scalars(1)[0];
    quotient_set = qs;
    quotient_answers = qa;
    have_quotient = true;
    offset = fmul(fmul(offset, offset), offset);   // stir.rs:1149-1155: pow(2), then times the old offset
    length /= 2;
    prev_root = cur_root;
  }
  const xfe r = ps.sponge.sample_scalars(1)[0];
  const XPoly poly = ps.polynomial();
  if (!poly.empty() && poly.size() - 1 > sp.final_degree) fail("LdtVerificationError: LastRoundPolynomialHasTooHighDegree");
  std::vector<StirQuery> queries;
  std::vector<std::vector<u64>> auth;
  size_t f_len;
  extract(sp.final_num_in_domain_queries, queries, auth, f_len);
  authenticate(queries, auth, f_len, prev_root);
  const std::vector<xfe> final_answers = answers(queries, r);
  for (size_t i = 0; i < queries.size(); i++)
    if (!xeq(peval(poly, xlift(queries[i].point)), final_answers[i])) fail("LdtVerificationError: LastRoundPolynomialEvaluationMismatch");
  remember_first(queries, f_len);
  return first;
}

}  // namespace
}  // namespace tvm

// Stir::verify as a stand-alone low-degree test (stir.rs:995-1108) for arbitrary StirParameters
extern "C" int tvm_stir_verify_k(uint32_t security_level, uint32_t soundness, uint32_t log2_folding_factor,
                                 uint32_t log2_initial_expansion_factor, uint32_t log2_high_degree_bound, const uint64_t *proof,
                                 size_t proof_len, uint32_t *indices_out, uint64_t *values_out, size_t *num_indices, char *failure,
                                 size_t failure_capacity) {
  using namespace tvm;
  set_failure(failure, failure_capacity, "");
  if (!proof || !proof_len || soundness > 1) return TVM_ERR_INVALID_ARG;
  StarkDerived d{};
  const char *why = "";
  if (int rc = stir_derive(security_level, log2_folding_factor, log2_initial_expansion_factor, log2_high_degree_bound, soundness == 1, d.stir,
                           &why)) {
    set_failure(failure, failure_capacity, why);
    return rc;
  }
  d.ldt = 2;
  d.ldt_len = (size_t)1 << (log2_high_degree_bound + log2_initial_expansion_factor);
  d.ldt_offset = 7;                                   // BFieldElement::generator(), stir.rs:589
  try {
    Transcript ps(proof, proof_len);
    LdtResult r = stir_verify(ps, d);
    if (ps.index != ps.items.size()) fail("VerificationError: SuperfluousProofItems");
    const size_t cap = num_indices ? *num_indices : 0;
    if (num_indices) *num_indices = r.indices.size();
    if (indices_out || values_out) {
      if (cap < r.indices.size()) return TVM_ERR_INVALID_ARG;
      for (size_t i = 0; i < r.indices.size(); i++) {
        if (indices_out) indices_out[i] = r.indices[i];
        if (values_out) { values_out[3 * i] = from_mont(r.values[i].c0); values_out[3 * i + 1] = from_mont(r.values[i].c1); values_out[3 * i + 2] = from_mont(r.values[i].c2); }
      }
    }
    return TVM_OK;
  } catch (const VerifyFailure &f) {
    set_failure(failure, failure_capacity, f.what);
    return TVM_ERR_VERIFICATION;
  } catch (const std::exception &e) {
    set_failure(failure, failure_capacity, e.what());
    return TVM_ERR_VERIFICATION;
  } catch (...) {
    set_failure(failure, failure_capacity, "internal error");
    return TVM_ERR_VERIFICATION;
  }
}

extern "C" int tvm_stir_verify(uint32_t security_level, uint32_t soundness, uint32_t log2_initial_expansion_factor,
                               uint32_t log2_high_degree_bound, const uint64_t *proof, size_t proof_len, uint32_t *indices_out,
                               uint64_t *values_out, size_t *num_indices, char *failure, size_t failure_capacity) {
  return tvm_stir_verify_k(security_level, soundness, tvm::STIR_LOG2_FOLDING_FACTOR, log2_initial_expansion_factor, log2_high_degree_bound,
                           proof, proof_len, indices_out, values_out, num_indices, failure, failure_capacity);
}

// Fri::verify as a stand-alone low-degree test (fri.rs:774-789) for arbitrary FriParameters: the fri_verify of tvm_verify
extern "C" int tvm_fri_verify(uint32_t security_level, uint32_t soundness, uint32_t log2_initial_expansion_factor,
                              uint32_t log2_high_degree_bound, const uint64_t *proof, size_t proof_len, uint32_t *indices_out,
                              uint64_t *values_out, size_t *num_indices, char *failure, size_t failure_capacity) {
  using namespace tvm;
  set_failure(failure, failure_capacity, "");
  if (!proof || !proof_len || soundness > 1) return TVM_ERR_INVALID_ARG;
  FriDerived d{};
  const char *why = "";
  if (int rc = fri_derive(security_level, soundness == 1, log2_initial_expansion_factor, log2_high_degree_bound, d, &why)) {
    set_failure(failure, failure_capacity, why);
    return rc;
  }
  if (d.domain_len > ((size_t)1 << 31)) {   // ProofStream::sample_indices takes upper bounds up to u32::MAX (proof_stream.rs:85-89)
    set_failure(failure, failure_capacity, "ProofStream::sample_indices: upper bound exceeds u32::MAX");
    return TVM_ERR_DOMAIN;
  }
  try {
    Transcript ps(proof, proof_len);
    LdtResult r = fri_verify(ps, d);
    if (ps.index != ps.items.size()) fail("VerificationError: SuperfluousProofItems");
    const size_t cap = num_indices ? *num_indices : 0;
    if (num_indices) *num_indices = r.indices.size();
    if (indices_out || values_out) {
      if (cap < r.indices.size()) return TVM_ERR_INVALID_ARG;
      for (size_t i = 0; i < r.indices.size(); i++) {
        if (indices_out) indices_out[i] = r.indices[i];
        if (values_out) { values_out[3 * i] = from_mont(r.values[i].c0); values_out[3 * i + 1] = from_mont(r.values[i].c1); values_out[3 * i + 2] = from_mont(r.values[i].c2); }
      }
    }
    return TVM_OK;
  } catch (const VerifyFailure &f) {
    set_failure(failure, failure_capacity, f.what);
    return TVM_ERR_VERIFICATION;
  } catch (const std::exception &e) {
    set_failure(failure, failure_capacity, e.what());
    return TVM_ERR_VERIFICATION;
  } catch (...) {
    set_failure(failure, failure_capacity, "internal error");
    return TVM_ERR_VERIFICATION;
  }
}

// Proof::padded_height (proof.rs:37-56): the one Log2PaddedHeight item of the proof stream
extern "C" int tvm_proof_padded_height(const uint64_t *proof, size_t proof_len, uint64_t *padded_height) {
  using namespace tvm;
  if (!proof || !proof_len || !padded_height) return TVM_ERR_INVALID_ARG;
  try {
    Transcript ps(proof, proof_len);
    int found = 0;
    for (const Item &it : ps.items)
      if (it.kind == (int)ItemKind::Log2PaddedHeight) {
        if (it.payload_len() != 1 || it.payload()[0] >= 64) return TVM_ERR_VERIFICATION;
        *padded_height = (uint64_t)1 << it.payload()[0];
        found++;
      }
    return found == 1 ? TVM_OK : TVM_ERR_VERIFICATION;   // NoLog2PaddedHeight / TooManyLog2PaddedHeights
  } catch (...) {
    return TVM_ERR_VERIFICATION;
  }
}

extern "C" int tvm_verify(const tvm_params *params, const tvm_claim *claim, const uint64_t *proof, size_t proof_len, int skip_air_check,
                          char *failure, size_t failure_capacity) {
  using namespace tvm;
  set_failure(failure, failure_capacity, "");
  if (!params || !claim || !proof || !proof_len || params->ldt_choice > 2 || !claim_ok(claim)) return TVM_ERR_INVALID_ARG;
  try {
    stark_verify(stark_params(*params), claim_view(*claim), proof, proof_len, !skip_air_check);
    return TVM_OK;
  } catch (const VerifyFailure &f) {
    set_failure(failure, failure_capacity, f.what);
    return TVM_ERR_VERIFICATION;
  } catch (const std::exception &e) {
    set_failure(failure, failure_capacity, e.what());
    return TVM_ERR_VERIFICATION;
  } catch (...) {
    set_failure(failure, failure_capacity, "internal error");
    return TVM_ERR_VERIFICATION;
  }
}

// Many proofs at once: proofs are independent, so the batch is spread over host threads (0 = one per hardware thread).
// results[i] receives what tvm_verify would return for proof i; the return value is TVM_OK iff every proof is accepted.
extern "C" int tvm_verify_batch(const tvm_params *params, const tvm_claim *claims, const uint64_t *const *proofs, const size_t *proof_lens,
                                size_t count, int skip_air_check, unsigned num_threads, int *results) {
  if (!params || (count && (!claims || !proofs || !proof_lens || !results))) return TVM_ERR_INVALID_ARG;
  if (!num_threads) num_threads = std::max(1u, std::thread::hardware_concurrency());
  num_threads = (unsigned)std::min<size_t>(num_threads, std::max<size_t>(count, 1));
  std::atomic<size_t> next{0};
  auto worker = [&]() {
    for (size_t i = next++; i < count; i = next++)
      results[i] = tvm_verify(params, &claims[i], proofs[i], proof_lens[i], skip_air_check, nullptr, 0);
  };
  std::vector<std::thread> pool;
  try {
    for (unsigned t = 1; t < num_threads; t++) pool.emplace_back(worker);
  } catch (...) {
    // std::system_error (no more threads): the threads already started plus this one finish the batch
  }
  worker();
  for (auto &th : pool) th.join();
  int rc = TVM_OK;
  for (size_t i = 0; i < count; i++)
    if (results[i] != TVM_OK) rc = results[i] == TVM_ERR_VERIFICATION && rc != TVM_ERR_INVALID_ARG ? TVM_ERR_VERIFICATION : TVM_ERR_INVALID_ARG;
  return rc;
}
