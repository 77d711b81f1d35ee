// STIR low-degree test, prover side, on the device-resident combination codeword.
//
// Restates Stir::prove (triton-vm/src/low_degree_test/stir.rs:885-993) with its helpers
// fold_polynomial (1132-1147), next_round_domain (1149-1155) and StirMerkleTree (1374-1433).
// The reference keeps the round polynomial in coefficient form and does the quotienting
//   poly' = (folded - Ans) / Zerofier * DegreeCorrection                 (stir.rs:950-966)
// with dense polynomial arithmetic.  Here the same polynomial is obtained in evaluation form on
// the next round's domain (whose points are disjoint from the quotient set: in-domain queries
// live in offset^k<g^k>, the next domain is offset^3<g^2>, offset = 7^(3^t), and offset^(k-3)
// is outside the 2-power subgroup for every k < 2^30; out-of-domain queries are X-field elements)
// followed by one inverse NTT — exact field arithmetic, hence the identical polynomial.  Ans and
// Zerofier (degree ~200) are interpolated on the host and evaluated on the domain by zero-padded NTTs.
// The folding factor k is any power of 2 from 4 on: k = 4 (Stark::ldt's) folds with one thread per
// output, larger factors with one quad per output; a stacked leaf is 3k base-field words.
//
// Layout: X-field vectors are 3 planes; every buffer of a round is packed [3][len].
#include <algorithm>
#include "prove_common.h"
#include "transcript.h"

namespace tvm {
namespace {

constexpr int ST_THREADS = 256;
inline unsigned st_grid(size_t n) { return (unsigned)((n + ST_THREADS - 1) / ST_THREADS); }
__device__ __forceinline__ u64 pt_get(const PowTab &t, u64 e) {
  return fmul(__ldg(t.lo + (e & ((1ULL << t.shift) - 1))), __ldg(t.hi + (e >> t.shift)));
}
int ilog2s(size_t x) { int l = 0; while (((size_t)1 << (l + 1)) <= x) l++; return l; }

// StirMerkleTree::stack (stir.rs:1407-1419): leaf i = [cw[i], cw[i + L/h], ..., cw[i + (h-1) L/h]];
// out is the [3h][L/h] column table whose row i is bfe_slice(leaf i) (x0.c0, x0.c1, x0.c2, x1.c0, ...).
__global__ void stir_stack_kernel(const u64 *cw, size_t len, unsigned h, u64 *out) {
  size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;   // over 3*len
  if (t >= 3 * len) return;
  size_t d = t / len, j = t - d * len;
  size_t lq = len / h, s = j / lq, i = j - s * lq;
  out[(3 * s + d) * lq + i] = cw[t];
}
// fold_polynomial: out_j = sum_{i<4} c_{4j+i} r^i   (stir.rs:1132-1147, folding factor 4, the factor Stark::ldt uses)
__global__ void stir_fold_kernel(const u64 *in, size_t in_len, xfe r1, xfe r2, xfe r3, u64 *out, size_t out_len) {
  size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= out_len) return;
  xfe acc = xzero();
  const xfe rp[4] = {xone(), r1, r2, r3};
#pragma unroll
  for (int i = 0; i < 4; i++) {
    size_t k = 4 * j + i;
    if (k < in_len) acc = xadd(acc, xmul(xmake(in[k], in[in_len + k], in[2 * in_len + k]), rp[i]));
  }
  out[j] = acc.c0; out[out_len + j] = acc.c1; out[2 * out_len + j] = acc.c2;
}
// fold_polynomial for k = 2^log_k >= 8: out_j = sum_{i<k} c_{kj+i} r^i over in[3][k * out_len].  The four lanes of a quad
// share one output: lane l reads the coefficients kj + l + 4m (m < k/4), so each load instruction of a warp reads eight whole
// 32-byte sectors of a plane.  A lane folds its k/4 coefficients by Horner in r^4 and scales the sum by r^l; two butterfly
// shuffles add up the quad.
__global__ void stir_fold_quad_kernel(const u64 *in, size_t in_len, unsigned log_k, xfe r1, xfe r2, xfe r3, xfe r4, u64 *out,
                                      size_t out_len) {
  const size_t j = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 2;
  const unsigned l = threadIdx.x & 3;
  xfe h = xzero();
  if (j < out_len) {            // no early return: every lane of the warp takes part in the shuffles
    const size_t base = (j << log_k) + l;
#pragma unroll 4
    for (size_t m = (size_t)1 << (log_k - 2); m-- > 0;) {
      const size_t i = base + 4 * m;
      h = xadd(xmul(h, r4), xmake(in[i], in[in_len + i], in[2 * in_len + i]));
    }
    if (l) h = xmul(h, l == 1 ? r1 : l == 2 ? r2 : r3);
  }
#pragma unroll
  for (int off = 1; off < 4; off <<= 1)
    h = xadd(h, xmake(__shfl_xor_sync(0xffffffffu, h.c0, off), __shfl_xor_sync(0xffffffffu, h.c1, off),
                      __shfl_xor_sync(0xffffffffu, h.c2, off)));
  if (l == 0 && j < out_len) { out[j] = h.c0; out[out_len + j] = h.c1; out[2 * out_len + j] = h.c2; }
}
// out[d][j] = j < in_len ? in[d][j] * s^j : 0   for j < out_len  (coset pre-scaling + zero padding before an NTT)
__global__ void stir_scale_pad_kernel(const u64 *in, size_t in_len, PowTab s, u64 *out, size_t out_len) {
  size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= out_len) return;
  if (j < in_len) {
    u64 f = pt_get(s, j);
    for (int d = 0; d < 3; d++) out[d * out_len + j] = fmul(in[d * in_len + j], f);
  } else {
    for (int d = 0; d < 3; d++) out[d * out_len + j] = 0;
  }
}
// values of the next round's polynomial on the next domain (stir.rs:950-966):
//   q(x) = (F(x) - A(x)) / Z(x) * sum_{i=0}^{m} (rho x)^i,   x = offset * g^j
__global__ void stir_quotient_kernel(const u64 *F, const u64 *A, const u64 *Z, size_t len, u64 offset, PowTab g, xfe rho, unsigned m_plus_1,
                                     u64 *out) {
  size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= len) return;
  u64 x = fmul(offset, pt_get(g, j));
  xfe f = xmake(F[j], F[len + j], F[2 * len + j]);
  xfe a = xmake(A[j], A[len + j], A[2 * len + j]);
  xfe z = xmake(Z[j], Z[len + j], Z[2 * len + j]);
  xfe common = xmulb(rho, x);
  xfe num = xsub(f, a);
  xfe res;
  if (xeq(common, xone())) {
    res = xmul(xmulb(num, to_mont((u64)m_plus_1)), xinv(z));
  } else {
    xfe one_minus = xsub(xone(), common);
    num = xmul(num, xsub(xone(), xpow(common, (u64)m_plus_1)));
    res = xmul(num, xinv(xmul(z, one_minus)));
  }
  out[j] = res.c0; out[len + j] = res.c1; out[2 * len + j] = res.c2;
}

// Zerofier and Lagrange interpolant of m <= blockDim.x points in one CTA (Polynomial::zerofier / ::interpolate,
// stir.rs:958-960).  pts/vals: [m][3] interleaved; Q: m*m X-field scratch (3 planes of m*m words);
// out_ans: [3][m] planar, out_z: [3][m+1] planar.
__global__ void stir_interpolate_kernel(const u64 *pts, const u64 *vals, unsigned m, u64 *Q, u64 *out_ans, u64 *out_z) {
  extern __shared__ u64 sm[];           // z[3][m+1], s[3][m]
  u64 *z = sm, *sc = sm + 3 * (m + 1);
  const unsigned t = threadIdx.x;
  const size_t mm = (size_t)m * m;
  // zerofier: multiply by (X - p_i) one point at a time; coefficient k is owned by thread k
  for (unsigned k = t; k <= m; k += blockDim.x) { z[k] = k == 0 ? MONT_ONE : 0; z[(m + 1) + k] = 0; z[2 * (m + 1) + k] = 0; }
  __syncthreads();
  for (unsigned i = 0; i < m; i++) {
    const xfe p = xmake(pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]);
    xfe nv = xzero();
    const bool mine = t <= i + 1 && t <= m;
    if (mine) {
      xfe cur = xmake(z[t], z[(m + 1) + t], z[2 * (m + 1) + t]);
      xfe prev = t ? xmake(z[t - 1], z[(m + 1) + t - 1], z[2 * (m + 1) + t - 1]) : xzero();
      nv = xsub(prev, xmul(cur, p));
    }
    __syncthreads();
    if (mine) { z[t] = nv.c0; z[(m + 1) + t] = nv.c1; z[2 * (m + 1) + t] = nv.c2; }
    __syncthreads();
  }
  for (unsigned k = t; k <= m; k += blockDim.x)
    for (int d = 0; d < 3; d++) out_z[d * (m + 1) + k] = z[d * (m + 1) + k];
  // q_i = z / (X - x_i) by synthetic division; s_i = y_i / q_i(x_i)
  if (t < m) {
    const xfe x = xmake(pts[3 * t], pts[3 * t + 1], pts[3 * t + 2]);
    xfe acc = xzero();
    for (unsigned k = m; k >= 1; k--) {
      acc = xadd(xmake(z[k], z[(m + 1) + k], z[2 * (m + 1) + k]), xmul(acc, x));
      Q[(size_t)t * m + (k - 1)] = acc.c0; Q[mm + (size_t)t * m + (k - 1)] = acc.c1; Q[2 * mm + (size_t)t * m + (k - 1)] = acc.c2;
    }
    xfe den = xzero();
    for (unsigned k = m; k-- > 0;) {
      xfe qk = xmake(Q[(size_t)t * m + k], Q[mm + (size_t)t * m + k], Q[2 * mm + (size_t)t * m + k]);
      den = xadd(xmul(den, x), qk);
    }
    xfe sv = xmul(xmake(vals[3 * t], vals[3 * t + 1], vals[3 * t + 2]), xinv(den));
    sc[t] = sv.c0; sc[m + t] = sv.c1; sc[2 * m + t] = sv.c2;
  }
  __syncthreads();
  if (t < m) {      // coefficient t of the interpolant: sum_i s_i q_i[t]
    xfe acc = xzero();
    for (unsigned i = 0; i < m; i++) {
      xfe qi = xmake(Q[(size_t)i * m + t], Q[mm + (size_t)i * m + t], Q[2 * mm + (size_t)i * m + t]);
      acc = xadd(acc, xmul(xmake(sc[i], sc[m + i], sc[2 * m + i]), qi));
    }
    out_ans[t] = acc.c0; out_ans[m + t] = acc.c1; out_ans[2 * m + t] = acc.c2;
  }
}

// ---- small host-side X-field polynomial arithmetic (Montgomery form, little-endian coefficients) ----
typedef std::vector<xfe> XPoly;
xfe xp_eval(const XPoly &c, xfe x) {
  xfe acc = xzero();
  for (size_t i = c.size(); i-- > 0;) acc = xadd(xmul(acc, x), c[i]);
  return acc;
}
XPoly xp_zerofier(const std::vector<xfe> &pts) {            // Polynomial::zerofier
  XPoly z(1, xone());
  for (const xfe &p : pts) {
    XPoly nz(z.size() + 1, xzero());
    for (size_t i = 0; i < z.size(); i++) {
      nz[i + 1] = xadd(nz[i + 1], z[i]);
      nz[i] = xsub(nz[i], xmul(z[i], p));
    }
    z.swap(nz);
  }
  return z;
}
XPoly xp_interpolate(const std::vector<xfe> &xs, const std::vector<xfe> &ys, const XPoly &z) {   // the unique interpolant (Lagrange)
  const size_t m = xs.size();
  XPoly out(m, xzero()), q(m);
  for (size_t i = 0; i < m; i++) {
    xfe acc = xzero();
    for (size_t k = m; k >= 1; k--) {        // z / (X - x_i) by synthetic division
      acc = xadd(z[k], xmul(acc, xs[i]));
      q[k - 1] = acc;
    }
    xfe s = xmul(ys[i], xinv(xp_eval(q, xs[i])));
    for (size_t k = 0; k < m; k++) out[k] = xadd(out[k], xmul(s, q[k]));
  }
  return out;
}

struct Commitment {        // StirMerkleTree: stacked leaves as a [3k][leaves] column table + the node array
  u64 *stack = nullptr, *nodes = nullptr;
  size_t leaves = 0;
};

}  // namespace

std::vector<uint32_t> stir_prove_run(Ctx &c, DevMem &mem, ProofStream &ps, const u64 *d_codeword, size_t len, u64 offset_mont,
                                     const StirDerived &sd, u64 *d_tmp) {
  const unsigned ff = (unsigned)sd.folding_factor;
  const unsigned log_ff = (unsigned)ilog2s(ff);
  if (ff < 4 || ff != 1u << log_ff || len % ff)
    throw ApiError{TVM_ERR_UNSUPPORTED, "STIR: the folding factor must be a power of 2, at least 4, dividing the domain length"};
  auto launch_check = [&](int k) { c.launches += k; TVM_CUDA(cudaGetLastError()); };
  // fold_polynomial (stir.rs:1132-1147) of d_in[3][k * out_len]
  auto fold = [&](const u64 *d_in, size_t in_len, xfe r, u64 *d_out, size_t out_len) {
    const xfe r2 = xmul(r, r), r3 = xmul(r2, r);
    if (ff == 4) {
      stir_fold_kernel<<<st_grid(out_len), ST_THREADS, 0, c.stream>>>(d_in, in_len, r, r2, r3, d_out, out_len);
    } else {
      stir_fold_quad_kernel<<<st_grid(4 * out_len), ST_THREADS, 0, c.stream>>>(d_in, in_len, log_ff, r, r2, r3, xmul(r2, r2), d_out,
                                                                               out_len);
    }
    launch_check(1);
  };

  auto commit = [&](const u64 *d_cw, size_t L) {
    Commitment cm;
    cm.leaves = L / ff;
    cm.stack = mem.words(3 * L);
    cm.nodes = mem.words(2 * cm.leaves * 5);
    stir_stack_kernel<<<st_grid(3 * L), ST_THREADS, 0, c.stream>>>(d_cw, L, ff, cm.stack);
    launch_check(1);
    TVM_CUDA(cudaMemsetAsync(cm.nodes, 0, 40, c.stream));
    const unsigned W = (unsigned)c.comm.world, rank = (unsigned)c.comm.rank;
    if (W > 1 && cm.leaves >= (size_t)4096 * W) {
      // multi-GPU: the codeword is replicated, so each rank hashes its 1/W of the stacked leaves; the leaf digests are
      // all-gathered and every rank builds the (much cheaper) tree itself: queries are answered from the complete node array
      const size_t per = cm.leaves / W;
      hash_rows_run(c, cm.stack + (size_t)rank * per, cm.leaves, per, 3 * ff, 0, cm.nodes + 5 * (cm.leaves + (size_t)rank * per));
      c.all_gather(cm.nodes + 5 * cm.leaves, per * 40);
      merkle_run(c, cm.nodes, cm.leaves);
    } else {
      hash_rows_run(c, cm.stack, cm.leaves, cm.leaves, 3 * ff, 0, cm.nodes + 5 * cm.leaves);
      merkle_run(c, cm.nodes, cm.leaves);
    }
    std::vector<u64> root = d2h(c, cm.nodes + 5, 5);
    for (auto &v : root) v = from_mont(v);
    ps.enqueue(ItemKind::MerkleRoot, root);
    return cm;
  };
  // evaluate the X-field polynomial d_coef[3][clen] on the coset off*<w_L> (clen <= L); result in d_out[3][L]
  auto evaluate = [&](const u64 *d_coef, size_t clen, u64 off, size_t L, u64 *d_out, u64 *d_scratch) {
    stir_scale_pad_kernel<<<st_grid(L), ST_THREADS, 0, c.stream>>>(d_coef, clen, c.get_pow_tab(off, ilog2s(L)), d_scratch, L);
    launch_check(1);
    NttJob f{};
    f.in = d_scratch; f.in_cstride = L; f.out = d_out; f.out_cstride = L; f.tmp = d_tmp;
    f.log_n = ilog2s(L); f.ncols = 3; f.inverse = false;
    ntt_run(c, f);
  };
  constexpr size_t MAXQ = 4096, MAXN = MAXQ * 40;      // queries per round / authentication-structure nodes
  unsigned *d_idx = (unsigned *)mem.words(MAXQ);
  unsigned *d_nidx = (unsigned *)mem.words(MAXN);
  // one response's leaves: no more distinct folded indices than leaves of the first (largest) tree, each of 3 * ff words
  const size_t max_leaves = std::min(MAXQ, len / ff);
  u64 *d_gather = mem.words(max_leaves * 3 * ff);
  u64 *d_dig = mem.words(MAXN * 5);
  // StirResponse {queried_leafs, auth_structure} of a commitment at the (folded, de-duplicated) indices
  auto respond = [&](const Commitment &cm, const std::vector<uint32_t> &idx) {
    if (idx.size() > max_leaves) throw ApiError{TVM_ERR_UNSUPPORTED, "STIR: more than 4096 distinct queried leaves in one round"};
    TVM_CUDA(cudaMemcpyAsync(d_idx, idx.data(), idx.size() * 4, cudaMemcpyHostToDevice, c.stream));
    gather_rows_run(c, cm.stack, cm.leaves, 3 * ff, d_idx, (unsigned)idx.size(), 0, -1, d_gather);
    std::vector<u64> rows = d2h(c, d_gather, idx.size() * 3 * ff);
    std::vector<unsigned> nodes = auth_structure_node_indices(cm.leaves, idx);
    std::vector<u64> auth;
    if (!nodes.empty()) {
      if (nodes.size() > MAXN) throw ApiError{TVM_ERR_UNSUPPORTED, "STIR: authentication structure too large"};
      TVM_CUDA(cudaMemcpyAsync(d_nidx, nodes.data(), nodes.size() * 4, cudaMemcpyHostToDevice, c.stream));
      gather_digests_run(c, cm.nodes, d_nidx, (unsigned)nodes.size(), d_dig);
      auth = d2h(c, d_dig, nodes.size() * 5);
    }
    // BFieldCodec: Vec<Vec<XFE>> = count, then every (dynamically sized) inner Vec prefixed with its length
    std::vector<u64> a, b;
    a.push_back(idx.size());
    for (size_t t = 0; t < idx.size(); t++) {
      a.push_back(1 + 3 * ff);
      a.push_back(ff);
      a.insert(a.end(), rows.begin() + t * 3 * ff, rows.begin() + (t + 1) * 3 * ff);
    }
    b.push_back(auth.size() / 5); b.insert(b.end(), auth.begin(), auth.end());
    std::vector<u64> e;
    const std::vector<u64> *order[2] = {&a, &b};
    for (int t = 0; t < 2; t++) {
      const std::vector<u64> &f = *order[BFIELDCODEC_STRUCT_FIELDS_REVERSED ? 1 - t : t];
      e.push_back(f.size());
      e.insert(e.end(), f.begin(), f.end());
    }
    ps.enqueue(ItemKind::StirResponse, e);
  };
  auto dedup_folded = [&](const std::vector<uint32_t> &queried, size_t f_len) {
    std::vector<uint32_t> out;
    std::set<uint32_t> seen;
    for (uint32_t q : queried) {
      uint32_t f = (uint32_t)(q % f_len);
      if (seen.insert(f).second) out.push_back(f);
    }
    return out;
  };

  // ---- initialize (stir.rs:891-908) ----
  size_t cur_len = len;
  u64 cur_off = offset_mont;
  Commitment commitment = commit(d_codeword, cur_len);
  u64 *d_poly = mem.words(3 * cur_len);     // coefficients of the round polynomial, [3][cur_len]
  {
    NttJob inv{};
    inv.in = d_codeword; inv.in_cstride = cur_len; inv.out = d_poly; inv.out_cstride = cur_len; inv.tmp = d_tmp;
    inv.log_n = ilog2s(cur_len); inv.ncols = 3; inv.inverse = true;
    ntt_run(c, inv);
    scale_by_powers_run(c, d_poly, cur_len, 3, cur_len, c.get_pow_tab(finv(cur_off), ilog2s(cur_len)));
  }
  std::vector<uint32_t> first_round_indices;
  bool have_first = false;

  for (int round = 0; round < sd.num_rounds; round++) {
    const xfe r = ps.sample_scalars(1)[0];
    const size_t f_len = cur_len / ff, n_len = cur_len / 2;
    const u64 n_off = fmul(fmul(cur_off, cur_off), cur_off);                 // next_round_domain: offset^2 * offset
    const u64 f_off = fpow(cur_off, ff);                                      // domain.pow(folding_factor)
    u64 *d_folded = mem.words(3 * f_len);
    fold(d_poly, cur_len, r, d_folded, f_len);
    u64 *d_scratch = mem.words(3 * n_len);
    u64 *d_fe = mem.words(3 * n_len);          // folded evaluations on the next round's domain
    evaluate(d_folded, f_len, n_off, n_len, d_fe, d_scratch);
    Commitment folded_commitment = commit(d_fe, n_len);

    // out-of-domain queries (stir.rs:921-926)
    const size_t num_ood = sd.out_of_domain[round];
    std::vector<xfe> ood_queries = ps.sample_scalars(num_ood);
    std::vector<xfe> ood_values(num_ood);
    {
      u64 *d_pw = d_scratch;                  // power vector [3][f_len] (d_scratch is free again)
      u64 *d_dots = mem.words(32);
      std::vector<u64> payload;
      payload.push_back(num_ood);
      for (size_t t = 0; t < num_ood; t++) {
        xpow_vector_run(c, ood_queries[t], d_pw, f_len, f_len);
        col_dot_run(c, d_folded, f_len, 3, f_len, d_pw, f_len, 3 * f_len, 1, d_dots);
        std::vector<u64> dv = d2h(c, d_dots, 9);
        ood_values[t] = combine_planes(xmake(dv[0], dv[1], dv[2]), xmake(dv[3], dv[4], dv[5]), xmake(dv[6], dv[7], dv[8]));
        push_xfe_canon(payload, ood_values[t]);
      }
      ps.enqueue(ItemKind::StirOutOfDomainValues, payload);
      mem.release(d_dots);
    }

    // in-domain queries against the previous commitment (stir.rs:928-940)
    std::vector<uint32_t> queried = ps.sample_indices((uint32_t)cur_len, sd.in_domain[round]);
    std::vector<uint32_t> folded_idx = dedup_folded(queried, f_len);
    respond(commitment, folded_idx);

    // answers of the folded polynomial at the queried points of the folded domain (stir.rs:942-957)
    std::vector<xfe> points, answers;
    {
      u64 *d_ff = d_scratch;                  // folded polynomial on offset^k <g^k>, [3][f_len]
      u64 *d_ff_in = mem.words(3 * f_len);
      evaluate(d_folded, f_len, f_off, f_len, d_ff, d_ff_in);
      mem.release(d_ff_in);
      TVM_CUDA(cudaMemcpyAsync(d_idx, folded_idx.data(), folded_idx.size() * 4, cudaMemcpyHostToDevice, c.stream));
      gather_rows_run(c, d_ff, f_len, 3, d_idx, (unsigned)folded_idx.size(), 0, -1, d_gather);
      std::vector<u64> vals = d2h(c, d_gather, folded_idx.size() * 3);     // canonical
      const u64 gf = root_of_unity_mont((unsigned)ilog2s(f_len));
      for (size_t t = 0; t < folded_idx.size(); t++) {
        points.push_back(xlift(fmul(f_off, fpow(gf, folded_idx[t]))));
        answers.push_back(xmake(to_mont(vals[3 * t]), to_mont(vals[3 * t + 1]), to_mont(vals[3 * t + 2])));
      }
      for (size_t t = 0; t < num_ood; t++) { points.push_back(ood_queries[t]); answers.push_back(ood_values[t]); }
    }
    const size_t m = points.size();
    // Ans and Zerofier (stir.rs:958-960): on the device when the point set fits one CTA, else on the host
    u64 *d_small = mem.words(3 * (2 * m + 1));      // ans [3][m] followed by zerofier [3][m+1]
    if (m < 1024) {
      std::vector<u64> hp(6 * m);
      for (size_t k = 0; k < m; k++) {
        hp[3 * k] = points[k].c0; hp[3 * k + 1] = points[k].c1; hp[3 * k + 2] = points[k].c2;
        hp[3 * m + 3 * k] = answers[k].c0; hp[3 * m + 3 * k + 1] = answers[k].c1; hp[3 * m + 3 * k + 2] = answers[k].c2;
      }
      u64 *d_pv = mem.words(6 * m);
      u64 *d_Q = mem.words(3 * m * m);
      TVM_CUDA(cudaMemcpyAsync(d_pv, hp.data(), hp.size() * 8, cudaMemcpyHostToDevice, c.stream));
      unsigned threads = 32;
      while (threads < m + 1) threads <<= 1;
      size_t smem = sizeof(u64) * (3 * (m + 1) + 3 * m);
      stir_interpolate_kernel<<<1, threads, smem, c.stream>>>(d_pv, d_pv + 3 * m, (unsigned)m, d_Q, d_small, d_small + 3 * m);
      launch_check(1);
      TVM_CUDA(cudaStreamSynchronize(c.stream));     // `hp` goes out of scope
      mem.release(d_pv); mem.release(d_Q);
    } else {
      const XPoly zf = xp_zerofier(points);
      const XPoly ans = xp_interpolate(points, answers, zf);
      std::vector<u64> host(3 * (2 * m + 1));
      for (size_t k = 0; k < m; k++) { host[k] = ans[k].c0; host[m + k] = ans[k].c1; host[2 * m + k] = ans[k].c2; }
      u64 *hz = host.data() + 3 * m;
      for (size_t k = 0; k <= m; k++) { hz[k] = zf[k].c0; hz[(m + 1) + k] = zf[k].c1; hz[2 * (m + 1) + k] = zf[k].c2; }
      TVM_CUDA(cudaMemcpyAsync(d_small, host.data(), host.size() * 8, cudaMemcpyHostToDevice, c.stream));
      TVM_CUDA(cudaStreamSynchronize(c.stream));
    }
    const xfe rho = ps.sample_scalars(1)[0];       // degree-correction randomness

    // next round's polynomial (stir.rs:958-972)
    {
      u64 *d_A = mem.words(3 * n_len), *d_Z = mem.words(3 * n_len);
      evaluate(d_small, m, n_off, n_len, d_A, d_scratch);
      evaluate(d_small + 3 * m, m + 1, n_off, n_len, d_Z, d_scratch);
      stir_quotient_kernel<<<st_grid(n_len), ST_THREADS, 0, c.stream>>>(d_fe, d_A, d_Z, n_len, n_off,
                                                                        c.get_pow_tab(root_of_unity_mont((unsigned)ilog2s(n_len)), ilog2s(n_len)),
                                                                        rho, (unsigned)(m + 1), d_scratch);
      launch_check(1);
      mem.release(d_poly);
      d_poly = mem.words(3 * n_len);
      NttJob inv{};
      inv.in = d_scratch; inv.in_cstride = n_len; inv.out = d_poly; inv.out_cstride = n_len; inv.tmp = d_tmp;
      inv.log_n = ilog2s(n_len); inv.ncols = 3; inv.inverse = true;
      ntt_run(c, inv);
      scale_by_powers_run(c, d_poly, n_len, 3, n_len, c.get_pow_tab(finv(n_off), ilog2s(n_len)));
      mem.release(d_A); mem.release(d_Z); mem.release(d_small);
    }
    mem.release(d_fe); mem.release(d_scratch); mem.release(d_folded);
    mem.release(commitment.stack); mem.release(commitment.nodes);
    commitment = folded_commitment;
    cur_len = n_len; cur_off = n_off;
    if (!have_first) { first_round_indices = queried; have_first = true; }
  }

  // ---- final round (stir.rs:975-991) ----
  {
    const xfe r = ps.sample_scalars(1)[0];
    const size_t f_len = cur_len / ff;
    u64 *d_final = mem.words(3 * f_len);
    fold(d_poly, cur_len, r, d_final, f_len);
    std::vector<u64> co = d2h(c, d_final, 3 * f_len);
    size_t deg_plus_1 = f_len;
    while (deg_plus_1 > 0 && co[deg_plus_1 - 1] == 0 && co[f_len + deg_plus_1 - 1] == 0 && co[2 * f_len + deg_plus_1 - 1] == 0) deg_plus_1--;
    std::vector<u64> payload;        // Polynomial { coefficients }: length of the Vec encoding, count, elements (see prover.cu)
    payload.push_back(1 + 3 * deg_plus_1);
    payload.push_back(deg_plus_1);
    for (size_t i = 0; i < deg_plus_1; i++)
      for (int dd = 0; dd < 3; dd++) payload.push_back(from_mont(co[dd * f_len + i]));
    ps.enqueue(ItemKind::Polynomial, payload);
    std::vector<uint32_t> queried = ps.sample_indices((uint32_t)cur_len, sd.final_num_in_domain_queries);
    respond(commitment, dedup_folded(queried, f_len));
    if (!have_first) first_round_indices = queried;
    mem.release(d_final);
  }
  mem.release(d_poly);
  mem.release(commitment.stack); mem.release(commitment.nodes);
  mem.release(d_idx); mem.release(d_nidx); mem.release(d_gather); mem.release(d_dig);
  return first_round_indices;
}

}  // namespace tvm
