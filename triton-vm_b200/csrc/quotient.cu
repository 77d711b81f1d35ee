// Quotient codeword: host-side driver of the generated AIR kernels.
// Restates Prover::compute_quotient_segments' cached branch up to the quotient codeword
// (triton-vm/src/stark.rs:770-782) = all_quotients_combined (master_table.rs:1264-1363).
#include "air.cuh"
#include "launch.h"
#include "air_gen/air_meta.inc"
#include "stark.h"
#include <cstdlib>

namespace tvm {

#define TVM_AIR_TU(name) void name##_launch(const AirArgs &lo, const AirArgs &hi, const u64 *d_wtab, const u64 *d_ch, cudaStream_t s, unsigned long long *launches);
#include "air_gen/air_chunks.inc"
#undef TVM_AIR_TU

namespace {
struct AirConstSlot {
  std::mutex m;
  cudaEvent_t last_use = nullptr;   // recorded at the end of every lease on this device (created by the first one)
};
AirConstSlot &air_const_slot(int device) {
  static std::mutex registry;
  static auto *slots = new std::map<int, AirConstSlot>();   // never destroyed: a context may outlive static destruction
  std::lock_guard<std::mutex> g(registry);
  return (*slots)[device];
}
}  // namespace

AirConstLease::AirConstLease(Ctx &c) : c_(c) {
  AirConstSlot &s = air_const_slot(c.device);
  std::unique_lock<std::mutex> lock(s.m);
  if (!s.last_use) TVM_CUDA(cudaEventCreateWithFlags(&s.last_use, cudaEventDisableTiming));
  TVM_CUDA(cudaStreamWaitEvent(c.stream, s.last_use, 0));
  last_use_ = s.last_use;
  lock_ = std::move(lock);
}

AirConstLease::~AirConstLease() { cudaEventRecord(last_use_, c_.stream); }

// weight table: 7 words per weight (air.cuh, AIR_WTAB_WORDS)
__global__ void air_weight_table_kernel(const u64 *w, unsigned count, u64 *tab) {
  unsigned j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= count) return;
  u64 b0 = w[3 * j], b1 = w[3 * j + 1], b2 = w[3 * j + 2];
  u64 *t = tab + (size_t)AIR_WTAB_WORDS * j;
  t[0] = b0; t[1] = b1; t[2] = b2; t[3] = fneg(b1); t[4] = fneg(b2); t[5] = fadd(b0, b2); t[6] = fsub(b1, b2);
}

// Per-row zerofier inverses.  Each thread owns ZF_PER rows and inverts
// their (x - 1) and (x - w_n^-1) with one shared field inversion (Montgomery's trick).
static constexpr int ZF_PER = 8;
struct ZerofierArgs {
  u64 *zi_init, *zi_tran, *zi_term;
  size_t nrows;
  int log_n;
  PowTab trace_gen;
  u64 trace_gen_inv;
  u64 coset_x[AIR_MAX_COSETS];
  u64 cons_zerofier_inv[AIR_MAX_COSETS];
};
__global__ void __launch_bounds__(256) air_zerofier_kernel(ZerofierArgs a) {
  // the ZF_PER rows of a thread are strided by the total thread count so that stores stay coalesced
  const size_t nthreads = (size_t)gridDim.x * blockDim.x;
  const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t n = (size_t)1 << a.log_n;
  u64 d[2 * ZF_PER], pre[2 * ZF_PER];
  u64 run = MONT_ONE;
#pragma unroll
  for (int j = 0; j < ZF_PER; j++) {
    size_t m = t + (size_t)j * nthreads;
    if (m >= a.nrows) m = a.nrows - 1;
    size_t coset = m >> a.log_n, k = m & (n - 1);
    u64 lo = __ldg(a.trace_gen.lo + (k & ((1ULL << a.trace_gen.shift) - 1)));
    u64 hi = __ldg(a.trace_gen.hi + (k >> a.trace_gen.shift));
    u64 x = fmul(a.coset_x[coset], fmul(lo, hi));
    d[2 * j] = fsub(x, MONT_ONE);
    d[2 * j + 1] = fsub(x, a.trace_gen_inv);
    pre[2 * j] = run; run = fmul(run, d[2 * j]);
    pre[2 * j + 1] = run; run = fmul(run, d[2 * j + 1]);
  }
  u64 inv = finv(run);
#pragma unroll
  for (int j = ZF_PER - 1; j >= 0; j--) {
    u64 i1 = fmul(inv, pre[2 * j + 1]); inv = fmul(inv, d[2 * j + 1]);
    u64 i0 = fmul(inv, pre[2 * j]);     inv = fmul(inv, d[2 * j]);
    size_t m = t + (size_t)j * nthreads;
    if (m < a.nrows) {
      a.zi_init[m] = i0;
      a.zi_term[m] = i1;
      a.zi_tran[m] = fmul(d[2 * j + 1], a.cons_zerofier_inv[m >> a.log_n]);
    }
  }
}

// Degree split, last step: out += sum over the four zerofier classes of zerofier_inverse_class(row) * S_class(row), where S_class
// (the weighted sum of the class's split constraints) sits in coset-major order for the even cosets (computed by the
// split chunks) and in NATURAL order of the half-size domain for the odd cosets (extended by two transforms, air_quotient_run).
__global__ void __launch_bounds__(256) air_low_combine_kernel(AirArgs a, const u64 *s_even, const u64 *s_odd, size_t ls, int log_half) {
  const size_t m = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= a.nrows) return;
  const size_t n = (size_t)1 << a.log_n;
  const size_t coset = m >> a.log_n, k = m & (n - 1), half = coset >> 1;
  const u64 *src = (coset & 1) ? s_odd + half + (k << log_half) : s_even + half * n + k;
  const u64 zi[4] = {a.zi_init[m], a.cons_zerofier_inv[coset], a.zi_tran[m], a.zi_term[m]};
  xfe acc = xzero();
#pragma unroll
  for (int t = 0; t < 4; t++) acc = xadd(acc, xmulb(xmake(src[(3 * t) * ls], src[(3 * t + 1) * ls], src[(3 * t + 2) * ls]), zi[t]));
  air_add_out(a, m, acc);
}

// ---- top-degree correction of the full degree split ------------------------------------------------------------------
// Columns are polynomials of degree <= D = n + h - 1 in u = x / offset (d_coef holds their u-coefficients).  A class sum C
// (the weighted sum of one zerofier class's constraints) has degree <= 4D; write C = r + u^{4n} q with deg r < 4n.  On the even
// cosets u^{4n} = 1, so their values interpolate to r + q; on the odd ones u^{4n} = -1 and C = r - q.  With
// s = 4n - 3D >= 1 every term of C of degree >= 4n comes from the degree-4 part H4 of C applied to the column tops
// T = coefficients s..D (4h - 3 of them): q_i = [u^(i + 12(h-1))] H4(T).  H4(T) has degree <= 16(h-1) and is evaluated on
// L >= 16h - 15 points as (C(2T) + C(-2T) - 4 (C(T) + C(-T)) + 6 C(0)) / 24, by the hi chunks on 5 "cosets" of L rows.
static constexpr int AIR_TOP_LAMBDAS = 5;   // slot l of a top column holds lambda_l * T at the L points, lambda = 0, 1, -1, 2, -2

// tops[q][i] (row stride L): coefficient s + i of column q, zero for i >= count; columns q >= ncur are the next-row
// polynomials col(w_n u) of columns q - ncur, whose coefficient j carries the extra factor w_n^j
__global__ void air_top_extract_kernel(const u64 *main_coef, const u64 *aux_coef, size_t coef_stride, unsigned nmain,
                                       unsigned ncur, size_t s, unsigned count, int log_n, PowTab wn, u64 *tops, size_t L) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned q = blockIdx.y;
  if (i >= L) return;
  u64 v = 0;
  if (i < count) {
    const unsigned qc = q % ncur;
    const u64 *col = qc < nmain ? main_coef + (size_t)qc * coef_stride : aux_coef + (size_t)(qc - nmain) * coef_stride;
    v = col[s + i];
    if (q >= ncur) {
      const u64 e = (s + i) & (((u64)1 << log_n) - 1);
      v = fmul(v, fmul(__ldg(wn.lo + (e & ((1ULL << wn.shift) - 1))), __ldg(wn.hi + (e >> wn.shift))));
    }
  }
  tops[(size_t)q * L + i] = v;
}

// slot 1 of every top column holds T at the L points: slots 0, 2, 3, 4 become 0, -T, 2T, -2T
__global__ void air_top_lambda_kernel(u64 *tab, size_t L) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= L) return;
  u64 *col = tab + (size_t)blockIdx.y * AIR_TOP_LAMBDAS * L;
  const u64 v = col[L + i], v2 = fadd(v, v);
  col[i] = 0; col[2 * L + i] = fneg(v); col[3 * L + i] = v2; col[4 * L + i] = fneg(v2);
}

// h4[p][i] = (S_2 + S_-2 - 4 (S_1 + S_-1) + 6 S_0) / 24 for the 12 planes of class sums S (slot stride L, plane stride 5L)
__global__ void air_top_h4_kernel(const u64 *sums, size_t L, u64 inv24, u64 *h4) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= L) return;
  const u64 *S = sums + (size_t)blockIdx.y * AIR_TOP_LAMBDAS * L + i;
  const u64 s1 = fadd(S[L], S[2 * L]), s2 = fadd(S[3 * L], S[4 * L]);
  const u64 s1x4 = fadd(fadd(s1, s1), fadd(s1, s1));
  const u64 s0x2 = fadd(S[0], S[0]), s0x6 = fadd(fadd(s0x2, s0x2), s0x2);
  h4[(size_t)blockIdx.y * L + i] = fmul(fadd(fsub(s2, s1x4), s0x6), inv24);
}

// coef[p][i] -= 2 q_p[i] = 2 h4coef[p][first + i] for i < count (12 planes, strides `stride` and L)
__global__ void air_top_subtract_kernel(u64 *coef, size_t stride, const u64 *h4coef, size_t L, size_t first, unsigned count) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  const u64 q = h4coef[(size_t)blockIdx.y * L + first + i];
  u64 *c = coef + (size_t)blockIdx.y * stride + i;
  *c = fsub(*c, fadd(q, q));
}

// Subtracts 2q from the 12 coefficient planes of the even-coset class sums (stride ls).  Scratch on the context pool.
static void air_top_correction(Ctx &c, const AirCoefs &cf, unsigned log_n, const u64 *d_wtab, const u64 *d_challenges, u64 *coef,
                               size_t ls) {
  const size_t n = (size_t)1 << log_n, h = cf.num_rand;
  const size_t s = n + 3 - 3 * h;                 // 4n - 3D
  const unsigned count = (unsigned)(4 * h - 3);    // D - s + 1
  int log_L = 6;
  while (((size_t)1 << log_L) < 16 * h - 15) log_L++;
  const size_t L = (size_t)1 << log_L, rows = AIR_TOP_LAMBDAS * L;
  const unsigned nmain = TVM_NUM_MAIN_COLUMNS, ncur = nmain + AIR_AUX_BCOLS, ncols = 2 * ncur;
  // top tables [cur main | cur aux | next main | next aux][5 slots][L] | class sums [12][5][L] | packed tops [ncols][L]
  // (later H4 values and coefficients) | NTT scratch [ncols][L]
  u64 *buf = (u64 *)c.pool_alloc(sizeof(u64) * ((size_t)ncols * rows + 12 * rows + 2 * (size_t)ncols * L));
  u64 *tab = buf, *sums = tab + (size_t)ncols * rows, *packed = sums + 12 * rows, *tmp = packed + (size_t)ncols * L;
  try {
    const dim3 blk(256);
    air_top_extract_kernel<<<dim3((unsigned)((L + 255) / 256), ncols), blk, 0, c.stream>>>(
        cf.main, cf.aux, cf.stride, nmain, ncur, s, count, (int)log_n, c.get_pow_tab(root_of_unity_mont(log_n), (int)log_n), packed, L);
    NttJob fwd{};
    fwd.in = packed; fwd.in_cstride = L; fwd.out = tab + L; fwd.out_cstride = rows; fwd.tmp = tmp;
    fwd.log_n = log_L; fwd.ncols = ncols; fwd.inverse = false;
    ntt_run(c, fwd);
    air_top_lambda_kernel<<<dim3((unsigned)((L + 255) / 256), ncols), blk, 0, c.stream>>>(tab, L);
    TVM_CUDA(cudaMemsetAsync(sums, 0, sizeof(u64) * 12 * rows, c.stream));
    c.launches += 2;
    AirArgs t{};
    t.main = tab; t.aux = tab + (size_t)nmain * rows;
    t.main_stride = t.aux_stride = rows;
    t.next_offset = (size_t)ncur * rows;           // the next-row columns follow the current ones in the same order
    t.nrows = rows; t.log_n = log_L; t.coset_mem_stride = 1;
    t.low_out = sums; t.low_stride = rows;
    t.min_degree = 4;                              // only degree-4 constraints reach H4
    AirArgs none{};
#define TVM_AIR_TU(name) name##_launch(none, t, d_wtab, d_challenges, c.stream, &c.launches);
#include "air_gen/air_chunks.inc"
#undef TVM_AIR_TU
    TVM_CUDA(cudaGetLastError());
    const u64 inv24 = finv(to_mont(24));
    air_top_h4_kernel<<<dim3((unsigned)((L + 255) / 256), 12), blk, 0, c.stream>>>(sums, L, inv24, packed);
    NttJob inv{};
    inv.in = packed; inv.in_cstride = L; inv.out = tmp + 12 * L; inv.out_cstride = L; inv.tmp = tmp;
    inv.log_n = log_L; inv.ncols = 12; inv.inverse = true;
    ntt_run(c, inv);
    air_top_subtract_kernel<<<dim3((count + 255) / 256, 12), blk, 0, c.stream>>>(coef, ls, tmp + 12 * L, L, 12 * (h - 1), count);
    c.launches += 2;
    TVM_CUDA(cudaGetLastError());
  } catch (...) {
    c.pool_release(buf);
    throw;
  }
  c.pool_release(buf);
}

// d_main: [>=379][r*n] coset-major LDE of the main table; d_aux: [>=270][r*n] (X-field columns as
// 3 planar B-field columns); d_challenges: 63 X-field (Montgomery); d_weights: 604 X-field;
// d_out: 3 planes of r*n words (memory order = coset-major), overwritten.
void air_quotient_run(Ctx &c, const u64 *d_main, size_t main_stride, const u64 *d_aux, size_t aux_stride,
                      const u64 *d_challenges, const u64 *d_weights, unsigned log_n, unsigned log_r,
                      unsigned coset_first, unsigned coset_step, unsigned num_cosets, unsigned coset_mem_stride,
                      u64 offset_mont, u64 *d_out, size_t out_stride, const AirCoefs *coefs) {
  if (num_cosets > (unsigned)AIR_MAX_COSETS) throw ApiError{TVM_ERR_UNSUPPORTED, "too many cosets"};
  // every chunk launch below (air_top_correction's too) uploads and reads the device's constant banks
  AirConstLease lease(c);
  // The degree split needs the whole domain in one call, at least 8n points of it, and the tables' degree D = n + h - 1
  // (known from their coefficients).  Constraints of degree <= 2 run on the even cosets when 2D < 4n (their class sums have
  // degree < 4n); all of them do when in addition 3D < 4n on exactly 8n points (air_top_correction).
  static const bool split_enabled = [] { const char *e = getenv("TVM_AIR_NO_DEGREE_SPLIT"); return !(e && e[0] == '1'); }();
  const size_t n = (size_t)1 << log_n;
  const size_t deg = coefs ? n + coefs->num_rand - 1 : 0;
  const bool split = TVM_AIR_HAS_LOW_CHUNKS && split_enabled && coefs && coset_first == 0 && coset_step == 1 &&
                     num_cosets == (1u << log_r) && log_r >= 3 && log_n + log_r - 1 <= 26 && 2 * deg < 4 * n;
  const bool full = split && log_r == 3 && 3 * deg < 4 * n;
  const unsigned num_weights = AIR_NUM_INIT + AIR_NUM_CONS + AIR_NUM_TRAN + AIR_NUM_TERM;
  AirArgs a{};
  a.main = d_main; a.main_stride = main_stride; a.aux = d_aux; a.aux_stride = aux_stride;
  a.out = d_out; a.out_stride = out_stride;
  a.nrows = (size_t)num_cosets << log_n;
  a.log_n = (int)log_n;
  a.coset_mem_stride = coset_mem_stride;
  ZerofierArgs z{};
  z.nrows = a.nrows; z.log_n = a.log_n;
  u64 wn = root_of_unity_mont(log_n);
  z.trace_gen = c.get_pow_tab(wn, (int)log_n);
  z.trace_gen_inv = finv(wn);
  u64 wrn = root_of_unity_mont(log_n + log_r);
  for (unsigned y = 0; y < num_cosets; y++) {
    u64 x = fmul(offset_mont, fpow(wrn, (u64)(coset_first + coset_step * y)));
    z.coset_x[y] = x;
    z.cons_zerofier_inv[y] = a.cons_zerofier_inv[y] = finv(fsub(fpow(x, (u64)1 << log_n), MONT_ONE));
  }
  u64 *low = nullptr;
  u64 *scratch = (u64 *)c.pool_alloc(sizeof(u64) * (3 * a.nrows + (size_t)AIR_WTAB_WORDS * num_weights));
  z.zi_init = scratch; z.zi_tran = scratch + a.nrows; z.zi_term = scratch + 2 * a.nrows;
  u64 *d_wtab = scratch + 3 * a.nrows;
  a.zi_init = z.zi_init; a.zi_tran = z.zi_tran; a.zi_term = z.zi_term;
  try {
    size_t zthreads = (a.nrows + ZF_PER - 1) / ZF_PER;
    air_zerofier_kernel<<<(unsigned)((zthreads + 255) / 256), 256, 0, c.stream>>>(z);
    air_weight_table_kernel<<<(num_weights + 127) / 128, 128, 0, c.stream>>>(d_weights, num_weights, d_wtab);
    c.launches += 2;
    TVM_CUDA(cudaMemsetAsync(d_out, 0, sizeof(u64) * a.nrows, c.stream));
    TVM_CUDA(cudaMemsetAsync(d_out + out_stride, 0, sizeof(u64) * a.nrows, c.stream));
    TVM_CUDA(cudaMemsetAsync(d_out + 2 * out_stride, 0, sizeof(u64) * a.nrows, c.stream));
    AirArgs lo = a;
    const size_t ls = a.nrows / 2;               // rows of the even cosets = plane stride of the class sums
    if (split) {
      low = (u64 *)c.pool_alloc(sizeof(u64) * 48 * ls);   // 12 planes each: class sums | natural order, later odd values | coefficients | NTT scratch
      TVM_CUDA(cudaMemsetAsync(low, 0, sizeof(u64) * 12 * ls, c.stream));
      lo.nrows = ls;
      lo.coset_mem_stride = 2 * coset_mem_stride;           // evaluated coset y of the lo chunks = domain coset 2y
      lo.low_out = low; lo.low_stride = ls;
    }
    const AirArgs &hi = full ? lo : a;
#define TVM_AIR_TU(name) name##_launch(lo, hi, d_wtab, d_challenges, c.stream, &c.launches);
#include "air_gen/air_chunks.inc"
#undef TVM_AIR_TU
    TVM_CUDA(cudaGetLastError());
    if (split) {
      // even cosets = the coset offset*<w_{rn}^2> of `ls` points: natural order, inverse transform (= coefficients times
      // offset^j), times w_{rn}^j, forward transform = the values on offset*w_{rn}*<w_{rn}^2>, the odd cosets, natural order
      u64 *nat = low + 12 * ls, *coef = low + 24 * ls, *ntt_tmp = low + 36 * ls;
      const int log_half = (int)log_r - 1, log_len = (int)(log_n + log_r) - 1;
      coset_to_natural_run(c, low, nat, ls, ls, (int)log_n, log_half, 12);
      NttJob inv{};
      inv.in = nat; inv.in_cstride = ls; inv.out = coef; inv.out_cstride = ls; inv.tmp = ntt_tmp;
      inv.log_n = log_len; inv.ncols = 12; inv.inverse = true;
      ntt_run(c, inv);
      if (full && coefs->num_rand) air_top_correction(c, *coefs, log_n, d_wtab, d_challenges, coef, ls);   // r + q -> r - q
      scale_by_powers_run(c, coef, ls, 12, ls, c.get_pow_tab(wrn, log_len));
      NttJob fwd{};
      fwd.in = coef; fwd.in_cstride = ls; fwd.out = nat; fwd.out_cstride = ls; fwd.tmp = ntt_tmp;
      fwd.log_n = log_len; fwd.ncols = 12; fwd.inverse = false;
      ntt_run(c, fwd);
      air_low_combine_kernel<<<(unsigned)((a.nrows + 255) / 256), 256, 0, c.stream>>>(a, low, nat, ls, log_half);
      c.launches++;
      TVM_CUDA(cudaGetLastError());
    }
  } catch (...) {
    c.pool_release(scratch);
    if (low) c.pool_release(low);
    throw;
  }
  c.pool_release(scratch);
  if (low) c.pool_release(low);
}

}  // namespace tvm
