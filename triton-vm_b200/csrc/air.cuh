// Shared declarations for the generated AIR quotient kernels (csrc/air_gen/*.cu).
// Semantics: triton-vm/src/table/master_table.rs:1194-1363 (zerofier inverses +
// all_quotients_combined).  Row layout: tables are column-major and coset-major, memory index
// m = coset * n + k  <->  quotient-domain row i = coset + r*k, x_i = offset * w_{rn}^i; the
// "next row" i + r (unit distance = quotient_len / trace_len, master_table.rs:1305-1306) is
// (coset, k+1 mod n).
#pragma once
#include "ctx.h"

namespace tvm {

#ifndef TVM_AIR_THREADS
#define TVM_AIR_THREADS 256
#endif
static constexpr int AIR_THREADS = TVM_AIR_THREADS;
static constexpr int AIR_MAX_COSETS = 64;

static constexpr unsigned AIR_AUX_BCOLS = 270;   // aux B-field columns the constraints read (X-field columns 0..89)
static constexpr int AIR_WTAB_WORDS = 7;   // per weight w = (b0,b1,b2): b0, b1, b2, -b1, -b2, b0+b2, b1-b2

struct AirArgs {
  const u64 *main;      // main column q at main + q*main_stride
  size_t main_stride;
  const u64 *aux;       // aux X-field column q, coordinate d at aux + (3q+d)*aux_stride
  size_t aux_stride;
  // 0: the "next row" is row (coset, k+1 mod n).  Otherwise it is read at the current row's index plus next_offset words in
  // both tables (quotient.cu's top-degree correction stores the next-row polynomials as separate columns)
  size_t next_offset;
  u64 *out;             // quotient codeword, planar: coordinate d at out + d*out_stride, memory order
  size_t out_stride;
  size_t nrows;         // (#cosets evaluated) * n
  int log_n;            // trace length n = 2^log_n
  unsigned coset_mem_stride;   // evaluated coset y sits at table coset y * coset_mem_stride (quotient domain = every
                               // (N/Q)-th coset of the LDT-domain tables when the expansion factor exceeds 4)
  // per-row zerofier inverses in memory order (air_zerofier_kernel):
  const u64 *zi_init;   // 1 / (x - 1)                         (master_table.rs:1194-1202)
  const u64 *zi_tran;   // (x - w_n^-1) / (x^n - 1)            (1216-1237)
  const u64 *zi_term;   // 1 / (x - w_n^-1)                    (1239-1252)
  u64 cons_zerofier_inv[AIR_MAX_COSETS];  // 1 / (x^n - 1), constant on a coset   (1204-1214)
  // Degree split (quotient.cu): the chunks given these arguments add their sums WITHOUT the zerofier inverse to low_out:
  // class t (init, cons, tran, term), coordinate d at low_out + (3t + d) * low_stride, compact row index.  nullptr: they
  // add the zerofier-weighted sums to `out`.
  u64 *low_out;
  size_t low_stride;
  int min_degree;       // chunks whose constraints all have a smaller degree are not launched with these arguments
};

// strides handed to the chunk bodies of a fused group kernel (generated code refers to them as a.main_stride / a.aux_stride)
struct AirStrides {
  size_t main_stride, aux_stride;
};

// ---- unreduced accumulation of  sum_j w_j * c_j ------------------------------------------------
// (c * w)_0 = c0 b0 - c1 b2 - c2 b1;  (c * w)_1 = c0 b1 + c1 (b0 + b2) + c2 (b1 - b2);
// (c * w)_2 = c0 b2 + c1 b1 + c2 (b0 + b2)           (X^3 = X - 1)
// Each coordinate sums 128-bit products of Montgomery words; `ov` counts carries out of bit 128.
struct AirAcc {
  u64 lo[3], hi[3];
  u32 ov[3];
};
__device__ __forceinline__ void air_acc_zero(AirAcc &c) {
#pragma unroll
  for (int i = 0; i < 3; i++) { c.lo[i] = 0; c.hi[i] = 0; c.ov[i] = 0; }
}
__device__ __forceinline__ void air_mac(u64 &lo, u64 &hi, u32 &ov, u64 x, u64 y) {
  const unsigned __int128 p128 = (unsigned __int128)x * y;   // one 128-bit product: 4 IMAD.WIDE (x * y and __umul64hi form the low half twice)
  u64 plo = (u64)p128, phi = (u64)(p128 >> 64);
  asm("add.cc.u64 %0, %0, %3;\n\taddc.cc.u64 %1, %1, %4;\n\taddc.u32 %2, %2, 0;"
      : "+l"(lo), "+l"(hi), "+r"(ov) : "l"(plo), "l"(phi));
}
__device__ __forceinline__ void air_acc_b(AirAcc &c, const u64 *w, u64 v) {
  air_mac(c.lo[0], c.hi[0], c.ov[0], v, w[0]);
  air_mac(c.lo[1], c.hi[1], c.ov[1], v, w[1]);
  air_mac(c.lo[2], c.hi[2], c.ov[2], v, w[2]);
}
__device__ __forceinline__ void air_acc_x(AirAcc &c, const u64 *w, xfe v) {
  air_mac(c.lo[0], c.hi[0], c.ov[0], v.c0, w[0]);
  air_mac(c.lo[0], c.hi[0], c.ov[0], v.c1, w[4]);
  air_mac(c.lo[0], c.hi[0], c.ov[0], v.c2, w[3]);
  air_mac(c.lo[1], c.hi[1], c.ov[1], v.c0, w[1]);
  air_mac(c.lo[1], c.hi[1], c.ov[1], v.c1, w[5]);
  air_mac(c.lo[1], c.hi[1], c.ov[1], v.c2, w[6]);
  air_mac(c.lo[2], c.hi[2], c.ov[2], v.c0, w[2]);
  air_mac(c.lo[2], c.hi[2], c.ov[2], v.c1, w[1]);
  air_mac(c.lo[2], c.hi[2], c.ov[2], v.c2, w[5]);
}
// (lo + 2^64 hi + 2^128 ov) * 2^-64  =  montyred(lo, 0) + hi + ov * 2^64   (mod p)
__device__ __forceinline__ u64 air_reduce160(u64 lo, u64 hi, u32 ov) {
  u64 h = hi >= P ? hi - P : hi;
  return fadd(fadd(montyred(lo, 0), h), (u64)ov * EPS);
}
__device__ __forceinline__ xfe air_acc_reduce(const AirAcc &c) {
  return xmake(air_reduce160(c.lo[0], c.hi[0], c.ov[0]), air_reduce160(c.lo[1], c.hi[1], c.ov[1]),
               air_reduce160(c.lo[2], c.hi[2], c.ov[2]));
}

__device__ __forceinline__ void air_add_out(const AirArgs &a, size_t m, xfe v) {
  u64 *o = a.out + m;
  o[0] = fadd(o[0], v.c0);
  o[a.out_stride] = fadd(o[a.out_stride], v.c1);
  o[2 * a.out_stride] = fadd(o[2 * a.out_stride], v.c2);
}

__device__ __forceinline__ void air_accumulate_init(const AirArgs &a, size_t m, size_t, xfe acc) {
  air_add_out(a, m, xmulb(acc, a.zi_init[m]));
}
__device__ __forceinline__ void air_accumulate_cons(const AirArgs &a, size_t m, size_t coset, xfe acc) {
  air_add_out(a, m, xmulb(acc, a.cons_zerofier_inv[coset]));
}
__device__ __forceinline__ void air_accumulate_tran(const AirArgs &a, size_t m, size_t, xfe acc) {
  air_add_out(a, m, xmulb(acc, a.zi_tran[m]));
}
__device__ __forceinline__ void air_accumulate_term(const AirArgs &a, size_t m, size_t, xfe acc) {
  air_add_out(a, m, xmulb(acc, a.zi_term[m]));
}

template <int TYPE>
__device__ __forceinline__ void air_accumulate_low(const AirArgs &a, size_t m, size_t coset, xfe acc) {
  if (a.low_out) {
    u64 *o = a.low_out + (size_t)(3 * TYPE) * a.low_stride + m;
    o[0] = fadd(o[0], acc.c0);
    o[a.low_stride] = fadd(o[a.low_stride], acc.c1);
    o[2 * a.low_stride] = fadd(o[2 * a.low_stride], acc.c2);
    return;
  }
  if (TYPE == 0) air_accumulate_init(a, m, coset, acc);
  else if (TYPE == 1) air_accumulate_cons(a, m, coset, acc);
  else if (TYPE == 2) air_accumulate_tran(a, m, coset, acc);
  else air_accumulate_term(a, m, coset, acc);
}

}  // namespace tvm
