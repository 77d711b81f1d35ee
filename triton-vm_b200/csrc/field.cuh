// B-field / X-field device arithmetic for sm_90a.
//
// Elements live in HBM and registers in MONTGOMERY form (R = 2^64), the same
// in-memory representation twenty-first's BFieldElement uses (reference
// triton-constraint-builder/src/codegen.rs:926-932), because Tip5's split-and-lookup
// S-box is defined on the bytes of that representation (tips/tip-0005/tip-0005.md:52-61,94-104).
// p = 2^64 - 2^32 + 1 (triton-vm/src/lib.rs:5-6).  X-field = F_p[X]/(X^3 - X + 1)
// (specification/src/isa.md:8).
#pragma once
#pragma nv_diag_suppress 550  // asm scratch outputs
#include <cstdint>
#include <cuda_runtime.h>

namespace tvm {

typedef uint64_t u64;
typedef unsigned int u32;

static constexpr u64 P = 0xFFFFFFFF00000001ULL;
static constexpr u64 MONT_ONE = 0xFFFFFFFFULL;          // R mod p
static constexpr u64 MONT_R2 = 0xFFFFFFFE00000001ULL;   // R^2 mod p
static constexpr u64 EPS = 0xFFFFFFFFULL;               // 2^64 mod p

#define TVM_HD __host__ __device__ __forceinline__
#define TVM_D __device__ __forceinline__

// ---- 128-bit product + Montgomery reduction -------------------------------------------
// x = lo + 2^64 hi  ->  x * 2^-64 mod p, result canonical when x < p * 2^64.
//
// Device versions are explicit 32-bit carry chains: the kernels that use them (NTT, Tip5, AIR)
// are bound by the integer-ALU pipe rather than by the IMAD (fma) pipe,
// and the compiler's compare/select sequences for the C versions cost 13 ALU instructions per
// fmul, 9 per fadd/fsub; the chains below cost 8 / 7 / 5.
// Contract for ANY x < 2^128: the result is < 2^64 and congruent to x * 2^-64 (hi - b with b < p, plus p on borrow).
TVM_HD u64 montyred(u64 lo, u64 hi) {
#ifdef __CUDA_ARCH__
  u32 x0 = (u32)lo, x1 = (u32)(lo >> 32), x2 = (u32)hi, x3 = (u32)(hi >> 32);
  u32 a1, b0, b1, r0, r1;
  // a = lo*(2^32+1) mod 2^64 = (x0, x1+x0), e = carry;  b = a - (a>>32) - e;  r = hi - b (+p on borrow)
  // (carry chains are kept homogeneous: an add.cc feeding a subc is not translated faithfully by ptxas)
  asm("{\n\t"
      ".reg .u32 t;\n\t"
      "add.u32 %0, %6, %5;\n\t"       // a1 = x1 + x0 (mod 2^32)
      "sub.cc.u32 t, %0, %5;\n\t"     // borrow <=> a1 < x0 <=> the addition carried (e)
      "subc.cc.u32 %1, %5, %0;\n\t"   // b0 = a0 - a1 - e
      "subc.u32 %2, %0, 0;\n\t"       // b1 = a1 - borrow
      "sub.cc.u32 %3, %7, %1;\n\t"    // r0 = x2 - b0
      "subc.cc.u32 %4, %8, %2;\n\t"   // r1 = x3 - b1 - borrow
      "subc.u32 %1, 0, 0;\n\t"        // m = borrow ? 0xffffffff : 0
      "sub.cc.u32 %3, %3, %1;\n\t"    // r -= eps & m   (== r += p mod 2^64)
      "subc.u32 %4, %4, 0;\n\t"
      "}"
      : "=&r"(a1), "=&r"(b0), "=&r"(b1), "=&r"(r0), "=&r"(r1)
      : "r"(x0), "r"(x1), "r"(x2), "r"(x3));
  return ((u64)r1 << 32) | r0;
#else
  u64 a = lo + (lo << 32);
  u64 e = a < lo;
  u64 b = a - (a >> 32) - e;
  u64 r = hi - b;
  u64 c = hi < b;
  return r - (EPS & (0 - c));
#endif
}

TVM_HD u64 fmul(u64 a, u64 b) {
  // one 128-bit product: nvcc turns this into 4 IMAD.WIDE (+3 carry fix-ups); separate `a * b` and
  // `__umul64hi(a, b)` cost 8 IMAD-class instructions because the low product is formed twice
  unsigned __int128 x = (unsigned __int128)a * b;
  u64 lo = (u64)x, hi = (u64)(x >> 64);
  return montyred(lo, hi);
}
// Squaring as the general product: a three-product form (a0^2 + 2^33 a0 a1 + 2^64 a1^2) saves one IMAD.WIDE but pays
// for doubling the cross term with shifts and a separate carry chain; in the Tip5 round it measured 20 SASS instructions
// MORE per round body (704 against 684 on sm_90a) than nvcc's four accumulating IMAD.WIDE.
TVM_HD u64 fsqr(u64 a) { return fmul(a, a); }
// the canonical representative of any x < 2^64
TVM_HD u64 fcanon(u64 x) { return x >= P ? x - P : x; }

TVM_HD u64 fsub(u64 a, u64 b) {  // canonical a, b in [0, p] -> canonical
#ifdef __CUDA_ARCH__
  u32 r0, r1, m;
  asm("{\n\t"
      "sub.cc.u32 %0, %3, %5;\n\t"
      "subc.cc.u32 %1, %4, %6;\n\t"
      "subc.u32 %2, 0, 0;\n\t"        // m = borrow ? 0xffffffff : 0
      "sub.cc.u32 %0, %0, %2;\n\t"    // += p  (== -= eps mod 2^64)
      "subc.u32 %1, %1, 0;\n\t"
      "}"
      : "=&r"(r0), "=&r"(r1), "=&r"(m)
      : "r"((u32)a), "r"((u32)(a >> 32)), "r"((u32)b), "r"((u32)(b >> 32)));
  return ((u64)r1 << 32) | r0;
#else
  u64 d = a - b;
  if (a < b) d += P;
  return d;
#endif
}
TVM_HD u64 fadd(u64 a, u64 b) {  // canonical in, canonical out
#ifdef __CUDA_ARCH__
  // a + b = a - (p - b); p - b in [1, p] is a valid subtrahend for fsub
  u32 n0, n1;
  asm("{\n\t"
      "sub.cc.u32 %0, 1, %2;\n\t"
      "subc.u32 %1, 0xffffffff, %3;\n\t"
      "}"
      : "=&r"(n0), "=&r"(n1)
      : "r"((u32)b), "r"((u32)(b >> 32)));
  return fsub(a, ((u64)n1 << 32) | n0);
#else
  u64 s = a + b;
  if (s < a || s >= P) s -= P;
  return s;
#endif
}
TVM_HD u64 fneg(u64 a) { return a ? P - a : 0; }
TVM_HD u64 to_mont(u64 canon) { return fmul(canon, MONT_R2); }
TVM_HD u64 from_mont(u64 m) { return montyred(m, 0); }

TVM_HD u64 fpow(u64 a, u64 e) {
  u64 r = MONT_ONE;
  while (e) {
    if (e & 1) r = fmul(r, a);
    a = fmul(a, a);
    e >>= 1;
  }
  return r;
}
TVM_HD u64 finv(u64 a) { return fpow(a, P - 2); }

// plain reduction of lo + 2^64*hi (hi < 2^32) mod p — for delayed-reduction sums
TVM_HD u64 reduce96(u64 lo, u64 hi) {
  u64 t = hi * EPS;  // hi*(2^32-1) < 2^64
  u64 s = lo + t;
  if (s < t) s += EPS;  // wrapped: +2^64 = +EPS mod p; cannot wrap twice
  if (s >= P) s -= P;
  return s;
}

// x * 2^K mod p for a compile-time K in [0, 96); x canonical (works on any representation:
// (aR)*2^K = (a*2^K)R).  Uses 2^64 = 2^32 - 1, 2^96 = -1 (mod p).
template <int K>
TVM_HD u64 fmul_2k(u64 x) {
  static_assert(K >= 0 && K < 96, "K out of range");
  if (K == 0) return x;
  if (K < 32) {
    u64 lo = x << K, hi = x >> (64 - K);  // hi < 2^32
    return reduce96(lo, hi);
  } else if (K == 32) {
    // x*2^32 = (x_lo<<32) + x_hi*2^64 -> x_hi*(2^32-1)
    u64 lo = x << 32, hi = x >> 32;
    return reduce96(lo, hi);
  } else if (K < 64) {
    // x*2^K = lo(64) + mid*2^64 + top*2^96, with (x >> (64-K)) = mid + top*2^32
    u64 lo = x << K;
    u64 h = x >> (64 - K);           // < 2^K
    u64 mid = h & 0xFFFFFFFFULL, top = h >> 32;  // top < 2^(K-32)
    u64 r = reduce96(lo, mid);
    return fsub(r, top);
  } else {
    // K >= 64: x*2^K = (x*2^(K-64))*2^64; x*2^(K-64) = lo' + hi'*2^64 ->
    //   lo'*2^64 + hi'*2^128 ;  2^64 = eps, 2^128 = -2^32  (2^96=-1)
    constexpr int J = K - 64;        // 0..31
    u64 lo = J ? (x << J) : x;
    u64 hi = J ? (x >> (64 - J)) : 0;  // < 2^J <= 2^31
    // lo * 2^64: lo = l0 + l1*2^32 -> l0*eps + l1*2^96 = l0*eps - l1
    u64 l0 = lo & 0xFFFFFFFFULL, l1 = lo >> 32;
    u64 r = fsub(l0 * EPS, l1);      // l0*eps < 2^64, may be >= p? l0*eps <= (2^32-1)^2 < p ok
    // hi * 2^128 = -hi*2^32
    return fsub(r, hi << 32);
  }
}

// ---- X-field --------------------------------------------------------------------------
struct xfe {
  u64 c0, c1, c2;
};
TVM_HD xfe xmake(u64 a, u64 b, u64 c) { xfe r; r.c0 = a; r.c1 = b; r.c2 = c; return r; }
TVM_HD xfe xzero() { return xmake(0, 0, 0); }
TVM_HD xfe xone() { return xmake(MONT_ONE, 0, 0); }
TVM_HD xfe xlift(u64 b) { return xmake(b, 0, 0); }
TVM_HD xfe xadd(xfe a, xfe b) { return xmake(fadd(a.c0, b.c0), fadd(a.c1, b.c1), fadd(a.c2, b.c2)); }
TVM_HD xfe xsub(xfe a, xfe b) { return xmake(fsub(a.c0, b.c0), fsub(a.c1, b.c1), fsub(a.c2, b.c2)); }
TVM_HD xfe xneg(xfe a) { return xmake(fneg(a.c0), fneg(a.c1), fneg(a.c2)); }
TVM_HD xfe xaddb(xfe a, u64 b) { return xmake(fadd(a.c0, b), a.c1, a.c2); }
TVM_HD xfe xsubb(xfe a, u64 b) { return xmake(fsub(a.c0, b), a.c1, a.c2); }
TVM_HD xfe xmulb(xfe a, u64 b) { return xmake(fmul(a.c0, b), fmul(a.c1, b), fmul(a.c2, b)); }
TVM_HD xfe xmul(xfe a, xfe b) {
  u64 d0 = fmul(a.c0, b.c0);
  u64 d1 = fadd(fmul(a.c0, b.c1), fmul(a.c1, b.c0));
  u64 d2 = fadd(fadd(fmul(a.c0, b.c2), fmul(a.c1, b.c1)), fmul(a.c2, b.c0));
  u64 d3 = fadd(fmul(a.c1, b.c2), fmul(a.c2, b.c1));
  u64 d4 = fmul(a.c2, b.c2);
  return xmake(fsub(d0, d3), fsub(fadd(d1, d3), d4), fadd(d2, d4));
}
TVM_HD bool xeq(xfe a, xfe b) { return a.c0 == b.c0 && a.c1 == b.c1 && a.c2 == b.c2; }
TVM_HD bool xis_zero(xfe a) { return (a.c0 | a.c1 | a.c2) == 0; }

// Inverse via the norm to the base field: for a in F_p^3, a^-1 = a^(p) a^(p^2) / N(a).
// Implemented with the adjugate of the multiplication-by-a matrix (no Frobenius tables).
TVM_HD xfe xinv(xfe a) {
  // columns of M: a*1, a*X, a*X^2 ;  X^3 = X - 1
  //   a*X   = (-a2, a0 + a2, a1)
  //   a*X^2 = (-a1, a1... ) computed by applying the same map again
  u64 m00 = a.c0, m10 = a.c1, m20 = a.c2;
  u64 m01 = fneg(a.c2), m11 = fadd(a.c0, a.c2), m21 = a.c1;
  u64 m02 = fneg(m21), m12 = fadd(m01, m21), m22 = m11;
  // first column of adj(M)/det solves M y = e0:  y = (C00, C01, C02)/det with cofactors of row 0
  u64 c00 = fsub(fmul(m11, m22), fmul(m12, m21));
  u64 c01 = fsub(fmul(m12, m20), fmul(m10, m22));
  u64 c02 = fsub(fmul(m10, m21), fmul(m11, m20));
  u64 det = fadd(fadd(fmul(m00, c00), fmul(m01, c01)), fmul(m02, c02));
  u64 di = finv(det);
  return xmake(fmul(c00, di), fmul(c01, di), fmul(c02, di));
}
TVM_HD xfe xpow(xfe a, u64 e) {
  xfe r = xone();
  while (e) {
    if (e & 1) r = xmul(r, a);
    a = xmul(a, a);
    e >>= 1;
  }
  return r;
}

}  // namespace tvm
