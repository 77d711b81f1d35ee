// Tip5 row hashing and Merkle tree construction for sm_90a.
//
// Reference behaviour: every low-degree-test-domain row of a master table is hashed with
// Tip5::hash_varlen (master_table.rs:455-465; quotient segments stark.rs:425-446), the digests
// are the leaves of MerkleTree::par_new (master_table.rs:443-453): node i = hash_pair(node 2i,
// node 2i+1), root = node 1, leaf j = node n + j (SURVEY.md A.4).  FRI codeword trees use the
// unhashed leaf Digest::from(xfe) = (c0,c1,c2,0,0) (fri.rs:343-347, 927-929).
//
// Mapping: rows and inner nodes go through the IMMA permutation, four lanes per state and two states
// per lane quad.  Thread-per-node kernels (the whole state in one thread's registers) handle Merkle
// levels narrower than 64 nodes and the top of the tree.
#include <cstdint>
#include "ctx.h"
#include "tip5.cuh"
#include "tip5_constants.inc"

namespace tvm {

const u64 TIP5_ROUND_CONSTANTS_HOST[80] = {TVM_TIP5_RC_MONT};
const unsigned char TIP5_LOOKUP_HOST[256] = {TVM_TIP5_LUT};
__constant__ u64 c_tip5_rc[80] = {TVM_TIP5_RC_MONT};
__constant__ unsigned char c_tip5_lut[256] = {TVM_TIP5_LUT};

struct DevLut {
  const unsigned char *s;
  __device__ __forceinline__ unsigned char operator()(unsigned i) const { return s[i]; }
};
struct DevRc {
  __device__ __forceinline__ u64 operator()(int i) const { return c_tip5_rc[i]; }
};

__device__ __forceinline__ void tip5_perm_dev(u64 (&s)[16], const unsigned char *lut_smem) {
  tip5_permutation_generic(s, DevLut{lut_smem}, DevRc{});
}

static constexpr int HASH_THREADS = 128;

// Row index mapping: the LDE tables are coset-major ([col][coset][k], row i = coset + r*k).
// `log_r` = log2(#cosets); log_r = 0 means plain row-major-in-index ([col][i]).
struct HashRowsParams {
  const u64 *table;     // column q at table + q*col_stride
  size_t col_stride;
  size_t nrows;         // total rows (all cosets)
  unsigned ncols;
  int log_r;
  u64 *digests;         // [nrows][5], natural row order
  unsigned coset_mem_stride;   // rows of coset c are read from table coset c * coset_mem_stride
};

// nodes: [2*nleaves][5]; computes nodes[lo .. lo+count) from their children.
__global__ void __launch_bounds__(HASH_THREADS) merkle_level_kernel(u64 *nodes, size_t lo, size_t count) {
  __shared__ unsigned char lut[256];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) lut[i] = c_tip5_lut[i];
  __syncthreads();
  size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= count) return;
  size_t i = lo + t;
  const u64 *ch = nodes + 10 * i;  // children 2i, 2i+1 are adjacent: 10 words
  u64 s[16];
#pragma unroll
  for (int k = 0; k < 10; k++) s[k] = ch[k];
#pragma unroll
  for (int k = 10; k < 16; k++) s[k] = MONT_ONE;
  tip5_perm_dev(s, lut);
#pragma unroll
  for (int k = 0; k < 5; k++) nodes[5 * i + k] = s[k];
}

// The last levels (<= 2*HASH_THREADS nodes wide) in one CTA.
__global__ void __launch_bounds__(HASH_THREADS) merkle_top_kernel(u64 *nodes, size_t top_width) {
  __shared__ unsigned char lut[256];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) lut[i] = c_tip5_lut[i];
  __syncthreads();
  for (size_t w = top_width; w >= 1; w >>= 1) {
    for (size_t t = threadIdx.x; t < w; t += blockDim.x) {
      size_t i = w + t;
      const u64 *ch = nodes + 10 * i;
      u64 s[16];
#pragma unroll
      for (int k = 0; k < 10; k++) s[k] = ch[k];
#pragma unroll
      for (int k = 10; k < 16; k++) s[k] = MONT_ONE;
      tip5_perm_dev(s, lut);
#pragma unroll
      for (int k = 0; k < 5; k++) nodes[5 * i + k] = s[k];
    }
    __threadfence_block();
    __syncthreads();
  }
}

// leaves of an X-field codeword tree: Digest::from(xfe) = (c0, c1, c2, 0, 0).
// codeword is planar: coordinate d of element i at cw[d*stride + i].
__global__ void xfe_leaves_kernel(const u64 *cw, size_t stride, size_t n, u64 *leaves) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  u64 *d = leaves + 5 * i;
  d[0] = cw[i]; d[1] = cw[stride + i]; d[2] = cw[2 * stride + i]; d[3] = 0; d[4] = 0;
}

// ---- four lanes per state, two states per lane quad ---------------------------------------------
// Lane l of a quad holds elements {l, l+4, l+8, l+12} of each of its two states: slot 0 is a
// split-and-lookup element and slots 1..3 take x^7, so quad_sbox is divergence-free.
// split-and-lookup (tip-0005.md:52-61) of one 32-bit half: byte extraction and re-assembly with PRMT (the shift/mask/or
// form costs ~6 instructions per byte, this one 11 per four bytes); the looked-up values are zero-extended bytes, so
// "byte 1 of l" is a zero for the unused selector positions
__device__ __forceinline__ unsigned lookup_word(unsigned w, const unsigned char *lut) {
  const unsigned l0 = lut[w & 0xFF], l1 = lut[__byte_perm(w, 0, 0x4441)], l2 = lut[__byte_perm(w, 0, 0x4442)], l3 = lut[w >> 24];
  return __byte_perm(__byte_perm(l0, l1, 0x1140), __byte_perm(l2, l3, 0x1140), 0x5410);
}
__device__ __forceinline__ u64 lookup_u64(u64 v, const unsigned char *lut) {
  return ((u64)lookup_word((unsigned)(v >> 32), lut) << 32) | lookup_word((unsigned)v, lut);
}
// x^7 (in Montgomery form: x^7 R^-6) of any representative < 2^64, by montyred's contract; the result is < 2^64
__device__ __forceinline__ u64 pow7(u64 x) {
  const u64 x2 = fsqr(x), x3 = fmul(x2, x), x4 = fsqr(x2);
  return fmul(x3, x4);
}
__device__ __forceinline__ void quad_sbox(u64 (&s)[4], const unsigned char *lut) {
  s[0] = lookup_u64(s[0], lut);   // slot 0: split-and-lookup (canonical input)
#pragma unroll
  for (int i = 1; i < 4; i++) s[i] = pow7(s[i]);
}

// ---- MDS on the tensor cores: IMMA.16832.U8.U8 -----------------------------------------------------
// The linear layer y = M x (tip-0005.md:100-104) is a dense 16x16 integer matrix product applied to every state:
// the one dense contraction on the prover's path.  M's entries are 16-bit and the state words 64-bit, so with
// byte limbs  x_e = sum_s 2^(8s) X_s[e],  M = M_0 + 2^8 M_1  the product is
//     y_o = sum_{s=0..8} 2^(8s) T_s[o],      T_s = M_0 X_s + M_1 X_{s-1}      (X_{-1} = X_8 = 0, T_s < 2^21),
// and T_s for 16 states x 8 outputs is exactly one mma.sync.m16n8k32 (u8 x u8 -> s32): K = 32 = 16 state elements x
// {limb s against M_0, limb s-1 against M_1}.  Layout: the quad layout above with two rows per quad
// IS the IMMA A-fragment layout (fragment row g / g+8 = first / second row of quad g, fragment k = 4l+t = element
// l+4t of lane l), and choosing the B-fragment column order as o(j, n) = (n >> 1) + 4 (2j + (n & 1)) makes the
// D fragment of N-block j land on the lane that owns the output element: c0/c1 = elements l+8j, l+8j+4 of the first row,
// c2/c3 of the second.  No shuffles, 18 IMMA + 16 IMAD.WIDE and 32 IMAD (limb recombination) per lane and round instead of
// 256 IMAD.WIDE + 64 SHFL + 64 SEL.  The M_0 / M_1 fragments are 4 constant registers per lane.
__device__ __forceinline__ void imma_16832_u8(int (&d)[4], unsigned a0, unsigned a1, unsigned a2, unsigned a3, unsigned b0,
                                              unsigned b1) {
  asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.u8.u8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%10,%10,%10,%10};"
               : "=r"(d[0]), "=r"(d[1]), "=r"(d[2]), "=r"(d[3])
               : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1), "r"(0));
}
__device__ __forceinline__ u64 mad_wide(unsigned a, unsigned b, u64 c) {
  u64 d;
  asm("mad.wide.u32 %0, %1, %2, %3;" : "=l"(d) : "r"(a), "r"(b), "l"(c));
  return d;
}
struct MdsFrag { unsigned b[2][2]; };   // [N-block][k < 16 : k >= 16]
__constant__ unsigned short c_mds_col[16] = TVM_MDS_COL;
__constant__ unsigned c_pow256[4] = {1u, 1u << 8, 1u << 16, 1u << 24};
__device__ __forceinline__ MdsFrag mds_fragments(int lane) {
  const int g = lane >> 2, l = lane & 3;
  MdsFrag f;
#pragma unroll
  for (int j = 0; j < 2; j++) {
    const int o = (g >> 1) + 4 * (2 * j + (g & 1));
    unsigned lo = 0, hi = 0;
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const unsigned m = c_mds_col[(o - (l + 4 * i)) & 15];
      lo |= (m & 0xFF) << (8 * i);
      hi |= (m >> 8) << (8 * i);
    }
    f.b[j][0] = lo; f.b[j][1] = hi;
  }
  return f;
}
// bytes s of four 32-bit words -> one register per s
__device__ __forceinline__ void byte_transpose4(unsigned w0, unsigned w1, unsigned w2, unsigned w3, unsigned (&o)[4]) {
  const unsigned t01l = __byte_perm(w0, w1, 0x5140), t01h = __byte_perm(w0, w1, 0x7362);
  const unsigned t23l = __byte_perm(w2, w3, 0x5140), t23h = __byte_perm(w2, w3, 0x7362);
  o[0] = __byte_perm(t01l, t23l, 0x5410); o[1] = __byte_perm(t01l, t23l, 0x7632);
  o[2] = __byte_perm(t01h, t23h, 0x5410); o[3] = __byte_perm(t01h, t23h, 0x7632);
}
// V = lo + 2^32 hi + 2^64 top + rc  (lo, hi < 2^47, top < 2^21, rc < 2^64) folded to s + n 2^64 with s < 2^64, n in {0, 1}.
// Homogeneous carry chains (the compare/select code nvcc emits for the C formulation is ~45 instructions):
//   V = w0 + 2^32 w1 + 2^64 w2 (w2 < 2^23);  2^64 = 2^32 - 1 (mod p):  s + n 2^64 = (w0, w1) - w2 + 2^32 w2
//   (a borrow of the subtraction is always cancelled by the carry of the addition, so n is 0 or 1, and n = 1 means
//   s < 2^32 w2 < 2^55).
struct MdsFold { u64 s; unsigned n; };
__device__ __forceinline__ MdsFold mds_fold(u64 lo, u64 hi, unsigned top, u64 rc) {
  unsigned s0, s1, n;
  asm("{\n\t"
      ".reg .u32 l0, l1, h0, h1, r0, r1, w0, w1, w2, m;\n\t"
      "mov.b64 {l0, l1}, %3;\n\t"
      "mov.b64 {h0, h1}, %4;\n\t"
      "mov.b64 {r0, r1}, %6;\n\t"
      "add.cc.u32 w0, l0, r0;\n\t"
      "addc.cc.u32 w1, l1, r1;\n\t"
      "addc.u32 w2, h1, %5;\n\t"
      "add.cc.u32 w1, w1, h0;\n\t"
      "addc.u32 w2, w2, 0;\n\t"
      "sub.cc.u32 %0, w0, w2;\n\t"
      "subc.cc.u32 %1, w1, 0;\n\t"
      "subc.u32 m, 0, 0;\n\t"
      "add.cc.u32 %1, %1, w2;\n\t"
      "addc.u32 %2, m, 0;\n\t"
      "}"
      : "=r"(s0), "=r"(s1), "=r"(n)
      : "l"(lo), "l"(hi), "r"(top), "l"(rc));
  return {((u64)s1 << 32) | s0, n};
}
// canonical: s + n 2^64 - p if that is >= 0, else s  (u = s + (2^32 - 1), and the carry / n select).  For the look-up
// element and for whatever leaves the permutation.
__device__ __forceinline__ u64 mds_finish(u64 lo, u64 hi, unsigned top, u64 rc) {
  const MdsFold f = mds_fold(lo, hi, top, rc);
  u64 r;
  asm("{\n\t"
      ".reg .u32 s0, s1, u0, u1, k;\n\t"
      ".reg .pred q;\n\t"
      "mov.b64 {s0, s1}, %1;\n\t"
      "add.cc.u32 u0, s0, 0xffffffff;\n\t"
      "addc.cc.u32 u1, s1, 0;\n\t"
      "addc.u32 k, %2, 0;\n\t"
      "setp.ne.u32 q, k, 0;\n\t"
      "selp.u32 s0, u0, s0, q;\n\t"
      "selp.u32 s1, u1, s1, q;\n\t"
      "mov.b64 %0, {s0, s1};\n\t"
      "}"
      : "=l"(r)
      : "l"(f.s), "r"(f.n));
  return r;
}
// lazy: a representative < 2^64, s + n (2^32 - 1) (no wrap: n = 1 implies s < 2^55), for the elements that only feed
// the x^7 power map.  One IMAD.WIDE; the multiplier comes from constant memory so that ptxas keeps it one instruction.
__constant__ unsigned c_eps32 = 0xFFFFFFFFu;
__device__ __forceinline__ u64 mds_finish_lazy(u64 lo, u64 hi, unsigned top, u64 rc) {
  const MdsFold f = mds_fold(lo, hi, top, rc);
  u64 d;
  asm("mad.wide.u32 %0, %1, %2, %3;" : "=l"(d) : "r"(f.n), "r"(c_eps32), "l"(f.s));
  return d;
}
__device__ __forceinline__ void quad2_mds_mma(u64 (&a)[4], u64 (&b)[4], int l, const MdsFrag &f, const u64 *rc_smem, int rnd) {
  unsigned La[8], Lb[8];
  {
    unsigned o[4];
    byte_transpose4((unsigned)a[0], (unsigned)a[1], (unsigned)a[2], (unsigned)a[3], o);
#pragma unroll
    for (int i = 0; i < 4; i++) La[i] = o[i];
    byte_transpose4((unsigned)(a[0] >> 32), (unsigned)(a[1] >> 32), (unsigned)(a[2] >> 32), (unsigned)(a[3] >> 32), o);
#pragma unroll
    for (int i = 0; i < 4; i++) La[4 + i] = o[i];
    byte_transpose4((unsigned)b[0], (unsigned)b[1], (unsigned)b[2], (unsigned)b[3], o);
#pragma unroll
    for (int i = 0; i < 4; i++) Lb[i] = o[i];
    byte_transpose4((unsigned)(b[0] >> 32), (unsigned)(b[1] >> 32), (unsigned)(b[2] >> 32), (unsigned)(b[3] >> 32), o);
#pragma unroll
    for (int i = 0; i < 4; i++) Lb[4 + i] = o[i];
  }
  // Recombination y = sum_s 2^(8s) T_s (T_s < 2^21): pairs e = T_s + 2^8 T_{s+1} < 2^30 in 32 bits, then
  // lo = e_01 + 2^16 e_23 and hi = e_45 + 2^16 e_67 (< 2^47) with one IMAD.WIDE each; T_8 goes to mds_fold as the
  // 2^64 word.  2^8 and 2^16 come from constant memory, which neither nvcc nor ptxas folds: a literal power of two is
  // strength-reduced from one IMAD into ALU shifts and carry adds.
  const unsigned pw8 = c_pow256[1], pw16 = c_pow256[2];
  // [row a/b][t = 2j + c]
  u64 lo[2][4], hi[2][4];
  unsigned e0[2][4], e1[2][4], top[2][4];
#pragma unroll
  for (int s = 0; s <= 8; s++) {
    const unsigned a0 = s < 8 ? La[s] : 0u, a1 = s < 8 ? Lb[s] : 0u;
    const unsigned a2 = s > 0 ? La[s - 1] : 0u, a3 = s > 0 ? Lb[s - 1] : 0u;
#pragma unroll
    for (int j = 0; j < 2; j++) {
      int d[4];
      imma_16832_u8(d, a0, a1, a2, a3, f.b[j][0], f.b[j][1]);
#pragma unroll
      for (int c = 0; c < 4; c++) {
        const int row = c >> 1, t = 2 * j + (c & 1);
        const unsigned v = (unsigned)d[c];
        if (s == 8) top[row][t] = v;
        else if ((s & 3) == 0) e0[row][t] = v;
        else if ((s & 3) == 1) e0[row][t] += v * pw8;
        else if ((s & 3) == 2) e1[row][t] = v;
        else {
          const u64 w = mad_wide(e1[row][t] + v * pw8, pw16, (u64)e0[row][t]);
          if (s == 3) lo[row][t] = w;
          else hi[row][t] = w;
        }
      }
    }
  }
  // slot 0 feeds the next round's look-up and must be canonical; the x^7 slots take any representative < 2^64
#pragma unroll
  for (int t = 0; t < 4; t++) {
    const u64 rc = rc_smem[16 * rnd + l + 4 * t];
    if (t == 0) {
      a[t] = mds_finish(lo[0][t], hi[0][t], top[0][t], rc);
      b[t] = mds_finish(lo[1][t], hi[1][t], top[1][t], rc);
    } else {
      a[t] = mds_finish_lazy(lo[0][t], hi[0][t], top[0][t], rc);
      b[t] = mds_finish_lazy(lo[1][t], hi[1][t], top[1][t], rc);
    }
  }
}
// The state leaves in lazy form: slot 0 (elements 0..3) is canonical, slots 1..3 are representatives < 2^64.  Callers
// canonicalise what they store (fcanon); capacity elements stay lazy from one absorption to the next.
__device__ __forceinline__ void tip5_perm_quad2_mma(u64 (&a)[4], u64 (&b)[4], int l, const MdsFrag &f, const unsigned char *lut,
                                                    const u64 *rc_smem) {
#pragma unroll 1
  for (int rnd = 0; rnd < TIP5_ROUNDS; rnd++) {
    quad_sbox(a, lut);
    quad_sbox(b, lut);
    quad2_mds_mma(a, b, l, f, rc_smem, rnd);
  }
}

// Kernel-level check of the permutation's arithmetic pieces: in [n][5] = (x, lo, hi, top, rc), out [n][4] =
// (fsqr(x), pow7(x), mds_finish_lazy(lo, hi, top, rc), mds_finish(lo, hi, top, rc)).  Inputs outside the finish's
// bounds (lo, hi < 2^47, top < 2^21) are the caller's error.
__global__ void tip5_arith_check_kernel(const u64 *in, size_t n, u64 *out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const u64 *v = in + 5 * i;
  u64 *o = out + 4 * i;
  o[0] = fsqr(v[0]);
  o[1] = pow7(v[0]);
  o[2] = mds_finish_lazy(v[1], v[2], (unsigned)v[3], v[4]);
  o[3] = mds_finish(v[1], v[2], (unsigned)v[3], v[4]);
}
void tip5_arith_check_run(Ctx &c, const u64 *in, size_t n, u64 *out) {
  tip5_arith_check_kernel<<<(unsigned)((n + 127) / 128), 128, 0, c.stream>>>(in, n, out);
  c.launches++;
  TVM_CUDA(cudaGetLastError());
}

static constexpr int HASHM_THREADS = 128;   // 32 quads, 64 rows per CTA
__global__ void __launch_bounds__(HASHM_THREADS) tip5_hash_rows_mma_kernel(HashRowsParams p) {
  __shared__ unsigned char lut[256];
  __shared__ u64 rc[80];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) lut[i] = c_tip5_lut[i];
  for (int i = threadIdx.x; i < 80; i += blockDim.x) rc[i] = c_tip5_rc[i];
  __syncthreads();
  const int lane = threadIdx.x & 31, l = lane & 3;
  const MdsFrag f = mds_fragments(lane);
  constexpr int QUADS = HASHM_THREADS / 4;
  size_t mrow[2];
  bool active[2];
  const u64 *base[2];
#pragma unroll
  for (int t = 0; t < 2; t++) {
    size_t m = (size_t)blockIdx.x * (2 * QUADS) + (threadIdx.x >> 2) + (size_t)t * QUADS;
    active[t] = m < p.nrows;
    if (!active[t]) m = p.nrows - 1;                              // the whole warp takes part in the IMMA
    mrow[t] = m;
    const size_t per_ = p.nrows >> p.log_r, cs_ = m / per_;
    base[t] = p.table + m + cs_ * (p.coset_mem_stride - 1) * per_;
  }
  u64 a[4] = {0, 0, 0, 0}, b[4] = {0, 0, 0, 0};
  unsigned c = 0;
  for (; c + 10 <= p.ncols; c += 10) {
    a[0] = base[0][(size_t)(c + l) * p.col_stride];
    b[0] = base[1][(size_t)(c + l) * p.col_stride];
    a[1] = base[0][(size_t)(c + l + 4) * p.col_stride];
    b[1] = base[1][(size_t)(c + l + 4) * p.col_stride];
    if (l < 2) {
      a[2] = base[0][(size_t)(c + l + 8) * p.col_stride];
      b[2] = base[1][(size_t)(c + l + 8) * p.col_stride];
    }
    tip5_perm_quad2_mma(a, b, l, f, lut, rc);
  }
  unsigned rem = p.ncols - c;
#pragma unroll
  for (int i = 0; i < 3; i++) {
    unsigned e = (unsigned)(l + 4 * i);
    if (e < 10) {
      u64 va = 0, vb = 0;
      if (e < rem) { va = base[0][(size_t)(c + e) * p.col_stride]; vb = base[1][(size_t)(c + e) * p.col_stride]; }
      else if (e == rem) { va = MONT_ONE; vb = MONT_ONE; }
      a[i] = va; b[i] = vb;
    }
  }
  tip5_perm_quad2_mma(a, b, l, f, lut, rc);
  const size_t per = p.nrows >> p.log_r;
#pragma unroll
  for (int t = 0; t < 2; t++) {
    if (!active[t]) continue;
    size_t m = mrow[t];
    size_t coset = m / per, k = m - coset * per;
    u64 *d = p.digests + (coset + (k << p.log_r)) * 5;
    const u64 *s = t ? b : a;
    d[l] = s[0];
    if (l == 0) d[4] = fcanon(s[1]);
  }
}

// ---- the same kernel with the table tiles staged by the TMA engine ---------------------------------------------------
// One absorption reads a [10 columns][64 rows] tile of the column-major table: ten 512-byte runs.  Thread 0 hands them to
// the bulk-copy engine (cp.async.bulk.shared::cluster.global -> UBLKCP, completion counted on an mbarrier) two absorptions
// AHEAD of the permutation that consumes them: the loads of block b + 2 are in flight while block b is permuted, no lane
// spends address arithmetic or a scoreboard wait on them.  Rows of a tile column sit 68 words apart in shared memory
// (16-byte aligned destinations; the quad layout then reads it bank-conflict free).  Needs full CTAs (nrows, and rows per
// coset, multiples of 64) and 16-byte aligned columns; hash_rows_run falls back to the LDG kernel otherwise.
static constexpr int STAGE_PITCH = 68;
__device__ __forceinline__ unsigned smem_addr(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(u64 *bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(u64 *bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, unsigned bytes, u64 *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_addr(dst)), "l"(src),
               "r"(bytes), "r"(smem_addr(bar))
               : "memory");
}
__device__ __forceinline__ void mbar_wait(u64 *bar, unsigned parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "TVM_MBAR_WAIT:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra TVM_MBAR_DONE;\n\t"
      "bra TVM_MBAR_WAIT;\n\t"
      "TVM_MBAR_DONE:\n\t"
      "}" ::"r"(smem_addr(bar)),
      "r"(parity)
      : "memory");
}

__global__ void __launch_bounds__(HASHM_THREADS) tip5_hash_rows_mma_tma_kernel(HashRowsParams p) {
  __shared__ unsigned char lut[256];
  __shared__ u64 rc[80];
  __shared__ __align__(16) u64 stage[2][10][STAGE_PITCH];
  __shared__ __align__(8) u64 mbar[2];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) lut[i] = c_tip5_lut[i];
  for (int i = threadIdx.x; i < 80; i += blockDim.x) rc[i] = c_tip5_rc[i];
  const int lane = threadIdx.x & 31, l = lane & 3;
  const MdsFrag f = mds_fragments(lane);
  constexpr int QUADS = HASHM_THREADS / 4, ROWS = 2 * QUADS;
  const size_t per = p.nrows >> p.log_r;
  const size_t m0 = (size_t)blockIdx.x * ROWS, cs0 = m0 / per;
  const u64 *tile0 = p.table + m0 + cs0 * (p.coset_mem_stride - 1) * per;      // first row of the CTA's tile, column 0
  const unsigned full = p.ncols / 10, rem = p.ncols - 10 * full, nblk = full + 1;
  auto issue = [&](unsigned b) {                       // thread 0 only
    const unsigned cols = b < full ? 10u : rem;
    if (!cols) return;
    u64 *bar = &mbar[b & 1];
    mbar_expect_tx(bar, cols * ROWS * 8);
    for (unsigned i = 0; i < cols; i++) bulk_g2s(&stage[b & 1][i][0], tile0 + (size_t)(10 * b + i) * p.col_stride, ROWS * 8, bar);
  };
  if (threadIdx.x == 0) {
    mbar_init(&mbar[0], 1);
    mbar_init(&mbar[1], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    issue(0);
    if (nblk > 1) issue(1);
  }
  const int ra = threadIdx.x >> 2, rb = ra + QUADS;    // this quad's two rows inside the tile
  u64 a[4] = {0, 0, 0, 0}, b[4] = {0, 0, 0, 0};
  for (unsigned blk = 0; blk < nblk; blk++) {
    const unsigned cols = blk < full ? 10u : rem;
    const u64(*st)[STAGE_PITCH] = stage[blk & 1];
    if (cols) mbar_wait(&mbar[blk & 1], (blk >> 1) & 1);
    if (blk < full) {
      a[0] = st[l][ra]; b[0] = st[l][rb];
      a[1] = st[l + 4][ra]; b[1] = st[l + 4][rb];
      if (l < 2) { a[2] = st[l + 8][ra]; b[2] = st[l + 8][rb]; }
    } else {
#pragma unroll
      for (int i = 0; i < 3; i++) {
        const unsigned e = (unsigned)(l + 4 * i);
        if (e < 10) {
          u64 va = 0, vb = 0;
          if (e < rem) { va = st[e][ra]; vb = st[e][rb]; }
          else if (e == rem) { va = MONT_ONE; vb = MONT_ONE; }
          a[i] = va; b[i] = vb;
        }
      }
    }
    __syncthreads();                                   // every lane has taken its words out of this stage
    if (threadIdx.x == 0 && blk + 2 < nblk) {
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy reads before the async-proxy overwrite
      issue(blk + 2);
    }
    tip5_perm_quad2_mma(a, b, l, f, lut, rc);
  }
#pragma unroll
  for (int t = 0; t < 2; t++) {
    const size_t m = m0 + (size_t)(t ? rb : ra);
    const size_t coset = m / per, k = m - coset * per;
    u64 *d = p.digests + (coset + (k << p.log_r)) * 5;
    const u64 *s = t ? b : a;
    d[l] = s[0];
    if (l == 0) d[4] = fcanon(s[1]);
  }
}

// Inner tree nodes on the same permutation: a quad computes nodes lo + q and lo + q + count/2... (two nodes per quad).
__global__ void __launch_bounds__(HASHM_THREADS) merkle_level_mma_kernel(u64 *nodes, size_t lo, size_t count) {
  __shared__ unsigned char lut[256];
  __shared__ u64 rc[80];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) lut[i] = c_tip5_lut[i];
  for (int i = threadIdx.x; i < 80; i += blockDim.x) rc[i] = c_tip5_rc[i];
  __syncthreads();
  const int lane = threadIdx.x & 31, l = lane & 3;
  const MdsFrag f = mds_fragments(lane);
  constexpr int QUADS = HASHM_THREADS / 4;
  size_t node[2];
  bool active[2];
  u64 s[2][4];
#pragma unroll
  for (int t = 0; t < 2; t++) {
    size_t q = (size_t)blockIdx.x * (2 * QUADS) + (threadIdx.x >> 2) + (size_t)t * QUADS;
    active[t] = q < count;
    if (!active[t]) q = count - 1;
    node[t] = lo + q;
    const u64 *ch = nodes + 10 * node[t];          // children 2i, 2i+1 are adjacent: 10 words
    s[t][0] = ch[l];
    s[t][1] = ch[l + 4];
    s[t][2] = l < 2 ? ch[l + 8] : MONT_ONE;
    s[t][3] = MONT_ONE;
  }
  tip5_perm_quad2_mma(s[0], s[1], l, f, lut, rc);
#pragma unroll
  for (int t = 0; t < 2; t++) {
    if (!active[t]) continue;
    u64 *d = nodes + 5 * node[t];
    d[l] = s[t][0];
    if (l == 0) d[4] = fcanon(s[t][1]);
  }
}

void hash_rows_run(Ctx &c, const u64 *table, size_t col_stride, size_t nrows, unsigned ncols, int log_r, u64 *digests,
                   unsigned coset_mem_stride) {
  HashRowsParams p{table, col_stride, nrows, ncols, log_r, digests, coset_mem_stride};
  const size_t rows_per_cta = HASHM_THREADS / 2;
  unsigned grid = (unsigned)((nrows + rows_per_cta - 1) / rows_per_cta);
  const size_t per = nrows >> log_r;
  const bool tma_ok = nrows % rows_per_cta == 0 && per % rows_per_cta == 0 && ((uintptr_t)table % 16) == 0 &&
                      (col_stride * sizeof(u64)) % 16 == 0;
  if (tma_ok) tip5_hash_rows_mma_tma_kernel<<<grid, HASHM_THREADS, 0, c.stream>>>(p);
  else tip5_hash_rows_mma_kernel<<<grid, HASHM_THREADS, 0, c.stream>>>(p);
  c.launches++;
  TVM_CUDA(cudaGetLastError());
}

static void merkle_level_launch(Ctx &c, u64 *nodes, size_t lo, size_t count) {
  if (count < 64) {
    unsigned grid = (unsigned)((count + HASH_THREADS - 1) / HASH_THREADS);
    merkle_level_kernel<<<grid, HASH_THREADS, 0, c.stream>>>(nodes, lo, count);
  } else {
    const size_t per_cta = HASHM_THREADS / 2;
    unsigned grid = (unsigned)((count + per_cta - 1) / per_cta);
    merkle_level_mma_kernel<<<grid, HASHM_THREADS, 0, c.stream>>>(nodes, lo, count);
  }
  c.launches++;
}

// leaves already stored at nodes[nleaves .. 2*nleaves)
// (measured and rejected: the levels of width <= 4096 / <= 512 fused into ONE launch of a single 1024-thread CTA on the
// IMMA permutation made a STIR prove slower than one launch per level: one SM against all of them.)
void merkle_run(Ctx &c, u64 *nodes, size_t nleaves) {
  size_t w = nleaves / 2;
  const size_t TOP = 64;
  for (; w > TOP; w >>= 1) {
    merkle_level_launch(c, nodes, w, w);
  }
  if (w >= 1) {
    merkle_top_kernel<<<1, HASH_THREADS, 0, c.stream>>>(nodes, w);
    c.launches++;
  }
  TVM_CUDA(cudaGetLastError());
}

// Multi-GPU: rank g builds only the subtree rooted at node W + g (its 1/W of every level of width >= W); the W
// subtree roots are all-gathered in place (node W + g sits at nodes + 5*(W + g)) and the top of the tree is built by
// every rank.  Node ownership for the authentication paths: gather_digests_run(log_w, rank).
void merkle_run_sharded(Ctx &c, u64 *nodes, size_t nleaves, unsigned rank, unsigned W) {
  if (W <= 1 || nleaves < 2 * (size_t)W) { merkle_run(c, nodes, nleaves); return; }
  for (size_t w = nleaves / 2; w >= W; w >>= 1) {
    const size_t cnt = w / W;
    merkle_level_launch(c, nodes, w + rank * cnt, cnt);
  }
  TVM_CUDA(cudaGetLastError());
  c.all_gather(nodes + 5 * (size_t)W, 40);
  if (W >= 2) {
    merkle_top_kernel<<<1, HASH_THREADS, 0, c.stream>>>(nodes, W / 2);
    c.launches++;
  }
  TVM_CUDA(cudaGetLastError());
}

void xfe_leaves_run(Ctx &c, const u64 *cw, size_t stride, size_t n, u64 *leaves) {
  xfe_leaves_kernel<<<(unsigned)((n + 255) / 256), 256, 0, c.stream>>>(cw, stride, n, leaves);
  c.launches++;
  TVM_CUDA(cudaGetLastError());
}

// ---- host Tip5 (transcript) -------------------------------------------------------------
struct HostLutF { unsigned char operator()(unsigned i) const { return TIP5_LOOKUP_HOST[i]; } };
struct HostRcF { u64 operator()(int i) const { return TIP5_ROUND_CONSTANTS_HOST[i]; } };

void tip5_permutation_host(u64 s[16]) {
  u64(&st)[16] = *reinterpret_cast<u64(*)[16]>(s);
  tip5_permutation_generic(st, HostLutF{}, HostRcF{});
}
void tip5_round_host(u64 s[16], int rnd) {
  u64(&st)[16] = *reinterpret_cast<u64(*)[16]>(s);
  tip5_round_generic(st, rnd, HostLutF{}, HostRcF{});
}
void tip5_hash_varlen_host(const u64 *w, size_t n, u64 digest[5]) {
  u64 s[16] = {0};
  size_t full = n / 10;
  for (size_t i = 0; i < full; i++) {
    for (int k = 0; k < 10; k++) s[k] = w[10 * i + k];
    tip5_permutation_host(s);
  }
  size_t rem = n - 10 * full;
  for (size_t k = 0; k < 10; k++) s[k] = k < rem ? w[10 * full + k] : (k == rem ? MONT_ONE : 0);
  tip5_permutation_host(s);
  for (int k = 0; k < 5; k++) digest[k] = s[k];
}
void tip5_hash_pair_host(const u64 l[5], const u64 r[5], u64 digest[5]) {
  u64 s[16];
  for (int k = 0; k < 5; k++) { s[k] = l[k]; s[5 + k] = r[k]; }
  for (int k = 10; k < 16; k++) s[k] = MONT_ONE;
  tip5_permutation_host(s);
  for (int k = 0; k < 5; k++) digest[k] = s[k];
}

}  // namespace tvm
