// Tip5 row hashing and Merkle tree construction for sm_90a.
//
// Reference behaviour: every low-degree-test-domain row of a master table is hashed with
// Tip5::hash_varlen (master_table.rs:455-465; quotient segments stark.rs:425-446), the digests
// are the leaves of MerkleTree::par_new (master_table.rs:443-453): node i = hash_pair(node 2i,
// node 2i+1), root = node 1, leaf j = node n + j (SURVEY.md A.4).  FRI codeword trees use the
// unhashed leaf Digest::from(xfe) = (c0,c1,c2,0,0) (fri.rs:343-347, 927-929).
//
// Mapping: one thread per row with the 16-lane sponge state resident in registers for the
// whole absorb loop (all 5 rounds fused; no state traffic), tables stored column-major so that
// a warp's loads of one column are a single coalesced 256-byte segment.  The S-box lookup table
// lives in shared memory; the round constants in constant memory (warp-uniform index).
#include <cstdint>
#include <cstdlib>
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

__global__ void __launch_bounds__(HASH_THREADS) tip5_hash_rows_kernel(HashRowsParams p) {
  __shared__ unsigned char lut[256];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) lut[i] = c_tip5_lut[i];
  __syncthreads();
  size_t m = (size_t)blockIdx.x * blockDim.x + threadIdx.x;  // memory-order index within a column
  if (m >= p.nrows) return;
  // memory index m = coset * (nrows >> log_r) + k  <->  row i = coset + (k << log_r)
  size_t per = p.nrows >> p.log_r;
  size_t coset = m / per, k = m - coset * per;
  size_t row = coset + (k << p.log_r);
  const u64 *base = p.table + m;
  u64 s[16];
#pragma unroll
  for (int i = 0; i < 16; i++) s[i] = 0;
  unsigned c = 0;
  for (; c + 10 <= p.ncols; c += 10) {
#pragma unroll
    for (int i = 0; i < 10; i++) s[i] = base[(size_t)(c + i) * p.col_stride];
    tip5_perm_dev(s, lut);
  }
  unsigned rem = p.ncols - c;
#pragma unroll
  for (int i = 0; i < 10; i++) {
    u64 v = 0;
    if ((unsigned)i < rem) v = base[(size_t)(c + i) * p.col_stride];
    else if ((unsigned)i == rem) v = MONT_ONE;
    s[i] = v;
  }
  tip5_perm_dev(s, lut);
  u64 *d = p.digests + row * 5;
#pragma unroll
  for (int i = 0; i < 5; i++) d[i] = s[i];
}

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


// ---- warp-resident variant: 4 lanes per row ---------------------------------------------------
// Lane l of a 4-lane group holds state elements {l, l+4, l+8, l+12}: every lane has one
// split-and-lookup element (slot 0) and three x^7 elements, so the S-box layer is divergence-free.
// The circulant MDS product gathers the 16 inputs by warp shuffle in a lane-rotated order
// (X[k] = x_{(k+l) mod 16}), which makes the matrix constants identical for all lanes
// (y_{l+4i} = sum_k M[(4i-k) mod 16] X[k]).  Compared with one thread per row this keeps the round
// body ~4x smaller (instruction-cache resident) and the register count low (more resident warps).
__device__ __forceinline__ u64 shfl64(u64 v, int src) {
  unsigned lo = __shfl_sync(0xffffffffu, (unsigned)v, src);
  unsigned hi = __shfl_sync(0xffffffffu, (unsigned)(v >> 32), src);
  return ((u64)hi << 32) | lo;
}

__device__ __forceinline__ void tip5_perm_quad(u64 (&s)[4], int l, int group_base, const unsigned char *lut, const u64 *rc_smem) {
  constexpr unsigned short MDS[16] = TVM_MDS_COL;
#pragma unroll 1
  for (int rnd = 0; rnd < TIP5_ROUNDS; rnd++) {
    {  // slot 0: split-and-lookup
      u64 v = s[0], o = 0;
#pragma unroll
      for (int b = 0; b < 8; b++) o |= (u64)lut[(unsigned)((v >> (8 * b)) & 0xFF)] << (8 * b);
      s[0] = o;
    }
#pragma unroll
    for (int i = 1; i < 4; i++) {
      u64 x = s[i], x2 = fmul(x, x), x3 = fmul(x2, x), x4 = fmul(x2, x2);
      s[i] = fmul(x3, x4);
    }
    u64 lo[4] = {0, 0, 0, 0}, hi[4] = {0, 0, 0, 0};
#pragma unroll
    for (int k = 0; k < 16; k++) {
      // this lane provides, to the lane l' that wants element (k + l') mod 16 with (k + l') mod 4 == l,
      // its slot ((k + ((l - k) & 3)) & 15) >> 2
      const int wrap = (((l - k) & 3) + (k & 3)) >> 2;          // 0 or 1
      const u64 provide = wrap ? s[((k >> 2) + 1) & 3] : s[k >> 2];
      const u64 X = shfl64(provide, group_base + ((k + l) & 3));
      const u64 xl = X & 0xFFFFFFFFULL, xh = X >> 32;
#pragma unroll
      for (int i = 0; i < 4; i++) {
        const u64 m = MDS[(4 * i - k) & 15];
        lo[i] += m * xl;
        hi[i] += m * xh;
      }
    }
#pragma unroll
    for (int i = 0; i < 4; i++) {
      u64 lsum = lo[i] + (hi[i] << 32);
      u64 carry = lsum < lo[i];
      u64 h = (hi[i] >> 32) + carry;
      s[i] = fadd(reduce96(lsum, h), rc_smem[16 * rnd + l + 4 * i]);
    }
  }
}

// ---- two rows per lane quad ---------------------------------------------------------------------
// The round of one state is a long FMA-pipe stretch (MDS: 128 IMAD.WIDE per lane) followed by
// ALU-pipe stretches (reductions, S-box bookkeeping); with every warp of an SM running the same
// stream the two pipes are used alternately rather than concurrently (ncu r01b: issue 54 %,
// `math_pipe_throttle` the top stall).  Each quad therefore carries two independent rows, half a
// round out of phase: the MDS of one state is scheduled together with the S-box of the other.
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
__device__ __forceinline__ void quad_sbox(u64 (&s)[4], const unsigned char *lut) {
  s[0] = lookup_u64(s[0], lut);   // slot 0: split-and-lookup
#pragma unroll
  for (int i = 1; i < 4; i++) {
    u64 x = s[i], x2 = fmul(x, x), x3 = fmul(x2, x), x4 = fmul(x2, x2);
    s[i] = fmul(x3, x4);
  }
}
__device__ __forceinline__ void quad_mds_rc(u64 (&s)[4], int l, int group_base, const u64 *rc_smem, int rnd) {
  constexpr unsigned short MDS[16] = TVM_MDS_COL;
  u64 lo[4] = {0, 0, 0, 0}, hi[4] = {0, 0, 0, 0};
#pragma unroll
  for (int k = 0; k < 16; k++) {
    const int wrap = (((l - k) & 3) + (k & 3)) >> 2;          // 0 or 1
    const u64 provide = wrap ? s[((k >> 2) + 1) & 3] : s[k >> 2];
    const u64 X = shfl64(provide, group_base + ((k + l) & 3));
    const u64 xl = X & 0xFFFFFFFFULL, xh = X >> 32;
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const u64 m = MDS[(4 * i - k) & 15];
      lo[i] += m * xl;
      hi[i] += m * xh;
    }
  }
#pragma unroll
  for (int i = 0; i < 4; i++) {
    u64 lsum = lo[i] + (hi[i] << 32);
    u64 carry = lsum < lo[i];
    u64 h = (hi[i] >> 32) + carry;
    s[i] = fadd(reduce96(lsum, h), rc_smem[16 * rnd + l + 4 * i]);
  }
}
// Same MDS step with the 16 inputs exchanged through shared memory instead of 32 shuffles + 32 selects (cost model:
// SHFL 4 clocks, SEL 2; LDS.64 ~2): the quad writes its state to a 20-word-strided slot (bank-conflict free: word index
// 20*s + e covers all 16 residues mod 16 for 4 consecutive quads, two wavefronts per 64-bit warp access) and every
// lane reads x_{(k+l) mod 16}.
static constexpr int XCH_STRIDE = 20;
__device__ __forceinline__ void quad_mds_rc_smem(u64 (&s)[4], int l, u64 *slot, const u64 *rc_smem, int rnd) {
  constexpr unsigned short MDS[16] = TVM_MDS_COL;
  __syncwarp();                                   // previous readers of this slot are done
#pragma unroll
  for (int i = 0; i < 4; i++) slot[l + 4 * i] = s[i];
  __syncwarp();
  u64 lo[4] = {0, 0, 0, 0}, hi[4] = {0, 0, 0, 0};
#pragma unroll
  for (int k = 0; k < 16; k++) {
    const u64 X = slot[(k + l) & 15];
    const u64 xl = X & 0xFFFFFFFFULL, xh = X >> 32;
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const u64 m = MDS[(4 * i - k) & 15];
      lo[i] += m * xl;
      hi[i] += m * xh;
    }
  }
#pragma unroll
  for (int i = 0; i < 4; i++) {
    u64 lsum = lo[i] + (hi[i] << 32);
    u64 carry = lsum < lo[i];
    u64 h = (hi[i] >> 32) + carry;
    s[i] = fadd(reduce96(lsum, h), rc_smem[16 * rnd + l + 4 * i]);
  }
}
template <bool SMEM>
__device__ __forceinline__ void quad_mds_sel(u64 (&s)[4], int l, int group_base, u64 *slot, const u64 *rc_smem, int rnd) {
  if (SMEM) quad_mds_rc_smem(s, l, slot, rc_smem, rnd);
  else quad_mds_rc(s, l, group_base, rc_smem, rnd);
}
template <bool SMEM>
__device__ __forceinline__ void tip5_perm_quad2x(u64 (&a)[4], u64 (&b)[4], int l, int group_base, const unsigned char *lut,
                                                 const u64 *rc_smem, u64 *slot_a, u64 *slot_b) {
  quad_sbox(a, lut);
#pragma unroll 1
  for (int rnd = 0; rnd < TIP5_ROUNDS - 1; rnd++) {
    quad_mds_sel<SMEM>(a, l, group_base, slot_a, rc_smem, rnd);
    quad_sbox(b, lut);
    quad_mds_sel<SMEM>(b, l, group_base, slot_b, rc_smem, rnd);
    quad_sbox(a, lut);
  }
  quad_mds_sel<SMEM>(a, l, group_base, slot_a, rc_smem, TIP5_ROUNDS - 1);
  quad_sbox(b, lut);
  quad_mds_sel<SMEM>(b, l, group_base, slot_b, rc_smem, TIP5_ROUNDS - 1);
}
__device__ __forceinline__ void tip5_perm_quad2(u64 (&a)[4], u64 (&b)[4], int l, int group_base, const unsigned char *lut,
                                                const u64 *rc_smem) {
  quad_sbox(a, lut);
#pragma unroll 1
  for (int rnd = 0; rnd < TIP5_ROUNDS - 1; rnd++) {
    quad_mds_rc(a, l, group_base, rc_smem, rnd);
    quad_sbox(b, lut);
    quad_mds_rc(b, l, group_base, rc_smem, rnd);
    quad_sbox(a, lut);
  }
  quad_mds_rc(a, l, group_base, rc_smem, TIP5_ROUNDS - 1);
  quad_sbox(b, lut);
  quad_mds_rc(b, l, group_base, rc_smem, TIP5_ROUNDS - 1);
}

static constexpr int HASHQ2_THREADS = 128;   // 32 quads, 64 rows per CTA
template <bool SMEM>
__global__ void __launch_bounds__(HASHQ2_THREADS) tip5_hash_rows_quad2_kernel(HashRowsParams p) {
  __shared__ unsigned char lut[256];
  __shared__ u64 rc[80];
  __shared__ u64 xch[SMEM ? 2 * (HASHQ2_THREADS / 4) * XCH_STRIDE : 1];
  u64 *slot_a = xch + (SMEM ? (threadIdx.x >> 2) * XCH_STRIDE : 0);
  u64 *slot_b = xch + (SMEM ? ((HASHQ2_THREADS / 4) + (threadIdx.x >> 2)) * XCH_STRIDE : 0);
  for (int i = threadIdx.x; i < 256; i += blockDim.x) lut[i] = c_tip5_lut[i];
  for (int i = threadIdx.x; i < 80; i += blockDim.x) rc[i] = c_tip5_rc[i];
  __syncthreads();
  const int lane = threadIdx.x & 31, l = lane & 3, group_base = lane & ~3;
  constexpr int QUADS = HASHQ2_THREADS / 4;
  size_t mrow[2];
  bool active[2];
  const u64 *base[2];
#pragma unroll
  for (int t = 0; t < 2; t++) {
    size_t m = (size_t)blockIdx.x * (2 * QUADS) + (threadIdx.x >> 2) + (size_t)t * QUADS;
    active[t] = m < p.nrows;
    if (!active[t]) m = p.nrows - 1;                              // keep the quad alive for the shuffles
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
    tip5_perm_quad2x<SMEM>(a, b, l, group_base, lut, rc, slot_a, slot_b);
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
  tip5_perm_quad2x<SMEM>(a, b, l, group_base, lut, rc, slot_a, slot_b);
  const size_t per = p.nrows >> p.log_r;
#pragma unroll
  for (int t = 0; t < 2; t++) {
    if (!active[t]) continue;
    size_t m = mrow[t];
    size_t coset = m / per, k = m - coset * per;
    u64 *d = p.digests + (coset + (k << p.log_r)) * 5;
    const u64 *s = t ? b : a;
    d[l] = s[0];
    if (l == 0) d[4] = s[1];
  }
}

// ---- MDS on the tensor cores: IMMA.16832.U8.U8 -----------------------------------------------------
// The linear layer y = M x (tip-0005.md:100-104) is a dense 16x16 integer matrix product applied to every state:
// the one dense contraction on the prover's path.  M's entries are 16-bit and the state words 64-bit, so with
// byte limbs  x_e = sum_s 2^(8s) X_s[e],  M = M_0 + 2^8 M_1  the product is
//     y_o = sum_{s=0..8} 2^(8s) T_s[o],      T_s = M_0 X_s + M_1 X_{s-1}      (X_{-1} = X_8 = 0, T_s < 2^21),
// and T_s for 16 states x 8 outputs is exactly one mma.sync.m16n8k32 (u8 x u8 -> s32): K = 32 = 16 state elements x
// {limb s against M_0, limb s-1 against M_1}.  Layout: the quad layout of the kernels above with two rows per quad
// IS the IMMA A-fragment layout (fragment row g / g+8 = first / second row of quad g, fragment k = 4l+t = element
// l+4t of lane l), and choosing the B-fragment column order as o(j, n) = (n >> 1) + 4 (2j + (n & 1)) makes the
// D fragment of N-block j land on the lane that owns the output element: c0/c1 = elements l+8j, l+8j+4 of the first row,
// c2/c3 of the second.  No shuffles, 18 IMMA + 64 IMAD.WIDE (limb recombination) per lane and round instead of
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
// lo + 2^32 hi + rc  (lo < 2^46, hi < 2^54, rc canonical) reduced to canonical form.  Four homogeneous carry chains
// (16 instructions; the compare/select code nvcc emits for the C formulation is ~45):
//   V = lo + rc + (hi << 32) = w0 + 2^32 w1 + 2^64 w2 (w2 < 2^23);  2^64 = 2^32 - 1 (mod p):  s = (w0, w1) - w2 + 2^32 w2
//   tracked as s + n 2^64 with n in {0, 1} (a borrow of the subtraction is always cancelled by the carry of the addition);
//   result = s + n 2^64 - p if that is >= 0, else s:  u = s + (2^32 - 1) and the carry / n select.
__device__ __forceinline__ u64 mds_finish(u64 lo, u64 hi, u64 rc) {
  u64 r;
  asm("{\n\t"
      ".reg .u32 l0, l1, h0, h1, r0, r1, w0, w1, w2, s0, s1, m, n, u0, u1, k;\n\t"
      ".reg .pred q;\n\t"
      "mov.b64 {l0, l1}, %1;\n\t"
      "mov.b64 {h0, h1}, %2;\n\t"
      "mov.b64 {r0, r1}, %3;\n\t"
      "add.cc.u32 w0, l0, r0;\n\t"
      "addc.cc.u32 w1, l1, r1;\n\t"
      "addc.u32 w2, h1, 0;\n\t"
      "add.cc.u32 w1, w1, h0;\n\t"
      "addc.u32 w2, w2, 0;\n\t"
      "sub.cc.u32 s0, w0, w2;\n\t"
      "subc.cc.u32 s1, w1, 0;\n\t"
      "subc.u32 m, 0, 0;\n\t"
      "add.cc.u32 s1, s1, w2;\n\t"
      "addc.u32 n, m, 0;\n\t"
      "add.cc.u32 u0, s0, 0xffffffff;\n\t"
      "addc.cc.u32 u1, s1, 0;\n\t"
      "addc.u32 k, n, 0;\n\t"
      "setp.ne.u32 q, k, 0;\n\t"
      "selp.u32 s0, u0, s0, q;\n\t"
      "selp.u32 s1, u1, s1, q;\n\t"
      "mov.b64 %0, {s0, s1};\n\t"
      "}"
      : "=l"(r)
      : "l"(lo), "l"(hi), "l"(rc));
  return r;
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
  // 2^8, 2^16, 2^24 from constant memory, which neither nvcc nor ptxas folds: a literal power of two is strength-reduced
  // from one IMAD.WIDE into SHL + HI + two carry adds
  const unsigned pw[4] = {1u, c_pow256[1], c_pow256[2], c_pow256[3]};
  // accumulators: [row a/b][t = 2j + c]
  u64 lo[2][4], hi[2][4];
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
        if (s == 0) lo[row][t] = v;
        else if (s < 4) lo[row][t] = mad_wide(v, pw[s], lo[row][t]);
        else if (s == 4) hi[row][t] = v;
        else if (s < 8) hi[row][t] = mad_wide(v, pw[s - 4], hi[row][t]);
        else hi[row][t] += (u64)v << 32;
      }
    }
  }
#pragma unroll
  for (int t = 0; t < 4; t++) {
    const u64 rc = rc_smem[16 * rnd + l + 4 * t];
    a[t] = mds_finish(lo[0][t], hi[0][t], rc);
    b[t] = mds_finish(lo[1][t], hi[1][t], rc);
  }
}
__device__ __forceinline__ void tip5_perm_quad2_mma(u64 (&a)[4], u64 (&b)[4], int l, const MdsFrag &f, const unsigned char *lut,
                                                    const u64 *rc_smem) {
#pragma unroll 1
  for (int rnd = 0; rnd < TIP5_ROUNDS; rnd++) {
    quad_sbox(a, lut);
    quad_sbox(b, lut);
    quad2_mds_mma(a, b, l, f, rc_smem, rnd);
  }
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
    if (l == 0) d[4] = s[1];
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
    if (l == 0) d[4] = s[1];
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
    if (l == 0) d[4] = s[t][1];
  }
}

// ---- two lanes per row ------------------------------------------------------------------------------
// Measured cost model (tools/microbench/field_ops.cu, SMSP-clocks per warp instruction group): the MDS step
// of the 4-lane layout costs 635 per round against 355 for the three x^7 - its 32 shuffles (4 clocks
// each) and 32 selects are paid by every lane for a quarter of a state.  With two lanes per row, lane l
// holding elements {l, l+2, ..., l+14} (slots 0,1 = split-and-lookup, slots 2..7 = x^7, again
// divergence-free), the rotated gather X[k] = x_{(k+l) mod 16} needs the partner only for odd k:
// 16 shuffles + 16 selects per lane for HALF a state, and the IMAD count per state is unchanged.
__device__ __forceinline__ void pair_sbox(u64 (&s)[8], const unsigned char *lut) {
#pragma unroll
  for (int j = 0; j < 2; j++) {
    u64 v = s[j], o = 0;
#pragma unroll
    for (int b = 0; b < 8; b++) o |= (u64)lut[(unsigned)((v >> (8 * b)) & 0xFF)] << (8 * b);
    s[j] = o;
  }
#pragma unroll
  for (int j = 2; j < 8; j++) {
    u64 x = s[j], x2 = fmul(x, x), x3 = fmul(x2, x), x4 = fmul(x2, x2);
    s[j] = fmul(x3, x4);
  }
}
__device__ __forceinline__ void pair_mds_rc(u64 (&s)[8], int l, const u64 *rc_smem, int rnd) {
  constexpr unsigned short MDS[16] = TVM_MDS_COL;
  u64 lo[8], hi[8];
#pragma unroll
  for (int i = 0; i < 8; i++) { lo[i] = 0; hi[i] = 0; }
#pragma unroll
  for (int k = 0; k < 16; k++) {
    u64 X;
    if ((k & 1) == 0) {
      X = s[k >> 1];                                           // own element k + l
    } else {
      // the partner wants x_{(k + l') mod 16}: lane 1 serves lane 0 with slot (k-1)/2, lane 0 serves lane 1
      // with slot ((k+1) mod 16)/2
      const u64 provide = l ? s[(k - 1) >> 1] : s[((k + 1) & 15) >> 1];
      unsigned plo = __shfl_xor_sync(0xffffffffu, (unsigned)provide, 1);
      unsigned phi = __shfl_xor_sync(0xffffffffu, (unsigned)(provide >> 32), 1);
      X = ((u64)phi << 32) | plo;
    }
    const u64 xl = X & 0xFFFFFFFFULL, xh = X >> 32;
#pragma unroll
    for (int i = 0; i < 8; i++) {
      const u64 m = MDS[(2 * i - k) & 15];
      lo[i] += m * xl;
      hi[i] += m * xh;
    }
  }
#pragma unroll
  for (int i = 0; i < 8; i++) {
    u64 lsum = lo[i] + (hi[i] << 32);
    u64 carry = lsum < lo[i];
    u64 h = (hi[i] >> 32) + carry;
    s[i] = fadd(reduce96(lsum, h), rc_smem[16 * rnd + l + 2 * i]);
  }
}
__device__ __forceinline__ void tip5_perm_pair(u64 (&s)[8], int l, const unsigned char *lut, const u64 *rc_smem) {
#pragma unroll 1
  for (int rnd = 0; rnd < TIP5_ROUNDS; rnd++) {
    pair_sbox(s, lut);
    pair_mds_rc(s, l, rc_smem, rnd);
  }
}

static constexpr int HASHP_THREADS = 128;    // 64 rows per CTA
__global__ void __launch_bounds__(HASHP_THREADS) tip5_hash_rows_pair_kernel(HashRowsParams p) {
  __shared__ unsigned char lut[256];
  __shared__ u64 rc[80];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) lut[i] = c_tip5_lut[i];
  for (int i = threadIdx.x; i < 80; i += blockDim.x) rc[i] = c_tip5_rc[i];
  __syncthreads();
  const int l = threadIdx.x & 1;
  size_t m = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 1;   // one row per 2 lanes
  const bool active = m < p.nrows;
  if (!active) m = p.nrows - 1;                                     // keep the pair alive for the shuffles
  const u64 *base = p.table + m;
  u64 s[8];
#pragma unroll
  for (int j = 0; j < 8; j++) s[j] = 0;
  unsigned c = 0;
  for (; c + 10 <= p.ncols; c += 10) {
#pragma unroll
    for (int j = 0; j < 5; j++) s[j] = base[(size_t)(c + l + 2 * j) * p.col_stride];
    tip5_perm_pair(s, l, lut, rc);
  }
  const unsigned rem = p.ncols - c;
#pragma unroll
  for (int j = 0; j < 5; j++) {
    const unsigned e = (unsigned)(l + 2 * j);
    u64 v = 0;
    if (e < rem) v = base[(size_t)(c + e) * p.col_stride];
    else if (e == rem) v = MONT_ONE;
    s[j] = v;
  }
  tip5_perm_pair(s, l, lut, rc);
  if (active) {
    const size_t per = p.nrows >> p.log_r;
    const size_t coset = m / per, k = m - coset * per;
    u64 *d = p.digests + (coset + (k << p.log_r)) * 5;
    d[l] = s[0];
    d[l + 2] = s[1];
    if (l == 0) d[4] = s[2];
  }
}

static constexpr int HASHQ_THREADS = 128;
__global__ void __launch_bounds__(HASHQ_THREADS) tip5_hash_rows_quad_kernel(HashRowsParams p) {
  __shared__ unsigned char lut[256];
  __shared__ u64 rc[80];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) lut[i] = c_tip5_lut[i];
  for (int i = threadIdx.x; i < 80; i += blockDim.x) rc[i] = c_tip5_rc[i];
  __syncthreads();
  const int lane = threadIdx.x & 31, l = lane & 3, group_base = lane & ~3;
  size_t m = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 2;   // one row per 4 lanes
  const bool active = m < p.nrows;
  if (!active) m = p.nrows - 1;                                     // keep the quad alive for the shuffles
  size_t per = p.nrows >> p.log_r;
  size_t coset = m / per, k = m - coset * per;
  size_t row = coset + (k << p.log_r);
  const u64 *base = p.table + m;
  u64 s[4] = {0, 0, 0, 0};
  unsigned c = 0;
  for (; c + 10 <= p.ncols; c += 10) {
    s[0] = base[(size_t)(c + l) * p.col_stride];
    s[1] = base[(size_t)(c + l + 4) * p.col_stride];
    if (l < 2) s[2] = base[(size_t)(c + l + 8) * p.col_stride];
    tip5_perm_quad(s, l, group_base, lut, rc);
  }
  unsigned rem = p.ncols - c;
#pragma unroll
  for (int i = 0; i < 3; i++) {
    unsigned e = (unsigned)(l + 4 * i);
    if (e < 10) {
      u64 v = 0;
      if (e < rem) v = base[(size_t)(c + e) * p.col_stride];
      else if (e == rem) v = MONT_ONE;
      s[i] = v;
    }
  }
  tip5_perm_quad(s, l, group_base, lut, rc);
  if (active) {
    u64 *d = p.digests + row * 5;
    d[l] = s[0];
    if (l == 0) d[4] = s[1];
  }
}

void hash_rows_run(Ctx &c, const u64 *table, size_t col_stride, size_t nrows, unsigned ncols, int log_r, u64 *digests,
                   unsigned coset_mem_stride) {
  HashRowsParams p{table, col_stride, nrows, ncols, log_r, digests, coset_mem_stride};
  static const bool use_thread_per_row = getenv("TVM_TIP5_THREAD_PER_ROW") != nullptr;
  static const bool use_imad_mds = getenv("TVM_TIP5_IMAD_MDS") != nullptr;   // A/B: the round-1 default (MDS on the integer pipe)
  if (!use_imad_mds && !use_thread_per_row && !getenv("TVM_TIP5_ONE_ROW_PER_QUAD") && !getenv("TVM_TIP5_TWO_LANES") &&
      !getenv("TVM_TIP5_SMEM_EXCHANGE")) {
    const size_t rows_per_cta = HASHM_THREADS / 2;
    unsigned grid = (unsigned)((nrows + rows_per_cta - 1) / rows_per_cta);
    static const bool no_tma = getenv("TVM_TIP5_NO_TMA") != nullptr;        // A/B: per-lane LDG instead of bulk-copy staging
    const size_t per = nrows >> log_r;
    const bool tma_ok = !no_tma && nrows % rows_per_cta == 0 && per % rows_per_cta == 0 && ((uintptr_t)table % 16) == 0 &&
                        (col_stride * sizeof(u64)) % 16 == 0;
    if (tma_ok) tip5_hash_rows_mma_tma_kernel<<<grid, HASHM_THREADS, 0, c.stream>>>(p);
    else tip5_hash_rows_mma_kernel<<<grid, HASHM_THREADS, 0, c.stream>>>(p);
  } else if (coset_mem_stride != 1) {   // of the A/B variants only quad2 knows about strided cosets
    const size_t rows_per_cta = HASHQ2_THREADS / 2;
    unsigned grid = (unsigned)((nrows + rows_per_cta - 1) / rows_per_cta);
    tip5_hash_rows_quad2_kernel<false><<<grid, HASHQ2_THREADS, 0, c.stream>>>(p);
  } else if (use_thread_per_row) {
    unsigned grid = (unsigned)((nrows + HASH_THREADS - 1) / HASH_THREADS);
    tip5_hash_rows_kernel<<<grid, HASH_THREADS, 0, c.stream>>>(p);
  } else if (getenv("TVM_TIP5_ONE_ROW_PER_QUAD")) {
    size_t threads = nrows * 4;
    unsigned grid = (unsigned)((threads + HASHQ_THREADS - 1) / HASHQ_THREADS);
    tip5_hash_rows_quad_kernel<<<grid, HASHQ_THREADS, 0, c.stream>>>(p);
  } else if (getenv("TVM_TIP5_TWO_LANES")) {   // A/B switch: measured 3 % slower than the default below at 2^20
    unsigned grid = (unsigned)((nrows * 2 + HASHP_THREADS - 1) / HASHP_THREADS);
    tip5_hash_rows_pair_kernel<<<grid, HASHP_THREADS, 0, c.stream>>>(p);
  } else {
    const size_t rows_per_cta = HASHQ2_THREADS / 2;
    unsigned grid = (unsigned)((nrows + rows_per_cta - 1) / rows_per_cta);
    // exchanging the MDS inputs through shared memory instead of shuffles measured 10 % SLOWER at 2^20 (191 vs 174 ms
    // for the main table): kept as an A/B switch only
    if (getenv("TVM_TIP5_SMEM_EXCHANGE")) tip5_hash_rows_quad2_kernel<true><<<grid, HASHQ2_THREADS, 0, c.stream>>>(p);
    else tip5_hash_rows_quad2_kernel<false><<<grid, HASHQ2_THREADS, 0, c.stream>>>(p);
  }
  c.launches++;
  TVM_CUDA(cudaGetLastError());
}

static void merkle_level_launch(Ctx &c, u64 *nodes, size_t lo, size_t count, bool thread_per_node) {
  if (thread_per_node || count < 64) {
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
  static const bool thread_per_node = getenv("TVM_TIP5_IMAD_MDS") != nullptr;
  for (; w > TOP; w >>= 1) {
    merkle_level_launch(c, nodes, w, w, thread_per_node);
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
    static const bool thread_per_node = getenv("TVM_TIP5_IMAD_MDS") != nullptr;
    merkle_level_launch(c, nodes, w + rank * cnt, cnt, thread_per_node);
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
