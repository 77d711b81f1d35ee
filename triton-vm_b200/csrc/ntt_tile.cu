// Round-2 NTT kernels: square two-round tiles with register-resident radix-R DFTs (R = 8, 16, 32).
//
// A transform of size n = n2 * n1 (reference semantics: ntt.cu header; call sites stark.rs:872-877,
// arithmetic_domain.rs:141-212, master_table.rs:258-322) is two passes over HBM/L2:
//   pass A: n1/T tiles; a tile is T adjacent strided rows (fixed j1, elements j = j1 + n1 j2) -> n2-point NTT over j2,
//           times the inter-pass twist, stored transposed (tmp[K n1 + j1]);
//   pass B: n2/T tiles of T contiguous rows of tmp -> n1-point NTT over j1, stored to natural order (k = K + n2 K_B).
// A tile row of M = R*R points is transformed in TWO rounds: thread (t, a) holds the R points j = a + R b in registers,
// does an R-point DFT whose twiddles are all powers of two (ntt_radix.cuh), multiplies by w_M^(a k2) and hands the
// results over through shared memory; thread (t, k2) then does the R-point DFT over a and owns X[k2 + R k1].  Per point
// and pass: one generic twiddle multiplication, one shared-memory round trip, no bit reversal (the register index
// permutation is free), against 3.3 rounds, 2.6 twiddles and the bit-reversed addressing of the radix-8 tiles in ntt.cu.
// The row index t occupies the low lane bits, so every warp-wide global access covers whole 32/64-byte runs of adjacent
// rows and the exchange buffer ((k2 (R+1) + a) T + t) is bank-conflict free in both directions.
//
// Pre-/post-operations fused into the passes (each costs what its arithmetic costs, no extra pass over memory):
//   * coset evaluation (LDE): pass A multiplies point j2 by S_c[j2] = w_{r n2}^(c j2) (a table of n2 entries per
//     coset) and folds the randomizer chunk (c'_j += w_r^c c'_{n+j}, j < fold_count); the factor w_{rn}^(c j1) that
//     remains of the coset shift is one more term in the twist exponent: twist = w_{rn}^(j1 (r K + c)).
//   * interpolation: pass B multiplies by n^-1 offset^k (the coefficients are kept pre-scaled by offset^k).
//   Both are geometric in k1 for a fixed thread: factor = base * step^k1, two table look-ups per thread and tile.
#include <algorithm>
#include <cstdint>
#include <cstdlib>
#include "ctx.h"
#include "launch.h"
#include "ntt_radix.cuh"

namespace tvm {

__device__ __forceinline__ u64 powtab_at(const PowTab &t, u64 e) {
  const u64 lo = __ldg(t.lo + (e & ((1ULL << t.shift) - 1)));
  const u64 hi = __ldg(t.hi + (e >> t.shift));
  return fmul(lo, hi);
}

// One batch of transforms, both passes: (column zz, coset yy) reads in[zz * in_col_stride + j], keeps its transposed
// intermediate at tmp[(zz * tmp_cosets + yy) n + K n1 + j1] and writes out[zz * out_col_stride + yy n + k].
struct TileJob {
  const u64 *in;
  u64 *tmp, *out;
  size_t in_col_stride, out_col_stride, n;
  unsigned tmp_cosets, log_n1, log_n2;
  const u64 *tw;             // w_MA^(+-e), e < MA = RA*RA (pass A); pass B reads w_MB^e = w_MA^(e MA/MB) from it
  // pass A pre-operation (coset evaluation)
  const u64 *prescale;       // [coset][n2]
  const u64 *fold_factor;    // [coset]
  unsigned fold_count;       // input elements at offset < fold_count receive + fold_factor * in[fold_offset + offset]
  size_t fold_offset;
  // pass A post-operation: twist Ga^(row (mula K + c)), c = coset_first + coset_step yy
  PowTab Ga;
  u64 exp_mask, mula;
  unsigned coset_first, coset_step;
  // pass B post-operation (POSTB = 2): scalar * Gb^(row + mulb K)
  PowTab Gb;
  u64 mulb, scalar;
};

// Work order of one persistent launch.  The batch is cut into pairs (a column group x a coset group) whose intermediate
// should stay in the L2 until pass B reads it; tickets are handed out as A_0 | A_1 B_0 | A_2 B_1 | ... | B_(P-1), so the
// A-tiles of pair p+1 run while the B-tiles of pair p wait for, and then consume, the last A-tiles of pair p.
struct TileSched {
  unsigned *sync;            // [0] next ticket, [1 + p] finished A-tiles of pair p; zeroed before every launch
  unsigned npairs, ncg;      // pair p: column group p / ncg, coset group p % ncg
  unsigned group, cos_per, ncols;
  unsigned nxa, nxb;         // A- and B-tiles per (column, coset)
};

struct TileTicket {
  bool a, live;              // live: the column exists (the last column group may be partial)
  unsigned pair, x, yy, zz;
};

__device__ __forceinline__ unsigned tile_ticket_count(const TileSched &s) {
  return s.npairs * s.group * s.cos_per * (s.nxa + s.nxb);
}

__device__ __forceinline__ TileTicket tile_ticket(const TileSched &s, unsigned t) {
  const unsigned sa = s.group * s.cos_per * s.nxa, sb = s.group * s.cos_per * s.nxb;
  TileTicket k;
  unsigned i;
  if (t < sa) {
    k.a = true; k.pair = 0; i = t;
  } else {
    const unsigned u = t - sa, q = u / (sa + sb), r = u % (sa + sb);
    const bool last = q + 1 == s.npairs;   // the last step holds B_(P-1) only
    k.a = !last && r < sa;
    k.pair = k.a ? q + 1 : q;
    i = k.a || last ? r : r - sa;
  }
  const unsigned nx = k.a ? s.nxa : s.nxb, yz = i / nx;
  k.x = i % nx;
  k.yy = (k.pair % s.ncg) * s.cos_per + yz % s.cos_per;
  k.zz = (k.pair / s.ncg) * s.group + yz / s.cos_per;
  k.live = k.zz < s.ncols;
  return k;
}

__device__ __forceinline__ unsigned tile_pair_a_count(const TileSched &s, unsigned pair) {
  const unsigned z0 = (pair / s.ncg) * s.group;
  return min(s.group, s.ncols - z0) * s.cos_per * s.nxa;
}

static constexpr int TILE_THREADS = 256;

// TMA bulk copies (cp.async.bulk, SASS UBLKCP) with mbarrier completion - used to stage the contiguous rows of a B-tile
__device__ __forceinline__ unsigned tile_smem_addr(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void tile_mbar_init(u64 *bar) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;\n\tfence.mbarrier_init.release.cluster;" ::"r"(tile_smem_addr(bar)) : "memory");
}
__device__ __forceinline__ void tile_mbar_expect_tx(u64 *bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(tile_smem_addr(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tile_bulk_g2s(void *dst, const void *src, unsigned bytes, u64 *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(tile_smem_addr(dst)), "l"(src),
               "r"(bytes), "r"(tile_smem_addr(bar))
               : "memory");
}
__device__ __forceinline__ void tile_mbar_wait(u64 *bar, unsigned parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "TVM_TILE_WAIT:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra TVM_TILE_DONE;\n\t"
      "bra TVM_TILE_WAIT;\n\t"
      "TVM_TILE_DONE:\n\t"
      "}" ::"r"(tile_smem_addr(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ unsigned tile_ld_acquire(const unsigned *p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void tile_red_release(unsigned *p, unsigned v) {
  asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// Thread 0 hands the T rows of B-tile k to the TMA engine: one bulk copy of M words per row into the exchange buffer's
// memory, row pitch M + 2 words (bank-conflict free for the (t, a) read-out).  The rows are pass-A output of pair k.pair:
// unless `block` is false (then nothing is issued and false returned) it first waits until every A-tile of that pair has
// released its completion.  The proxy fences order the A-tiles' generic stores (seen through the acquire) and this CTA's
// own generic accesses of ex before the copy's async-proxy reads and writes.
template <int LOGR>
__device__ __forceinline__ bool tile_stage_b(const TileJob &p, const TileSched &s, const TileTicket &k, u64 *ex, u64 *bar, bool block) {
  constexpr int R = 1 << LOGR, M = R * R, T = TILE_THREADS / R;
  const unsigned need = tile_pair_a_count(s, k.pair);
  const unsigned *done = s.sync + 1 + k.pair;
  if (!block && tile_ld_acquire(done) < need) return false;
  while (tile_ld_acquire(done) < need) __nanosleep(64);
  asm volatile("fence.proxy.async.global;\n\tfence.proxy.async.shared::cta;" ::: "memory");
  tile_mbar_expect_tx(bar, (unsigned)(T * M * sizeof(u64)));
  const u64 *src = p.tmp + ((size_t)k.zz * p.tmp_cosets + k.yy) * p.n + ((size_t)k.x * T) * M;
  for (int r = 0; r < T; r++) tile_bulk_g2s(ex + (size_t)r * (M + 2), src + (size_t)r * M, (unsigned)(M * sizeof(u64)), bar);
  return true;
}

// One tile of either pass.  HAS_A / HAS_B: which tile kinds this instance serves; when both passes use the same radix the
// kernel instantiates one body for both (is_a decided at run time around the loads and stores), so that the two unrolled
// DFT copies exist once in the kernel and not twice, which keeps the kernel's SASS near the size of one pass.
// Round 1: thread (t, a) holds the R points a + R b of row t (pass A: strided loads and the coset pre-scale; pass B: the
// staged rows in ex), R-point DFT, twiddle w_M^(a k2), exchange through ex; round 2: thread (t, k2) does the R-point DFT
// over a and owns X[k2 + R k1].  `mid` runs between the round-2 read-out of ex and the second DFT.  tw holds w_M'^e for
// M' = M 2^TWS (the roots are successive squares: w_M = w_M'^(2^TWS)).
template <int LOGR, int TWS, bool INV, bool PRE, int POSTB, bool HAS_A, bool HAS_B, class Mid>
__device__ __forceinline__ void tile_body(bool is_a_rt, const TileJob &p, const TileTicket &k, const u64 *tw, u64 *ex, u64 *bar,
                                          unsigned phase, Mid mid) {
  constexpr int R = 1 << LOGR, M = R * R, LOGT = 8 - LOGR, T = 1 << LOGT;
  const bool is_a = HAS_A && (!HAS_B || is_a_rt);
  const int tid = threadIdx.x, t = tid & (T - 1), a = tid >> LOGT;
  const size_t row = (size_t)k.x * T + t;
  const size_t tmp_off = ((size_t)k.zz * p.tmp_cosets + k.yy) * p.n;
  u64 v[R];
  if (is_a) {
    const u64 *in = p.in + (size_t)k.zz * p.in_col_stride;
    const size_t off0 = row + ((size_t)a << p.log_n1), step = (size_t)R << p.log_n1;
#pragma unroll
    for (int b = 0; b < R; b++) v[b] = in[off0 + b * step];
    if (PRE) {
      if (off0 < p.fold_count) v[0] = fadd(v[0], fmul(__ldg(p.fold_factor + k.yy), in[p.fold_offset + off0]));
      const u64 *S = p.prescale + (size_t)k.yy * M + a;
#pragma unroll
      for (int b = 0; b < R; b++) v[b] = fmul(v[b], __ldg(S + b * R));
    }
  } else {
    tile_mbar_wait(bar, phase);
    const u64 *st = ex + (size_t)t * (M + 2) + a;
#pragma unroll
    for (int b = 0; b < R; b++) v[b] = st[b * R];
  }
  dft_pow2<LOGR, INV>(v);
  __syncthreads();           // pass B: every staged row read before the exchange overwrites it
#pragma unroll
  for (int k2 = 0; k2 < R; k2++) {
    u64 z = v[bitrev_c(k2, LOGR)];
    if (k2) z = fmul(z, tw[(a * k2) << TWS]);   // a == 0: tw[0] = 1 (kept branch-free)
    ex[(k2 * (R + 1) + a) * T + t] = z;
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < R; i++) v[i] = ex[(a * (R + 1) + i) * T + t];
  mid();
  dft_pow2<LOGR, INV>(v);
  const int k2 = a;
  if (is_a) {
    // the intermediate is read again by pass B of this launch: plain stores, so that it stays in the L2
    u64 *out = p.tmp + tmp_off;
    const size_t ooff0 = row + ((size_t)k2 << p.log_n1), ostep = (size_t)R << p.log_n1;
    const u64 c = p.coset_first + p.coset_step * k.yy;
    u64 f = powtab_at(p.Ga, (row * (p.mula * k2 + c)) & p.exp_mask);
    const u64 st = powtab_at(p.Ga, (row * p.mula * R) & p.exp_mask);
#pragma unroll
    for (int k1 = 0; k1 < R; k1++) {
      out[ooff0 + k1 * ostep] = fmul(v[bitrev_c(k1, LOGR)], f);
      if (k1 + 1 < R) f = fmul(f, st);
    }
  } else {
    u64 *out = p.out + (size_t)k.zz * p.out_col_stride + (size_t)k.yy * p.n;
    const size_t ooff0 = row + ((size_t)k2 << p.log_n2), ostep = (size_t)R << p.log_n2;
    if (POSTB == 0) {
      // coset evaluation: the output is not read again by the LDE (st.global.cs = evict first)
#pragma unroll
      for (int k1 = 0; k1 < R; k1++) __stcs(out + ooff0 + k1 * ostep, v[bitrev_c(k1, LOGR)]);
    } else {
      u64 f = fmul(p.scalar, powtab_at(p.Gb, row + p.mulb * k2));
      const u64 st = powtab_at(p.Gb, p.mulb * R);
#pragma unroll
      for (int k1 = 0; k1 < R; k1++) {
        out[ooff0 + k1 * ostep] = fmul(v[bitrev_c(k1, LOGR)], f);
        if (k1 + 1 < R) f = fmul(f, st);
      }
    }
  }
}

// The persistent tile kernel: every CTA takes tickets (tile_ticket) until the batch is done.  Pass A of the ticket is
// LOGRA-radix, pass B LOGRB-radix; PRE: coset pre-scale and randomizer fold in pass A; POSTB: 0 none, 2 n^-1 offset^k.
// A CTA takes its next ticket right after the round-2 read-out of ex; when that is a B-tile whose pair is complete, it
// issues the tile's bulk copy into ex at once, so the load overlaps the second DFT and the stores of the current tile.
//
// Deadlock freedom: only B-tiles wait, and only for the A-tiles of their own pair, whose tickets precede them (A_p is
// handed out one step before B_p).  A ticket is held only by a CTA that is already running, and a CTA holding an A ticket
// finishes it without waiting on anything.  So every wait ends, however many CTAs are resident: one CTA is enough.
template <int LOGRA, int LOGRB, bool INV, bool PRE, int POSTB>
__global__ void __launch_bounds__(TILE_THREADS, 2) ntt_tile_kernel(TileJob p, TileSched s) {
  constexpr int MA = 1 << (2 * LOGRA);
  constexpr bool SAME = LOGRA == LOGRB;
  extern __shared__ __align__(16) u64 smem[];
  u64 *tw = smem;            // [MA], both passes
  u64 *ex = smem + MA;
  __shared__ __align__(8) u64 bulk_bar;
  __shared__ unsigned s_next, s_staged;
  const int tid = threadIdx.x;
  const unsigned total = tile_ticket_count(s);
  if (tid == 0) {
    tile_mbar_init(&bulk_bar);
    s_next = atomicAdd(s.sync, 1u);
    s_staged = 0;
  }
  for (int i = tid; i < MA; i += TILE_THREADS) tw[i] = __ldg(p.tw + i);
  __syncthreads();
  unsigned phase = 0;        // parity of the bulk barrier's current phase: one phase per B-tile
  for (;;) {
    const unsigned tk = s_next;
    if (tk >= total) break;
    const TileTicket k = tile_ticket(s, tk);
    const bool staged = s_staged;
    // next ticket, after every thread has read ex in round 2 (ex is free for the next B-tile's rows)
    auto mid = [&]() {
      __syncthreads();
      if (tid == 0) {
        const unsigned t2 = atomicAdd(s.sync, 1u);
        bool st = false;
        if (t2 < total) {
          const TileTicket k2 = tile_ticket(s, t2);
          if (!k2.a && k2.live) st = tile_stage_b<LOGRB>(p, s, k2, ex, &bulk_bar, false);
        }
        s_next = t2;
        s_staged = st;
      }
    };
    if (!k.live) {
      mid();
      __syncthreads();
      continue;
    }
    if (!k.a && !staged && tid == 0) tile_stage_b<LOGRB>(p, s, k, ex, &bulk_bar, true);
    if (SAME) {
      tile_body<LOGRA, 0, INV, PRE, POSTB, true, true>(k.a, p, k, tw, ex, &bulk_bar, phase, mid);
    } else if (k.a) {
      tile_body<LOGRA, 0, INV, PRE, POSTB, true, false>(true, p, k, tw, ex, &bulk_bar, phase, mid);
    } else {
      tile_body<LOGRB, 2 * (LOGRA - LOGRB), INV, PRE, POSTB, false, true>(false, p, k, tw, ex, &bulk_bar, phase, mid);
    }
    __syncthreads();         // the tile's stores are done; s_next / s_staged are visible
    if (k.a) {
      if (tid == 0) {
        asm volatile("fence.proxy.async.global;" ::: "memory");
        tile_red_release(s.sync + 1 + k.pair, 1u);
      }
    } else {
      phase ^= 1;
    }
  }
}

// randomizer fold-in after the interpolation (master_table.rs:392-403: interpolant + zerofier * randomizer, zerofier
// X^n - 1 on the trace domain): coef[k] -= rand[k] post^k, coef[n + k] = rand[k] post^(n + k), zero up to rand_pad.
__global__ void lde_randomizer_kernel(u64 *coef, size_t coef_stride, size_t n, const u64 *rand, unsigned rand_count,
                                      unsigned rand_pad, PowTab post) {
  const unsigned k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= rand_pad) return;
  u64 *c = coef + (size_t)blockIdx.y * coef_stride;
  if (k < rand_count) {
    const u64 r = rand[(size_t)blockIdx.y * rand_count + k];
    c[k] = fsub(c[k], fmul(r, powtab_at(post, k)));
    c[n + k] = fmul(r, powtab_at(post, n + k));
  } else {
    c[n + k] = 0;
  }
}

__global__ void prescale_table_kernel(u64 *S, u64 *ff, PowTab pre, unsigned log_n, unsigned log_n1, unsigned M, unsigned coset_first,
                                      unsigned coset_step, u64 exp_mask) {
  const unsigned i = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  const u64 c = coset_first + coset_step * y;
  if (i < M) S[(size_t)y * M + i] = powtab_at(pre, ((c << log_n1) * i) & exp_mask);
  if (i == 0) ff[y] = powtab_at(pre, (c << log_n) & exp_mask);
}

u64 *Ctx::get_prescale(unsigned log_n, unsigned log_r, unsigned log_n1, unsigned M, unsigned first, unsigned step, unsigned count,
                        const std::function<void(u64 *, u64 *)> &fill) {
  auto key = std::make_tuple(log_n, log_r, log_n1, M, first, step, count);
  auto it = prescale_tabs.find(key);
  if (it != prescale_tabs.end()) return it->second;
  u64 *d = (u64 *)alloc(((size_t)count * M + count) * sizeof(u64));
  fill(d, d + (size_t)count * M);
  prescale_tabs[key] = d;
  return d;
}

static int tile_logr(int log_m) { return (log_m == 6 || log_m == 8 || log_m == 10) ? log_m / 2 : 0; }

// bytes of transposed intermediate one pair may produce: pass B should find it in the L2 (50 MB on H100, shared with the
// pair whose A-tiles run meanwhile and with the streaming output).  Measured with the launch-pair kernels that preceded
// the persistent one (16 columns at 2^20, 8 cosets; H100 SXM 80 GB at a 700 W limit, one run each): 3.41 ms with 16 MB
// pairs, 3.52 ms with 32 MB, 4.00 ms with 8 MB.
static size_t tile_tmp_budget() {
  static const size_t mb = getenv("TVM_NTT_TMP_MB") ? (size_t)atoi(getenv("TVM_NTT_TMP_MB")) : 16;
  return std::max<size_t>(1, mb) << 20;
}

// Picks n = n2 * n1 with both factors in {2^6, 2^8, 2^10}; false if this size is left to ntt.cu's kernels.
bool ntt_tile_supported(int log_n, int *log_n2, int *log_n1) {
  static const bool off = getenv("TVM_NTT_RADIX8_TILES") != nullptr;   // A/B: the round-1 kernels
  if (off) return false;
  for (int la = 10; la >= 6; la -= 2) {
    const int lb = log_n - la;
    if (lb > la) return false;
    if (lb == 6 || lb == 8 || lb == 10) { *log_n2 = la; *log_n1 = lb; return true; }
  }
  return false;
}

// One persistent launch of both passes over the batch.  The grid is the number of CTAs that fit on the device at once
// (TVM_NTT_TILE_CTAS=k sets it to k instead, for tests of the pair waits; nothing else changes).
template <bool INV, bool PRE, int POSTB>
static void run_tiles(Ctx &c, int ra, int rb, const TileJob &j, TileSched s) {
  const size_t sa = (size_t)s.group * s.cos_per * s.nxa, sb = (size_t)s.group * s.cos_per * s.nxb;
  const size_t total = s.npairs * (sa + sb);
  if (total >= ((size_t)1 << 31)) throw CudaError{cudaErrorInvalidValue, __FILE__, __LINE__};
  auto ex_words = [](int lr, bool staged) {
    const size_t R = (size_t)1 << lr, T = TILE_THREADS / R;
    return std::max(R * (R + 1) * T, staged ? T * (R * R + 2) : 0);
  };
  const size_t smem = (((size_t)1 << (2 * ra)) + std::max(ex_words(ra, false), ex_words(rb, true))) * sizeof(u64);
  auto go = [&](auto kernel) {
    TVM_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    TVM_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, TILE_THREADS, smem));
    size_t grid = (size_t)std::max(1, per_sm) * (size_t)c.num_sms;
    if (const char *e = getenv("TVM_NTT_TILE_CTAS")) grid = std::max(1, atoi(e));
    grid = std::min(grid, total);
    if (c.tile_sync_words < s.npairs + 1) {
      if (c.tile_sync) c.free_tracked(c.tile_sync);
      c.tile_sync_words = std::max<size_t>(s.npairs + 1, 1024);
      c.tile_sync = (unsigned *)c.alloc(c.tile_sync_words * sizeof(unsigned));
    }
    s.sync = c.tile_sync;
    TVM_CUDA(cudaMemsetAsync(s.sync, 0, (s.npairs + 1) * sizeof(unsigned), c.stream));
    c.launches++;                            // the memset is a device operation of its own
    kernel<<<(unsigned)grid, TILE_THREADS, smem, c.stream>>>(j, s);
    c.launches++;
    TVM_CUDA(cudaGetLastError());
  };
  if (ra == 5 && rb == 5) go(ntt_tile_kernel<5, 5, INV, PRE, POSTB>);
  else if (ra == 3 && rb == 3) go(ntt_tile_kernel<3, 3, INV, PRE, POSTB>);
  else throw CudaError{cudaErrorInvalidValue, __FILE__, __LINE__};   // mixed radices take the launch pairs
}

struct PairJob {
  const u64 *in;
  u64 *out;
  size_t in_col_stride, in_coset_stride, out_col_stride, out_coset_stride;   // per blockIdx.z (column), blockIdx.y (coset)
  size_t in_row_stride, in_elem_stride, out_row_stride, out_elem_stride;     // element idx of row r at r*row + idx*elem
  const u64 *tw;             // w_M^(+-e), e < M = R*R
  // pre-operation (coset evaluation)
  const u64 *prescale;       // [gridDim.y][M] or nullptr
  const u64 *fold_factor;    // [gridDim.y]
  unsigned fold_count;       // input elements at offset < fold_count receive + fold_factor * in[fold_offset + offset]
  size_t fold_offset;
  // post-operation: 0 none; 1 twist G^(row (mul K + c_y)), c_y = coset_first + coset_step y; 2 scalar * G^(row + mul K)
  int post_mode;
  PowTab G;
  u64 exp_mask;
  u64 mul;
  unsigned coset_first, coset_step;
  u64 scalar;
};

// PRE: coset pre-scale + randomizer fold on the way in; POST: 0 none, 1 twist, 2 scalar * power on the way out (compile-time:
// the unused variants would otherwise double the unrolled code, ~100 KB of SASS, past the instruction cache)
// STREAM: second pass - its input is the intermediate that should live in L2 only (last use: ld.global.cs = evict first) and
// its output is not read again by the LDE (st.global.cs), so that the NEXT column's intermediate finds room in the L2.
// BULK: the tile's rows are contiguous in memory (second pass): thread 0 hands the T rows to the TMA engine (one bulk copy of
// M words per row into the exchange buffer's memory, row pitch M + 2 words: bank-conflict free for the (t, a) read-out), the
// CTA waits on the mbarrier and fills its registers from shared memory; no lane issues a global load.
template <int LOGR, bool INV, bool PRE, int POST, bool STREAM, bool BULK>
__global__ void __launch_bounds__(TILE_THREADS, 2) ntt_pair_kernel(PairJob p) {
  constexpr int R = 1 << LOGR, M = R * R, LOGT = 8 - LOGR, T = 1 << LOGT;
  extern __shared__ __align__(16) u64 smem[];
  u64 *tw = smem;            // [M]
  u64 *ex = smem + M;        // [(k2 (R+1) + a) T + t]
  const int tid = threadIdx.x, t = tid & (T - 1), a = tid >> LOGT;
  const size_t row = (size_t)blockIdx.x * T + t;
  const unsigned y = blockIdx.y;
  const u64 *in = p.in + (size_t)blockIdx.z * p.in_col_stride + (size_t)y * p.in_coset_stride;
  u64 *out = p.out + (size_t)blockIdx.z * p.out_col_stride + (size_t)y * p.out_coset_stride;
  __shared__ __align__(8) u64 bulk_bar;
  if (BULK) {
    if (tid == 0) tile_mbar_init(&bulk_bar);
    __syncthreads();
    if (tid == 0) {
      tile_mbar_expect_tx(&bulk_bar, (unsigned)(T * M * sizeof(u64)));
      const u64 *src = in + ((size_t)blockIdx.x * T) * p.in_row_stride;
      for (int r = 0; r < T; r++) tile_bulk_g2s(ex + (size_t)r * (M + 2), src + (size_t)r * p.in_row_stride, (unsigned)(M * sizeof(u64)), &bulk_bar);
    }
  }
  for (int i = tid; i < M; i += TILE_THREADS) tw[i] = __ldg(p.tw + i);

  u64 v[R];
#pragma unroll 2
  for (int rnd = 0; rnd < 2; rnd++) {
    if (rnd == 0) {
      const size_t off0 = row * p.in_row_stride + (size_t)a * p.in_elem_stride;
      const size_t step = (size_t)R * p.in_elem_stride;
      if (BULK) {
        tile_mbar_wait(&bulk_bar, 0);
        const u64 *st = ex + (size_t)t * (M + 2) + a;
#pragma unroll
        for (int b = 0; b < R; b++) v[b] = st[b * R];
      } else {
#pragma unroll
        for (int b = 0; b < R; b++) v[b] = STREAM ? __ldcs(in + off0 + b * step) : in[off0 + b * step];
      }
      if (PRE) {
        if (off0 < p.fold_count) v[0] = fadd(v[0], fmul(__ldg(p.fold_factor + y), in[p.fold_offset + off0]));
        const u64 *S = p.prescale + (size_t)y * M + a;
#pragma unroll
        for (int b = 0; b < R; b++) v[b] = fmul(v[b], __ldg(S + b * R));
      }
    } else {
      // second round: this thread owns outputs K = k2 + R k1 of row t, k2 = a
#pragma unroll
      for (int i = 0; i < R; i++) v[i] = ex[(a * (R + 1) + i) * T + t];
    }
    dft_pow2<LOGR, INV>(v);
    if (rnd == 0) {
      __syncthreads();           // tw[] complete
#pragma unroll
      for (int k2 = 0; k2 < R; k2++) {
        u64 z = v[bitrev_c(k2, LOGR)];
        if (k2) z = fmul(z, tw[a * k2]);          // a == 0: tw[0] = 1 (kept branch-free)
        ex[(k2 * (R + 1) + a) * T + t] = z;
      }
      __syncthreads();
    } else {
      const int k2 = a;
      const size_t ooff0 = row * p.out_row_stride + (size_t)k2 * p.out_elem_stride;
      const size_t ostep = (size_t)R * p.out_elem_stride;
      if (POST == 0) {
#pragma unroll
        for (int k1 = 0; k1 < R; k1++) {
          if (STREAM) __stcs(out + ooff0 + k1 * ostep, v[bitrev_c(k1, LOGR)]);
          else out[ooff0 + k1 * ostep] = v[bitrev_c(k1, LOGR)];
        }
      } else {
        u64 f, st;
        if (POST == 1) {
          const u64 c = p.coset_first + p.coset_step * y;
          f = powtab_at(p.G, (row * (p.mul * k2 + c)) & p.exp_mask);
          st = powtab_at(p.G, (row * p.mul * R) & p.exp_mask);
        } else {
          f = fmul(p.scalar, powtab_at(p.G, row + p.mul * k2));
          st = powtab_at(p.G, p.mul * R);
        }
#pragma unroll
        for (int k1 = 0; k1 < R; k1++) {
          const u64 o = fmul(v[bitrev_c(k1, LOGR)], f);
          if (STREAM) __stcs(out + ooff0 + k1 * ostep, o);
          else out[ooff0 + k1 * ostep] = o;
          if (k1 + 1 < R) f = fmul(f, st);
        }
      }
    }
  }
}

template <bool INV, bool PRE, int POST, bool STREAM>
static void launch_pair(int logr, dim3 grid, cudaStream_t s, const PairJob &j) {
  const int R = 1 << logr, M = R * R, T = TILE_THREADS / R;
  const size_t smem = ((size_t)M + (size_t)R * (R + 1) * T) * sizeof(u64);
  auto go = [&](auto kernel) {
    TVM_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kernel<<<grid, TILE_THREADS, smem, s>>>(j);
  };
  // contiguous, 16-byte aligned rows of exactly M words (every second pass): staged by the TMA engine
  const bool bulk = !PRE && j.in_elem_stride == 1 && j.in_row_stride == (size_t)M && ((uintptr_t)j.in % 16) == 0 &&
                    (j.in_col_stride * 8) % 16 == 0 && (j.in_coset_stride * 8) % 16 == 0;
  if (logr == 5) go(ntt_pair_kernel<5, INV, PRE, POST, STREAM, false>);
  else if (logr == 4 && bulk) go(ntt_pair_kernel<4, INV, false, POST, STREAM, true>);
  else if (logr == 4) go(ntt_pair_kernel<4, INV, PRE, POST, STREAM, false>);
  else if (bulk) go(ntt_pair_kernel<3, INV, false, POST, STREAM, true>);
  else go(ntt_pair_kernel<3, INV, PRE, POST, STREAM, false>);
  TVM_CUDA(cudaGetLastError());
}

// Mixed radices (n = 2^14, 2^16, 2^18): pass A and pass B have different R, and one kernel holding both unrolled bodies
// spills and outgrows the instruction cache (measured slower than this).  Here the passes stay separate kernels, launched
// per pair; pairs alternate between the context's stream and a second one, which fills the other's partial last wave.
static void evaluate_pairs(Ctx &c, const u64 *d_coef, size_t coef_stride, unsigned fold_count, unsigned log_n, unsigned log_r,
                           unsigned coset_first, unsigned coset_step, unsigned num_cosets, size_t ncols, u64 *d_out, u64 *d_tmp,
                           int la, int lb, const u64 *S, PowTab pre, u64 mask) {
  const size_t n = (size_t)1 << log_n, n2 = (size_t)1 << la, n1 = (size_t)1 << lb;
  const int ra = tile_logr(la), rb = tile_logr(lb);
  const unsigned TA = TILE_THREADS >> ra, TB = TILE_THREADS >> rb;
  const u64 *ff = S + (size_t)num_cosets * n2;
  PairJob a{};
  a.in = d_coef; a.out = d_tmp;
  a.in_col_stride = coef_stride; a.in_coset_stride = 0;
  a.out_col_stride = (size_t)num_cosets * n; a.out_coset_stride = n;
  a.in_row_stride = 1; a.in_elem_stride = n1;
  a.out_row_stride = 1; a.out_elem_stride = n1;
  a.tw = c.get_tile_tw(la, false);
  a.prescale = S; a.fold_factor = ff; a.fold_count = fold_count; a.fold_offset = n;
  a.post_mode = 1; a.G = pre; a.exp_mask = mask; a.mul = (u64)1 << log_r;
  a.coset_first = coset_first; a.coset_step = coset_step;
  PairJob b{};
  b.in = d_tmp; b.out = d_out;
  b.in_col_stride = (size_t)num_cosets * n; b.in_coset_stride = n;
  b.out_col_stride = (size_t)num_cosets * n; b.out_coset_stride = n;
  b.in_row_stride = n1; b.in_elem_stride = 1;
  b.out_row_stride = 1; b.out_elem_stride = n2;
  b.tw = c.get_tile_tw(lb, false);
  b.post_mode = 0;
  // launch pairs of (columns x cosets) whose transposed intermediate fits the budget
  const size_t budget_words = tile_tmp_budget() / 8;
  size_t cos_per = std::min<size_t>(num_cosets, std::max<size_t>(1, budget_words / n));
  while (num_cosets % cos_per) cos_per--;
  const size_t group = cos_per == num_cosets ? std::max<size_t>(1, budget_words / ((size_t)num_cosets * n)) : 1;
  const size_t pair_words = group * cos_per * n;
  const size_t npairs = ((ncols + group - 1) / group) * (num_cosets / cos_per);
  const bool two = npairs >= 2 && 2 * pair_words <= ncols * (size_t)num_cosets * n;
  cudaStream_t st[2] = {c.stream, c.stream};
  if (two) {
    st[1] = c.get_pair_stream();
    TVM_CUDA(cudaEventRecord(c.pair_fork, c.stream));
    TVM_CUDA(cudaStreamWaitEvent(st[1], c.pair_fork, 0));
  }
  size_t pi = 0;
  for (size_t c0 = 0; c0 < ncols; c0 += group) {
    const size_t g = std::min(group, ncols - c0);
    for (size_t y0 = 0; y0 < num_cosets; y0 += cos_per, pi++) {
      const int k = two ? (int)(pi & 1) : 0;
      PairJob aa = a, bb = b;
      aa.in += c0 * coef_stride;
      aa.out += (size_t)k * pair_words;
      aa.prescale += y0 * n2; aa.fold_factor += y0;
      aa.coset_first = coset_first + coset_step * (unsigned)y0;
      aa.out_col_stride = cos_per * n;                       // the intermediate of this pair only
      bb.in += (size_t)k * pair_words;
      bb.in_col_stride = cos_per * n;
      bb.out += (c0 * (size_t)num_cosets + y0) * n;
      launch_pair<false, true, 1, false>(ra, dim3((unsigned)(n1 / TA), (unsigned)cos_per, (unsigned)g), st[k], aa);
      launch_pair<false, false, 0, true>(rb, dim3((unsigned)(n2 / TB), (unsigned)cos_per, (unsigned)g), st[k], bb);
      c.launches += 2;
    }
  }
  if (two) {
    TVM_CUDA(cudaEventRecord(c.pair_join, st[1]));
    TVM_CUDA(cudaStreamWaitEvent(c.stream, c.pair_join, 0));
  }
}

static void interpolate_pairs(Ctx &c, const u64 *d_trace, unsigned log_n, u64 offset_mont, size_t ncols, u64 *d_coef,
                              size_t coef_stride, u64 *d_tmp, int la, int lb) {
  const size_t n = (size_t)1 << log_n, n2 = (size_t)1 << la, n1 = (size_t)1 << lb;
  const int ra = tile_logr(la), rb = tile_logr(lb);
  const unsigned TA = TILE_THREADS >> ra, TB = TILE_THREADS >> rb;
  const u64 wn_inv = finv(root_of_unity_mont(log_n));
  PairJob a{};
  a.in = d_trace; a.out = d_tmp;
  a.in_col_stride = n; a.out_col_stride = n;
  a.in_row_stride = 1; a.in_elem_stride = n1;
  a.out_row_stride = 1; a.out_elem_stride = n1;
  a.tw = c.get_tile_tw(la, true);
  a.post_mode = 1; a.G = c.get_pow_tab(wn_inv, (int)log_n); a.exp_mask = n - 1; a.mul = 1;
  PairJob b{};
  b.in = d_tmp; b.out = d_coef;
  b.in_col_stride = n; b.out_col_stride = coef_stride;
  b.in_row_stride = n1; b.in_elem_stride = 1;
  b.out_row_stride = 1; b.out_elem_stride = n2;
  b.tw = c.get_tile_tw(lb, true);
  b.post_mode = 2; b.G = c.get_pow_tab(offset_mont, (int)log_n + 1); b.mul = n2;
  b.scalar = finv(to_mont((u64)n));
  size_t group = std::max<size_t>(1, tile_tmp_budget() / 8 / n);
  for (size_t c0 = 0; c0 < ncols; c0 += group) {
    const size_t g = std::min(group, ncols - c0);
    PairJob aa = a, bb = b;
    aa.in += c0 * n;
    bb.out += c0 * coef_stride;
    launch_pair<true, false, 1, false>(ra, dim3((unsigned)(n1 / TA), 1, (unsigned)g), c.stream, aa);
    launch_pair<true, false, 2, false>(rb, dim3((unsigned)(n2 / TB), 1, (unsigned)g), c.stream, bb);
    c.launches += 2;
  }
}

// B-tiles read their rows with 16-byte bulk copies: the intermediate must be 16-byte aligned (n >= 2^12 keeps every
// column and coset at a multiple of 16 bytes)
static bool tile_tmp_aligned(const u64 *d_tmp) { return ((uintptr_t)d_tmp % 16) == 0; }

// Coset evaluation of pre-scaled coefficient columns (lde_evaluate_run's contract).
bool lde_evaluate_tiles(Ctx &c, const u64 *d_coef, size_t coef_stride, unsigned fold_count, unsigned log_n, unsigned log_r,
                        unsigned coset_first, unsigned coset_step, unsigned num_cosets, size_t ncols, u64 *d_out, u64 *d_tmp) {
  int la, lb;
  if (!ntt_tile_supported((int)log_n, &la, &lb) || !tile_tmp_aligned(d_tmp)) return false;
  const size_t n = (size_t)1 << log_n, n2 = (size_t)1 << la, n1 = (size_t)1 << lb;
  const int ra = tile_logr(la), rb = tile_logr(lb);
  if (fold_count > (n1 << ra) || fold_count > n) return false;
  const unsigned TA = TILE_THREADS >> ra, TB = TILE_THREADS >> rb;
  if (n1 % TA || n2 % TB) return false;
  const u64 wrn = root_of_unity_mont(log_n + log_r);
  PowTab pre = c.get_pow_tab(wrn, (int)(log_n + log_r));
  const u64 mask = ((u64)1 << (log_n + log_r)) - 1;
  // prescale table + fold factors of this coset set (cached per job shape)
  u64 *S = c.get_prescale(log_n, log_r, (unsigned)lb, (unsigned)n2, coset_first, coset_step, num_cosets, [&](u64 *dS, u64 *dff) {
    prescale_table_kernel<<<dim3((unsigned)((n2 + 255) / 256), num_cosets), 256, 0, c.stream>>>(dS, dff, pre, log_n, (unsigned)lb,
                                                                                                  (unsigned)n2, coset_first, coset_step, mask);
    c.launches++;
    TVM_CUDA(cudaGetLastError());
  });
  if (ra != rb) {
    evaluate_pairs(c, d_coef, coef_stride, fold_count, log_n, log_r, coset_first, coset_step, num_cosets, ncols, d_out, d_tmp, la, lb,
                   S, pre, mask);
    return true;
  }
  TileJob j{};
  j.in = d_coef; j.in_col_stride = coef_stride;
  j.tmp = d_tmp; j.tmp_cosets = num_cosets;
  j.out = d_out; j.out_col_stride = (size_t)num_cosets * n;
  j.n = n; j.log_n1 = (unsigned)lb; j.log_n2 = (unsigned)la;
  j.tw = c.get_tile_tw(la, false);
  j.prescale = S; j.fold_factor = S + (size_t)num_cosets * n2; j.fold_count = fold_count; j.fold_offset = n;
  j.Ga = pre; j.exp_mask = mask; j.mula = (u64)1 << log_r;
  j.coset_first = coset_first; j.coset_step = coset_step;
  // pairs of (columns x cosets) whose transposed intermediate fits the budget
  const size_t budget_words = tile_tmp_budget() / 8;
  size_t cos_per = std::min<size_t>(num_cosets, std::max<size_t>(1, budget_words / n));
  while (num_cosets % cos_per) cos_per--;
  const size_t group = cos_per == num_cosets ? std::max<size_t>(1, std::min(ncols, budget_words / ((size_t)num_cosets * n))) : 1;
  TileSched s{};
  s.ncg = (unsigned)(num_cosets / cos_per);
  s.npairs = (unsigned)((ncols + group - 1) / group) * s.ncg;
  s.group = (unsigned)group; s.cos_per = (unsigned)cos_per; s.ncols = (unsigned)ncols;
  s.nxa = (unsigned)(n1 / TA); s.nxb = (unsigned)(n2 / TB);
  run_tiles<false, true, 0>(c, ra, rb, j, s);
  return true;
}

// Interpolation of trace columns to pre-scaled coefficients (lde_interpolate_run's contract).
bool lde_interpolate_tiles(Ctx &c, const u64 *d_trace, const u64 *d_rand, unsigned num_rand, unsigned rand_pad, unsigned log_n,
                           u64 offset_mont, size_t ncols, u64 *d_coef, size_t coef_stride, u64 *d_tmp) {
  int la, lb;
  if (!ntt_tile_supported((int)log_n, &la, &lb) || !tile_tmp_aligned(d_tmp)) return false;
  const size_t n = (size_t)1 << log_n, n2 = (size_t)1 << la, n1 = (size_t)1 << lb;
  const int ra = tile_logr(la), rb = tile_logr(lb);
  const unsigned TA = TILE_THREADS >> ra, TB = TILE_THREADS >> rb;
  if (n1 % TA || n2 % TB) return false;
  const u64 wn_inv = finv(root_of_unity_mont(log_n));
  TileJob j{};
  j.in = d_trace; j.in_col_stride = n;
  j.tmp = d_tmp; j.tmp_cosets = 1;
  j.out = d_coef; j.out_col_stride = coef_stride;
  j.n = n; j.log_n1 = (unsigned)lb; j.log_n2 = (unsigned)la;
  j.tw = c.get_tile_tw(la, true);
  j.Ga = c.get_pow_tab(wn_inv, (int)log_n); j.exp_mask = n - 1; j.mula = 1;
  j.Gb = c.get_pow_tab(offset_mont, (int)log_n + 1); j.mulb = n2;
  j.scalar = finv(to_mont((u64)n));
  const size_t group = std::max<size_t>(1, std::min(ncols, tile_tmp_budget() / 8 / n));
  TileSched s{};
  s.ncg = 1; s.cos_per = 1;
  s.npairs = (unsigned)((ncols + group - 1) / group);
  s.group = (unsigned)group; s.ncols = (unsigned)ncols;
  s.nxa = (unsigned)(n1 / TA); s.nxb = (unsigned)(n2 / TB);
  if (ra != rb) interpolate_pairs(c, d_trace, log_n, offset_mont, ncols, d_coef, coef_stride, d_tmp, la, lb);
  else run_tiles<true, false, 2>(c, ra, rb, j, s);
  const unsigned pad = d_rand ? std::max(rand_pad, num_rand) : 0;
  if (pad) {
    lde_randomizer_kernel<<<dim3((pad + 127) / 128, (unsigned)ncols), 128, 0, c.stream>>>(d_coef, coef_stride, n, d_rand, num_rand, pad, j.Gb);
    c.launches++;
    TVM_CUDA(cudaGetLastError());
  }
  return true;
}

}  // namespace tvm
