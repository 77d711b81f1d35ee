// Auxiliary-table extension on the device: MasterMainTable::extend (master_table.rs:1006-1075) + the generated
// fill_derived_aux_columns (substitutions.rs:163-205, 336-368) — SURVEY.md 8(f).1.
//
// The reference fills each of the 49 auxiliary base columns with a sequential loop over the rows (processor.rs:139-640,
// op_stack.rs:213-290, ram.rs:105-255, jump_stack.rs:207-280, hash.rs:304-460, cascade.rs:68-130, lookup.rs:118-180,
// u32.rs:156-230, program.rs:115-190), one rayon task per column.  Every one of those loops is a first-order linear
// recurrence   aux[i] = a_i * aux[i-1] + b_i   (running product: b = 0; running evaluation: a = indeterminate;
// logarithmic derivative: a = 1, b = multiplicity / (indeterminate - value)), so on the device a column is the inclusive
// SCAN of its row maps under composition, parallel over rows as well as columns:
//
//   aux_scan_kernel          one CTA per (256-row chunk, column): row maps, CTA scan; stores the scanned map of every row
//                            (48 B per row and column) and the chunk total                                 -> maps, tot
//   aux_scan_tops_kernel     one warp per column: the chunk totals in order                            -> value entering each chunk
//   aux_apply_kernel         scanned map of the row applied to the value entering its chunk, store
//                            (round 1 recomputed the row maps and the scan here: ncu r02i, 2^18 rows, 47 columns: 6 780
//                            instructions per row and column in EACH pass, half of them the map itself - logarithmic
//                            derivatives cost a field inversion per row; 48 B of traffic are far cheaper)
//
// twice: 47 columns depend on the main table only, two (program table: send-chunk evaluation; RAM table: formal
// derivative) read a finished column of the first pass.  The row maps (a_i, b_i) are not hand-written: airgen/extend_gen.py
// derives them from the AIR's own initial/transition constraints by symbolic differentiation (aux_gen/aux_extend_gen.inc),
// so they cannot drift from what the quotient kernels enforce.  Then one kernel fills the 41 degree-lowering columns row by
// row.  Integer work on the FMA/ALU pipes like the rest of the prover; HBM traffic is one read of the touched main columns
// per pass and one write of the auxiliary table — no tensor-core shape anywhere.
//
// Layout: main table [379][n] Montgomery, auxiliary table [91*3][n] Montgomery planes (the layout the LDE consumes).
#include <cstdlib>
#include <cstring>
#include "prove_common.h"

namespace tvm {
namespace {

struct auxctx {
  u64 *main_t;     // written only by the derived-main-column kernels
  u64 *aux_t;
  const u64 *ch;
  size_t n, cur, nxt;
};

TVM_D xfe aux_load(const auxctx &c, int col, size_t row) {
  return xmake(c.aux_t[(size_t)(3 * col) * c.n + row], c.aux_t[(size_t)(3 * col + 1) * c.n + row], c.aux_t[(size_t)(3 * col + 2) * c.n + row]);
}
TVM_D void aux_store(const auxctx &c, int col, size_t row, xfe v) {
  c.aux_t[(size_t)(3 * col) * c.n + row] = v.c0;
  c.aux_t[(size_t)(3 * col + 1) * c.n + row] = v.c1;
  c.aux_t[(size_t)(3 * col + 2) * c.n + row] = v.c2;
}
TVM_D xfe ch_load(const auxctx &c, int i) { return xmake(c.ch[3 * i], c.ch[3 * i + 1], c.ch[3 * i + 2]); }

#define AUXGEN_FN static __device__ __noinline__
#define AUXGEN_ARGS const auxctx &c
#define AUXGEN_PASS c
#define AUXGEN_TOUCH (void)c
#define MC(col) (c.main_t[(size_t)(col) * c.n + c.cur])
#define MN(col) (c.main_t[(size_t)(col) * c.n + c.nxt])
#define AC(col) aux_load(c, (col), c.cur)
#define AN(col) aux_load(c, (col), c.nxt)
#define CH(i) ch_load(c, (i))
#define AW(col, v) aux_store(c, (col), c.cur, (v))
#define MW(col, v) (c.main_t[(size_t)(col) * c.n + c.cur] = (v))
#include "aux_gen/aux_extend_gen.inc"
#undef MC
#undef MN
#undef AC
#undef AN
#undef CH
#undef AW
#undef MW

constexpr int AUX_CHUNK = 256;

struct AffMap {   // v -> a * v + b
  xfe a, b;
};
TVM_D AffMap compose(const AffMap &later, const AffMap &earlier) {
  AffMap r;
  r.a = xmul(later.a, earlier.a);
  r.b = xadd(xmul(later.a, earlier.b), later.b);
  return r;
}
TVM_D void map_store(u64 (*sm)[AUX_CHUNK], int t, const AffMap &m) {
  sm[0][t] = m.a.c0; sm[1][t] = m.a.c1; sm[2][t] = m.a.c2;
  sm[3][t] = m.b.c0; sm[4][t] = m.b.c1; sm[5][t] = m.b.c2;
}
TVM_D AffMap map_load(u64 (*sm)[AUX_CHUNK], int t) {
  AffMap m;
  m.a = xmake(sm[0][t], sm[1][t], sm[2][t]);
  m.b = xmake(sm[3][t], sm[4][t], sm[5][t]);
  return m;
}
// inclusive scan over the CTA's AUX_CHUNK maps (thread t holds map t); double-buffered Hillis-Steele
TVM_D AffMap cta_scan(AffMap m, u64 (*sm)[6][AUX_CHUNK]) {
  const int t = threadIdx.x;
  int src = 0;
  map_store(sm[0], t, m);
  __syncthreads();
  for (int d = 1; d < AUX_CHUNK; d <<= 1) {
    if (t >= d) m = compose(m, map_load(sm[src], t - d));
    map_store(sm[src ^ 1], t, m);
    __syncthreads();
    src ^= 1;
  }
  return m;
}

struct AuxScanArgs {
  const u64 *main_t;
  u64 *aux_t;
  const u64 *ch;
  size_t n, nchunks;
  u64 *tot;   // [ncols][nchunks][6]   chunk totals
  u64 *vin;   // [ncols][nchunks][3]   value of the column before the chunk's first row
  u64 *maps;  // [ncols][6][n]         scanned (within its chunk) map of every row
  int ncols;
  int cols[AUXGEN_NUM_BASE];
};

__global__ void __launch_bounds__(AUX_CHUNK, 2) aux_scan_kernel(AuxScanArgs p) {
  __shared__ u64 sm[2][6][AUX_CHUNK];
  const int q = p.cols[blockIdx.y];
  const size_t i = (size_t)blockIdx.x * AUX_CHUNK + threadIdx.x;
  AffMap m;
  m.a = xone();
  m.b = xzero();
  if (i < p.n) {
    auxctx c{const_cast<u64 *>(p.main_t), p.aux_t, p.ch, p.n, i ? i - 1 : 0, i};
    xfe a = xone(), b = xzero();
    if (i == 0) {                       // the initial constraint fixes row 0: constant map
      auxgen_init(q, c, &b);
      m.a = xzero();
      m.b = b;
    } else if (auxgen_tran(q, c, &a, &b)) {
      m.a = a;
      m.b = b;
    }                                   // no rule moves the column on this row: identity
  }
  m = cta_scan(m, sm);
  const size_t slot = (size_t)blockIdx.y * p.nchunks + blockIdx.x;
  if (i < p.n) {                        // scanned map of row i: planes [column of the level][6][n]
    u64 *o = p.maps + (size_t)blockIdx.y * 6 * p.n + i;
    o[0] = m.a.c0; o[p.n] = m.a.c1; o[2 * p.n] = m.a.c2; o[3 * p.n] = m.b.c0; o[4 * p.n] = m.b.c1; o[5 * p.n] = m.b.c2;
  }
  if (threadIdx.x == AUX_CHUNK - 1) {
    u64 *o = p.tot + slot * 6;
    o[0] = m.a.c0; o[1] = m.a.c1; o[2] = m.a.c2; o[3] = m.b.c0; o[4] = m.b.c1; o[5] = m.b.c2;
  }
}

__global__ void __launch_bounds__(AUX_CHUNK) aux_apply_kernel(AuxScanArgs p) {
  const int q = p.cols[blockIdx.y];
  const size_t i = (size_t)blockIdx.x * AUX_CHUNK + threadIdx.x;
  if (i >= p.n) return;
  const u64 *o = p.maps + (size_t)blockIdx.y * 6 * p.n + i;
  const xfe a = xmake(o[0], o[p.n], o[2 * p.n]), b = xmake(o[3 * p.n], o[4 * p.n], o[5 * p.n]);
  const u64 *vi = p.vin + ((size_t)blockIdx.y * p.nchunks + blockIdx.x) * 3;
  const xfe v = xadd(xmul(a, xmake(vi[0], vi[1], vi[2])), b);
  u64 *w = p.aux_t + (size_t)(3 * q) * p.n + i;
  w[0] = v.c0; w[p.n] = v.c1; w[2 * p.n] = v.c2;
}

// one warp per column, lane 0 walks the chunk totals in order (n / 256 compositions: 4096 at 2^20, ~1.5 ms for all columns
// in parallel; a CTA-wide scan of the totals is the obvious next step once this stage shows up in a profile).
// vin[k] = value of the column before chunk k's first row; row 0's map is constant, so the value fed in is irrelevant.
__global__ void aux_scan_tops_kernel(AuxScanArgs p) {
  if (threadIdx.x != 0) return;
  const u64 *tot = p.tot + (size_t)blockIdx.x * p.nchunks * 6;
  u64 *vin = p.vin + (size_t)blockIdx.x * p.nchunks * 3;
  xfe v = xzero();
  for (size_t k = 0; k < p.nchunks; k++) {
    vin[3 * k] = v.c0; vin[3 * k + 1] = v.c1; vin[3 * k + 2] = v.c2;
    xfe a = xmake(tot[6 * k], tot[6 * k + 1], tot[6 * k + 2]), b = xmake(tot[6 * k + 3], tot[6 * k + 4], tot[6 * k + 5]);
    v = xadd(xmul(a, v), b);
  }
}

// CTA-wide variant of the above (TVM_AUX_TOPS_PARALLEL=1; not yet run on a GPU — the sequential kernel is the default until
// it has been compared): thread t composes its `per` consecutive chunk totals, the CTA scans the 256 thread totals with
// the same cta_scan the row kernels use, and each thread walks its range again from its exclusive prefix.
__global__ void __launch_bounds__(AUX_CHUNK) aux_scan_tops_parallel_kernel(AuxScanArgs p) {
  __shared__ u64 sm[2][6][AUX_CHUNK];
  __shared__ u64 ex[6][AUX_CHUNK];
  const int t = threadIdx.x;
  const size_t per = (p.nchunks + AUX_CHUNK - 1) / AUX_CHUNK;
  const size_t k0 = (size_t)t * per < p.nchunks ? (size_t)t * per : p.nchunks;
  const size_t k1 = k0 + per < p.nchunks ? k0 + per : p.nchunks;
  const u64 *tot = p.tot + (size_t)blockIdx.x * p.nchunks * 6;
  u64 *vin = p.vin + (size_t)blockIdx.x * p.nchunks * 3;
  AffMap m;
  m.a = xone();
  m.b = xzero();
  for (size_t k = k0; k < k1; k++) {
    AffMap x;
    x.a = xmake(tot[6 * k], tot[6 * k + 1], tot[6 * k + 2]);
    x.b = xmake(tot[6 * k + 3], tot[6 * k + 4], tot[6 * k + 5]);
    m = compose(x, m);
  }
  const AffMap incl = cta_scan(m, sm);
  map_store(ex, t, incl);
  __syncthreads();
  xfe v = xzero();                                   // value before this thread's first chunk
  if (t > 0) v = map_load(ex, t - 1).b;              // the prefix map applied to 0 (row 0's map is constant)
  for (size_t k = k0; k < k1; k++) {
    vin[3 * k] = v.c0; vin[3 * k + 1] = v.c1; vin[3 * k + 2] = v.c2;
    xfe a = xmake(tot[6 * k], tot[6 * k + 1], tot[6 * k + 2]), b = xmake(tot[6 * k + 3], tot[6 * k + 4], tot[6 * k + 5]);
    v = xadd(xmul(a, v), b);
  }
}

// the 41 degree-lowering columns: row i from rows i, i+1 of the main table and of the 49 base columns; last row zero
__global__ void __launch_bounds__(128) aux_derived_kernel(const u64 *main_t, u64 *aux_t, const u64 *ch, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  auxctx c{const_cast<u64 *>(main_t), aux_t, ch, n, i, i + 1};
  if (i + 1 < n) {
    auxgen_derived_tran(c);
  } else {
    for (int k = 0; k < AUXGEN_NUM_DERIVED_TRAN; k++) aux_store(c, AUXGEN_DERIVED_START_TRAN + k, i, xzero());
  }
}

// DegreeLoweringTable::fill_derived_main_columns (substitutions.rs:128-161, 237-300): main columns 149..378 from 0..148.
// Sections init | cons read their own row (pass 0, every row); section tran reads rows i and i+1 including the next row's
// init / cons columns (pass 1, after pass 0 has completed; the last row's tran columns are 0).
template <int PASS>
__global__ void __launch_bounds__(128) main_derived_kernel(u64 *main_t, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  auxctx c{main_t, nullptr, nullptr, n, i, PASS ? i + 1 : i};
  if (PASS == 0) {
    auxgen_derived_main_init(c);
    auxgen_derived_main_cons(c);
  } else if (i + 1 < n) {
    auxgen_derived_main_tran(c);
  } else {
    for (int k = 0; k < AUXGEN_NUM_DERIVED_MAIN_TRAN; k++) main_t[(size_t)(AUXGEN_DERIVED_MAIN_START_TRAN + k) * n + i] = 0;
  }
}

// [ncols][3 planes][n] Montgomery -> [ncols][n][3] canonical (the ABI's X-field layout)
__global__ void interleave3_from_mont_kernel(const u64 *in, u64 *out, size_t n, size_t ncols) {
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= ncols * n) return;
  size_t q = idx / n, j = idx - q * n;
  for (int d = 0; d < 3; d++) out[3 * idx + d] = from_mont(in[(3 * q + d) * n + j]);
}

}  // namespace

size_t aux_extend_scratch_words(size_t n) { return (size_t)AUXGEN_NUM_BASE * (((n + AUX_CHUNK - 1) / AUX_CHUNK) * 9 + 6 * n); }

// d_main [379][n], d_ch [63*3], d_aux [273][n] (all Montgomery; the batch-randomizer planes 270..272 are the caller's)
void aux_extend_run(Ctx &c, const u64 *d_main, size_t n, const u64 *d_ch, u64 *d_aux, u64 *d_scratch) {
  AuxScanArgs p{};
  p.main_t = d_main; p.aux_t = d_aux; p.ch = d_ch; p.n = n;
  p.nchunks = (n + AUX_CHUNK - 1) / AUX_CHUNK;
  p.tot = d_scratch;
  p.vin = d_scratch + (size_t)AUXGEN_NUM_BASE * p.nchunks * 6;
  p.maps = d_scratch + (size_t)AUXGEN_NUM_BASE * p.nchunks * 9;
  for (int level = 0; level < AUXGEN_NUM_LEVELS; level++) {
    p.ncols = 0;
    for (int q = 0; q < AUXGEN_NUM_BASE; q++)
      if (AUXGEN_LEVEL[q] == level) p.cols[p.ncols++] = q;
    if (!p.ncols) continue;
    dim3 grid((unsigned)p.nchunks, (unsigned)p.ncols);
    aux_scan_kernel<<<grid, AUX_CHUNK, 0, c.stream>>>(p);
    static const bool tops_parallel = getenv("TVM_AUX_TOPS_PARALLEL") && atoi(getenv("TVM_AUX_TOPS_PARALLEL"));
    if (tops_parallel) aux_scan_tops_parallel_kernel<<<(unsigned)p.ncols, AUX_CHUNK, 0, c.stream>>>(p);
    else aux_scan_tops_kernel<<<(unsigned)p.ncols, 32, 0, c.stream>>>(p);
    aux_apply_kernel<<<grid, AUX_CHUNK, 0, c.stream>>>(p);
    c.launches += 3;
    TVM_CUDA(cudaGetLastError());
  }
  aux_derived_kernel<<<(unsigned)((n + 127) / 128), 128, 0, c.stream>>>(d_main, d_aux, d_ch, n);
  c.launches++;
  TVM_CUDA(cudaGetLastError());
}

void aux_extend_on_device(Ctx &c, DevMem &mem, const u64 *d_main, size_t n, const u64 *d_ch, const u64 *randomizer_column, u64 *d_aux) {
  const size_t NA = TVM_NUM_AUX_COLUMNS;
  u64 *d_scratch = mem.words(aux_extend_scratch_words(n) + (randomizer_column ? 3 * n : 0));
  u64 *d_rplanes = d_aux + 3 * (NA - 1) * n;
  if (randomizer_column) {
    u64 *d_rc = d_scratch + aux_extend_scratch_words(n);
    TVM_CUDA(cudaMemcpyAsync(d_rc, randomizer_column, 3 * n * 8, cudaMemcpyDefault, c.stream));
    to_mont_run(c, d_rc, 3 * n);
    deinterleave3_run(c, d_rc, d_rplanes, n, 1);
  } else {
    TVM_CUDA(cudaMemsetAsync(d_rplanes, 0, 3 * n * 8, c.stream));
  }
  aux_extend_run(c, d_main, n, d_ch, d_aux, d_scratch);
  mem.release(d_scratch);
}

// d_main [379][n] Montgomery, columns 149.. overwritten
void main_derived_run(Ctx &c, u64 *d_main, size_t n) {
  const unsigned grid = (unsigned)((n + 127) / 128);
  main_derived_kernel<0><<<grid, 128, 0, c.stream>>>(d_main, n);
  main_derived_kernel<1><<<grid, 128, 0, c.stream>>>(d_main, n);
  c.launches += 2;
  TVM_CUDA(cudaGetLastError());
}

void interleave3_from_mont_run(Ctx &c, const u64 *in, u64 *out, size_t n, size_t ncols) {
  interleave3_from_mont_kernel<<<(unsigned)((ncols * n + 255) / 256), 256, 0, c.stream>>>(in, out, n, ncols);
  c.launches++;
  TVM_CUDA(cudaGetLastError());
}

}  // namespace tvm
