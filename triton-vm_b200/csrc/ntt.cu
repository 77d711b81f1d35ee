// Batched radix-2 NTT / iNTT / coset-LDE over GF(p), p = 2^64 - 2^32 + 1, for sm_90a.
//
// Semantics (reference triton-vm/src/arithmetic_domain.rs:141-212, A.2 of SURVEY.md):
//   ntt(x)[k] = sum_j x_j w^{jk}, natural order in and out, w = primitive_root_of_unity(n)
//   (twenty-first's table); intt is its inverse.  The LDE entry point restates
//   master_table.rs:258-322 / 392-403: interpolate the trace column on the trace domain
//   (offset 1), add zerofier*randomizer, evaluate on the coset offset*<w_{rn}>.
//
// Decomposition (GPU-first, not the reference's per-column recursive NTT):
//   * 4-step: n = n1*n2.  Pass A does n1/T tiles of T interleaved n2-point NTTs on strided
//     rows (64-byte segments), multiplies by the inter-pass twist w_n^{j1*k2} on the way out.
//     Pass B does n2/T tiles of T contiguous n1-point NTTs and scatters rows to natural order.
//   * inside a tile: data in shared memory, radix-8 decimation-in-frequency rounds held in
//     registers; the three inner stages use only w_8 = -2^24, w_4 = 2^48 (shift-and-reduce,
//     no multiplier), followed by 7 general twiddles per group.  Bit reversal is absorbed in
//     the global row addressing of the store.
//   * LDE: evaluation domain = r cosets of the size-n trace domain.  Coset c of column q is
//     an n-point NTT of the folded, pre-scaled coefficients
//         (c'_j + w_r^c c'_{n+j}) * w_{rn}^{c j},   c'_j = coeff_j * offset^j,
//     so the 8x blow-up is never a zero-padded transform.  Output layout is coset-major:
//     out[q][c][k] holds evaluation-domain row i = c + r*k.
#include "ctx.h"
#include "launch.h"

namespace tvm {

static constexpr int NTT_THREADS = 512;
static constexpr int LT_MAX = 13;   // two passes cover transforms up to 2^26 (LDT domain of padded height 2^23)

__device__ __forceinline__ u64 powtab_get(const PowTab &t, u64 e) {
  u64 lo = __ldg(t.lo + (e & ((1ULL << t.shift) - 1)));
  u64 hi = __ldg(t.hi + (e >> t.shift));
  return fmul(lo, hi);
}

__device__ __forceinline__ unsigned bitrev(unsigned x, int bits) { return bits ? (__brev(x) >> (32 - bits)) : 0; }

// 8-point DIF network with constant twiddles.  Forward root w_8 = -2^24 (twenty-first's
// primitive_root_of_unity(8) = 18446744069397807105 = p - 2^24), w_8^2 = 2^48, w_8^3 = -2^72.
template <bool INV>
__device__ __forceinline__ void dft8(u64 (&e)[8]) {
  {
    u64 u, v;
    u = e[0]; v = e[4]; e[0] = fadd(u, v); e[4] = fsub(u, v);
    u = e[1]; v = e[5]; e[1] = fadd(u, v);
    e[5] = INV ? fmul_2k<72>(fsub(u, v)) : fmul_2k<24>(fsub(v, u));
    u = e[2]; v = e[6]; e[2] = fadd(u, v);
    e[6] = INV ? fmul_2k<48>(fsub(v, u)) : fmul_2k<48>(fsub(u, v));
    u = e[3]; v = e[7]; e[3] = fadd(u, v);
    e[7] = INV ? fmul_2k<24>(fsub(u, v)) : fmul_2k<72>(fsub(v, u));
  }
#pragma unroll
  for (int h = 0; h < 8; h += 4) {
    u64 u, v;
    u = e[h]; v = e[h + 2]; e[h] = fadd(u, v); e[h + 2] = fsub(u, v);
    u = e[h + 1]; v = e[h + 3]; e[h + 1] = fadd(u, v);
    e[h + 3] = INV ? fmul_2k<48>(fsub(v, u)) : fmul_2k<48>(fsub(u, v));
  }
#pragma unroll
  for (int q = 0; q < 8; q += 2) {
    u64 u = e[q], v = e[q + 1];
    e[q] = fadd(u, v);
    e[q + 1] = fsub(u, v);
  }
}

// In-place DIF NTT of T rows of length N = 2^LT in shared memory (row pitch `pitch`),
// natural order in, bit-reversed order out.  tw[e] = w_N^(+-e), e < N.
template <bool INV>
__device__ void tile_dif(u64 *tile, int pitch, const u64 *tw, int LT, int log_t) {
  const int N = 1 << LT;
  int m_log = LT;
  while (m_log >= 3) {
    const int groups_row = N >> 3;
    const int total = groups_row << log_t;
    const int sub = m_log - 3;
    for (int gi = threadIdx.x; gi < total; gi += blockDim.x) {
      int g = gi & (groups_row - 1);
      int t = gi >> (LT - 3);
      int j0 = g & ((1 << sub) - 1);
      int b = (g >> sub) << m_log;
      u64 *p = tile + t * pitch + b + j0;
      u64 e[8];
#pragma unroll
      for (int i = 0; i < 8; i++) e[i] = p[i << sub];
      dft8<INV>(e);
      if (j0 != 0) {
        const int sh = LT - m_log;
        // output i carries the twist w_m^{j0 * bitrev3(i)}
        e[1] = fmul(e[1], tw[(j0 * 4) << sh]);
        e[2] = fmul(e[2], tw[(j0 * 2) << sh]);
        e[3] = fmul(e[3], tw[(j0 * 6) << sh]);
        e[4] = fmul(e[4], tw[(j0 * 1) << sh]);
        e[5] = fmul(e[5], tw[(j0 * 5) << sh]);
        e[6] = fmul(e[6], tw[(j0 * 3) << sh]);
        e[7] = fmul(e[7], tw[(j0 * 7) << sh]);
      }
#pragma unroll
      for (int i = 0; i < 8; i++) p[i << sub] = e[i];
    }
    __syncthreads();
    m_log -= 3;
  }
  if (m_log == 2) {
    const int total = (N >> 2) << log_t;
    for (int gi = threadIdx.x; gi < total; gi += blockDim.x) {
      int g = gi & ((N >> 2) - 1);
      int t = gi >> (LT - 2);
      u64 *p = tile + t * pitch + 4 * g;
      u64 a = p[0], b = p[1], c = p[2], d = p[3];
      u64 s0 = fadd(a, c), s1 = fadd(b, d), d0 = fsub(a, c);
      u64 d1 = INV ? fmul_2k<48>(fsub(d, b)) : fmul_2k<48>(fsub(b, d));
      p[0] = fadd(s0, s1); p[1] = fsub(s0, s1); p[2] = fadd(d0, d1); p[3] = fsub(d0, d1);
    }
    __syncthreads();
  } else if (m_log == 1) {
    const int total = (N >> 1) << log_t;
    for (int gi = threadIdx.x; gi < total; gi += blockDim.x) {
      int g = gi & ((N >> 1) - 1);
      int t = gi >> (LT - 1);
      u64 *p = tile + t * pitch + 2 * g;
      u64 a = p[0], b = p[1];
      p[0] = fadd(a, b); p[1] = fsub(a, b);
    }
    __syncthreads();
  }
}

struct PassA {
  const u64 *in;       // [col][...]: element j of (col) at in[col*in_cstride + j]
  u64 *out;            // [(col*num_cosets + coset)][n] in Y layout
  size_t in_cstride;
  int log_n, LT, log_t;   // n2 = 2^LT (tile), n1 = 2^(log_n - LT), T = 2^log_t interleaved rows
  PowTab twist;        // w_n^(+-e)
  int has_pre;         // coset pre-scale enabled
  PowTab pre;          // w_{r n}^e
  unsigned fold_count; // #coefficients j < fold_count that receive + w_r^c * in[n + j]
  unsigned coset_first, coset_step;   // grid.y index y evaluates coset coset_first + coset_step*y (shard of the r cosets)
};

template <bool INV>
__global__ void __launch_bounds__(NTT_THREADS) ntt_pass_a_kernel(PassA p, const u64 *tile_tw) {
  extern __shared__ u64 smem[];
  const int N = 1 << p.LT, T = 1 << p.log_t;
  const int pitch = N + 2;
  u64 *tw = smem, *tile = smem + N;
  const int log_n1 = p.log_n - p.LT;
  const size_t n = (size_t)1 << p.log_n;
  const unsigned coset = p.coset_first + p.coset_step * blockIdx.y, col = blockIdx.z;
  const unsigned j1_0 = blockIdx.x << p.log_t;
  const u64 *in = p.in + (size_t)col * p.in_cstride;
  u64 *out = p.out + ((size_t)col * gridDim.y + blockIdx.y) * n;

  for (int i = threadIdx.x; i < N; i += blockDim.x) tw[i] = __ldg(tile_tw + i);
  u64 fold_factor = 0;
  if (p.fold_count) fold_factor = powtab_get(p.pre, (u64)coset << p.log_n);
  for (int idx = threadIdx.x; idx < (N << p.log_t); idx += blockDim.x) {
    int t = idx & (T - 1), pos = idx >> p.log_t;
    size_t j = (size_t)(j1_0 + t) + ((size_t)pos << log_n1);
    u64 v = in[j];
    if (j < p.fold_count) v = fadd(v, fmul(fold_factor, in[n + j]));
    if (p.has_pre && coset) v = fmul(v, powtab_get(p.pre, (u64)coset * j));
    tile[t * pitch + pos] = v;
  }
  __syncthreads();
  tile_dif<INV>(tile, pitch, tw, p.LT, p.log_t);
  for (int idx = threadIdx.x; idx < (N << p.log_t); idx += blockDim.x) {
    int t = idx & (T - 1), pos = idx >> p.log_t;
    unsigned k2 = bitrev(pos, p.LT);
    unsigned j1 = j1_0 + t;
    u64 v = tile[t * pitch + pos];
    v = fmul(v, powtab_get(p.twist, (u64)j1 * k2));
    out[(size_t)j1 + ((size_t)k2 << log_n1)] = v;
  }
}

struct PassB {
  const u64 *in;       // [colB][n] Y layout (colB = col*num_cosets + coset)
  u64 *out;            // [colB] at out[colB*out_cstride + k]
  size_t out_cstride;
  int log_n, LT, log_t;   // n1 = 2^LT (tile, contiguous), n2 = 2^(log_n - LT)
  u64 post_mul;        // scalar applied to every output (Montgomery); MONT_ONE for none
  int has_post;        // multiply output k by post^(k)
  PowTab post;
  // randomizer fold-in (LDE): out[k] = (v - rand[k]) * post^k, out[n + k] = rand[k] * post^(n+k)
  const u64 *rand;     // [colB][rand_count] or nullptr
  unsigned rand_count;
  unsigned rand_pad;   // out[n + k] = 0 for rand_count <= k < rand_pad
};

template <bool INV>
__global__ void __launch_bounds__(NTT_THREADS) ntt_pass_b_kernel(PassB p, const u64 *tile_tw) {
  extern __shared__ u64 smem[];
  const int N = 1 << p.LT, T = 1 << p.log_t;
  const int pitch = N + 2;
  u64 *tw = smem, *tile = smem + N;
  const int log_n2 = p.log_n - p.LT;
  const size_t n = (size_t)1 << p.log_n;
  const size_t row0 = (size_t)blockIdx.x << p.log_t;  // row = colB * n2 + k2

  for (int i = threadIdx.x; i < N; i += blockDim.x) tw[i] = __ldg(tile_tw + i);
  for (int idx = threadIdx.x; idx < (N << p.log_t); idx += blockDim.x) {
    int pos = idx & (N - 1), t = idx >> p.LT;
    tile[t * pitch + pos] = p.in[((row0 + t) << p.LT) + pos];
  }
  __syncthreads();
  tile_dif<INV>(tile, pitch, tw, p.LT, p.log_t);
  for (int idx = threadIdx.x; idx < (N << p.log_t); idx += blockDim.x) {
    int t = idx & (T - 1), pos = idx >> p.log_t;
    size_t row = row0 + t;
    size_t colB = row >> log_n2;
    size_t k2 = row & (((size_t)1 << log_n2) - 1);
    size_t k = k2 + ((size_t)bitrev(pos, p.LT) << log_n2);
    u64 v = tile[t * pitch + pos];
    if (p.post_mul != MONT_ONE) v = fmul(v, p.post_mul);
    u64 *o = p.out + colB * p.out_cstride;
    if (p.rand) {
      if (k < p.rand_count) {
        u64 r = p.rand[colB * p.rand_count + k];
        v = fsub(v, r);
        o[n + k] = p.has_post ? fmul(r, powtab_get(p.post, n + k)) : r;
      } else if (k < p.rand_pad) {
        o[n + k] = 0;
      }
    }
    if (p.has_post) v = fmul(v, powtab_get(p.post, k));
    o[k] = v;
  }
}

// ---- table generation -------------------------------------------------------------------
__global__ void pow_table_kernel(u64 *out, u64 base, size_t count) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < count) out[i] = fpow(base, i);
}

static const u64 ROOT_2_32_CANON = 1753635133440165772ULL;
u64 root_of_unity_mont(unsigned log2n) {
  u64 r = to_mont(ROOT_2_32_CANON);
  for (unsigned i = log2n; i < 32; i++) r = fmul(r, r);
  return r;
}

void Ctx::all_gather(void *dev_buf, size_t bytes_per_rank) {
  if (comm.world <= 1) return;
  if (!comm.all_gather || comm.all_gather(comm.user, dev_buf, bytes_per_rank, (void *)stream))
    throw ApiError{TVM_ERR_INVALID_ARG, "all_gather callback failed"};
}
void Ctx::all_reduce_sum(u64 *dev_buf, size_t count) {
  if (comm.world <= 1) return;
  if (!comm.all_reduce_sum_u64 || comm.all_reduce_sum_u64(comm.user, dev_buf, count, (void *)stream))
    throw ApiError{TVM_ERR_INVALID_ARG, "all_reduce callback failed"};
}

cudaStream_t Ctx::get_pair_stream() {
  if (!pair_stream) {
    TVM_CUDA(cudaStreamCreateWithFlags(&pair_stream, cudaStreamNonBlocking));
    TVM_CUDA(cudaEventCreateWithFlags(&pair_fork, cudaEventDisableTiming));
    TVM_CUDA(cudaEventCreateWithFlags(&pair_join, cudaEventDisableTiming));
  }
  return pair_stream;
}
cudaStream_t Ctx::get_copy_stream() {
  if (!copy_stream) TVM_CUDA(cudaStreamCreateWithFlags(&copy_stream, cudaStreamNonBlocking));
  return copy_stream;
}
cudaEvent_t Ctx::get_copy_event(size_t i) {
  while (copy_events.size() <= i) {
    cudaEvent_t e;
    TVM_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    copy_events.push_back(e);
  }
  return copy_events[i];
}

void *Ctx::pool_alloc(size_t bytes) {
  if (!bytes) bytes = 8;
  auto it = pool_free.lower_bound(bytes);
  if (it != pool_free.end() && it->first <= bytes + bytes / 4 + 4096) {
    void *p = it->second;
    pool_live[p] = it->first;
    pool_free.erase(it);
    return p;
  }
  void *p = nullptr;
  cudaError_t e = cudaMalloc(&p, bytes);
  if (e != cudaSuccess) {
    // give cached blocks back to the driver and retry once
    cudaGetLastError();
    for (auto &kv : pool_free) cudaFree(kv.second);
    pool_free.clear();
    e = cudaMalloc(&p, bytes);
    if (e != cudaSuccess) throw CudaError{e, __FILE__, __LINE__};
  }
  pool_live[p] = bytes;
  return p;
}
void Ctx::pool_release(void *p) {
  auto it = pool_live.find(p);
  if (it == pool_live.end()) return;
  pool_free.emplace(it->second, p);
  pool_live.erase(it);
}

Ctx::~Ctx() {
  for (auto &kv : pool_free) cudaFree(kv.second);
  for (auto &kv : pool_live) cudaFree(kv.first);
  for (void *p : owned) cudaFree(p);
  for (auto &s : scratch)
    if (s.p) cudaFree(s.p);
  if (pair_stream) { cudaStreamDestroy(pair_stream); cudaEventDestroy(pair_fork); cudaEventDestroy(pair_join); }
  if (copy_stream) cudaStreamDestroy(copy_stream);
  for (cudaEvent_t e : copy_events) cudaEventDestroy(e);
  if (own_stream && stream) cudaStreamDestroy(stream);
}

void *Ctx::alloc(size_t bytes) {
  void *p = nullptr;
  cudaError_t e = cudaMalloc(&p, bytes ? bytes : 8);
  if (e != cudaSuccess) throw CudaError{e, __FILE__, __LINE__};
  owned.push_back(p);
  return p;
}
void Ctx::free_tracked(void *p) {
  for (size_t i = 0; i < owned.size(); i++)
    if (owned[i] == p) {
      cudaFree(p);
      owned.erase(owned.begin() + i);
      return;
    }
}
void *Ctx::scratch_get(int slot, size_t bytes) {
  DevBuf &s = scratch[slot];
  if (s.bytes < bytes) {
    if (s.p) {
      TVM_CUDA(cudaStreamSynchronize(stream));
      cudaFree(s.p);
      s.p = nullptr;
      s.bytes = 0;
    }
    cudaError_t e = cudaMalloc(&s.p, bytes);
    if (e != cudaSuccess) throw CudaError{e, __FILE__, __LINE__};
    s.bytes = bytes;
  }
  return s.p;
}

static u64 *make_pow_table(Ctx &c, u64 base, size_t count) {
  u64 *d = (u64 *)c.alloc(count * sizeof(u64));
  pow_table_kernel<<<(unsigned)((count + 255) / 256), 256, 0, c.stream>>>(d, base, count);
  c.launches++;
  TVM_CUDA(cudaGetLastError());
  return d;
}

const u64 *Ctx::get_tile_tw(int LT, bool inverse) {
  auto key = std::make_pair(LT, (int)inverse);
  auto it = tile_tw.find(key);
  if (it != tile_tw.end()) return it->second;
  u64 w = root_of_unity_mont(LT);
  if (inverse) w = finv(w);
  u64 *d = make_pow_table(*this, w, (size_t)1 << LT);
  tile_tw[key] = d;
  return d;
}

PowTab Ctx::get_pow_tab(u64 base, int log_count) {
  int shift = (log_count + 1) / 2;
  auto key = std::make_tuple(base, log_count, shift);
  auto it = pow_tabs.find(key);
  if (it == pow_tabs.end()) {
    u64 *lo = make_pow_table(*this, base, (size_t)1 << shift);
    u64 *hi = make_pow_table(*this, fpow(base, 1ULL << shift), (size_t)1 << (log_count - shift > 0 ? log_count - shift : 0));
    it = pow_tabs.emplace(key, std::make_pair(lo, hi)).first;
  }
  return PowTab{it->second.first, it->second.second, shift};
}

// ---- launchers --------------------------------------------------------------------------
static int pick_log_t(int LT) {
  // T interleaved rows per tile: keep the tile <= 128 KB of shared memory
  if (LT <= 10) return 3;
  if (LT == 11) return 3;
  if (LT == 12) return 2;
  return 1;
}
static size_t tile_smem_bytes(int LT, int log_t) {
  size_t N = (size_t)1 << LT;
  return (N + ((N + 2) << log_t)) * sizeof(u64);
}

// The dynamic shared-memory limit is an attribute of the kernel on a device, shared by every context of the process, and these
// kernels launch with a size that depends on the transform.  So the limit only ever grows: setting it to this launch's size
// could lower it between another context's set and launch, and that launch would fail with cudaErrorInvalidValue.
template <class K>
static void set_smem(K kernel, size_t bytes) {
  static std::mutex m;
  static auto *limits = new std::map<std::pair<int, const void *>, size_t>();   // (device, kernel) -> limit set; never destroyed
  int dev = 0;
  TVM_CUDA(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> g(m);
  size_t &limit = (*limits)[{dev, (const void *)kernel}];
  if (bytes <= limit) return;
  TVM_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  limit = bytes;
}

void ntt_run(Ctx &c, const NttJob &job) {
  const int L = job.log_n;
  int LA, LB;
  if (L <= LT_MAX && job.num_cosets == 1 && !job.coset_pre && job.fold_count == 0) {
    LA = 0; LB = L;
  } else {
    LB = (L + 1) / 2; LA = L - LB;
    if (LB > LT_MAX) throw CudaError{cudaErrorInvalidValue, __FILE__, __LINE__};
  }
  const size_t n = (size_t)1 << L;
  const size_t ncolsB = job.ncols * job.num_cosets;
  const u64 *b_in = job.in;
  if (LA > 0 || job.num_cosets > 1 || job.coset_pre || job.fold_count) {
    PassA a{};
    a.in = job.in; a.out = job.tmp; a.in_cstride = job.in_cstride;
    a.log_n = L; a.LT = LA;
    int log_n1 = L - LA;
    a.log_t = pick_log_t(LA);
    if (a.log_t > log_n1) a.log_t = log_n1;
    u64 wn = root_of_unity_mont(L);
    if (job.inverse) wn = finv(wn);
    a.twist = c.get_pow_tab(wn, L);
    a.has_pre = job.coset_pre;
    a.fold_count = job.fold_count;
    if (job.coset_pre || job.fold_count) {
      const int tot = job.total_cosets ? job.total_cosets : job.num_cosets;
      int lr = 0;
      while ((1 << lr) < tot) lr++;
      a.pre = c.get_pow_tab(root_of_unity_mont(L + lr), L + lr);
    }
    a.coset_first = job.coset_first; a.coset_step = job.coset_step;
    size_t smem = tile_smem_bytes(LA, a.log_t);
    dim3 grid((unsigned)(((size_t)1 << log_n1) >> a.log_t), job.num_cosets, (unsigned)job.ncols);
    const u64 *tw = c.get_tile_tw(LA, job.inverse);
    if (job.inverse) {
      set_smem(ntt_pass_a_kernel<true>, smem);
      ntt_pass_a_kernel<true><<<grid, NTT_THREADS, smem, c.stream>>>(a, tw);
    } else {
      set_smem(ntt_pass_a_kernel<false>, smem);
      ntt_pass_a_kernel<false><<<grid, NTT_THREADS, smem, c.stream>>>(a, tw);
    }
    c.launches++;
    TVM_CUDA(cudaGetLastError());
    b_in = job.tmp;
  } else if (job.in_cstride != n) {
    throw CudaError{cudaErrorInvalidValue, __FILE__, __LINE__};  // single-pass needs packed columns
  }
  PassB b{};
  b.in = b_in; b.out = job.out; b.out_cstride = job.out_cstride;
  b.log_n = L; b.LT = LB;
  b.log_t = pick_log_t(LB);
  // rows = ncolsB * n2 must be a multiple of T
  size_t rows = ncolsB << (L - LB);
  while (b.log_t > 0 && (rows & (((size_t)1 << b.log_t) - 1))) b.log_t--;
  b.post_mul = job.post_mul;
  if (job.inverse) b.post_mul = fmul(b.post_mul, finv(to_mont((u64)n)));
  b.has_post = job.has_post; b.post = job.post;
  b.rand = job.rand; b.rand_count = job.rand_count; b.rand_pad = job.rand_pad;
  size_t smem = tile_smem_bytes(LB, b.log_t);
  unsigned grid = (unsigned)(rows >> b.log_t);
  const u64 *tw = c.get_tile_tw(LB, job.inverse);
  if (job.inverse) {
    set_smem(ntt_pass_b_kernel<true>, smem);
    ntt_pass_b_kernel<true><<<grid, NTT_THREADS, smem, c.stream>>>(b, tw);
  } else {
    set_smem(ntt_pass_b_kernel<false>, smem);
    ntt_pass_b_kernel<false><<<grid, NTT_THREADS, smem, c.stream>>>(b, tw);
  }
  c.launches++;
  TVM_CUDA(cudaGetLastError());
}

}  // namespace tvm
