// extern "C" boundary of libtvm_b200 (kernel-level entry points).  See include/tvm_b200.h.
#include "../../include/tvm_b200.h"
#include "ctx.h"
#include "air.cuh"
#include "launch.h"
#include "transcript.h"
#include "prove_common.h"
#include "stark.h"
#include "vm.h"
#include <algorithm>
#include <cstring>
#include <memory>
#include <new>
#include <stdexcept>

using namespace tvm;

struct tvm_ctx {
  Ctx c;
  ProveTimings timings;
};

namespace tvm {

int translate_exception(Ctx *c) {
  try {
    throw;
  } catch (const CudaError &e) {
    if (c) {
      char buf[512];
      snprintf(buf, sizeof buf, "CUDA error %d (%s) at %s:%d", (int)e.err, cudaGetErrorString(e.err), e.file, e.line);
      c->last_error = buf;
    }
    cudaGetLastError();
    return e.err == cudaErrorMemoryAllocation ? TVM_ERR_OOM : (e.err == cudaErrorInvalidValue ? TVM_ERR_INVALID_ARG : TVM_ERR_CUDA);
  } catch (const std::bad_alloc &) {
    if (c) c->last_error = "host allocation failed";
    return TVM_ERR_OOM;
  } catch (const ApiError &e) {
    if (c) c->last_error = e.msg;
    return e.code;
  } catch (const TranscriptCallbackError &) {
    if (c) c->last_error = "a transcript callback failed (or returned an index outside its range)";
    return TVM_ERR_INVALID_ARG;
  } catch (...) {
    if (c) c->last_error = "unknown internal error";
    return TVM_ERR_CUDA;
  }
}

__global__ void to_mont_kernel(u64 *d, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) d[i] = to_mont(d[i]);
}
__global__ void from_mont_kernel(u64 *d, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) d[i] = from_mont(d[i]);
}
// coset-major [c][k] -> natural i = c + r*k, fused with from_mont (host-facing outputs)
__global__ void coset_to_natural_canon_kernel(const u64 *in, u64 *out, size_t n, int log_r, size_t total) {
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;  // over ncols * r * n, output order
  if (idx >= total) return;
  size_t rn = n << log_r;
  size_t q = idx / rn, i = idx - q * rn;
  size_t c = i & (((size_t)1 << log_r) - 1), k = i >> log_r;
  out[idx] = from_mont(in[q * rn + c * n + k]);
}

void to_mont_run(Ctx &c, u64 *d, size_t n) {
  if (!n) return;
  to_mont_kernel<<<(unsigned)((n + 255) / 256), 256, 0, c.stream>>>(d, n);
  c.launches++;
  TVM_CUDA(cudaGetLastError());
}
void from_mont_run(Ctx &c, u64 *d, size_t n) {
  if (!n) return;
  from_mont_kernel<<<(unsigned)((n + 255) / 256), 256, 0, c.stream>>>(d, n);
  c.launches++;
  TVM_CUDA(cudaGetLastError());
}

// 1) interpolate on the trace domain (offset 1), fold in zerofier*randomizer, pre-scale by offset^j:
//    d_coef[col*coef_stride + j], j < n + rand_pad (entries num_rand <= j-n < rand_pad are zeroed)
void lde_interpolate_run(Ctx &c, const u64 *d_trace, const u64 *d_rand, unsigned num_rand, unsigned rand_pad, unsigned log2_trace,
                         u64 offset_mont, size_t ncols, u64 *d_coef, size_t coef_stride, u64 *d_tmp) {
  const size_t n = (size_t)1 << log2_trace;
  if (num_rand > n) throw ApiError{TVM_ERR_INVALID_ARG, "more trace randomizers than trace rows"};
  if (lde_interpolate_tiles(c, d_trace, d_rand, num_rand, rand_pad, log2_trace, offset_mont, ncols, d_coef, coef_stride, d_tmp)) return;
  NttJob inv{};
  inv.in = d_trace; inv.in_cstride = n;
  inv.out = d_coef; inv.out_cstride = coef_stride;
  inv.tmp = d_tmp;
  inv.log_n = (int)log2_trace; inv.ncols = ncols; inv.inverse = true;
  inv.has_post = true;
  inv.post = c.get_pow_tab(offset_mont, (int)log2_trace + 1);
  inv.rand = d_rand; inv.rand_count = d_rand ? num_rand : 0; inv.rand_pad = d_rand ? std::max(rand_pad, num_rand) : 0;
  ntt_run(c, inv);
}
// 2) evaluate pre-scaled coefficient columns on `num_cosets` of the 2^log2_cosets cosets
//    (domain coset coset_first + coset_step*y for y < num_cosets): d_out[(col*num_cosets + y)*n + k]
void lde_evaluate_run(Ctx &c, const u64 *d_coef, size_t coef_stride, unsigned fold_count, unsigned log2_trace, unsigned log2_cosets,
                      unsigned coset_first, unsigned coset_step, unsigned num_cosets, size_t ncols, u64 *d_out, u64 *d_tmp) {
  const size_t n = (size_t)1 << log2_trace;
  if (lde_evaluate_tiles(c, d_coef, coef_stride, fold_count, log2_trace, log2_cosets, coset_first, coset_step, num_cosets, ncols, d_out,
                         d_tmp))
    return;
  NttJob fwd{};
  fwd.in = d_coef; fwd.in_cstride = coef_stride;
  fwd.out = d_out; fwd.out_cstride = n;  // per (col*num_cosets + y)
  fwd.tmp = d_tmp;
  fwd.log_n = (int)log2_trace; fwd.ncols = ncols; fwd.inverse = false;
  fwd.num_cosets = (int)num_cosets; fwd.total_cosets = 1 << log2_cosets;
  fwd.coset_first = coset_first; fwd.coset_step = coset_step;
  fwd.coset_pre = true;
  fwd.fold_count = fold_count;
  ntt_run(c, fwd);
}
void lde_run(Ctx &c, const u64 *d_trace, const u64 *d_rand, unsigned num_rand, unsigned log2_trace,
             unsigned log2_cosets, u64 offset_mont, size_t ncols, u64 *d_coef, u64 *d_out, u64 *d_tmp) {
  const size_t n = (size_t)1 << log2_trace;
  lde_interpolate_run(c, d_trace, d_rand, num_rand, num_rand, log2_trace, offset_mont, ncols, d_coef, 2 * n, d_tmp);
  lde_evaluate_run(c, d_coef, 2 * n, d_rand ? num_rand : 0, log2_trace, log2_cosets, 0, 1, 1u << log2_cosets, ncols, d_out, d_tmp);
}

}  // namespace tvm

#define TVM_API_BEGIN(ctx) \
  Ctx *c__ = (ctx) ? &(ctx)->c : nullptr; \
  try { \
    if (c__) TVM_CUDA(cudaSetDevice(c__->device));
#define TVM_API_END \
    return TVM_OK; \
  } catch (...) { \
    return translate_exception(c__); \
  }

// the prover's randomness for `seed` in device memory of `mem` (canonical; main, aux, column 90, quotient segments)
struct SeededRandomness {
  const u64 *main_rand, *aux_rand, *randomizer_column, *quot_rand;
  size_t n, h, nq;   // trace length, trace randomizers, quotient randomizer coefficients
};
static SeededRandomness seeded_randomness(Ctx &c, DevMem &mem, const StarkParams &sp, uint64_t padded_height, const uint8_t *seed) {
  StarkDerived d{};
  if (int rc = stark_derive(sp, padded_height, d)) throw ApiError{rc, "parameter derivation failed"};
  const ProverRandomnessLayout L = prover_randomness_layout(d.trace_len, d.num_trace_randomizers, d.num_quotient_randomizer_coefficients);
  u64 *d_r = mem.words(L.total);
  prover_randomness_run(c, seed, d.trace_len, d.num_trace_randomizers, d.num_quotient_randomizer_coefficients, d_r);
  return {d_r + L.main, d_r + L.aux, d_r + L.randomizer_column, d_r + L.quot, d.trace_len, d.num_trace_randomizers,
          d.num_quotient_randomizer_coefficients};
}

// the proof into the caller's buffer; *proof_len receives the proof's length even when the buffer is missing or too small,
// so that the caller can size a second attempt
static void copy_proof_out(const std::vector<u64> &proof, uint64_t *proof_out, size_t *proof_len) {
  const size_t cap = *proof_len;
  *proof_len = proof.size();
  if (!proof_out || cap < proof.size()) throw ApiError{TVM_ERR_INVALID_ARG, "proof buffer too small"};
  memcpy(proof_out, proof.data(), proof.size() * 8);
}

// a low-degree test's revealed indices: *num_indices (optional) receives their count, indices_out (optional) the indices
static void copy_indices_out(const std::vector<uint32_t> &revealed, uint32_t *indices_out, size_t *num_indices) {
  const size_t cap = num_indices ? *num_indices : 0;
  if (num_indices) *num_indices = revealed.size();
  if (indices_out) {
    if (cap < revealed.size()) throw ApiError{TVM_ERR_INVALID_ARG, "index buffer too small"};
    memcpy(indices_out, revealed.data(), revealed.size() * sizeof(uint32_t));
  }
}

// What every tvm_prove* entry point does after its own argument checks.  With a seed the randomness is drawn into device
// memory first (after whatever the caller already holds there, so before the prove reads free memory to choose its mode).
// Then the prove, and the proof copied out, unless proof_len is NULL: an external transcript keeps the proof stream.
static void run_prove(tvm_ctx *ctx, const tvm_params &params, const ClaimView &cv, uint64_t padded_height, ProveInputs in,
                      const uint8_t *seed, uint64_t *proof_out, size_t *proof_len) {
  Ctx &c = ctx->c;
  const StarkParams sp = stark_params(params);
  std::vector<u64> proof;
  {
    DevMem mem(c);
    if (seed) {
      const SeededRandomness r = seeded_randomness(c, mem, sp, padded_height, seed);
      in.main_rand = r.main_rand; in.aux_rand = r.aux_rand; in.randomizer_column = r.randomizer_column; in.quot_rand = r.quot_rand;
    }
    stark_prove(c, sp, cv, padded_height, in, proof, &ctx->timings);
  }
  if (proof_len) copy_proof_out(proof, proof_out, proof_len);
}

extern "C" {

int tvm_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}

int tvm_ctx_create(tvm_ctx **out, int device) {
  if (!out) return TVM_ERR_INVALID_ARG;
  *out = nullptr;
  int n = tvm_device_count();
  if (device < 0 || device >= n) return TVM_ERR_CUDA;  // no CPU fallback: fail loudly without a GPU
  tvm_ctx *ctx = new (std::nothrow) tvm_ctx();
  if (!ctx) return TVM_ERR_OOM;
  ctx->c.device = device;
  if (cudaSetDevice(device) != cudaSuccess || cudaDeviceGetAttribute(&ctx->c.num_sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess ||
      cudaStreamCreateWithFlags(&ctx->c.stream, cudaStreamNonBlocking) != cudaSuccess) {
    cudaGetLastError();
    delete ctx;
    return TVM_ERR_CUDA;
  }
  ctx->c.own_stream = true;
  *out = ctx;
  return TVM_OK;
}

void tvm_ctx_destroy(tvm_ctx *ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->c.device);
  cudaStreamSynchronize(ctx->c.stream);
  delete ctx;
}

int tvm_ctx_set_stream(tvm_ctx *ctx, void *stream) {
  if (!ctx) return TVM_ERR_INVALID_ARG;
  TVM_API_BEGIN(ctx)
  TVM_CUDA(cudaStreamSynchronize(c__->stream));
  if (c__->own_stream) { cudaStreamDestroy(c__->stream); c__->own_stream = false; }
  if (stream) c__->stream = (cudaStream_t)stream;
  else { TVM_CUDA(cudaStreamCreateWithFlags(&c__->stream, cudaStreamNonBlocking)); c__->own_stream = true; }
  TVM_API_END
}

int tvm_ctx_set_comm(tvm_ctx *ctx, const tvm_comm *comm) {
  if (!ctx) return TVM_ERR_INVALID_ARG;
  TVM_API_BEGIN(ctx)
  if (!comm) { c__->comm = tvm_comm{0, 1, nullptr, nullptr, nullptr}; return TVM_OK; }
  const int w = comm->world;
  if (!(w == 1 || w == 2 || w == 4 || w == 8) || comm->rank < 0 || comm->rank >= w) throw ApiError{TVM_ERR_INVALID_ARG, "comm: world must be 1, 2, 4 or 8 and 0 <= rank < world"};
  if (w > 1 && (!comm->all_gather || !comm->all_reduce_sum_u64)) throw ApiError{TVM_ERR_INVALID_ARG, "comm: missing collective callbacks"};
  c__->comm = *comm;
  TVM_API_END
}

int tvm_ctx_set_low_memory(tvm_ctx *ctx, int mode) {
  if (!ctx || mode < 0 || mode > 2) return TVM_ERR_INVALID_ARG;
  ctx->c.low_memory_mode = mode;
  return TVM_OK;
}
int tvm_last_prove_low_memory(const tvm_ctx *ctx) { return ctx && ctx->timings.low_memory ? 1 : 0; }

int tvm_ctx_release_cached_memory(tvm_ctx *ctx) {
  if (!ctx) return TVM_ERR_INVALID_ARG;
  TVM_API_BEGIN(ctx)
  TVM_CUDA(cudaStreamSynchronize(c__->stream));
  while (!c__->pool_free.empty()) {         // each block leaves the pool before it is freed: no double free on an error
    void *p = c__->pool_free.begin()->second;
    c__->pool_free.erase(c__->pool_free.begin());
    TVM_CUDA(cudaFree(p));
  }
  for (auto &s : c__->scratch) {
    void *p = s.p;
    s.p = nullptr;
    s.bytes = 0;
    if (p) TVM_CUDA(cudaFree(p));
  }
  TVM_API_END
}

int tvm_ctx_synchronize(tvm_ctx *ctx) {
  if (!ctx) return TVM_ERR_INVALID_ARG;
  TVM_API_BEGIN(ctx)
  TVM_CUDA(cudaStreamSynchronize(c__->stream));
  TVM_API_END
}

const char *tvm_strerror(int code) {
  switch (code) {
    case TVM_OK: return "ok";
    case TVM_ERR_INVALID_ARG: return "invalid argument";
    case TVM_ERR_CUDA: return "CUDA failure (or no CUDA device: this library has no CPU fallback)";
    case TVM_ERR_OOM: return "out of memory (ProvingError::OutOfMemory)";
    case TVM_ERR_ZK_VIOLATION: return "out-of-domain point collides with a revealed row (ProvingError::ZeroKnowledgeViolation)";
    case TVM_ERR_DOMAIN: return "arithmetic domain error";
    case TVM_ERR_LDT_PARAMS: return "low-degree-test parameter error";
    case TVM_ERR_STATE: return "entry point called out of order";
    case TVM_ERR_UNSUPPORTED: return "unsupported configuration";
    case TVM_ERR_VERIFICATION: return "proof rejected (VerificationError)";
    case TVM_ERR_VM: return "the program cannot be executed (VMError / ProgramDecodingError)";
    default: return "unknown error";
  }
}
const char *tvm_last_error(const tvm_ctx *ctx) { return ctx ? ctx->c.last_error.c_str() : ""; }
uint64_t tvm_launch_count(const tvm_ctx *ctx) { return ctx ? ctx->c.launches : 0; }

int tvm_to_mont_dev(tvm_ctx *ctx, uint64_t *d, size_t n) {
  if (!ctx) return TVM_ERR_INVALID_ARG;
  TVM_API_BEGIN(ctx)
  to_mont_run(*c__, (u64 *)d, n);
  TVM_API_END
}
int tvm_from_mont_dev(tvm_ctx *ctx, uint64_t *d, size_t n) {
  if (!ctx) return TVM_ERR_INVALID_ARG;
  TVM_API_BEGIN(ctx)
  from_mont_run(*c__, (u64 *)d, n);
  TVM_API_END
}

int tvm_ntt_bfe_dev(tvm_ctx *ctx, const uint64_t *d_in, uint64_t *d_out, uint64_t *d_tmp, unsigned log2n, size_t ncols, int inverse) {
  if (!ctx || !d_in || !d_out || log2n > 32) return TVM_ERR_INVALID_ARG;
  TVM_API_BEGIN(ctx)
  if (!ncols) return TVM_OK;
  NttJob j{};
  size_t n = (size_t)1 << log2n;
  j.in = (const u64 *)d_in; j.in_cstride = n; j.out = (u64 *)d_out; j.out_cstride = n; j.tmp = (u64 *)d_tmp;
  j.log_n = (int)log2n; j.ncols = ncols; j.inverse = inverse != 0;
  if (log2n > 13 && !d_tmp) throw ApiError{TVM_ERR_INVALID_ARG, "tvm_ntt_bfe_dev: d_tmp required for log2n > 13"};
  if (log2n > 26) throw ApiError{TVM_ERR_UNSUPPORTED, "tvm_ntt_bfe_dev: log2n > 26 not supported"};
  ntt_run(*c__, j);
  TVM_API_END
}

int tvm_ntt_bfe(tvm_ctx *ctx, uint64_t *host, unsigned log2n, size_t ncols, int inverse) {
  if (!ctx || !host) return TVM_ERR_INVALID_ARG;
  TVM_API_BEGIN(ctx)
  size_t n = (size_t)1 << log2n, total = n * ncols;
  if (!total) return TVM_OK;
  u64 *d = (u64 *)c__->scratch_get(0, total * 8);
  u64 *t = (u64 *)c__->scratch_get(1, total * 8);
  u64 *o = (u64 *)c__->scratch_get(2, total * 8);
  TVM_CUDA(cudaMemcpyAsync(d, host, total * 8, cudaMemcpyHostToDevice, c__->stream));
  to_mont_run(*c__, d, total);
  int rc = tvm_ntt_bfe_dev(ctx, d, o, t, log2n, ncols, inverse);
  if (rc) return rc;
  from_mont_run(*c__, o, total);
  TVM_CUDA(cudaMemcpyAsync(host, o, total * 8, cudaMemcpyDeviceToHost, c__->stream));
  TVM_CUDA(cudaStreamSynchronize(c__->stream));
  TVM_API_END
}

int tvm_lde_bfe_dev(tvm_ctx *ctx, const uint64_t *d_trace, const uint64_t *d_rand, unsigned num_rand, unsigned log2_trace,
                    unsigned log2_cosets, uint64_t offset_canon, size_t ncols, uint64_t *d_coef, uint64_t *d_out, uint64_t *d_tmp) {
  if (!ctx || !d_trace || !d_coef || !d_out || !d_tmp) return TVM_ERR_INVALID_ARG;
  if (log2_trace > 26 || log2_cosets > 6 || offset_canon >= P || offset_canon == 0) return TVM_ERR_DOMAIN;
  TVM_API_BEGIN(ctx)
  if (!ncols) return TVM_OK;
  lde_run(*c__, (const u64 *)d_trace, (const u64 *)d_rand, num_rand, log2_trace, log2_cosets, to_mont(offset_canon), ncols,
          (u64 *)d_coef, (u64 *)d_out, (u64 *)d_tmp);
  TVM_API_END
}

int tvm_lde_bfe_cosets_dev(tvm_ctx *ctx, const uint64_t *d_trace, const uint64_t *d_rand, unsigned num_rand, unsigned log2_trace,
                           unsigned log2_cosets, uint64_t offset_canon, unsigned coset_first, unsigned coset_step,
                           unsigned num_cosets, size_t ncols, uint64_t *d_coef, uint64_t *d_out, uint64_t *d_tmp) {
  if (!ctx || !d_trace || !d_coef || !d_out || !d_tmp) return TVM_ERR_INVALID_ARG;
  if (log2_trace > 26 || log2_cosets > 6 || offset_canon >= P || offset_canon == 0) return TVM_ERR_DOMAIN;
  if (num_cosets == 0 || coset_first + (uint64_t)coset_step * (num_cosets - 1) >= (1ull << log2_cosets)) return TVM_ERR_DOMAIN;
  TVM_API_BEGIN(ctx)
  if (!ncols) return TVM_OK;
  const size_t n = (size_t)1 << log2_trace;
  lde_interpolate_run(*c__, (const u64 *)d_trace, (const u64 *)d_rand, num_rand, num_rand, log2_trace, to_mont(offset_canon), ncols,
                      (u64 *)d_coef, 2 * n, (u64 *)d_tmp);
  lde_evaluate_run(*c__, (const u64 *)d_coef, 2 * n, d_rand ? num_rand : 0, log2_trace, log2_cosets, coset_first, coset_step, num_cosets,
                   ncols, (u64 *)d_out, (u64 *)d_tmp);
  TVM_API_END
}

int tvm_lde_bfe(tvm_ctx *ctx, const uint64_t *trace, const uint64_t *rand, unsigned num_rand, unsigned log2_trace,
                unsigned log2_cosets, uint64_t offset_canon, size_t ncols, uint64_t *out) {
  if (!ctx || !trace || !out) return TVM_ERR_INVALID_ARG;
  TVM_API_BEGIN(ctx)
  size_t n = (size_t)1 << log2_trace, rn = n << log2_cosets;
  if (!ncols) return TVM_OK;
  // slot 0: trace + rand ; slot 1: coef ; slot 2: out (coset-major) ; slot 3: tmp, later natural-order output
  size_t in_words = ncols * n + (rand ? ncols * (size_t)num_rand : 0);
  u64 *d_in = (u64 *)c__->scratch_get(0, in_words * 8);
  u64 *d_coef = (u64 *)c__->scratch_get(1, ncols * 2 * n * 8);
  u64 *d_out = (u64 *)c__->scratch_get(2, ncols * rn * 8);
  u64 *d_tmp = (u64 *)c__->scratch_get(3, ncols * rn * 8);
  TVM_CUDA(cudaMemcpyAsync(d_in, trace, ncols * n * 8, cudaMemcpyHostToDevice, c__->stream));
  u64 *d_rand = nullptr;
  if (rand && num_rand) {
    d_rand = d_in + ncols * n;
    TVM_CUDA(cudaMemcpyAsync(d_rand, rand, ncols * (size_t)num_rand * 8, cudaMemcpyHostToDevice, c__->stream));
  }
  to_mont_run(*c__, d_in, in_words);
  int rc = tvm_lde_bfe_dev(ctx, d_in, d_rand, num_rand, log2_trace, log2_cosets, offset_canon, ncols, d_coef, d_out, d_tmp);
  if (rc) return rc;
  size_t total = ncols * rn;
  coset_to_natural_canon_kernel<<<(unsigned)((total + 255) / 256), 256, 0, c__->stream>>>(d_out, d_tmp, n, (int)log2_cosets, total);
  c__->launches++;
  TVM_CUDA(cudaGetLastError());
  TVM_CUDA(cudaMemcpyAsync(out, d_tmp, total * 8, cudaMemcpyDeviceToHost, c__->stream));
  TVM_CUDA(cudaStreamSynchronize(c__->stream));
  TVM_API_END
}

int tvm_tip5_hash_rows_dev(tvm_ctx *ctx, const uint64_t *d_table, size_t col_stride, size_t nrows, unsigned ncols,
                           unsigned log2_cosets, uint64_t *d_digests) {
  if (!ctx || !d_table || !d_digests) return TVM_ERR_INVALID_ARG;
  TVM_API_BEGIN(ctx)
  if (!nrows) return TVM_OK;
  if (log2_cosets && (nrows & (((size_t)1 << log2_cosets) - 1))) throw ApiError{TVM_ERR_INVALID_ARG, "nrows not a multiple of the coset count"};
  hash_rows_run(*c__, (const u64 *)d_table, col_stride, nrows, ncols, (int)log2_cosets, (u64 *)d_digests);
  TVM_API_END
}

int tvm_tip5_hash_rows(tvm_ctx *ctx, const uint64_t *table, size_t nrows, unsigned ncols, uint64_t *digests) {
  if (!ctx || !digests || (!table && nrows && ncols)) return TVM_ERR_INVALID_ARG;
  TVM_API_BEGIN(ctx)
  if (!nrows) return TVM_OK;
  size_t words = nrows * (size_t)ncols;
  u64 *d = (u64 *)c__->scratch_get(0, (words ? words : 1) * 8);
  u64 *dg = (u64 *)c__->scratch_get(1, nrows * 5 * 8);
  if (words) {
    TVM_CUDA(cudaMemcpyAsync(d, table, words * 8, cudaMemcpyHostToDevice, c__->stream));
    to_mont_run(*c__, d, words);
  }
  hash_rows_run(*c__, d, nrows, nrows, ncols, 0, dg);
  from_mont_run(*c__, dg, nrows * 5);
  TVM_CUDA(cudaMemcpyAsync(digests, dg, nrows * 5 * 8, cudaMemcpyDeviceToHost, c__->stream));
  TVM_CUDA(cudaStreamSynchronize(c__->stream));
  TVM_API_END
}

int tvm_tip5_hash_varlen(const uint64_t *words, size_t n, uint64_t digest[5]) {
  if (!digest || (!words && n)) return TVM_ERR_INVALID_ARG;
  try {
    std::vector<u64> w(n);
    for (size_t i = 0; i < n; i++) {
      if (words[i] >= P) return TVM_ERR_INVALID_ARG;
      w[i] = to_mont(words[i]);
    }
    u64 d[5];
    tip5_hash_varlen_host(w.data(), n, d);
    for (int i = 0; i < 5; i++) digest[i] = from_mont(d[i]);
    return TVM_OK;
  } catch (...) {
    return TVM_ERR_OOM;
  }
}

int tvm_merkle_build_dev(tvm_ctx *ctx, uint64_t *d_nodes, size_t nleaves) {
  if (!ctx || !d_nodes || nleaves == 0 || (nleaves & (nleaves - 1))) return TVM_ERR_INVALID_ARG;
  TVM_API_BEGIN(ctx)
  merkle_run(*c__, (u64 *)d_nodes, nleaves);
  TVM_API_END
}

int tvm_tip5_arith_check_dev(tvm_ctx *ctx, const uint64_t *d_in, size_t n, uint64_t *d_out) {
  if (!ctx || (n && (!d_in || !d_out))) return TVM_ERR_INVALID_ARG;
  TVM_API_BEGIN(ctx)
  if (!n) return TVM_OK;
  tip5_arith_check_run(*c__, (const u64 *)d_in, n, (u64 *)d_out);
  TVM_API_END
}

int tvm_merkle_build(tvm_ctx *ctx, const uint64_t *leaves, size_t nleaves, uint64_t *nodes_out, uint64_t root[5]) {
  if (!ctx || !leaves || !root || nleaves == 0 || (nleaves & (nleaves - 1))) return TVM_ERR_INVALID_ARG;
  TVM_API_BEGIN(ctx)
  u64 *d = (u64 *)c__->scratch_get(0, 2 * nleaves * 5 * 8);
  TVM_CUDA(cudaMemsetAsync(d, 0, 40, c__->stream));
  TVM_CUDA(cudaMemcpyAsync(d + 5 * nleaves, leaves, nleaves * 40, cudaMemcpyHostToDevice, c__->stream));
  to_mont_run(*c__, d + 5 * nleaves, nleaves * 5);
  merkle_run(*c__, d, nleaves);
  from_mont_run(*c__, d, 2 * nleaves * 5);
  if (nodes_out) TVM_CUDA(cudaMemcpyAsync(nodes_out, d, 2 * nleaves * 40, cudaMemcpyDeviceToHost, c__->stream));
  TVM_CUDA(cudaMemcpyAsync(root, d + 5, 40, cudaMemcpyDeviceToHost, c__->stream));
  TVM_CUDA(cudaStreamSynchronize(c__->stream));
  TVM_API_END
}

int tvm_air_quotient_dev(tvm_ctx *ctx, const uint64_t *d_main, size_t main_stride, const uint64_t *d_aux, size_t aux_stride,
                         const uint64_t *challenges, const uint64_t *weights, unsigned log2_trace, unsigned log2_cosets,
                         uint64_t offset_canon, uint64_t *d_out, size_t out_stride) {
  if (!ctx || !d_main || !d_aux || !challenges || !weights || !d_out) return TVM_ERR_INVALID_ARG;
  if (offset_canon == 0 || offset_canon >= P || log2_trace + log2_cosets > 32) return TVM_ERR_DOMAIN;
  TVM_API_BEGIN(ctx)
  const size_t nc = 3 * TVM_NUM_CHALLENGES, nw = 3 * TVM_NUM_CONSTRAINTS;
  std::vector<u64> h(nc + nw);
  for (size_t i = 0; i < nc; i++) h[i] = to_mont(challenges[i] % P);
  for (size_t i = 0; i < nw; i++) h[nc + i] = to_mont(weights[i] % P);
  u64 *d = (u64 *)c__->scratch_get(3, (nc + nw) * 8);
  TVM_CUDA(cudaMemcpyAsync(d, h.data(), (nc + nw) * 8, cudaMemcpyHostToDevice, c__->stream));
  TVM_CUDA(cudaStreamSynchronize(c__->stream));  // h is a stack-owned staging buffer
  air_quotient_run(*c__, (const u64 *)d_main, main_stride, (const u64 *)d_aux, aux_stride, d, d + nc, log2_trace, log2_cosets, 0, 1, 1u << log2_cosets, 1,
                   to_mont(offset_canon), (u64 *)d_out, out_stride);
  TVM_API_END
}

int tvm_air_quotient_coef_dev(tvm_ctx *ctx, const uint64_t *d_main_coef, const uint64_t *d_aux_coef, size_t coef_stride,
                              unsigned num_rand, const uint64_t *challenges, const uint64_t *weights, unsigned log2_trace,
                              uint64_t offset_canon, uint64_t *d_out, size_t out_stride) {
  if (!ctx || !d_main_coef || !d_aux_coef || !challenges || !weights || !d_out) return TVM_ERR_INVALID_ARG;
  if (offset_canon == 0 || offset_canon >= P || log2_trace < 1 || log2_trace + 3 > 27) return TVM_ERR_DOMAIN;
  const size_t n = (size_t)1 << log2_trace, len = n + num_rand;
  if (num_rand > n || coef_stride < len || out_stride < 8 * n) return TVM_ERR_INVALID_ARG;
  TVM_API_BEGIN(ctx)
  Ctx &c = *c__;
  const size_t nc = 3 * TVM_NUM_CHALLENGES, nw = 3 * TVM_NUM_CONSTRAINTS;
  std::vector<u64> hw(nc + nw);
  for (size_t i = 0; i < nc; i++) hw[i] = to_mont(challenges[i] % P);
  for (size_t i = 0; i < nw; i++) hw[nc + i] = to_mont(weights[i] % P);
  const size_t nmain = TVM_NUM_MAIN_COLUMNS, ncols = nmain + AIR_AUX_BCOLS, tmp_cols = 16;
  // [consts | coefficients pre-scaled by offset^j [ncols][len] | LDE [ncols][8n] | transform scratch]
  u64 *buf = (u64 *)c.pool_alloc(sizeof(u64) * (nc + nw + ncols * len + ncols * 8 * n + tmp_cols * 8 * n));
  u64 *d = buf, *coef = d + nc + nw, *lde = coef + ncols * len, *tmp = lde + ncols * 8 * n;
  try {
    TVM_CUDA(cudaMemcpyAsync(d, hw.data(), (nc + nw) * 8, cudaMemcpyHostToDevice, c.stream));
    TVM_CUDA(cudaMemcpy2DAsync(coef, len * 8, d_main_coef, coef_stride * 8, len * 8, nmain, cudaMemcpyDeviceToDevice, c.stream));
    TVM_CUDA(cudaMemcpy2DAsync(coef + nmain * len, len * 8, d_aux_coef, coef_stride * 8, len * 8, AIR_AUX_BCOLS,
                               cudaMemcpyDeviceToDevice, c.stream));
    const u64 off = to_mont(offset_canon);
    scale_by_powers_run(c, coef, len, (int)ncols, len, c.get_pow_tab(off, (int)log2_trace + 1));
    for (size_t c0 = 0; c0 < ncols; c0 += tmp_cols)   // coefficients n..len-1 fold into 0..num_rand-1 (u^n = w_8^coset)
      lde_evaluate_run(c, coef + c0 * len, len, num_rand, log2_trace, 3, 0, 1, 8, std::min(tmp_cols, ncols - c0), lde + c0 * 8 * n, tmp);
    const AirCoefs cf{coef, coef + nmain * len, len, num_rand};
    air_quotient_run(c, lde, 8 * n, lde + nmain * 8 * n, 8 * n, d, d + nc, log2_trace, 3, 0, 1, 8, 1, off, (u64 *)d_out, out_stride, &cf);
    TVM_CUDA(cudaStreamSynchronize(c.stream));   // hw is a stack-owned staging buffer
  } catch (...) {
    c.pool_release(buf);
    throw;
  }
  c.pool_release(buf);
  TVM_API_END
}

int tvm_derive_domains(const tvm_params *p, uint64_t padded_height, tvm_domains *out) {
  if (!p || !out) return TVM_ERR_INVALID_ARG;
  StarkDerived d{};
  int rc = stark_derive(stark_params(*p), padded_height, d);
  if (rc) return rc;
  out->padded_height = d.padded_height; out->num_trace_randomizers = d.num_trace_randomizers;
  out->randomized_trace_len = d.randomized_trace_len; out->trace_len = d.trace_len; out->quotient_len = d.quotient_len;
  out->ldt_len = d.ldt_len; out->ldt_offset = d.ldt_offset; out->num_collinearity_checks = d.fri.num_collinearity_checks;
  out->fri_num_rounds = d.fri.num_rounds; out->fri_last_round_max_degree = d.fri.last_round_max_degree;
  out->num_quotient_randomizer_coefficients = d.num_quotient_randomizer_coefficients;
  out->ldt = (uint64_t)d.ldt; out->num_first_round_queries = d.num_first_round_queries;
  out->stir_num_rounds = d.ldt == 2 ? (uint64_t)d.stir.num_rounds : 0;
  for (int i = 0; i < 16; i++) {
    out->stir_in_domain_queries[i] = d.ldt == 2 && i < d.stir.num_rounds ? d.stir.in_domain[i] : 0;
    out->stir_out_of_domain_queries[i] = d.ldt == 2 && i < d.stir.num_rounds ? d.stir.out_of_domain[i] : 0;
  }
  out->stir_final_num_queries = d.ldt == 2 ? d.stir.final_num_in_domain_queries : 0;
  out->stir_final_degree = d.ldt == 2 ? d.stir.final_degree : 0;
  return TVM_OK;
}

int tvm_aux_extend(tvm_ctx *ctx, const uint64_t *main_trace, unsigned log2_n, const uint64_t *challenges,
                   const uint64_t *randomizer_column, uint64_t *aux_trace_out) {
  if (!ctx || !main_trace || !challenges || !aux_trace_out) return TVM_ERR_INVALID_ARG;
  if (log2_n > 26) return TVM_ERR_DOMAIN;
  TVM_API_BEGIN(ctx)
  const size_t n = (size_t)1 << log2_n, NM = TVM_NUM_MAIN_COLUMNS, NA = TVM_NUM_AUX_COLUMNS;
  Ctx &c = *c__;
  DevMem mem(c);      // RAII: every block goes back to the pool on all exit paths (an allocation failure used to strand the earlier ones)
  u64 *d_main = mem.words(NM * n);
  u64 *d_aux = mem.words(3 * NA * n);      // planes; reused as staging for the interleaved output
  u64 *d_out = mem.words(3 * NA * n);
  u64 *d_ch = mem.words(3 * TVM_NUM_CHALLENGES);
  TVM_CUDA(cudaMemcpyAsync(d_main, main_trace, NM * n * 8, cudaMemcpyDefault, c.stream));
  TVM_CUDA(cudaMemcpyAsync(d_ch, challenges, 3 * TVM_NUM_CHALLENGES * 8, cudaMemcpyDefault, c.stream));
  to_mont_run(c, d_main, NM * n);
  to_mont_run(c, d_ch, 3 * TVM_NUM_CHALLENGES);
  aux_extend_on_device(c, mem, d_main, n, d_ch, (const u64 *)randomizer_column, d_aux);
  interleave3_from_mont_run(c, d_aux, d_out, n, NA);
  TVM_CUDA(cudaMemcpyAsync(aux_trace_out, d_out, 3 * NA * n * 8, cudaMemcpyDefault, c.stream));
  TVM_CUDA(cudaStreamSynchronize(c.stream));
  TVM_API_END
}

int tvm_fill_derived_main_columns(tvm_ctx *ctx, uint64_t *main_trace, unsigned log2_n) {
  if (!ctx || !main_trace) return TVM_ERR_INVALID_ARG;
  if (log2_n > 26) return TVM_ERR_DOMAIN;
  TVM_API_BEGIN(ctx)
  const size_t n = (size_t)1 << log2_n, NM = TVM_NUM_MAIN_COLUMNS, NB = TVM_NUM_MAIN_TABLE_COLUMNS;
  Ctx &c = *c__;
  u64 *d_main = (u64 *)c.pool_alloc(NM * n * 8);
  try {
    TVM_CUDA(cudaMemcpyAsync(d_main, main_trace, NB * n * 8, cudaMemcpyDefault, c.stream));
    to_mont_run(c, d_main, NB * n);
    main_derived_run(c, d_main, n);
    from_mont_run(c, d_main + NB * n, (NM - NB) * n);
    TVM_CUDA(cudaMemcpyAsync(main_trace + NB * n, d_main + NB * n, (NM - NB) * n * 8, cudaMemcpyDefault, c.stream));
    TVM_CUDA(cudaStreamSynchronize(c.stream));
  } catch (...) {
    cudaStreamSynchronize(c.stream);
    c.pool_release(d_main);
    throw;
  }
  c.pool_release(d_main);
  TVM_API_END
}

int tvm_prove(tvm_ctx *ctx, const tvm_params *params, const tvm_claim *claim, uint64_t padded_height, const uint64_t *main_trace,
              const uint64_t *main_rand, tvm_aux_callback aux_cb, void *aux_user, const uint64_t *quot_rand, uint64_t *proof_out,
              size_t *proof_len) {
  if (!ctx || !params || !claim || !main_trace || !main_rand || !aux_cb || !quot_rand || !proof_len) return TVM_ERR_INVALID_ARG;
  if (params->ldt_choice > 2 || !claim_ok(claim)) return TVM_ERR_INVALID_ARG;
  TVM_API_BEGIN(ctx)
  ProveInputs in;
  in.main_trace = (const u64 *)main_trace; in.main_rand = (const u64 *)main_rand; in.quot_rand = (const u64 *)quot_rand;
  in.aux_cb = (AuxCallback)aux_cb; in.aux_user = aux_user;
  run_prove(ctx, *params, claim_view(*claim), padded_height, in, nullptr, proof_out, proof_len);
  TVM_API_END
}

int tvm_prove_transcript(tvm_ctx *ctx, const tvm_params *params, const tvm_claim *claim, uint64_t padded_height, const uint64_t *main_trace,
                         const uint64_t *main_rand, tvm_aux_callback aux_cb, void *aux_user, const uint64_t *quot_rand,
                         const tvm_transcript *transcript) {
  if (!ctx || !params || !claim || !main_trace || !main_rand || !aux_cb || !quot_rand || !transcript) return TVM_ERR_INVALID_ARG;
  if (!transcript->alter_fiat_shamir_state || !transcript->enqueue || !transcript->sample_scalars || !transcript->sample_indices)
    return TVM_ERR_INVALID_ARG;
  if (params->ldt_choice > 2 || !claim_ok(claim)) return TVM_ERR_INVALID_ARG;
  TVM_API_BEGIN(ctx)
  const ExternalTranscript ext{transcript->user, transcript->alter_fiat_shamir_state, transcript->enqueue, transcript->sample_scalars,
                               transcript->sample_indices};
  ProveInputs in;
  in.main_trace = (const u64 *)main_trace; in.main_rand = (const u64 *)main_rand; in.quot_rand = (const u64 *)quot_rand;
  in.aux_cb = (AuxCallback)aux_cb; in.aux_user = aux_user;
  in.ext = &ext;
  run_prove(ctx, *params, claim_view(*claim), padded_height, in, nullptr, nullptr, nullptr);
  TVM_API_END
}

int tvm_prove_tables(tvm_ctx *ctx, const tvm_params *params, const tvm_claim *claim, uint64_t padded_height, const uint64_t *main_table,
                     int fill_derived_main_columns, const uint64_t *main_rand, const uint64_t *aux_rand, const uint64_t *randomizer_column,
                     const uint64_t *quot_rand, uint64_t *proof_out, size_t *proof_len) {
  if (!ctx || !params || !claim || !main_table || !main_rand || !aux_rand || !quot_rand || !proof_len) return TVM_ERR_INVALID_ARG;
  if (params->ldt_choice > 2 || !claim_ok(claim)) return TVM_ERR_INVALID_ARG;
  TVM_API_BEGIN(ctx)
  ProveInputs in;
  in.main_trace = (const u64 *)main_table; in.fill_derived_main = fill_derived_main_columns != 0;
  in.main_rand = (const u64 *)main_rand; in.aux_rand = (const u64 *)aux_rand; in.randomizer_column = (const u64 *)randomizer_column;
  in.quot_rand = (const u64 *)quot_rand;
  run_prove(ctx, *params, claim_view(*claim), padded_height, in, nullptr, proof_out, proof_len);
  TVM_API_END
}

int tvm_main_table_from_aet(tvm_ctx *ctx, const tvm_aet *aet, uint64_t num_rows, uint64_t *main_table_out, uint64_t *table_lengths_out) {
  if (!ctx || !aet || !main_table_out) return TVM_ERR_INVALID_ARG;
  if (num_rows < 256 || (num_rows & (num_rows - 1)) || num_rows > ((uint64_t)1 << 26)) return TVM_ERR_DOMAIN;
  TVM_API_BEGIN(ctx)
  Ctx &c = *c__;
  const size_t n = (size_t)num_rows, NM = TVM_NUM_MAIN_COLUMNS;
  DevMem mem(c);
  u64 *d_main = mem.words(NM * n);
  main_table_on_device(c, d_main, n, *aet, table_lengths_out);
  from_mont_run(c, d_main, NM * n);
  TVM_CUDA(cudaMemcpyAsync(main_table_out, d_main, NM * n * 8, cudaMemcpyDefault, c.stream));
  TVM_CUDA(cudaStreamSynchronize(c.stream));
  TVM_API_END
}

int tvm_prove_aet(tvm_ctx *ctx, const tvm_params *params, const tvm_claim *claim, uint64_t padded_height, const tvm_aet *aet,
                  const uint64_t *main_rand, const uint64_t *aux_rand, const uint64_t *randomizer_column, const uint64_t *quot_rand,
                  uint64_t *proof_out, size_t *proof_len) {
  if (!ctx || !params || !claim || !aet || !main_rand || !aux_rand || !quot_rand || !proof_len) return TVM_ERR_INVALID_ARG;
  if (params->ldt_choice > 2 || !claim_ok(claim)) return TVM_ERR_INVALID_ARG;
  TVM_API_BEGIN(ctx)
  ProveInputs in;
  in.aet = aet;
  in.main_rand = (const u64 *)main_rand; in.aux_rand = (const u64 *)aux_rand; in.randomizer_column = (const u64 *)randomizer_column;
  in.quot_rand = (const u64 *)quot_rand;
  run_prove(ctx, *params, claim_view(*claim), padded_height, in, nullptr, proof_out, proof_len);
  TVM_API_END
}

int tvm_prover_randomness(tvm_ctx *ctx, const tvm_params *params, uint64_t padded_height, const uint8_t seed[32], uint64_t *main_rand_out,
                          uint64_t *aux_rand_out, uint64_t *randomizer_column_out, uint64_t *quot_rand_out) {
  if (!ctx || !params || !seed || params->ldt_choice > 2) return TVM_ERR_INVALID_ARG;
  TVM_API_BEGIN(ctx)
  Ctx &c = *c__;
  DevMem mem(c);
  const SeededRandomness r = seeded_randomness(c, mem, stark_params(*params), padded_height, seed);
  if (main_rand_out) TVM_CUDA(cudaMemcpyAsync(main_rand_out, r.main_rand, TVM_NUM_MAIN_COLUMNS * r.h * 8, cudaMemcpyDefault, c.stream));
  if (aux_rand_out) TVM_CUDA(cudaMemcpyAsync(aux_rand_out, r.aux_rand, TVM_NUM_AUX_COLUMNS * r.h * 3 * 8, cudaMemcpyDefault, c.stream));
  if (randomizer_column_out) TVM_CUDA(cudaMemcpyAsync(randomizer_column_out, r.randomizer_column, r.n * 3 * 8, cudaMemcpyDefault, c.stream));
  if (quot_rand_out) TVM_CUDA(cudaMemcpyAsync(quot_rand_out, r.quot_rand, r.nq * 3 * 8, cudaMemcpyDefault, c.stream));
  TVM_CUDA(cudaStreamSynchronize(c.stream));
  TVM_API_END
}

int tvm_prove_aet_seeded(tvm_ctx *ctx, const tvm_params *params, const tvm_claim *claim, uint64_t padded_height, const tvm_aet *aet,
                         const uint8_t seed[32], uint64_t *proof_out, size_t *proof_len) {
  if (!ctx || !params || !claim || !aet || !seed || !proof_len) return TVM_ERR_INVALID_ARG;
  if (params->ldt_choice > 2 || !claim_ok(claim)) return TVM_ERR_INVALID_ARG;
  TVM_API_BEGIN(ctx)
  ProveInputs in;
  in.aet = aet;
  run_prove(ctx, *params, claim_view(*claim), padded_height, in, seed, proof_out, proof_len);
  TVM_API_END
}

int tvm_prove_tables_seeded(tvm_ctx *ctx, const tvm_params *params, const tvm_claim *claim, uint64_t padded_height,
                            const uint64_t *main_table, int fill_derived_main_columns, const uint8_t seed[32], uint64_t *proof_out,
                            size_t *proof_len) {
  if (!ctx || !params || !claim || !main_table || !seed || !proof_len) return TVM_ERR_INVALID_ARG;
  if (params->ldt_choice > 2 || !claim_ok(claim)) return TVM_ERR_INVALID_ARG;
  TVM_API_BEGIN(ctx)
  ProveInputs in;
  in.main_trace = (const u64 *)main_table; in.fill_derived_main = fill_derived_main_columns != 0;
  run_prove(ctx, *params, claim_view(*claim), padded_height, in, seed, proof_out, proof_len);
  TVM_API_END
}

int tvm_trace_execution(const uint64_t *program, size_t program_len, const uint64_t *public_input, size_t num_input,
                        const tvm_nondeterminism *nd, tvm_execution **out, char *failure, size_t failure_capacity) {
  set_failure(failure, failure_capacity, "");
  if (!out) return TVM_ERR_INVALID_ARG;
  *out = nullptr;
  static const tvm_nondeterminism empty{};
  if (!nd) nd = &empty;
  if ((program_len && !program) || (num_input && !public_input) || (nd->num_individual_tokens && !nd->individual_tokens) ||
      (nd->num_digests && !nd->digests) || (nd->num_ram && (!nd->ram_addresses || !nd->ram_values)))
    return TVM_ERR_INVALID_ARG;
  auto canonical = [](const uint64_t *w, size_t n) {
    for (size_t i = 0; i < n; i++) if (w[i] >= P) return false;
    return true;
  };
  if (!canonical(program, program_len) || !canonical(public_input, num_input) ||
      !canonical(nd->individual_tokens, nd->num_individual_tokens) || !canonical(nd->digests, 5 * nd->num_digests) ||
      !canonical(nd->ram_addresses, nd->num_ram) || !canonical(nd->ram_values, nd->num_ram)) {
    set_failure(failure, failure_capacity, "a word is not a canonical field element (>= p)");
    return TVM_ERR_INVALID_ARG;
  }
  try {
    std::vector<uint64_t> addresses(nd->ram_addresses, nd->ram_addresses + nd->num_ram);
    std::sort(addresses.begin(), addresses.end());
    if (std::adjacent_find(addresses.begin(), addresses.end()) != addresses.end()) {
      set_failure(failure, failure_capacity, "a RAM address is given twice");
      return TVM_ERR_INVALID_ARG;
    }
    std::unique_ptr<tvm_execution> ex(new tvm_execution());
    std::string why;
    const VmInputs in{program, program_len, public_input, num_input, nd->individual_tokens, nd->num_individual_tokens,
                      nd->digests, nd->num_digests, nd->ram_addresses, nd->ram_values, nd->num_ram};
    if (int rc = trace_execution(in, *ex, why)) {
      set_failure(failure, failure_capacity, why.c_str());
      return rc;
    }
    *out = ex.release();
    return TVM_OK;
  } catch (const std::bad_alloc &) {
    set_failure(failure, failure_capacity, "host allocation failed");
    return TVM_ERR_OOM;
  }
}

int tvm_execution_info(const tvm_execution *ex, tvm_execution_summary *out, uint64_t *output) {
  if (!ex || !out) return TVM_ERR_INVALID_ARG;
  memcpy(out->program_digest, ex->digest, sizeof ex->digest);
  out->padded_height = ex->padded_height;
  memcpy(out->table_heights, ex->table_heights, sizeof ex->table_heights);
  out->num_output = ex->output.size();
  if (output && !ex->output.empty()) memcpy(output, ex->output.data(), ex->output.size() * 8);
  return TVM_OK;
}

// the execution's AET with host arrays; the three hash traces NULL
static tvm_aet execution_aet_host(const tvm_execution &ex) {
  tvm_aet a{};
  a.program = ex.program.data(); a.program_len = ex.program.size();
  a.instruction_multiplicities = ex.instruction_multiplicities.data();
  a.processor_trace = ex.processor_trace.data(); a.processor_rows = ex.processor_trace.size() / 39;
  a.op_stack_underflow_trace = ex.op_stack_trace.data(); a.op_stack_rows = ex.op_stack_trace.size() / 4;
  a.ram_trace = ex.ram_trace.data(); a.ram_rows = ex.ram_trace.size() / 7;
  a.program_hash_rows = ex.hash_rows[0]; a.sponge_rows = ex.hash_rows[1]; a.hash_rows = ex.hash_rows[2];
  a.u32_entries = ex.u32_entries.data(); a.u32_count = ex.u32_entries.size() / 4;
  a.cascade_table_lookup_multiplicities = ex.cascade_multiplicities.data(); a.cascade_count = ex.cascade_multiplicities.size() / 2;
  a.lookup_table_lookup_multiplicities = ex.lookup_multiplicities;
  return a;
}

// the execution's AET with the three hash traces expanded into device memory of `mem`
static tvm_aet execution_aet_device(Ctx &c, DevMem &mem, const tvm_execution &ex) {
  tvm_aet a = execution_aet_host(ex);
  u64 *d[3];
  hash_trace_run(c, mem, ex, d);
  a.program_hash_trace = d[0]; a.sponge_trace = d[1]; a.hash_trace = d[2];
  return a;
}

// the claim an execution proves (Claim::about_program(..).with_input(..).with_output(..))
static ClaimView execution_claim(const tvm_execution &ex) {
  return {ex.digest, TVM_CURRENT_VERSION, ex.input.data(), ex.input.size(), ex.output.data(), ex.output.size()};
}

int tvm_execution_aet(tvm_ctx *ctx, const tvm_execution *ex, tvm_aet *out) {
  if (!ex || !out) return TVM_ERR_INVALID_ARG;
  *out = execution_aet_host(*ex);
  if (!ctx) return TVM_OK;
  TVM_API_BEGIN(ctx)
  Ctx &c = *c__;
  if (!ex->expanded) {
    DevMem mem(c);
    const tvm_aet a = execution_aet_device(c, mem, *ex);
    const uint64_t *d[3] = {a.program_hash_trace, a.sponge_trace, a.hash_trace};
    for (int s = 0; s < 3; s++) {
      ex->hash_cache[s].resize(ex->hash_rows[s] * 67);
      if (ex->hash_rows[s])
        TVM_CUDA(cudaMemcpyAsync(ex->hash_cache[s].data(), d[s], ex->hash_cache[s].size() * 8, cudaMemcpyDeviceToHost, c.stream));
    }
    TVM_CUDA(cudaStreamSynchronize(c.stream));
    ex->expanded = true;
  }
  out->program_hash_trace = ex->hash_cache[0].data();
  out->sponge_trace = ex->hash_cache[1].data();
  out->hash_trace = ex->hash_cache[2].data();
  TVM_API_END
}

int tvm_prove_execution(tvm_ctx *ctx, const tvm_params *params, const tvm_execution *ex, const uint8_t seed[32], uint64_t *proof_out,
                        size_t *proof_len) {
  if (!ctx || !params || !ex || !seed || !proof_len || params->ldt_choice > 2) return TVM_ERR_INVALID_ARG;
  TVM_API_BEGIN(ctx)
  DevMem mem(*c__);   // the hash traces, allocated before the seeded randomness and live throughout the prove
  const tvm_aet a = execution_aet_device(*c__, mem, *ex);
  ProveInputs in;
  in.aet = &a;
  run_prove(ctx, *params, execution_claim(*ex), ex->padded_height, in, seed, proof_out, proof_len);
  TVM_API_END
}

void tvm_execution_destroy(tvm_execution *ex) { delete ex; }

int tvm_air_check(tvm_ctx *ctx, const uint64_t *main_table, const uint64_t *aux_table, unsigned log2_n, const uint64_t *challenges,
                  uint64_t *counts, uint64_t *first_rows, uint64_t *last_rows, uint64_t *num_violated) {
  if (!ctx || !main_table || !aux_table || !challenges || !counts || !first_rows || !last_rows || !num_violated) return TVM_ERR_INVALID_ARG;
  if (log2_n > 26) return TVM_ERR_DOMAIN;
  TVM_API_BEGIN(ctx)
  for (size_t i = 0; i < 3 * TVM_NUM_CHALLENGES; i++)
    if (challenges[i] >= P) throw ApiError{TVM_ERR_INVALID_ARG, "challenge word >= p at index " + std::to_string(i)};
  Ctx &c = *c__;
  const size_t n = (size_t)1 << log2_n;
  std::vector<u64> ch_mont(3 * TVM_NUM_CHALLENGES);
  for (size_t i = 0; i < ch_mont.size(); i++) ch_mont[i] = to_mont(challenges[i]);
  DevMem mem(c);
  u64 *d_main, *d_aux;
  air_check_upload(c, mem, (const u64 *)main_table, (const u64 *)aux_table, n, &d_main, &d_aux);
  air_check_run(c, mem, d_main, d_aux, n, ch_mont.data(), counts, first_rows, last_rows, num_violated);
  TVM_API_END
}

// the witness tvm_prove_aet builds (fill, padding, degree-lowering columns, Challenges::new, extend with a zero randomizer
// column), by the prover's own table stages, checked in place
static void air_check_witness(Ctx &c, DevMem &mem, const tvm_aet &aet, const ClaimView &cv, size_t n, const uint64_t *sampled,
                              uint64_t *counts, uint64_t *first_rows, uint64_t *last_rows, uint64_t *num_violated) {
  std::vector<xfe> ch;
  for (int i = 0; i < 59; i++) ch.push_back(xmake(to_mont(sampled[3 * i]), to_mont(sampled[3 * i + 1]), to_mont(sampled[3 * i + 2])));
  challenges_derive(cv, ch);
  std::vector<u64> ch_mont;
  for (xfe x : ch) { ch_mont.push_back(x.c0); ch_mont.push_back(x.c1); ch_mont.push_back(x.c2); }
  u64 *d_main = mem.words(TVM_NUM_MAIN_COLUMNS * n);
  main_table_on_device(c, d_main, n, aet);
  u64 *d_aux = mem.words(3 * TVM_NUM_AUX_COLUMNS * n);
  u64 *d_ch = mem.words(3 * TVM_NUM_CHALLENGES);
  TVM_CUDA(cudaMemcpyAsync(d_ch, ch_mont.data(), 3 * TVM_NUM_CHALLENGES * 8, cudaMemcpyHostToDevice, c.stream));
  aux_extend_on_device(c, mem, d_main, n, d_ch, nullptr, d_aux);
  mem.release(d_ch);
  air_check_run(c, mem, d_main, d_aux, n, ch_mont.data(), counts, first_rows, last_rows, num_violated);
}

static bool canonical_words(const uint64_t *w, size_t n) {
  for (size_t i = 0; i < n; i++) if (w[i] >= P) return false;
  return true;
}

int tvm_air_check_aet(tvm_ctx *ctx, const tvm_aet *aet, const tvm_claim *claim, uint64_t num_rows, const uint64_t *sampled_challenges,
                      uint64_t *counts, uint64_t *first_rows, uint64_t *last_rows, uint64_t *num_violated) {
  if (!ctx || !aet || !claim || !sampled_challenges || !counts || !first_rows || !last_rows || !num_violated) return TVM_ERR_INVALID_ARG;
  if (!claim_ok(claim) || !canonical_words(sampled_challenges, 3 * 59)) return TVM_ERR_INVALID_ARG;
  if (num_rows < 256 || (num_rows & (num_rows - 1)) || num_rows > ((uint64_t)1 << 26)) return TVM_ERR_DOMAIN;
  TVM_API_BEGIN(ctx)
  DevMem mem(*c__);
  air_check_witness(*c__, mem, *aet, claim_view(*claim), (size_t)num_rows, sampled_challenges, counts, first_rows, last_rows, num_violated);
  TVM_API_END
}

int tvm_air_check_execution(tvm_ctx *ctx, const tvm_execution *ex, const uint64_t *sampled_challenges, uint64_t *counts,
                            uint64_t *first_rows, uint64_t *last_rows, uint64_t *num_violated) {
  if (!ctx || !ex || !sampled_challenges || !counts || !first_rows || !last_rows || !num_violated) return TVM_ERR_INVALID_ARG;
  if (!canonical_words(sampled_challenges, 3 * 59)) return TVM_ERR_INVALID_ARG;
  TVM_API_BEGIN(ctx)
  DevMem mem(*c__);
  const tvm_aet a = execution_aet_device(*c__, mem, *ex);
  air_check_witness(*c__, mem, a, execution_claim(*ex), ex->padded_height, sampled_challenges, counts, first_rows, last_rows, num_violated);
  TVM_API_END
}

int tvm_bezout_coefficients(tvm_ctx *ctx, const uint64_t *roots, uint64_t m, uint64_t *a_out, uint64_t *b_out) {
  if (!ctx || (m && (!roots || !a_out || !b_out))) return TVM_ERR_INVALID_ARG;
  if (m > ((uint64_t)1 << 24)) return TVM_ERR_DOMAIN;
  if (!m) return TVM_OK;
  TVM_API_BEGIN(ctx)
  Ctx &c = *c__;
  DevMem mem(c);
  u64 *d_r = mem.words(m), *d_a = mem.words(m), *d_b = mem.words(m);
  TVM_CUDA(cudaMemcpyAsync(d_r, roots, m * 8, cudaMemcpyDefault, c.stream));
  to_mont_run(c, d_r, m);
  try {
    bezout_run(c, mem, d_r, (size_t)m, d_a, d_b);
  } catch (const std::runtime_error &e) {
    throw ApiError{TVM_ERR_UNSUPPORTED, e.what()};
  }
  from_mont_run(c, d_a, m);
  from_mont_run(c, d_b, m);
  TVM_CUDA(cudaMemcpyAsync(a_out, d_a, m * 8, cudaMemcpyDefault, c.stream));
  TVM_CUDA(cudaMemcpyAsync(b_out, d_b, m * 8, cudaMemcpyDefault, c.stream));
  TVM_CUDA(cudaStreamSynchronize(c.stream));
  TVM_API_END
}

int tvm_stir_derive(uint32_t security_level, uint32_t soundness, uint32_t log2_folding_factor, uint32_t log2_initial_expansion_factor,
                    uint32_t log2_high_degree_bound, tvm_stir_info *out) {
  if (!out || soundness > 1) return TVM_ERR_INVALID_ARG;
  StirDerived sd{};
  if (int rc = stir_derive(security_level, log2_folding_factor, log2_initial_expansion_factor, log2_high_degree_bound, soundness == 1, sd))
    return rc;
  *out = tvm_stir_info{};
  out->domain_len = (uint64_t)1 << (log2_high_degree_bound + log2_initial_expansion_factor);
  out->domain_offset = 7;                                   // BFieldElement::generator(), stir.rs:589
  out->folding_factor = sd.folding_factor;
  out->num_rounds = (uint64_t)sd.num_rounds;
  for (int i = 0; i < sd.num_rounds; i++) {
    out->in_domain_queries[i] = sd.in_domain[i];
    out->out_of_domain_queries[i] = sd.out_of_domain[i];
  }
  out->final_num_queries = sd.final_num_in_domain_queries;
  out->final_degree = sd.final_degree;
  return TVM_OK;
}

int tvm_stir_prove_k(tvm_ctx *ctx, uint32_t security_level, uint32_t soundness, uint32_t log2_folding_factor,
                     uint32_t log2_initial_expansion_factor, uint32_t log2_high_degree_bound, const uint64_t *codeword, uint64_t *proof_out,
                     size_t *proof_len, uint32_t *indices_out, size_t *num_indices) {
  if (!ctx || !codeword || !proof_len || soundness > 1) return TVM_ERR_INVALID_ARG;
  TVM_API_BEGIN(ctx)
  Ctx &c = *c__;
  StirDerived sd{};
  const char *why = "";
  if (int rc = stir_derive(security_level, log2_folding_factor, log2_initial_expansion_factor, log2_high_degree_bound, soundness == 1, sd,
                           &why))
    throw ApiError{rc, why};
  if (log2_high_degree_bound + log2_initial_expansion_factor > 26)
    throw ApiError{TVM_ERR_DOMAIN, "STIR: the device prover supports initial domains of up to 2^26 points"};
  const size_t len = (size_t)1 << (log2_high_degree_bound + log2_initial_expansion_factor);
  std::vector<u64> proof;
  std::vector<uint32_t> revealed;
  {
    DevMem mem(c);
    u64 *d_in = mem.words(3 * len), *d_cw = mem.words(3 * len), *d_tmp = mem.words(3 * len);
    TVM_CUDA(cudaMemcpyAsync(d_in, codeword, 3 * len * 8, cudaMemcpyDefault, c.stream));
    to_mont_run(c, d_in, 3 * len);
    deinterleave3_run(c, d_in, d_cw, len, 1);
    ProofStream ps;
    revealed = stir_prove_run(c, mem, ps, d_cw, len, to_mont(7), sd, d_tmp);
    proof = ps.encode();
  }
  copy_indices_out(revealed, indices_out, num_indices);
  copy_proof_out(proof, proof_out, proof_len);
  TVM_API_END
}

int tvm_stir_prove(tvm_ctx *ctx, uint32_t security_level, uint32_t soundness, uint32_t log2_initial_expansion_factor,
                   uint32_t log2_high_degree_bound, const uint64_t *codeword, uint64_t *proof_out, size_t *proof_len,
                   uint32_t *indices_out, size_t *num_indices) {
  if (!ctx || !codeword || !proof_len || soundness > 1) return TVM_ERR_INVALID_ARG;
  if (log2_high_degree_bound + log2_initial_expansion_factor > 26) return TVM_ERR_DOMAIN;
  return tvm_stir_prove_k(ctx, security_level, soundness, STIR_LOG2_FOLDING_FACTOR, log2_initial_expansion_factor, log2_high_degree_bound,
                          codeword, proof_out, proof_len, indices_out, num_indices);
}

int tvm_fri_derive(uint32_t security_level, uint32_t soundness, uint32_t log2_initial_expansion_factor, uint32_t log2_high_degree_bound,
                   tvm_fri_info *out) {
  if (!out || soundness > 1) return TVM_ERR_INVALID_ARG;
  FriDerived fd{};
  if (int rc = fri_derive(security_level, soundness == 1, log2_initial_expansion_factor, log2_high_degree_bound, fd)) return rc;
  out->domain_len = fd.domain_len; out->domain_offset = fd.domain_offset; out->expansion_factor = fd.expansion_factor;
  out->max_degree = fd.max_degree; out->num_collinearity_checks = fd.num_collinearity_checks; out->num_rounds = fd.num_rounds;
  out->last_round_max_degree = fd.last_round_max_degree;
  return TVM_OK;
}

int tvm_fri_prove(tvm_ctx *ctx, uint32_t security_level, uint32_t soundness, uint32_t log2_initial_expansion_factor,
                  uint32_t log2_high_degree_bound, const uint64_t *codeword, size_t codeword_len, uint64_t *proof_out, size_t *proof_len,
                  uint32_t *indices_out, size_t *num_indices) {
  if (!ctx || !codeword || !proof_len || soundness > 1) return TVM_ERR_INVALID_ARG;
  TVM_API_BEGIN(ctx)
  Ctx &c = *c__;
  FriDerived fd{};
  const char *why = "";
  if (int rc = fri_derive(security_level, soundness == 1, log2_initial_expansion_factor, log2_high_degree_bound, fd, &why))
    throw ApiError{rc, why};
  if (log2_high_degree_bound + log2_initial_expansion_factor > 26)
    throw ApiError{TVM_ERR_DOMAIN, "FRI: the device prover supports initial domains of up to 2^26 points"};
  const size_t len = fd.domain_len;
  if (codeword_len != len)   // LdtProvingError, fri.rs:323-330
    throw ApiError{TVM_ERR_INVALID_ARG, "InitialCodewordMismatch { domain_len: " + std::to_string(len) + ", codeword_len: " +
                                            std::to_string(codeword_len) + " }"};
  std::vector<u64> proof;
  std::vector<uint32_t> revealed;
  {
    DevMem mem(c);
    u64 *d_in = mem.words(3 * len), *d_cw = mem.words(3 * len);
    TVM_CUDA(cudaMemcpyAsync(d_in, codeword, 3 * len * 8, cudaMemcpyDefault, c.stream));
    to_mont_run(c, d_in, 3 * len);
    deinterleave3_run(c, d_in, d_cw, len, 1);
    ProofStream ps;
    revealed = fri_prove_run(c, mem, ps, d_cw, len, to_mont(fd.domain_offset), fd, d_in /* free again: scratch */);
    proof = ps.encode();
  }
  copy_indices_out(revealed, indices_out, num_indices);
  copy_proof_out(proof, proof_out, proof_len);
  TVM_API_END
}

int tvm_last_prove_timings(const tvm_ctx *ctx, const char **names, float *ms) {
  if (!ctx) return 0;
  int n = 0;
  for (auto &st : ctx->timings.stages) {
    if (n >= 20) break;
    if (names) names[n] = st.first.c_str();
    if (ms) ms[n] = st.second;
    n++;
  }
  return n;
}

}  // extern "C"
