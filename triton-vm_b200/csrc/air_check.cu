// The AIR constraint checker: every constraint of the degree-lowered AIR on the trace rows where it must vanish, with the
// reference's row rules (check_constraints_fn!, triton-vm/src/stark.rs:2899-3015; zerofiers master_table.rs:1194-1252).
// The chunk kernels are generated (airgen/codegen_check.py -> air_check_gen/); this file holds the upload, the launch order
// and the constraint metadata.
#include <cstring>
#include <string>
#include "air_check.cuh"
#include "launch.h"
#include "prove_common.h"
#include "stark.h"

namespace tvm {
#include "air_gen/air_meta.inc"

#define TVM_AIR_CHECK_TU(tu) void tu##_launch(const AirCheckArgs args[4], const u64 *d_challenges, cudaStream_t s, unsigned long long *launches);
#define TVM_AIR_CHECK_CHUNK(body, cat, first, count)
#define TVM_AIR_CHECK_ORIGINS
#include "air_check_gen/air_check_meta.inc"
#undef TVM_AIR_CHECK_TU

namespace {

static constexpr int NUM_CHECKED_AUX = TVM_NUM_AUX_COLUMNS - 1;   // column 90, the randomizer, is read by no constraint

// canonical -> Montgomery, column-major [379][n]; `bad` keeps the smallest index of a word >= p
__global__ void check_main_in_kernel(const u64 *in, u64 *out, size_t total, unsigned long long *bad) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    u64 v = in[i];
    if (v >= P) {
      atomicMin(bad, (unsigned long long)i);
      v = 0;
    }
    out[i] = to_mont(v);
  }
}

// canonical [91][n][3] -> Montgomery planes [270][n] (coordinate d of column q at plane 3q + d); every word is validated
__global__ void check_aux_in_kernel(const u64 *in, u64 *out, size_t n, unsigned long long *bad) {
  const size_t total = (size_t)TVM_NUM_AUX_COLUMNS * 3 * n;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    u64 v = in[i];
    if (v >= P) {
      atomicMin(bad, (unsigned long long)i);
      v = 0;
    }
    const size_t q = i / (3 * n), rest = i - q * 3 * n, row = rest / 3, d = rest - 3 * row;
    if (q < (size_t)NUM_CHECKED_AUX) out[(3 * q + d) * n + row] = to_mont(v);
  }
}

unsigned grid_for(const Ctx &c, size_t total) {
  const size_t want = (total + 255) / 256, cap = (size_t)c.num_sms * 64;
  return (unsigned)std::max<size_t>(1, std::min(want, cap));
}

// a table already in this device's memory is read in place; anything else is copied first (cudaMemcpyDefault)
const u64 *device_view(Ctx &c, DevMem &mem, const u64 *p, size_t words) {
  cudaPointerAttributes at{};
  if (cudaPointerGetAttributes(&at, p) == cudaSuccess && at.type == cudaMemoryTypeDevice && at.device == c.device) return p;
  cudaGetLastError();
  u64 *d = mem.words(words);
  TVM_CUDA(cudaMemcpyAsync(d, p, words * 8, cudaMemcpyDefault, c.stream));
  return d;
}

}  // namespace

void air_check_upload(Ctx &c, DevMem &mem, const u64 *main, const u64 *aux, size_t n, u64 **d_main, u64 **d_aux) {
  const size_t NM = TVM_NUM_MAIN_COLUMNS, NA = TVM_NUM_AUX_COLUMNS;
  u64 *d_bad = mem.words(2);
  TVM_CUDA(cudaMemsetAsync(d_bad, 0xff, 16, c.stream));
  *d_main = mem.words(NM * n);
  *d_aux = mem.words(3 * NUM_CHECKED_AUX * n);
  const u64 *src_main = device_view(c, mem, main, NM * n);
  check_main_in_kernel<<<grid_for(c, NM * n), 256, 0, c.stream>>>(src_main, *d_main, NM * n, (unsigned long long *)d_bad);
  c.launches++;
  TVM_CUDA(cudaGetLastError());
  if (src_main != main) mem.release((void *)src_main);
  const u64 *src_aux = device_view(c, mem, aux, 3 * NA * n);
  check_aux_in_kernel<<<grid_for(c, 3 * NA * n), 256, 0, c.stream>>>(src_aux, *d_aux, n, (unsigned long long *)d_bad + 1);
  c.launches++;
  TVM_CUDA(cudaGetLastError());
  if (src_aux != aux) mem.release((void *)src_aux);
  const std::vector<u64> bad = d2h(c, d_bad, 2);
  if (bad[0] != UINT64_MAX)
    throw ApiError{TVM_ERR_INVALID_ARG, "main table: word >= p at column " + std::to_string(bad[0] / n) + ", row " + std::to_string(bad[0] % n)};
  if (bad[1] != UINT64_MAX) {
    const u64 q = bad[1] / (3 * n), row = (bad[1] % (3 * n)) / 3, d = bad[1] % 3;
    throw ApiError{TVM_ERR_INVALID_ARG, "aux table: word >= p at column " + std::to_string(q) + ", row " + std::to_string(row) + ", coordinate " +
                                            std::to_string(d)};
  }
}

void air_check_run(Ctx &c, DevMem &mem, const u64 *d_main, const u64 *d_aux, size_t n, const u64 *ch_mont, uint64_t *counts,
                   uint64_t *first, uint64_t *last, uint64_t *num_violated) {
  const size_t NC = TVM_NUM_CONSTRAINTS, nch = 3 * TVM_NUM_CHALLENGES;
  // one upload: the challenges and the initial results (count 0, first row UINT64_MAX, last row 0)
  std::vector<u64> h(nch + 3 * NC, 0);
  memcpy(h.data(), ch_mont, nch * 8);
  for (size_t j = 0; j < NC; j++) h[nch + 3 * j + 1] = UINT64_MAX;
  u64 *d = mem.words(h.size());
  TVM_CUDA(cudaMemcpyAsync(d, h.data(), h.size() * 8, cudaMemcpyHostToDevice, c.stream));
  unsigned long long *d_out = (unsigned long long *)(d + nch);
  AirCheckArgs args[4];
  for (int k = 0; k < 4; k++) args[k] = AirCheckArgs{d_main, n, d_aux, n, 0, 0, d_out};
  args[0].nrows = 1;                                      // init: row 0
  args[1].nrows = n;                                      // cons: every row
  args[2].nrows = n - 1;                                  // tran: (i, i+1) for i < n - 1
  args[3].first_row = n - 1; args[3].nrows = 1;           // term: row n - 1
#define TVM_AIR_CHECK_TU(tu) tu##_launch(args, d, c.stream, &c.launches);
#include "air_check_gen/air_check_meta.inc"
#undef TVM_AIR_CHECK_TU
  TVM_CUDA(cudaGetLastError());
  const std::vector<u64> out = d2h(c, d + nch, 3 * NC);   // synchronises: `h` may go
  uint64_t violated = 0;
  for (size_t j = 0; j < NC; j++) {
    counts[j] = out[3 * j];
    first[j] = out[3 * j] ? out[3 * j + 1] : UINT64_MAX;
    last[j] = out[3 * j] ? out[3 * j + 2] : UINT64_MAX;
    violated += out[3 * j] != 0;
  }
  *num_violated = violated;
}

}  // namespace tvm

#ifndef __CUDA_ARCH__   // host code: the origin table exists in the host compilation only
extern "C" int tvm_air_constraint_info(unsigned index, tvm_air_constraint *out) {
  using namespace tvm;
  if (!out || index >= TVM_NUM_CONSTRAINTS) return TVM_ERR_INVALID_ARG;
  const unsigned *o = AIR_CHECK_ORIGIN[index];
  static const unsigned char *const DEGREES[4] = {AIR_DEGREES_INIT, AIR_DEGREES_CONS, AIR_DEGREES_TRAN, AIR_DEGREES_TERM};
  out->category = o[0];
  out->index_in_category = o[1];
  out->degree = DEGREES[o[0]][o[1]];
  out->origin = o[2];
  out->origin_index = o[3];
  out->derived_column = o[2] != AIR_CHECK_ORIGIN_DEGREE_LOWERING ? TVM_AIR_DERIVED_NONE
                        : o[3] >= TVM_NUM_MAIN_TABLE_COLUMNS   ? TVM_AIR_DERIVED_MAIN
                                                               : TVM_AIR_DERIVED_AUX;
  out->origin_name = AIR_CHECK_ORIGIN_NAME[o[2]];
  return TVM_OK;
}
#endif
