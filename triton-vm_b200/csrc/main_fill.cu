// MasterMainTable::new + pad on the device (SURVEY.md 8(f).4; reference triton-vm/src/table/master_table.rs:881-974):
// the CUDA executor of fill/main_fill.cuh — one generic grid-stride kernel per stage body, cub's radix sort and scan for
// the memory-like tables and the u32 sections, the batched NTT of ntt.cu for the polynomial passes of the RAM table's
// Bezout coefficients — plus the upload of the AlgebraicExecutionTrace.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include "ctx.h"
#include "launch.h"
#include "prove_common.h"
#include "stark.h"
#include "tip5.cuh"
#include "fill/main_fill.cuh"
#include "fill/hash_trace.cuh"
#include "vm.h"

namespace tvm {

template <class F>
__global__ void __launch_bounds__(256) fill_stage_kernel(size_t count, F body) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < count; i += (size_t)gridDim.x * blockDim.x) body(i);
}

namespace fill_cuda {

struct CudaExec {
  Ctx &c;
  DevMem &mem;
  u64 *alloc(size_t words) { return mem.words(words); }
  template <class F>
  void launch(size_t count, F body) {
    if (!count) return;
    const size_t blocks = (count + 255) / 256, cap = (size_t)c.num_sms * 32;
    fill_stage_kernel<<<(unsigned)(blocks < cap ? blocks : cap), 256, 0, c.stream>>>(count, body);
    c.launches++;
    TVM_CUDA(cudaGetLastError());
  }
  void sort_perm(const u64 *keys, u64 *perm, size_t n) {
    u64 *keys_out = mem.words(n), *iota = mem.words(n);
    launch(n, TVM_FILL_BODY(size_t i) { iota[i] = i; });
    size_t bytes = 0;
    TVM_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, bytes, keys, keys_out, iota, perm, n, 0, 64, c.stream));
    void *tmp = mem.words(bytes / 8 + 1);
    TVM_CUDA(cub::DeviceRadixSort::SortPairs(tmp, bytes, keys, keys_out, iota, perm, n, 0, 64, c.stream));   // LSD radix sort: stable
    c.launches += 8;
    mem.release(tmp); mem.release(iota); mem.release(keys_out);
  }
  void exclusive_sum(const u64 *in, u64 *out, size_t n) {
    size_t bytes = 0;
    TVM_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, bytes, in, out, n, c.stream));
    void *tmp = mem.words(bytes / 8 + 1);
    TVM_CUDA(cub::DeviceScan::ExclusiveSum(tmp, bytes, in, out, n, c.stream));
    c.launches += 2;
    mem.release(tmp);
  }
  void ntt(const u64 *in, u64 *out, unsigned lg, size_t count, bool inverse) {
    const size_t n = (size_t)1 << lg;
    NttJob j{};
    j.in = in; j.in_cstride = n; j.out = out; j.out_cstride = n;
    j.log_n = (int)lg; j.ncols = count; j.inverse = inverse;
    u64 *tmp = nullptr;
    if (lg > 13) j.tmp = tmp = mem.words(count * n);
    ntt_run(c, j);
    if (tmp) mem.release(tmp);
  }
  u64 read_word(const u64 *p) {
    u64 v = 0;
    TVM_CUDA(cudaMemcpyAsync(&v, p, 8, cudaMemcpyDeviceToHost, c.stream));
    TVM_CUDA(cudaStreamSynchronize(c.stream));
    return v;
  }
};

u64 *upload(Ctx &c, DevMem &mem, const u64 *host, size_t words) {
  u64 *d = mem.words(words);
  if (words) TVM_CUDA(cudaMemcpyAsync(d, host, words * 8, cudaMemcpyDefault, c.stream));
  return d;
}

}  // namespace fill_cuda
using fill_cuda::CudaExec;
using fill_cuda::upload;

// d_table: [>= 149][n] words, column stride n; receives the nine tables' columns in CANONICAL form.
void main_fill_run(Ctx &c, DevMem &mem, const tvm_aet &a, size_t n, u64 *d_table, uint64_t *lengths9) {
  if (!a.processor_trace || !a.processor_rows || (a.program_len && (!a.program || !a.instruction_multiplicities)) ||
      (a.op_stack_rows && !a.op_stack_underflow_trace) || (a.ram_rows && !a.ram_trace) || (a.program_hash_rows && !a.program_hash_trace) ||
      (a.sponge_rows && !a.sponge_trace) || (a.hash_rows && !a.hash_trace) || (a.u32_count && !a.u32_entries) ||
      (a.cascade_count && !a.cascade_table_lookup_multiplicities) || !a.lookup_table_lookup_multiplicities)
    throw ApiError{TVM_ERR_INVALID_ARG, "tvm_aet: a trace with rows has no data"};
  u64 rc0[16];
  for (int k = 0; k < 16; k++) rc0[k] = from_mont(TIP5_ROUND_CONSTANTS_HOST[k]);
  const std::vector<u64> consts = fill::fill_constants(rc0, TIP5_LOOKUP_HOST);
  std::vector<u64> mult(a.program_len);
  for (size_t i = 0; i < a.program_len; i++) mult[i] = a.instruction_multiplicities[i];
  fill::AetView v{};
  v.program = upload(c, mem, a.program, a.program_len); v.program_len = a.program_len;
  v.instruction_multiplicities = upload(c, mem, mult.data(), mult.size());
  v.processor_trace = upload(c, mem, a.processor_trace, a.processor_rows * fill::W_PROCESSOR); v.processor_rows = a.processor_rows;
  v.op_stack_trace = upload(c, mem, a.op_stack_underflow_trace, a.op_stack_rows * fill::W_OP_STACK); v.op_stack_rows = a.op_stack_rows;
  v.ram_trace = upload(c, mem, a.ram_trace, a.ram_rows * fill::W_RAM); v.ram_rows = a.ram_rows;
  v.program_hash_trace = upload(c, mem, a.program_hash_trace, a.program_hash_rows * fill::W_HASH); v.program_hash_rows = a.program_hash_rows;
  v.sponge_trace = upload(c, mem, a.sponge_trace, a.sponge_rows * fill::W_HASH); v.sponge_rows = a.sponge_rows;
  v.hash_trace = upload(c, mem, a.hash_trace, a.hash_rows * fill::W_HASH); v.hash_rows = a.hash_rows;
  v.u32_entries = upload(c, mem, a.u32_entries, a.u32_count * 4); v.u32_count = a.u32_count;
  v.cascade_multiplicities = upload(c, mem, a.cascade_table_lookup_multiplicities, a.cascade_count * 2); v.cascade_count = a.cascade_count;
  v.lookup_multiplicities = upload(c, mem, a.lookup_table_lookup_multiplicities, 256);
  const u64 *d_consts = upload(c, mem, consts.data(), consts.size());
  TVM_CUDA(cudaStreamSynchronize(c.stream));   // `mult` and `consts` are pageable host vectors of this frame
  CudaExec ex{c, mem};
  fill::FillInfo info;
  try {
    info = fill::main_table_from_aet(ex, v, d_consts, n, d_table);
  } catch (const std::invalid_argument &e) {
    throw ApiError{TVM_ERR_INVALID_ARG, e.what()};
  } catch (const std::runtime_error &e) {
    throw ApiError{TVM_ERR_UNSUPPORTED, e.what()};
  }
  if (lengths9) {
    const uint64_t l[9] = {info.program_len_padded, info.processor_len, info.op_stack_len, info.ram_len, info.processor_len,
                           info.hash_len, info.cascade_len, 256, info.u32_len};
    for (int i = 0; i < 9; i++) lengths9[i] = l[i];
  }
}

void main_table_on_device(Ctx &c, u64 *d_main, size_t n, const tvm_aet &aet, uint64_t *lengths9) {
  {
    DevMem fill_mem(c);   // the AET's device copy and the fill's scratch go back to the pool right after
    main_fill_run(c, fill_mem, aet, n, d_main, lengths9);
  }
  to_mont_run(c, d_main, (size_t)TVM_NUM_MAIN_TABLE_COLUMNS * n);
  main_derived_run(c, d_main, n);
}

void bezout_run(Ctx &c, DevMem &mem, const u64 *d_roots_mont, size_t m, u64 *d_a, u64 *d_b) {
  CudaExec ex{c, mem};
  fill::bezout_coefficients(ex, d_roots_mont, m, d_a, d_b);
}

void hash_trace_run(Ctx &c, DevMem &mem, const tvm_execution &e, u64 *d_out[3]) {
  const size_t count = e.perm_meta.size();
  const std::vector<u64> k = hash_trace::constants(TIP5_ROUND_CONSTANTS_HOST, TIP5_LOOKUP_HOST);
  const u64 *d_states = upload(c, mem, e.perm_states.data(), 16 * count), *d_meta = upload(c, mem, e.perm_meta.data(), count);
  const u64 *d_k = upload(c, mem, k.data(), k.size());
  for (int s = 0; s < 3; s++) d_out[s] = mem.words(e.hash_rows[s] * hash_trace::H_WIDTH);
  CudaExec ex{c, mem};
  hash_trace::expand(ex, d_states, d_meta, count, d_k, d_out[0], d_out[1], d_out[2]);
  TVM_CUDA(cudaStreamSynchronize(c.stream));   // `k` is a pageable host vector of this frame
}

}  // namespace tvm
