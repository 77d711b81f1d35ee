// The prover's randomness on the device (reference stark.rs:192, 293-328; master_table.rs:423-434, 630-662, 1006-1025):
// the CUDA executor of rand/prover_randomness.cuh — one generic grid-stride kernel per stage body.
#include "ctx.h"
#include "launch.h"
#include "prove_common.h"
#include "stark.h"
#include "rand/prover_randomness.cuh"

namespace tvm {

template <class F>
__global__ void __launch_bounds__(256) rand_stage_kernel(size_t count, F body) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < count; i += (size_t)gridDim.x * blockDim.x) body(i);
}

namespace {

struct RandExec {
  Ctx &c;
  DevMem &mem;
  u64 *alloc(size_t words) { return mem.words(words); }
  template <class F>
  void launch(size_t count, F body) {
    if (!count) return;
    const size_t blocks = (count + 255) / 256, cap = (size_t)c.num_sms * 16;
    rand_stage_kernel<<<(unsigned)(blocks < cap ? blocks : cap), 256, 0, c.stream>>>(count, body);
    c.launches++;
    TVM_CUDA(cudaGetLastError());
  }
  u64 read_word(const u64 *p) {
    u64 v = 0;
    TVM_CUDA(cudaMemcpyAsync(&v, p, 8, cudaMemcpyDeviceToHost, c.stream));
    TVM_CUDA(cudaStreamSynchronize(c.stream));
    return v;
  }
};

}  // namespace

ProverRandomnessLayout prover_randomness_layout(size_t n, size_t h, size_t nq) {
  const prand::Layout L = prand::prover_layout(n, h, nq);
  ProverRandomnessLayout r;
  r.main = L.g[0].out0; r.aux = L.g[1].out0; r.randomizer_column = L.g[2].out0; r.quot = L.g[3].out0; r.total = L.total_out;
  return r;
}

void prover_randomness_run(Ctx &c, const uint8_t seed[32], size_t n, size_t h, size_t nq, u64 *d_out) {
  prand::Seed s;
  for (int i = 0; i < 8; i++)
    s.w[i] = (uint32_t)seed[4 * i] | ((uint32_t)seed[4 * i + 1] << 8) | ((uint32_t)seed[4 * i + 2] << 16) | ((uint32_t)seed[4 * i + 3] << 24);
  DevMem scratch(c);   // keystream and flag tables go back to the pool as soon as the samples are written
  RandExec ex{c, scratch};
  prand::generate(ex, prand::prover_layout(n, h, nq), s, d_out);
}

}  // namespace tvm
