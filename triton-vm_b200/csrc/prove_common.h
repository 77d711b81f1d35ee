// Host-side helpers shared by the prover's translation units (prover.cu, stir.cu).
#pragma once
#include <set>
#include <vector>
#include "launch.h"
#include "stark.h"

namespace tvm {

struct DevMem {   // RAII device buffers of one prove() call, recycled through the context's block pool
  Ctx &c;
  std::vector<void *> ptrs;
  explicit DevMem(Ctx &ctx) : c(ctx) {}
  ~DevMem() {
    cudaStreamSynchronize(c.stream);
    for (void *p : ptrs) c.pool_release(p);
  }
  u64 *words(size_t n) {
    void *p = c.pool_alloc((n ? n : 1) * sizeof(u64));
    ptrs.push_back(p);
    return (u64 *)p;
  }
  void release(void *p) {   // stream-ordered reuse: later kernels on the same stream see earlier ones complete
    for (size_t i = 0; i < ptrs.size(); i++)
      if (ptrs[i] == p) { c.pool_release(p); ptrs.erase(ptrs.begin() + i); return; }
  }
};

inline xfe xmul_by_X(xfe a) { return xmake(fneg(a.c2), fadd(a.c0, a.c2), a.c1); }   // X^3 = X - 1
// value of an X-field column stored as 3 planar B-field columns from the 3 per-plane dot products
inline xfe combine_planes(xfe r0, xfe r1, xfe r2) { return xadd(r0, xadd(xmul_by_X(r1), xmul_by_X(xmul_by_X(r2)))); }

inline std::vector<unsigned> auth_structure_node_indices(size_t num_leafs, const std::vector<uint32_t> &leaf_indices) {
  // twenty-first MerkleTree::authentication_structure (SURVEY.md A.4): needed-but-not-computable
  // sibling nodes, descending node index
  std::set<size_t> needed, computable;
  for (uint32_t li : leaf_indices) {
    size_t node = (size_t)li + num_leafs;
    while (node > 1) {
      computable.insert(node);
      needed.insert(node ^ 1);
      node >>= 1;
    }
  }
  std::vector<unsigned> out;
  for (auto it = needed.rbegin(); it != needed.rend(); ++it)
    if (!computable.count(*it)) out.push_back((unsigned)*it);
  return out;
}

inline std::vector<u64> d2h(Ctx &c, const u64 *d, size_t n) {
  std::vector<u64> h(n);
  TVM_CUDA(cudaMemcpyAsync(h.data(), d, n * sizeof(u64), cudaMemcpyDeviceToHost, c.stream));
  TVM_CUDA(cudaStreamSynchronize(c.stream));
  return h;
}

struct ProofStream;
// STIR prover (stir.rs:885-993) on a device-resident codeword [3 planes][len] in natural order; enqueues into
// `ps` and returns the revealed first-round indices.
std::vector<uint32_t> stir_prove_run(Ctx &c, DevMem &mem, ProofStream &ps, const u64 *d_codeword, size_t len, u64 offset_mont,
                                     const StirDerived &sd, u64 *d_tmp /* >= 3*len words */);
// FRI prover (fri.rs:212-366, 754-772) on a device-resident codeword [3 planes][len] in natural order, Montgomery form, on the
// domain offset_mont * <g_len>; enqueues into `ps` and returns the first-round collinearity-check indices.
std::vector<uint32_t> fri_prove_run(Ctx &c, DevMem &mem, ProofStream &ps, const u64 *d_codeword, size_t len, u64 offset_mont,
                                    const FriDerived &fd, u64 *d_tmp /* >= 3*len words */);

}  // namespace tvm
