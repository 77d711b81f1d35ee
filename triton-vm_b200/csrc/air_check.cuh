// The AIR constraint checker's shared declarations: the generated chunk bodies (csrc/air_check_gen/air_check_bodies.cuh),
// the recorders they report to, and the kernels' row mapping.  Included by the library (air_check.cu and the generated
// translation units) and by the sequential host harness tests/host/air_check_host.cu.
//
// Semantics: check_constraints_fn! (triton-vm/src/stark.rs:2899-3015) on the degree-lowered AIR: init on row 0, cons on every
// row, tran on the pairs (i, i+1) for i < n - 1 (no wrap-around), term on row n - 1.  Per constraint the result is the number
// of rows where its value is non-zero and the first and last such row.
#pragma once
#include "field.cuh"

namespace tvm {

#ifndef TVM_AIR_CHECK_THREADS
#define TVM_AIR_CHECK_THREADS 256
#endif
static constexpr int AIR_CHECK_THREADS = TVM_AIR_CHECK_THREADS;

// what the generated bodies call the strides (a.main_stride, a.aux_stride, as the quotient's bodies do)
struct AirCheckStrides {
  size_t main_stride, aux_stride;
};

// the rows one category's kernels check: row first_row + t for t < nrows, the next row is row + 1
struct AirCheckArgs {
  const u64 *main;      // main column q at main + q*main_stride, Montgomery
  size_t main_stride;
  const u64 *aux;       // aux X-field column q, coordinate d at aux + (3q+d)*aux_stride, Montgomery
  size_t aux_stride;
  size_t first_row, nrows;
  unsigned long long *out;   // [604][3]: count, first row, last row
};

#ifdef __CUDACC__
struct AirCheckRow {
  size_t row, next, warp_base;
  bool active;
};
// Every lane of a warp stays alive (the recorder's ballots are warp-wide): a lane past the last row evaluates the first row
// again and records nothing.
__device__ __forceinline__ AirCheckRow air_check_row(const AirCheckArgs &a) {
  const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  AirCheckRow r;
  r.active = t < a.nrows;
  r.warp_base = a.first_row + (t & ~(size_t)31);
  r.row = a.first_row + (r.active ? t : 0);
  r.next = r.row + 1;   // read by the transition bodies only, whose rows stop at n - 2
  return r;
}
static inline unsigned air_check_grid(const AirCheckArgs &a) { return (unsigned)((a.nrows + AIR_CHECK_THREADS - 1) / AIR_CHECK_THREADS); }

// Warp-aggregated recording: one ballot per constraint; if any lane's row violates it, the lowest such lane adds the
// warp's count and folds the warp's first and last violating row into the constraint's minimum and maximum.  Counts,
// minima and maxima are order-independent, so the result does not depend on the launch order.
struct AirCheckDeviceRecorder {
  unsigned long long *out;
  size_t warp_base;
  bool active;
  __device__ __forceinline__ void operator()(int j, bool nonzero) {
    const unsigned m = __ballot_sync(0xffffffffu, nonzero && active);
    if (m && (threadIdx.x & 31) == (unsigned)(__ffs(m) - 1)) {
      atomicAdd(out + 3 * j, (unsigned long long)__popc(m));
      atomicMin(out + 3 * j + 1, (unsigned long long)(warp_base + __ffs(m) - 1));
      atomicMax(out + 3 * j + 2, (unsigned long long)(warp_base + 31 - __clz(m)));
    }
  }
};
#endif

// the sequential recorder (host harness): one row at a time
struct AirCheckHostRecorder {
  uint64_t *count, *first, *last;
  uint64_t row;
  __host__ __device__ void operator()(int j, bool nonzero) {
    if (!nonzero) return;
    count[j]++;
    if (row < first[j]) first[j] = row;
    if (last[j] == UINT64_MAX || row > last[j]) last[j] = row;
  }
};

}  // namespace tvm
