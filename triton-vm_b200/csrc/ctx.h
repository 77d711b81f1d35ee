// Library context: device, stream, cached power/twiddle tables, scratch memory.
#pragma once
#include <cuda_runtime.h>
#include <cstdio>
#include <functional>
#include <map>
#include <mutex>
#include <string>
#include <tuple>
#include <vector>
#include "field.cuh"
#include "../../include/tvm_b200.h"

namespace tvm {


struct CudaError {
  cudaError_t err;
  const char *file;
  int line;
};

#define TVM_CUDA(x)                                              \
  do {                                                           \
    cudaError_t e__ = (x);                                       \
    if (e__ != cudaSuccess) throw tvm::CudaError{e__, __FILE__, __LINE__}; \
  } while (0)

// two-level power table: base^e = lo[e & ((1<<shift)-1)] * hi[e >> shift]
struct PowTab {
  const u64 *lo;
  const u64 *hi;
  int shift;
};

struct DevBuf {
  void *p = nullptr;
  size_t bytes = 0;
};

struct Ctx {
  int device = 0;
  int num_sms = 132;                    // multiprocessor count of `device` (read in tvm_ctx_create; grid sizing)
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  // multi-GPU communication layer supplied by the host (tvm_ctx_set_comm); world == 1: no-ops
  tvm_comm comm{0, 1, nullptr, nullptr, nullptr};
  void all_gather(void *dev_buf, size_t bytes_per_rank);
  void all_reduce_sum(u64 *dev_buf, size_t count);
  int low_memory_mode = 0;              // 0 = automatic, 1 = always just-in-time LDE, 2 = never (tvm_ctx_set_low_memory)
  cudaStream_t copy_stream = nullptr;   // host<->device staging overlapped with compute (created on first use)
  std::vector<cudaEvent_t> copy_events; // recycled per-batch "upload done" events
  // second compute stream of the tile NTT's launch pairs (ntt_tile.cu, mixed radices): alternate pairs fill each other's
  // partial last waves
  cudaStream_t pair_stream = nullptr;
  cudaEvent_t pair_fork = nullptr, pair_join = nullptr;
  cudaStream_t get_pair_stream();
  // ticket and pair-completion counters of the persistent tile NTT (ntt_tile.cu), grown on demand
  unsigned *tile_sync = nullptr;
  size_t tile_sync_words = 0;
  cudaStream_t get_copy_stream();
  cudaEvent_t get_copy_event(size_t i);
  std::string last_error;
  unsigned long long launches = 0;  // kernels launched through this context

  // caches
  std::map<std::pair<int, int>, u64 *> tile_tw;                     // (LT, inverse) -> omega_{2^LT}^(+-e)
  std::map<std::tuple<u64, int, int>, std::pair<u64 *, u64 *>> pow_tabs;  // (base, log_count, shift)
  std::vector<void *> owned;
  // coset pre-scale tables of the tile NTT (ntt_tile.cu): key = (log_n, log_r, log_n1, M, first, step, count)
  std::map<std::tuple<unsigned, unsigned, unsigned, unsigned, unsigned, unsigned, unsigned>, u64 *> prescale_tabs;
  u64 *get_prescale(unsigned log_n, unsigned log_r, unsigned log_n1, unsigned M, unsigned first, unsigned step, unsigned count,
                    const std::function<void(u64 *, u64 *)> &fill);

  // scratch arena (grown on demand, reused)
  DevBuf scratch[4];
  // block pool for prove(): cudaMalloc/cudaFree are synchronising and slow (ms each for GB-sized
  // blocks); blocks are recycled across prove() calls instead.
  std::multimap<size_t, void *> pool_free;
  std::map<void *, size_t> pool_live;
  void *pool_alloc(size_t bytes);
  void pool_release(void *p);

  ~Ctx();
  void *alloc(size_t bytes);  // tracked device allocation (freed with the ctx)
  void free_tracked(void *p);
  void *scratch_get(int slot, size_t bytes);
  const u64 *get_tile_tw(int LT, bool inverse);
  PowTab get_pow_tab(u64 base_mont, int log_count);  // exponents < 2^log_count
};

// Exclusive use of the device's AIR constant banks.  The generated AIR kernels (air_gen/, air_check_gen/) read the weights
// and challenges from __constant__ memory, which every context on a device shares, and their launch functions upload it on
// the caller's stream.  A lease holds the device's process-wide mutex and makes c.stream wait for the previous owner's last
// AIR work (an event recorded when that lease ended); its destructor records the event on c.stream and unlocks, on an
// exception too.  The mutex is held only while work is enqueued (DESIGN.md §6j: why that cannot deadlock).
class AirConstLease {
 public:
  explicit AirConstLease(Ctx &c);
  ~AirConstLease();
  AirConstLease(const AirConstLease &) = delete;
  AirConstLease &operator=(const AirConstLease &) = delete;

 private:
  Ctx &c_;
  std::unique_lock<std::mutex> lock_;
  cudaEvent_t last_use_ = nullptr;
};

u64 root_of_unity_mont(unsigned log2n);  // twenty-first's PRIMITIVE_ROOTS, Montgomery form

}  // namespace tvm
