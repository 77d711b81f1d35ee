/* Plain-C client that proves on several contexts of one GPU at the same time: K POSIX threads, each with its own tvm_ctx on
 * device 0, trace and prove ProgramToBench::spin(k) (triton-dev-util/src/lib.rs:49-75) for its own k, all at once, and verify
 * their proofs, the AIR included.  This is the shape of a proving job queue: one context per worker thread.  A context is
 * driven by one thread at a time; contexts on the same device overlap everything but their AIR stages (DESIGN.md §6j).
 *   tvm_trace_execution   runs the VM on the host (VM::trace_execution)
 *   tvm_prove_execution   hash traces, table fill, extension and proof on the GPU (fixed seed: a demonstration only, a fixed
 *                         seed breaks zero knowledge)
 *   tvm_verify            checks the proof, the AIR included
 *
 *   prove_concurrent [K [k0]]   (default K = 4, k0 = 10): thread t proves spin(k0 + t)
 *   gcc -std=c99 -pthread -Iinclude examples/prove_concurrent.c -Ltriton-vm_b200/lib -ltvm_b200 -o prove_concurrent
 *
 * Exit status: 0 every proof verified, 1 a verification failed, 2 usage error, 3 no usable GPU (there is no CPU fallback),
 * 4 the library reported an error. */
#define _POSIX_C_SOURCE 200809L
#include <pthread.h>
#include <stdio.h>
#include <stdlib.h>
#include "tvm_b200.h"

/* read_io 1 addi -3 push 2 pow place 5 call spin halt  spin: pick 5 addi -1 place 5 recurse_or_return */
static const uint64_t SPIN[] = {73, 1, 65, 18446744069414584318ULL, 1, 2, 30, 25, 5, 49, 12, 0, 17, 5, 65, 18446744069414584320ULL,
                                25, 5, 32};
enum { MAX_THREADS = 16 };

typedef struct {
  uint64_t k;
  int status;               /* the exit status of this thread's proof */
  uint64_t padded_height;
  size_t proof_len;
  char why[256];
} job;

static pthread_barrier_t start;

static void *prove_one(void *arg) {
  job *j = arg;
  const tvm_params params = {160, 2, 0, 0}; /* Stark::default() */
  tvm_execution *ex = NULL;
  tvm_ctx *ctx = NULL;
  uint64_t *proof = NULL;
  uint64_t output[1];
  tvm_execution_summary info;
  int rc = tvm_trace_execution(SPIN, sizeof SPIN / sizeof SPIN[0], &j->k, 1, NULL, &ex, j->why, sizeof j->why);
  if (!rc) rc = tvm_execution_info(ex, &info, output);
  j->status = rc ? 4 : 0;
  if (!rc && tvm_ctx_create(&ctx, 0)) {
    snprintf(j->why, sizeof j->why, "tvm_ctx_create: no usable GPU (there is no CPU fallback)");
    j->status = 3;
  }
  pthread_barrier_wait(&start); /* every thread proves at the same time */
  if (j->status) goto done;
  uint8_t seed[32];
  for (int i = 0; i < 32; i++) seed[i] = (uint8_t)(i + j->k);
  j->proof_len = (size_t)1 << 22;
  proof = malloc(j->proof_len * sizeof *proof);
  if (!proof) { snprintf(j->why, sizeof j->why, "out of host memory"); j->status = 4; goto done; }
  rc = tvm_prove_execution(ctx, &params, ex, seed, proof, &j->proof_len);
  if (rc) { snprintf(j->why, sizeof j->why, "tvm_prove_execution: %s (%s)", tvm_strerror(rc), tvm_last_error(ctx)); j->status = 4; goto done; }
  tvm_claim claim;
  for (int i = 0; i < 5; i++) claim.program_digest[i] = info.program_digest[i];
  claim.version = TVM_CURRENT_VERSION;
  claim.input = &j->k; claim.num_input = 1;
  claim.output = output; claim.num_output = (size_t)info.num_output;
  j->padded_height = info.padded_height;
  rc = tvm_verify(&params, &claim, proof, j->proof_len, 0, j->why, sizeof j->why);
  j->status = rc == TVM_OK ? 0 : 1;
done:
  free(proof);
  tvm_ctx_destroy(ctx);
  tvm_execution_destroy(ex);
  return NULL;
}

int main(int argc, char **argv) {
  const long K = argc > 1 ? strtol(argv[1], NULL, 10) : 4;
  const long k0 = argc > 2 ? strtol(argv[2], NULL, 10) : 10;
  if (argc > 3 || K < 1 || K > MAX_THREADS || k0 < 8 || k0 + K - 1 > 26) {
    fprintf(stderr, "usage: %s [K [k0]], 1 <= K <= %d, 8 <= k0, k0 + K - 1 <= 26\n", argv[0], MAX_THREADS);
    return 2;
  }
  job jobs[MAX_THREADS] = {{0}};
  pthread_t threads[MAX_THREADS];
  if (pthread_barrier_init(&start, NULL, (unsigned)K)) { fprintf(stderr, "pthread_barrier_init failed\n"); return 4; }
  long started = 0;
  for (; started < K; started++) {
    jobs[started].k = (uint64_t)(k0 + started);
    if (pthread_create(&threads[started], NULL, prove_one, &jobs[started])) break;
  }
  if (started < K) { fprintf(stderr, "pthread_create failed\n"); return 4; } /* ends the threads waiting at the barrier */
  int status = 0;
  for (long t = 0; t < K; t++) {
    pthread_join(threads[t], NULL);
    const job *j = &jobs[t];
    if (j->status == 0 || j->status == 1)
      printf("thread %ld: spin(%llu), padded height %llu, proof of %zu words, %s\n", t, (unsigned long long)j->k,
             (unsigned long long)j->padded_height, j->proof_len, j->status == 0 ? "verified" : j->why);
    else
      fprintf(stderr, "thread %ld: spin(%llu): %s\n", t, (unsigned long long)j->k, j->why);
    if (j->status > status) status = j->status;
  }
  pthread_barrier_destroy(&start);
  return status;
}
