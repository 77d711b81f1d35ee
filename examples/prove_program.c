/* Plain-C client of the whole pipeline from a program and its input, without the reference crate: what
 * triton_vm::prove_program (lib.rs:228-267) does.  The program is the reference's benchmark workload ProgramToBench::spin
 * (triton-dev-util/src/lib.rs:49-75), embedded as its encoded words; its public input `k` makes the padded height 2^k.
 *   tvm_trace_execution   runs the VM on the host (VM::trace_execution)
 *   tvm_execution_info    program digest, padded height, public output
 *   tvm_prove_execution   hash traces expanded on the GPU, table fill, extension and proof (fixed seed: a demonstration only,
 *                         a fixed seed breaks zero knowledge)
 *   tvm_verify            checks the proof, the AIR included
 *
 *   prove_program [k]     (default 10)
 *   gcc -std=c99 -Iinclude examples/prove_program.c -Ltriton-vm_b200/lib -ltvm_b200 -o prove_program
 *
 * Exit status: 0 proof verified, 1 verification failed, 2 usage error, 3 no usable GPU (there is no CPU fallback), 4 the library
 * reported an error. */
#include <stdio.h>
#include <stdlib.h>
#include "tvm_b200.h"

/* read_io 1 addi -3 push 2 pow place 5 call spin halt  spin: pick 5 addi -1 place 5 recurse_or_return */
static const uint64_t SPIN[] = {73, 1, 65, 18446744069414584318ULL, 1, 2, 30, 25, 5, 49, 12, 0, 17, 5, 65, 18446744069414584320ULL,
                                25, 5, 32};

int main(int argc, char **argv) {
  const uint64_t k = argc > 1 ? strtoull(argv[1], NULL, 10) : 10;
  if (argc > 2 || k < 8 || k > 26) { fprintf(stderr, "usage: %s [k], 8 <= k <= 26\n", argv[0]); return 2; }
  char why[256];
  tvm_execution *ex = NULL;
  int rc = tvm_trace_execution(SPIN, sizeof SPIN / sizeof SPIN[0], &k, 1, NULL, &ex, why, sizeof why);
  if (rc) { fprintf(stderr, "tvm_trace_execution: %s (%s)\n", tvm_strerror(rc), why); return 4; }
  tvm_execution_summary info;
  uint64_t output[1];
  rc = tvm_execution_info(ex, &info, output);
  if (rc || info.num_output > 1) { fprintf(stderr, "tvm_execution_info: %s\n", tvm_strerror(rc)); return 4; }

  tvm_ctx *ctx = NULL;
  rc = tvm_ctx_create(&ctx, 0);
  if (rc) { fprintf(stderr, "tvm_ctx_create: %s\n", tvm_strerror(rc)); tvm_execution_destroy(ex); return 3; }
  const tvm_params params = {160, 2, 0, 0}; /* Stark::default() */
  uint8_t seed[32];
  for (int i = 0; i < 32; i++) seed[i] = (uint8_t)i;
  size_t proof_len = (size_t)1 << 22;
  uint64_t *proof = malloc(proof_len * sizeof *proof);
  if (!proof) return 2;
  rc = tvm_prove_execution(ctx, &params, ex, seed, proof, &proof_len);
  if (rc) { fprintf(stderr, "tvm_prove_execution: %s (%s)\n", tvm_strerror(rc), tvm_last_error(ctx)); return 4; }
  tvm_ctx_destroy(ctx);

  tvm_claim claim;
  for (int i = 0; i < 5; i++) claim.program_digest[i] = info.program_digest[i];
  claim.version = TVM_CURRENT_VERSION;
  claim.input = &k; claim.num_input = 1;
  claim.output = output; claim.num_output = (size_t)info.num_output;
  rc = tvm_verify(&params, &claim, proof, proof_len, 0, why, sizeof why);
  printf("spin(%llu): %llu cycles, padded height %llu, proof of %zu words, %s\n", (unsigned long long)k,
         (unsigned long long)info.table_heights[1], (unsigned long long)info.padded_height, proof_len, rc == TVM_OK ? "verified" : why);
  free(proof);
  tvm_execution_destroy(ex);
  return rc == TVM_OK ? 0 : 1;
}
