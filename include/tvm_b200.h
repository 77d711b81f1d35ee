/* libtvm_b200 — C ABI of the H100-native (sm_90a) backend for Triton VM's Stark::prove() hot path.
 *
 * The reference (TritonVM/triton-vm @ 8cd9a0eb) has no FFI for this path; its seams are
 * Rust-internal (SURVEY.md §8(b)).  Each entry point below names the reference function(s) it
 * replaces.  INTEGRATION.md shows the Rust `extern "C"` declarations and the patched
 * `Prover::prove` that would call them.
 *
 * Conventions
 *  - Host-buffer entry points take/return CANONICAL field elements (u64 < p, p = 2^64-2^32+1);
 *    X-field elements are 3 consecutive u64 (c0,c1,c2); digests are 5 u64.
 *  - `_dev` entry points take device pointers to HBM-resident data in MONTGOMERY form
 *    (R = 2^64; twenty-first's in-memory representation) and never touch host memory.
 *  - All functions return 0 on success or a negative TVM_ERR_* code; no exceptions or panics
 *    cross the ABI.  tvm_last_error() gives a human-readable description.
 *  - A tvm_ctx is single-caller (like the reference's prove(): one driving thread); several
 *    contexts may run concurrently on different devices.
 *  - Caller owns every host pointer, for the duration of the call only.
 */
#ifndef TVM_B200_H
#define TVM_B200_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define TVM_OK 0
#define TVM_ERR_INVALID_ARG (-1)
#define TVM_ERR_CUDA (-2)
#define TVM_ERR_OOM (-3)          /* ProvingError::OutOfMemory, triton-vm/src/error.rs:184-185 */
#define TVM_ERR_ZK_VIOLATION (-4) /* ProvingError::ZeroKnowledgeViolation, stark.rs:648-663 */
#define TVM_ERR_DOMAIN (-5)       /* ArithmeticDomainError, error.rs */
#define TVM_ERR_LDT_PARAMS (-6)   /* LdtParameterError */
#define TVM_ERR_STATE (-7)
#define TVM_ERR_UNSUPPORTED (-8)
#define TVM_ERR_VERIFICATION (-9) /* VerificationError / LdtVerificationError, error.rs:190-260: the proof is rejected */

typedef struct tvm_ctx tvm_ctx;

/* ---- context ------------------------------------------------------------------------- */
int tvm_ctx_create(tvm_ctx **out, int cuda_device);
void tvm_ctx_destroy(tvm_ctx *ctx);
int tvm_ctx_set_stream(tvm_ctx *ctx, void *cuda_stream /* cudaStream_t, NULL = own stream */);
int tvm_ctx_synchronize(tvm_ctx *ctx);
/* Memory mode of tvm_prove.  The reference either caches the low-degree-extended tables or recomputes them just in
 * time (TVM_LDE_TRACE / MasterTable::maybe_low_degree_extend_all_columns, master_table.rs:258-322; JIT branch
 * stark.rs:805-1006).  0 = decide from the free device memory (default), 1 = always just in time (the extended
 * main/aux tables are never stored: every coset is re-evaluated for row hashing, for the AIR and for the openings),
 * 2 = always cache.  The proof is identical in both modes. */
int tvm_ctx_set_low_memory(tvm_ctx *ctx, int mode);
int tvm_last_prove_low_memory(const tvm_ctx *ctx); /* 1 if the last tvm_prove ran just in time */

/* Multi-GPU: one process (and one context) per GPU.  A proof is sharded by evaluation-domain cosets
 * (SURVEY.md 8(e), mirroring the reference's own coset decomposition, stark.rs:824-885): rank g of
 * `world` owns the LDT-domain rows i with (i mod 8) mod world == g; trace columns are interpolated
 * column-sharded.  The library needs two collectives from the host's communication layer (NCCL through
 * torch.distributed in this repo, ncclAllGather / ncclAllReduce directly from Rust).  Both operate IN
 * PLACE on device memory and must be ordered on `cuda_stream` (or complete before returning):
 *   all_gather:  rank g contributes the bytes_per_rank bytes at dev_buf + g*bytes_per_rank; afterwards
 *                every rank holds all world*bytes_per_rank bytes;
 *   all_reduce_sum_u64: element-wise wrapping sum of `count` uint64 over all ranks.
 * Return 0 on success.  world must be 1, 2, 4 or 8.  Every rank must call tvm_prove with identical
 * arguments (each rank only reads its own column slice of the traces) and obtains the identical proof. */
typedef struct tvm_comm {
  int rank, world;
  void *user;
  int (*all_gather)(void *user, void *dev_buf, size_t bytes_per_rank, void *cuda_stream);
  int (*all_reduce_sum_u64)(void *user, uint64_t *dev_buf, size_t count, void *cuda_stream);
} tvm_comm;
int tvm_ctx_set_comm(tvm_ctx *ctx, const tvm_comm *comm /* NULL = single GPU */);
const char *tvm_strerror(int code);
const char *tvm_last_error(const tvm_ctx *ctx);
uint64_t tvm_launch_count(const tvm_ctx *ctx); /* CUDA kernels launched through this ctx */
int tvm_device_count(void);

/* ---- field representation ------------------------------------------------------------ */
int tvm_to_mont_dev(tvm_ctx *ctx, uint64_t *d_data, size_t n);
int tvm_from_mont_dev(tvm_ctx *ctx, uint64_t *d_data, size_t n);

/* ---- NTT: twenty_first::math::ntt::{ntt,intt} (call sites stark.rs:872,877,997,1002,1176;
 *      arithmetic_domain.rs:150,188).  ncols independent transforms of 2^log2n elements,
 *      packed [ncols][n], natural order in and out. ------------------------------------- */
int tvm_ntt_bfe_dev(tvm_ctx *ctx, const uint64_t *d_in, uint64_t *d_out, uint64_t *d_tmp /* ncols*n */,
                    unsigned log2n, size_t ncols, int inverse);
int tvm_ntt_bfe(tvm_ctx *ctx, uint64_t *host_data, unsigned log2n, size_t ncols, int inverse);

/* ---- column LDE: MasterTable::maybe_low_degree_extend_all_columns (master_table.rs:258-322)
 *      = randomized_column_interpolant (392-403) + ArithmeticDomain::evaluate
 *      (arithmetic_domain.rs:141-170) for every column.
 *      d_trace [ncols][n]; d_rand [ncols][num_rand] trace-randomizer coefficients or NULL;
 *      evaluation domain = offset * <w_{r n}>, r = 2^log2_cosets.
 *      d_coef  [ncols][2n]  out: interpolant coefficients pre-scaled by offset^j (kept for
 *                           later stages: OOD evaluation, row re-extrapolation)
 *      d_out   [ncols][r*n] out: COSET-MAJOR codewords, d_out[q][c*n + k] = value at
 *                           evaluation-domain index i = c + r*k
 *      d_tmp   [ncols][r*n] scratch */
int tvm_lde_bfe_dev(tvm_ctx *ctx, const uint64_t *d_trace, const uint64_t *d_rand, unsigned num_rand,
                    unsigned log2_trace, unsigned log2_cosets, uint64_t offset_canon, size_t ncols,
                    uint64_t *d_coef, uint64_t *d_out, uint64_t *d_tmp);
/* host buffers, canonical; out is [ncols][r*n] in NATURAL evaluation-domain order */
int tvm_lde_bfe(tvm_ctx *ctx, const uint64_t *trace_colmajor, const uint64_t *rand, unsigned num_rand,
                unsigned log2_trace, unsigned log2_cosets, uint64_t offset_canon, size_t ncols, uint64_t *out);

/* ---- Tip5 row hashing: MasterTable::hash_all_ldt_domain_rows (master_table.rs:455-465),
 *      quotient-segment rows (stark.rs:425-446).  Table is column-major, column q at
 *      d_table + q*col_stride; if log2_cosets > 0 each column is coset-major as produced by
 *      tvm_lde_bfe_dev.  Digests are written in natural row order, [nrows][5]. ----------- */
int tvm_tip5_hash_rows_dev(tvm_ctx *ctx, const uint64_t *d_table, size_t col_stride, size_t nrows,
                           unsigned ncols, unsigned log2_cosets, uint64_t *d_digests);
int tvm_tip5_hash_rows(tvm_ctx *ctx, const uint64_t *table_colmajor /* [ncols][nrows] */, size_t nrows,
                       unsigned ncols, uint64_t *digests /* [nrows][5] */);
/* Tip5::hash_varlen on the host (transcript-side helper; program/claim hashing) */
int tvm_tip5_hash_varlen(const uint64_t *words, size_t n, uint64_t digest[5]);

/* ---- Merkle tree: MerkleTree::par_new (master_table.rs:449, stark.rs:443, fri.rs:346).
 *      d_nodes [2*nleaves][5]; leaves must already be at d_nodes[nleaves..2*nleaves);
 *      node i = hash_pair(node 2i, node 2i+1); root = node 1. -------------------------- */
int tvm_merkle_build_dev(tvm_ctx *ctx, uint64_t *d_nodes, size_t nleaves);
int tvm_merkle_build(tvm_ctx *ctx, const uint64_t *leaves /* [nleaves][5] */, size_t nleaves,
                     uint64_t *nodes_out /* [2*nleaves][5] or NULL */, uint64_t root[5]);

/* ---- AIR quotient codeword: all_quotients_combined (master_table.rs:1264-1363) with the
 *      build-time generated constraint evaluators (constraint-builder/src/codegen.rs:59-269)
 *      and the four zerofier inverses (master_table.rs:1194-1252).
 *      d_main [>=379 columns][r*n], d_aux [>=270 B-field columns = 90 X-field columns x 3][r*n],
 *      both coset-major LDE tables on the quotient domain offset*<w_{rn}>;
 *      challenges: 63 X-field elements, weights: 604 X-field elements (host, canonical);
 *      d_out: 3 planes (coordinate d at d_out + d*out_stride) of r*n words, coset-major order:
 *      d_out[c*n + k] = quotient value at domain index i = c + r*k. ----------------------- */
#define TVM_NUM_MAIN_COLUMNS 379
#define TVM_NUM_MAIN_TABLE_COLUMNS 149 /* the nine tables' columns; 149..378 are degree-lowering columns */
#define TVM_NUM_AUX_COLUMNS 91
#define TVM_NUM_CHALLENGES 63
#define TVM_NUM_CONSTRAINTS 604
int tvm_air_quotient_dev(tvm_ctx *ctx, const uint64_t *d_main, size_t main_stride, const uint64_t *d_aux,
                         size_t aux_stride, const uint64_t *challenges, const uint64_t *weights,
                         unsigned log2_trace, unsigned log2_cosets, uint64_t offset_canon,
                         uint64_t *d_out, size_t out_stride);

/* ---- STARK parameters: Stark::{ldt,fri,max_degree,randomized_trace_len,num_trace_randomizers}
 *      (stark.rs:1885-2089), ProverDomains::derive (263-286), FriParameters (fri.rs:799-924),
 *      ReedSolomonCode (low_degree_test/mod.rs:215-300).  Pure function, no GPU needed. ------- */
typedef struct tvm_params {
  uint32_t security_level;            /* Stark::default(): 160 */
  uint32_t log2_ldt_expansion_factor; /* Stark::default(): 2   */
  uint32_t ldt_choice;                /* 0 = the reference's heuristic (Stark::default(): FRI below padded height 2^16,
                                         STIR from there on, stark.rs:1942-1957); 1 = LdtChoice::Fri; 2 = LdtChoice::Stir */
  uint32_t soundness;                 /* ProximityRegime (low_degree_test/mod.rs:60-80): 0 = Proven (default), 1 = Conjectured */
} tvm_params;
typedef struct tvm_domains {
  uint64_t padded_height, num_trace_randomizers, randomized_trace_len, trace_len, quotient_len, ldt_len;
  uint64_t ldt_offset;                /* canonical; trace and randomized-trace domains have offset 1 */
  uint64_t num_collinearity_checks, fri_num_rounds, fri_last_round_max_degree;
  uint64_t num_quotient_randomizer_coefficients; /* (h + 1) * 5 X-field coefficients, stark.rs:1320-1322 */
  /* low-degree test actually used and its round structure (stir.rs:437-567) */
  uint64_t ldt;                       /* 1 = FRI, 2 = STIR */
  uint64_t num_first_round_queries;   /* rows opened from each table; h = this + 4*3*2 + 1 (stark.rs:2083-2089) */
  uint64_t stir_num_rounds;           /* full rounds (0 for FRI) */
  uint64_t stir_in_domain_queries[16], stir_out_of_domain_queries[16];
  uint64_t stir_final_num_queries, stir_final_degree;
} tvm_domains;
int tvm_derive_domains(const tvm_params *params, uint64_t padded_height, tvm_domains *out);

/* ---- Stark::prove (stark.rs:1845-1851 -> Prover::prove 331-719) for already generated traces.
 *      claim: program digest (5 words), version, public input / output (proof.rs:68-88).
 *      main_trace   [379][trace_len]  column-major, canonical (MasterMainTable after pad(),
 *                                      master_table.rs:881-983, trace_table is column-major: 888)
 *      main_rand    [379][h]          trace-randomizer coefficients per column (master_table.rs:423-434)
 *      aux_cb       called once with the 63 challenges (canonical X-field, challenges.rs:88-135); must
 *                   provide aux_trace [91][trace_len][3] (MasterMainTable::extend, 1006-1075, incl. the
 *                   batch-randomizer column 90) and aux_rand [91][h][3] by setting *aux_trace / *aux_rand
 *                   to caller-owned (ideally pinned) buffers that stay valid until tvm_prove returns
 *      quot_rand    [(h+1)*5][3]      quotient-segment randomizer (stark.rs:1316-1322)
 *      proof_out    receives Proof.0 (Vec<BFieldElement>, canonical); *proof_len in: capacity, out: needed
 *                   length (TVM_ERR_INVALID_ARG with *proof_len set if the capacity is too small).
 *      All randomness is the caller's: the backend is a deterministic function of its inputs. --- */
typedef int (*tvm_aux_callback)(void *user, const uint64_t *challenges /*[63][3]*/, uint64_t **aux_trace, uint64_t **aux_rand);
typedef struct tvm_claim {
  uint64_t program_digest[5];
  uint32_t version;
  const uint64_t *input; size_t num_input;
  const uint64_t *output; size_t num_output;
} tvm_claim;
int tvm_prove(tvm_ctx *ctx, const tvm_params *params, const tvm_claim *claim, uint64_t padded_height,
              const uint64_t *main_trace, const uint64_t *main_rand, tvm_aux_callback aux_cb, void *aux_user,
              const uint64_t *quot_rand, uint64_t *proof_out, size_t *proof_len);
/* ---- Stark::prove with the HOST keeping the transcript (SURVEY.md 8(b), "who keeps the sponge"): a Rust host hands callbacks
 *      into its own `ProofStream` (proof_stream.rs:19-104); the library then only PRODUCES proof items and CONSUMES challenges,
 *      in exactly the order of Prover::prove (stark.rs:331-719) - Fiat-Shamir, the item list, `Proof` and its BFieldCodec stay on
 *      the host side.  All words canonical.
 *        alter_fiat_shamir_state  ProofStream::alter_fiat_shamir_state_with(&claim): called once, first, with the Claim's encoding
 *        enqueue                  ProofStream::enqueue(item): `variant` = index of the ProofItem variant in declaration order
 *                                 (proof_item.rs:96-147: 0 MerkleRoot, 1 Log2PaddedHeight, 2 OutOfDomainMainRow, 3 OutOfDomainAuxRow,
 *                                 4 OutOfDomainQuotientSegments, 5 Polynomial, 6 StirOutOfDomainValues, 7 AuthenticationStructure,
 *                                 8 MasterMainTableRows, 9 MasterAuxTableRows, 10 QuotientSegmentsElements, 11 FriCodeword,
 *                                 12 FriResponse, 13 StirResponse), `payload` = the variant's BFieldCodec payload
 *        sample_scalars           ProofStream::sample_scalars(n) -> n X-field elements ([n][3])
 *        sample_indices           ProofStream::sample_indices(upper_bound, n)
 *      Every callback returns 0 on success.  Other arguments as tvm_prove; no proof buffer: the host's stream holds the items. --- */
typedef struct tvm_transcript {
  void *user;
  int (*alter_fiat_shamir_state)(void *user, const uint64_t *words, size_t n);
  int (*enqueue)(void *user, unsigned variant, const uint64_t *payload, size_t n);
  int (*sample_scalars)(void *user, size_t n, uint64_t *out);
  int (*sample_indices)(void *user, unsigned upper_bound, size_t n, unsigned *out);
} tvm_transcript;
int tvm_prove_transcript(tvm_ctx *ctx, const tvm_params *params, const tvm_claim *claim, uint64_t padded_height,
                         const uint64_t *main_trace, const uint64_t *main_rand, tvm_aux_callback aux_cb, void *aux_user,
                         const uint64_t *quot_rand, const tvm_transcript *transcript);
/* ---- Stark::prove with the table stages on the device (SURVEY.md 8(f).1): what Prover::prove does between
 *      MasterMainTable::new/pad and the proof (stark.rs:331-719 together with master_table.rs:975-983, 1006-1075).  The main
 *      trace is uploaded once and stays resident: MasterMainTable::extend (the nine tables' `extend` +
 *      fill_derived_aux_columns) runs on it as soon as the challenges are known, no callback, no host round trip of the
 *      auxiliary table.
 *      main_table   [379][trace_len] canonical, column-major; with fill_derived_main_columns != 0 only columns 0..148 (the
 *                   nine tables) are read and uploaded, the 230 degree-lowering columns are computed on the device
 *                   (DegreeLoweringTable::fill_derived_main_columns, substitutions.rs:128-161)
 *      aux_rand     [91][h][3]  trace-randomizer coefficients of the auxiliary columns
 *      randomizer_column [trace_len][3]  auxiliary column 90 (master_table.rs:1019-1025); NULL = zeros
 *      other arguments and the proof: as tvm_prove (identical proof words for identical tables and randomness).
 *      With tvm_ctx_set_comm (world > 1) every rank is handed the same table: each holds the whole main trace, runs the
 *      extension itself and interpolates its own block of columns; the cosets are sharded as in tvm_prove. --- */
int tvm_prove_tables(tvm_ctx *ctx, const tvm_params *params, const tvm_claim *claim, uint64_t padded_height,
                     const uint64_t *main_table, int fill_derived_main_columns, const uint64_t *main_rand, const uint64_t *aux_rand,
                     const uint64_t *randomizer_column, const uint64_t *quot_rand, uint64_t *proof_out, size_t *proof_len);
/* ---- The witness at the boundary: AlgebraicExecutionTrace (aet.rs:41-91) -> MasterMainTable::new + pad + the proof
 *      (SURVEY.md 8(f).4).  Every array is what the reference's AET holds, row-major, canonical words:
 *        program                    Program::to_bwords()
 *        instruction_multiplicities [program_len]                          (aet.rs:52)
 *        processor_trace            [processor_rows][39]                   (aet.rs:55; ProcessorMainColumn order)
 *        op_stack_underflow_trace   [op_stack_rows][4]                     (aet.rs:57; clk, IB1 shrink, stack pointer, element)
 *        ram_trace                  [ram_rows][7]                          (aet.rs:59; columns 4..6 unused, as RamTableCall::to_table_row leaves them)
 *        program_hash_trace / sponge_trace / hash_trace  [rows][67]        (aet.rs:67-76; HashMainColumn order, CI set, Mode unset)
 *        u32_entries                [u32_count][4]: opcode, left operand, right operand, multiplicity, in IndexMap order (aet.rs:85)
 *        cascade_table_lookup_multiplicities [cascade_count][2]: 16-bit limb, multiplicity, in IndexMap order (aet.rs:90)
 *        lookup_table_lookup_multiplicities  [256]                         (aet.rs:93) --- */
typedef struct tvm_aet {
  const uint64_t *program; uint64_t program_len;
  const uint32_t *instruction_multiplicities;
  const uint64_t *processor_trace; uint64_t processor_rows;
  const uint64_t *op_stack_underflow_trace; uint64_t op_stack_rows;
  const uint64_t *ram_trace; uint64_t ram_rows;
  const uint64_t *program_hash_trace; uint64_t program_hash_rows;
  const uint64_t *sponge_trace; uint64_t sponge_rows;
  const uint64_t *hash_trace; uint64_t hash_rows;
  const uint64_t *u32_entries; uint64_t u32_count;
  const uint64_t *cascade_table_lookup_multiplicities; uint64_t cascade_count;
  const uint64_t *lookup_table_lookup_multiplicities;
} tvm_aet;
/*      tvm_main_table_from_aet: MasterMainTable::new + pad (master_table.rs:881-974) on the device: the nine tables' `fill`
 *      (sorting the memory-like tables, clock-jump-difference multiplicities, the RAM table's Bezout coefficient
 *      polynomials ram.rs:162-214, the u32 sections u32.rs:193-290), their `pad`, and the degree-lowering columns.
 *        num_rows       rows of the table (a power of two >= every table's length; the trace-domain length)
 *        main_table_out [379][num_rows] canonical, column-major (host memory)
 *        table_lengths_out (optional) [9]: program, processor, op stack, ram, jump stack, hash, cascade, lookup, u32
 *      tvm_prove_aet: the same fill as the first stage of tvm_prove_tables; nothing but the AET and the randomness is
 *      uploaded, the table never exists on the host.  Other arguments (and the multi-GPU behaviour) as tvm_prove_tables. --- */
int tvm_main_table_from_aet(tvm_ctx *ctx, const tvm_aet *aet, uint64_t num_rows, uint64_t *main_table_out, uint64_t *table_lengths_out);
int tvm_prove_aet(tvm_ctx *ctx, const tvm_params *params, const tvm_claim *claim, uint64_t padded_height, const tvm_aet *aet,
                  const uint64_t *main_rand, const uint64_t *aux_rand, const uint64_t *randomizer_column, const uint64_t *quot_rand,
                  uint64_t *proof_out, size_t *proof_len);
/* ---- Seeded proving: the prover's randomness drawn on the device from ONE 32-byte seed, exactly as Prover::prove draws it
 *      from its `randomness_seed` (stark.rs:192, 293-328): every array comes from its own
 *      StdRng::from_seed(offset_rng_seed(seed, k)) stream (master_table.rs:630-662; StdRng = ChaCha12, each B-field element one
 *      sample of rand's `random_range(0..=p-1)`, each X-field element three):
 *        main_rand          [379][h]     k = column                     (trace_randomizer_for_column, master_table.rs:423-434)
 *        aux_rand           [91][h][3]   k = 379 + column               (offset_rng_seed(offset_rng_seed(seed, 379), column))
 *        randomizer_column  [n][3]       k = 379 + 91                   (auxiliary column 90, master_table.rs:1016-1023)
 *        quot_rand          [(h+1)*5][3] k = 379 + 91 + 1               (quotient-segment randomizer, stark.rs:1316-1322)
 *      h, n and the quotient coefficient count as tvm_derive_domains reports them for `params` and `padded_height`.
 *      WARNING (as the reference's Prover::set_randomness_seed_which_may_break_zero_knowledge): the proof is zero-knowledge
 *      only if the seed comes from a cryptographically secure RNG that the verifier can neither predict nor influence (what
 *      Prover::new does with `random()`).  A fixed or reused seed breaks zero knowledge.  The library never draws entropy
 *      itself: it stays a deterministic function of its inputs, and a NULL seed is TVM_ERR_INVALID_ARG.
 *
 *      tvm_prover_randomness: kernel-level entry point; the four arrays (canonical) into host or device memory, any of them
 *      may be NULL.
 *      tvm_prove_aet_seeded / tvm_prove_tables_seeded: the proof words tvm_prove_aet / tvm_prove_tables give when handed the
 *      arrays tvm_prover_randomness returns for the same seed.  The randomness is generated in device memory and never
 *      crosses PCIe.  With tvm_ctx_set_comm every rank is handed the same seed and derives the identical randomness itself. */
int tvm_prover_randomness(tvm_ctx *ctx, const tvm_params *params, uint64_t padded_height, const uint8_t seed[32], uint64_t *main_rand_out,
                          uint64_t *aux_rand_out, uint64_t *randomizer_column_out, uint64_t *quot_rand_out);
int tvm_prove_aet_seeded(tvm_ctx *ctx, const tvm_params *params, const tvm_claim *claim, uint64_t padded_height, const tvm_aet *aet,
                         const uint8_t seed[32], uint64_t *proof_out, size_t *proof_len);
int tvm_prove_tables_seeded(tvm_ctx *ctx, const tvm_params *params, const tvm_claim *claim, uint64_t padded_height,
                            const uint64_t *main_table, int fill_derived_main_columns, const uint8_t seed[32], uint64_t *proof_out,
                            size_t *proof_len);
/* ---- Proving a program from its inputs: VM::trace_execution (vm.rs:159-196) and triton_vm::prove_program (lib.rs:228-267).
 *      tvm_trace_execution runs the program on the host and keeps what AlgebraicExecutionTrace (aet.rs:41-91) records, except
 *      the three Hash-table traces: of those only the 16-word input state of every Tip5 permutation is kept, and the traces
 *      (67 columns, 6 rows per permutation) are expanded on the device when they are needed.
 *        program      Program::to_bwords() (no length prefix), decoded as Program::decode (program.rs:65-108) decodes it
 *        public_input PublicInput; nd: NonDeterminism (vm.rs:1467-1471), NULL = empty
 *      Words >= p in the program, inputs, digests or RAM, and a RAM address given twice, are TVM_ERR_INVALID_ARG.  A program
 *      the VM rejects is TVM_ERR_VM; `failure` (optional) then names the reference's variant and, for a VMError, the clock
 *      cycle and instruction pointer: "VMError: AssertionFailed (clk 17, ip 9)", "ProgramDecodingError: MissingArgument(6, push)".
 *      DIVERGENCE: the reference runs a program that never halts until memory is exhausted.  Here execution stops with
 *      TVM_ERR_DOMAIN as soon as any table would grow beyond 2^26 rows, the largest height tvm_main_table_from_aet takes: nothing
 *      taller can be proved by this library.
 *      The execution is host memory only; any number of contexts may use it concurrently. --- */
#define TVM_ERR_VM (-10)          /* VMError / ProgramDecodingError: the program cannot be executed */
#define TVM_CURRENT_VERSION 6     /* proof.rs:33; the version tvm_prove_execution puts into the claim (Claim::new) */
typedef struct tvm_nondeterminism {                                     /* NonDeterminism (vm.rs:1467-1471) */
  const uint64_t *individual_tokens; size_t num_individual_tokens;     /* secret input, consumed by `divine` */
  const uint64_t *digests; size_t num_digests;                         /* [num_digests][5], consumed by `merkle_step` */
  const uint64_t *ram_addresses, *ram_values; size_t num_ram;          /* initial RAM */
} tvm_nondeterminism;
typedef struct tvm_execution tvm_execution;
typedef struct tvm_execution_summary {
  uint64_t program_digest[5];   /* Program::hash */
  uint64_t padded_height;       /* AlgebraicExecutionTrace::padded_height (aet.rs:133-146) */
  uint64_t table_heights[9];    /* height_of_table, in the order of tvm_main_table_from_aet's table_lengths_out */
  uint64_t num_output;
} tvm_execution_summary;
/* host code, no GPU */
int tvm_trace_execution(const uint64_t *program, size_t program_len, const uint64_t *public_input, size_t num_input,
                        const tvm_nondeterminism *nd, tvm_execution **out, char *failure, size_t failure_capacity);
/* output: [num_output] public output, or NULL */
int tvm_execution_info(const tvm_execution *ex, tvm_execution_summary *out, uint64_t *output);
/* the reference's AET as tvm_aet: pointers into storage owned by `ex`, valid until tvm_execution_destroy.  The three hash traces
 * are expanded on the device of `ctx` (and kept with `ex`); with ctx == NULL they are NULL, their row counts are still set. */
int tvm_execution_aet(tvm_ctx *ctx, const tvm_execution *ex, tvm_aet *out);
/* Stark::prove(Claim::new(digest).with_input(input).with_output(output), aet) with Prover::prove's randomness drawn from `seed`:
 * the proof words tvm_prove_aet_seeded gives for that claim (version TVM_CURRENT_VERSION), tvm_execution_aet's AET and the
 * execution's padded height.  The hash traces are expanded into device memory and never cross PCIe.  The proof-capacity
 * protocol is tvm_prove's; a retry proves again but does not execute again.  With tvm_ctx_set_comm every rank traces the same
 * inputs itself and calls this with the same seed.  The seed WARNING of the seeded entry points applies. */
int tvm_prove_execution(tvm_ctx *ctx, const tvm_params *params, const tvm_execution *ex, const uint8_t seed[32],
                        uint64_t *proof_out, size_t *proof_len);
void tvm_execution_destroy(tvm_execution *ex);
/* Bezout coefficient polynomials of rp = prod (x - roots[i]) and its formal derivative (ram.rs:162-214), kernel-level entry
 * point: `roots` m distinct canonical elements; a_out, b_out [m] canonical coefficients, lowest first. */
int tvm_bezout_coefficients(tvm_ctx *ctx, const uint64_t *roots, uint64_t m, uint64_t *a_out, uint64_t *b_out);
/* ---- STIR as a stand-alone low-degree test: Stir::prove / Stir::verify (low_degree_test/stir.rs:885-993, 995-1108) of the sealed
 *      `LowDegreeTest` trait (mod.rs:48-100) for ARBITRARY StirParameters (stir.rs:395-435; folding factor 2^2 as Stark::ldt fixes
 *      it, stark.rs:2023).  Used by the restated property tests of the reference (stir.rs:1813-2010) and by hosts that keep
 *      Prover::prove's orchestration.  The initial domain has 2^(log2_high_degree_bound + log2_initial_expansion_factor) points and
 *      offset BFieldElement::generator() (stir.rs:589).
 *      codeword   [len][3] canonical X-field evaluations on that domain (host or device memory)
 *      proof_out  the encoded proof stream of the STIR items alone (Proof.0 layout; same capacity protocol as tvm_prove)
 *      indices_out (optional) receives the revealed first-round indices; *num_indices in: capacity, out: count. --- */
int tvm_stir_prove(tvm_ctx *ctx, uint32_t security_level, uint32_t soundness, uint32_t log2_initial_expansion_factor,
                   uint32_t log2_high_degree_bound, const uint64_t *codeword, uint64_t *proof_out, size_t *proof_len,
                   uint32_t *indices_out, size_t *num_indices);
/* host code, no GPU; TVM_OK = accepted, TVM_ERR_VERIFICATION = rejected (`failure` names the LdtVerificationError variant);
 * on acceptance the verifier's postscript: first-round indices and the partial first codeword [count][3] (optional outputs) */
int tvm_stir_verify(uint32_t security_level, uint32_t soundness, uint32_t log2_initial_expansion_factor, uint32_t log2_high_degree_bound,
                    const uint64_t *proof, size_t proof_len, uint32_t *indices_out, uint64_t *values_out, size_t *num_indices,
                    char *failure, size_t failure_capacity);
/* ---- FRI as a stand-alone low-degree test: Fri::prove / Fri::verify (low_degree_test/fri.rs:212-366, 393-735, 754-789) of the
 *      sealed `LowDegreeTest` trait for ARBITRARY FriParameters (fri.rs:799-845): the prover Stark::default() uses below padded
 *      height 2^16 and LdtChoice::Fri everywhere, for hosts that keep Prover::prove's orchestration and for the restated
 *      property tests of the reference (fri.rs:989-1425).  The initial domain has 2^(log2_high_degree_bound +
 *      log2_initial_expansion_factor) points and offset BFieldElement::generator() (fri.rs:829).  The whole prove and
 *      tvm_verify run the same prover and verifier.
 *      Parameter errors are LdtParameterError's (fri.rs:800-829): TVM_ERR_LDT_PARAMS for log2_initial_expansion_factor == 0
 *      (TooSmallInitialExpansionFactor), >= 32 (TooBigInitialExpansionFactor) or an initial domain beyond 2^32 points
 *      (InitialDomainTooBig); the variant is named in tvm_last_error / `failure`. --- */
typedef struct tvm_fri_info {
  uint64_t domain_len, domain_offset, expansion_factor, max_degree;   /* domain_offset canonical; max_degree = Fri::max_degree */
  uint64_t num_collinearity_checks, num_rounds, last_round_max_degree;
} tvm_fri_info;
/* host code, no GPU: FriParameters::try_into_fri and Fri::{max_degree, num_rounds, last_round_max_degree} (fri.rs:799-924) */
int tvm_fri_derive(uint32_t security_level, uint32_t soundness, uint32_t log2_initial_expansion_factor, uint32_t log2_high_degree_bound,
                   tvm_fri_info *out);
/*      codeword     [codeword_len][3] canonical X-field evaluations on the initial domain (host or device memory);
 *                   codeword_len != domain length is TVM_ERR_INVALID_ARG, "InitialCodewordMismatch { domain_len, codeword_len }"
 *                   (LdtProvingError, fri.rs:323-330).  Initial domains beyond 2^26 points are TVM_ERR_DOMAIN.
 *      proof_out    the encoded proof stream of the FRI items alone (Proof.0 layout; same capacity protocol as tvm_prove)
 *      indices_out  (optional) receives the first-round collinearity-check indices; *num_indices in: capacity, out: count.
 *      Argument and parameter errors return before any kernel is launched. */
int tvm_fri_prove(tvm_ctx *ctx, uint32_t security_level, uint32_t soundness, uint32_t log2_initial_expansion_factor,
                  uint32_t log2_high_degree_bound, const uint64_t *codeword, size_t codeword_len, uint64_t *proof_out, size_t *proof_len,
                  uint32_t *indices_out, size_t *num_indices);
/* host code, no GPU; TVM_OK = accepted, TVM_ERR_VERIFICATION = rejected (`failure` names the LdtVerificationError variant);
 * on acceptance the verifier's postscript: first-round indices and the partial first codeword [count][3] (optional outputs).
 * An initial domain of 2^32 points is TVM_ERR_DOMAIN: the proof stream samples indices below u32::MAX only
 * (proof_stream.rs:85-89). */
int tvm_fri_verify(uint32_t security_level, uint32_t soundness, uint32_t log2_initial_expansion_factor, uint32_t log2_high_degree_bound,
                   const uint64_t *proof, size_t proof_len, uint32_t *indices_out, uint64_t *values_out, size_t *num_indices,
                   char *failure, size_t failure_capacity);
/* ---- auxiliary table: MasterMainTable::extend (master_table.rs:1006-1075) = the nine tables' `extend`
 *      (TraceTable::extend, table.rs:29-48; e.g. processor.rs:97-137, hash.rs:304-460, ram.rs:105-255) followed by
 *      DegreeLoweringTable::fill_derived_aux_columns (substitutions.rs:163-205).  SURVEY.md 8(f).1: the stage a host
 *      otherwise runs inside tvm_aux_callback.
 *      main_trace         [379][n]  canonical, column-major (the tvm_prove layout), host or device memory
 *      challenges         [63][3]   canonical, host memory (what tvm_aux_callback receives)
 *      randomizer_column  [n][3]    canonical, host or device: the batch-randomizer column 90 (master_table.rs:1019-1025;
 *                                   the reference draws it from its own seeded RNG); NULL = zeros
 *      aux_trace_out      [91][n][3] canonical, host or device memory — directly usable as tvm_aux_callback's *aux_trace
 *      n = 2^log2_n rows.  May be called from inside tvm_aux_callback on the same or on another context. --- */
int tvm_aux_extend(tvm_ctx *ctx, const uint64_t *main_trace, unsigned log2_n, const uint64_t *challenges,
                   const uint64_t *randomizer_column, uint64_t *aux_trace_out);
/* DegreeLoweringTable::fill_derived_main_columns (generated in the reference: triton-constraint-builder/src/
 * substitutions.rs:128-161, 237-300; called from MasterMainTable::new, master_table.rs:975-983): fills the 230
 * degree-lowering columns 149..378 of main_trace [379][n] (canonical, column-major, host or device memory, IN PLACE) from
 * the 149 table columns 0..148, which are not modified. */
int tvm_fill_derived_main_columns(tvm_ctx *ctx, uint64_t *main_trace, unsigned log2_n);
/* ---- AIR constraint check of a witness: the reference's test-suite check check_constraints_fn! (stark.rs:2899-3015) on the
 *      device, for the degree-lowered AIR the prover enforces.  A witness that violates a constraint still gives a proof, which
 *      tvm_verify then rejects without saying where; these entry points name every violated constraint, its origin and rows.
 *      All 604 constraints are checked in evaluator order (init | cons | tran | term, base-field-valued before
 *      extension-field-valued; the order of tvm_air_quotient_dev's weights): init on row 0, cons on every row, tran on the pairs
 *      (i, i+1) for i < n - 1 (no wrap-around), term on row n - 1.
 *      Outputs, per constraint j: counts[j] rows where its value is non-zero, first_rows[j] / last_rows[j] the first and last
 *      such row (UINT64_MAX when counts[j] == 0); *num_violated the number of constraints with counts[j] != 0.  Violations are
 *      results: the call returns TVM_OK whenever the check ran.  The result does not depend on the launch order.
 *
 *      tvm_air_check: main_table [379][n] and aux_table [91][n][3] canonical, column-major (the tvm_aux_extend layout, host or
 *      device memory; aux column 90 is read by no constraint); challenges [63][3] canonical (host), the order tvm_aux_extend
 *      takes them; n = 2^log2_n, log2_n <= 26 (else TVM_ERR_DOMAIN).  NULL pointers are TVM_ERR_INVALID_ARG before any
 *      kernel is launched.  A word >= p is TVM_ERR_INVALID_ARG too, found by the upload pass that converts the tables (no
 *      check kernel runs); tvm_last_error names the table, column and row of the first one. */
int tvm_air_check(tvm_ctx *ctx, const uint64_t *main_table, const uint64_t *aux_table, unsigned log2_n, const uint64_t *challenges,
                  uint64_t *counts, uint64_t *first_rows, uint64_t *last_rows, uint64_t *num_violated);
/*      tvm_air_check_aet: the witness as tvm_prove_aet builds it, checked without leaving the device: MasterMainTable::new +
 *      pad from the AET (num_rows as tvm_main_table_from_aet takes it), the degree-lowering columns, Challenges::new (the 4
 *      challenges derived from `claim` and the lookup table, challenges.rs:88-135) on top of sampled_challenges [59][3]
 *      (canonical), MasterMainTable::extend with a zero randomizer column, then the check.
 *      tvm_air_check_execution: the same for an execution (tvm_trace_execution): its claim and padded height, the hash traces
 *      expanded on the device as tvm_prove_execution does.  A valid witness satisfies the AIR for every challenge value. */
int tvm_air_check_aet(tvm_ctx *ctx, const tvm_aet *aet, const tvm_claim *claim, uint64_t num_rows, const uint64_t *sampled_challenges,
                      uint64_t *counts, uint64_t *first_rows, uint64_t *last_rows, uint64_t *num_violated);
int tvm_air_check_execution(tvm_ctx *ctx, const tvm_execution *ex, const uint64_t *sampled_challenges, uint64_t *counts,
                            uint64_t *first_rows, uint64_t *last_rows, uint64_t *num_violated);
/*      tvm_air_constraint_info (host code, no GPU): constraint `index` < 604 of the evaluator order.
 *        origin        0..8 the table, in the order of tvm_main_table_from_aet's table_lengths_out; 9 the Grand Cross-Table
 *                      Argument; 10 degree lowering (a substitution constraint, which defines a derived column)
 *        origin_index  an original constraint's position in its table's list for that category before degree lowering (the
 *                      idx of the reference's ConstraintError); for a substitution constraint the derived column it defines
 *        derived_column TVM_AIR_DERIVED_MAIN (origin_index is a main column 149..378), TVM_AIR_DERIVED_AUX (an aux column
 *                      49..89) or TVM_AIR_DERIVED_NONE
 *        degree        the constraint's degree (the reference's generated quotient degree bounds)
 *        origin_name   static string: "ProcessorTable", ..., "GrandCrossTableArg", "DegreeLowering" */
#define TVM_AIR_DERIVED_NONE 0
#define TVM_AIR_DERIVED_MAIN 1
#define TVM_AIR_DERIVED_AUX 2
typedef struct tvm_air_constraint {
  uint32_t category;            /* 0 initial, 1 consistency, 2 transition, 3 terminal */
  uint32_t index_in_category;
  uint32_t degree;
  uint32_t origin;
  uint32_t origin_index;
  uint32_t derived_column;
  const char *origin_name;
} tvm_air_constraint;
int tvm_air_constraint_info(unsigned index, tvm_air_constraint *out);
/* ---- Stark::verify (stark.rs:1388-1763, Verifier::verify) — SURVEY.md 8(f).4.
 *      Replays the Fiat-Shamir transcript of `proof` (Proof.0, canonical words) against `claim` under `params`: AIR / quotient
 *      identity at the out-of-domain point, FRI or STIR, Merkle openings, DEEP combination.  Host code — one proof is a few
 *      milliseconds of strictly sequential work; needs neither a context nor a GPU.
 *      Returns TVM_OK if the proof is accepted, TVM_ERR_VERIFICATION if it is rejected (then `failure`, if given, receives the
 *      name of the reference's error variant, e.g. "VerificationError: CombinationCodewordMismatch").
 *      skip_air_check != 0 skips only the out-of-domain AIR identity (for proofs over synthetic, non-satisfying traces as
 *      used by tests and benchmarks); production callers pass 0. --- */
int tvm_verify(const tvm_params *params, const tvm_claim *claim, const uint64_t *proof, size_t proof_len, int skip_air_check,
               char *failure, size_t failure_capacity);
/* `count` independent proofs verified on `num_threads` host threads (0 = all hardware threads); results[i] = what tvm_verify
 * returns for (claims[i], proofs[i]).  Returns TVM_OK iff all are accepted, else TVM_ERR_VERIFICATION (or TVM_ERR_INVALID_ARG). */
int tvm_verify_batch(const tvm_params *params, const tvm_claim *claims, const uint64_t *const *proofs, const size_t *proof_lens,
                     size_t count, int skip_air_check, unsigned num_threads, int *results);
/* Proof::padded_height (proof.rs:37-56): TVM_ERR_VERIFICATION unless the proof decodes and holds exactly one such item. */
int tvm_proof_padded_height(const uint64_t *proof, size_t proof_len, uint64_t *padded_height);
/* device time per stage of the last tvm_prove on this ctx, reference profiler labels; returns #stages */
int tvm_last_prove_timings(const tvm_ctx *ctx, const char **names /*[20]*/, float *ms /*[20]*/);

#ifdef __cplusplus
}
#endif
#endif /* TVM_B200_H */
