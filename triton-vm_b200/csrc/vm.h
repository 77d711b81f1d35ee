// Host-side Triton VM (csrc/vm.cu): VM::trace_execution and the log it keeps for tvm_execution_aet / tvm_prove_execution.
#pragma once
#include <cstdint>
#include <string>
#include <vector>
#include "field.cuh"
#include "../../include/tvm_b200.h"

// What AlgebraicExecutionTrace (aet.rs:41-91) records, except the three hash traces: of those only the 16-word input state of
// every permutation is kept (fill/hash_trace.cuh expands them).  All words canonical unless stated otherwise.
struct tvm_execution {
  std::vector<uint64_t> program;                     // Program::to_bwords()
  std::vector<uint32_t> instruction_multiplicities;  // [program_len]
  std::vector<uint64_t> processor_trace;             // [rows][39]
  std::vector<uint64_t> op_stack_trace;              // [rows][4]
  std::vector<uint64_t> ram_trace;                   // [rows][7]
  std::vector<uint64_t> u32_entries;                 // [count][4]: opcode, lhs, rhs, multiplicity (IndexMap order)
  std::vector<uint64_t> cascade_multiplicities;      // [count][2]: limb, multiplicity (IndexMap order)
  uint64_t lookup_multiplicities[256] = {};
  std::vector<uint64_t> perm_states;                 // [permutations][16] MONTGOMERY, execution order (program hash first)
  std::vector<uint64_t> perm_meta;                   // [permutations]: hash_trace::meta_encode
  uint64_t hash_rows[3] = {};                        // rows of the program-hash, sponge and hash traces
  uint64_t digest[5] = {};
  std::vector<uint64_t> input, output;
  uint64_t table_heights[9] = {};                    // program, processor, op stack, ram, jump stack, hash, cascade, lookup, u32
  uint64_t padded_height = 0;
  mutable std::vector<uint64_t> hash_cache[3];       // tvm_execution_aet's expansion, kept for the lifetime of the execution
  mutable bool expanded = false;
};

namespace tvm {

struct VmInputs {
  const uint64_t *program; size_t program_len;
  const uint64_t *public_input; size_t num_input;
  const uint64_t *secret_input; size_t num_secret;
  const uint64_t *digests; size_t num_digests;       // [num_digests][5]
  const uint64_t *ram_addresses, *ram_values; size_t num_ram;
};

// VM::trace_execution (vm.rs:159-196).  TVM_OK, or TVM_ERR_VM / TVM_ERR_DOMAIN with `failure` naming the cause.  The inputs
// must already be canonical and the RAM addresses distinct.
int trace_execution(const VmInputs &in, tvm_execution &ex, std::string &failure);

// the largest table height the device fill takes (tvm_main_table_from_aet)
static constexpr uint64_t VM_MAX_TABLE_HEIGHT = (uint64_t)1 << 26;

}  // namespace tvm
