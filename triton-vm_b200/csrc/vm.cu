// VM::trace_execution (triton-vm/src/vm.rs:159-196) on the host: Program::decode (triton-isa/src/program.rs:65-108), the
// instruction semantics and helper variables (vm.rs:270-1111), the co-processor logs (op-stack underflow op_stack.rs:61-255,
// RAM, u32, Tip5 permutations) and the program-attestation hashing and look-up multiplicities of the AET (aet.rs:95-215,
// 305-348).  The interpretation loop is sequential by nature; the wide part of the AET, the Hash-table traces, is left as
// the permutations' input states and expanded on the device (fill/hash_trace.cuh).  Restated from the project's oracle
// (oracle/tracegen.py: execute, _program_hash, _lookup_multiplicities, aet_arrays).
#include <cstdio>
#include <unordered_map>
#include "tip5.cuh"
#include "vm.h"
#include "fill/hash_trace.cuh"

namespace tvm {
namespace {

enum : unsigned {
  HALT = 0, PUSH = 1, SKIZ = 2, POP = 3, SPLIT = 4, LT = 6, NOP = 8, DIVINE = 9, ASSERT = 10, WRITE_MEM = 11, LOG_2_FLOOR = 12,
  AND = 14, RETURN = 16, PICK = 17, HASH = 18, WRITE_IO = 19, DIV_MOD = 20, XOR = 22, RECURSE = 24, PLACE = 25,
  ASSERT_VECTOR = 26, POP_COUNT = 28, POW = 30, RECURSE_OR_RETURN = 32, DUP = 33, SPONGE_ABSORB = 34, MERKLE_STEP = 36,
  SPONGE_INIT = 40, SWAP = 41, ADD = 42, MERKLE_STEP_MEM = 44, SPONGE_ABSORB_MEM = 48, CALL = 49, MUL = 50, SPONGE_SQUEEZE = 56,
  READ_MEM = 57, EQ = 58, INVERT = 64, ADDI = 65, XX_ADD = 66, X_INVERT = 72, READ_IO = 73, XX_MUL = 74, B_HORNER_STEP = 80,
  XB_MUL = 82, X_HORNER_STEP = 88
};
enum Arg { NO_ARG, ANY_ARG, NUM_WORDS, STACK_ELEMENT };   // Instruction::change_arg (instruction.rs:612-640)

struct OpInfo { const char *name; Arg arg; };
const OpInfo *op_info(u64 opcode) {
  static const struct { unsigned op; OpInfo info; } TABLE[] = {
      {HALT, {"halt", NO_ARG}}, {PUSH, {"push", ANY_ARG}}, {SKIZ, {"skiz", NO_ARG}}, {POP, {"pop", NUM_WORDS}},
      {SPLIT, {"split", NO_ARG}}, {LT, {"lt", NO_ARG}}, {NOP, {"nop", NO_ARG}}, {DIVINE, {"divine", NUM_WORDS}},
      {ASSERT, {"assert", NO_ARG}}, {WRITE_MEM, {"write_mem", NUM_WORDS}}, {LOG_2_FLOOR, {"log_2_floor", NO_ARG}},
      {AND, {"and", NO_ARG}}, {RETURN, {"return", NO_ARG}}, {PICK, {"pick", STACK_ELEMENT}}, {HASH, {"hash", NO_ARG}},
      {WRITE_IO, {"write_io", NUM_WORDS}}, {DIV_MOD, {"div_mod", NO_ARG}}, {XOR, {"xor", NO_ARG}}, {RECURSE, {"recurse", NO_ARG}},
      {PLACE, {"place", STACK_ELEMENT}}, {ASSERT_VECTOR, {"assert_vector", NO_ARG}}, {POP_COUNT, {"pop_count", NO_ARG}},
      {POW, {"pow", NO_ARG}}, {RECURSE_OR_RETURN, {"recurse_or_return", NO_ARG}}, {DUP, {"dup", STACK_ELEMENT}},
      {SPONGE_ABSORB, {"sponge_absorb", NO_ARG}}, {MERKLE_STEP, {"merkle_step", NO_ARG}}, {SPONGE_INIT, {"sponge_init", NO_ARG}},
      {SWAP, {"swap", STACK_ELEMENT}}, {ADD, {"add", NO_ARG}}, {MERKLE_STEP_MEM, {"merkle_step_mem", NO_ARG}},
      {SPONGE_ABSORB_MEM, {"sponge_absorb_mem", NO_ARG}}, {CALL, {"call", ANY_ARG}}, {MUL, {"mul", NO_ARG}},
      {SPONGE_SQUEEZE, {"sponge_squeeze", NO_ARG}}, {READ_MEM, {"read_mem", NUM_WORDS}}, {EQ, {"eq", NO_ARG}},
      {INVERT, {"invert", NO_ARG}}, {ADDI, {"addi", ANY_ARG}}, {XX_ADD, {"xx_add", NO_ARG}}, {X_INVERT, {"x_invert", NO_ARG}},
      {READ_IO, {"read_io", NUM_WORDS}}, {XX_MUL, {"xx_mul", NO_ARG}}, {B_HORNER_STEP, {"b_horner_step", NO_ARG}},
      {XB_MUL, {"xb_mul", NO_ARG}}, {X_HORNER_STEP, {"x_horner_step", NO_ARG}}};
  for (const auto &e : TABLE)
    if (e.op == opcode) return &e.info;
  return nullptr;
}

struct Instr { unsigned op; u64 arg; bool has_arg; };

constexpr u64 U32_MAX = 0xFFFFFFFFULL;

// canonical arithmetic on top of field.cuh's Montgomery routines
u64 mulc(u64 a, u64 b) { return fmul(to_mont(a), b); }
u64 invc(u64 a) { return from_mont(finv(to_mont(a))); }
u64 inv_or_zero(u64 a) { return a ? invc(a) : 0; }
u64 powc(u64 a, u64 e) { return from_mont(fpow(to_mont(a), e)); }
struct X3 { u64 c[3]; };
xfe xm(const X3 &a) { return xmake(to_mont(a.c[0]), to_mont(a.c[1]), to_mont(a.c[2])); }
X3 xc(const xfe &a) { return {{from_mont(a.c0), from_mont(a.c1), from_mont(a.c2)}}; }
X3 xaddc(const X3 &a, const X3 &b) { return {{fadd(a.c[0], b.c[0]), fadd(a.c[1], b.c[1]), fadd(a.c[2], b.c[2])}}; }
X3 xmulc(const X3 &a, const X3 &b) { return xc(xmul(xm(a), xm(b))); }

struct VmError { std::string text; };               // VMError / ProgramDecodingError, formatted
struct DomainError { std::string text; };

struct U32Key {
  unsigned op; u64 lhs, rhs;
  bool operator==(const U32Key &o) const { return op == o.op && lhs == o.lhs && rhs == o.rhs; }
};
struct U32Hash {
  size_t operator()(const U32Key &k) const { return (size_t)(k.lhs * 0x9E3779B97F4A7C15ULL ^ (k.rhs + 0x632BE59BD9B4E019ULL) * 31 ^ k.op); }
};

unsigned bit_length(u64 x) { return x ? 64 - (unsigned)__builtin_clzll(x) : 0; }

struct Vm {
  tvm_execution &ex;
  std::vector<Instr> prog;                    // one entry per word: an instruction repeated over its argument (program.rs:97)
  std::vector<u64> stack;                     // index 0 = deepest element
  std::vector<std::pair<u64, u64>> jump_stack;
  std::vector<u64> input, secret;
  size_t input_pos = 0, secret_pos = 0, digest_pos = 0;
  const u64 *digests; size_t num_digests;
  std::unordered_map<u64, u64> ram;
  bool sponge_ok = false;
  u64 sponge[16] = {};                        // Montgomery
  std::vector<int32_t> cascade_index = std::vector<int32_t>(1 << 16, -1);
  std::unordered_map<U32Key, size_t, U32Hash> u32_index;
  uint64_t u32_height = 0;
  u64 clk = 0, ip = 0;
  std::vector<std::pair<bool, u64>> io;       // underflow IO of the current instruction: (is_write, payload)

  explicit Vm(tvm_execution &e) : ex(e) {}

  [[noreturn]] void fail(const char *variant) {
    char buf[160];
    snprintf(buf, sizeof buf, "VMError: %s (clk %llu, ip %llu)", variant, (unsigned long long)clk, (unsigned long long)ip);
    throw VmError{buf};
  }
  u64 st(size_t i) const { return stack[stack.size() - 1 - i]; }
  u64 &st_ref(size_t i) { return stack[stack.size() - 1 - i]; }
  u64 underflow() const { return stack.size() > 16 ? stack[stack.size() - 17] : 0; }
  void push(u64 e) {
    stack.push_back(e);
    io.push_back({true, underflow()});
  }
  u64 pop() {
    io.push_back({false, underflow()});
    if (stack.size() <= 16) fail("TooShallow");
    const u64 v = stack.back();
    stack.pop_back();
    return v;
  }
  void need_u32(size_t i) { if (st(i) > U32_MAX) fail("FailedU32Conversion"); }
  X3 pop_x() { X3 x; for (int k = 0; k < 3; k++) x.c[k] = pop(); return x; }
  void push_x(const X3 &x) { for (int k = 2; k >= 0; k--) push(x.c[k]); }
  u64 ram_get(u64 p) const { auto it = ram.find(p); return it == ram.end() ? 0 : it->second; }
  u64 ram_read(u64 p) {
    const u64 v = ram_get(p);
    const u64 row[7] = {clk, 1, p, v, 0, 0, 0};
    ex.ram_trace.insert(ex.ram_trace.end(), row, row + 7);
    return v;
  }
  void ram_write(u64 p, u64 v) {
    const u64 row[7] = {clk, 0, p, v, 0, 0, 0};
    ex.ram_trace.insert(ex.ram_trace.end(), row, row + 7);
    ram[p] = v;
  }
  void u32_call(unsigned op, u64 lhs, u64 rhs) {
    const U32Key key{op, lhs, rhs};
    auto it = u32_index.find(key);
    if (it != u32_index.end()) { ex.u32_entries[4 * it->second + 3]++; return; }
    u32_index.emplace(key, ex.u32_entries.size() / 4);
    const u64 row[4] = {op, lhs, rhs, 1};
    ex.u32_entries.insert(ex.u32_entries.end(), row, row + 4);
    const u64 m = std::max(op == POW ? 0 : lhs, rhs);   // rows of the section (aet.rs:137-168)
    u32_height += m ? 1 + bit_length(m) : 1;
  }

  // one Tip5 permutation of the Montgomery state `s` in place: recorded for the hash traces, its S-box look-ups counted
  // (aet.rs:305-344: rows 0..4 x state elements 0..3 x the four 16-bit limbs, first-use order)
  void permutation(u64 (&s)[16], unsigned section, unsigned ci) {
    ex.perm_states.insert(ex.perm_states.end(), s, s + 16);
    ex.perm_meta.push_back(hash_trace::meta_encode(ex.hash_rows[section], ci, section, false));
    ex.hash_rows[section] += 6;
    for (int rnd = 0; rnd < TIP5_ROUNDS; rnd++) {
      for (int e = 0; e < 4; e++)
        for (int l = 0; l < 4; l++) {
          const unsigned limb = (unsigned)(s[e] >> (16 * l)) & 0xFFFF;
          int32_t &k = cascade_index[limb];
          if (k >= 0) { ex.cascade_multiplicities[2 * k + 1]++; continue; }
          k = (int32_t)(ex.cascade_multiplicities.size() / 2);
          ex.cascade_multiplicities.push_back(limb);
          ex.cascade_multiplicities.push_back(1);
          ex.lookup_multiplicities[limb & 0xFF]++;
          ex.lookup_multiplicities[limb >> 8]++;
        }
      tip5_round_host(s, rnd);
    }
  }

  // Program::decode on the length-prefixed words (program.rs:65-108)
  void decode(const u64 *w, size_t n) {
    char buf[200];
    prog.reserve(n);
    size_t i = 0;
    while (i < n) {
      const OpInfo *info = op_info(w[i]);
      if (!info) {
        if (w[i] > U32_MAX) snprintf(buf, sizeof buf, "ProgramDecodingError: InvalidInstruction(%zu, OutOfRangeOpcode)", i);
        else snprintf(buf, sizeof buf, "ProgramDecodingError: InvalidInstruction(%zu, InvalidOpcode(%llu))", i, (unsigned long long)w[i]);
        throw VmError{buf};
      }
      Instr ins{(unsigned)w[i], 0, info->arg != NO_ARG};
      if (ins.has_arg) {
        if (i + 2 > n) {
          snprintf(buf, sizeof buf, "ProgramDecodingError: MissingArgument(%zu, %s)", i, info->name);
          throw VmError{buf};
        }
        const u64 a = w[i + 1];
        if ((info->arg == NUM_WORDS && (a < 1 || a > 5)) || (info->arg == STACK_ELEMENT && a > 15)) {
          snprintf(buf, sizeof buf, "ProgramDecodingError: InvalidInstruction(%zu, IllegalArgument(%s, %llu))", i, info->name,
                   (unsigned long long)a);
          throw VmError{buf};
        }
        ins.arg = a;
      }
      prog.push_back(ins);
      if (ins.has_arg) prog.push_back(ins);
      i += ins.has_arg ? 2 : 1;
    }
  }

  // aet.rs:150-190: absorb the padded program, trace every permutation -> program digest
  void hash_program(const u64 *w, size_t n) {
    const size_t padded = (n + 1 + 9) / 10 * 10;
    u64 s[16] = {};
    for (size_t c0 = 0; c0 < padded; c0 += 10) {
      for (size_t k = 0; k < 10; k++) {
        const size_t j = c0 + k;
        s[k] = j < n ? to_mont(w[j]) : (j == n ? MONT_ONE : 0);
      }
      permutation(s, hash_trace::SECTION_PROGRAM_HASH, HASH);
    }
    for (int k = 0; k < 5; k++) ex.digest[k] = from_mont(s[k]);
    ex.table_heights[0] = padded;
  }

  // hash / merkle_step: Tip5 in fixed-length mode on 10 words (capacity of ones), digest = first five words
  void hash10(const u64 (&words)[10], u64 (&out)[5]) {
    u64 s[16];
    for (int k = 0; k < 10; k++) s[k] = to_mont(words[k]);
    for (int k = 10; k < 16; k++) s[k] = MONT_ONE;
    permutation(s, hash_trace::SECTION_HASH, HASH);
    for (int k = 0; k < 5; k++) out[k] = from_mont(s[k]);
  }

  void merkle_step(const u64 (&sibling)[5]) {     // vm.rs:1026-1062
    need_u32(5);
    const u64 node_index = st(5);
    u64 acc[5];
    for (int k = 0; k < 5; k++) acc[k] = pop();
    u64 words[10], out[5];
    const bool left = node_index % 2 == 0;
    for (int k = 0; k < 5; k++) { words[k] = left ? acc[k] : sibling[k]; words[5 + k] = left ? sibling[k] : acc[k]; }
    hash10(words, out);
    for (int k = 4; k >= 0; k--) push(out[k]);
    st_ref(5) = node_index / 2;
    u32_call(SPLIT, node_index, node_index / 2);
  }

  void horner_step(const X3 &coefficient) {          // vm.rs:1064-1111
    const X3 x{{st(0), st(1), st(2)}}, acc0{{st(7), st(8), st(9)}};
    const X3 acc = xaddc(xmulc(acc0, x), coefficient);
    for (int k = 0; k < 3; k++) st_ref(7 + k) = acc.c[k];
  }

  void check_heights() {
    const uint64_t hash = ex.hash_rows[0] + ex.hash_rows[1] + ex.hash_rows[2];
    const uint64_t h = std::max({(uint64_t)ex.processor_trace.size() / 39, (uint64_t)ex.op_stack_trace.size() / 4,
                                 (uint64_t)ex.ram_trace.size() / 7, hash, u32_height});
    if (h > VM_MAX_TABLE_HEIGHT) {
      char buf[200];
      snprintf(buf, sizeof buf, "a table of the execution passes 2^26 rows, the largest height that can be proved (clk %llu, ip %llu)",
               (unsigned long long)clk, (unsigned long long)ip);
      throw DomainError{buf};
    }
  }

  // executes the instruction at `ip`; true once the VM halts
  bool step() {
    if (ip >= prog.size()) fail("InstructionPointerOverflow");
    const Instr &in = prog[ip];
    const unsigned op = in.op;
    const u64 arg = in.arg;
    const size_t nxt = ip + (in.has_arg ? 2 : 1);
    const u64 nia = in.has_arg ? arg : (nxt < prog.size() ? (u64)prog[nxt].op : 1);     // vm.rs:1178-1189
    u64 hv[6] = {};                                                                     // vm.rs:270-345
    switch (op) {
      case POP: case DIVINE: case PICK: case PLACE: case DUP: case SWAP: case READ_MEM: case WRITE_MEM: case READ_IO: case WRITE_IO:
        for (int k = 0; k < 4; k++) hv[k] = (arg >> k) & 1;
        break;
      case SKIZ:
        hv[0] = inv_or_zero(st(0));
        hv[1] = nia % 2; hv[2] = (nia >> 1) % 4; hv[3] = (nia >> 3) % 4; hv[4] = (nia >> 5) % 4; hv[5] = nia >> 7;
        break;
      case RECURSE_OR_RETURN: hv[0] = inv_or_zero(fsub(st(6), st(5))); break;
      case SPLIT:
        if (st(0) & U32_MAX) hv[0] = inv_or_zero(fsub(st(0) >> 32, U32_MAX));
        break;
      case EQ: hv[0] = inv_or_zero(fsub(st(1), st(0))); break;
      case SPONGE_ABSORB_MEM:
        for (int k = 0; k < 6; k++) hv[k] = ram_get(fadd(st(0), 4 + k));
        break;
      case MERKLE_STEP:
        if (digest_pos < num_digests) for (int k = 0; k < 5; k++) hv[k] = digests[5 * digest_pos + k];
        hv[5] = st(5) % 2;
        break;
      case MERKLE_STEP_MEM:
        for (int k = 0; k < 5; k++) hv[k] = ram_get(fadd(st(7), k));
        hv[5] = st(5) % 2;
        break;
      case B_HORNER_STEP: hv[0] = ram_get(st(5)); break;
      case X_HORNER_STEP:
        hv[2] = ram_get(st(5)); hv[1] = ram_get(fsub(st(5), 1)); hv[0] = ram_get(fsub(st(5), 2));
        break;
      default: break;
    }
    {   // processor row (aet.rs:55, vm.rs:1113-1190)
      const auto &js = jump_stack;
      u64 row[39];
      row[0] = clk; row[1] = 0; row[2] = ip; row[3] = op; row[4] = nia;
      for (int b = 0; b < 7; b++) row[5 + b] = (op >> b) & 1;
      row[12] = js.size(); row[13] = js.empty() ? 0 : js.back().first; row[14] = js.empty() ? 0 : js.back().second;
      for (int k = 0; k < 16; k++) row[15 + k] = st(k);
      row[31] = stack.size();
      for (int k = 0; k < 6; k++) row[32 + k] = hv[k];
      row[38] = 0;
      ex.processor_trace.insert(ex.processor_trace.end(), row, row + 39);
    }
    ex.instruction_multiplicities[ip]++;
    io.clear();
    bool halting = false;
    u64 ip_after = nxt;
    switch (op) {
      case HALT: halting = true; break;
      case NOP: break;
      case PUSH: push(arg); break;
      case POP: for (u64 k = 0; k < arg; k++) pop(); break;
      case DIVINE:
        if (secret.size() - secret_pos < arg) fail("EmptySecretInput");
        for (u64 k = 0; k < arg; k++) push(secret[secret_pos++]);
        break;
      case PICK: {
        io.push_back({false, underflow()});
        const size_t at = stack.size() - 1 - arg;
        const u64 e = stack[at];
        stack.erase(stack.begin() + at);
        push(e);
        break;
      }
      case PLACE: {
        const u64 e = pop();
        stack.insert(stack.end() - arg, e);
        io.push_back({true, underflow()});
        break;
      }
      case DUP: push(st(arg)); break;
      case SWAP: std::swap(st_ref(0), st_ref(arg)); break;
      case SKIZ:
        if (pop() == 0) {
          if (nxt >= prog.size()) fail("InstructionPointerOverflow");
          ip_after = nxt + (prog[nxt].has_arg ? 2 : 1);
        }
        break;
      case CALL: jump_stack.push_back({ip + 2, arg}); ip_after = arg; break;
      case RETURN:
        if (jump_stack.empty()) fail("JumpStackIsEmpty");
        ip_after = jump_stack.back().first;
        jump_stack.pop_back();
        break;
      case RECURSE:
        if (jump_stack.empty()) fail("JumpStackIsEmpty");
        ip_after = jump_stack.back().second;
        break;
      case RECURSE_OR_RETURN:
        if (jump_stack.empty()) fail("JumpStackIsEmpty");
        if (st(5) == st(6)) { ip_after = jump_stack.back().first; jump_stack.pop_back(); }
        else ip_after = jump_stack.back().second;
        break;
      case ASSERT:
        if (st(0) != 1) fail("AssertionFailed");
        pop();
        break;
      case READ_MEM: {
        u64 p = pop();
        for (u64 k = 0; k < arg; k++) { push(ram_read(p)); p = fsub(p, 1); }
        push(p);
        break;
      }
      case WRITE_MEM: {
        u64 p = pop();
        for (u64 k = 0; k < arg; k++) { const u64 v = pop(); ram_write(p, v); p = fadd(p, 1); }
        push(p);
        break;
      }
      case HASH: {
        u64 words[10], out[5];
        for (int k = 0; k < 10; k++) words[k] = pop();
        hash10(words, out);
        for (int k = 4; k >= 0; k--) push(out[k]);
        break;
      }
      case ASSERT_VECTOR:
        for (int k = 0; k < 5; k++) if (st(k) != st(k + 5)) fail("VectorAssertionFailed");
        for (int k = 0; k < 5; k++) pop();
        break;
      case SPONGE_INIT: {
        for (auto &w : sponge) w = 0;
        sponge_ok = true;
        ex.perm_states.insert(ex.perm_states.end(), sponge, sponge + 16);
        ex.perm_meta.push_back(hash_trace::meta_encode(ex.hash_rows[1], SPONGE_INIT, hash_trace::SECTION_SPONGE, true));
        ex.hash_rows[1] += 1;
        break;
      }
      case SPONGE_ABSORB:
        if (!sponge_ok) fail("SpongeNotInitialized");
        for (int k = 0; k < 10; k++) sponge[k] = to_mont(pop());
        permutation(sponge, hash_trace::SECTION_SPONGE, SPONGE_ABSORB);
        break;
      case SPONGE_ABSORB_MEM: {                        // vm.rs:699-729: st1..st4 receive the first four absorbed words
        if (!sponge_ok) fail("SpongeNotInitialized");
        u64 p = pop();
        for (int k = 0; k < 10; k++) {
          const u64 v = ram_read(p);
          sponge[k] = to_mont(v);
          p = fadd(p, 1);
          if (k < 4) st_ref(k) = v;
        }
        push(p);
        permutation(sponge, hash_trace::SECTION_SPONGE, SPONGE_ABSORB);
        break;
      }
      case SPONGE_SQUEEZE:
        if (!sponge_ok) fail("SpongeNotInitialized");
        for (int k = 9; k >= 0; k--) push(from_mont(sponge[k]));
        permutation(sponge, hash_trace::SECTION_SPONGE, SPONGE_SQUEEZE);
        break;
      case MERKLE_STEP: {
        if (digest_pos >= num_digests) fail("EmptySecretDigestInput");
        u64 sibling[5];
        for (int k = 0; k < 5; k++) sibling[k] = digests[5 * digest_pos + k];
        digest_pos++;
        merkle_step(sibling);
        break;
      }
      case MERKLE_STEP_MEM: {
        need_u32(5);
        u64 p = st(7), sibling[5];
        for (int k = 0; k < 5; k++) { sibling[k] = ram_read(p); p = fadd(p, 1); }
        st_ref(7) = p;
        merkle_step(sibling);
        break;
      }
      case B_HORNER_STEP: {
        const u64 p = st(5);
        const u64 c0 = ram_read(p);
        st_ref(5) = fsub(p, 1);
        horner_step(X3{{c0, 0, 0}});
        break;
      }
      case X_HORNER_STEP: {
        const u64 p = st(5);
        const u64 c2 = ram_read(p), c1 = ram_read(fsub(p, 1)), c0 = ram_read(fsub(p, 2));
        st_ref(5) = fsub(p, 3);
        horner_step(X3{{c0, c1, c2}});
        break;
      }
      case ADD: { const u64 x = pop(), y = pop(); push(fadd(x, y)); break; }
      case ADDI: st_ref(0) = fadd(st(0), arg); break;
      case MUL: { const u64 x = pop(), y = pop(); push(mulc(x, y)); break; }
      case INVERT:
        if (st(0) == 0) fail("InverseOfZero");
        push(invc(pop()));
        break;
      case EQ: { const u64 x = pop(), y = pop(); push(x == y ? 1 : 0); break; }
      case SPLIT: {
        const u64 top = pop(), lo = top & U32_MAX, hi = top >> 32;
        push(hi); push(lo);
        u32_call(SPLIT, lo, hi);
        break;
      }
      case LT: {
        need_u32(0); need_u32(1);
        const u64 lhs = pop(), rhs = pop();
        push(lhs < rhs ? 1 : 0);
        u32_call(LT, lhs, rhs);
        break;
      }
      case AND: case XOR: {                            // a ^ b = a + b - 2 (a & b): `xor` is looked up as `and` (vm.rs:860-865)
        need_u32(0); need_u32(1);
        const u64 lhs = pop(), rhs = pop();
        push(op == AND ? (lhs & rhs) : (lhs ^ rhs));
        u32_call(AND, lhs, rhs);
        break;
      }
      case LOG_2_FLOOR: {
        need_u32(0);
        if (st(0) == 0) fail("LogarithmOfZero");
        const u64 top = pop();
        push(bit_length(top) - 1);
        u32_call(LOG_2_FLOOR, top, 0);
        break;
      }
      case POW: {
        need_u32(1);
        const u64 base = pop(), exponent = pop();
        push(powc(base, exponent));
        u32_call(POW, base, exponent);
        break;
      }
      case DIV_MOD: {
        need_u32(0); need_u32(1);
        if (st(1) == 0) fail("DivisionByZero");
        const u64 num = pop(), den = pop(), quot = num / den, rem = num % den;
        push(quot); push(rem);
        u32_call(LT, rem, den);
        u32_call(SPLIT, num, quot);
        break;
      }
      case POP_COUNT: {
        need_u32(0);
        const u64 top = pop();
        push((u64)__builtin_popcountll(top));
        u32_call(POP_COUNT, top, 0);
        break;
      }
      case XX_ADD: { const X3 x = pop_x(), y = pop_x(); push_x(xaddc(x, y)); break; }
      case XX_MUL: { const X3 x = pop_x(), y = pop_x(); push_x(xmulc(x, y)); break; }
      case X_INVERT: {
        if ((st(0) | st(1) | st(2)) == 0) fail("InverseOfZero");
        const X3 x = pop_x();
        push_x(xc(xinv(xm(x))));
        break;
      }
      case XB_MUL: { const u64 x = pop(); const X3 y = pop_x(); push_x(xmulc(X3{{x, 0, 0}}, y)); break; }
      case READ_IO:
        if (input.size() - input_pos < arg) fail("EmptyPublicInput");
        for (u64 k = 0; k < arg; k++) push(input[input_pos++]);
        break;
      case WRITE_IO: for (u64 k = 0; k < arg; k++) ex.output.push_back(pop()); break;
      default: fail("InvalidOpcode");                // unreachable: decode admits the 46 opcodes only
    }
    // the op-stack underflow IO of this instruction, canonicalised (op_stack.rs:61-87) and turned into table rows (234-255)
    for (bool changed = true; changed;) {
      changed = false;
      for (size_t k = 0; k + 1 < io.size(); k++)
        if (io[k].first != io[k + 1].first && io[k].second == io[k + 1].second) {
          io.erase(io.begin() + k, io.begin() + k + 2);
          changed = true;
          break;
        }
    }
    if (!io.empty()) {
      u64 p = io[0].first ? stack.size() - io.size() : stack.size() + io.size();
      for (const auto &e : io) {
        if (!e.first) p--;
        const u64 row[4] = {clk, e.first ? 0ULL : 1ULL, p, e.second};
        ex.op_stack_trace.insert(ex.op_stack_trace.end(), row, row + 4);
        if (e.first) p++;
      }
    }
    ip = ip_after;
    clk++;
    check_heights();
    return halting;
  }

  void run(const VmInputs &in) {
    ex.program.assign(in.program, in.program + in.program_len);
    ex.instruction_multiplicities.assign(in.program_len, 0);
    ex.input.assign(in.public_input, in.public_input + in.num_input);
    input = ex.input;
    secret.assign(in.secret_input, in.secret_input + in.num_secret);
    digests = in.digests;
    num_digests = in.num_digests;
    for (size_t i = 0; i < in.num_ram; i++) ram[in.ram_addresses[i]] = in.ram_values[i];
    decode(in.program, in.program_len);
    hash_program(in.program, in.program_len);
    stack.assign(16, 0);                              // OpStack::new: the reversed program digest at the bottom
    for (int k = 0; k < 5; k++) stack[k] = ex.digest[4 - k];
    while (!step()) {
    }
    const uint64_t rows = ex.processor_trace.size() / 39;
    const uint64_t h[9] = {ex.table_heights[0], rows, ex.op_stack_trace.size() / 4, ex.ram_trace.size() / 7, rows,
                           ex.hash_rows[0] + ex.hash_rows[1] + ex.hash_rows[2], ex.cascade_multiplicities.size() / 2, 256, u32_height};
    uint64_t m = 0;
    for (int i = 0; i < 9; i++) { ex.table_heights[i] = h[i]; m = std::max(m, h[i]); }
    ex.padded_height = 1;
    while (ex.padded_height < m) ex.padded_height <<= 1;
  }
};

}  // namespace

int trace_execution(const VmInputs &in, tvm_execution &ex, std::string &failure) {
  Vm vm(ex);
  try {
    vm.run(in);
  } catch (const VmError &e) {
    failure = e.text;
    return TVM_ERR_VM;
  } catch (const DomainError &e) {
    failure = e.text;
    return TVM_ERR_DOMAIN;
  }
  return TVM_OK;
}

}  // namespace tvm
