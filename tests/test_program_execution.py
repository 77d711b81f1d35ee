"""VM::trace_execution in the library (tvm_trace_execution, csrc/vm.cu; host code, no GPU) against the oracle's VM
(oracle/tracegen.execute + aet_arrays), which the reference's whole-proof known-answer tests pin: every array of the AET except
the three hash traces, the output, the program digest, the table heights and the padded height, word for word.  The hash
traces are expanded from the recorded permutation inputs by fill/hash_trace.cuh; its stage body runs here under the sequential
host executor of tests/host/hash_trace_host.cu on the oracle's permutation inputs.  The GPU runs of the same expansion, and
proofs from (program, inputs, seed) alone, are tests/test_zzzz_gpu_program.py."""
import ctypes
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "triton-vm_b200"), os.path.join(ROOT, "triton-vm_b200", "py"), os.path.dirname(os.path.abspath(__file__))]
from oracle import tip5, tracegen as tg   # noqa: E402
import tvm_b200                           # noqa: E402
import test_golden as TG                  # noqa: E402
import test_vm_programs as tvp            # noqa: E402
from test_main_fill_host import _program as fill_program   # noqa: E402

P = tg.P
SRC = os.path.join(ROOT, "tests", "host", "hash_trace_host.cu")
SO = os.path.join(ROOT, "tests", "host", "_build", "libhash_trace_host.so")
HDRS = [os.path.join(ROOT, "triton-vm_b200", "csrc", f) for f in ("fill/hash_trace.cuh", "fill/main_fill.cuh", "tip5.cuh", "field.cuh")]
HASH_KEYS = ("program_hash_trace", "sponge_trace", "hash_trace")


def every_instruction_inputs():
    """the inputs of stark.rs:2433-2460 as test_golden.every_instruction_instance builds them: public input = Merkle node [5; 5],
    secret input = reversed root ++ [1337; 10], one secret digest [4; 5], RAM = {i: 42 + i} and node [3; 5] at 100000"""
    n5, n4, n3 = [5] * 5, [4] * 5, [3] * 5
    n2 = [int(v) for v in tip5.hash_pair(n4, n5)]
    n1 = [int(v) for v in tip5.hash_pair(n2, n3)]
    ram = {i: 42 + i for i in range(1000)}
    ram.update({100000 + k: v for k, v in enumerate(n3)})
    return n5, list(reversed(n1)) + [1337] * 10, ram, [n4]


def program(name):
    """-> (words, public input, secret input, RAM, digests)"""
    if name == "kitchen_sink":
        return tg.assemble(tvp.KITCHEN_SINK), tvp.SINK_INPUT, tvp.SINK_SECRET, None, []
    if name == "memory_and_merkle":
        return tg.assemble(tvp.MEMORY_AND_MERKLE), [], [], tvp.MEM_RAM, [tvp.MEM_SIBLING]
    if name == "every_instruction":
        inp, sec, ram, digests = every_instruction_inputs()
        return tg.assemble(TG.EVERY_INSTRUCTION_PROGRAM), inp, sec, ram, digests
    words, inp, ram = fill_program(name)
    return list(words), inp, [], ram, []


PROGRAMS = ["halt", "fib_100", "spin_9", "kitchen_sink", "memory_and_merkle", "every_instruction", "u32_mix", "verifier_3", "verifier_40"]


def run_both(name):
    words, inp, sec, ram, digests = program(name)
    ex = tvm_b200.trace_execution(words, inp, sec, digests, ram)
    want = tg.execute(list(words), inp, sec, ram, digests)
    return words, ex, want


@pytest.mark.parametrize("name", PROGRAMS)
def test_execution_matches_the_oracle(name):
    words, ex, want = run_both(name)
    got = ex.aet()
    arrays = tg.aet_arrays(list(words), want)
    assert set(got) == set(arrays)
    for key, w in arrays.items():
        if key in HASH_KEYS:
            assert got[key] is None or len(w) == 0         # not expanded without a device
            continue
        assert got[key].dtype == w.dtype and got[key].shape == w.shape, key
        assert np.array_equal(got[key], w), key
    assert ex.output == want.output and ex.program_digest == want.digest
    assert ex.table_heights == tg.table_heights(list(words), want)
    _, inp, sec, ram, digests = program(name)
    assert ex.padded_height == tg.padded_height(list(words), inp, sec, ram, digests)
    assert ex.claim == (want.digest, list(inp), want.output)
    ex.close()


# ---- the expansion's stage body on the host ---------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def host():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    stale = not os.path.exists(SO) or any(os.path.getmtime(f) > os.path.getmtime(SO) for f in [SRC] + HDRS)
    if stale:
        if not os.path.exists(nvcc):
            pytest.skip("nvcc not available to build the host harness")
        os.makedirs(os.path.dirname(SO), exist_ok=True)
        subprocess.run([nvcc, "-O2", "-std=c++17", "--extended-lambda", "--expt-relaxed-constexpr", "-shared", "-Xcompiler", "-fPIC",
                        SRC, "-o", SO], check=True, capture_output=True)
    return ctypes.CDLL(SO)


def oracle_permutations(words, ex):
    """the oracle's permutation inputs in the order the VM records them: (state, section, CI, single row)"""
    recs = [(t[0], 0, tg.OP_HASH, 0) for t in tg._program_hash(list(words))[2]]
    i, rows = 0, ex.sponge_rows
    while i < len(rows):
        ci, _, st = rows[i]
        single = ci == tg.OPCODES["sponge_init"]
        recs.append((st, 1, ci, int(single)))
        i += 1 if single else 6
    recs += [(t[0], 2, tg.OP_HASH, 0) for t in ex.hash_traces]
    return recs


def host_expand(lib, recs):
    vp = ctypes.c_void_p
    states = np.array([r[0] for r in recs], dtype=np.uint64).reshape(-1, 16)
    section, ci, single = (np.array([r[k] for r in recs], dtype=np.uint32) for k in (1, 2, 3))
    rows = np.zeros(3, dtype=np.uint64)
    args = [states.ctypes.data_as(vp), section.ctypes.data_as(vp), ci.ctypes.data_as(vp), single.ctypes.data_as(vp), ctypes.c_size_t(len(recs)),
            rows.ctypes.data_as(vp)]
    lib.hash_trace_host_expand(*args, None, None, None)
    out = [np.zeros((int(r), 67), dtype=np.uint64) for r in rows]
    lib.hash_trace_host_expand(*args, *[o.ctypes.data_as(vp) for o in out])
    return dict(zip(HASH_KEYS, out))


@pytest.mark.parametrize("name", PROGRAMS)
def test_hash_trace_expansion_matches_the_oracle(host, name):
    words, inp, sec, ram, digests = program(name)
    want = tg.execute(list(words), inp, sec, ram, digests)
    arrays = tg.aet_arrays(list(words), want)
    got = host_expand(host, oracle_permutations(words, want))
    for key in HASH_KEYS:
        assert got[key].shape == arrays[key].shape and np.array_equal(got[key], arrays[key]), key


# ---- failures -----------------------------------------------------------------------------------------------------------------
FAILURES = [
    ("InvalidOpcode", [5], {}),
    ("OutOfRangeOpcode", [1 << 40], {}),
    ("IllegalArgument", [tg.OPCODES["pop"], 7, 0], {}),
    ("IllegalArgument", [tg.OPCODES["dup"], 100, 0], {}),
    ("MissingArgument", [tg.OPCODES["push"]], {}),
    ("InstructionPointerOverflow", "push 1 pop 1", {}),
    ("InstructionPointerOverflow", [], {}),
    ("JumpStackIsEmpty", "return halt", {}),
    ("JumpStackIsEmpty", "recurse halt", {}),
    ("AssertionFailed", "push 0 assert halt", {}),
    ("VectorAssertionFailed", "push 1 assert_vector halt", {}),
    ("InverseOfZero", "push 0 invert halt", {}),
    ("InverseOfZero", "push 0 push 0 push 0 x_invert halt", {}),
    ("DivisionByZero", "push 0 push 5 div_mod halt", {}),
    ("LogarithmOfZero", "push 0 log_2_floor halt", {}),
    ("SpongeNotInitialized", "sponge_squeeze halt", {}),
    ("SpongeNotInitialized", "push 0 push 0 push 0 push 0 push 0 push 0 push 0 push 0 push 0 push 0 sponge_absorb halt", {}),
    ("SpongeNotInitialized", "push 7 sponge_absorb_mem halt", {}),
    ("EmptyPublicInput", "read_io 2 halt", dict(public_input=[1])),
    ("EmptySecretInput", "divine 1 halt", {}),
    ("EmptySecretDigestInput", "merkle_step halt", {}),
    ("TooShallow", "pop 1 halt", {}),
    ("FailedU32Conversion", "push 18446744069414584320 push 1 lt halt", {}),
    ("FailedU32Conversion", "push 1 push 4294967296 div_mod halt", {}),
]


@pytest.mark.parametrize("variant,prog,kw", FAILURES, ids=[f"{v}-{i}" for i, (v, _, _) in enumerate(FAILURES)])
def test_vm_failures_name_the_variant(variant, prog, kw):
    words = tg.assemble(prog) if isinstance(prog, str) else prog
    with pytest.raises(Exception):                           # the oracle rejects the same program
        tg.execute(list(words), kw.get("public_input", ()))
    with pytest.raises(tvm_b200.TvmError) as e:
        tvm_b200.trace_execution(words, **kw)
    assert e.value.code == tvm_b200.TVM_ERR_VM
    assert variant in str(e.value)
    kind = "ProgramDecodingError" if variant in ("InvalidOpcode", "OutOfRangeOpcode", "IllegalArgument", "MissingArgument") else "VMError"
    assert kind in str(e.value)


def test_failure_text_names_clock_cycle_and_instruction_pointer():
    with pytest.raises(tvm_b200.TvmError) as e:
        tvm_b200.trace_execution(tg.assemble("push 2 push 0 assert halt"))
    assert "VMError: AssertionFailed (clk 2, ip 4)" in str(e.value)
    with pytest.raises(tvm_b200.TvmError) as e:
        tvm_b200.trace_execution([tg.OPCODES["nop"]] * 6 + [tg.OPCODES["push"]])
    assert "ProgramDecodingError: MissingArgument(6, push)" in str(e.value)


def test_an_argument_word_executes_its_instruction():
    """program.rs:97: the program is a list of instructions repeated over their argument words — `call 3` lands on the argument
    of `push 7` and executes `push 7`, whose successor is two words further on"""
    words = [tg.OPCODES["call"], 3, tg.OPCODES["push"], 7, tg.OPCODES["nop"], tg.OPCODES["halt"]]
    ex = tvm_b200.trace_execution(words)
    proc = ex.aet()["processor_trace"]
    assert [int(v) for v in proc[:, 2]] == [0, 3, 5] and [int(v) for v in proc[:, 3]] == [49, 1, 0]
    assert int(proc[2, 15]) == 7                             # st0 after `push 7`
    assert [int(v) for v in ex.aet()["instruction_multiplicities"]] == [1, 0, 0, 1, 0, 1]


def _raw_trace(words, inp=(), sec=(), digests=(), ram_addresses=(), ram_values=()):
    """tvm_trace_execution on raw arrays (the RAM may repeat an address); -> return code"""
    arr = [np.array(list(x), dtype=np.uint64) for x in (words, inp, sec, [w for d in digests for w in d], ram_addresses, ram_values)]
    p = [a.ctypes.data_as(tvm_b200._u64p) for a in arr]
    nd = tvm_b200.NondeterminismStruct(p[2], arr[2].size, p[3], len(digests), p[4], p[5], arr[4].size)
    h = ctypes.c_void_p()
    rc = tvm_b200.lib().tvm_trace_execution(p[0], arr[0].size, p[1], arr[1].size, ctypes.byref(nd), ctypes.byref(h), None, 0)
    if rc == 0:
        tvm_b200.lib().tvm_execution_destroy(h)
    return rc


def test_words_outside_the_field_and_repeated_ram_addresses_are_argument_errors():
    halt = [tg.OP_HALT]
    assert _raw_trace(halt, ram_addresses=[1, 2], ram_values=[3, 4]) == 0
    for kw in (dict(words=[P]), dict(words=halt, inp=[P]), dict(words=halt, sec=[P + 5]), dict(words=halt, digests=[[0, 0, 0, 0, P]]),
               dict(words=halt, ram_addresses=[P], ram_values=[0]), dict(words=halt, ram_addresses=[0], ram_values=[(1 << 64) - 1]),
               dict(words=halt, ram_addresses=[7, 8, 7], ram_values=[1, 2, 3])):
        kw.setdefault("words", halt)
        assert _raw_trace(**kw) == -1, kw
    assert tvm_b200.lib().tvm_trace_execution(None, 1, None, 0, None, ctypes.byref(ctypes.c_void_p()), None, 0) == -1


def test_plain_c_program_client_builds_and_fails_loudly_without_a_gpu(tmp_path):
    """examples/prove_program.c under the tests' -pedantic -Werror line; the execution runs on the host, the prove needs a GPU"""
    from test_native_verifier import _build_example
    exe = _build_example(tmp_path, "prove_program")
    r = subprocess.run([exe, "8"], capture_output=True, text=True)
    if tvm_b200.lib().tvm_device_count() == 0:
        assert r.returncode == 3 and "no CPU fallback" in r.stderr
    else:
        assert r.returncode == 0 and "verified" in r.stdout, r.stderr
