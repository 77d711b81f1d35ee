"""The seeded program corpus of tests/program_corpus.py through everything that turns a program into a witness, on the host:
the library's VM (tvm_trace_execution, csrc/vm.cu) against the oracle's VM, the hash-trace expansion's stage body
(fill/hash_trace.cuh) and the table fill's stage bodies (fill/main_fill.cuh) under their sequential host executors against
the oracle's traces and tables, and — the check that does not assume the oracle is right — the oracle's witness, extended
under sampled challenges (two draws for the random programs), against every AIR constraint (`oracle_check`, the C
evaluators tests/test_air.py pins to the reference's constraint circuits).  The device runs of the same corpus are
tests/test_zzzzzzz_gpu_program_corpus.py."""
import contextlib
import ctypes
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

sys.path[:0] = [os.path.dirname(os.path.abspath(__file__))]
import program_corpus as PC                                                    # noqa: E402
from oracle import corc, tracegen as tg                                        # noqa: E402
import tvm_b200                                                                # noqa: E402
from test_air_check import challenges63, oracle_check, sampled_challenges      # noqa: E402
import test_main_fill_host as TMF                                              # noqa: E402
import test_program_execution as TPE                                           # noqa: E402
from test_main_fill_host import host_bezout, host_main_table                    # noqa: E402
from test_program_execution import HASH_KEYS, host_expand, oracle_permutations   # noqa: E402

P = tg.P
CASES = PC.cases()
IDS = [c.name for c in CASES]
TABLES = ("program", "processor", "op_stack", "ram", "jump_stack", "hash", "cascade", "lookup", "u32")
BEZOUT_ORACLE_LIMIT = 300          # tg.bezout_coefficients is cubic in the number of unique RAM pointers


def run_oracle(case):
    return tg.execute(list(case.words), case.public_input, case.secret_input, case.ram, case.digests)


def padded_height(heights):
    return 1 << (max(heights.values()) - 1).bit_length()


def checked_bezout(lib):
    """Bezout coefficients for root sets too large for the oracle's Lagrange interpolation: the host executor's, accepted
    only if a rp + b rp' = 1 holds at three points outside the roots (with deg a < m - 1 and deg b < m, that determines
    a and b)"""
    def bezout(roots):
        a, b, _ = host_bezout(lib, roots, 5)
        assert len(a) == len(b) == len(roots) and a[-1] == 0
        for z in (3, 12345678901234567, P - 2):
            rp, fd = 1, 0
            for r in roots:
                fd = (fd * (z - r) + rp) % P
                rp = rp * (z - r) % P
            ev = lambda poly: sum(c * pow(z, k, P) for k, c in enumerate(poly)) % P       # noqa: E731
            assert (ev(a) * rp + ev(b) * fd) % P == 1
        return a, b
    return bezout


@contextlib.contextmanager
def oracle_bezout(case, ex, lib):
    """tg.main_table with checked_bezout when the case has more unique RAM pointers than the oracle's Bezout handles"""
    if len({c[2] for c in ex.ram_calls}) <= BEZOUT_ORACLE_LIMIT:
        yield
        return
    saved = tg.bezout_coefficients
    tg.bezout_coefficients = checked_bezout(lib)
    try:
        yield
    finally:
        tg.bezout_coefficients = saved


def oracle_main_table(case, ex, n, lib):
    """the oracle's [379, n] main table (derived columns included) and the claim"""
    with oracle_bezout(case, ex, lib):
        T, digest, out = tg.main_table(list(case.words), case.public_input, n, case.secret_input, case.ram, case.digests)
    return np.asarray(T, dtype=np.uint64), (list(digest), list(case.public_input), list(out))


def load_harness(src, so, deps):
    """a host harness of tests/host (the stage bodies under the sequential host executor), built with the line its own
    test module uses when a source is newer than the library; skips the calling test without nvcc"""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(so) or any(os.path.getmtime(f) > os.path.getmtime(so) for f in [src] + list(deps)):
        if not os.path.exists(nvcc):
            pytest.skip("nvcc not available to build the host harness")
        os.makedirs(os.path.dirname(so), exist_ok=True)
        subprocess.run([nvcc, "-O2", "-std=c++17", "--extended-lambda", "--expt-relaxed-constexpr", "-shared", "-Xcompiler", "-fPIC",
                        src, "-o", so], check=True, capture_output=True)
    return ctypes.CDLL(so)


@pytest.fixture(scope="module")
def fill_host():
    return load_harness(TMF.SRC, TMF.SO, [TMF.HDR])


@pytest.fixture(scope="module")
def hash_host():
    return load_harness(TPE.SRC, TPE.SO, TPE.HDRS)


def challenge_seeds(case):
    return (5, 6) if case.name.startswith("random") else (5,)


# ---- 1. the VM -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_vm_matches_the_oracle(case):
    """what test_program_execution.test_execution_matches_the_oracle compares: every AET array but the hash traces (not
    expanded without a device), the output, the digest, the table heights, the padded height and the claim"""
    ex = tvm_b200.trace_execution(case.words, case.public_input, case.secret_input, case.digests, case.ram)
    want = run_oracle(case)
    got, arrays = ex.aet(), tg.aet_arrays(list(case.words), want)
    assert set(got) == set(arrays)
    for key, w in arrays.items():
        if key in HASH_KEYS:
            assert got[key] is None or len(w) == 0
            continue
        assert got[key].dtype == w.dtype and got[key].shape == w.shape, key
        assert np.array_equal(got[key], w), key
    assert ex.output == want.output and ex.program_digest == want.digest
    heights = tg.table_heights(list(case.words), want)
    assert ex.table_heights == heights
    assert ex.padded_height == padded_height(heights)           # tg.padded_height without a second run of the oracle's VM
    assert ex.claim == (want.digest, list(case.public_input), want.output)
    ex.close()


# ---- 2. the hash traces --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_hash_traces_match_the_oracle(hash_host, case):
    want = run_oracle(case)
    arrays = tg.aet_arrays(list(case.words), want)
    got = host_expand(hash_host, oracle_permutations(case.words, want))
    for key in HASH_KEYS:
        assert got[key].shape == arrays[key].shape and np.array_equal(got[key], arrays[key]), key


# ---- 3 + 4. the table fill, and the AIR on the oracle's witness ----------------------------------------------------------------
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_tables_match_the_oracle_and_satisfy_the_air(fill_host, case):
    ex = run_oracle(case)
    heights = tg.table_heights(list(case.words), ex)
    n = max(256, padded_height(heights))
    main, claim = oracle_main_table(case, ex, n, fill_host)
    got, lengths = host_main_table(fill_host, tg.aet_arrays(list(case.words), ex), n)
    bad = [c for c in range(149) if not np.array_equal(got[c], main[c])]
    assert not bad, [tg.column_name(True, c) for c in bad[:8]]
    assert lengths == [heights[k] for k in TABLES]
    for seed in challenge_seeds(case):
        ch = challenges63(sampled_challenges(seed), claim)
        counts, first, last = oracle_check(main, corc.aux_extend(main, ch), ch)
        info = tvm_b200.air_constraint_info()
        violated = [(info[j]["origin"], info[j]["category"], info[j]["index_in_category"], int(first[j])) for j in np.nonzero(counts)[0]]
        assert not violated, f"challenge seed {seed}: (table, category, index, first row) {violated[:8]}"


# ---- the shapes the shape cases are named for ----------------------------------------------------------------------------------
def test_shape_cases_have_their_shapes():
    h = {c.name: tg.table_heights(list(c.words), run_oracle(c)) for c in CASES if c.name.startswith("shape")}
    u32 = h["shape-u32-dominated"]
    assert u32["u32"] >= 1 << 14 and u32["u32"] == max(u32.values())
    exact = h["shape-u32-exactly-2^12"]
    assert exact["u32"] == 1 << 12 == padded_height(exact)
    ram = h["shape-ram-dominated"]
    assert ram["ram"] == max(ram.values())
    assert len({c[2] for c in run_oracle(PC.by_name("shape-ram-dominated")).ram_calls}) > 1 << 13
    hsh = h["shape-hash-dominated"]
    assert hsh["hash"] > max(hsh[k] for k in ("processor", "op_stack", "ram", "u32", "program"))
    ops = h["shape-op-stack-dominated"]
    assert ops["op_stack"] == max(ops.values())
    proc = h["shape-processor-exactly-2^13"]
    assert proc["processor"] == proc["jump_stack"] == 1 << 13 == padded_height(proc)
    ex = run_oracle(PC.by_name("shape-processor-exactly-2^13"))
    assert max(r["jsp"] for r in ex.rows) >= 1000
    assert max(r["osp"] for r in run_oracle(PC.by_name("shape-op-stack-dominated")).rows) >= 2000


# ---- 5. coverage --------------------------------------------------------------------------------------------------------------
def test_every_instruction_runs_on_an_edge_operand():
    """every one of the 46 instructions executes in an edge case (a case that is neither random nor a shape case), and
    the u32 table entries and RAM pointers the edge cases are written for are recorded"""
    executed, u32, pointers = set(), set(), set()
    for c in CASES:
        if c.name.startswith(("random", "shape")):
            continue
        ex = run_oracle(c)
        executed |= {tg._NAME[r["ci"]] for r in ex.rows}
        u32 |= set(ex.u32_entries)
        pointers |= {call[2] for call in ex.ram_calls}
    assert executed == set(tg.OPCODES), sorted(set(tg.OPCODES) - executed)
    U = PC.U32
    for entry in [("split", 0, U), ("split", U, 0), ("split", 0, 1), ("lt", U, 0), ("lt", 0, U), ("lt", U, U), ("lt", 0, 0),
                  ("and", U, U), ("and", 0xAAAAAAAA, 0x55555555), ("log_2_floor", U, 0), ("log_2_floor", 1, 0), ("pop_count", U, 0),
                  ("pop_count", 0, 0), ("pow", P - 1, U), ("pow", U, 1 << 31), ("pow", 0, 0), ("lt", 0, U),
                  ("split", U, 1), ("split", U, U // 7)]:
        assert entry in u32, entry
    assert {0, 1, 2, 3, P - 1, P - 2, P - 3, P - 5} <= pointers
