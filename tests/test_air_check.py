"""The AIR constraint checker (check_constraints_fn!, stark.rs:2899-3015) without a GPU: the constraint metadata of
tvm_air_constraint_info against the reference's constraint counts, the built generated sources against a fresh generator run, and the generated chunk
bodies of csrc/air_check_gen/ run by the sequential host recorder of tests/host/air_check_host.cu against `oracle_check`
(tests/host/air_check_oracle.c: an OpenMP loop over the oracle's generated `orc_air_eval_*` evaluators, which tests/test_air.py
pins to the reference) on all 604 (count, first row, last row) triples.  The device runs of the same cases are tests/test_zzzzzz_gpu_air_check.py."""
import collections
import ctypes
import filecmp
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "triton-vm_b200"), os.path.join(ROOT, "triton-vm_b200", "py"), os.path.dirname(os.path.abspath(__file__))]
from oracle import corc, stark as S, tracegen as tg   # noqa: E402
import tvm_b200                                         # noqa: E402
import test_program_execution as tpe                    # noqa: E402

P = tg.P
GEN = os.path.join(ROOT, "triton-vm_b200", "csrc", "air_check_gen")
SRC = os.path.join(ROOT, "tests", "host", "air_check_host.cu")
SO = os.path.join(ROOT, "tests", "host", "_build", "libair_check_host.so")
ORACLE_SRC = os.path.join(ROOT, "tests", "host", "air_check_oracle.c")
ORACLE_SO = os.path.join(ROOT, "tests", "host", "_build", "libair_check_oracle.so")
ORACLE_DEPS = [ORACLE_SRC] + [os.path.join(ROOT, "oracle", "c", f) for f in ("air_eval_gen.c", "field_inline.h")]
HDRS = [os.path.join(ROOT, "triton-vm_b200", "csrc", f) for f in ("air_check.cuh", "field.cuh")] + \
    [os.path.join(GEN, f) for f in ("air_check_bodies.cuh", "air_check_meta.inc")]
CATS = ("init", "cons", "tran", "term")
TABLES = ["ProgramTable", "ProcessorTable", "OpStackTable", "RamTable", "JumpStackTable", "HashTable", "CascadeTable", "LookupTable",
          "U32Table", "GrandCrossTableArg"]
# specification/src/arithmetization-overview.md, "Before automatic degree lowering": init / cons / tran / term per table
BEFORE = {"ProgramTable": (6, 5, 10, 2), "ProcessorTable": (29, 10, 42, 1), "OpStackTable": (3, 1, 5, 0), "RamTable": (7, 1, 12, 1),
          "JumpStackTable": (6, 0, 6, 0), "HashTable": (22, 45, 48, 2), "CascadeTable": (2, 1, 3, 0), "LookupTable": (3, 1, 4, 1),
          "U32Table": (1, 15, 22, 2), "GrandCrossTableArg": (0, 0, 0, 14)}
AFTER_TOTAL = (81, 97, 403, 23)
DERIVED = 160      # a derived main column of a consistency substitution: defined on every row
PROGRAMS = ["halt", "fib_100", "spin_9", "kitchen_sink", "memory_and_merkle", "every_instruction", "u32_mix"]


# ---- metadata --------------------------------------------------------------------------------------------------------
def test_constraint_counts_per_category_and_origin():
    info = tvm_b200.air_constraint_info()
    assert [i["index"] for i in info] == list(range(604))
    per_cat = collections.Counter(i["category"] for i in info)
    assert tuple(per_cat[c] for c in CATS) == AFTER_TOTAL
    for c in CATS:   # evaluator order: the categories in turn, indices within a category consecutive
        assert [i["index_in_category"] for i in info if i["category"] == c] == list(range(per_cat[c]))
    for t in TABLES:
        for k, c in enumerate(CATS):
            idx = sorted(i["origin_index"] for i in info if i["origin"] == t and i["category"] == c)
            assert idx == list(range(BEFORE[t][k])), (t, c)      # each original constraint exactly once, positions 0..count-1
            assert all(i["derived_column"] is None for i in info if i["origin"] == t)
    assert {i["origin_id"]: i["origin"] for i in info} == dict(enumerate(TABLES + ["DegreeLowering"]))


def test_substitution_constraints_define_every_derived_column_once():
    info = tvm_b200.air_constraint_info()
    sub = [i for i in info if i["origin"] == "DegreeLowering"]
    for k, c in enumerate(CATS):
        assert sum(1 for i in sub if i["category"] == c) == AFTER_TOTAL[k] - sum(b[k] for b in BEFORE.values())
    assert all(i["derived_column"] == (("main" if i["origin_index"] >= 149 else "aux"), i["origin_index"]) for i in sub)
    assert sorted(i["origin_index"] for i in sub if i["derived_column"][0] == "main") == list(range(149, 379))
    assert sorted(i["origin_index"] for i in sub if i["derived_column"][0] == "aux") == list(range(49, 90))


def test_degrees_equal_the_quotient_metadata():
    meta = open(os.path.join(ROOT, "triton-vm_b200", "csrc", "air_gen", "air_meta.inc")).read()
    degs = []
    for c in CATS:
        line = next(l for l in meta.splitlines() if l.startswith(f"static const unsigned char AIR_DEGREES_{c.upper()}[]"))
        degs += [int(v) for v in line.split("{")[1].split("}")[0].split(",")]
    assert [i["degree"] for i in tvm_b200.air_constraint_info()] == degs


def test_constraint_info_argument_errors():
    l = tvm_b200.lib()
    c = tvm_b200.AirConstraintStruct()
    assert l.tvm_air_constraint_info(604, ctypes.byref(c)) == -1
    assert l.tvm_air_constraint_info(0, None) == -1
    out = [(ctypes.c_uint64 * 604)() for _ in range(3)]
    nv = ctypes.c_uint64()
    ch = np.zeros(189, dtype=np.uint64)
    t = np.zeros(4, dtype=np.uint64)
    pt = t.ctypes.data_as(tvm_b200._u64p)
    assert l.tvm_air_check(None, pt, pt, 1, ch.ctypes.data_as(tvm_b200._u64p), *out, ctypes.byref(nv)) == -1
    assert l.tvm_air_check_aet(None, None, None, 256, ch.ctypes.data_as(tvm_b200._u64p), *out, ctypes.byref(nv)) == -1
    assert l.tvm_air_check_execution(None, None, ch.ctypes.data_as(tvm_b200._u64p), *out, ctypes.byref(nv)) == -1


def test_generated_sources_are_fresh(tmp_path):
    subprocess.run([sys.executable, "-m", "airgen.codegen_check", str(tmp_path)], cwd=os.path.join(ROOT, "triton-vm_b200"), check=True,
                   capture_output=True)
    names = sorted(os.listdir(tmp_path))
    assert names == sorted(os.listdir(GEN))
    for f in names:
        assert filecmp.cmp(os.path.join(tmp_path, f), os.path.join(GEN, f), shallow=False), f


# ---- cases: valid and corrupted witnesses -----------------------------------------------------------------------------
def sampled_challenges(seed=5):
    return np.random.default_rng(seed).integers(0, P, size=(59, 3), dtype=np.uint64)


def challenges63(sampled, claim):
    return np.array(S.derive_challenges([tuple(int(v) for v in r) for r in sampled], S.Claim(*claim)), dtype=np.uint64)


_TABLES = {}


def program_tables(name):
    """oracle tables of a program at its padded height -> (main [379, n], aux [91, n, 3], challenges [63, 3], claim, sampled)"""
    if name not in _TABLES:
        words, inp, sec, ram, digests = tpe.program(name)
        ph = tg.padded_height(list(words), inp, sec, ram, digests)
        T, digest, out = tg.main_table(list(words), inp, ph, sec, ram, digests)
        main = np.array(T, dtype=np.uint64)
        claim = (list(digest), list(inp), list(out))
        sampled = sampled_challenges()
        ch = challenges63(sampled, claim)
        _TABLES[name] = (main, corc.aux_extend(main, ch), ch, claim, sampled)
    return _TABLES[name]


def corrupt_cases(main, aux):
    """(label, main, aux): one cell changed in each of the nine tables' main columns, in a derived main column and in an aux
    column, at row 0, a middle row and row n - 1; and two processor rows swapped"""
    from airgen.columns import MAIN
    n = main.shape[1]
    cols = [getattr(MAIN["program"], "Address"), getattr(MAIN["processor"], "ST0"), getattr(MAIN["op_stack"], "StackPointer"),
            getattr(MAIN["ram"], "RamValue"), getattr(MAIN["jump_stack"], "JSP"), getattr(MAIN["hash"], "State5"),
            getattr(MAIN["cascade"], "LookInHi"), getattr(MAIN["lookup"], "LookIn"), getattr(MAIN["u32"], "Result")]
    out = []
    for row in (0, n // 2 + 1, n - 1):
        for col in cols + [DERIVED]:
            m = main.copy()
            m[col, row] = (int(m[col, row]) + 1) % P
            out.append((f"main[{col}][{row}]", m, aux))
        a = aux.copy()
        a[7, row, 1] = (int(a[7, row, 1]) + 3) % P
        out.append((f"aux[7][{row}]", main, a))
    m = main.copy()
    proc = slice(MAIN["processor"].start, MAIN["processor"].start + MAIN["processor"].COUNT)
    m[proc, 3:5] = m[proc, 4:2:-1]
    out.append(("swap processor rows 3, 4", m, aux))
    return out


def random_tables(log_n, seed):
    rng = np.random.default_rng(seed)
    n = 1 << log_n
    return (rng.integers(0, P, size=(379, n), dtype=np.uint64), rng.integers(0, P, size=(91, n, 3), dtype=np.uint64),
            rng.integers(0, P, size=(63, 3), dtype=np.uint64))


def boundary_tables(log_n, kind):
    """tables whose Montgomery words are all p - 1, or whose columns alternate between 0 and Montgomery p - 1"""
    n = 1 << log_n
    pm1 = int(corc.from_mont(np.array([P - 1], dtype=np.uint64))[0])    # canonical value whose Montgomery word is p - 1
    if kind == "max":
        main, aux, ch = np.full((379, n), pm1, np.uint64), np.full((91, n, 3), pm1, np.uint64), np.full((63, 3), pm1, np.uint64)
    else:
        alt = np.where(np.arange(n) % 2 == 0, 0, pm1).astype(np.uint64)
        main, aux = np.tile(alt, (379, 1)), np.repeat(np.tile(alt, (91, 1))[:, :, None], 3, axis=2).copy()
        ch = np.full((63, 3), pm1, np.uint64)
    return main, aux, ch


def cpu_cases():
    """(label, main, aux, challenges) of the comparison with the oracle"""
    cases = []
    for name in PROGRAMS:
        main, aux, ch, claim, _ = program_tables(name)
        cases.append((name, main, aux, ch))
        if name in ("fib_100", "kitchen_sink"):
            cases += [(f"{name} {lab}", m, a, ch) for lab, m, a in corrupt_cases(main, aux)]
            bad = challenges63(sampled_challenges(), (claim[0], claim[1], [(claim[2][0] + 1) % P] + claim[2][1:]))
            cases.append((f"{name} wrong output", main, corc.aux_extend(main, bad), bad))
    for log_n in range(4, 9):
        cases.append((f"random 2^{log_n}",) + random_tables(log_n, log_n))
    for kind in ("max", "alternating"):
        cases.append((f"{kind} 2^5",) + boundary_tables(5, kind))
    cases.append(("random n = 2",) + random_tables(1, 99))
    return cases


@pytest.fixture(scope="module")
def host():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    stale = not os.path.exists(SO) or any(os.path.getmtime(f) > os.path.getmtime(SO) for f in [SRC] + HDRS)
    if stale:
        if not os.path.exists(nvcc):
            pytest.skip("nvcc not available to build the host harness")
        os.makedirs(os.path.dirname(SO), exist_ok=True)
        subprocess.run([nvcc, "-O1", "-std=c++17", "--expt-relaxed-constexpr", "-shared", "-Xcompiler", "-fPIC", SRC, "-o", SO], check=True,
                       capture_output=True)
    return ctypes.CDLL(SO)


def host_check(lib, main, aux, ch):
    m, a, c = (np.ascontiguousarray(x, dtype=np.uint64) for x in (main, aux, ch))
    out = [np.zeros(604, dtype=np.uint64) for _ in range(3)]
    vp = ctypes.c_void_p
    lib.air_check_host(m.ctypes.data_as(vp), a.ctypes.data_as(vp), ctypes.c_size_t(m.shape[1]), c.ctypes.data_as(vp),
                       *[o.ctypes.data_as(vp) for o in out])
    return out


_ORACLE = None


def oracle_check(main_table, aux_table, challenges):
    """check_constraints_fn! on the CPU (tests/host/air_check_oracle.c).  main_table [379][n], aux_table [91][n][3] (column 90
    unread), challenges 63 X-field triples, all canonical -> (counts, first_rows, last_rows), uint64 [604] each; first / last
    are 2^64 - 1 where the count is 0"""
    global _ORACLE
    if _ORACLE is None:
        if not os.path.exists(ORACLE_SO) or any(os.path.getmtime(f) > os.path.getmtime(ORACLE_SO) for f in ORACLE_DEPS):
            os.makedirs(os.path.dirname(ORACLE_SO), exist_ok=True)
            cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"   # the distro gcc ships libgomp (as oracle/Makefile)
            subprocess.run([cc, "-O2", "-fopenmp", "-shared", "-fPIC", ORACLE_SRC, "-o", ORACLE_SO], check=True, capture_output=True)
        _ORACLE = ctypes.CDLL(ORACLE_SO)
    T = corc.to_mont(np.ascontiguousarray(main_table, dtype=np.uint64))
    ncols, n = T.shape
    assert ncols == 379
    A = np.asarray(aux_table, dtype=np.uint64).reshape(91, n, 3)[:90]
    A = corc.to_mont(np.ascontiguousarray(A.transpose(0, 2, 1)).reshape(270, n))
    ch = corc.to_mont(np.asarray(challenges, dtype=np.uint64).reshape(63, 3))
    out = [np.zeros(604, dtype=np.uint64) for _ in range(3)]
    vp = ctypes.c_void_p
    _ORACLE.air_check_oracle(T.ctypes.data_as(vp), A.ctypes.data_as(vp), ctypes.c_size_t(n), ch.ctypes.data_as(vp),
                             *[o.ctypes.data_as(vp) for o in out])
    return out


def assert_same(got, want, label):
    for k, what in enumerate(("count", "first row", "last row")):
        bad = np.nonzero(got[k] != want[k])[0]
        assert bad.size == 0, f"{label}: {what} differs at constraints {bad[:8].tolist()}"


_CASES = None


def all_cases():
    global _CASES
    if _CASES is None:
        _CASES = cpu_cases()
    return _CASES


def test_host_bodies_equal_the_oracle(host):
    for label, main, aux, ch in all_cases():
        want = oracle_check(main, aux, ch)
        assert_same(host_check(host, main, aux, ch), want, label)


def test_valid_witnesses_satisfy_every_constraint():
    for name in PROGRAMS:
        main, aux, ch, _, _ = program_tables(name)
        counts, first, last = oracle_check(main, aux, ch)
        assert not counts.any() and (first == 2**64 - 1).all() and (last == 2**64 - 1).all(), name


def test_corruptions_are_located():
    info = tvm_b200.air_constraint_info()
    main, aux, ch, claim, _ = program_tables("fib_100")
    n = main.shape[1]
    from airgen.columns import MAIN
    j = next(i["index"] for i in info if i["derived_column"] == ("main", DERIVED))
    assert info[j]["category"] == "cons"
    for label, m, a in corrupt_cases(main, aux):
        counts, first, last = oracle_check(m, a, ch)
        if label.startswith(f"main[{DERIVED}]"):       # its substitution constraint fires on that row only
            row = int(label.split("[")[2].rstrip("]"))
            assert counts[j] == 1 and first[j] == last[j] == row, label
        if label == f"main[{MAIN['processor'].ST0}][0]":  # the processor's initial stack
            assert any(info[k]["origin"] == "ProcessorTable" and info[k]["category"] == "init" for k in np.nonzero(counts)[0])
        if label.startswith("swap"):
            assert any(info[k]["origin"] == "ProcessorTable" for k in np.nonzero(counts)[0])
    bad = challenges63(sampled_challenges(), (claim[0], claim[1], [(claim[2][0] + 1) % P] + claim[2][1:]))
    counts, first, last = oracle_check(main, corc.aux_extend(main, bad), bad)
    fired = [info[j] for j in np.nonzero(counts)[0]]
    assert fired and all(i["origin"] == "GrandCrossTableArg" and i["category"] == "term" for i in fired)
    assert all(first[i["index"]] == n - 1 for i in fired)
