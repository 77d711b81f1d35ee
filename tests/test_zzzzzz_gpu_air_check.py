"""The AIR constraint checker on the device (tvm_air_check, tvm_air_check_aet, tvm_air_check_execution) against the oracle's
CPU check (tests/host/air_check_oracle.c) on all 604 (count, first row, last row) triples, with tables in host memory and as device tensors; the
witness the library builds itself (fill, degree lowering, Challenges::new, extension) checked at production heights; and the
reported rows of a corrupted 2^20 table re-evaluated on the host.  The CPU cases are those of tests/test_air_check.py."""
import ctypes

import numpy as np
import pytest

from test_air_check import P, all_cases, assert_same, boundary_tables, challenges63, oracle_check, random_tables, sampled_challenges
from oracle import corc, tracegen as tg
import test_program_execution as tpe
import test_vm_programs as tvp

pytestmark = pytest.mark.gpu


def triples(res):
    return [np.asarray(x) for x in res]


def test_device_check_equals_the_oracle_on_the_cpu_cases(backend):
    for label, main, aux, ch in all_cases():
        assert_same(triples(backend.air_check(main, aux, ch, arrays=True)), oracle_check(main, aux, ch), label)


def test_device_check_of_device_tensors(backend):
    import torch
    for label, main, aux, ch in all_cases()[::7]:
        got = backend.air_check(torch.from_numpy(main.view(np.int64)).cuda(), torch.from_numpy(aux.view(np.int64)).cuda(), ch, arrays=True)
        assert_same(triples(got), oracle_check(main, aux, ch), label + " (device tensors)")


@pytest.mark.parametrize("log_n", [12, 16])
def test_device_check_at_larger_heights(backend, log_n):
    cases = [("random",) + random_tables(log_n, 7 * log_n), ("max",) + boundary_tables(log_n, "max"),
             ("alternating",) + boundary_tables(log_n, "alternating")]
    for label, main, aux, ch in cases:
        assert_same(triples(backend.air_check(main, aux, ch, arrays=True)), oracle_check(main, aux, ch), f"{label} 2^{log_n}")


def _aet(name):
    words, inp, sec, ram, digests = tpe.program(name)
    ex = tg.execute(list(words), inp, sec, ram, digests)
    return tg.aet_arrays(list(words), ex), (list(ex.digest), list(inp), list(ex.output)), tg.padded_height(list(words), inp, sec, ram, digests)


def _via_tables(backend, aet, claim, n, sampled):
    main, _ = backend.main_table_from_aet(aet, n)
    ch = challenges63(sampled, claim)
    return backend.air_check(main, backend.aux_extend(main, ch), ch, arrays=True)


@pytest.mark.parametrize("name", ["halt", "fib_100", "kitchen_sink", "memory_and_merkle", "every_instruction", "u32_mix"])
def test_aet_check_equals_the_table_check(backend, name):
    aet, claim, n = _aet(name)
    sampled = sampled_challenges(11)
    got = triples(backend.air_check_aet(aet, claim, n, sampled, arrays=True))
    assert not got[0].any(), name
    assert_same(got, triples(_via_tables(backend, aet, claim, n, sampled)), name)


# a changed u32 multiplicity leaves the U32 table consistent in itself (the fill rebuilds its sections): what breaks is the
# lookup argument between the processor and the U32 table, a Grand Cross-Table Argument terminal constraint
@pytest.mark.parametrize("what, table", [("processor_trace", "ProcessorTable"), ("ram_trace", "RamTable"), ("u32_entries", "GrandCrossTableArg")])
def test_aet_check_locates_a_changed_aet_word(backend, what, table):
    aet, claim, n = _aet("kitchen_sink")
    aet = {k: (v.copy() if hasattr(v, "copy") else v) for k, v in aet.items()}
    a = aet[what]
    if what == "processor_trace":
        a[5, 15] = (int(a[5, 15]) + 1) % P          # ST0 of row 5
    elif what == "ram_trace":
        a[2, 3] = (int(a[2, 3]) + 1) % P            # a RAM value
    else:
        a[1, 3] = int(a[1, 3]) + 1                  # a u32 entry's multiplicity
    sampled = sampled_challenges(12)
    got = backend.air_check_aet(aet, claim, n, sampled)
    assert got and table in {v["origin"] for v in got}, (what, sorted({v["origin"] for v in got}))
    assert_same(triples(backend.air_check_aet(aet, claim, n, sampled, arrays=True)), triples(_via_tables(backend, aet, claim, n, sampled)), what)


@pytest.mark.parametrize("workload, log_ph", [("spin_16", 16), ("spin_20", 20), ("verifier_11500", 20)])
def test_programs_satisfy_every_constraint_at_production_height(backend, workload, log_ph):
    program, inp, ram = tvp._workload(workload)
    ex = __import__("tvm_b200").trace_execution(tg.assemble(program), inp, (), (), ram)
    assert ex.padded_height == 1 << log_ph
    counts, first, last = triples(backend.air_check_execution(ex, sampled_challenges(3), arrays=True))
    ex.close()
    assert not counts.any() and (first == 2**64 - 1).all() and (last == 2**64 - 1).all()
    if log_ph == 16:
        assert backend.check_program(tg.assemble(program), inp, ram=ram) == []


def test_reported_rows_of_a_corrupted_2_20_table_reevaluate(backend):
    import torch
    import tvm_b200
    program, inp, ram = tvp._workload("spin_20")
    ex = tvm_b200.trace_execution(tg.assemble(program), inp, (), (), ram)
    aet = ex.aet(backend)
    n = ex.padded_height
    main, _ = backend.main_table_from_aet(aet, n)
    claim = ex.claim
    ex.close()
    from airgen.columns import MAIN
    main[MAIN["processor"].ST1, 77777] = (int(main[MAIN["processor"].ST1, 77777]) + 5) % P
    main[MAIN["hash"].State7, n - 3] = (int(main[MAIN["hash"].State7, n - 3]) + 1) % P
    ch = challenges63(sampled_challenges(4), claim)
    d_main = torch.from_numpy(main.view(np.int64)).cuda()
    d_aux = torch.empty((91, n, 3), dtype=torch.int64, device="cuda")
    backend.aux_extend(d_main, ch, out=d_aux)
    got = backend.air_check(d_main, d_aux, ch)
    assert got
    rows_of = {"init": (0, 1), "cons": (0, n), "tran": (0, n - 1), "term": (n - 1, n)}
    cats = ("init", "cons", "tran", "term")

    def value(v, r):
        nx = min(r + 1, n - 1)
        a = d_aux[:90, [r, nx], :].cpu().numpy().view(np.uint64)
        vals = corc.air_eval_category(cats.index(v["category"]), main[:, r], a[:, 0, :].reshape(-1), main[:, nx], a[:, 1, :].reshape(-1), ch)
        return vals[v["index_in_category"]]
    for v in got:
        assert value(v, v["first_row"]).any() and value(v, v["last_row"]).any(), v
        lo, hi = rows_of[v["category"]]
        for r in (v["first_row"] - 1, v["last_row"] + 1, (v["first_row"] + v["last_row"]) // 2):
            if lo <= r < hi and not (v["first_row"] <= r <= v["last_row"]):
                assert not value(v, r).any(), (v, r)
        if v["count"] == v["last_row"] - v["first_row"] + 1:
            assert value(v, (v["first_row"] + v["last_row"]) // 2).any(), v


def test_argument_errors(backend):
    import tvm_b200
    lib, before = tvm_b200.lib(), backend.launches
    out = [(ctypes.c_uint64 * 604)() for _ in range(3)]
    nv = ctypes.c_uint64()
    main, aux, ch = random_tables(4, 1)
    mp, ap, cp = (x.ctypes.data_as(tvm_b200._u64p) for x in (main, aux, ch))
    assert lib.tvm_air_check(backend._h, None, ap, 4, cp, *out, ctypes.byref(nv)) == -1
    assert lib.tvm_air_check(backend._h, mp, None, 4, cp, *out, ctypes.byref(nv)) == -1
    assert lib.tvm_air_check(backend._h, mp, ap, 4, None, *out, ctypes.byref(nv)) == -1
    assert lib.tvm_air_check(backend._h, mp, ap, 4, cp, out[0], out[1], out[2], None) == -1
    assert lib.tvm_air_check(backend._h, mp, ap, 27, cp, *out, ctypes.byref(nv)) == -5
    bad_ch = ch.copy()
    bad_ch[5, 1] = P
    assert lib.tvm_air_check(backend._h, mp, ap, 4, bad_ch.ctypes.data_as(tvm_b200._u64p), *out, ctypes.byref(nv)) == -1
    aet, claim, _ = _aet("halt")
    s, keep = tvm_b200.aet_struct(aet)
    cs, keep2 = backend._claim(claim)
    sp = sampled_challenges().copy()
    assert lib.tvm_air_check_aet(backend._h, ctypes.byref(s), ctypes.byref(cs), 100, sp.ctypes.data_as(tvm_b200._u64p), *out, ctypes.byref(nv)) == -5
    sp[0, 0] = P
    assert lib.tvm_air_check_aet(backend._h, ctypes.byref(s), ctypes.byref(cs), 256, sp.ctypes.data_as(tvm_b200._u64p), *out, ctypes.byref(nv)) == -1
    assert backend.launches == before
    # a word >= p: found by the upload pass, named by column and row; no check kernel runs
    m2 = main.copy()
    m2[17, 9] = P + 3
    with pytest.raises(tvm_b200.TvmError, match="main table: word >= p at column 17, row 9"):
        backend.air_check(m2, aux, ch)
    a2 = aux.copy()
    a2[40, 3, 2] = 2**64 - 1
    with pytest.raises(tvm_b200.TvmError, match="aux table: word >= p at column 40, row 3, coordinate 2"):
        backend.air_check(main, a2, ch)
    assert backend.launches == before + 4
