"""The seeded program corpus of tests/program_corpus.py on the device: the hash traces tvm_execution_aet expands, the table
fill (tvm_main_table_from_aet) at the padded height and at twice it, the degree-lowering columns, the auxiliary extension
and the AIR check, each against the oracle on every row; the shape cases and three random programs proved and verified
with the AIR; and one shape case and one random program proved word for word like the oracle.  The host runs of the same
corpus are tests/test_program_corpus.py; this file sorts last."""
import numpy as np
import pytest

import tvm_b200
from oracle import corc, fast, reference_prover as RP, stark as S, tracegen as tg

import program_corpus as PC
from test_air_check import assert_same, challenges63, oracle_check, sampled_challenges
from test_program_corpus import CASES, IDS, TABLES, fill_host, oracle_main_table, run_oracle   # noqa: F401  (fixture)
from test_program_execution import HASH_KEYS
from test_zzzzz_gpu_production_shapes import first_difference

pytestmark = pytest.mark.gpu

SEED = bytes(range(40, 72))
PROVED = [c.name for c in CASES if c.name.startswith("shape")] + ["random-seed=0", "random-seed=7", "random-seed=13"]
WORD_FOR_WORD = ["shape-u32-exactly-2^12", "random-seed=7"]


def _trace(case):
    return tvm_b200.trace_execution(case.words, case.public_input, case.secret_input, case.digests, case.ram)


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_device_witness_matches_the_oracle(backend, fill_host, case):
    want_ex = run_oracle(case)
    arrays = tg.aet_arrays(list(case.words), want_ex)
    ex = _trace(case)
    aet = ex.aet(backend)
    for key in HASH_KEYS:
        assert aet[key].shape == arrays[key].shape and np.array_equal(aet[key], arrays[key]), key
    heights = tg.table_heights(list(case.words), want_ex)
    n = ex.padded_height
    for rows in (n, 2 * n):
        want, claim = oracle_main_table(case, want_ex, rows, fill_host)
        got, lengths = backend.main_table_from_aet(aet, rows)
        bad = [c for c in range(379) if not np.array_equal(got[c], want[c])]
        assert not bad, (rows, [tg.column_name(True, c) for c in bad[:8]])
        assert lengths == [heights[k] for k in TABLES]
    derived = want.copy()
    derived[149:] = 0
    backend.fill_derived_main_columns(derived)
    assert np.array_equal(derived, want)
    for seed in ((5, 6) if case.name.startswith("random") else (5,)):
        ch = challenges63(sampled_challenges(seed), claim)
        aux = backend.aux_extend(want, ch)
        want_aux = corc.aux_extend(want, ch)
        bad = [q for q in range(91) if not np.array_equal(aux[q], want_aux[q])]
        assert not bad, f"aux columns {bad[:8]} differ"
        triples = [np.asarray(x) for x in backend.air_check(want, aux, ch, arrays=True)]
        assert_same(triples, oracle_check(want, want_aux, ch), case.name)
        assert not triples[0].any()
        counts, first, last = (np.asarray(x) for x in backend.air_check_execution(ex, sampled_challenges(seed), arrays=True))
        assert not counts.any() and (first == 2**64 - 1).all() and (last == 2**64 - 1).all()
    ex.close()


@pytest.mark.parametrize("name", PROVED)
def test_proof_verifies_with_the_air(backend, name):
    ex = _trace(PC.by_name(name))
    proof = backend.prove_execution(ex, SEED, security_level=8)
    assert tvm_b200.proof_padded_height(proof) == ex.padded_height
    assert tvm_b200.verify(ex.claim, proof, 8, 2) == (True, "")
    ex.close()


@pytest.mark.parametrize("name", WORD_FOR_WORD)
def test_proof_equals_the_oracles(backend, name):
    case = PC.by_name(name)
    inst = RP.instance(S.Stark(8, 2), list(case.words), case.public_input, SEED, case.secret_input, case.ram, case.digests)
    want = np.array(fast.prove(inst["stark"], inst["claim"], inst["main"], inst["main_rand"], inst["extend"], inst["quot_rand"],
                               padded_height=inst["padded_height"]), dtype=np.uint64)
    ex = _trace(case)
    got = backend.prove_execution(ex, SEED, security_level=8)
    assert ex.claim == (inst["claim"].program_digest, inst["claim"].input, inst["claim"].output)
    ex.close()
    assert np.array_equal(got, want), f"first differing proof item: {first_difference(got, want)}"
