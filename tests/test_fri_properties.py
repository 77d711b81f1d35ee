"""The reference's FRI property tests (low_degree_test/fri.rs:989-1425) restated against this repository's FRI: the native
verifier `tvm_fri_verify` and parameter derivation `tvm_fri_derive` (host code, run everywhere) and, on a GPU, the device prover
`tvm_fri_prove` — for ARBITRARY FriParameters, not only the ones Stark::fri derives from a padded height.  The oracle is the
checker: its prover (oracle/stark.py::fri_prove) feeds the CPU tests, its proof words are what the device prover must reproduce.
The proof streams are mutated on their encoded words: FriCodeword, FriResponse and its authentication structure are outside
Fiat-Shamir (proof_item.rs:140-145), so an item can be decoded, modified and re-encoded without touching the transcript."""
import math
import random

import numpy as np
import pytest

from oracle import codec, field as F, merkle, stark as S, stir as ST
from oracle.field import P

REGIMES = ("proven", "conjectured")
# (security, log2 expansion, log2 high-degree bound, regime); codewords of at most 2^14 points keep the CPU suite fast
PARAMS = [(1, 1, 0, "conjectured"), (64, 1, 3, "proven"), (16, 1, 8, "proven"), (20, 2, 6, "conjectured"), (160, 2, 8, "proven"),
          (192, 1, 9, "proven"), (40, 3, 9, "conjectured"), (12, 4, 10, "proven"), (8, 5, 6, "conjectured"), (30, 6, 8, "proven"),
          (80, 2, 12, "proven")]
LDT_PARAMS = -6


def oracle_fri_derive(security, log2_exp, log2_hdb, soundness="proven"):
    """FriParameters::try_into_fri + Fri::{max_degree, num_rounds, last_round_max_degree} (fri.rs:799-924) -> the parameter dict
    oracle.stark.fri_prove / fri_verify consume"""
    proximity_parameter = ST.rs_proximity_parameter(log2_exp, soundness)               # mod.rs:243-320
    checks = int(math.ceil(-float(security) / math.log2(1.0 - proximity_parameter)))   # fri.rs:832-836
    domain_len, expansion = 1 << (log2_hdb + log2_exp), 1 << log2_exp
    max_degree = domain_len // expansion - 1                                           # fri.rs:872-874
    max_num_rounds = (max_degree + 1).bit_length() - 1
    skip = (checks.bit_length() - 1 if checks else 0) + 1                              # fri.rs:907-920
    rounds = max(0, max_num_rounds - skip)
    return dict(ldt_offset=F.GENERATOR, ldt_len=domain_len, num_collinearity_checks=checks, fri_num_rounds=rounds,
                fri_last_round_max_degree=max_degree >> rounds, max_degree=max_degree, expansion_factor=expansion)


def _poly(degree, seed):
    rng = np.random.default_rng(seed)
    c = rng.integers(0, P, size=(max(degree + 1, 0), 3), dtype=np.uint64)
    if degree >= 0 and not c[-1].any():
        c[-1, 0] = 1
    return [tuple(int(t) for t in row) for row in c]


def _codeword(d, poly):
    """[domain_len, 3] canonical evaluations on the initial domain"""
    return ST.xevaluate(poly, d["ldt_offset"], d["ldt_len"])


def _at(cw, idx):
    return [tuple(int(t) for t in cw[i]) for i in idx]


def _oracle_proof(d, cw):
    ps = codec.ProofStream()
    idx, _ = S.fri_prove(ps, cw, d)
    return ps.encode(), idx, ps


def _verify(params, proof):
    import tvm_b200
    security, log2_exp, log2_hdb, regime = params
    return tvm_b200.fri_verify(security, log2_exp, log2_hdb, proof, conjectured=regime == "conjectured")


def _ids(params):
    return [f"s{s}-e{e}-h{h}-{r[:4]}" for s, e, h, r in params]


# ---- parameters ---------------------------------------------------------------------------------------------------------------
def test_derivation_matches_oracle_and_num_rounds_are_reasonable():
    """num_rounds_are_reasonable (fri.rs:989-997), over security 1..192 x log2 expansion 1..6 x log2 high-degree bound 0..15 x both
    proximity regimes: tvm_fri_derive equals the stand-alone oracle derivation; with rounds, checks <= last-round max degree <
    2 checks"""
    import tvm_b200
    for regime in REGIMES:
        for log2_exp in range(1, 7):
            for log2_hdb in range(16):
                for security in range(1, 193):
                    got = tvm_b200.fri_derive(security, log2_exp, log2_hdb, conjectured=regime == "conjectured")
                    want = oracle_fri_derive(security, log2_exp, log2_hdb, regime)
                    assert (got["domain_len"], got["domain_offset"], got["expansion_factor"], got["max_degree"],
                            got["num_collinearity_checks"], got["num_rounds"], got["last_round_max_degree"]) == \
                        (want["ldt_len"], want["ldt_offset"], want["expansion_factor"], want["max_degree"], want["num_collinearity_checks"],
                         want["fri_num_rounds"], want["fri_last_round_max_degree"]), (security, log2_exp, log2_hdb, regime)
                    assert got["last_round_max_degree"] == got["max_degree"] >> got["num_rounds"]
                    if got["num_rounds"] > 0:
                        assert got["num_collinearity_checks"] <= got["last_round_max_degree"] < 2 * got["num_collinearity_checks"]


def test_stark_derivation_uses_the_stand_alone_fri():
    """Stark::fri (stark.rs:1972-1995): the FRI fields of tvm_derive_domains are tvm_fri_derive at the final high-degree bound"""
    import tvm_b200
    for security, log2_exp, ph, regime in [(160, 2, 1 << 10, "proven"), (80, 1, 1 << 8, "conjectured"), (128, 4, 1 << 14, "proven")]:
        for ldt in (tvm_b200.LDT_FRI, tvm_b200.LDT_STIR):
            dom = tvm_b200.derive_domains(security, log2_exp, ph, ldt, conjectured=regime == "conjectured")
            log2_hdb = dom["ldt_len"].bit_length() - 1 - log2_exp
            fri = tvm_b200.fri_derive(security, log2_exp, log2_hdb, conjectured=regime == "conjectured")
            assert (dom["ldt_offset"], dom["num_collinearity_checks"], dom["fri_num_rounds"], dom["fri_last_round_max_degree"]) == \
                (fri["domain_offset"], fri["num_collinearity_checks"], fri["num_rounds"], fri["last_round_max_degree"])


def test_smallest_possible_fri():
    """smallest_possible_fri_has_no_rounds, ..._can_only_verify_constant_polynomials (fri.rs:1065-1084)"""
    import tvm_b200
    fd = tvm_b200.fri_derive(1, 1, 0, conjectured=True)
    assert fd["num_rounds"] == 0 and fd["max_degree"] == 0 and fd["domain_len"] == 2 and fd["last_round_max_degree"] == 0


def test_too_small_and_too_big_expansion_factors_are_rejected():
    """too_small_expansion_factor_is_rejected, too_big_expansion_factor_is_rejected (fri.rs:1086-1110); a domain beyond 2^32
    points is InitialDomainTooBig (fri.rs:815-829)"""
    import tvm_b200
    cases = [(0, 0, "TooSmallInitialExpansionFactor"), (0, 5, "TooSmallInitialExpansionFactor")] + \
        [(e, 0, "TooBigInitialExpansionFactor") for e in (32, 33, 63, 64, 1000, (1 << 32) - 1)] + \
        [(1, 32, "InitialDomainTooBig"), (16, 17, "InitialDomainTooBig"), (1, (1 << 32) - 1, "InitialDomainTooBig")]
    for log2_exp, log2_hdb, variant in cases:
        for regime in REGIMES:
            with pytest.raises(tvm_b200.TvmError) as e:
                tvm_b200.fri_derive(1, log2_exp, log2_hdb, conjectured=regime == "conjectured")
            assert e.value.code == LDT_PARAMS
            with pytest.raises(tvm_b200.TvmError) as e:
                _verify((1, log2_exp, log2_hdb, regime), [1, 0])
            assert e.value.code == LDT_PARAMS and variant in str(e.value), str(e.value)
    assert tvm_b200.fri_derive(1, 31, 1)["domain_len"] == 1 << 32    # the largest domain the reference accepts


# ---- prove and verify ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("params", PARAMS, ids=_ids(PARAMS))
def test_prove_and_verify_low_degree_polynomial(params):
    """prove_and_verify_low_degree_polynomial (fri.rs:1013-1027), postscript_is_integral (1371-1424): accepted; the first-round
    indices are the prover's, the partial first codeword is the codeword at those indices and authenticates against the first
    root; the last polynomial is the interpolant of the last codeword"""
    security, log2_exp, log2_hdb, regime = params
    d = oracle_fri_derive(security, log2_exp, log2_hdb, regime)
    max_degree = d["max_degree"]
    for degree in sorted({-1, 0, max_degree // 3, max_degree}):
        cw = _codeword(d, _poly(degree, seed=degree + 11))
        proof, idx, ps = _oracle_proof(d, cw)
        ok, why, vidx, vals = _verify(params, proof)
        assert ok, (degree, why)
        assert vidx == idx and len(idx) == d["num_collinearity_checks"]
        assert [tuple(int(t) for t in v) for v in vals] == _at(cw, idx)
        items = codec.decode_proof(proof).items
        first_root = items[0][1]
        leafs = [(i, list(v) + [0, 0]) for i, v in zip(idx, _at(cw, idx))]
        assert merkle.verify_inclusion(first_root, d["ldt_len"].bit_length() - 1, leafs, items[d["fri_num_rounds"] + 3][1][1])
        last_cw = items[d["fri_num_rounds"] + 1][1]
        assert len(last_cw) == d["ldt_len"] >> d["fri_num_rounds"]
        assert items[d["fri_num_rounds"] + 2][1] == ST.xinterpolate(last_cw, 1)


@pytest.mark.parametrize("params", [p for p in PARAMS if oracle_fri_derive(*p)["max_degree"] >= 3], ids=_ids([p for p in PARAMS if oracle_fri_derive(*p)["max_degree"] >= 3]))
def test_prove_and_verify_low_degree_of_twice_cubing_plus_one(params):
    """prove_and_verify_low_degree_of_twice_cubing_plus_one (fri.rs:999-1011)"""
    d = oracle_fri_derive(*params)
    proof, idx, _ = _oracle_proof(d, _codeword(d, [(1, 0, 0), (0, 0, 0), (0, 0, 0), (2, 0, 0)]))
    ok, why, vidx, _ = _verify(params, proof)
    assert ok and vidx == idx, why


@pytest.mark.parametrize("params", PARAMS, ids=_ids(PARAMS))
def test_high_degree_polynomial_is_rejected(params):
    """prove_and_fail_to_verify_high_degree_polynomial (fri.rs:1048-1063),
    codeword_corresponding_to_high_degree_polynomial_results_in_verification_failure (1347-1361)"""
    d = oracle_fri_derive(*params)
    too_high = d["max_degree"] + 1
    for degree in sorted({too_high, too_high + too_high // 2, 2 * too_high - 1}):
        proof, _, _ = _oracle_proof(d, _codeword(d, _poly(degree, seed=degree)))
        ok, why, _, _ = _verify(params, proof)
        assert not ok and why == "LdtVerificationError: LastRoundPolynomialHasTooHighDegree", (degree, why)


def test_serialization():
    """serialization (fri.rs:1112-1137): the encoded proof stream decodes to the prover's items"""
    for params in PARAMS:
        d = oracle_fri_derive(*params)
        proof, _, ps = _oracle_proof(d, _codeword(d, _poly(d["max_degree"] // 2, seed=3)))
        items = codec.decode_proof(proof).items
        assert [k for k, _ in items] == [k for k, _ in ps.items]
        for (k, p), (_, v) in zip(ps.items, items):
            assert codec.encode_item(k, p) == codec.encode_item(k, v)
        assert [k for k, _ in items] == ["MerkleRoot"] * (d["fri_num_rounds"] + 1) + ["FriCodeword", "Polynomial"] + \
            ["FriResponse"] * (d["fri_num_rounds"] + 1)


# ---- corrupted proofs ---------------------------------------------------------------------------------------------------------
def _mutated(proof, mutate):
    ps = codec.decode_proof(proof)
    ps.items = [(k, p) for k, p in ps.items]
    mutate(ps.items)
    return ps.encode()


def _find(items, kind):
    return [i for i, (k, _) in enumerate(items) if k == kind]


MUTATION_PARAMS = [p for p in PARAMS if p[2] > 0]


@pytest.mark.parametrize("params", MUTATION_PARAMS, ids=_ids(MUTATION_PARAMS))
def test_corrupted_proofs_are_rejected_with_the_reference_variant(params):
    """last_round_codeword_unequal_to_last_round_commitment_results_in_validation_failure (fri.rs:1139-1158),
    revealing_wrong_number_of_leaves_results_in_validation_failure (1183-1202),
    incorrect_authentication_structure_results_in_validation_failure (1232-1255),
    too_short_last_round_codeword_doesnt_panic (1288-1310),
    incorrect_last_round_polynomial_results_in_verification_failure (1312-1345)"""
    d = oracle_fri_derive(*params)
    proof, _, _ = _oracle_proof(d, _codeword(d, _poly(d["max_degree"], seed=21)))
    assert _verify(params, proof)[0]
    rnd = random.Random(params[0] * 1000 + params[2])
    rx = lambda: (rnd.randrange(P), rnd.randrange(P), rnd.randrange(P))
    for _ in range(4):
        def change_last_codeword(items):
            k = _find(items, "FriCodeword")[0]
            cw = list(items[k][1])
            cw[rnd.randrange(len(cw))] = rx()
            items[k] = ("FriCodeword", cw)
        assert _verify(params, _mutated(proof, change_last_codeword))[1] == "LdtVerificationError: BadMerkleRootForLastCodeword"

        def change_number_of_leaves(items):
            k = rnd.choice(_find(items, "FriResponse"))
            leaves, auth = items[k][1]
            leaves = list(leaves)
            j = rnd.randrange(len(leaves))
            if rnd.random() < 0.5:
                leaves.pop(j)
            else:
                leaves.insert(j, rx())
            items[k] = ("FriResponse", (leaves, auth))
        assert _verify(params, _mutated(proof, change_number_of_leaves))[1] == "LdtVerificationError: IncorrectNumberOfRevealedLeaves"

        def shorten_last_codeword(items):
            k = _find(items, "FriCodeword")[0]
            items[k] = ("FriCodeword", list(items[k][1])[:-1])
        assert _verify(params, _mutated(proof, shorten_last_codeword))[1] == "LdtVerificationError: LastCodewordMismatch"

        wrong = _poly(d["fri_last_round_max_degree"], seed=rnd.randrange(1 << 30))

        def replace_last_polynomial(items):
            k = _find(items, "Polynomial")[0]
            items[k] = ("Polynomial", wrong)
        assert _verify(params, _mutated(proof, replace_last_polynomial))[1] in (
            "LdtVerificationError: LastRoundPolynomialEvaluationMismatch", "LdtVerificationError: BadMerkleAuthenticationPath")

    responses = [k for k in _find(codec.decode_proof(proof).items, "FriResponse") if codec.decode_proof(proof).items[k][1][1]]
    if d["num_collinearity_checks"] >= d["ldt_len"]:
        assert not responses                 # every leaf is revealed: all authentication structures are empty
        return
    assert responses
    for how in range(3):
        for _ in range(3):
            def change_auth_structure(items):
                k = rnd.choice(responses)
                leaves, auth = items[k][1]
                auth = [list(a) for a in auth]
                j = rnd.randrange(len(auth))
                if how == 0:
                    auth.pop(j)
                elif how == 1:
                    auth.insert(j, [rnd.randrange(P) for _ in range(5)])
                else:
                    auth[j] = [rnd.randrange(P) for _ in range(5)]
                items[k] = ("FriResponse", (leaves, auth))
            assert _verify(params, _mutated(proof, change_auth_structure))[1] == "LdtVerificationError: BadMerkleAuthenticationPath"


@pytest.mark.parametrize("params", [PARAMS[0], PARAMS[1], PARAMS[4], PARAMS[7]], ids=_ids([PARAMS[0], PARAMS[1], PARAMS[4], PARAMS[7]]))
def test_any_corrupted_word_is_rejected(params):
    """one corrupted word anywhere - Merkle root, last codeword, last polynomial, revealed leaves, authentication structure, any
    length prefix - is rejected; so are truncated streams"""
    d = oracle_fri_derive(*params)
    proof, _, _ = _oracle_proof(d, _codeword(d, _poly(d["max_degree"], seed=5)))
    proof = np.array(proof, dtype=np.uint64)
    rnd = random.Random(7)
    for j in sorted(set(rnd.randrange(proof.size) for _ in range(60)) | {0, 1, 2, proof.size - 1}):
        bad = proof.copy()
        bad[j] = (int(bad[j]) + 1 + rnd.randrange(P - 2)) % P
        ok, why, _, _ = _verify(params, bad)
        assert not ok and why, j
    for cut in (1, 3, proof.size // 2):
        assert not _verify(params, proof[:-cut])[0]


def test_verifying_arbitrary_proof_does_not_panic():
    """verifying_arbitrary_proof_does_not_panic (fri.rs:1363-1369): junk words of many lengths, and valid proofs checked under
    parameters they were not made for (also with security levels whose collinearity checks exceed the proof), are rejected"""
    import tvm_b200
    rnd = random.Random(1)
    for params in PARAMS[:6]:
        for n in (1, 2, 3, 7, 100, 5000):
            junk = np.array([rnd.randrange(P) for _ in range(n)], dtype=np.uint64)
            assert _verify(params, junk)[0] is False
            junk[0] = n - 1                                    # a consistent length prefix gets past the first check
            assert _verify(params, junk)[0] is False
    for params in PARAMS[1:6]:
        security, log2_exp, log2_hdb, regime = params
        d = oracle_fri_derive(*params)
        proof, _, _ = _oracle_proof(d, _codeword(d, _poly(d["max_degree"], seed=9)))
        others = [(security + 9, log2_exp, log2_hdb, regime), (security, log2_exp + 1, log2_hdb, regime),
                  (security, log2_exp, log2_hdb + 1, regime), (security, log2_exp + 1, max(log2_hdb - 1, 0), regime),
                  (security, log2_exp, log2_hdb, REGIMES[regime == "proven"]), ((1 << 32) - 1, log2_exp, log2_hdb, regime)]
        for other in others:
            if oracle_fri_derive(*other) == d:
                continue
            ok, why, _, _ = _verify(other, proof)
            assert not ok and why, other
    with pytest.raises(tvm_b200.TvmError) as e:                # a domain of 2^32 points: indices cannot be sampled below it
        _verify((1, 1, 31, "proven"), [1, 0])
    assert e.value.code == -5


# ---- the device prover --------------------------------------------------------------------------------------------------------
GPU_PARAMS = [(1, 1, 0, "conjectured"), (1, 1, 0, "proven"), (64, 1, 3, "proven"), (192, 2, 4, "conjectured"),
              (16, 1, 8, "proven"), (16, 1, 8, "conjectured"), (160, 1, 11, "proven"), (160, 1, 11, "conjectured"),
              (192, 1, 12, "proven"), (192, 1, 12, "conjectured"), (160, 2, 12, "proven"), (160, 3, 10, "conjectured"),
              (40, 4, 9, "proven"), (16, 5, 8, "conjectured"), (192, 6, 7, "proven"), (160, 6, 15, "proven"), (24, 2, 15, "conjectured")]


@pytest.mark.gpu
@pytest.mark.parametrize("params", GPU_PARAMS, ids=_ids(GPU_PARAMS))
def test_device_fri_prover_for_arbitrary_parameters(backend, params):
    """the device prover under arbitrary FriParameters: word for word the oracle's proof stream with the same indices, accepted
    by the native verifier (low degree), rejected for a too-high degree"""
    security, log2_exp, log2_hdb, regime = params
    conj = regime == "conjectured"
    d = oracle_fri_derive(*params)
    max_degree = d["max_degree"]
    for degree in sorted({-1, 0, max_degree}):
        cw = _codeword(d, _poly(degree, seed=degree + 3))
        want, want_idx, _ = _oracle_proof(d, cw)
        got, idx = backend.fri_prove(security, log2_exp, log2_hdb, cw, conjectured=conj)
        assert [int(v) for v in got] == want and idx == want_idx, degree
        ok, why, vidx, vals = _verify(params, got)
        assert ok and vidx == idx, why
        assert [tuple(int(t) for t in v) for v in vals] == _at(cw, idx)
    cw = _codeword(d, _poly(max_degree + 1 + max_degree // 2, seed=2))
    got, _ = backend.fri_prove(security, log2_exp, log2_hdb, cw, conjectured=conj)
    assert _verify(params, got)[1] == "LdtVerificationError: LastRoundPolynomialHasTooHighDegree"


@pytest.mark.gpu
def test_device_fri_prover_reads_device_memory(backend):
    """a codeword in device memory gives the same words as the same codeword in host memory"""
    import torch
    d = oracle_fri_derive(160, 2, 10, "proven")
    cw = _codeword(d, _poly(d["max_degree"], seed=4))
    host = backend.fri_prove(160, 2, 10, cw)
    dev = backend.fri_prove(160, 2, 10, torch.from_numpy(cw.view(np.int64)).cuda())
    assert np.array_equal(host[0], dev[0]) and host[1] == dev[1]


@pytest.mark.gpu
def test_device_fri_prover_rejects_bad_arguments_without_a_launch(backend):
    """codeword_len != domain length is InitialCodewordMismatch (fri.rs:323-330, fail_to_prove_codeword_of_incorrect_length
    1029-1046); bad expansion factors are LdtParameterError's; domains beyond 2^26 points are TVM_ERR_DOMAIN - all before any
    kernel is launched"""
    import ctypes
    import tvm_b200
    lib = backend._l
    cw = np.zeros((1 << 12, 3), dtype=np.uint64)
    cwp = cw.ctypes.data_as(ctypes.POINTER(ctypes.c_uint64))
    out = np.zeros(1 << 16, dtype=np.uint64)
    cases = [(2, 6, 63, -1, "InitialCodewordMismatch { domain_len: 256, codeword_len: 63 }"),
             (2, 6, 257, -1, "InitialCodewordMismatch { domain_len: 256, codeword_len: 257 }"),
             (0, 6, 64, LDT_PARAMS, "TooSmallInitialExpansionFactor"), (32, 0, 64, LDT_PARAMS, "TooBigInitialExpansionFactor"),
             (40, 6, 64, LDT_PARAMS, "TooBigInitialExpansionFactor"), (1, 32, 64, LDT_PARAMS, "InitialDomainTooBig"),
             (2, 25, 64, -5, "2^26")]
    before = backend.launches
    for log2_exp, log2_hdb, n, code, text in cases:
        cap = ctypes.c_size_t(out.size)
        rc = lib.tvm_fri_prove(backend._h, 160, 0, log2_exp, log2_hdb, cwp, n, out.ctypes.data_as(ctypes.POINTER(ctypes.c_uint64)),
                               ctypes.byref(cap), None, None)
        assert rc == code, (log2_exp, log2_hdb, n, rc)
        assert text in lib.tvm_last_error(backend._h).decode()
    assert backend.launches == before
    with pytest.raises(tvm_b200.TvmError) as e:
        backend.fri_prove(160, 2, 6, cw[:100])
    assert e.value.code == -1 and "InitialCodewordMismatch" in str(e.value)
    assert backend.launches == before
