"""STIR at every folding factor: `log2_folding_factor` through tvm_stir_derive, tvm_stir_verify_k and the device prover
tvm_stir_prove_k, with the oracle (oracle/stir.py, oracle/fast.py) as the checker.

The reference draws the factor of its STIR property tests (low_degree_test/stir.rs:1813-2010) from 2^2..2^5 (stir.rs:77);
tests/test_stir_properties.py restates them at 2^2, the factor Stark::ldt uses.  Here they run at 2^3, 2^4 and 2^5, and the
device prover is checked word for word against the oracle at 2^3, 2^4 and 2^5 up to the size of a padded-height-2^20 prove."""
import random

import numpy as np
import pytest

import tvm_b200
from oracle import codec, corc, fast, stir as ST
from oracle.field import P

LDT_PARAMS = -6


def _native_derive(security, log2_ff, log2_exp, log2_hdb, soundness):
    """-> dict like oracle.stir.derive, or the LdtParameterError variant the native code names"""
    try:
        return tvm_b200.stir_derive(security, log2_exp, log2_hdb, soundness == "conjectured", log2_ff)
    except tvm_b200.TvmError as e:
        assert e.code == LDT_PARAMS, e
    try:   # tvm_stir_derive has no failure buffer: the verifier checks the same parameters first and names the variant
        tvm_b200.stir_verify(security, log2_exp, log2_hdb, np.array([0], dtype=np.uint64), soundness == "conjectured", log2_ff)
    except tvm_b200.TvmError as e:
        assert e.code == LDT_PARAMS, e
        return str(e).rsplit("LdtParameterError: ", 1)[1]
    raise AssertionError("the verifier accepted parameters tvm_stir_derive rejects")


def _oracle_derive(security, log2_ff, log2_exp, log2_hdb, soundness):
    try:
        return ST.derive(security, log2_ff, log2_exp, log2_hdb, soundness)
    except ValueError as e:
        return str(e)


@pytest.mark.parametrize("soundness", ["proven", "conjectured"])
@pytest.mark.parametrize("log2_ff", [2, 3, 4, 5, 6])
def test_derive_equals_the_oracle(log2_ff, soundness):
    """StirParameters::try_into_stir: every round's query counts, the final round and the initial domain"""
    for security in (8, 33, 100, 160):
        for log2_exp in range(1, 7):
            for log2_hdb in range(log2_ff, 21):
                want = _oracle_derive(security, log2_ff, log2_exp, log2_hdb, soundness)
                assert _native_derive(security, log2_ff, log2_exp, log2_hdb, soundness) == want, (security, log2_exp, log2_hdb)


@pytest.mark.parametrize("log2_ff,log2_exp,log2_hdb", [
    (0, 2, 10), (1, 2, 10), (1, 0, 0),                   # TooSmallLog2FoldingFactor, checked first
    (2, 0, 10), (5, 0, 3),                               # TooSmallInitialExpansionFactor before TooLowDegree...
    (3, 2, 2), (6, 1, 5), (20, 1, 19),                   # TooLowDegreeOfHighDegreePolynomials
    (3, 4, 29), (2, 1, 32), (5, 31, 5),                  # InitialDomainTooBig
])
def test_parameter_errors_name_the_oracles_variant(log2_ff, log2_exp, log2_hdb):
    for soundness in ("proven", "conjectured"):
        want = _oracle_derive(16, log2_ff, log2_exp, log2_hdb, soundness)
        assert isinstance(want, str)
        assert _native_derive(16, log2_ff, log2_exp, log2_hdb, soundness) == want


def test_too_big_folding_factor():
    """stir.rs:450-459: a factor 2^log2_folding_factor that overflows usize, checked after TooLowDegreeOfHighDegreePolynomials
    and before the initial domain (the oracle stops at InitialDomainTooBig, which comes later)"""
    assert _native_derive(16, 64, 1, 64, "proven") == "TooBigLog2FoldingFactor"
    assert _native_derive(16, 64, 1, 63, "proven") == "TooLowDegreeOfHighDegreePolynomials"
    assert _native_derive(16, 63, 1, 63, "proven") == "InitialDomainTooBig"


# ---- the reference's property tests at folding factors 2^3, 2^4, 2^5 (CPU: oracle prover, native verifier) -------------
PARAMS = {   # (security, log2 expansion, log2 high-degree bound); the first has no full round (high-degree bound = factor)
    3: [(8, 1, 3), (20, 1, 9), (6, 2, 10), (8, 3, 10), (4, 2, 13)],
    4: [(8, 2, 4), (12, 1, 9), (6, 3, 11), (8, 2, 12)],
    5: [(8, 1, 5), (16, 1, 11), (6, 3, 13), (4, 2, 13)],
}
CASES = [(f, *t) for f, ts in PARAMS.items() for t in ts]


def _instance(security, log2_ff, log2_exp, log2_hdb, degree, seed):
    rnd = random.Random(seed)
    sp = ST.derive(security, log2_ff, log2_exp, log2_hdb)
    poly = [tuple(rnd.randrange(P) for _ in range(3)) for _ in range(degree + 1)]
    cw = ST.xevaluate(poly, sp["initial_offset"], sp["initial_domain_len"]) if poly else np.zeros((sp["initial_domain_len"], 3), dtype=np.uint64)
    return sp, [tuple(int(t) for t in v) for v in cw]


def _oracle_proof(sp, cw):
    ps = codec.ProofStream()
    idx = ST.prove(ps, cw, sp)
    return ps.encode(), idx


def test_the_cases_cover_zero_and_several_full_rounds():
    rounds = {f: [len(ST.derive(s, f, e, h)["round_queries"]) for s, e, h in ts] for f, ts in PARAMS.items()}
    assert all(r[0] == 0 and max(r) >= 1 for r in rounds.values()), rounds


@pytest.mark.parametrize("log2_ff,security,log2_exp,log2_hdb", CASES)
def test_verifier_accepts_low_degree_and_zero_polynomials(log2_ff, security, log2_exp, log2_hdb):
    """prove_and_verify_low_degree_polynomial (stir.rs:1869-1900), prove_and_verify_zero_polynomial (1813-1822): accepted, the
    oracle's first-round indices, and the partial first codeword is the codeword at those indices"""
    max_degree = (1 << log2_hdb) - 1
    for degree in (max_degree, max_degree // 3, 0, -1):
        sp, cw = _instance(security, log2_ff, log2_exp, log2_hdb, degree, seed=degree + 11)
        proof, idx = _oracle_proof(sp, cw)
        ok, why, vidx, vals = tvm_b200.stir_verify(security, log2_exp, log2_hdb, proof, log2_folding_factor=log2_ff)
        assert ok, why
        assert vidx == idx
        assert [tuple(int(t) for t in v) for v in vals] == [cw[i] for i in idx]


@pytest.mark.parametrize("log2_ff,security,log2_exp,log2_hdb", CASES)
def test_verifier_rejects_too_high_degree(log2_ff, security, log2_exp, log2_hdb):
    """prove_and_fail_to_verify_high_degree_polynomial (stir.rs:1903-1920)"""
    too_high = 1 << log2_hdb
    for degree in (too_high, too_high + too_high // 2, 2 * too_high - 1):
        sp, cw = _instance(security, log2_ff, log2_exp, log2_hdb, degree, seed=degree)
        proof, _ = _oracle_proof(sp, cw)
        ok, why, _, _ = tvm_b200.stir_verify(security, log2_exp, log2_hdb, proof, log2_folding_factor=log2_ff)
        assert not ok and why.startswith("LdtVerificationError: "), why


def _reencode(items):
    ps = codec.ProofStream()
    ps.items = items
    return np.array(ps.encode(), dtype=np.uint64)


def _corruptions(items, rnd):
    """(item index, corrupted item) for the reference's corruptions (stir.rs:1967-2010): a Merkle root digest, an
    out-of-domain value, a revealed leaf's element, an authentication-structure digest, a final-polynomial coefficient"""
    def other():
        return tuple(rnd.randrange(P) for _ in range(3))
    for i, (kind, payload) in enumerate(items):
        if kind == "MerkleRoot":
            d = list(payload); d[rnd.randrange(5)] = (d[0] + 1) % P
            yield i, (kind, d)
        elif kind in ("StirOutOfDomainValues", "Polynomial") and payload:
            v = list(payload); v[rnd.randrange(len(v))] = other()
            yield i, (kind, v)
        elif kind == "StirResponse":
            leafs, auth = payload
            j = rnd.randrange(len(leafs))
            bad = [list(l) for l in leafs]; bad[j][rnd.randrange(len(bad[j]))] = other()
            yield i, (kind, (bad, auth))
            if auth:
                a = [list(d) for d in auth]; a[rnd.randrange(len(a))][0] ^= 1
                yield i, (kind, (leafs, a))


@pytest.mark.parametrize("log2_ff,security,log2_exp,log2_hdb", CASES)
def test_modified_proof_stream_fails_with_the_oracles_variant(log2_ff, security, log2_exp, log2_hdb):
    """modified_proof_stream_results_in_verification_failure (stir.rs:1967-2010): every corruption is rejected, and where
    the oracle's verifier names an LdtVerificationError the native verifier names the same one"""
    sp, cw = _instance(security, log2_ff, log2_exp, log2_hdb, (1 << log2_hdb) - 1, seed=log2_hdb)
    proof, _ = _oracle_proof(sp, cw)
    items = codec.decode_proof(proof).items
    rnd = random.Random(log2_ff * 100 + log2_hdb)
    kinds = set()
    for i, item in _corruptions(items, rnd):
        bad = _reencode(items[:i] + [item] + items[i + 1:])
        ok, why, _, _ = tvm_b200.stir_verify(security, log2_exp, log2_hdb, bad, log2_folding_factor=log2_ff)
        assert not ok, (item[0], i)
        try:
            ST.verify(codec.decode_proof(bad), sp)
            raise AssertionError("the oracle accepted a corrupted proof")
        except ValueError as e:
            want = str(e)
        if want in ("BadMerkleAuthenticationPath", "LastRoundPolynomialEvaluationMismatch", "IncorrectNumberOfRevealedLeaves",
                    "LastRoundPolynomialHasTooHighDegree"):
            assert why == "LdtVerificationError: " + want, (item[0], i, why, want)
        kinds.add(item[0])
    assert kinds >= {"MerkleRoot", "StirResponse", "Polynomial"} | ({"StirOutOfDomainValues"} if sp["round_queries"] else set())


@pytest.mark.parametrize("log2_ff,security,log2_exp,log2_hdb", [c for c in CASES if c[3] > c[0]])
def test_wrong_number_or_width_of_revealed_leaves(log2_ff, security, log2_exp, log2_hdb):
    """a StirResponse with one leaf too few (stir.rs:1174-1176), or with a leaf of k - 1 or k + 1 elements instead of k:
    IncorrectNumberOfRevealedLeaves"""
    sp, cw = _instance(security, log2_ff, log2_exp, log2_hdb, (1 << log2_hdb) - 1, seed=3)
    proof, _ = _oracle_proof(sp, cw)
    items = codec.decode_proof(proof).items
    i = next(n for n, (kind, _) in enumerate(items) if kind == "StirResponse")
    leafs, auth = items[i][1]
    k = 1 << log2_ff
    assert all(len(l) == k for l in leafs)
    for bad_leafs in (leafs[:-1], [leafs[0][:-1]] + leafs[1:], leafs[:-1] + [leafs[-1] + [leafs[-1][0]]]):
        bad = _reencode(items[:i] + [("StirResponse", (bad_leafs, auth))] + items[i + 1:])
        ok, why, _, _ = tvm_b200.stir_verify(security, log2_exp, log2_hdb, bad, log2_folding_factor=log2_ff)
        assert not ok and why == "LdtVerificationError: IncorrectNumberOfRevealedLeaves", why
    # the proof made for factor k is not a proof for factor 2k or k/2
    for other in (log2_ff - 1, log2_ff + 1):
        if other >= 2 and other <= log2_hdb:
            assert not tvm_b200.stir_verify(security, log2_exp, log2_hdb, proof, log2_folding_factor=other)[0]


@pytest.mark.parametrize("log2_ff", [3, 4, 5])
def test_verifying_arbitrary_words_does_not_crash(log2_ff):
    """verifying_arbitrary_proof_does_not_panic (stir.rs:1960-1963)"""
    rnd = random.Random(log2_ff)
    for n in (1, 2, 7, 100, 5000):
        junk = np.array([rnd.randrange(P) for _ in range(n)], dtype=np.uint64)
        assert tvm_b200.stir_verify(12, 2, 10, junk, log2_folding_factor=log2_ff)[0] is False
    # a well-formed proof of the right shape with random contents
    sp, cw = _instance(12, log2_ff, 2, 10, 100, seed=1)
    items = codec.decode_proof(_oracle_proof(sp, cw)[0]).items
    junk_items = []
    for kind, payload in items:
        if kind == "MerkleRoot":
            junk_items.append((kind, [rnd.randrange(P) for _ in range(5)]))
        elif kind in ("StirOutOfDomainValues", "Polynomial"):
            junk_items.append((kind, [tuple(rnd.randrange(1, P) for _ in range(3)) for _ in payload]))
        else:
            leafs, auth = payload
            junk_items.append((kind, ([[tuple(rnd.randrange(P) for _ in range(3)) for _ in l] for l in leafs],
                                      [[rnd.randrange(P) for _ in range(5)] for _ in auth])))
    assert tvm_b200.stir_verify(12, 2, 10, _reencode(junk_items), log2_folding_factor=log2_ff)[0] is False


# ---- the device prover ---------------------------------------------------------------------------------------------------
DEVICE_CASES = [(f, *t) for f in (3, 4, 5) for t in PARAMS[f]]


@pytest.mark.gpu
@pytest.mark.parametrize("log2_ff,security,log2_exp,log2_hdb", DEVICE_CASES)
def test_device_prover_equals_the_oracle(backend, log2_ff, security, log2_exp, log2_hdb):
    """tvm_stir_prove_k: the oracle's proof words and first-round indices, accepted by tvm_stir_verify_k; a codeword of too
    high a degree is rejected"""
    max_degree = (1 << log2_hdb) - 1
    for degree in (max_degree, max_degree // 2, -1):
        sp, cw = _instance(security, log2_ff, log2_exp, log2_hdb, degree, seed=degree + 5)
        want, want_idx = _oracle_proof(sp, cw)
        got, idx = backend.stir_prove(security, log2_exp, log2_hdb, np.array(cw, dtype=np.uint64), log2_folding_factor=log2_ff)
        assert [int(v) for v in got] == want and idx == want_idx
        ok, why, vidx, vals = tvm_b200.stir_verify(security, log2_exp, log2_hdb, got, log2_folding_factor=log2_ff)
        assert ok and vidx == idx, why
        assert [tuple(int(t) for t in v) for v in vals] == [cw[i] for i in idx]
    sp, cw = _instance(security, log2_ff, log2_exp, log2_hdb, max_degree + 1 + max_degree // 2, seed=2)
    got, _ = backend.stir_prove(security, log2_exp, log2_hdb, np.array(cw, dtype=np.uint64), log2_folding_factor=log2_ff)
    assert not tvm_b200.stir_verify(security, log2_exp, log2_hdb, got, log2_folding_factor=log2_ff)[0]


def _raw_stir_prove(backend, entry, *args, codeword):
    """one call of tvm_stir_prove / tvm_stir_prove_k (args: everything between the context and the codeword)"""
    import ctypes
    cw = np.ascontiguousarray(codeword, dtype=np.uint64)
    cap, icap = ctypes.c_size_t(1 << 22), ctypes.c_size_t(8192)
    buf, idx = np.empty(1 << 22, dtype=np.uint64), (ctypes.c_uint32 * 8192)()
    backend._chk(entry(backend._h, *args, cw.ctypes.data_as(tvm_b200._u64p), buf.ctypes.data_as(tvm_b200._u64p), ctypes.byref(cap), idx,
                       ctypes.byref(icap)))
    return buf[:cap.value].copy(), [int(idx[i]) for i in range(icap.value)]


@pytest.mark.gpu
@pytest.mark.parametrize("security,log2_exp,log2_hdb", [(8, 1, 5), (20, 2, 8), (160, 2, 12), (40, 2, 9)])
def test_factor_4_is_tvm_stir_prove(backend, security, log2_exp, log2_hdb):
    """tvm_stir_prove is tvm_stir_prove_k at log2_folding_factor 2, word for word"""
    sp, cw = _instance(security, 2, log2_exp, log2_hdb, (1 << log2_hdb) - 1, seed=log2_hdb)
    old = _raw_stir_prove(backend, backend._l.tvm_stir_prove, security, 0, log2_exp, log2_hdb, codeword=cw)
    new = _raw_stir_prove(backend, backend._l.tvm_stir_prove_k, security, 0, 2, log2_exp, log2_hdb, codeword=cw)
    assert np.array_equal(old[0], new[0]) and old[1] == new[1]
    assert [int(v) for v in new[0]] == _oracle_proof(sp, cw)[0]


@pytest.mark.gpu
def test_device_prover_parameter_errors_name_the_variant(backend):
    """parameter errors return before any kernel launch, with the variant in tvm_last_error"""
    cw = np.zeros((1 << 8, 3), dtype=np.uint64)
    for log2_ff, log2_exp, log2_hdb, want in [(1, 2, 6, "TooSmallLog2FoldingFactor"), (3, 0, 8, "TooSmallInitialExpansionFactor"),
                                              (5, 4, 4, "TooLowDegreeOfHighDegreePolynomials")]:
        before = backend.launches
        with pytest.raises(tvm_b200.TvmError) as e:
            backend.stir_prove(16, log2_exp, log2_hdb, cw, log2_folding_factor=log2_ff)
        assert e.value.code == LDT_PARAMS and str(e.value).endswith("LdtParameterError: " + want), e.value
        assert backend.launches == before


# ---- large domains, against the C-backed oracle -------------------------------------------------------------------------
def _low_degree_codeword(backend, log2_domain, log2_exp, seed):
    """[2^log2_domain, 3] canonical: an X-field polynomial of degree < 2^(log2_domain - log2_exp) on 7 * <w>, by the device
    LDE of random values"""
    vals = np.random.default_rng(seed).integers(0, P, size=(3, 1 << (log2_domain - log2_exp)), dtype=np.uint64)
    return np.ascontiguousarray(backend.lde(vals, None, log2_exp, 7).T)


@pytest.mark.gpu
@pytest.mark.parametrize("log2_ff,log2_domain", [(3, 23), (4, 23), (5, 23), (4, 25)])
def test_device_prover_at_large_domains(backend, log2_ff, log2_domain):
    """security 160, expansion 2^2: at 2^23 points the size of a padded-height-2^20 prove's STIR, word for word the C oracle;
    at 2^25 accepted by the native verifier with the prover's indices and the codeword's values"""
    log2_exp = 2
    hdb = log2_domain - log2_exp
    cw = _low_degree_codeword(backend, log2_domain, log2_exp, 0x5346 + 64 * log2_ff + log2_domain)
    got, idx = backend.stir_prove(160, log2_exp, hdb, cw, log2_folding_factor=log2_ff)
    if log2_domain <= 23:
        sp = ST.derive(160, log2_ff, log2_exp, hdb)
        assert sp["round_queries"]
        ps = codec.ProofStream()
        want_idx = fast.stir_prove(ps, corc.to_mont(cw).reshape(-1, 3), sp)
        assert idx == want_idx, "first-round indices differ"
        want = np.array(ps.encode(), dtype=np.uint64)
        if not np.array_equal(got, want):
            g, w = codec.decode_proof(got).items, codec.decode_proof(want).items
            bad = next((i for i, (a, b) in enumerate(zip(g, w)) if a != b), None)
            raise AssertionError(f"proof item {bad} differs" if bad is not None else f"{len(g)} items, the oracle has {len(w)}")
    ok, why, vidx, vals = tvm_b200.stir_verify(160, log2_exp, hdb, got, log2_folding_factor=log2_ff)
    assert ok, why
    assert vidx == idx and np.array_equal(vals, cw[np.array(idx)])
