"""The LDE, NTT, row-hashing, Merkle, STIR and FRI kernels and the just-in-time prove at the sizes of padded heights 2^20 to
2^23, word for word against the C oracle (oracle/corc.py, oracle/fast.py).

The library proves padded heights whose tables do not fit one H100 (from 2^21 on) in just-in-time (JIT) mode, and ntt.cu
serves every transform the tile kernels of ntt_tile.cu do not: all LDEs of trace length above 2^20 and plain transforms
up to 2^26 points.  The smaller tests of these kernels stop at 2^20 (2^17 for whole proofs against the oracle), so the
tile shapes, coset subsets, tree levels and domain sizes only these heights reach are checked here.  Where an
oracle-side pass over the whole output would take minutes (the 2^24-row tables, the 2^26-leaf tree), the check covers a
seeded sample plus the rows or levels where an index computation is most likely to go wrong.  Every failure names the
first bad column, coset, row, node or proof item."""
import functools
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import tvm_b200
from oracle import codec, corc, fast, stir as ST

import test_fri_properties as TF
import test_zzzzz_gpu_production_shapes as PS

pytestmark = pytest.mark.gpu

P = (1 << 64) - (1 << 32) + 1
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEED = bytes(range(200, 232))
DEV = torch.device("cuda:0")


@pytest.fixture(scope="module", autouse=True)
def _oracle_cores():
    PS._oracle_threads()


@pytest.fixture
def backend(backend):
    """a context of its own for every test: the gigabytes of scratch and pooled memory these sizes leave in a context go
    back to the device when the test ends, so that the whole proofs below, in interpreters of their own, find it free.  The
    suite's shared context (the fixture this one overrides) first gives back what earlier tests left in its pool."""
    backend.release_cached_memory()
    torch.cuda.empty_cache()
    b = tvm_b200.Backend(0)
    yield b
    b.close()
    torch.cuda.empty_cache()


def _rand(log2n, ncols, seed):
    return np.random.default_rng(seed).integers(0, P, size=(ncols, 1 << log2n), dtype=np.uint64)


def _dev_random(shape, seed):
    """uniform words below 2^64 - 2^32 (< p, so canonical and also valid Montgomery forms) generated on the device"""
    g = torch.Generator(device=DEV)
    g.manual_seed(seed)
    hi = torch.randint(0, (1 << 32) - 1, shape, dtype=torch.int64, device=DEV, generator=g)
    lo = torch.randint(0, 1 << 32, shape, dtype=torch.int64, device=DEV, generator=g)
    out = (hi << 32) | lo
    torch.cuda.synchronize()        # the library runs on a stream of its own, unordered with torch's
    return out


def _first_bad(got, want):
    """index of the first differing entry along the last axis of two equal-shape arrays (rows of a 2-D array), or None"""
    bad = np.nonzero(got != want)[0] if got.ndim == 1 else np.nonzero((got != want).any(axis=tuple(range(1, got.ndim))))[0]
    return (int(bad[0]), int(bad.size)) if bad.size else None


# ---- 1. plain NTT at every two-pass split above 2^20 ----------------------------------------------------------------------------
# ntt_run: LB = ceil(L/2), LA = L - LB; rows per CTA (pick_log_t) 8 for a tile of <= 2^11 points, 4 for 2^12, 2 for 2^13.
#   L   LA  LB   pass-A rows/CTA   pass-B rows/CTA
#   21  10  11   8                 8
#   22  11  11   8                 8
#   23  11  12   8                 4
#   24  12  12   4                 4
#   26  13  13   2                 2          (L = 20 and 25 are in test_gpu_kernels.py)
@pytest.mark.parametrize("inverse", [False, True])
@pytest.mark.parametrize("log2n", [21, 22, 23, 24, 26])
def test_ntt_above_2_20(backend, log2n, inverse):
    x = _rand(log2n, 1, 0x4E54 + log2n)
    got = backend.ntt(x, inverse=inverse)[0]
    want = corc.ntt(x[0], inverse=inverse)
    bad = _first_bad(got, want)
    assert bad is None, f"2^{log2n} {'inverse' if inverse else 'forward'}: first bad index {bad[0]} of {bad[1]} bad"


# ---- 2. column LDE through ntt.cu: randomizer fold, coset pre-scale, coset subsets ---------------------------------------------
R, LOG_R, OFFSET, LDE_COLS = 8, 3, 7, 2


def _lde_case(log2n, h):
    """(trace, randomizers, the oracle's natural-order LDE [ncols, n, 8]: row c + 8k at [:, k, c])"""
    rng = np.random.default_rng([0x4C44, log2n, h])
    n = 1 << log2n
    trace = rng.integers(0, P, size=(LDE_COLS, n), dtype=np.uint64)
    rand = rng.integers(0, P, size=(LDE_COLS, h), dtype=np.uint64) if h else None
    want = corc.lde_table(trace, rand, OFFSET, log2n + LOG_R).reshape(LDE_COLS, n, R)
    return trace, rand, want


_lde_case_kept = functools.lru_cache(maxsize=None)(_lde_case)   # the 2^21 and 2^22 cases the coset-subset test reuses


def _lde_mismatch(got, want):
    """got, want [ncols, n, cosets] -> None, or a message naming the first bad column, coset and row"""
    for q in range(got.shape[0]):
        for c in range(got.shape[2]):
            bad = _first_bad(got[q, :, c], want[q, :, c])
            if bad:
                return f"column {q}, coset {c}: first bad k = {bad[0]} (row {c + R * bad[0]}), {bad[1]} bad rows"
    return None


@pytest.mark.parametrize("h", [0, 228])
@pytest.mark.parametrize("log2n", [21, 22, 23])
def test_lde_through_ntt_cu(backend, log2n, h):
    """Backend.lde at trace lengths the tile kernels do not take: 8 cosets, offset 7, with and without the randomizer fold
    (228 trace randomizers, the 2^20 STIR prove's count)"""
    trace, rand, want = (_lde_case_kept if h and log2n <= 22 else _lde_case)(log2n, h)
    got = backend.lde(trace, rand, LOG_R, OFFSET).reshape(LDE_COLS, 1 << log2n, R)
    msg = _lde_mismatch(got, want)
    assert msg is None, f"2^{log2n}, h = {h}: {msg}"


@pytest.mark.parametrize("log2n", [21, 22])
def test_lde_coset_subsets_through_ntt_cu(backend, log2n):
    """lde_cosets_dev on the subsets a prove evaluates: one coset at a time (a JIT prove's coset loop) and every rank's share
    of a coset-sharded prove, against the oracle's full LDE"""
    h = 228
    trace, rand, want = _lde_case_kept(log2n, h)
    n = 1 << log2n
    d_trace = torch.from_numpy(trace.view(np.int64)).to(DEV)
    d_rand = torch.from_numpy(rand.view(np.int64)).to(DEV)
    d_coef = torch.empty((LDE_COLS, 2 * n), dtype=torch.int64, device=DEV)
    d_tmp = torch.empty((LDE_COLS, R * n), dtype=torch.int64, device=DEV)
    torch.cuda.synchronize()        # the library runs on a stream of its own, unordered with torch's
    backend.to_mont_(d_trace)
    backend.to_mont_(d_rand)
    subsets = [(c, 1, 1) for c in range(R)] + [(1, 2, 4), (3, 4, 2), (2, 3, 2), (0, 1, 8)]
    for first, step, count in subsets:
        d_out = torch.empty((LDE_COLS, count * n), dtype=torch.int64, device=DEV)
        backend.lde_cosets_dev(d_trace, d_rand, h, log2n, LOG_R, OFFSET, first, step, count, LDE_COLS, d_coef, d_out, d_tmp)
        backend.from_mont_(d_out)
        backend.synchronize()
        got = d_out.cpu().numpy().view(np.uint64).reshape(LDE_COLS, count, n).transpose(0, 2, 1)
        cosets = [first + step * y for y in range(count)]
        msg = _lde_mismatch(got, want[:, :, cosets])
        assert msg is None, f"2^{log2n}, cosets {cosets}: {msg} (coset index within the subset)"


# ---- 3. row hashing of coset-major tables of 2^24 rows (8 cosets x 2^21) ---------------------------------------------------------
HASH_LOG_ROWS = 24


def _hash_sample_rows():
    """memory rows m = c * 2^21 + k: the last 2^12 rows k of every coset, plus 2^16 seeded rows"""
    per = 1 << (HASH_LOG_ROWS - LOG_R)
    tail = np.concatenate([c * per + np.arange(per - 4096, per) for c in range(R)])
    sample = np.random.default_rng(0x5257).integers(0, 1 << HASH_LOG_ROWS, size=1 << 16)
    return np.unique(np.concatenate([tail, sample]))


@pytest.mark.parametrize("kernel,pad", [("tma", 2), ("per_lane_load", 1)])
@pytest.mark.parametrize("ncols", [10, 11, 20])
def test_hash_rows_coset_major_2_24(backend, ncols, kernel, pad):
    """random canonical words with a column stride of 2^24 + 2 (16-byte aligned columns: the TMA-staged kernel) or 2^24 + 1
    (8-byte aligned, which hash_rows_run's tma_ok rejects: the per-lane-load kernel)"""
    nrows = 1 << HASH_LOG_ROWS
    stride = nrows + pad
    table = _dev_random((ncols, stride), 0x4854 + ncols)
    m = _hash_sample_rows()
    per = nrows >> LOG_R
    natural = (m // per) + R * (m % per)        # digests are stored in natural row order: row c + 8k
    rows = np.ascontiguousarray(table[:, torch.from_numpy(m).to(DEV)].cpu().numpy().view(np.uint64))
    backend.to_mont_(table)
    d_dig = torch.empty((nrows, 5), dtype=torch.int64, device=DEV)
    backend.hash_rows_dev(table, stride, nrows, ncols, LOG_R, d_dig)
    backend.from_mont_(d_dig)
    backend.synchronize()
    got = d_dig[torch.from_numpy(natural).to(DEV)].cpu().numpy().view(np.uint64)
    del d_dig, table
    want = corc.hash_rows_colmajor(rows)
    bad = _first_bad(got, want)
    if bad:
        i = bad[0]
        small = np.array_equal(backend.hash_rows(rows[:, :300]), want[:300])   # the same rows through the small-table path
        pytest.fail(f"{kernel}, {ncols} columns: coset {m[i] // per}, k = {m[i] % per} (row {natural[i]}) differs; {bad[1]} of "
                    f"{m.size} checked rows bad (their first 300 through tvm_tip5_hash_rows: {'equal' if small else 'also bad'})")


# ---- 4. Merkle trees of 2^24 and 2^26 leaves -----------------------------------------------------------------------------------
def _node_name(i):
    lvl = int(i).bit_length() - 1
    return f"node {i} (level of width 2^{lvl}, index {i - (1 << lvl)})"


def test_merkle_2_24_whole_tree(backend):
    nl = 1 << 24
    d_nodes = torch.zeros((2 * nl, 5), dtype=torch.int64, device=DEV)
    d_nodes[nl:] = _dev_random((nl, 5), 0x4D24)
    torch.cuda.synchronize()
    backend.merkle_dev(d_nodes, nl)
    backend.synchronize()
    nodes = d_nodes.cpu().numpy().view(np.uint64)
    del d_nodes
    want = corc.merkle_build(nodes[nl:], mont_io=True)
    bad = _first_bad(nodes[1:nl], want[1:nl])
    assert bad is None, f"{_node_name(bad[0] + 1)} differs; {bad[1]} bad nodes"


def _pair_hashes(children):
    """[2k, 5] Montgomery children (k a power of two) -> [k, 5]: the oracle's Tip5 pair hash of rows 2j and 2j + 1"""
    k = children.shape[0] // 2
    return corc.merkle_build(np.ascontiguousarray(children), mont_io=True)[k:2 * k]


def test_merkle_2_26_levels(backend):
    """every node of the levels of width <= 2^12; on every wider level, down to the one hashed from the leaves, its first
    and last 64 nodes and a seeded sample, 4096 in all, recomputed from their two stored children"""
    log_nl = 26
    nl = 1 << log_nl
    d_nodes = torch.zeros((2 * nl, 5), dtype=torch.int64, device=DEV)
    d_nodes[nl:] = _dev_random((nl, 5), 0x4D26)
    torch.cuda.synchronize()
    backend.merkle_dev(d_nodes, nl)
    backend.synchronize()
    top = d_nodes[:1 << 14].cpu().numpy().view(np.uint64)
    want = corc.merkle_build(top[1 << 13:], mont_io=True)
    bad = _first_bad(top[1:1 << 13], want[1:1 << 13])
    assert bad is None, f"{_node_name(bad[0] + 1)} differs; {bad[1]} bad nodes"
    rng = np.random.default_rng(0x4D53)
    for lvl in range(13, log_nl):
        w = 1 << lvl
        inner = 64 + rng.choice(w - 128, size=4096 - 128, replace=False)
        idx = w + np.sort(np.concatenate([np.arange(64), inner, np.arange(w - 64, w)]))
        kids = np.stack([2 * idx, 2 * idx + 1], axis=1).reshape(-1)
        got = d_nodes[torch.from_numpy(idx).to(DEV)].cpu().numpy().view(np.uint64)
        ch = d_nodes[torch.from_numpy(kids).to(DEV)].cpu().numpy().view(np.uint64)
        bad = _first_bad(got, _pair_hashes(ch))
        assert bad is None, f"{_node_name(idx[bad[0]])} is not the hash of its children; {bad[1]} of 4096 sampled bad"
    del d_nodes
    torch.cuda.empty_cache()


# ---- 5. stand-alone STIR and FRI at the LDT domains of 2^20..2^23 proves ---------------------------------------------------------
SECURITY, LOG_EXP = 160, 2


def _low_degree_codeword(backend, log2_domain, offset, seed):
    """[2^log2_domain, 3] canonical: an X-field polynomial of degree < 2^(log2_domain - 2) on offset * <w>, by the device
    LDE of random trace-domain values (its correctness is what test_lde_through_ntt_cu checks)"""
    log2n = log2_domain - LOG_EXP
    vals = _rand(log2n, 3, seed)
    return np.ascontiguousarray(backend.lde(vals, None, LOG_EXP, offset).T)


def _proof_mismatch(got, want):
    if np.array_equal(got, want):
        return None
    g, w = codec.decode_proof(got).items, codec.decode_proof(want).items
    for i, (a, b) in enumerate(zip(g, w)):
        if a != b:
            return f"proof item {i} ({b[0]}) differs"
    return f"{len(g)} proof items, the oracle has {len(w)}"


@pytest.mark.parametrize("log2_domain", [23, 24])
def test_stir_prove_equals_the_oracle(backend, log2_domain):
    hdb = log2_domain - LOG_EXP
    sp = ST.derive(SECURITY, 2, LOG_EXP, hdb)
    cw = _low_degree_codeword(backend, log2_domain, sp["initial_offset"], 0x5354 + log2_domain)
    got, idx = backend.stir_prove(SECURITY, LOG_EXP, hdb, cw)
    ps = codec.ProofStream()
    want_idx = fast.stir_prove(ps, corc.to_mont(cw).reshape(-1, 3), sp)
    want = np.array(ps.encode(), dtype=np.uint64)
    assert idx == want_idx, "first-round indices differ"
    msg = _proof_mismatch(got, want)
    assert msg is None, msg


@pytest.mark.parametrize("log2_domain", [23, 24])
def test_fri_prove_equals_the_oracle(backend, log2_domain):
    hdb = log2_domain - LOG_EXP
    d = TF.oracle_fri_derive(SECURITY, LOG_EXP, hdb)
    cw = _low_degree_codeword(backend, log2_domain, d["ldt_offset"], 0x4652 + log2_domain)
    got, idx = backend.fri_prove(SECURITY, LOG_EXP, hdb, cw)
    ps = codec.ProofStream()
    want_idx = fast.fri_prove(ps, corc.to_mont(cw).reshape(-1, 3), d)
    want = np.array(ps.encode(), dtype=np.uint64)
    assert idx == want_idx, "first-round indices differ"
    msg = _proof_mismatch(got, want)
    assert msg is None, msg


@pytest.mark.parametrize("log2_domain", [25, 26])
def test_stir_and_fri_verify_at_large_domains(backend, log2_domain):
    """the native verifiers accept the device proofs of a low-degree codeword and return the prover's indices; at 2^26 they
    reject a codeword of too high a degree"""
    hdb = log2_domain - LOG_EXP
    cw = _low_degree_codeword(backend, log2_domain, 7, 0x5646 + log2_domain)
    for name, prove, verify in [("STIR", backend.stir_prove, tvm_b200.stir_verify), ("FRI", backend.fri_prove, tvm_b200.fri_verify)]:
        proof, idx = prove(SECURITY, LOG_EXP, hdb, cw)
        ok, why, vidx, vals = verify(SECURITY, LOG_EXP, hdb, proof)
        assert ok, f"{name} 2^{log2_domain}: rejected: {why}"
        assert vidx == idx, f"{name} 2^{log2_domain}: the verifier's indices differ from the prover's"
        assert np.array_equal(vals, cw[np.array(idx)]), f"{name} 2^{log2_domain}: revealed values differ from the codeword"
    if log2_domain == 26:
        high = np.ascontiguousarray(_rand(log2_domain, 3, 0x4844).T)      # random values: degree ~ 2^26 > 2^24 - 1
        for name, prove, verify in [("STIR", backend.stir_prove, tvm_b200.stir_verify), ("FRI", backend.fri_prove, tvm_b200.fri_verify)]:
            ok, _, _, _ = verify(SECURITY, LOG_EXP, hdb, prove(SECURITY, LOG_EXP, hdb, high)[0])
            assert not ok, f"{name} 2^{log2_domain}: a codeword of too high a degree was accepted"


# ---- 6. whole proofs, each in a fresh interpreter ---------------------------------------------------------------------------------
def _run_fresh(code, tmp_path, timeout=1200):
    """run `code` in a new interpreter with the tests' import paths; it prints one JSON line last"""
    prelude = "import sys, json, time, numpy as np\nsys.path[:0] = [%r, %r, %r]\n" % (
        ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "triton-vm_b200", "py"))
    r = subprocess.run([sys.executable, "-c", prelude + code], capture_output=True, text=True, timeout=timeout, cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def test_jit_proof_equals_the_cached_proof_at_2_20(backend, tmp_path):
    """bench.py-shaped synthetic tables under Stark::default() at padded height 2^20: the just-in-time proof is the cached
    proof word for word, and the native verifier accepts it (AIR identity skipped: the tables are random)"""
    proofs = {}
    for name, mode in [("cached", PS.CACHED), ("jit", PS.JUST_IN_TIME)]:
        out = str(tmp_path / f"{name}.npy")
        _run_fresh("""
import tvm_b200
import test_zzzzz_gpu_production_shapes as M
b = tvm_b200.Backend(0)
np.save(%r, M._device_proof(b, 20, "auto", 2, %d))
b.close()
print(json.dumps({}))
""" % (out, mode), tmp_path)
        proofs[name] = np.load(out)
    jit, cached = proofs["jit"], proofs["cached"]
    assert np.array_equal(jit, cached), f"first differing proof item: {PS.first_difference(jit, cached)}"
    assert tvm_b200.verify((PS.CLAIM.program_digest, PS.CLAIM.input, PS.CLAIM.output), jit, 160, 2,
                           skip_air_check=True) == (True, "")


def test_spin_2_21_proves_just_in_time_and_verifies_with_the_air(backend, tmp_path):
    """ProgramToBench::spin(21): its tables exceed one H100, so the automatic mode must choose JIT; the proof verifies with
    the AIR identity, and forcing JIT gives the same words"""
    proofs = {}
    for name, mode in [("auto", 0), ("jit", 1)]:
        out = str(tmp_path / f"{name}.npy")
        res = _run_fresh("""
import tvm_b200
from oracle import tracegen as tg
import test_vm_programs as tvp
b = tvm_b200.Backend(0)
b.set_low_memory(%d)
t0 = time.perf_counter()
claim, proof = b.prove_program(tg.assemble(tvp.SPIN), [21], seed=%r)
seconds = time.perf_counter() - t0
np.save(%r, proof)
print(json.dumps(dict(claim=[list(map(int, claim[0])), list(map(int, claim[1])), list(map(int, claim[2]))],
                      low_memory=b.last_prove_low_memory, seconds=seconds)))
b.close()
""" % (mode, SEED, out), tmp_path)
        proofs[name] = np.load(out)
        assert res["low_memory"], f"{name}: the 2^21 prove did not run just in time"
        claim = tuple(res["claim"])
        print(f"spin(21), low-memory mode {mode}: prove_program {res['seconds']:.1f} s")
    auto, jit = proofs["auto"], proofs["jit"]
    assert tvm_b200.proof_padded_height(auto) == 1 << 21
    assert tvm_b200.verify(claim, auto) == (True, "")
    assert np.array_equal(auto, jit), f"first differing proof item: {PS.first_difference(jit, auto)}"
