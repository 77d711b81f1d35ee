"""Whole proofs at the benchmark's shapes against the C + OpenMP oracle (oracle/fast.py, itself pinned to oracle/stark.py by
tests/test_oracle_fast.py and to the reference's digests by tests/test_golden.py), word for word, and the AIR quotient and
auxiliary-table extension kernels on every row.

The native verifier opens a few hundred rows, so a kernel that is wrong on a few rows still gives a proof that verifies; and a
GPU-vs-GPU comparison misses a bug both arms share.  A proof that equals the oracle's word for word does neither: every Merkle
root feeds Fiat-Shamir, so one wrong row changes every later word.  These shapes reach paths the small parity tests do not:
the tile LDE (even trace lengths 2^12..2^20) and its column/coset grouping, ntt.cu at odd lengths, the TMA row hashes, the MMA
Merkle levels above width 64, the quotient's degree split over 2^19 rows, multi-round STIR and FRI over 2^19 and 2^20
domains, and quotient domains that differ from the LDT domain.  On failure `first_difference` names the first differing proof
item, and so the stage: main LDE/hash, aux, quotient, out-of-domain rows, DEEP or the low-degree test."""
import functools
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import tvm_b200
from oracle import codec, corc, fast, reference_prover as RP, stark as S, tracegen as tg

import test_vm_programs as tvp

gpu = pytest.mark.gpu      # the CPU tests of this file (the helper, the oracle at other expansions) run without a GPU

P = (1 << 64) - (1 << 32) + 1
NM, NA = 379, 91
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEED = bytes(range(200, 232))
CLAIM = S.Claim([1, 2, 3, 4, 5], [7, 8, 9], [10])
LDT = {"auto": tvm_b200.LDT_AUTO, "fri": tvm_b200.LDT_FRI, "stir": tvm_b200.LDT_STIR}


# ---- naming the first differing proof item -------------------------------------------------------------------------------
def _item_names(items):
    """kind of each proof item; a MerkleRoot also names its commitment: main, aux, quotient, then LDT round k"""
    names, roots = [], 0
    for kind, _ in items:
        if kind == "MerkleRoot":
            names.append("MerkleRoot (%s)" % (("main", "aux", "quotient")[roots] if roots < 3 else f"LDT round {roots - 3}"))
            roots += 1
        else:
            names.append(kind)
    return names


def first_difference(got, want):
    """None if the two proofs are equal, else (index, name) of the first proof item in which they differ"""
    g, w = codec.decode_proof(got).items, codec.decode_proof(want).items
    if len(g) == len(w) and all(a == b for a, b in zip(g, w)):
        return None
    names = _item_names(w)
    for i, (a, b) in enumerate(zip(g, w)):
        if a != b:
            return i, names[i] if a[0] == b[0] else f"{names[i]} (got a {a[0]})"
    i = min(len(g), len(w))
    return i, f"{names[i]} missing" if i < len(w) else f"extra {g[i][0]}"


def _item_offsets(words):
    """word offset of each proof item's encoding (its variant index) in the proof"""
    offs, pos = [], 2
    for _ in range(int(words[1])):
        offs.append(pos + 1)
        pos += 1 + int(words[pos])
    return offs


def _oracle_threads():
    """one OpenMP thread per physical core: with two threads per core the memory-bound NTTs of the C oracle run several
    times slower on hyper-threaded hosts"""
    try:
        import psutil
        phys = psutil.cpu_count(logical=False) or 0
    except ImportError:
        phys = 0
    if phys and phys != corc.num_threads():
        corc.set_num_threads(phys)


def test_first_difference_names_the_item():
    st = S.Stark(160, 2)
    d = st.derive(16)
    rng = np.random.default_rng(16)
    r = lambda *shape: rng.integers(0, P, size=shape, dtype=np.uint64)
    n, h = d["trace_len"], d["num_trace_randomizers"]
    aux, arand = r(NA, n, 3), r(NA, h, 3)
    want = np.array(fast.prove(st, CLAIM, r(NM, n), r(NM, h), lambda ch: (aux, arand), r(d["num_quotient_randomizer_coefficients"], 3),
                               padded_height=16), dtype=np.uint64)
    assert first_difference(want, want.copy()) is None
    kinds = [k for k, _ in codec.decode_proof(want).items]
    offs = _item_offsets(want)
    roots = [i for i, k in enumerate(kinds) if k == "MerkleRoot"]
    last_ldt = kinds.index("MasterMainTableRows") - 1
    assert kinds[last_ldt] == "FriResponse"
    for item, word, name in [(roots[1], offs[roots[1]] + 3, "MerkleRoot (aux)"),          # a word inside the aux root
                             (last_ldt, offs[last_ldt + 1] - 2, "FriResponse"),           # the last word of the last LDT item
                             (roots[3], offs[roots[3]] + 1, "MerkleRoot (LDT round 0)")]:
        got = want.copy()
        got[word] = (int(got[word]) + 1) % P
        assert first_difference(got, want) == (item, name)


# ---- synthetic whole proofs at Stark::default() vs oracle/fast.py -----------------------------------------------------------
def _instance(log2_height, ldt, log2_exp):
    """random main and aux tables and randomizers of the benchmark's shape (bench.py's OracleInstance), fixed seed"""
    st = S.Stark(160, log2_exp, None if ldt == "auto" else ldt)
    d = st.derive(1 << log2_height)
    n, h = d["trace_len"], d["num_trace_randomizers"]
    rng = np.random.default_rng([0x5452_4954, log2_height, log2_exp])
    r = lambda *shape: rng.integers(0, P, size=shape, dtype=np.uint64)
    main, mrand, aux, arand = r(NM, n), r(NM, h), r(NA, n, 3), r(NA, h, 3)
    return dict(stark=st, main=main, mrand=mrand, aux=aux, arand=arand, qrand=r(d["num_quotient_randomizer_coefficients"], 3),
                padded_height=1 << log2_height)


@functools.lru_cache(maxsize=None)
def _oracle_proof(log2_height, ldt, log2_exp):
    """each shape is proved once on the CPU"""
    _oracle_threads()
    x = _instance(log2_height, ldt, log2_exp)
    return np.array(fast.prove(x["stark"], CLAIM, x["main"], x["mrand"], lambda ch: (x["aux"], x["arand"]), x["qrand"],
                               padded_height=x["padded_height"]), dtype=np.uint64)


def _device_proof(backend, log2_height, ldt, log2_exp, low_memory):
    x = _instance(log2_height, ldt, log2_exp)
    backend.set_low_memory(low_memory)
    try:
        proof = backend.prove((CLAIM.program_digest, CLAIM.input, CLAIM.output), x["main"], x["mrand"], lambda ch: (x["aux"], x["arand"]),
                              x["qrand"], 160, log2_exp, x["padded_height"], LDT[ldt])
        assert backend.last_prove_low_memory == (low_memory == 1)
    finally:
        backend.set_low_memory(0)
    return proof


CACHED, JUST_IN_TIME = 2, 1


@gpu
@pytest.mark.parametrize("log2_height,ldt,log2_exp,low_memory", [
    (12, "auto", 2, CACHED),            # tile LDE, 6 x 6
    (14, "auto", 2, CACHED),            # tile LDE, 8 x 6
    (13, "auto", 2, CACHED),            # ntt.cu at the odd lengths the tiles skip
    (15, "auto", 2, CACHED),
    (16, "auto", 2, CACHED),            # the benchmark's 2^16 config: 10 x 6 tiles, degree split over 2^19 rows, multi-round STIR
    (16, "auto", 2, JUST_IN_TIME),
    (16, "fri", 2, CACHED),             # FRI folds, leaves and gathers at 2^19
    (17, "stir", 2, CACHED),            # odd trace length at scale: ntt.cu LDE, 2^20 LDT domain
    (14, "fri", 1, CACHED),             # LDT domain 2^16 < quotient domain 2^17
    (14, "fri", 4, CACHED),             # LDT domain 2^19 > quotient domain 2^17
])
def test_whole_proof_equals_the_oracle(backend, log2_height, ldt, log2_exp, low_memory):
    want = _oracle_proof(log2_height, ldt, log2_exp)
    got = _device_proof(backend, log2_height, ldt, log2_exp, low_memory)
    assert np.array_equal(got, want), f"first differing proof item: {first_difference(got, want)}"
    assert tvm_b200.verify((CLAIM.program_digest, CLAIM.input, CLAIM.output), got, 160, log2_exp, ldt_choice=LDT[ldt],
                           skip_air_check=True) == (True, "")


@pytest.mark.parametrize("log2_exp", [1, 4])
def test_fast_oracle_equals_the_python_oracle_at_expansion(log2_exp):
    """tests/test_oracle_fast.py pins fast.prove at expansion 4 only; the two expansions above rest on this"""
    st = S.Stark(160, log2_exp, "fri")
    d = st.derive(16)
    rng = np.random.default_rng(log2_exp)
    r = lambda *shape: rng.integers(0, P, size=shape, dtype=np.uint64)
    n, h = d["trace_len"], d["num_trace_randomizers"]
    main, mrand, aux, arand = r(NM, n), r(NM, h), r(NA, n, 3), r(NA, h, 3)
    qrand = r(d["num_quotient_randomizer_coefficients"], 3)
    want, _ = S.prove(st, CLAIM, main, mrand, lambda ch: (aux, arand), qrand, padded_height=16)
    got = fast.prove(st, CLAIM, main, mrand, lambda ch: (aux, arand), qrand, padded_height=16)
    assert got == want, f"first differing proof item: {first_difference(got, want)}"


# ---- a real program at 2^16: the device fills, extends and draws the randomness itself ---------------------------------------
@gpu
def test_spin_16_equals_the_oracle_from_the_aet_and_seed(backend):
    """ProgramToBench::spin(16) at Stark::default(), the first BASELINE.json config: the oracle proves its own table fill,
    extension and randomness; the device gets only the AET and the seed"""
    _oracle_threads()
    words = tg.assemble(tvp.SPIN)
    inst = RP.instance(S.Stark(160, 2), words, [16], SEED)
    assert inst["padded_height"] == 1 << 16
    want = np.array(fast.prove(inst["stark"], inst["claim"], inst["main"], inst["main_rand"], inst["extend"], inst["quot_rand"],
                               padded_height=inst["padded_height"]), dtype=np.uint64)
    claim = (inst["claim"].program_digest, inst["claim"].input, inst["claim"].output)
    got = backend.prove_aet_seeded(claim, tg.aet_arrays(words, inst["execution"]), SEED, 1 << 16)
    assert np.array_equal(got, want), f"first differing proof item: {first_difference(got, want)}"
    assert tvm_b200.verify(claim, got) == (True, "")


# ---- process-wide variants at 2^16, each in a fresh interpreter -------------------------------------------------------------
@gpu
@pytest.mark.parametrize("env", [
    # tile_tmp_budget(): 1 MB = 2^17 words.  At trace length 2^16 that holds 2 cosets of one column (cos_per = 2 of the 8
    # cosets, group = 1, the coset-split launch pairs), the grouping the default 16 MB budget (2^21 words) selects only at
    # trace length 2^20; at 2^16 the default puts all 8 cosets of 4 columns in one pair
    {"TVM_NTT_TMP_MB": "1"},
    # the quotient without the degree split: both AIR paths must give the same proof at the production shape
    {"TVM_AIR_NO_DEGREE_SPLIT": "1"},
], ids=["ntt_tmp_1mb", "no_degree_split"])
def test_variant_proof_equals_the_oracle(env, tmp_path):
    """both variables are read once per process"""
    out = str(tmp_path / "proof.npy")
    code = """
import sys, numpy as np
sys.path[:0] = [%r, %r, %r]
import tvm_b200
import test_zzzzz_gpu_production_shapes as M
b = tvm_b200.Backend(0)
np.save(%r, M._device_proof(b, 16, "auto", 2, M.CACHED))
b.close()
""" % (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "triton-vm_b200", "py"), out)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=900, env=dict(os.environ, **env))
    assert r.returncode == 0, r.stderr[-2000:]
    got, want = np.load(out), _oracle_proof(16, "auto", 2)
    assert np.array_equal(got, want), f"first differing proof item: {first_difference(got, want)}"


# ---- kernels on every row -------------------------------------------------------------------------------------------------
def _mont_max(shape):
    """canonical values whose Montgomery words are p - 1: every 128-bit product summed into the quotient's unreduced
    accumulator (AirAcc) is as large as it gets, and so is its carry count"""
    return corc.from_mont(np.full(shape, P - 1, dtype=np.uint64)).reshape(shape)


def _alternating(shape, log_r):
    """columns alternating between 0 and Montgomery p - 1 along the trace (row i and its next row i + r differ), with
    neighbouring columns out of phase"""
    ncols, rn = shape
    k = np.arange(rn) >> log_r
    on = ((k[None, :] + np.arange(ncols)[:, None]) & 1).astype(bool)
    return np.where(on, _mont_max(shape), np.uint64(0))


@gpu
@pytest.mark.parametrize("kind", ["random", "mont_max", "alternating"])
@pytest.mark.parametrize("log_n,log_r", [(10, 3), (12, 3), (11, 2)])
def test_air_quotient_on_every_row(backend, log_n, log_r, kind):
    n, r = 1 << log_n, 1 << log_r
    rn = n * r
    rng = np.random.default_rng([log_n, log_r, len(kind)])
    rand = lambda *shape: rng.integers(0, P, size=shape, dtype=np.uint64)
    ch = rand(63, 3)
    if kind == "random":
        main, aux, w = rand(NM, rn), rand(270, rn), rand(604, 3)
    elif kind == "mont_max":
        main, aux, w = _mont_max((NM, rn)), _mont_max((270, rn)), _mont_max((604, 3))
    else:
        main, aux, w = _alternating((NM, rn), log_r), _alternating((270, rn), log_r), _mont_max((604, 3))
    want = corc.air_quotient(main, aux, log_n, 7, ch, w)                          # natural order: row i at 7 * w_rn^i
    # the device reads and writes coset-major memory: index c * n + k holds row i = c + r * k
    to_mem = lambda t: np.ascontiguousarray(t.reshape(t.shape[0], n, r).transpose(0, 2, 1).reshape(t.shape[0], rn))
    dev = torch.device("cuda:0")
    d_main = torch.from_numpy(to_mem(main).view(np.int64)).to(dev)
    d_aux = torch.from_numpy(to_mem(aux).view(np.int64)).to(dev)
    backend.to_mont_(d_main); backend.to_mont_(d_aux)
    d_out = torch.zeros((3, rn), dtype=torch.int64, device=dev)
    backend.air_quotient_dev(d_main, rn, d_aux, rn, ch, w, log_n, log_r, 7, d_out, rn)
    backend.from_mont_(d_out)
    backend.synchronize()
    got = d_out.cpu().numpy().view(np.uint64).reshape(3, r, n).transpose(2, 1, 0).reshape(rn, 3)
    bad = np.nonzero((got != want).any(axis=1))[0]
    assert bad.size == 0, f"{bad.size} of {rn} rows differ; first: row {bad[0]} (coset {bad[0] % r}, k = {bad[0] // r})"


@gpu
@pytest.mark.parametrize("log_n", [16, 17])       # 256 and 512 scan chunks
def test_aux_extension_on_every_row(backend, log_n):
    n = 1 << log_n
    rng = np.random.default_rng(log_n)
    T = rng.integers(0, P, size=(NM, n), dtype=np.uint64)
    ch = rng.integers(0, P, size=(63, 3), dtype=np.uint64)
    rc = rng.integers(0, P, size=(n, 3), dtype=np.uint64)
    want = corc.aux_extend(T, ch, rc)
    got = backend.aux_extend(T, ch, rc)
    bad = [q for q in range(NA) if not np.array_equal(got[q], want[q])]
    where = {q: (int(np.nonzero((got[q] != want[q]).any(axis=1))[0][0]), int((got[q] != want[q]).any(axis=1).sum())) for q in bad[:8]}
    assert bad == [], f"columns {bad} differ; (first bad row, #bad rows) = {where}"
