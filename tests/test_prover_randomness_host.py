"""The prover's randomness from its 32-byte seed (stark.rs:192, 293-328; master_table.rs:423-434, 630-662, 1006-1025): the
sampler stages of triton-vm_b200/csrc/rand/prover_randomness.cuh, run by the sequential host executor of
tests/host/prover_randomness_host.cu (test infrastructure; the library instantiates the same header with the CUDA executor
only), against the oracle's StdRng restatement (oracle/rand_compat.py), which the reference's whole-proof known-answer tests
pin.  The GPU run of the same checks is tests/test_zzz_gpu_seeded_randomness.py."""
import ctypes
import json
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "triton-vm_b200", "py")]
from oracle import reference_prover as RP, stark as S   # noqa: E402
from oracle.rand_compat import StdRng, chacha_block     # noqa: E402

P = (1 << 64) - (1 << 32) + 1
M64 = (1 << 64) - 1
SRC = os.path.join(ROOT, "tests", "host", "prover_randomness_host.cu")
SO = os.path.join(ROOT, "tests", "host", "_build", "libprover_randomness_host.so")
HDR = os.path.join(ROOT, "triton-vm_b200", "csrc", "rand", "prover_randomness.cuh")
FIXTURE = os.path.join(ROOT, "tests", "golden", "short_draw_seed.json")
vp = ctypes.c_void_p


def build_host():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    stale = not os.path.exists(SO) or any(os.path.getmtime(f) > os.path.getmtime(SO) for f in (SRC, HDR))
    if stale:
        if not os.path.exists(nvcc):
            pytest.skip("nvcc not available to build the host harness")
        os.makedirs(os.path.dirname(SO), exist_ok=True)
        subprocess.run([nvcc, "-O3", "-std=c++17", "--extended-lambda", "--expt-relaxed-constexpr", "-shared", "-Xcompiler", "-fPIC",
                        SRC, "-o", SO], check=True, capture_output=True)
    return ctypes.CDLL(SO)


@pytest.fixture(scope="module")
def host():
    return build_host()


def host_stream(lib, seed, count):
    out, stats = np.zeros(count, dtype=np.uint64), np.zeros(2, dtype=np.uint64)
    assert lib.prand_host_stream(bytes(seed), ctypes.c_uint64(count), out.ctypes.data_as(vp), stats.ctypes.data_as(vp)) == 0
    return [int(v) for v in out], [int(v) for v in stats]


def host_words(lib, words, count, cap=1024):
    w = np.array(words, dtype=np.uint64)
    assert w.size == 2 * count
    out = np.zeros(count, dtype=np.uint64)
    assert lib.prand_host_words(w.ctypes.data_as(vp), ctypes.c_uint64(count), ctypes.c_uint64(cap), out.ctypes.data_as(vp)) == 0
    return [int(v) for v in out]


def host_randomness(lib, seed, n, h, nq):
    sizes = [379 * h, 91 * h * 3, n * 3, nq * 3]
    out = np.zeros(sum(sizes), dtype=np.uint64)
    assert lib.prand_host_randomness(bytes(seed), ctypes.c_uint64(n), ctypes.c_uint64(h), ctypes.c_uint64(nq), out.ctypes.data_as(vp)) == 0
    parts = np.split(out, np.cumsum(sizes)[:-1])
    return parts[0].reshape(379, h), parts[1].reshape(91, h, 3), parts[2].reshape(n, 3), parts[3].reshape(nq, 3)


def short_word(t):
    """a u64 x with lo(x p) = t: Canon draws no second u64 for it when t < 2^32"""
    return t * pow((1 - (1 << 32)) % (1 << 64), -1, 1 << 64) % (1 << 64)


def canon(words, count):
    """rand's Canon single-sample method over [0, p - 1] driven by a word list -> (samples, indices of the short samples)"""
    out, shorts, k = [], [], 0
    for j in range(count):
        prod = words[k] * P
        r, lo = prod >> 64, prod & M64
        if lo > (1 << 32) - 1:
            if lo + ((words[k + 1] * P) >> 64) > M64:
                r += 1
            k += 2
        else:
            shorts.append(j)
            k += 1
        out.append(r % P)
    return out, shorts


# ---- ChaCha12 and offset_rng_seed --------------------------------------------------------------------------------------
@pytest.mark.parametrize("counter", [0, 1, 7, (1 << 32) - 1, 1 << 32, (1 << 32) + 5, (1 << 63) + 12345, M64])
def test_chacha_blocks_match_the_oracle(host, counter):
    rng = np.random.default_rng(counter % 1000)
    for key in ([0] * 8, [0xFFFFFFFF] * 8, [int(v) for v in rng.integers(0, 1 << 32, size=8)]):
        for rounds in (12, 20):
            out = (ctypes.c_uint32 * 16)()
            host.prand_host_chacha_block((ctypes.c_uint32 * 8)(*key), ctypes.c_uint64(counter), rounds, out)
            assert list(out) == chacha_block(key, counter, 0, rounds)


@pytest.mark.parametrize("seed,offset", [(bytes(32), 0), (bytes(32), 471), (b"\xff" * 32, 1), (b"\xff" * 32, 471),
                                         (b"\xff" * 8 + bytes(24), 1), (bytes(range(32)), (1 << 64) - 1),
                                         (b"\xff" * 31 + b"\x00", 1 << 40)])
def test_offset_rng_seed_matches_the_oracle(host, seed, offset):
    out = (ctypes.c_uint8 * 32)()
    host.prand_host_offset_seed(seed, ctypes.c_uint64(offset), out)
    assert bytes(out) == RP.offset_rng_seed(seed, offset)


# ---- draw sequences ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("count", [1, 7, 8, 9, 100, 4097])
def test_bfe_draws_match_stdrng(host, count):
    for seed in (bytes(32), bytes(range(32)), b"\xff" * 32):
        r = StdRng(seed)
        assert host_stream(host, seed, count)[0] == [r.bfe() for _ in range(count)]


@pytest.mark.parametrize("xfes", [1, 3, 33])
def test_xfe_draws_match_stdrng(host, xfes):
    seed = bytes(range(1, 33))
    r = StdRng(seed)
    want = [c for _ in range(xfes) for c in r.xfe()]
    assert host_stream(host, seed, 3 * xfes)[0] == want


# ---- injected streams: short samples at chosen positions ---------------------------------------------------------------
def _stream(count, plant, seed):
    rng = np.random.default_rng(seed)
    words = [int(v) for v in rng.integers(0, 1 << 64, size=2 * count, dtype=np.uint64)]
    assert not any(canon(words, count)[1])                  # random words: no short sample of their own
    for k in plant:
        words[k] = short_word(int(rng.integers(0, 1 << 32)))
    return words


COUNT = 24
CASES = {                                                   # planted positions, expected short samples
    "position_0": ([0], [0]),
    "last_sample": ([2 * (COUNT - 1)], [COUNT - 1]),
    "two_consecutive": ([4, 5], [2, 3]),
    "both_parities": ([4, 9], [2, 5]),                      # sample 3 starts at 5, 4 at 7, 5 at 9
    "stride_2_trap": ([0, 2], [0]),                         # after the short at 0, position 2 is sample 1's SECOND u64
    "odd_without_a_short": ([3, 11], []),                   # second u64s of long samples
    "everything_short": (list(range(2 * COUNT)), list(range(COUNT))),
    "last_then_tail": ([2 * (COUNT - 1), 2 * COUNT - 1], [COUNT - 1]),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_injected_short_samples(host, case):
    plant, want_shorts = CASES[case]
    words = _stream(COUNT, plant, len(case))
    want, shorts = canon(words, COUNT)
    assert shorts == want_shorts
    assert host_words(host, words, COUNT) == want
    assert host_words(host, words, COUNT, cap=1) == want     # more flags than room: the flags are recounted


def test_injected_random_short_patterns(host):
    rng = np.random.default_rng(5)
    for trial in range(200):
        count = int(rng.integers(1, 40))
        plant = [k for k in range(2 * count) if rng.random() < 0.2]
        words = _stream(count, plant, 1000 + trial)
        want, _ = canon(words, count)
        assert host_words(host, words, count, cap=int(rng.integers(1, 8))) == want


# ---- a real seed with a short sample -----------------------------------------------------------------------------------
def fixture_seed():
    fx = json.load(open(FIXTURE))
    return bytes.fromhex(fx["seed_hex"]), fx["short_sample"]


def test_short_draw_fixture_seed(host):
    seed, j = fixture_seed()
    r = StdRng(seed)
    want = [r.bfe() for _ in range(j)]
    before = r.index + 16 * r.counter
    want.append(r.bfe())
    assert r.index + 16 * r.counter - before == 2              # the oracle's sample j consumes one u64 (two words)
    want += [r.bfe() for _ in range(300)]
    got, stats = host_stream(host, seed, len(want))
    assert stats[1] >= 1 and got == want


# ---- whole proves ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("padded_height,security", [(1 << 8, 160), (1 << 11, 32)])
def test_prover_randomness_matches_the_oracle(host, padded_height, security):
    d = S.Stark(security, 2).derive(padded_height)
    n, h, nq = d["trace_len"], d["num_trace_randomizers"], d["num_quotient_randomizer_coefficients"]
    for seed in (bytes(range(32)), b"\xff" * 32):
        got = host_randomness(host, seed, n, h, nq)
        want = RP.randomness(seed, n, h, nq)
        for g, w in zip(got, want):
            assert np.array_equal(g, w)


def test_prover_randomness_on_the_short_draw_seed(host):
    """the fixture seed is main column 0's stream: its randomizers take the short path"""
    seed, j = fixture_seed()
    d = S.Stark(160, 2).derive(1 << 8)
    n, h, nq = d["trace_len"], d["num_trace_randomizers"], d["num_quotient_randomizer_coefficients"]
    assert j < h
    got = host_randomness(host, seed, n, h, nq)
    for g, w in zip(got, RP.randomness(seed, n, h, nq)):
        assert np.array_equal(g, w)
