"""Several contexts proving on one GPU at the same time, each driven by its own thread (DESIGN.md §6j).  The generated AIR kernels
read their weights and challenges from constant memory, which all contexts of a device share; the library hands it to one
context at a time.  Every test makes its own Backends, starts its threads behind a barrier, and asserts that the calls' host
time windows overlapped, so that a run whose calls happened one after another cannot pass.  Results must equal the known
answers, or what the same context computes alone."""
import os
import subprocess
import threading
import time

import numpy as np
import pytest

import tvm_b200
from oracle import reference_prover as RP, tip5, tracegen as tg
from oracle.rand_compat import StdRng

import test_golden as TG
import test_vm_programs as tvp
from test_air_check import P, sampled_challenges
from test_program_execution import every_instruction_inputs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEED = bytes(range(100, 132))
SPIN = tg.assemble(tvp.SPIN)


def run_concurrently(calls):
    """calls[i]() on thread i, all released by one barrier -> (results, host time windows); re-raises a thread's exception"""
    barrier = threading.Barrier(len(calls))
    results, windows, errors = [None] * len(calls), [None] * len(calls), []

    def worker(i):
        barrier.wait()
        t0 = time.perf_counter()
        try:
            results[i] = calls[i]()
        except BaseException as e:  # noqa: BLE001
            errors.append(e)
        windows[i] = (t0, time.perf_counter())
    threads = [threading.Thread(target=worker, args=(i,)) for i in range(len(calls))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    if errors:
        raise errors[0]
    return results, windows


def assert_overlapped(windows):
    """every call was still running when the last one started"""
    assert max(w[0] for w in windows) < min(w[1] for w in windows), windows


def backends(k):
    return [tvm_b200.Backend(0) for _ in range(k)]


def close(bs):
    for b in bs:
        b.close()


# ---- 1: known-answer digests -------------------------------------------------------------------------------------------------
_SPIN_FIXTURES = None


def _spin_fixture(name):
    global _SPIN_FIXTURES
    if _SPIN_FIXTURES is None:
        import json
        _SPIN_FIXTURES = json.load(open(os.path.join(ROOT, "tests", "golden", "spin_digests.json")))
    return _SPIN_FIXTURES[name]


def _kat_jobs():
    """[(name, prove(backend) -> proof, want digest, want length or None)]: proof.rs:200-226 (FRI), stark.rs:2433-2460
    (security 32), spin_13 (FRI) and spin_16 (STIR) of tests/golden/spin_digests.json, through the entry points of the
    existing tests of each"""
    ref_words = tg.assemble(TG.REFERENCE_PROGRAM)
    ref_digest = [int(v) for v in tip5.hash_varlen(ref_words)]
    ref_seed = RP.seed_from_rng(StdRng.seed_from_u64(TG.REFERENCE_SEED_OF_SEED))
    every_words = tg.assemble(TG.EVERY_INSTRUCTION_PROGRAM)
    inp, sec, ram, digests = every_instruction_inputs()
    every_seed = RP.seed_from_rng(StdRng.seed_from_u64(TG.EVERY_INSTRUCTION_SEED_OF_SEED))
    jobs = [("proof.rs", lambda b: b.prove_program(ref_words, ref_digest, seed=ref_seed)[1], TG.REFERENCE_PROOF_DIGEST, None),
            ("every_instruction", lambda b: b.prove_program(every_words, inp, sec, digests, ram, seed=every_seed, security_level=32)[1],
             TG.EVERY_INSTRUCTION_PROOF_DIGEST, None)]
    for name, ldt in (("spin_13", "fri"), ("spin_16", "stir")):
        inst = tvp.program_instance(tvp.SPIN, [int(name.split("_")[1])], 160, None)
        fixture = _spin_fixture(name)
        assert inst["derived"]["ldt"] == fixture["ldt"] == ldt
        blank = inst["main"].copy()
        blank[149:] = 0
        c = inst["claim"]

        def prove(b, inst=inst, blank=blank, c=c):
            return b.prove_tables((c.program_digest, c.input, c.output), blank, inst["main_rand"], inst["aux_rand"],
                                  inst["randomizer_column"], inst["quot_rand"], security_level=160, log2_expansion=2,
                                  padded_height=inst["padded_height"])
        jobs.append((name, prove, fixture["tip5_digest"], fixture["proof_words"]))
    return jobs


@pytest.mark.gpu
def test_known_answer_digests_under_concurrency():
    jobs = _kat_jobs()
    bs = backends(4)
    try:
        for rotation in range(2):
            assign = [jobs[(i + rotation) % 4] for i in range(4)]
            proofs, windows = run_concurrently([lambda b=b, job=job: job[1](b) for b, job in zip(bs, assign)])
            assert_overlapped(windows)
            for (name, _, digest, length), proof in zip(assign, proofs):
                assert RP.proof_digest([int(v) for v in proof]) == digest, (rotation, name)
                assert length is None or len(proof) == length, (rotation, name)
    finally:
        close(bs)


# ---- 2 and 3: the same instance on several contexts ----------------------------------------------------------------------------
@pytest.mark.gpu
def test_same_instance_on_four_contexts():
    bs = backends(4)
    try:
        claim, alone = bs[0].prove_program(SPIN, [16], seed=SEED)
        proofs, windows = run_concurrently([lambda b=b: b.prove_program(SPIN, [16], seed=SEED) for b in bs])
        assert_overlapped(windows)
        for got_claim, proof in proofs:
            assert got_claim == claim and np.array_equal(proof, alone)
        assert tvm_b200.verify(claim, alone) == (True, "")
    finally:
        close(bs)


@pytest.mark.gpu
def test_just_in_time_and_cached_side_by_side():
    jit, cached = backends(2)
    try:
        jit.set_low_memory(1)
        cached.set_low_memory(2)
        _, alone = cached.prove_program(SPIN, [16], seed=SEED)
        proofs, windows = run_concurrently([lambda b=b: b.prove_program(SPIN, [16], seed=SEED)[1] for b in (jit, cached)])
        assert_overlapped(windows)
        assert jit.last_prove_low_memory and not cached.last_prove_low_memory
        assert np.array_equal(proofs[0], alone) and np.array_equal(proofs[1], alone)
    finally:
        close((jit, cached))


# ---- 4: the constant banks directly --------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_air_quotient_dev_keeps_each_contexts_challenges_and_weights():
    """Two contexts evaluate the AIR quotient on their own 2^16-row, 8-coset tables with their own challenges and weights, several
    times at once: every result equals what that context computes alone.  A context whose constant upload lands under the
    other's running kernels computes with the other's weights and challenges."""
    import torch
    log_n, log_r, calls = 16, 3, 4
    rn = 1 << (log_n + log_r)
    bs = backends(2)
    try:
        ins, alone = [], []
        for i, b in enumerate(bs):
            g = torch.Generator(device="cuda").manual_seed(1000 + i)
            d_main = torch.randint(0, 1 << 62, (379, rn), dtype=torch.int64, device="cuda", generator=g)   # canonical: < 2^62 < p
            d_aux = torch.randint(0, 1 << 62, (270, rn), dtype=torch.int64, device="cuda", generator=g)
            torch.cuda.synchronize()
            b.to_mont_(d_main); b.to_mont_(d_aux)
            rng = np.random.default_rng(2000 + i)
            ch = rng.integers(0, P, size=(63, 3), dtype=np.uint64)
            w = rng.integers(0, P, size=(604, 3), dtype=np.uint64)
            out = torch.empty((3, rn), dtype=torch.int64, device="cuda")
            b.air_quotient_dev(d_main, rn, d_aux, rn, ch, w, log_n, log_r, 7, out, rn)
            b.synchronize()
            ins.append((d_main, d_aux, ch, w))
            alone.append(out)
        assert not torch.equal(alone[0], alone[1])

        def work(i):
            b, (d_main, d_aux, ch, w) = bs[i], ins[i]
            outs = [torch.empty((3, rn), dtype=torch.int64, device="cuda") for _ in range(calls)]
            for out in outs:
                b.air_quotient_dev(d_main, rn, d_aux, rn, ch, w, log_n, log_r, 7, out, rn)
            b.synchronize()
            return [torch.equal(out, alone[i]) for out in outs]
        same, windows = run_concurrently([lambda i=i: work(i) for i in range(2)])
        assert_overlapped(windows)
        assert same == [[True] * calls] * 2, same
    finally:
        close(bs)


# ---- 5: the AIR check ----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_air_check_of_a_valid_and_a_corrupted_witness_side_by_side():
    """check_program on spin(16) (every constraint holds) next to the check of the same witness's AET with a changed ST0 word
    (tvm_air_check_aet): the violated constraints, their counts and first and last rows equal those found alone"""
    valid, corrupt = backends(2)
    try:
        ex = tvm_b200.trace_execution(SPIN, [16])
        aet = {k: (v.copy() if hasattr(v, "copy") else v) for k, v in ex.aet(valid).items()}
        claim, n = ex.claim, ex.padded_height
        ex.close()
        aet["processor_trace"][1000, 15] = (int(aet["processor_trace"][1000, 15]) + 1) % P   # ST0 of row 1000
        sampled = sampled_challenges(5)
        want = [np.asarray(x) for x in corrupt.air_check_aet(aet, claim, n, sampled, arrays=True)]
        assert want[0].any()
        assert valid.check_program(SPIN, [16]) == []
        reps = 3
        results, windows = run_concurrently([
            lambda: [valid.check_program(SPIN, [16], arrays=True) for _ in range(reps)],
            lambda: [corrupt.air_check_aet(aet, claim, n, sampled, arrays=True) for _ in range(reps)]])
        assert_overlapped(windows)
        for counts, first, last in (tuple(np.asarray(x) for x in r) for r in results[0]):
            assert not counts.any() and (first == 2**64 - 1).all() and (last == 2**64 - 1).all()
        for got in results[1]:
            for g, w in zip(got, want):
                assert np.array_equal(np.asarray(g), w)
    finally:
        close((valid, corrupt))


# ---- 6: the plain-C client -----------------------------------------------------------------------------------------------------
def _build_prove_concurrent(tmp_path):
    libdir = os.path.join(ROOT, "triton-vm_b200", "lib")
    exe = str(tmp_path / "prove_concurrent")
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-pthread", "-I" + os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "examples", "prove_concurrent.c"), "-L" + libdir, "-ltvm_b200", "-Wl,-rpath," + libdir, "-o", exe],
                   check=True)
    return exe


def test_plain_c_concurrent_client_builds_and_fails_loudly_without_a_gpu(tmp_path):
    if not os.path.exists(tvm_b200.LIB_PATH):
        tvm_b200.build()
    exe = _build_prove_concurrent(tmp_path)
    assert subprocess.run([exe, "0"], capture_output=True, text=True).returncode == 2
    if tvm_b200.lib().tvm_device_count() == 0:
        r = subprocess.run([exe, "2"], capture_output=True, text=True)
        assert r.returncode == 3 and "no CPU fallback" in r.stderr, r.stdout + r.stderr


@pytest.mark.gpu
def test_plain_c_concurrent_client_proves_and_verifies(tmp_path):
    exe = _build_prove_concurrent(tmp_path)
    r = subprocess.run([exe, "4"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = r.stdout.splitlines()
    assert len(lines) == 4 and all("verified" in line for line in lines), r.stdout
    assert sorted(int(line.split("padded height ")[1].split(",")[0]) for line in lines) == [1 << k for k in range(10, 14)]
