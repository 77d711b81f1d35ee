"""Seeded proving on the device: the prover's randomness drawn from its 32-byte seed (tvm_prover_randomness; sampler stages
of csrc/rand/prover_randomness.cuh) against the oracle's restatement of Prover::prove's draws, and tvm_prove_aet_seeded /
tvm_prove_tables_seeded reproducing the reference's two whole-proof known-answer digests from (AET, seed) alone — no
randomness computed in Python.  The same stage bodies are checked on the host by tests/test_prover_randomness_host.py; this
file sorts last: its kernels are the newest."""
import functools
import os
import socket

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

import tvm_b200
from oracle import reference_prover as RP, stark as S, tip5, tracegen as tg
from oracle.rand_compat import StdRng

import test_golden as TG
import test_vm_programs as tvp
from test_prover_randomness_host import fixture_seed

pytestmark = pytest.mark.gpu

SEED = bytes(range(100, 132))


@functools.lru_cache(maxsize=None)
def oracle_randomness(seed, padded_height, security=160):
    d = S.Stark(security, 2).derive(padded_height)
    return RP.randomness(seed, d["trace_len"], d["num_trace_randomizers"], d["num_quotient_randomizer_coefficients"])


def _equal(got, want):
    return all(np.array_equal(np.asarray(g).reshape(np.shape(w)), w) for g, w in zip(got, want))


@pytest.mark.parametrize("log2_ph", [8, 11, 16])
def test_device_randomness_matches_the_oracle(backend, log2_ph):
    ph = 1 << log2_ph
    want = oracle_randomness(SEED, ph)
    assert _equal(backend.prover_randomness(SEED, ph), want)
    dev = tuple(torch.empty(w.shape, dtype=torch.int64, device="cuda") for w in want)   # device outputs
    backend.prover_randomness(SEED, ph, out=dev)
    torch.cuda.synchronize()
    assert _equal([t.cpu().numpy().view(np.uint64) for t in dev], want)
    part = backend.prover_randomness(SEED, ph, out=(None, None, np.empty(want[2].shape, dtype=np.uint64), None))   # any output may be NULL
    assert part[0] is None and np.array_equal(part[2], want[2])


def test_device_randomness_on_the_short_draw_seed(backend):
    """main column 0 is the fixture seed's own stream: a short sample among its randomizers"""
    seed, j = fixture_seed()
    d = S.Stark(160, 2).derive(256)
    assert j < d["num_trace_randomizers"]
    assert _equal(backend.prover_randomness(seed, 256), oracle_randomness(seed, 256))
    r = StdRng(seed)
    assert [int(v) for v in backend.prover_randomness(seed, 256)[0][0, :j + 2]] == [r.bfe() for _ in range(j + 2)]


# ---- the reference's whole-proof known-answer tests, from (AET, seed) alone ------------------------------------------------
def _claim(inst):
    c = inst["claim"]
    return (c.program_digest, c.input, c.output)


def test_reference_proof_digest_from_the_seed(backend):
    """proof.rs:200-226 `current_proof_version_is_still_current`"""
    words = tg.assemble(TG.REFERENCE_PROGRAM)
    seed = RP.seed_from_rng(StdRng.seed_from_u64(TG.REFERENCE_SEED_OF_SEED))
    inst = RP.instance(S.Stark(160, 2), words, [int(v) for v in tip5.hash_varlen(words)], seed)     # as test_golden.py builds it
    aet = tg.aet_arrays(words, inst["execution"])
    got = backend.prove_aet_seeded(_claim(inst), aet, seed, inst["padded_height"])
    assert RP.proof_digest([int(v) for v in got]) == TG.REFERENCE_PROOF_DIGEST
    got = backend.prove_tables_seeded(_claim(inst), inst["main"], seed, padded_height=inst["padded_height"])
    assert RP.proof_digest([int(v) for v in got]) == TG.REFERENCE_PROOF_DIGEST


def test_every_instruction_proof_digest_from_the_seed(backend):
    """stark.rs:2433-2460 `supplying_prover_randomness_seed_fully_derandomizes_produced_proof` (Stark::low_security())"""
    inst = TG.every_instruction_instance()
    seed = RP.seed_from_rng(StdRng.seed_from_u64(TG.EVERY_INSTRUCTION_SEED_OF_SEED))
    aet = tg.aet_arrays(tg.assemble(TG.EVERY_INSTRUCTION_PROGRAM), inst["execution"])
    got = backend.prove_aet_seeded(_claim(inst), aet, seed, inst["padded_height"], security_level=32)
    assert RP.proof_digest([int(v) for v in got]) == TG.EVERY_INSTRUCTION_PROOF_DIGEST
    assert tvm_b200.verify(_claim(inst), got, 32, 2) == (True, "")
    got = backend.prove_tables_seeded(_claim(inst), inst["main"], seed, security_level=32, padded_height=inst["padded_height"])
    assert RP.proof_digest([int(v) for v in got]) == TG.EVERY_INSTRUCTION_PROOF_DIGEST


def test_seeded_spin_16_equals_the_prove_fed_with_the_oracles_randomness(backend):
    """ProgramToBench::spin(16) at Stark::default() (STIR at 2^16)"""
    words = tg.assemble(tvp.SPIN)
    ex = tg.execute(words, [16])
    ph = tg.padded_height(words, [16])
    assert ph == 1 << 16
    aet = tg.aet_arrays(words, ex)
    claim = (ex.digest, [16], list(ex.output))
    seeded = backend.prove_aet_seeded(claim, aet, SEED, ph)
    assert np.array_equal(seeded, backend.prove_aet(claim, aet, *oracle_randomness(SEED, ph), padded_height=ph))
    assert tvm_b200.derive_domains(padded_height=ph)["ldt"] == tvm_b200.LDT_STIR
    assert tvm_b200.verify(claim, seeded) == (True, "")


def test_null_seed_is_an_argument_error(backend):
    words = [tg.OP_HALT]
    ex = tg.execute(words)
    with pytest.raises(tvm_b200.TvmError) as e:
        backend.prover_randomness(None, 256)
    assert e.value.code == -1
    with pytest.raises(tvm_b200.TvmError) as e:
        backend.prove_aet_seeded((ex.digest, [], []), tg.aet_arrays(words, ex), None, 256)
    assert e.value.code == -1
    n = tvm_b200.derive_domains(padded_height=256)["trace_len"]
    with pytest.raises(tvm_b200.TvmError) as e:
        backend.prove_tables_seeded((ex.digest, [], []), np.zeros((379, n), dtype=np.uint64), None, padded_height=256)
    assert e.value.code == -1


# ---- two ranks: every rank derives the identical randomness from the same seed ---------------------------------------------
def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _worker(rank, world, port, q):
    import torch.distributed as dist
    from tvm_b200.dist import TorchDistComm
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    one_gpu_each = torch.cuda.device_count() >= world
    dev = rank if one_gpu_each else 0
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl" if one_gpu_each else "gloo", rank=rank, world_size=world)
    try:
        src, inp, ram = tvp._workload("fib_100")
        words = tg.assemble(src)
        ex = tg.execute(words, inp, (), ram)
        ph = tg.padded_height(words, inp)
        aet = tg.aet_arrays(words, ex)
        claim = (ex.digest, inp, list(ex.output))
        kw = dict(security_level=8, ldt_choice=tvm_b200.LDT_FRI)
        b = tvm_b200.Backend(dev)
        single = b.prove_aet_seeded(claim, aet, SEED, ph, **kw)
        assert np.array_equal(single, b.prove_aet(claim, aet, *b.prover_randomness(SEED, ph, security_level=8, ldt_choice=tvm_b200.LDT_FRI),
                                                  padded_height=ph, **kw))
        comm = TorchDistComm(f"cuda:{dev}")
        b.set_comm(comm)
        assert np.array_equal(single, b.prove_aet_seeded(claim, aet, SEED, ph, **kw)), "sharded tvm_prove_aet_seeded differs"
        assert not comm.errors, comm.errors
        b.set_comm(None)
        q.put((rank, "ok", len(single)))
    except Exception as e:  # noqa: BLE001
        q.put((rank, repr(e), 0))
        raise
    finally:
        dist.destroy_process_group()


def test_sharded_seeded_prove_equals_the_single_gpu_proof():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    ps = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in ps: p.start()
    for p in ps: p.join(600)
    res = sorted(q.get(timeout=10) for _ in range(2))
    assert all(r[1] == "ok" for r in res), res
    assert all(p.exitcode == 0 for p in ps)
