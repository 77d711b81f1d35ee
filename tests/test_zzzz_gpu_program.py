"""Proving a program from its inputs on the device: the hash traces of tvm_execution_aet expanded by fill/hash_trace.cuh's CUDA
executor against the oracle's, and tvm_prove_execution / Backend.prove_program reproducing the reference's two whole-proof
known-answer digests from (program, inputs, seed) alone — no AET, table or randomness computed in Python.  The VM and the stage
body are checked on the host by tests/test_program_execution.py; this file sorts last: its kernels are the newest."""
import os
import socket
import subprocess

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

import tvm_b200
from oracle import reference_prover as RP, tip5, tracegen as tg
from oracle.rand_compat import StdRng

import test_golden as TG
import test_vm_programs as tvp
from test_program_execution import HASH_KEYS, PROGRAMS, every_instruction_inputs, program

pytestmark = pytest.mark.gpu

SEED = bytes(range(100, 132))


def _verifier(name):
    src, inp, ram = tvp._workload(name)
    return tg.assemble(src), inp, [], ram, []


@pytest.mark.parametrize("name", PROGRAMS + ["verifier_2000"])
def test_device_hash_traces_match_the_oracle(backend, name):
    """verifier_2000: about 16 000 permutations, 96 000 rows, in one launch"""
    words, inp, sec, ram, digests = _verifier(name) if name == "verifier_2000" else program(name)
    ex = tvm_b200.trace_execution(words, inp, sec, digests, ram)
    want = tg.aet_arrays(list(words), tg.execute(list(words), inp, sec, ram, digests))
    launches = backend.launches
    got = ex.aet(backend)
    assert backend.launches > launches
    for key in HASH_KEYS:
        assert got[key].shape == want[key].shape and np.array_equal(got[key], want[key]), key
    if name == "verifier_2000":
        assert len(got["hash_trace"]) + len(got["sponge_trace"]) > 90_000
    assert ex.aet(backend)["sponge_trace"].shape == want["sponge_trace"].shape      # kept with the execution
    ex.close()


def test_reference_proof_digest_from_the_program(backend):
    """proof.rs:200-226: public input = the program's digest, Prover::default()"""
    words = tg.assemble(TG.REFERENCE_PROGRAM)
    seed = RP.seed_from_rng(StdRng.seed_from_u64(TG.REFERENCE_SEED_OF_SEED))
    digest = [int(v) for v in tip5.hash_varlen(words)]
    claim, proof = backend.prove_program(words, digest, seed=seed)
    assert claim == (digest, digest, [])
    assert RP.proof_digest([int(v) for v in proof]) == TG.REFERENCE_PROOF_DIGEST


def test_every_instruction_proof_digest_from_the_program(backend):
    """stark.rs:2433-2460 (Stark::low_security()), the nondeterminism of test_golden.every_instruction_instance"""
    inp, sec, ram, digests = every_instruction_inputs()
    seed = RP.seed_from_rng(StdRng.seed_from_u64(TG.EVERY_INSTRUCTION_SEED_OF_SEED))
    claim, proof = backend.prove_program(tg.assemble(TG.EVERY_INSTRUCTION_PROGRAM), inp, sec, digests, ram, seed=seed, security_level=32)
    assert RP.proof_digest([int(v) for v in proof]) == TG.EVERY_INSTRUCTION_PROOF_DIGEST
    assert tvm_b200.verify(claim, proof, 32, 2) == (True, "")


def test_spin_16_equals_the_seeded_prove_of_the_oracles_aet(backend):
    """ProgramToBench::spin(16) at Stark::default() (STIR at 2^16)"""
    words = tg.assemble(tvp.SPIN)
    ex = tvm_b200.trace_execution(words, [16])
    assert ex.padded_height == 1 << 16
    want = tg.execute(words, [16])
    got = backend.prove_execution(ex, SEED)
    assert np.array_equal(got, backend.prove_aet_seeded(ex.claim, tg.aet_arrays(words, want), SEED, ex.padded_height))
    assert ex.claim == (want.digest, [16], want.output)


def test_spin_20_proof_verifies_with_the_air(backend):
    claim, proof = backend.prove_program(tg.assemble(tvp.SPIN), [20], seed=SEED)
    assert tvm_b200.proof_padded_height(proof) == 1 << 20
    assert tvm_b200.verify(claim, proof) == (True, "")


def test_argument_errors_launch_nothing(backend):
    import ctypes
    ex = tvm_b200.trace_execution(tg.assemble(tvp.SPIN), [8])
    lib, before = tvm_b200.lib(), backend.launches
    p = tvm_b200.Params(160, 2, 0, 0)
    buf, cap = np.empty(1 << 16, dtype=np.uint64), ctypes.c_size_t(1 << 16)
    bp = buf.ctypes.data_as(tvm_b200._u64p)
    assert lib.tvm_prove_execution(backend._h, ctypes.byref(p), ex._h, None, bp, ctypes.byref(cap)) == -1        # NULL seed
    assert lib.tvm_prove_execution(backend._h, ctypes.byref(p), None, SEED, bp, ctypes.byref(cap)) == -1         # no execution
    assert lib.tvm_prove_execution(backend._h, None, ex._h, SEED, bp, ctypes.byref(cap)) == -1                   # no parameters
    assert lib.tvm_prove_execution(backend._h, ctypes.byref(p), ex._h, SEED, bp, None) == -1                    # no length
    bad = tvm_b200.Params(160, 2, 3, 0)
    assert lib.tvm_prove_execution(backend._h, ctypes.byref(bad), ex._h, SEED, bp, ctypes.byref(cap)) == -1      # ldt_choice
    assert backend.launches == before
    small = ctypes.c_size_t(4)                           # capacity protocol: the needed length comes back
    assert lib.tvm_prove_execution(backend._h, ctypes.byref(p), ex._h, SEED, bp, ctypes.byref(small)) == -1 and small.value > 4
    assert np.array_equal(backend.prove_execution(ex, SEED)[:small.value], backend.prove_execution(ex, SEED))
    ex.close()


def test_plain_c_program_client_proves_and_verifies(tmp_path):
    from test_native_verifier import _build_example
    exe = _build_example(tmp_path, "prove_program")
    r = subprocess.run([exe, "10"], capture_output=True, text=True)
    assert r.returncode == 0 and "verified" in r.stdout and "padded height 1024" in r.stdout, r.stdout + r.stderr


# ---- two ranks: every rank traces the same inputs and proves with the same seed ---------------------------------------------
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
        ex = tvm_b200.trace_execution(tg.assemble(src), inp, ram=ram)
        kw = dict(security_level=8, ldt_choice=tvm_b200.LDT_FRI)
        b = tvm_b200.Backend(dev)
        single = b.prove_execution(ex, SEED, **kw)
        comm = TorchDistComm(f"cuda:{dev}")
        b.set_comm(comm)
        assert np.array_equal(single, b.prove_execution(ex, SEED, **kw)), "sharded tvm_prove_execution differs"
        assert not comm.errors, comm.errors
        b.set_comm(None)
        q.put((rank, "ok", len(single)))
    except Exception as e:  # noqa: BLE001
        q.put((rank, repr(e), 0))
        raise
    finally:
        dist.destroy_process_group()


def test_sharded_program_prove_equals_the_single_gpu_proof():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    ps = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in ps: p.start()
    for p in ps: p.join(600)
    res = sorted(q.get(timeout=10) for _ in range(2))
    assert all(r[1] == "ok" for r in res), res
    assert all(p.exitcode == 0 for p in ps)
