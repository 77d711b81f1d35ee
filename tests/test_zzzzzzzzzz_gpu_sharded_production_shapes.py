"""One proof sharded over W ranks (tvm_ctx_set_comm) at Stark::default() parameters (security 160, expansion 4), every rank's
proof word for word against the C + OpenMP oracle (oracle/fast.py).

tests/test_gpu_sharded_prove.py compares sharded proofs with the single-GPU proof at padded heights 64..4096 and security
6..32: one GPU run against another, at shapes where nothing else pins the single-GPU proof.  Here the oracle is the
reference, and every Merkle root feeds Fiat-Shamir, so a kernel that is wrong on a few rows of one rank changes every later
proof word even though `tvm_verify` would still accept the proof.  The oracle proofs come from
test_zzzzz_gpu_production_shapes (its `lru_cache`), so the shapes both modules prove are proved once per session.

What each shape reaches, from the dispatch conditions (n = trace length = padded height here; r = 8 cosets; rank g owns the
cosets g, g + W, ...: NL = 8n / W rows; column blocks of ceil(ncols / W), the last one short):

* LDE (prover.cu `extend_table` -> all_gather of the coefficient blocks -> `evaluate_cols` on the rank's cosets; ntt_tile.cu
  `ntt_tile_supported`): tiles for log n in {12, 14, 16, 18, 20} as n2 x n1 = 2^6 x 2^6, 2^8 x 2^6, 2^10 x 2^6, 2^10 x 2^8;
  equal radices (2^12) run the persistent `ntt_tile_kernel`, unequal ones `evaluate_pairs` / `interpolate_pairs`.  Odd log n
  falls to ntt.cu.  (The quotient-segment and DEEP LDEs fold n coefficients, more than a tile takes: ntt.cu at every shape.)
* Row hashing (hash.cu `hash_rows_run`, `log_r = 0` over NL rows, or n rows per coset just in time): NL and n are multiples
  of 64 and the shards 16-byte aligned, so the TMA kernel at every shape; the per-lane-load kernel is not reached.
* Merkle (`merkle_run_sharded`): rank g builds levels w = 4n .. W of its subtree, w / W nodes each: the MMA level kernel
  while w / W >= 64, the thread-per-node kernel below; then the all-gather of the W subtree roots and `merkle_top_kernel`.
* AIR quotient (quotient.cu): strided coset subset (first = g, step = W), no degree split (`coefs == nullptr`), then
  `shards_to_natural_kernel`; the out-of-domain rows as column-sharded `col_dot_run` blocks (main 379, aux 273 planes).
* STIR (stir.cu `commit`): commitments of N/4, N/8, ... leaves (one per round plus the first); those with
  leaves >= 4096 W hash their 1/W of the leaves per rank and all-gather the digests.

| W | height | LDT | mode | LDE (interpolate / evaluate) | cosets per rank, NL | column blocks main / aux / OOD aux | Merkle levels per rank | STIR commitments sharded |
|---|---|---|---|---|---|---|---|---|
| 2 | 2^12 | auto: FRI | cached | persistent tiles 6x6 | 4, 2^14 | 190+189 / 46+45 / 137+136 | MMA w >= 128 | - (FRI, 173 queries, 2^15) |
| 4 | 2^14 | auto: FRI | cached | tile pairs 8x6 | 2, 2^15 | 95..94 / 23..22 / 69..66 | MMA w >= 256 | - (FRI at 2^17) |
| 2 | 2^17 | STIR | cached | ntt.cu (odd length) | 4, 2^19 | 190+189 / 46+45 / 137+136 | MMA w >= 128 | 5 of 5 (2^18..2^14 leaves, 4 rounds) |
| 4 | 2^16 | auto: STIR | cached | tile pairs 10x6 | 2, 2^17 | 95..94 / 23..22 / 69..66 | MMA w >= 256 | 4 of 5 (2^17..2^14; not 2^13) |
| 8 | 2^16 | auto: STIR | cached | tile pairs 10x6 | 1, 2^16 | 48..43 / 12..7 / 35..28 | MMA w >= 512 | 3 of 5 (2^17..2^15) |
| 8 | 2^16 | FRI | just in time | tile pairs 10x6, one coset at a time | 1, 2^16 | 48..43 / 12..7 / 35..28 | MMA w >= 512 | - (FRI at 2^19) |
| 4 | 2^18 | auto: STIR | cached | tile pairs 10x8 | 2, 2^19 | 95..94 / 23..22 / 69..66 | MMA w >= 256 | 6 of 6 (2^19..2^14, 5 rounds) |
| 4 | spin(16) | auto: STIR | seeded, from the AET | tile pairs 10x6 (device-table branch) | 2, 2^17 | 95..94 / 23..22 / 69..66 | MMA w >= 256 | 4 of 5 |

Every row opens the 173 (FRI) or 208..215 (STIR) queried rows of each table: `gather_rows_kernel` / `gather_digests_kernel`
with their rank masks, then `all_reduce_sum`; the just-in-time row instead evaluates coset by coset for hashing, the AIR and
the openings, which `gather_rows_scatter_kernel` writes into a zeroed buffer reduced across ranks.  What no other test
reaches: the 2^12 row, the oracle pin of the W = 2 tile path with 173 queries; 2^14, the tile pairs on a strided coset subset;
2^17, ntt.cu on a coset subset and multi-round STIR sharded; 2^16 at W = 4 and 8, sharded STIR leaf hashing there and the
shortest last column blocks; the just-in-time row, every sharded coset-by-coset path at production size; 2^18, the largest
shape here (its four ranks on one H100 80GB HBM3, 700 W limit, held at most 28.3 GB together, nvidia-smi); spin(16), the
device-table branch of `extend_table` on several ranks against the oracle.  Sharded proofs above 2^18 are not tested: with W
ranks on one shared GPU each would need tens of GB.

On a box with fewer GPUs than ranks the ranks share cuda:0 and the collectives run over gloo; otherwise NCCL, one GPU each.
Each rank sets its LDE mode explicitly: under the automatic choice the other ranks' allocations on the same GPU could flip it."""
import datetime
import functools
import os
import socket
import time
import traceback

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

import tvm_b200
from oracle import fast, reference_prover as RP, stark as S, tracegen as tg
from test_zzzzz_gpu_production_shapes import (CACHED, CLAIM, JUST_IN_TIME, LDT, SEED, _instance, _oracle_proof, _oracle_threads,
                                              first_difference)
import test_vm_programs as tvp

gpu = pytest.mark.gpu      # the CPU test of this file (the expected collective counts) runs without a GPU

RANK_TIMEOUT_S = 1800      # wall-clock limit for all ranks of one proof; a rank still running then is killed


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _expected_all_gathers(stark, padded_height, world):
    """all_gather calls of one sharded prove: the main and aux coefficient blocks (2); for each of the three table
    commitments the leaf digests and the subtree roots (6); the quotient (1); the main and aux out-of-domain blocks (2);
    the DEEP codeword (1); and one per STIR commitment whose leaves are hashed sharded (stir.cu: leaves >= 4096 W).  The
    first STIR commitment stacks the codeword of N points into N / 4 leaves, each round's commitment has half as many."""
    d = stark.derive(padded_height)
    sharded_stir = 0
    if d["ldt"] == "stir":
        leaves = d["ldt_len"] // 4
        for _ in range(len(d["stir"]["round_queries"]) + 1):
            sharded_stir += leaves >= 4096 * world
            leaves //= 2
    return 12 + sharded_stir


def test_expected_all_gathers_of_the_shapes():
    """the counts the docstring's table states; a shape whose parameters drift away from a sharded path fails here first"""
    want = {(12, None, 2): 12, (14, None, 4): 12, (17, "stir", 2): 17, (16, None, 4): 16, (16, None, 8): 15, (16, "fri", 8): 12,
            (18, None, 4): 18}
    got = {k: _expected_all_gathers(S.Stark(160, 2, k[1]), 1 << k[0], k[2]) for k in want}
    assert got == want


# ---- one rank ---------------------------------------------------------------------------------------------------------------
def _worker(rank, world, port, job, out_dir):
    """proves on rank `rank`; the proof goes to out_dir/rank<r>.npy, a failure's traceback to out_dir/rank<r>.err"""
    try:
        _prove_on_rank(rank, world, port, job, out_dir)
    except BaseException:
        with open(os.path.join(out_dir, f"rank{rank}.err"), "w") as f:
            f.write(traceback.format_exc())
        raise


def _prove_on_rank(rank, world, port, job, out_dir):
    import torch.distributed as dist
    from tvm_b200.dist import TorchDistComm
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    one_gpu_each = torch.cuda.device_count() >= world
    dev = rank if one_gpu_each else 0
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl" if one_gpu_each else "gloo", rank=rank, world_size=world, timeout=datetime.timedelta(minutes=10))
    b = None
    try:
        b = tvm_b200.Backend(dev)
        b.set_low_memory(job["low_memory"])
        comm = TorchDistComm(f"cuda:{dev}")
        b.set_comm(comm)
        if job["kind"] == "synthetic":
            x = _instance(job["log2_height"], job["ldt"], 2)
            proof = b.prove((CLAIM.program_digest, CLAIM.input, CLAIM.output), x["main"], x["mrand"], lambda ch: (x["aux"], x["arand"]),
                            x["qrand"], 160, 2, x["padded_height"], LDT[job["ldt"]])
        else:
            proof = b.prove_aet_seeded(job["claim"], job["aet"], SEED, job["padded_height"])
        assert b.last_prove_low_memory == (job["low_memory"] == JUST_IN_TIME)
        assert comm.errors == [], comm.errors
        assert comm.calls["all_gather"] == job["all_gathers"] and comm.calls["all_reduce"] == 6, \
            f"collectives {comm.calls}, expected {job['all_gathers']} all_gather and 6 all_reduce calls"
        np.save(os.path.join(out_dir, f"rank{rank}.npy"), proof)
    finally:
        try:
            if b is not None:
                b.release_cached_memory()
                b.close()
        finally:
            dist.destroy_process_group()


def _prove_on_ranks(world, job, out_dir, oracle):
    """starts the W ranks, computes the oracle proof while they run, returns (oracle proof, every rank's proof)"""
    ctx = mp.get_context("spawn")
    port = _free_port()
    ps = [ctx.Process(target=_worker, args=(r, world, port, job, str(out_dir))) for r in range(world)]
    for p in ps:
        p.start()
    try:
        want = oracle()
        deadline = time.monotonic() + RANK_TIMEOUT_S
        # a rank that failed leaves the others waiting in a collective: stop them then instead of at the deadline
        while any(p.is_alive() for p in ps) and time.monotonic() < deadline:
            if any(p.exitcode not in (None, 0) for p in ps):
                break
            time.sleep(0.5)
    finally:
        for p in ps:
            if p.is_alive():
                p.kill()
                p.join()
    errors = {r: (out_dir / f"rank{r}.err").read_text() for r in range(world) if (out_dir / f"rank{r}.err").exists()}
    assert not errors, "\n".join(f"rank {r}:\n{e}" for r, e in errors.items())
    assert [p.exitcode for p in ps] == [0] * world
    return want, [np.load(out_dir / f"rank{r}.npy") for r in range(world)]


@pytest.fixture
def free_device_memory(backend):
    """the suite's shared context gives back what earlier tests left in its pool: the W ranks need that device memory"""
    backend.release_cached_memory()
    torch.cuda.empty_cache()


def _assert_every_rank_equals(proofs, want):
    for r, got in enumerate(proofs[1:], 1):
        assert np.array_equal(got, proofs[0]), f"rank {r} differs from rank 0; first differing proof item: {first_difference(got, proofs[0])}"
    for r, got in enumerate(proofs):
        assert np.array_equal(got, want), f"rank {r}: first differing proof item vs the oracle: {first_difference(got, want)}"


# ---- synthetic tables at the production shapes ------------------------------------------------------------------------------
@gpu
@pytest.mark.usefixtures("free_device_memory")
@pytest.mark.parametrize("world,log2_height,ldt,low_memory", [
    (2, 12, "auto", CACHED),
    (4, 14, "auto", CACHED),
    (2, 17, "stir", CACHED),
    (4, 16, "auto", CACHED),
    (8, 16, "auto", CACHED),
    (8, 16, "fri", JUST_IN_TIME),
    (4, 18, "auto", CACHED),
], ids=["w2_2e12_fri", "w4_2e14_fri", "w2_2e17_stir", "w4_2e16_stir", "w8_2e16_stir", "w8_2e16_fri_jit", "w4_2e18_stir"])
def test_sharded_proof_equals_the_oracle(world, log2_height, ldt, low_memory, tmp_path):
    stark = S.Stark(160, 2, None if ldt == "auto" else ldt)
    job = dict(kind="synthetic", log2_height=log2_height, ldt=ldt, low_memory=low_memory,
               all_gathers=_expected_all_gathers(stark, 1 << log2_height, world))
    want, proofs = _prove_on_ranks(world, job, tmp_path, lambda: _oracle_proof(log2_height, ldt, 2))
    _assert_every_rank_equals(proofs, want)
    assert tvm_b200.verify((CLAIM.program_digest, CLAIM.input, CLAIM.output), proofs[0], 160, 2, ldt_choice=LDT[ldt],
                           skip_air_check=True) == (True, "")


# ---- a real program: spin(16) from its AET and seed, the table stages on the device of every rank -----------------------------
@functools.lru_cache(maxsize=None)
def _spin16_instance():
    words = tg.assemble(tvp.SPIN)
    inst = RP.instance(S.Stark(160, 2), words, [16], SEED)
    assert inst["padded_height"] == 1 << 16
    return words, inst


@functools.lru_cache(maxsize=None)
def _spin16_oracle_proof():
    """the oracle proof test_zzzzz_gpu_production_shapes' spin(16) test builds: its own table fill, extension and randomness"""
    _oracle_threads()
    _, inst = _spin16_instance()
    return np.array(fast.prove(inst["stark"], inst["claim"], inst["main"], inst["main_rand"], inst["extend"], inst["quot_rand"],
                               padded_height=inst["padded_height"]), dtype=np.uint64)


@gpu
@pytest.mark.usefixtures("free_device_memory")
def test_sharded_spin_16_from_the_aet_and_seed_equals_the_oracle(tmp_path):
    """`prove_aet_seeded` on 4 ranks: every rank fills and extends the whole main table from the AET (the device-table branch
    of extend_table), draws the randomness from the seed, and interpolates its block of columns"""
    world = 4
    words, inst = _spin16_instance()
    claim = (inst["claim"].program_digest, inst["claim"].input, inst["claim"].output)
    job = dict(kind="aet_seeded", claim=claim, aet=tg.aet_arrays(words, inst["execution"]), padded_height=inst["padded_height"],
               low_memory=CACHED, all_gathers=_expected_all_gathers(inst["stark"], inst["padded_height"], world))
    want, proofs = _prove_on_ranks(world, job, tmp_path, _spin16_oracle_proof)
    _assert_every_rank_equals(proofs, want)
    assert tvm_b200.verify(claim, proofs[0]) == (True, "")
