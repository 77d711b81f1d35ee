#!/usr/bin/env python3
"""Proofs per second on one GPU with 1, 2 and 4 contexts proving at the same time, one thread per context (DESIGN.md §6j):

    python tools/concurrent_time.py [--ks 10,13,16,18] [--contexts 1,2,4] [--runs 3] [--proves 24,16,8,4] [--out FILE]

For each seeded spin(k) (tests/test_vm_programs.SPIN, padded height 2^k, Stark::default()) and each context count K: K
Backends on device 0, one warm-up prove each, then --runs runs in which every thread runs the same number of proves
(tvm_prove_execution of one shared Execution, one seed) behind a barrier; host clock from the barrier to the last thread's
return.  Reported per (k, K), median over the runs: proofs per second, and the seconds of the quotient(AIR) stage summed over
the run's proves (tvm_last_prove_timings: device events on each context's stream, so under concurrency it includes the wait
for the device's AIR constant banks), next to the seconds the same proves spend in that stage with one context (the serialised
lower bound).  Every proof must equal the first context's warm-up proof.  The card's name, power limit and SM clocks are read
in the same call (read-only nvidia-smi query).  Prints one JSON line per (k, K)."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "triton-vm_b200", "py"), os.path.join(ROOT, "tests")]
import tvm_b200   # noqa: E402

SEED = bytes(range(100, 132))
AIR_STAGE = "quotient(AIR)"


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader,nounits"], capture_output=True, text=True,
                         timeout=30, check=True).stdout.strip().split(", ")
    return dict(zip(("name", "power_limit_w", "sm_clock_mhz", "max_sm_clock_mhz"), out))


def air_ms(b):
    return dict(b.last_prove_timings()).get(AIR_STAGE, 0.0)


def one_run(bs, ex, proves, want):
    barrier = threading.Barrier(len(bs))
    air, errors, done = [0.0] * len(bs), [], [0.0] * len(bs)

    def worker(i):
        barrier.wait()
        try:
            for _ in range(proves):
                proof = bs[i].prove_execution(ex, SEED)
                air[i] += air_ms(bs[i])
                if not np.array_equal(proof, want):
                    raise AssertionError(f"context {i}: proof differs from the warm-up proof")
        except BaseException as e:   # noqa: BLE001
            errors.append(e)
        done[i] = time.perf_counter()
    threads = [threading.Thread(target=worker, args=(i,)) for i in range(len(bs))]
    t0 = time.perf_counter()
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    if errors:
        raise errors[0]
    return max(done) - t0, sum(air) / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="10,13,16,18")
    ap.add_argument("--contexts", default="1,2,4")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--proves", default="24,16,8,4", help="proves per thread and run, one per k")
    ap.add_argument("--out")
    a = ap.parse_args()
    from oracle import tracegen as tg
    import test_vm_programs as tvp
    ks = [int(v) for v in a.ks.split(",")]
    counts = [int(v) for v in a.contexts.split(",")]
    proves = [int(v) for v in a.proves.split(",")]
    assert len(proves) == len(ks), "--proves needs one count per k"
    info = card()
    lines = []
    for k, n in zip(ks, proves):
        ex = tvm_b200.trace_execution(tg.assemble(tvp.SPIN), [k])
        assert ex.padded_height == 1 << k
        want, air_alone_ms = None, None
        for K in counts:
            bs = [tvm_b200.Backend(0) for _ in range(K)]
            for b in bs:                                   # warm-up: module load, pool blocks, tables
                proof = b.prove_execution(ex, SEED)
                if want is None:
                    want = proof
                assert np.array_equal(proof, want)
            if air_alone_ms is None:                       # the AIR stage of one prove with nothing else on the GPU
                alone = []
                for _ in range(3):
                    bs[0].prove_execution(ex, SEED)
                    alone.append(air_ms(bs[0]))
                air_alone_ms = statistics.median(alone)
            runs = [one_run(bs, ex, n, want) for _ in range(a.runs)]
            low_memory = [b.last_prove_low_memory for b in bs]
            for b in bs:
                b.close()
            wall = statistics.median(r[0] for r in runs)
            line = dict(k=k, contexts=K, proves_per_run=K * n, runs=a.runs, proofs_per_s=round(K * n / wall, 2),
                        run_s=[round(r[0], 4) for r in runs], air_stage_s=round(statistics.median(r[1] for r in runs), 4),
                        air_alone_s=round(K * n * air_alone_ms / 1e3, 4), low_memory=low_memory, card=info)
            lines.append(line)
            print(json.dumps(line), flush=True)
        ex.close()
    if a.out:
        with open(a.out, "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
