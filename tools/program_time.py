#!/usr/bin/env python3
"""Times proving a program from its inputs, in one process, for the workloads spin_20 and verifier_11500 (program words from
tests/test_vm_programs._workload; both pad to 2^20):

    python tools/program_time.py [--workloads spin_20,verifier_11500] [--reps 3] [--out /tmp/program_time.json]

  1. tvm_trace_execution: host wall time of the VM run (median of --reps runs);
  2. the hash-trace expansion on the device: kernel time of fill/hash_trace.cuh's stage from torch.profiler (one expansion,
     after a warm-up expansion of another execution), and CUDA events around the whole tvm_execution_aet call (upload of the
     permutation inputs, expansion, copy of the three traces back to the host);
  3. tvm_prove_execution against tvm_prove_aet_seeded handed the same AET as pinned host arrays, alternating the two, host
     clock around each call (both return after the proof is on the host); both must give identical proof words.
Prints one JSON line per workload with the card's name and power limit (read-only nvidia-smi query)."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "triton-vm_b200"), os.path.join(ROOT, "triton-vm_b200", "py"), os.path.join(ROOT, "tests")]
import tvm_b200   # noqa: E402

SEED = bytes(range(7, 39))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"], capture_output=True,
                             text=True, timeout=30).stdout.strip().split(", ")
        return out[0], float(out[1])
    except Exception:   # noqa: BLE001
        import torch
        return torch.cuda.get_device_name(0), None


def pinned(aet):
    import torch
    out = {}
    for name, arr in aet.items():
        if name not in tvm_b200._AET_WIDTHS:
            out[name] = arr
            continue
        t = torch.empty(arr.shape, dtype=torch.int64, pin_memory=True)
        t.numpy().view(np.uint64)[...] = arr
        out[name] = t
    return out


def measure(b, stream, workload, reps):
    import torch
    from oracle import tracegen as tg
    import test_vm_programs as tvp
    src, inp, ram = tvp._workload(workload)
    words = tg.assemble(src)

    def trace():
        return tvm_b200.trace_execution(words, inp, ram=ram)
    trace_ms = []
    for _ in range(reps):
        t0 = time.perf_counter()
        ex = trace()
        trace_ms.append((time.perf_counter() - t0) * 1e3)
        ex.close()
    ex = trace()
    trace().aet(b)                                         # warm-up expansion (module load, pool blocks)
    fresh = trace()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    fresh.aet(b)
    e1.record(stream)
    e1.synchronize()
    aet_call_ms = e0.elapsed_time(e1)
    fresh.close()
    fresh = trace()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fresh.aet(b)
        torch.cuda.synchronize()
    kernel_us = sum(e.device_time for e in prof.events() if "hash_trace" in e.name)
    fresh.close()
    aet = pinned(ex.aet(b))
    rows = sum(len(aet[k]) for k in ("program_hash_trace", "sponge_trace", "hash_trace"))

    def from_execution():
        return b.prove_execution(ex, SEED)

    def from_aet():
        return b.prove_aet_seeded(ex.claim, aet, SEED, ex.padded_height)
    want = from_aet()
    assert np.array_equal(want, from_execution()), "tvm_prove_execution differs from tvm_prove_aet_seeded on the same AET"
    t_ex, t_aet = [], []
    for _ in range(reps):
        for fn, acc in ((from_execution, t_ex), (from_aet, t_aet)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            proof = fn()
            acc.append((time.perf_counter() - t0) * 1e3)
            assert np.array_equal(proof, want)
    ok, _ = tvm_b200.verify(ex.claim, want)
    res = dict(workload=workload, padded_height=ex.padded_height, cycles=ex.table_heights["processor"],
               permutations=int(len(aet["program_hash_trace"]) // 6 + len(aet["hash_trace"]) // 6 + len(aet["sponge_trace"]) // 6),
               hash_rows=rows, hash_trace_mb=round(rows * 67 * 8 / 1e6, 1),
               trace_execution_ms=[round(v, 1) for v in trace_ms], trace_execution_median_ms=round(float(np.median(trace_ms)), 1),
               hash_expansion_kernel_ms=round(kernel_us / 1e3, 3), execution_aet_call_ms=round(aet_call_ms, 2),
               prove_execution_ms=[round(v, 1) for v in t_ex], prove_aet_seeded_ms=[round(v, 1) for v in t_aet],
               prove_execution_median_ms=round(float(np.median(t_ex)), 1), prove_aet_seeded_median_ms=round(float(np.median(t_aet)), 1),
               identical_proofs=True, proof_words=int(want.size), verified=bool(ok))
    ex.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="spin_20,verifier_11500")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out")
    a = ap.parse_args()
    import torch
    torch.cuda.set_device(0)
    b = tvm_b200.Backend(0)
    stream = torch.cuda.Stream()
    b.set_stream(stream.cuda_stream)
    name, power = card()
    lines = []
    for w in a.workloads.split(","):
        res = measure(b, stream, w, a.reps)
        res.update(gpu=name, power_limit_w=power)
        lines.append(json.dumps(res))
        print(lines[-1], flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")
    b.close()


if __name__ == "__main__":
    main()
