#!/usr/bin/env python3
"""Times seeded proving on the device, in one process:

    python tools/make_workload.py spin_20 /tmp/spin20 --aet
    python tools/seeded_time.py /tmp/spin20 [--reps 5] [--out /tmp/seeded_time.json]

  1. tvm_prover_randomness at the workload's padded height (all four arrays into device memory, and into pinned host
     memory), CUDA events on the context's stream after warm-up.  The window is the whole call: it includes the one host
     round trip of the call (the count of flagged positions is read back before the samples are drawn);
  2. tvm_prove_aet_seeded (the AET and the 32-byte seed cross the boundary) against tvm_prove_aet handed the same
     randomness as pinned host arrays (≈ 26 MB at 2^20 uploaded per prove), alternating the two, host clock around each call
     (both return after the proof is on the host); both must give identical proof words.
Prints one JSON line with the card's name and power limit (read-only nvidia-smi query)."""
import argparse
import glob
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "triton-vm_b200", "py")]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("workload_dir")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out")
    a = ap.parse_args()
    import torch
    torch.cuda.set_device(0)
    txt = open(os.path.join(a.workload_dir, "claim.txt")).read().split()
    security, log2_exp, ldtc, ph = (int(v) for v in txt[:4])
    ni = int(txt[9]); no = int(txt[10 + ni])
    claim = ([int(v) for v in txt[4:9]], [int(v) for v in txt[10:10 + ni]], [int(v) for v in txt[11 + ni:11 + ni + no]])
    kw = dict(security_level=security, log2_expansion=log2_exp, ldt_choice=ldtc)
    aet = {}
    for f in sorted(glob.glob(os.path.join(a.workload_dir, "aet_*.u*"))):
        name, ext = os.path.basename(f)[4:].rsplit(".", 1)
        arr = np.fromfile(f, dtype="<u4" if ext == "u32" else "<u8")
        if name in ("program", "instruction_multiplicities", "lookup_table_lookup_multiplicities"):
            aet[name] = arr
            continue
        width = tvm_b200._AET_WIDTHS[name]
        t = torch.empty((arr.size // width, width), dtype=torch.int64, pin_memory=True)
        t.numpy().view(np.uint64)[...] = arr.reshape(-1, width)
        aet[name] = t
    assert len(aet) == 11, "no AET in the workload directory: tools/make_workload.py --aet"

    b = tvm_b200.Backend(0)
    stream = torch.cuda.Stream()
    b.set_stream(stream.cuda_stream)
    dom = tvm_b200.derive_domains(security, log2_exp, ph, ldtc)
    shapes = [(379, dom["num_trace_randomizers"]), (91, dom["num_trace_randomizers"], 3), (dom["trace_len"], 3),
              (dom["num_quotient_randomizer_coefficients"], 3)]
    words = sum(int(np.prod(s)) for s in shapes)
    dev = tuple(torch.empty(s, dtype=torch.int64, device="cuda") for s in shapes)
    pinned = tuple(torch.empty(s, dtype=torch.int64, pin_memory=True) for s in shapes)

    def event_ms(out, reps):
        for _ in range(3):
            b.prover_randomness(SEED, ph, out=out, **kw)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ms = []
        for _ in range(reps):
            e0.record(stream)
            b.prover_randomness(SEED, ph, out=out, **kw)
            e1.record(stream)
            e1.synchronize()
            ms.append(e0.elapsed_time(e1))
        return ms
    rand_dev_ms = event_ms(dev, 20)
    rand_host_ms = event_ms(pinned, 20)
    host_rand = tuple(t.numpy().view(np.uint64) for t in pinned)
    assert all(np.array_equal(d.cpu().numpy().view(np.uint64), h) for d, h in zip(dev, host_rand))

    def arrays():
        return b.prove_aet(claim, aet, pinned[0], pinned[1], pinned[2], host_rand[3], padded_height=ph, **kw)

    def seeded():
        return b.prove_aet_seeded(claim, aet, SEED, ph, **kw)
    want = arrays()
    assert np.array_equal(want, seeded()), "tvm_prove_aet_seeded differs from tvm_prove_aet on the same randomness"
    t_arr, t_seed = [], []
    for _ in range(a.reps):
        for fn, acc in ((arrays, t_arr), (seeded, t_seed)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            proof = fn()
            acc.append((time.perf_counter() - t0) * 1e3)
            assert np.array_equal(proof, want)
    ok, why = tvm_b200.verify(claim, want, security, log2_exp, ldtc)
    name, power = card()
    res = dict(gpu=name, power_limit_w=power, padded_height=ph, randomness_words=words, randomness_mb=round(8 * words / 1e6, 2),
               prover_randomness_ms_device_out=round(float(np.median(rand_dev_ms)), 3),
               prover_randomness_ms_host_out=round(float(np.median(rand_host_ms)), 3),
               prove_aet_ms=[round(v, 1) for v in t_arr], prove_aet_seeded_ms=[round(v, 1) for v in t_seed],
               prove_aet_median_ms=round(float(np.median(t_arr)), 1), prove_aet_seeded_median_ms=round(float(np.median(t_seed)), 1),
               identical_proofs=True, proof_words=int(want.size), verified=bool(ok))
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")
    b.close()


if __name__ == "__main__":
    main()
