#!/usr/bin/env python3
"""Times the AIR constraint checker, in one process, for the workloads spin_20 and verifier_11500 (both pad to 2^20):

    python tools/air_check_time.py [--workloads spin_20,verifier_11500] [--reps 5] [--out /tmp/air_check_time.json]

  1. tvm_trace_execution: host wall time of the VM run;
  2. tvm_air_check_execution: host clock around the call (it returns after the results are on the host): hash-trace expansion,
     table fill, degree-lowering columns, extension and the check;
  3. tvm_air_check on the same witness held in device memory (torch tensors built by tvm_main_table_from_aet and
     tvm_aux_extend): host clock around the call, which includes the upload pass (validation, Montgomery form, planar aux)
     and the check kernels.  The difference of 2 and 3 is what the fill and the extension cost inside 2;
  4. the kernels launched per call (tvm_launch_count).
Medians of --reps runs after one warm-up.  Prints one JSON line per workload with the card's name and power limit (read-only
nvidia-smi query)."""
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


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"], capture_output=True,
                             text=True, timeout=30).stdout.strip().split(", ")
        return out[0], float(out[1])
    except Exception:   # noqa: BLE001
        import torch
        return torch.cuda.get_device_name(0), None


def timed(fn, reps):
    import torch
    fn()
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts)), ts


def measure(b, workload, reps):
    import torch
    from oracle import tracegen as tg
    import test_vm_programs as tvp
    src, inp, ram = tvp._workload(workload)
    words = tg.assemble(src)
    sampled = np.random.default_rng(1).integers(0, tvm_b200.P, size=(59, 3), dtype=np.uint64)
    t0 = time.perf_counter()
    ex = tvm_b200.trace_execution(words, inp, (), (), ram)
    trace_ms = (time.perf_counter() - t0) * 1e3
    n = ex.padded_height
    res = {}
    before = b.launches
    assert b.air_check_execution(ex, sampled) == []
    launches_exec = b.launches - before
    res["check_execution_ms"], res["check_execution_runs"] = timed(lambda: b.air_check_execution(ex, sampled), reps)
    # the same witness in device memory
    aet = ex.aet(b)
    main, _ = b.main_table_from_aet(aet, n)
    from oracle import stark as S
    ch = np.array(S.derive_challenges([tuple(int(v) for v in r) for r in sampled], S.Claim(*ex.claim)), dtype=np.uint64)
    d_main = torch.from_numpy(main.view(np.int64)).cuda()
    del main
    d_aux = torch.empty((91, n, 3), dtype=torch.int64, device="cuda")
    b.aux_extend(d_main, ch, out=d_aux)
    before = b.launches
    assert b.air_check(d_main, d_aux, ch) == []
    launches_tables = b.launches - before
    res["check_device_tables_ms"], res["check_device_tables_runs"] = timed(lambda: b.air_check(d_main, d_aux, ch), reps)
    ex.close()
    del d_main, d_aux
    torch.cuda.empty_cache()
    return dict(workload=workload, padded_height=n, trace_execution_ms=trace_ms, **res,
                fill_and_extend_ms=res["check_execution_ms"] - res["check_device_tables_ms"],
                launches_per_check_execution=launches_exec, launches_per_check_tables=launches_tables)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="spin_20,verifier_11500")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out")
    a = ap.parse_args()
    name, power = card()
    b = tvm_b200.Backend(0)
    rows = []
    for w in a.workloads.split(","):
        r = dict(measure(b, w, a.reps), gpu=name, power_limit_w=power)
        print(json.dumps(r), flush=True)
        rows.append(r)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)
    b.close()


if __name__ == "__main__":
    main()
