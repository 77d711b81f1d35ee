"""The AIR quotient stage at the prove's shape (padded height 2^20: 2^20 trace rows on 8 cosets, Stark::default()), two
library builds compared in one run, with the stage's time split by kernel.

    python tools/air_time.py --parent-lib OLD.so [--reps 3] [--iters 3] [--out DIR]

The parent build (OLD.so, selected through TVM_B200_LIB, with the bindings of its own tree: OLD.so's ../py) and this
tree's build run alternately, each in its own process, `--reps` times.  Every process proves the same seeded random tables
(device-resident, as bench.py's `value` leg) `--iters` times after one warm-up; the stage time is the median of the
prover's own CUDA-event stage marks ("quotient(AIR)").  Each process then proves once more under torch.profiler and sums
the device time of the kernels in that stage's window by kernel family.  The proofs of the two builds are compared word for
word.  The card's name, power limit and SM clock are sampled with nvidia-smi during the timed region.
"""
import argparse
import hashlib
import json
import os
import re
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEFAULT_LIB = os.path.join(ROOT, "triton-vm_b200", "lib", "libtvm_b200.so")
LOG2_HEIGHT = 20
STAGE = "quotient(AIR)"


def family(name):
    """kernel family of a demangled kernel name"""
    if "air_chunk" in name:
        return "chunks (even cosets)" if name.split("(")[0].endswith("_lo") else "chunks"
    for key in ("air_top_", "air_zerofier", "air_low_combine", "air_weight_table", "ntt_pass", "coset_to_natural",
                "scale_by_powers"):
        if key in name:
            return key.rstrip("_")
    return "other: " + name.split("(")[0][:60]


def worker(iters):
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.environ["TVM_B200_LIB"])), "py"))
    import numpy as np
    import torch
    import tvm_b200
    dev = torch.device("cuda:0")
    dom = tvm_b200.derive_domains(160, 2, 1 << LOG2_HEIGHT, tvm_b200.LDT_AUTO)
    n, h, nqr = dom["trace_len"], dom["num_trace_randomizers"], dom["num_quotient_randomizer_coefficients"]
    g = torch.Generator(device=dev)
    g.manual_seed(7)
    rnd = lambda *shape: torch.randint(0, 2**62, shape, dtype=torch.int64, device=dev, generator=g)   # < p: canonical
    main, mrand, aux, arand = rnd(379, n), rnd(379, h), rnd(91, n, 3), rnd(91, h, 3)
    qrand = np.random.default_rng(7).integers(0, 2**62, size=(nqr, 3), dtype=np.uint64)
    b = tvm_b200.Backend(0)
    claim = ([1, 2, 3, 4, 5], [7, 8, 9], [10])

    def prove():
        return b.prove(claim, main, mrand, lambda _c: (aux, arand), qrand, 160, 2, 1 << LOG2_HEIGHT, tvm_b200.LDT_AUTO)

    proof = prove()
    torch.cuda.synchronize()
    stage_ms = []
    for _ in range(iters):
        proof = prove()
        stage_ms.append(dict(b.last_prove_timings())[STAGE])
    # one profiled prove
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        prove()
        torch.cuda.synchronize()
    stages = list(b.last_prove_timings())
    kern = sorted((e for e in prof.events() if e.device_type.name == "CUDA"), key=lambda e: e.time_range.start)
    # the stage starts at the first chunk or zerofier kernel and ends with the last AIR kernel
    air = [i for i, e in enumerate(kern) if re.search(r"air_(chunk|zerofier|low_combine|top_)", e.name)]
    fam = {}
    if air:
        t0, t1 = kern[air[0]].time_range.start, kern[air[-1]].time_range.end
        for e in kern[air[0]:air[-1] + 1]:
            f = family(e.name)
            c, t = fam.get(f, (0, 0.0))
            fam[f] = (c + 1, t + (e.time_range.end - e.time_range.start) / 1e3)
        window = (t1 - t0) / 1e3
    else:
        window = None
    res = {"n": n, "h": h, "stage_ms": stage_ms, "stage_median_ms": statistics.median(stage_ms),
           "profiled_window_ms": window, "profiled_stages_ms": dict(stages),
           "kernels": {k: {"launches": c, "ms": round(t, 3)} for k, (c, t) in sorted(fam.items(), key=lambda x: -x[1][1])},
           "proof_sha256": hashlib.sha256(np.asarray(proof, dtype=np.uint64).tobytes()).hexdigest()}
    print("RESULT " + json.dumps(res), flush=True)


class Clocks:
    Q = "name,power.limit,clocks.sm,clocks.max.sm"

    def __init__(self):
        self.f = tempfile.TemporaryFile("w+")
        try:
            self.p = subprocess.Popen(["nvidia-smi", "-i", "0", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                                       "-lms", "200"], stdout=self.f, stderr=subprocess.DEVNULL)
        except OSError:
            self.p = None

    def stop(self):
        if self.p is None:
            return {"gpu": None, "reasons": ["nvidia-smi unavailable"]}
        self.p.terminate()
        try:
            self.p.wait(timeout=10)
        except subprocess.TimeoutExpired:
            self.p.kill()
            self.p.wait()
        self.f.seek(0)
        rows = [[x.strip() for x in line.split(",")] for line in self.f.read().splitlines()]
        rows = [r for r in rows if len(r) == 4 and r[2].replace(".", "").isdigit()]
        if not rows:
            return {"gpu": None, "reasons": ["no nvidia-smi samples"]}
        sm = [float(r[2]) for r in rows]
        return {"gpu": rows[-1][0], "power_limit_w": float(rows[-1][1]), "sm_mhz_peak_sampled": max(sm),
                "sm_mhz_median": statistics.median(sm), "sm_max_mhz": float(rows[-1][3]), "samples": len(rows)}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--lib", default=DEFAULT_LIB, help="this tree's build")
    ap.add_argument("--parent-lib", help="the build to compare against (required)")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--out", help="directory for air_time.json")
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        return worker(a.iters)
    if not a.parent_lib:
        raise SystemExit("--parent-lib is required")
    libs = {"parent": os.path.abspath(a.parent_lib), "new": os.path.abspath(a.lib)}
    runs = {k: [] for k in libs}
    report = {}
    clocks = Clocks()
    try:                                      # the sampler is stopped on every way out, a failed worker included
        for _ in range(a.reps):
            for k in ("parent", "new"):
                env = dict(os.environ, TVM_B200_LIB=libs[k])
                p = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", "--iters", str(a.iters)],
                                   env=env, capture_output=True, text=True)
                line = [x for x in p.stdout.splitlines() if x.startswith("RESULT ")]
                if p.returncode or not line:
                    raise SystemExit(f"worker for {k} failed ({p.returncode}):\n{p.stdout[-2000:]}\n{p.stderr[-4000:]}")
                runs[k].append(json.loads(line[0][7:]))
    finally:
        report["clocks"] = clocks.stop()
    for k in runs:
        med = [r["stage_median_ms"] for r in runs[k]]
        report[k] = {"stage_median_ms_per_rep": [round(x, 3) for x in med], "stage_median_ms": round(statistics.median(med), 3),
                     "spread_ms": round(max(med) - min(med), 3), "kernels_last_rep": runs[k][-1]["kernels"],
                     "profiled_window_ms": runs[k][-1]["profiled_window_ms"], "profiled_stages_ms": runs[k][-1]["profiled_stages_ms"]}
    report["n"], report["h"] = runs["new"][0]["n"], runs["new"][0]["h"]
    report["proofs_equal"] = len({r["proof_sha256"] for k in runs for r in runs[k]}) == 1
    report["speedup"] = round(report["parent"]["stage_median_ms"] / report["new"]["stage_median_ms"], 4)
    text = json.dumps(report, indent=1)
    print(text)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "air_time.json"), "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
