"""Column LDE at the prove's shapes (padded height 2^20), two library builds compared in one run, and the SASS
instruction mix of the tile-NTT kernels with the ALU-pipe floor derived from it.

    python tools/lde_ab.py --sass-only [--parent-lib OLD.so]      # any machine with cuobjdump; no GPU
    python tools/lde_ab.py --parent-lib OLD.so [--reps 3] [--log2n 20] [--out DIR]

Workload: the main LDE (379 B-field columns) and the aux LDE (273 B-field planes), n = 2^20 (`--log2n`), 8 cosets, h = 228
randomizers, through lde_interpolate_run + lde_evaluate_run (`tvm_lde_bfe_dev`) in the prover's batches: 16 columns
per batch for the main table, 15 planes (5 X-field columns) for the aux table.

Timing: the parent build (OLD.so, selected through TVM_B200_LIB, with the bindings of its own tree: OLD.so's ../py) and
this tree's build run alternately, each in its own process, `--reps` times.  A stage's time is the median of `--iters`
CUDA-event timings of all its batches; an output fingerprint of every stage is printed so that the two builds can be seen
to agree.  One more process per build runs each stage once under torch.profiler and reports the sum of the tile-kernel
times against the stage's wall time on the device.  The card's name, power limit and SM clock are sampled with
nvidia-smi during the timed region.

Floor (derived, not measured): an ALU-pipe warp instruction (IADD3, LOP3, LEA, SHF, ISETP, SEL, PRMT, MOV, ...) takes 2
issue cycles of an SM sub-partition (16 INT32 lanes); 132 SMs x 4 sub-partitions at 1980 MHz.  A tile of 256 threads
transforms 256 x R points with 8 warps, so pass X handles 1024 x 5.227e11 / alu_X points per second at R = 32.
"""
import argparse
import collections
import json
import os
import re
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEFAULT_LIB = os.path.join(ROOT, "triton-vm_b200", "lib", "libtvm_b200.so")
LOG2_COSETS, H = 3, 228
STAGES = [("main", 379, 16), ("aux", 273, 15)]          # (name, B-field columns, columns per prover batch)
ALU_OPS = ("IADD3", "LOP3", "LEA", "SHF", "ISETP", "SEL", "PRMT", "MOV", "IABS", "FLO", "POPC", "BMSK", "PLOP3", "LOP", "SGXT",
           "VIADD", "IMNMX", "VIMNMX", "UIADD3", "ULOP3", "ULEA", "USHF", "UISETP", "USEL", "UMOV", "UPRMT")
ALU_RATE = 132 * 4 * 1980e6 / 2                          # ALU-pipe warp instructions per second, whole device


# ---- SASS ------------------------------------------------------------------------------------------------------------
def opclass(op):
    base = op.split(".")[0]
    if base.startswith("IMAD") or base in ("IMUL",):
        return "IMAD"
    if base in ALU_OPS:
        return "ALU"
    return "other"


def sass(lib):
    """{kernel (demangled template arguments): {"total", "ALU", "IMAD", "other"}}"""
    out = subprocess.run(["cuobjdump", "-sass", lib], check=True, capture_output=True, text=True).stdout
    res = {}
    for m in re.finditer(r"Function : (_ZN3tvm15ntt_tile_kernel\S*)\n(.*?)(?=\n\s*Function : |\Z)", out, re.S):
        ops = []
        for line in m.group(2).splitlines():
            t = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(.*?);", line)
            if not t:
                continue
            body = re.sub(r"^@!?U?P[T0-9]+\s+", "", t.group(2).strip())
            op = body.split()[0]
            if op != "NOP":
                ops.append(op)
        c = collections.Counter(opclass(o) for o in ops)
        args = re.search(r"ntt_tile_kernel(I.*?E)(?:Ev|EEv)", m.group(1))
        res[(args.group(1) if args else m.group(1))] = {"total": len(ops), **{k: c.get(k, 0) for k in ("ALU", "IMAD", "other")}}
    return res


def floor_ms(alu_a, alu_b, R=32, cols=379 + 273, log2n=20):
    """derived ALU-pipe floor of the column LDE at 2^20: evaluation (8 cosets) + interpolation, both passes"""
    rate = lambda alu: 256 * R / 8 * ALU_RATE / alu          # points per second of one pass
    ev = cols * (1 << (log2n + LOG2_COSETS))
    it = cols * (1 << log2n)
    return {"pass_a_gpts": round(rate(alu_a) / 1e9, 1), "pass_b_gpts": round(rate(alu_b) / 1e9, 1),
            "evaluate_ms": round(1e3 * (ev / rate(alu_a) + ev / rate(alu_b)), 1),
            "interpolate_ms": round(1e3 * (it / rate(alu_a) + it / rate(alu_b)), 1),
            "floor_ms": round(1e3 * ((ev + it) / rate(alu_a) + (ev + it) / rate(alu_b)), 1)}


# ---- timing (one process per library) --------------------------------------------------------------------------------
def worker(iters, profile, log2n):
    # the Python bindings of the same build: <build>/lib/libtvm_b200.so -> <build>/py
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.environ["TVM_B200_LIB"])), "py"))
    import torch
    import tvm_b200
    dev = torch.device("cuda:0")
    b = tvm_b200.Backend(0)
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    b.set_stream(stream.cuda_stream)
    n = 1 << log2n
    rn = n << LOG2_COSETS
    g = torch.Generator(device=dev)
    g.manual_seed(1)
    maxc = max(c for _, c, _ in STAGES)
    maxb = max(bt for _, _, bt in STAGES)
    trace = torch.randint(0, 2**62, (maxc, n), dtype=torch.int64, device=dev, generator=g)   # < p: canonical
    rand = torch.randint(0, 2**62, (maxc, H), dtype=torch.int64, device=dev, generator=g)
    coef = torch.empty((maxc, 2 * n), dtype=torch.int64, device=dev)
    out = torch.empty((maxc, rn), dtype=torch.int64, device=dev)
    tmp = torch.empty((maxb, rn), dtype=torch.int64, device=dev)
    wcol = torch.arange(maxc, device=dev, dtype=torch.int64) * 2 + 1

    def run(ncols, bt):
        for c0 in range(0, ncols, bt):
            k = min(bt, ncols - c0)
            b.lde_dev(trace[c0:], rand[c0:], H, log2n, LOG2_COSETS, 7, k, coef[c0:], out[c0:], tmp)

    def fingerprint(ncols):
        return int((out[:ncols].sum(dim=1) * wcol[:ncols]).sum().item()) & ((1 << 64) - 1)

    res = {}
    for name, ncols, bt in STAGES:
        run(ncols, bt)
        torch.cuda.synchronize()
        if profile:
            from torch.profiler import ProfilerActivity, profile as prof
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            with prof(activities=[ProfilerActivity.CUDA]) as p:
                s.record()
                run(ncols, bt)
                e.record()
                e.synchronize()
            by = collections.Counter()
            count = collections.Counter()
            for ev in p.events():
                if ev.device_type.name != "CUDA":
                    continue
                key = "tile" if "ntt_tile" in ev.name else ("randomizer" if "randomizer" in ev.name else
                                                            ("memset" if "emset" in ev.name else "other"))
                by[key] += ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
                count[key] += 1
            res[name] = {"stage_ms_profiled": s.elapsed_time(e), "kernel_ms": {k: v / 1e3 for k, v in by.items()},
                         "kernel_count": dict(count)}
            continue
        ms = []
        for _ in range(iters):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            run(ncols, bt)
            e.record()
            e.synchronize()
            ms.append(s.elapsed_time(e))
        res[name] = {"ms": statistics.median(ms), "calls_ms": [round(x, 3) for x in ms], "fingerprint": fingerprint(ncols)}
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
        # the samples include the idle gaps between worker processes (the card then clocks down): the peak is the clock
        # under load
        return {"gpu": rows[-1][0], "power_limit_w": float(rows[-1][1]), "sm_mhz_peak_sampled": max(sm),
                "sm_mhz_median": statistics.median(sm), "sm_max_mhz": float(rows[-1][3]), "samples": len(rows)}


def spawn(lib, args):
    env = dict(os.environ, TVM_B200_LIB=lib)
    p = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", *args], env=env, capture_output=True, text=True)
    line = [x for x in p.stdout.splitlines() if x.startswith("RESULT ")]
    if p.returncode or not line:
        raise SystemExit(f"worker for {lib} failed ({p.returncode}):\n{p.stdout[-2000:]}\n{p.stderr[-4000:]}")
    return json.loads(line[0][7:])


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--lib", default=DEFAULT_LIB, help="this tree's build")
    ap.add_argument("--parent-lib", help="the build to compare against")
    ap.add_argument("--sass-only", action="store_true")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--log2n", type=int, default=20, choices=[12, 14, 16, 18, 20], help="trace length (tile-covered sizes)")
    ap.add_argument("--out", help="directory for lde_ab_2^<log2n>.json")
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--profile", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        return worker(a.iters, a.profile, a.log2n)
    libs = {"new": os.path.abspath(a.lib)}
    if a.parent_lib:
        libs["parent"] = os.path.abspath(a.parent_lib)
    report = {"sass": {k: sass(v) for k, v in libs.items()}}
    if "parent" in libs:
        # the parent's radix-32 forward passes: pass A <5,fwd,PRE,POST=1> and pass B <5,fwd,STREAM,BULK>
        ps = report["sass"]["parent"]
        pa = ps.get("ILi5ELb0ELb1ELi1ELb0ELb0ELb0E")
        pb = ps.get("ILi5ELb0ELb0ELi0ELb0ELb1ELb1E")
        if pa and pb:
            report["parent_floor"] = {"pass_a_sass": pa, "pass_b_sass": pb, **floor_ms(pa["ALU"], pb["ALU"])}
    if not a.sass_only:
        if "parent" not in libs:
            raise SystemExit("--parent-lib is required for timing")
        runs = {k: [] for k in libs}
        clocks = Clocks()
        try:                                  # the sampler is stopped on every way out, a failed worker included
            for _ in range(a.reps):
                for k in ("parent", "new"):
                    runs[k].append(spawn(libs[k], ["--iters", str(a.iters), "--log2n", str(a.log2n)]))
            report["profile"] = {k: spawn(libs[k], ["--profile", "--log2n", str(a.log2n)]) for k in ("parent", "new")}
        finally:
            report["clocks"] = clocks.stop()
        summary = {}
        for stage in runs["new"][0]:
            per = {k: [r[stage]["ms"] for r in runs[k]] for k in runs}
            med = {k: statistics.median(v) for k, v in per.items()}
            summary[stage] = {
                "parent_ms": [round(x, 3) for x in per["parent"]], "new_ms": [round(x, 3) for x in per["new"]],
                "parent_median_ms": round(med["parent"], 3), "new_median_ms": round(med["new"], 3),
                "spread_ms": round(max(max(v) - min(v) for v in per.values()), 3),
                "speedup": round(med["parent"] / med["new"], 4),
                "outputs_equal": len({r[stage]["fingerprint"] for k in runs for r in runs[k]}) == 1,
            }
        report["timing"] = summary
    text = json.dumps(report, indent=1)
    print(text)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, f"lde_ab_2^{a.log2n}.json"), "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
