"""Tip5 row hashing and Merkle build at the prove's shapes (padded height 2^20 -> 2^23 LDT rows), two library builds
compared in one run, and the SASS instruction mix of the hashing kernels.

    python tools/hash_time.py --sass-only [--parent-lib OLD.so]      # any machine with cuobjdump; no GPU
    python tools/hash_time.py --parent-lib OLD.so [--reps 3] [--out DIR]

Timing: the parent build (OLD.so, selected through TVM_B200_LIB, with the bindings of its own tree: OLD.so's
../py) and this tree's build run alternately, each in its own process, `--reps` times.  Every process hashes 379, 273 and
15 columns x 2^23 rows (8 cosets of 2^20, the main, aux and quotient-segment commitments) and builds a Merkle tree over
2^23 leaves; a shape's time is the median of `--iters` calls timed with CUDA events.  A fingerprint of every output is printed so that the two builds can be seen to agree.  The card's
name, power limit and SM clock are sampled with nvidia-smi during the timed region.
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
KERNELS = {
    "merkle_level_mma_kernel": "_ZN3tvm23merkle_level_mma_kernelEPmmm",
    "tip5_hash_rows_mma_tma_kernel": "_ZN3tvm29tip5_hash_rows_mma_tma_kernelENS_14HashRowsParamsE",
    "tip5_hash_rows_mma_kernel": "_ZN3tvm25tip5_hash_rows_mma_kernelENS_14HashRowsParamsE",
}
LOG2_ROWS, LOG2_COSETS = 23, 3
SHAPES = [("main", 379), ("aux", 273), ("quotient", 15)]
PERMS_PER_WARP_CALL = 16          # 8 quads x 2 rows share one round loop


# ---- SASS ------------------------------------------------------------------------------------------------------------
def opclass(op):
    if op.startswith("IMAD.WIDE"):
        return "IMAD.WIDE"
    for c in ("IADD3", "IMAD", "IMMA", "PRMT", "LOP3", "ISETP", "SEL", "SHF", "LEA", "LDS", "MOV"):
        if op == c or op.startswith(c + "."):
            return c
    return "other"


def sass(lib):
    """{kernel: {"total": n, "total_by_class": {...}, "round_body": n, "round_body_by_class": {...}}}"""
    out = subprocess.run(["cuobjdump", "-sass", "-fun", ",".join(KERNELS.values()), lib], check=True, capture_output=True,
                         text=True).stdout
    res = {}
    for name, mangled in KERNELS.items():
        m = re.search(r"Function : " + re.escape(mangled) + r"\n(.*?)(?=\n\s*Function : |\Z)", out, re.S)
        if not m:
            raise SystemExit(f"{name} not found in {lib}")
        ins = []                                    # (address, opcode, branch target or None)
        for line in m.group(1).splitlines():
            t = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(.*?);", line)
            if not t:
                continue
            body = re.sub(r"^@!?U?P[T0-9]+\s+", "", t.group(2).strip())
            op = body.split()[0]
            if op == "NOP":
                continue
            tgt = re.search(r"BRA\S*\s+(?:`\()?.*?0x([0-9a-f]+)", body) if op.startswith("BRA") else None
            ins.append((int(t.group(1), 16), op, int(tgt.group(1), 16) if tgt else None))
        # the round loop: the shortest backward branch whose body holds the IMMAs
        loops = [(a - t, t, a) for a, op, t in ins if t is not None and t < a
                 and any(o == "IMMA" or o.startswith("IMMA.") for x, o, _ in ins if t <= x <= a)]
        if not loops:
            raise SystemExit(f"{name}: no round loop found")
        _, lo, hi = min(loops)
        body = [op for a, op, _ in ins if lo <= a <= hi]
        count = lambda ops: dict(sorted(collections.Counter(opclass(o) for o in ops).items()))
        res[name] = {"total": len(ins), "total_by_class": count([op for _, op, _ in ins]), "round_body": len(body),
                     "round_body_by_class": count(body),
                     "warp_instructions_per_permutation": round(5 * len(body) / PERMS_PER_WARP_CALL, 1)}
    return res


# ---- timing (one process per library) --------------------------------------------------------------------------------
def worker(iters):
    # the Python bindings of the same build: <build>/lib/libtvm_b200.so -> <build>/py
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.environ["TVM_B200_LIB"])), "py"))
    import torch
    import tvm_b200
    dev = torch.device("cuda:0")
    b = tvm_b200.Backend(0)
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    b.set_stream(stream.cuda_stream)
    n = 1 << LOG2_ROWS
    g = torch.Generator(device=dev)
    g.manual_seed(1)
    maxc = max(c for _, c in SHAPES)
    table = torch.randint(0, 2**62, (maxc, n), dtype=torch.int64, device=dev, generator=g)   # < p: canonical
    nodes = torch.zeros((2 * n, 5), dtype=torch.int64, device=dev)
    idx = torch.arange(nodes.numel(), device=dev, dtype=torch.int64) * 2 + 1

    def fingerprint(t):
        return int((t.reshape(-1) * idx[: t.numel()]).sum().item()) & ((1 << 64) - 1)

    def timed(fn):
        fn()
        torch.cuda.synchronize()
        ms = []
        for _ in range(iters):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            fn()
            e.record()
            e.synchronize()
            ms.append(s.elapsed_time(e))
        return ms

    res = {}
    for name, ncols in SHAPES:
        ms = timed(lambda: b.hash_rows_dev(table, n, n, ncols, LOG2_COSETS, nodes[n:]))
        perms = n * (ncols // 10 + 1)
        res[f"hash_rows_{name}_{ncols}x2^{LOG2_ROWS}"] = {"ms": statistics.median(ms), "calls_ms": [round(x, 3) for x in ms],
                                                         "gperm_s": perms / statistics.median(ms) / 1e6,
                                                         "fingerprint": fingerprint(nodes[n:])}
    # the tree over the last shape's digests: leaves stay in place, every inner node is rewritten by each build
    ms = timed(lambda: b.merkle_dev(nodes, n))
    res[f"merkle_2^{LOG2_ROWS}"] = {"ms": statistics.median(ms), "calls_ms": [round(x, 3) for x in ms],
                                   "gperm_s": (n - 1) / statistics.median(ms) / 1e6, "fingerprint": fingerprint(nodes[1:n])}
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


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--lib", default=DEFAULT_LIB, help="this tree's build")
    ap.add_argument("--parent-lib", help="the build to compare against")
    ap.add_argument("--sass-only", action="store_true")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--out", help="directory for hash_time.json")
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        return worker(a.iters)
    libs = {"new": os.path.abspath(a.lib)}
    if a.parent_lib:
        libs["parent"] = os.path.abspath(a.parent_lib)
    report = {"sass": {k: sass(v) for k, v in libs.items()}}
    if not a.sass_only:
        if "parent" not in libs:
            raise SystemExit("--parent-lib is required for timing")
        runs = {k: [] for k in libs}
        clocks = Clocks()
        try:                                  # the sampler is stopped on every way out, a failed worker included
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
        summary = {}
        for shape in runs["new"][0]:
            per = {k: [r[shape]["ms"] for r in runs[k]] for k in runs}
            med = {k: statistics.median(v) for k, v in per.items()}
            summary[shape] = {
                "parent_ms": [round(x, 3) for x in per["parent"]], "new_ms": [round(x, 3) for x in per["new"]],
                "parent_median_ms": round(med["parent"], 3), "new_median_ms": round(med["new"], 3),
                "spread_ms": round(max(max(v) - min(v) for v in per.values()), 3),
                "speedup": round(med["parent"] / med["new"], 4),
                "new_gperm_s": round(statistics.median(r[shape]["gperm_s"] for r in runs["new"]), 3),
                "parent_gperm_s": round(statistics.median(r[shape]["gperm_s"] for r in runs["parent"]), 3),
                "outputs_equal": len({r[shape]["fingerprint"] for k in runs for r in runs[k]}) == 1,
            }
        report["timing"] = summary
    text = json.dumps(report, indent=1)
    print(text)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "hash_time.json"), "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
