"""Time the stand-alone STIR prover tvm_stir_prove_k at the size of a padded-height-2^20 prove's low-degree test (security
160, expansion 2^2, 2^23 points), with the codeword already in device memory, at folding factors 4, 8 and 16.

Prints one JSON line: the card's name and power limit (read in the same run), and per factor the milliseconds per call
(median, min and max of --calls calls after two warm-up calls), kernel launches per call and the proof length in words.

With --baseline-lib PATH (a libtvm_b200.so built from another commit) the factor-4 calls alternate between that
library's tvm_stir_prove and this tree's tvm_stir_prove_k, so that both see the same machine state; both proofs must be
the same words.  Needs a GPU and the built library of this tree."""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "triton-vm_b200", "py")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

import tvm_b200  # noqa: E402

SECURITY, LOG2_EXP, LOG2_DOMAIN = 160, 2, 23
_vp, _u64p = ctypes.c_void_p, ctypes.POINTER(ctypes.c_uint64)
_szp, _u32p = ctypes.POINTER(ctypes.c_size_t), ctypes.POINTER(ctypes.c_uint32)


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                         text=True, check=True).stdout.strip()
    name, power = [s.strip() for s in out.split(",")]
    return name, power


class Prover:
    """one library's context and its STIR entry point; call(log2_ff) -> (seconds, launches, proof words)"""
    def __init__(self, lib, k_entry):
        lib.tvm_ctx_create.argtypes = [ctypes.POINTER(_vp), ctypes.c_int]
        lib.tvm_ctx_destroy.argtypes = [_vp]
        lib.tvm_launch_count.argtypes, lib.tvm_launch_count.restype = [_vp], ctypes.c_uint64
        lib.tvm_last_error.argtypes, lib.tvm_last_error.restype = [_vp], ctypes.c_char_p
        self.lib, self.k_entry, self.h = lib, k_entry, _vp()
        assert lib.tvm_ctx_create(ctypes.byref(self.h), 0) == 0
        self.buf = np.empty(1 << 22, dtype=np.uint64)
        self.idx = (ctypes.c_uint32 * 8192)()

    def call(self, log2_ff, cw_ptr):
        cap, icap = ctypes.c_size_t(self.buf.size), ctypes.c_size_t(8192)
        hdb = LOG2_DOMAIN - LOG2_EXP
        before = self.lib.tvm_launch_count(self.h)
        t0 = time.perf_counter()
        if self.k_entry:
            rc = self.lib.tvm_stir_prove_k(self.h, SECURITY, 0, log2_ff, LOG2_EXP, hdb, cw_ptr, self.buf.ctypes.data_as(_u64p),
                                           ctypes.byref(cap), self.idx, ctypes.byref(icap))
        else:
            assert log2_ff == 2
            rc = self.lib.tvm_stir_prove(self.h, SECURITY, 0, LOG2_EXP, hdb, cw_ptr, self.buf.ctypes.data_as(_u64p), ctypes.byref(cap),
                                         self.idx, ctypes.byref(icap))
        dt = time.perf_counter() - t0      # the call returns after the proof words are back on the host
        assert rc == 0, (rc, self.lib.tvm_last_error(self.h))
        return dt, self.lib.tvm_launch_count(self.h) - before, self.buf[:cap.value].copy()


def summary(times):
    ms = [1e3 * t for t in times]
    return {"median_ms": round(statistics.median(ms), 3), "min_ms": round(min(ms), 3), "max_ms": round(max(ms), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--factors", default="2,3,4", help="log2 folding factors")
    ap.add_argument("--baseline-lib", default=None, help="libtvm_b200.so of another build, alternated with this one at factor 4")
    args = ap.parse_args()
    name, power = card()

    new_lib = tvm_b200.lib()
    vp = [_vp] + [ctypes.c_uint32] * 5 + [_vp, _u64p, _szp, _u32p, _szp]
    new_lib.tvm_stir_prove_k.argtypes = vp
    b = tvm_b200.Backend(0)
    vals = np.random.default_rng(0x5354).integers(0, tvm_b200.P, size=(3, 1 << (LOG2_DOMAIN - LOG2_EXP)), dtype=np.uint64)
    cw = torch.from_numpy(np.ascontiguousarray(b.lde(vals, None, LOG2_EXP, 7).T)).cuda()
    torch.cuda.synchronize()
    ptr = ctypes.c_void_p(cw.data_ptr())
    new = Prover(new_lib, True)
    old = None
    if args.baseline_lib:
        old_lib = ctypes.CDLL(os.path.abspath(args.baseline_lib))
        old_lib.tvm_stir_prove.argtypes = [_vp] + [ctypes.c_uint32] * 4 + [_vp, _u64p, _szp, _u32p, _szp]
        old = Prover(old_lib, False)

    result = {"card": name, "power_limit": power, "security": SECURITY, "log2_expansion": LOG2_EXP, "log2_domain": LOG2_DOMAIN,
              "calls": args.calls, "factors": {}}
    for log2_ff in [int(f) for f in args.factors.split(",")]:
        for _ in range(2):
            new.call(log2_ff, ptr)
            if old and log2_ff == 2:
                old.call(log2_ff, ptr)
        t_new, t_old = [], []
        for _ in range(args.calls):
            if old and log2_ff == 2:
                dt, _, proof_old = old.call(log2_ff, ptr)
                t_old.append(dt)
            dt, launches, proof = new.call(log2_ff, ptr)
            t_new.append(dt)
        entry = dict(summary(t_new), launches_per_call=int(launches), proof_words=int(proof.size))
        if old and log2_ff == 2:
            assert np.array_equal(proof, proof_old), "the two builds' proofs differ"
            entry["baseline"] = summary(t_old)
            entry["within_baseline_spread"] = entry["baseline"]["min_ms"] <= entry["median_ms"] <= entry["baseline"]["max_ms"]
        result["factors"][str(1 << log2_ff)] = entry
    new.lib.tvm_ctx_destroy(new.h)
    if old:
        old.lib.tvm_ctx_destroy(old.h)
    b.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
