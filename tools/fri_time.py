"""tvm_fri_prove alone at the size the FRI of a padded-height-2^20 prove has (Stark::default()'s security 160 and expansion 4:
initial domain of 2^23 points, log2 high-degree bound 21): host clock around each call on a codeword already in device memory
(the call returns after the proof is on the host), median over --reps calls after --warmup.  The time includes the codeword's
conversion to Montgomery form and planar layout (one pass over 200 MB) and every per-round host round trip for the Merkle root.
Prints one JSON line with the card's name and power limit (read-only nvidia-smi query)."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "triton-vm_b200", "py"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import tvm_b200  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"], capture_output=True,
                             text=True, timeout=30).stdout.strip().split(", ")
        return out[0], float(out[1])
    except Exception:   # noqa: BLE001
        return torch.cuda.get_device_name(0), None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--security", type=int, default=160)
    ap.add_argument("--log2-expansion", type=int, default=2)
    ap.add_argument("--log2-hdb", type=int, default=21)
    ap.add_argument("--conjectured", action="store_true")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    b = tvm_b200.Backend(0)
    fd = tvm_b200.fri_derive(a.security, a.log2_expansion, a.log2_hdb, a.conjectured)
    g = torch.Generator(device="cuda")
    g.manual_seed(1)
    # canonical words below 2^62 < P, [domain_len][3]
    cw = torch.randint(0, 2**62, (fd["domain_len"], 3), dtype=torch.int64, device="cuda", generator=g)
    args = (a.security, a.log2_expansion, a.log2_hdb, cw, a.conjectured)
    for _ in range(a.warmup):
        want = b.fri_prove(*args)
    torch.cuda.synchronize()
    ms, l0 = [], b.launches
    for _ in range(a.reps):
        t0 = time.perf_counter()
        proof, idx = b.fri_prove(*args)
        ms.append((time.perf_counter() - t0) * 1e3)
        assert np.array_equal(proof, want[0]) and idx == want[1]
    ok = tvm_b200.fri_verify(a.security, a.log2_expansion, a.log2_hdb, proof, a.conjectured)[0]
    name, power = card()
    print(json.dumps(dict(gpu=name, power_limit_w=power, security=a.security, log2_expansion=a.log2_expansion, log2_hdb=a.log2_hdb,
                          domain_len=fd["domain_len"], num_rounds=fd["num_rounds"], num_collinearity_checks=fd["num_collinearity_checks"],
                          fri_prove_ms_median=round(float(np.median(ms)), 2), fri_prove_ms=[round(v, 2) for v in ms],
                          launches_per_call=(b.launches - l0) / a.reps, proof_words=int(proof.size),
                          random_codeword_rejected=not ok)))
    b.close()


if __name__ == "__main__":
    main()
