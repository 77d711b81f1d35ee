"""Searches for a 32-byte prover seed whose StdRng stream has a SHORT sample among its first 64 B-field draws and writes it to
tests/golden/short_draw_seed.json.

A short sample is one where rand's Canon method needs only one u64 of the stream instead of two (probability 2^-32 per
draw, see triton-vm_b200/csrc/rand/prover_randomness.cuh); every later sample of the stream then starts one u64 earlier.
Random seeds practically never reach that path, so the tests use this fixture.  With it as the prover's seed, main column
0's trace randomizers (drawn from the seed itself) take the short path.

The search runs the sampler's own ChaCha12 and Canon code through the host harness of tests/host/prover_randomness_host.cu
on all CPU threads: about 2^26 seeds of 16 ChaCha blocks each, minutes.  The result is then checked against the oracle's
StdRng (oracle/rand_compat.py).

    python tests/golden/make_short_draw_seed.py"""
import ctypes
import json
import os
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.dirname(HERE)]

from oracle.rand_compat import StdRng   # noqa: E402
import test_prover_randomness_host as T  # noqa: E402

PREFIX = b"triton-vm short draw seed"[:24]
SAMPLES = 64
CHUNK = 1 << 24


def main():
    lib = T.build_host()
    found_i, found_j = ctypes.c_uint64(), ctypes.c_uint64()
    threads = os.cpu_count() or 1
    first, t0 = 0, time.time()
    while not lib.prand_host_search(PREFIX, ctypes.c_uint64(first), ctypes.c_uint64(CHUNK), SAMPLES, threads, ctypes.byref(found_i),
                                    ctypes.byref(found_j)):
        first += CHUNK
        print(f"{first} seeds searched, {time.time() - t0:.0f} s", flush=True)
    seed = PREFIX + int(found_i.value).to_bytes(8, "little")
    j = int(found_j.value)
    r = StdRng(seed)                         # the oracle must agree: sample j consumes exactly one u64
    for _ in range(j):
        r.bfe()
    before = r.index + 16 * r.counter
    r.bfe()
    assert r.index + 16 * r.counter - before == 2, "the oracle does not see a short sample there"
    out = {"seed_hex": seed.hex(), "short_sample": j, "samples_searched": SAMPLES, "seeds_searched": int(found_i.value) + 1}
    with open(os.path.join(HERE, "short_draw_seed.json"), "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")
    print(out, f"{time.time() - t0:.0f} s")


if __name__ == "__main__":
    main()
