"""Row hashing and Merkle trees through the device entry points (tvm_tip5_hash_rows_dev, tvm_merkle_build_dev) against the
C oracle, on Montgomery words chosen at the boundaries of the representation, and the permutation's arithmetic pieces
(fsqr, the power map x^7, the lazy and the canonical MDS finish) against Python integers.

Inside the permutation only the look-up element of each lane (state elements 0..3) is kept canonical; the x^7 elements
carry any representative < 2^64 from one round to the next (and the capacity from one absorption to the next), and the
stored digest words are canonicalised once.  A lazy element is >= p only when the folded MDS sum lands in [p, 2^64): for
uniformly distributed state that is (2^64 - p) / 2^64 = (2^32 - 1) / 2^64, about 2^-32 per element and round.  Random
rows therefore almost never reach that case: 2^16 rows x 3 absorptions x 5 rounds x 12 lazy elements x 2^-32 is about
2^-8.5 expected occurrences.  test_arith_check covers it with constructed operands; the row and tree tests cover the common
path at volume.  Two properties are NOT exercised by any input here, because no feasible input drives them to a
non-canonical word: that the stored digest word 4 is canonicalised (fcanon at every digest store of the three kernels), and
that only slot 0 (elements 0..3, always finished canonically) feeds a look-up.  Both rest on the code of
tip5_perm_quad2_mma and its callers.  No input here is outside what the entry points accept."""
import numpy as np
import pytest
import torch

from oracle import corc

pytestmark = pytest.mark.gpu

P = (1 << 64) - (1 << 32) + 1
R_INV = pow(1 << 64, -1, P)
M64 = (1 << 64) - 1

# canonical Montgomery words at the edges: 0, 1, 2^32 - 1, 2^32, p - 1, words just under p made of 0xFF bytes, and a
# word of every repeated byte value below 0xFF, so that the first round's look-up lanes see every byte
BOUNDARY = sorted({0, 1, (1 << 32) - 1, 1 << 32, P - 1, P - 2, 0xFFFFFFFEFFFFFFFF, 0xFFFFFFFEFFFFFF00, 0xFFFFFFFEFF00FFFF,
                   0xFEFFFFFFFFFFFFFF, 0xFFFFFFFE00000000, 0x00000000FFFFFFFF, 0xFFFFFFFF00000000 - 0xFF}
                  | {b * 0x0101010101010101 for b in range(255)})
assert all(w < P for w in BOUNDARY)


def to_dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint64).view(np.int64)).to("cuda:0")


def to_host(t):
    return t.cpu().numpy().view(np.uint64)


def hash_rows_dev(backend, table_mont, log2_cosets=0):
    ncols, nrows = table_mont.shape
    d_tab = to_dev(table_mont)
    d_dig = torch.zeros((nrows, 5), dtype=torch.int64, device="cuda:0")
    backend.hash_rows_dev(d_tab, nrows, nrows, ncols, log2_cosets, d_dig)
    backend.synchronize()
    return to_host(d_dig)


def coset_major_to_natural(table, log2_cosets):
    """the device reads column q as coset-major ([coset][k] = row coset + r*k); the oracle takes natural row order"""
    ncols, nrows = table.shape
    r = 1 << log2_cosets
    return table.reshape(ncols, r, nrows // r).transpose(0, 2, 1).reshape(ncols, nrows)


@pytest.mark.parametrize("nrows,log2_cosets", [(512, 3), (300, 0)])   # bulk-copy staged kernel / per-lane loads
@pytest.mark.parametrize("ncols", [1, 9, 10, 11, 379, 273])
def test_hash_rows_boundary_words(backend, ncols, nrows, log2_cosets):
    rng = np.random.default_rng(1000 * ncols + nrows)
    words = np.array(BOUNDARY, dtype=np.uint64)
    tab = words[rng.integers(0, words.size, size=(ncols, nrows))]
    tab[:, 0] = words[np.arange(ncols) % words.size]                 # every boundary word in some column of row 0 ...
    tab[0, : min(nrows, words.size)] = words[: min(nrows, words.size)]   # ... and every one in look-up lane 0
    got = hash_rows_dev(backend, tab, log2_cosets)
    want = corc.hash_rows_colmajor(coset_major_to_natural(tab, log2_cosets), mont_io=True)
    assert np.array_equal(got, want)


def test_hash_rows_random_rows(backend):
    rng = np.random.default_rng(77)
    ncols, nrows, log2_cosets = 21, 1 << 16, 3
    tab = rng.integers(0, P, size=(ncols, nrows), dtype=np.uint64)
    got = hash_rows_dev(backend, tab, log2_cosets)
    want = corc.hash_rows_colmajor(coset_major_to_natural(tab, log2_cosets), mont_io=True)
    assert np.array_equal(got, want)


@pytest.mark.parametrize("leaves_kind", ["boundary", "random"])
def test_merkle_build_dev(backend, leaves_kind):
    rng = np.random.default_rng(5)
    if leaves_kind == "boundary":
        n = 1 << 10
        words = np.array(BOUNDARY, dtype=np.uint64)
        leaves = words[rng.integers(0, words.size, size=(n, 5))]
        leaves[: words.size // 5] = words[: 5 * (words.size // 5)].reshape(-1, 5)
    else:
        n = 1 << 16
        leaves = rng.integers(0, P, size=(n, 5), dtype=np.uint64)
    d_nodes = torch.zeros((2 * n, 5), dtype=torch.int64, device="cuda:0")
    d_nodes[n:] = to_dev(leaves)
    backend.merkle_dev(d_nodes, n)
    backend.synchronize()
    got = to_host(d_nodes)
    want = corc.merkle_build(leaves, mont_io=True)
    assert np.array_equal(got[1:], want[1:])


def test_arith_check(backend):
    """fsqr and the power map x^7 against Python integers on canonical and non-canonical words; the lazy MDS finish returns a
    representative < 2^64 (and >= p for the constructed cases below), the canonical finish the canonical value."""
    rng = np.random.default_rng(9)
    xs = [0, 1, 2, (1 << 32) - 1, 1 << 32, (1 << 32) + 1, 1 << 63, P - 1, P, P + 1, M64 - 1, M64]
    xs += [int(v) for v in rng.integers(0, 1 << 64, size=200, dtype=np.uint64)]
    L = (1 << 47) - 1
    T = (1 << 21) - 1
    fin = [(lo, hi, top, rc) for lo in (0, 1, L) for hi in (0, 1, L) for top in (0, 1, T) for rc in (0, 1, P - 1, P, M64)]
    # the fold lands in [p, 2^64) and n = 0: the lazy result is the non-canonical word itself
    fin += [(0, 0, 0, P), (0, 0, 0, M64), (5, 0, 0, P - 1), (0, (1 << 32) - 1, 0, (1 << 32) * 0xFFFFFFFF)]
    # n = 1 (a carry into 2^64 after the fold), and the borrow that the carry cancels
    fin += [(L, L, T, M64), (0, 0, T, 0), (0, 0, 1, 0), (1, 0, T, 0)]
    fin += [(int(rng.integers(0, L + 1)), int(rng.integers(0, L + 1)), int(rng.integers(0, T + 1)),
             int(rng.integers(0, 1 << 64, dtype=np.uint64))) for _ in range(200)]
    n = max(len(xs), len(fin))
    xs += [xs[i % len(xs)] for i in range(n - len(xs))]
    fin += [fin[i % len(fin)] for i in range(n - len(fin))]
    inp = np.array([[x, *f] for x, f in zip(xs, fin)], dtype=np.uint64)
    d_in = to_dev(inp)
    d_out = torch.zeros((n, 4), dtype=torch.int64, device="cuda:0")
    backend.tip5_arith_check_dev(d_in, n, d_out)
    backend.synchronize()
    out = to_host(d_out)
    lazy_noncanonical = 0
    for (x, lo, hi, top, rc), (sq, p7, lazy, canon) in zip(inp.tolist(), out.tolist()):
        assert sq % P == x * x * R_INV % P, hex(x)
        assert p7 % P == pow(x, 7, P) * pow(R_INV, 6, P) % P, hex(x)   # Montgomery form: x^7 R^-6
        if x < P:
            assert sq < P and p7 < P, hex(x)
        v = lo + (hi << 32) + (top << 64) + rc
        assert canon == v % P, (lo, hi, top, rc)
        assert lazy % P == v % P, (lo, hi, top, rc)
        lazy_noncanonical += lazy >= P
    assert lazy_noncanonical >= 3
