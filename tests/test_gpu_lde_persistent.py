"""The persistent tile-NTT launch (ntt_tile.cu) behind tvm_lde_bfe_dev, word for word against the C oracle.

One launch runs both passes of a batch: CTAs take tiles from a ticket counter, and a pass-B tile waits until every
pass-A tile of its pair (a column group x a coset group) has finished.  The shapes below give several pairs in flight,
a partial last column group (tickets that map to no column), and both fold counts.  TVM_NTT_TILE_CTAS forces the grid to
one CTA (every wait is then on tiles this CTA has already finished) and to sizes that divide no ticket count, so that the
pair waits run with CTAs at different points of the ticket order; it changes the grid size and nothing else."""
import numpy as np
import pytest

from conftest import rand_bfes
from oracle import corc

pytestmark = pytest.mark.gpu

# (log2 n, columns): with the default 16 MB pair budget a pair is 2 cosets of one column at 2^20, all 8 cosets of one
# column at 2^18, all 8 cosets of 4 / 16 / 64 columns at 2^16 / 2^14 / 2^12; the interpolation pairs 2 / 8 / 32 / 128 /
# 512 columns.  Every column count leaves a partial last group for the evaluation or the interpolation.
SHAPES = [(12, 70), (14, 20), (16, 10), (18, 3), (20, 3)]


def _check(backend, log2n, ncols, h, seed):
    rng = np.random.default_rng(seed)
    n = 1 << log2n
    trace = rand_bfes(rng, (ncols, n))
    rand = rand_bfes(rng, (ncols, h)) if h else None
    got = backend.lde(trace, rand, 3, 7)
    want = corc.lde_table(trace, rand, 7, log2n + 3)
    bad = [c for c in range(ncols) if not np.array_equal(got[c], want[c])]
    assert not bad, f"2^{log2n} x {ncols}, h = {h}: columns {bad[:8]} differ"


@pytest.mark.parametrize("log2n,ncols", SHAPES)
@pytest.mark.parametrize("h", [0, 228])
def test_lde_tiles_match_oracle(backend, log2n, ncols, h):
    _check(backend, log2n, ncols, h, 1000 * log2n + ncols + h)


@pytest.mark.parametrize("ctas", ["1", "7", "263"])
@pytest.mark.parametrize("log2n,ncols", [(16, 10), (20, 1)])
def test_lde_tiles_forced_grid(backend, monkeypatch, ctas, log2n, ncols):
    monkeypatch.setenv("TVM_NTT_TILE_CTAS", ctas)
    _check(backend, log2n, ncols, 228, 77 + log2n)


@pytest.mark.parametrize("log2n,first,step,count", [(20, 1, 2, 4), (18, 3, 4, 2), (16, 2, 3, 2)])
def test_lde_tiles_coset_subset(backend, log2n, first, step, count):
    """cosets first + step*y, y < count, of the 8 (one rank of a coset-sharded prove), against the oracle's full LDE"""
    import torch
    ncols, h, r = 3, 228, 8
    n = 1 << log2n
    rng = np.random.default_rng(31 + log2n)
    trace = rand_bfes(rng, (ncols, n))
    rand = rand_bfes(rng, (ncols, h))
    dev = torch.device("cuda:0")
    d_trace = backend.to_mont_(torch.from_numpy(trace.view(np.int64)).to(dev))
    d_rand = backend.to_mont_(torch.from_numpy(rand.view(np.int64)).to(dev))
    d_coef = torch.empty((ncols, 2 * n), dtype=torch.int64, device=dev)
    d_out = torch.empty((ncols, count * n), dtype=torch.int64, device=dev)
    d_tmp = torch.empty((ncols, r * n), dtype=torch.int64, device=dev)
    backend.lde_cosets_dev(d_trace, d_rand, h, log2n, 3, 7, first, step, count, ncols, d_coef, d_out, d_tmp)
    backend.from_mont_(d_out)
    backend.synchronize()
    got = d_out.cpu().numpy().view(np.uint64).reshape(ncols, count, n)
    want = corc.lde_table(trace, rand, 7, log2n + 3).reshape(ncols, n, r)   # natural index c + r*k
    for y in range(count):
        assert np.array_equal(got[:, y], want[:, :, first + step * y]), f"2^{log2n}: coset {first + step * y} differs"
