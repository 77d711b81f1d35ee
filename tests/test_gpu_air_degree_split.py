"""The AIR quotient with every constraint evaluated on the even cosets (csrc/quotient.cu, the degree split and its top-degree
correction), against the C oracle's all_quotients_combined on every row of the 8n-point quotient domain.

Columns of degree D = n + h - 1 put the split in one of three modes: all constraints on half of the domain when 3D < 4n
(s = 4n - 3D >= 1), only those of degree <= 2 when 2D < 4n <= 3D, none otherwise.  Whole proofs reach only the heights
Stark::default() gives them; these shapes sit on either side of each boundary: s = 1 (the smallest top split), s = -2 (the
next h, n + 3 is never a multiple of 3: the degree <= 2 split), h = 0 (no top coefficients at all), a typical h, and h = n,
the largest h the degree <= 2 split takes."""
import numpy as np
import pytest
import torch

from oracle import corc

P = (1 << 64) - (1 << 32) + 1
NM, NA3 = 379, 270
OFFSET = 7


@pytest.mark.gpu
@pytest.mark.parametrize("log_n,h", [(10, 342), (10, 343), (10, 0), (11, 228), (9, 512)])
def test_quotient_from_coefficients_on_every_row(backend, log_n, h):
    n = 1 << log_n
    s = 4 * n - 3 * (n + h - 1)
    assert (log_n, h) != (10, 342) or s == 1
    assert (log_n, h) != (10, 343) or s == -2
    N, ln = 8 * n, log_n + 3
    rng = np.random.default_rng([log_n, h])
    coef = rng.integers(0, P, size=(NM + NA3, n + h), dtype=np.uint64)      # columns of degree exactly n + h - 1 (almost surely)
    ch = rng.integers(0, P, size=(63, 3), dtype=np.uint64)
    w = rng.integers(0, P, size=(604, 3), dtype=np.uint64)
    lde = np.stack([corc.coset_evaluate(c, OFFSET, ln) for c in coef])    # natural order: row i at 7 * w_N^i
    want = corc.air_quotient(lde[:NM], lde[NM:], log_n, OFFSET, ch, w)
    dev = torch.device("cuda:0")
    d_coef = torch.from_numpy(coef.view(np.int64)).to(dev)
    backend.to_mont_(d_coef)
    d_out = torch.zeros((3, N), dtype=torch.int64, device=dev)
    backend.air_quotient_coef_dev(d_coef[:NM], d_coef[NM:], n + h, h, ch, w, log_n, OFFSET, d_out, N)
    backend.from_mont_(d_out)
    backend.synchronize()
    got = d_out.cpu().numpy().view(np.uint64).reshape(3, 8, n).transpose(2, 1, 0).reshape(N, 3)   # coset-major -> natural
    bad = np.nonzero((got != want).any(axis=1))[0]
    assert bad.size == 0, f"{bad.size} of {N} rows differ; first: row {bad[0]} (coset {bad[0] % 8}, k = {bad[0] // 8})"
