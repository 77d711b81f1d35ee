"""The degree split's top-degree correction (csrc/quotient.cu, air_top_correction), restated with the oracle's AIR
evaluators on random columns at a small trace length.

Columns are random polynomials of degree D = n + h - 1 in u (the coefficient arrays' variable).  For each zerofier class
the weighted constraint sum C has degree <= 4D and C = r + u^{4n} q with deg r < 4n.  Its values on the 4n even points
u in <w_{8n}^2> interpolate to r + q; with q read off the degree-4 part H4 of C applied to the column tops,
q_i = [u^(i + 12(h-1))] H4(T), the odd points u in w_{8n}<w_{8n}^2> carry r - q.  The restatement must equal direct
evaluation on all 8n points when s = 4n - 3D >= 1, and must not when q is read one coefficient off, when the factor 2 is
dropped, or when s < 1."""
import functools

import numpy as np
import pytest

from oracle import corc
from oracle.field import P, xmul, xadd, xsub, xscale, inv

NM, NAX = 379, 90                     # main columns, aux X-field columns the constraints read
COUNTS = (81, 97, 403, 23)            # init, cons, tran, term


def root(log_len):
    e = np.zeros(1 << log_len, dtype=np.uint64)
    e[1] = 1
    return int(corc.ntt(e)[1])        # the transforms' own w_{2^log_len}


@functools.lru_cache(maxsize=None)
def case(log_n, h):
    n = 1 << log_n
    rng = np.random.default_rng([log_n, h, 5])
    coef = rng.integers(0, P, size=(NM + 3 * NAX, n + h), dtype=np.uint64)
    ch = rng.integers(0, P, size=(63, 3), dtype=np.uint64)
    w = [tuple(int(v) for v in row) for row in rng.integers(0, P, size=(604, 3), dtype=np.uint64)]
    return n, coef, ch, w


def class_sums(ch, w, main, aux, main_next, aux_next):
    """the four weighted constraint sums (init, cons, tran, term) at one point, from the column values there"""
    out, off = [], 0
    for cat in range(4):
        vals = corc.air_eval_category(cat, main, aux.reshape(NAX, 3), main_next, aux_next.reshape(NAX, 3), ch)
        acc = (0, 0, 0)
        for j in range(COUNTS[cat]):
            acc = xadd(acc, xmul(w[off + j], tuple(int(v) for v in vals[j])))
        out.append(acc)
        off += COUNTS[cat]
    return out


@functools.lru_cache(maxsize=None)
def direct(log_n, h):
    """class sums on all 8n points u = w_{8n}^i (natural order): [8n][4] X-field"""
    n, coef, ch, w = case(log_n, h)
    vals = np.stack([corc.coset_evaluate(c, 1, log_n + 3) for c in coef])   # [cols][8n]
    nxt = np.roll(vals, -8, axis=1)                                           # col(w_n u): w_n = w_{8n}^8
    return [class_sums(ch, w, vals[:NM, i], vals[NM:, i], nxt[:NM, i], nxt[NM:, i]) for i in range(8 * n)]


def odd_by_method(log_n, h, q_shift=0, factor=2):
    """the odd points' class sums from the even points' and the tops, as the device computes them: [4n][4]"""
    n, coef, ch, w = case(log_n, h)
    D = n + h - 1
    s, count = 4 * n - 3 * D, 4 * h - 3
    even = direct(log_n, h)[0::2]
    log_L = max(6, (16 * h - 15 - 1).bit_length())
    L = 1 << log_L
    # tops of the current and next-row polynomials at the L points
    wn = root(log_n)
    tops = np.zeros((2 * coef.shape[0], L), dtype=np.uint64)
    first = max(s, 0)                 # (s < 1 is the misuse one test makes: the tops are then cut at coefficient 0)
    for q in range(coef.shape[0]):
        t = [int(v) for v in coef[q, first:D + 1]]
        tops[q, :len(t)] = t
        tops[coef.shape[0] + q, :len(t)] = [v * pow(wn, first + i, P) % P for i, v in enumerate(t)]
    tv = np.stack([corc.ntt(t) for t in tops])
    ncur = coef.shape[0]
    h4 = [[None] * L for _ in range(4)]
    inv24 = inv(24)
    for t in range(L):
        sums = {}
        for lam in (0, 1, -1, 2, -2):
            col = [(lam * int(v)) % P for v in tv[:, t]]
            cur, nx = np.array(col[:ncur], dtype=np.uint64), np.array(col[ncur:], dtype=np.uint64)
            sums[lam] = class_sums(ch, w, cur[:NM], cur[NM:], nx[:NM], nx[NM:])
        for k in range(4):
            v = xadd(xadd(sums[2][k], sums[-2][k]), xscale(sums[0][k], 6))
            v = xsub(v, xscale(xadd(sums[1][k], sums[-1][k]), 4))
            h4[k][t] = xscale(v, inv24)
    w8n = root(log_n + 3)
    out = []
    for k in range(4):
        hc = corc.xntt(np.array(h4[k], dtype=np.uint64), inverse=True)               # coefficients of H4(T)
        rq = corc.xntt(np.array([even[i][k] for i in range(4 * n)], dtype=np.uint64), inverse=True)   # r + q
        for i in range(count):
            qi = tuple(int(v) for v in hc[i + 12 * (h - 1) + q_shift])
            rq[i] = [int(v) for v in xsub(tuple(int(x) for x in rq[i]), xscale(qi, factor))]
        shifted = np.array([[int(v) * pow(w8n, j, P) % P for v in rq[j]] for j in range(4 * n)], dtype=np.uint64)
        out.append(corc.xntt(shifted))                                                # values at w_{8n} w_{4n}^i
    return [[tuple(int(v) for v in out[k][i]) for k in range(4)] for i in range(4 * n)]


def test_roots_are_one_family():
    assert pow(root(6), 2, P) == root(5) and pow(root(6), 8, P) == root(3)


@pytest.mark.parametrize("log_n,h", [(3, 2), (4, 3)])     # s = 5 and s = 10
def test_odd_cosets_from_even_cosets_and_tops(log_n, h):
    assert 4 * (1 << log_n) - 3 * ((1 << log_n) + h - 1) >= 1
    assert odd_by_method(log_n, h) == direct(log_n, h)[1::2]


@pytest.mark.parametrize("kw", [{"q_shift": 1}, {"q_shift": -1}, {"factor": 1}])
def test_a_wrong_correction_is_caught(kw):
    assert odd_by_method(3, 2, **kw) != direct(3, 2)[1::2]


def test_the_correction_needs_s_at_least_one():
    # n = 8, h = 4: 3D = 33 > 4n = 32, so terms of degree >= 4n also come from products of lower coefficients
    assert odd_by_method(3, 4) != direct(3, 4)[1::2]
