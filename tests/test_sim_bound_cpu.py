"""Without a GPU: every instance of tests/sim_bound_cases.py has the properties the GPU tests rely on.

- the restated operands: the centres are exact, the query centring flag is what the case asks for, A rounds down and the
  competitors round up;
- exactness: every fp32 partial sum of the column sums and of the tensor-core accumulation, and every fp64 dot product;
- the inversion: A is the exact best (or tied with its twin at a higher index), every competitor's bf16 score is above A's;
- the realized error: A's bf16 rounding costs at least 0.9 of eps's bf16 terms, and no row's error exceeds eps.
"""
import numpy as np
import pytest

from tests import sim_bound_cases as sbc

CASES = [(name, d, centred) for name in ("k1_first", "k10_second", "k16_brute", "k10_shared", "k10_tie")
         for d in sbc.DIMS for centred in (False, True)]


def _case(name, d, centred):
    c = sbc.topk_case(name, d, centred)
    return c, sbc.operands(c.q, c.g)


@pytest.mark.parametrize("name,d,centred", CASES)
def test_operands_are_restated_exactly(name, d, centred):
    c, op = _case(name, d, centred)
    # centres: mu = 0 from the +- pairs, nu = c (8 p or 0); the flag follows the case
    assert not op.mu.any()
    assert op.flag == centred
    p = np.concatenate([np.ones(d // 2), -np.ones(d // 2)]).astype(np.float32)
    assert np.array_equal(op.nu, 8 * p if centred else np.zeros(d, np.float32))
    # col_sum_kernel's fp32 partial sums are exact: every column's sum of |x| stays below 2^24 quanta
    assert (np.abs(sbc.as_integers(c.g, sbc.U)).sum(axis=0) < 2 ** 24).all()
    assert (np.abs(sbc.as_integers(c.q, 0.5)).sum(axis=0) ** 2 < 2 ** 24).all()
    # the centred queries are +-w: bf16-exact, no query residual
    assert np.array_equal(np.abs(op.qv), np.ones_like(op.qv)) and np.array_equal(op.qh, op.qv)
    for i in range(c.q.shape[0]):
        s = np.sign(op.qv[i, 0])
        a = s * op.gh[c.target[i]]
        assert np.array_equal(a, np.ones(d, np.float32))                       # A rounds down to 1 ...
        assert np.array_equal(s * op.gv[c.target[i]] - a, np.full(d, 7 * sbc.U, np.float32))   # ... by 7 quanta each
        for b in c.comps[i]:
            vals = s * op.gh[b]                                                 # B rounds up to 1 + 2^-7 or 1
            assert np.isin(vals, np.float32([1.0, 1.0 + 2 ** -7])).all()
            assert (s * (op.gv[b] - op.gh[b]) < 0).all()


@pytest.mark.parametrize("name,d,centred", CASES)
def test_scores_are_exact(name, d, centred):
    c, op = _case(name, d, centred)
    qi, gi = sbc.as_integers(c.q, 0.5), sbc.as_integers(c.g, sbc.U)
    ints = qi @ gi.T                                                             # exact, in units of 2^-12
    assert np.abs(ints).max() < 2 ** 53
    assert np.array_equal(sbc.exact(c.q, c.g), ints * (0.5 * sbc.U))
    # the tensor-core accumulation: bf16 products on a 2^-9 grid whose absolute sum stays below 2^24 of them
    hq, hg = sbc.as_integers(op.qh, 0.5), sbc.as_integers(op.gh, 2.0 ** -8)
    assert (np.abs(hq) @ np.abs(hg).T).max() < 2 ** 24
    # the column offset nu.(g - mu) is exact in fp32
    bias64 = op.gv.astype(np.float64) @ op.nu.astype(np.float64)
    assert np.array_equal(op.bias.astype(np.float64), bias64 if op.flag else np.zeros_like(bias64))


@pytest.mark.parametrize("name,d,centred", CASES)
def test_bf16_order_inverts_exact_order(name, d, centred):
    c, op = _case(name, d, centred)
    ex, ap = sbc.exact(c.q, c.g), sbc.approx(op)
    e = sbc.eps(op, d)
    for i in range(c.q.shape[0]):
        a, comps, tw = c.target[i], c.comps[i], c.twin[i]
        others = np.setdiff1d(np.arange(c.g.shape[0]), [a, tw])
        assert (ex[i, others] < ex[i, a]).all()                                 # A is the exact best ...
        assert (ap[i, comps] > ap[i, a]).all()                                  # ... below every competitor in bf16
        assert ex[i, a] - ex[i, comps].max() <= 24 * d * sbc.U                  # close competitors
        if tw >= 0:                                                             # exact tie, higher index, better bf16
            assert ex[i, tw] == ex[i, a] and tw > a and ap[i, tw] - ap[i, a] > e[i]
        fillers = np.setdiff1d(others, comps)
        assert ex[i, fillers].max() < ex[i, a] - 4 * e[i]                       # fillers never compete
        # the fp32 scores keep the order: the threshold search at A's score sees the competitors below it
        assert (ex[i, comps].astype(np.float32) < np.float32(ex[i, a])).all()
        assert (ap[i, comps] >= np.float32(ex[i, a])).all()


@pytest.mark.parametrize("name,d,centred", CASES)
def test_realized_error_reaches_the_bound(name, d, centred):
    c, op = _case(name, d, centred)
    e, terms = sbc.eps(op, d), sbc.bf16_terms(op)
    r = sbc.realized(c, op)
    assert (r >= 0.9 * terms).all(), r / terms
    assert (r <= e).all()
    # the bound holds for every pair, so the instance is one the kernel must rank exactly
    err = np.abs(c.q.astype(np.float64) @ op.gv.astype(np.float64).T - sbc.approx(op))
    assert (err <= e[:, None]).all()
    # A's rows hold the largest residual, competitor or twin rows the largest norm
    res = np.linalg.norm(op.gv.astype(np.float64) - op.gh, axis=1)
    assert set(np.flatnonzero(res == res.max())) <= set(c.target)
    nrm = np.linalg.norm(op.gv.astype(np.float64), axis=1)
    special = set(c.target) | set(np.concatenate(c.comps)) | set(c.twin[c.twin >= 0])
    assert set(np.flatnonzero(nrm == nrm.max())) <= special


def test_many_query_instance():
    """The threshold-search instance with 3 scales x 43 query pairs: centres still exact, both centring branches."""
    for centred in (False, True):
        c = sbc.build(512, 20, centred=centred, scales=(1.0, 2.0, 0.5) * 43)
        op = sbc.operands(c.q, c.g)
        assert op.flag == centred and not op.mu.any()
        r, terms = sbc.realized(c, op), sbc.bf16_terms(op)
        assert (r >= 0.9 * terms).all() and (r <= sbc.eps(op, 512)).all()
