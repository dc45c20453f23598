"""Without a GPU: every split-score instance of tests/sim_bound_cases.py has the properties the GPU tests rely on.

- exactness: every fp32 partial sum of the tensor-core accumulation of every part, and every fp64 part dot product;
- the inversion: A is the exact best (or tied with its twin at a higher index); every competitor's bf16 split score is
  above A's while its fp32 split score is below A's;
- the realized error: A's bf16 rounding costs at least 0.9 of its part's bf16 terms, and no pair's error exceeds eps;
- quiet layout: eps comes from the instance part, every other part's term is at most 1e-3 of it, so a bound that reads
  another part's norms or gallery maxima, or that stops before the instance part, falls below A's realized error.
"""
import dataclasses

import numpy as np
import pytest

from tests import sim_bound_cases as sbc

# every instance at every placement of the shapes up to 4 parts; with 40 and 197 parts (the same p = 64 instances, 5 and
# 25 MB galleries) the tie and the threshold-search instance, which hold every kind of row the others do
CASES = [(name, c, p, layout, part, other)
         for c, p in sbc.RANGE_SPLIT_SHAPES
         for name in (("k1_first", "k10_second", "k16_brute", "k10_shared", "k10_tie", "range") if c <= 4
                      else ("k10_tie", "range"))
         for layout, part, other in sbc.split_placements(c)]


def _id(case):
    name, c, p, layout, part, other = case
    return f"{name}-C{c}-p{p}-{layout}{part}" + (f"-{other}" if other >= 0 else "")


def _case(name, c, p, layout, part, other):
    case = sbc.split_case(name, p, c, part, layout, other)
    return case, sbc.split_operands(case.q, case.g, c)


@pytest.mark.parametrize("name,c,p,layout,part,other", CASES, ids=[_id(x) for x in CASES])
def test_scores_are_exact(name, c, p, layout, part, other):
    case, op = _case(name, c, p, layout, part, other)
    qi, gi = sbc.as_integers(case.q, 0.5), sbc.as_integers(case.g, sbc.U)
    hq, hg = sbc.as_integers(op.qh, 0.5), sbc.as_integers(op.gh, sbc.U)
    # integers of at most 12 bits over at most 1024 terms: their fp64 part products are exact
    assert max(np.abs(qi).max(), np.abs(gi).max(), np.abs(hq).max(), np.abs(hg).max()) < 2 ** 12 and p <= 1024
    ints = sbc.part_products(qi, gi, c)                                # in units of 2^-12
    assert np.array_equal(sbc.split_exact(case.q, case.g, c), ints.max(axis=0) * (0.5 * sbc.U))
    # the tensor-core accumulation of every part: products on a 2^-12 grid whose absolute sum stays below 2^24 of them
    assert sbc.part_products(np.abs(hq), np.abs(hg), c).max() < 2 ** 24
    if layout == "quiet":                                              # the quiet parts score exactly 0
        others = [j for j in range(c) if j != part]
        assert not case.q.reshape(-1, c, p)[:, others].any()
        assert np.array_equal(hg.reshape(-1, c, p)[:, others], gi.reshape(-1, c, p)[:, others])


@pytest.mark.parametrize("name,c,p,layout,part,other", CASES, ids=[_id(x) for x in CASES])
def test_bf16_order_inverts_exact_order(name, c, p, layout, part, other):
    case, op = _case(name, c, p, layout, part, other)
    ex, ap = sbc.split_exact(case.q, case.g, c), sbc.split_approx(op, c)
    e = sbc.split_eps(op, sbc.d_pad(p))
    ex_parts = sbc.part_products(case.q, case.g, c)
    b_part = other if layout == "cross" else part
    for i in range(case.q.shape[0]):
        a, comps, tw = case.target[i], case.comps[i], case.twin[i]
        others = np.setdiff1d(np.arange(case.g.shape[0]), [a, tw])
        assert (ex[i, others] < ex[i, a]).all()                                 # A is the exact best ...
        assert (ap[i, comps] > ap[i, a]).all()                                  # ... below every competitor in bf16
        assert ex[i, a] - ex[i, comps].max() <= 24 * p * sbc.U                  # close competitors
        assert ex_parts[part][i, a] == ex[i, a]                                 # A scores in its part ...
        assert (ex_parts[b_part][i, comps] == ex[i, comps]).all()               # ... the competitors in theirs
        if layout == "cross":
            assert (np.delete(ex_parts[:, i, comps], other, axis=0) < ex[i, comps] - 4 * e[i]).all()
            assert (np.delete(ex_parts[:, i, a], part) < ex[i, a] - 4 * e[i]).all()
        if tw >= 0:                                                             # exact tie, higher index, better bf16
            assert ex[i, tw] == ex[i, a] and tw > a and ap[i, tw] - ap[i, a] > e[i]
        fillers = np.setdiff1d(others, comps)
        assert ex[i, fillers].max() < ex[i, a] - 4 * e[i]                       # fillers never compete
        # the fp32 scores keep the order: the threshold search at A's score sees the competitors below it
        assert (ex[i, comps].astype(np.float32) < np.float32(ex[i, a])).all()
        assert (ap[i, comps] >= np.float32(ex[i, a])).all()


@pytest.mark.parametrize("name,c,p,layout,part,other", CASES, ids=[_id(x) for x in CASES])
def test_realized_error_reaches_the_bound(name, c, p, layout, part, other):
    case, op = _case(name, c, p, layout, part, other)
    p_pad = sbc.d_pad(p)
    e, terms = sbc.split_eps(op, p_pad), sbc.split_bf16_terms(op)[:, part]
    r = sbc.split_realized(case, op)
    assert (r >= 0.9 * terms).all(), r / terms
    assert (r <= e).all()
    # the bound holds for every pair, so the instance is one the kernel must rank exactly
    err = np.abs(sbc.split_exact(case.q, case.g, c) - sbc.split_approx(op, c))
    assert (err <= e[:, None]).all()
    # the instance part's term is the row's eps
    assert np.array_equal(sbc.split_part_eps(op, p_pad)[:, part], e)


@pytest.mark.parametrize("name,c,p,layout,part,other",
                         [x for x in CASES if x[3] == "quiet"], ids=[_id(x) for x in CASES if x[3] == "quiet"])
def test_quiet_parts_leave_eps_to_the_instance_part(name, c, p, layout, part, other):
    """Every other part's term is at most 1e-3 of the instance part's.  So each of these misreadings of split_row_bound
    gives a bound below A's realized error wherever it changes the bound at all: the gallery maxima of part 0 for every
    part, the query norms of part 0 for every part, a part loop that stops after 32 parts.  A p in place of p_pad only
    shrinks the fp32-accumulation term, a few per cent of eps at most: these instances cannot show it."""
    case, op = _case(name, c, p, layout, part, other)
    p_pad = sbc.d_pad(p)
    terms = sbc.split_part_eps(op, p_pad)
    rest = np.delete(terms, part, axis=1)
    assert (rest <= 1e-3 * terms[:, part:part + 1]).all()
    r = sbc.split_realized(case, op)
    misread = {
        "g_max of part 0": dataclasses.replace(op, g_norm=np.repeat(op.g_norm[:1], c), g_res=np.repeat(op.g_res[:1], c)),
        "query norms of part 0": dataclasses.replace(op, qnh=np.repeat(op.qnh[:, :1], c, 1),
                                                     qnr=np.repeat(op.qnr[:, :1], c, 1), qnx=np.repeat(op.qnx[:, :1], c, 1)),
    }
    for what, bad in misread.items():
        e_bad = sbc.split_eps(bad, p_pad)
        assert (e_bad < 0.01 * r).all() if part > 0 else np.array_equal(e_bad, sbc.split_eps(op, p_pad)), what
    e_32 = terms[:, :32].max(axis=1)
    assert (e_32 < 0.01 * r).all() if part >= 32 else np.array_equal(e_32, terms.max(axis=1))


def test_many_query_instance():
    """The threshold-search instance with 3 scales x 43 query pairs, in part 33 of 197 and in the last part of 4: the
    bound still reaches every query, whatever its scale."""
    for c, p, part in ((197, 64, 33), (4, 516, 3)):
        case = sbc.split_case("range", p, c, part, scales=(1.0, 2.0, 0.5) * 43)
        op = sbc.split_operands(case.q, case.g, c)
        r, terms = sbc.split_realized(case, op), sbc.split_bf16_terms(op)[:, part]
        assert (r >= 0.9 * terms).all() and (r <= sbc.split_eps(op, sbc.d_pad(p))).all()


def test_second_half_moves_the_competitors_only():
    case = sbc.split_case("range", 64, 4, 1, "cross", 3, tie=True)
    moved = sbc.second_half(case)
    assert (np.concatenate(moved.comps) % 128 >= 64).all()
    assert np.array_equal(moved.target, case.target) and np.array_equal(moved.twin, case.twin)
    for i in range(case.q.shape[0]):
        assert np.array_equal(moved.g[moved.comps[i]], case.g[case.comps[i]])
    assert np.array_equal(np.sort(moved.g, axis=0), np.sort(case.g, axis=0))
