"""Without a GPU: the cross split-score instances of tests/sim_bound_cases.py, the 258-query forms and the mixed-stage
instance of the aligned split score have the properties the GPU tests rely on.

- exactness: every fp32 partial sum of the tensor-core accumulation of every (query part, gallery part) pair, and every
  fp64 pair dot product;
- the inversion: A is the exact best (or tied with its twin at a higher index); every competitor's bf16 cross score is
  above A's while its fp32 cross score is below A's;
- the realized error: A's bf16 rounding costs at least 0.9 of its pair's bf16 terms, and no pair's error exceeds eps;
- pair and quiet layouts: every other pair's term is at most 1e-3 of the instance pair's, so a bound read from the
  aligned pairs only (split_row_bound's), or from another part's norms or maxima, falls below A's realized error.

It also restates cross_staged_parts and checks the staged-group shapes the GPU tests walk against the constant in
sim_sweep.cuh.
"""
import re
from pathlib import Path

import numpy as np
import pytest

from tests import sim_bound_cases as sbc

# shapes of the threshold search and of the top-k stage matrix
SHAPES = tuple(dict.fromkeys(sbc.CROSS_RANGE_SHAPES + ((2, 64),)))


def _names(c):
    # every kind of row at up to 8 parts; with 40 parts the tie and the threshold-search instances, and with 197 (a
    # 25 MB gallery, C^2 pairs) the threshold search's tie instance, which holds every kind of row the others do
    return ("k1_first", "k10_second", "k16_brute", "k10_shared", "k10_tie", "range", "range_tie") if c <= 8 \
        else ("k10_tie", "range", "range_tie") if c <= 40 else ("range_tie",)


CASES = [(name, c, p, layout, part, other) for c, p in SHAPES for name in _names(c)
         for layout, part, other in sbc.cross_placements(c)]


def _id(x):
    name, c, p, layout, part, other = x
    return f"{name}-C{c}-p{p}-{layout}{part}" + (f"-{other}" if other >= 0 else "")


def _case(name, c, p, layout, part, other, **kw):
    if name.startswith("range"):
        kw["tie"] = name == "range_tie"
        name = "range"
    case = sbc.cross_case(name, p, c, layout, part, other, **kw)
    return case, sbc.split_operands(case.q, case.g, c)


def _scores(case, op, c, p):
    """(fp64 exact, bf16 approximate, eps) of every pair, and the exactness of both: integers of at most 12 bits over
    at most 1024 terms make every fp64 pair product exact; the tensor-core accumulation of every pair has products on a
    2^-12 grid whose absolute sum stays below 2^24 of them."""
    qi, gi = sbc.as_integers(case.q, 0.5), sbc.as_integers(case.g, sbc.U)
    hq, hg = sbc.as_integers(op.qh, 0.5), sbc.as_integers(op.gh, sbc.U)
    assert max(np.abs(qi).max(), np.abs(gi).max(), np.abs(hq).max(), np.abs(hg).max()) < 2 ** 12 and p <= 1024
    assert sbc.cross_exact(np.abs(hq), np.abs(hg), c).max() < 2 ** 24
    return sbc.cross_exact(case.q, case.g, c), sbc.cross_approx(op, c), sbc.cross_eps(op, sbc.d_pad(p))


def _inverted(case, ex, ap, e):
    for i in range(case.q.shape[0]):
        a, comps, tw = case.target[i], case.comps[i], case.twin[i]
        others = np.setdiff1d(np.arange(case.g.shape[0]), [a, tw])
        assert (ex[i, others] < ex[i, a]).all()                                 # A is the exact best ...
        assert (ap[i, comps] > ap[i, a]).all()                                  # ... below every competitor in bf16
        if tw >= 0:                                                             # exact tie, higher index, better bf16
            assert ex[i, tw] == ex[i, a] and tw > a and ap[i, tw] - ap[i, a] > e[i]
        fillers = np.setdiff1d(others, comps)
        assert ex[i, fillers].max() < ex[i, a] - 4 * e[i]                       # fillers never compete
        # the fp32 scores keep the order: the threshold search at A's score sees the competitors below it
        assert (ex[i, comps].astype(np.float32) < np.float32(ex[i, a])).all()
        assert (ap[i, comps] >= np.float32(ex[i, a])).all()


def _bound(case, op, ex, ap, e):
    """A's realized error against its pair's bf16 term and eps; every pair's error within eps.  Returns it."""
    pa, pb = sbc.instance_pair(case)
    rows = np.arange(case.q.shape[0])
    r = ex[rows, case.target] - ap[rows, case.target].astype(np.float64)
    assert (r >= 0.9 * sbc.cross_bf16_terms(op)[:, pa, pb]).all()
    assert (r <= e).all()
    assert (np.abs(ex - ap) <= e[:, None]).all()
    return r


def _isolated(case, op, p, r):
    """Every other pair's term is at most 1e-3 of the instance pair's, which is the row's eps; the aligned pairs'
    largest term (split_row_bound's eps) lies below 1% of A's realized error when the instance pair is not aligned."""
    terms = sbc.cross_part_eps(op, sbc.d_pad(p))
    pa, pb = sbc.instance_pair(case)
    inst = terms[:, pa, pb]
    rest = terms.copy()
    rest[:, pa, pb] = 0
    assert (rest.max(axis=(1, 2)) <= 1e-3 * inst).all()
    assert np.array_equal(inst, sbc.cross_eps(op, sbc.d_pad(p)))
    aligned = sbc.split_eps(op, sbc.d_pad(p))
    assert (aligned < 0.01 * r).all() if pa != pb else np.array_equal(aligned, inst)


@pytest.mark.parametrize("name,c,p,layout,part,other", CASES, ids=[_id(x) for x in CASES])
def test_cross_instance(name, c, p, layout, part, other):
    case, op = _case(name, c, p, layout, part, other)
    ex, ap, e = _scores(case, op, c, p)
    _inverted(case, ex, ap, e)
    r = _bound(case, op, ex, ap, e)
    if layout in ("pair", "quiet"):
        _isolated(case, op, p, r)


# the 258-query forms the GPU tests run under the cross score: the stage matrix's instances and the full CSR's
MANY = [(name, c, p, "pair", a, b) for c, p, a, b in sbc.CROSS_PLACES[:3]
        for name in (("k1_first", "k1_second", "k1_brute", "k10_first", "k10_second", "k10_brute") if c <= 4 else ("k10_second",))] \
    + [("range", 2, 256, "pair", 0, 1), ("range", 40, 64, "pair", 33, 1)]


@pytest.mark.parametrize("name,c,p,layout,part,other", MANY, ids=[_id(x) for x in MANY])
def test_many_query_forms(name, c, p, layout, part, other):
    """The scaled queries keep every property, and every query's scores and eps are its scale times those of the
    2-query instance: the powers of two change no rounding."""
    case, op = _case(name, c, p, layout, part, other, scales=sbc.MANY_SCALES)
    base, bop = _case(name, c, p, layout, part, other)
    assert case.q.shape[0] == 258 and np.array_equal(case.g, base.g)
    s = np.repeat(np.array(sbc.MANY_SCALES, np.float32), 2)
    assert np.array_equal(case.q, base.q[np.arange(258) % 2] * s[:, None])
    ex, ap, e = _scores(case, op, c, p)
    _inverted(case, ex, ap, e)
    bex, bap = sbc.cross_exact(base.q, base.g, c), sbc.cross_approx(bop, c)
    be = sbc.cross_eps(bop, sbc.d_pad(p))
    j = np.arange(258) % 2
    assert np.array_equal(ex, bex[j] * s[:, None]) and np.array_equal(ap, bap[j] * s[:, None])
    np.testing.assert_allclose(e, be[j] * s, rtol=1e-6)
    _isolated(case, op, p, _bound(case, op, ex, ap, e))


@pytest.mark.parametrize("k", [1, 10])
@pytest.mark.parametrize("c,p,parts,nan_part", sbc.MIXED_PLACES, ids=[f"C{x[0]}-p{x[1]}" for x in sbc.MIXED_PLACES])
def test_mixed_instance_takes_eps_from_each_querys_part(c, p, parts, nan_part, k):
    """The aligned split score on the three-part mix: each query's part holds the row's eps (every other part's term is at
    most 1e-3 of it), the bound is reached there, and the bf16 order inverts the exact order for every query."""
    case = sbc.mixed_case(k, p, c, parts)
    op = sbc.split_operands(case.q, case.g, c)
    types = case.info["types"]
    assert case.q.shape[0] == 258 and np.array_equal(np.bincount(types), [86, 86, 86])
    assert [sbc.stage_of(n) for n in sbc.MIXED[k]] == ["first", "second", "brute"]
    own = np.array(parts)[types]
    rows = np.arange(258)
    terms = sbc.split_part_eps(op, sbc.d_pad(p))
    e = sbc.split_eps(op, sbc.d_pad(p))
    assert np.array_equal(terms[rows, own], e)
    rest = terms.copy()
    rest[rows, own] = 0
    assert (rest.max(axis=1) <= 1e-3 * e).all()
    r = sbc.split_realized(case, op)
    assert (r >= 0.9 * sbc.split_bf16_terms(op)[rows, own]).all() and (r <= e).all()
    ex, ap = sbc.split_exact(case.q, case.g, c), sbc.split_approx(op, c)
    assert (np.abs(ex - ap) <= e[:, None]).all()
    for i in rows:
        a, comps = case.target[i], case.comps[i]
        assert (np.delete(ex[i], a) < ex[i, a]).all() and (ap[i, comps] > ap[i, a]).all()
    # the NaN part is a zero part of every query
    assert nan_part not in parts
    nanned = sbc.with_nan(case, sbc.nan_rows(258), nan_part)
    assert np.isnan(nanned.q).sum() == sbc.nan_rows(258).size


def test_nan_rows():
    rows = sbc.nan_rows(258)
    assert rows.size == 40 and {0, 7, 252, 127, 128, 257} <= set(rows.tolist())
    assert (rows < 128).sum() >= 1 and ((rows >= 128) & (rows < 256)).sum() >= 1 and (rows >= 256).sum() >= 1
    assert sbc.nan_rows(40).tolist() == [0, 7, 14, 21, 28, 35, 39]


def test_cross_staged_parts_restates_the_kernel():
    """The Python restatement uses the header's constant and formula, and every staged-group shape has the groups it
    was chosen for: one group of 78 and a remainder of 1, two full groups, three with a remainder of 41, and at the
    longest parts 2 + 1, 1 + 1 and 1 + 1 + 1."""
    src = (Path(__file__).resolve().parent.parent / "dcr_b200" / "csrc" / "sim_sweep.cuh").read_text()
    m = re.search(r"constexpr size_t kCrossStageBytes = (\d+) \* 1024;", src)
    assert m and int(m.group(1)) * 1024 == sbc.CROSS_STAGE_BYTES
    assert "const size_t per_part = (static_cast<size_t>(pl) + 8) * sizeof(double);" in src
    for (c, p), groups in sbc.STAGED_SHAPES.items():
        assert sbc.cross_groups(c, p) == groups, (c, p)
    assert sbc.cross_staged_parts(197, 2808) == 2 and sbc.cross_staged_parts(197, 2812) == 1
    assert sbc.cross_staged_parts(3, 2804) == 2 and sbc.cross_staged_parts(1, 8192) == 1
