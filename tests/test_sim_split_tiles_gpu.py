"""GPU: both split scores at production query counts.  dcr_sim_topk_split and dcr_sim_topk_cross on 258 queries (query
tiles of 128 + 128 + 2) of the bound instances of tests/sim_bound_cases.py, every query decided by a known stage: the
first pass, the second-chance pass on a flagged subset that is no prefix and spans every query tile, or the brute-force
path over several batches.  Every case is checked three ways: indices and score bits of the fp64 oracle, the bits of
dcr_split_rescore with every gallery row as a candidate, and the stage counts of sim_topk_stats() exactly.  Also: a
query's answer does not depend on the batch it is in, and the longest parts (p = 4096 and 8192) with the brute-force
path at its smallest batch."""
import numpy as np
import pytest
import torch

from dcr_b200 import _lib, similarity, synthetic
from oracle import similarity as osim
from tests import sim_bound_cases as sbc
from tests.test_sim_cross_cpu import cross_topk
from tests.test_sim_range_split_cpu import split_range

pytestmark = pytest.mark.gpu


def _topk(q, g, k, c, cross, block, monkeypatch):
    if block:
        monkeypatch.setenv("DCR_B200_TUNING", "1")
        monkeypatch.setenv("DCR_SIM_RESCORE_BLOCK", "1")
    v, i = similarity.sim_topk_split(torch.from_numpy(q).cuda(), torch.from_numpy(g).cuda(), k, c, cross=cross)
    torch.cuda.synchronize()
    st = similarity.sim_topk_stats()
    monkeypatch.delenv("DCR_SIM_RESCORE_BLOCK", raising=False)
    monkeypatch.delenv("DCR_B200_TUNING", raising=False)
    return v.cpu().numpy(), i.cpu().numpy(), st


def _split_topk(q, g, k, c):
    """The fp64 split-score top-k with fmax over the parts (a NaN part is ignored), ties to the lowest row."""
    nq, d = q.shape
    p = d // c
    q64, g64 = q.astype(np.float64).reshape(nq, c, p), g.astype(np.float64).reshape(g.shape[0], c, p)
    s = np.full((nq, g.shape[0]), -np.inf)
    for part in range(c):
        s = np.fmax(s, q64[:, part] @ g64[:, part].T)
    idx = np.stack([osim._rank_row(row, k) for row in s])
    return np.take_along_axis(s, idx, axis=1).astype(np.float32), idx


def _rescore_every_row(q, g, k, c, cross):
    """dcr_split_rescore with every gallery row as a candidate: the exact score of every pair, then the top-k."""
    lib = _lib.load()
    qd, gd = torch.from_numpy(q).cuda(), torch.from_numpy(g).cuda()
    nq, d = qd.shape
    ng = gd.shape[0]
    cand = torch.arange(ng, dtype=torch.int64, device="cuda").repeat(nq, 1).contiguous()
    out_s = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    out_i = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    rc = lib.dcr_split_rescore(qd.data_ptr(), gd.data_ptr(), nq, d, c, int(cross), cand.data_ptr(), ng, k,
                               out_s.data_ptr(), out_i.data_ptr(), torch.cuda.current_stream().cuda_stream)
    _lib.check(rc, "dcr_split_rescore")
    torch.cuda.synchronize()
    return out_s.cpu().numpy(), out_i.cpu().numpy()


def _check(q, g, k, c, cross, block, monkeypatch):
    """The search's indices and bits equal the fp64 oracle's and dcr_split_rescore's over every row (ng <= 4096)."""
    v, i, st = _topk(q, g, k, c, cross, block, monkeypatch)
    ov, oi = cross_topk(q, g, k, c) if cross else _split_topk(q, g, k, c)
    bad = np.nonzero((i != oi).any(axis=1))[0]
    assert bad.size == 0, f"{bad.size} query rows differ, first {bad[:5]}: got {i[bad[:3]]} want {oi[bad[:3]]}"
    assert np.array_equal(v.view(np.uint32), ov.view(np.uint32))
    assert g.shape[0] <= 4096
    rv, ri = _rescore_every_row(q, g, k, c, cross)
    assert np.array_equal(i, ri) and np.array_equal(v.view(np.uint32), rv.view(np.uint32))
    return v, i, st


def _expect(st, k, n_second, n_flagged):
    assert st["kp"] == sbc.KP0[k]
    assert st["n_second"] == n_second and st["n_flagged"] == n_flagged, (st["n_second"], st["n_flagged"], n_second, n_flagged)


# (score, C, p, part, other): aligned in part `part` (quiet layout), or cross in the pair (part, other).  3 query tiles x
# 4 gallery tiles = 12 work units, one gallery tile each, as with the 2-query instances: the stages are theirs.
SHAPES = [("aligned", 2, 64, 1, -1), ("aligned", 4, 516, 3, -1), ("aligned", 40, 64, 33, -1),
          ("cross", 2, 64, 0, 1), ("cross", 4, 516, 3, 0), ("cross", 40, 64, 33, 1)]
NAMES = ("k1_first", "k1_second", "k1_brute", "k10_first", "k10_second", "k10_brute")
MATRIX = [(name, *s, block) for s in SHAPES for name in NAMES for block in ((False, True) if s[0] == "aligned" else (False,))]


def _many(name, score, c, p, part, other):
    if score == "aligned":
        return sbc.split_case(name, p, c, part, scales=sbc.MANY_SCALES)
    return sbc.cross_embed(sbc.topk_case(name, p, False, scales=sbc.MANY_SCALES), c, part, other)


@pytest.mark.parametrize("name,score,c,p,part,other,block", MATRIX,
                         ids=[f"{x[0]}-{x[1]}-C{x[2]}-p{x[3]}-{x[4]}" + (f"-{x[5]}" if x[5] >= 0 else "")
                              + ("-block" if x[6] else "") for x in MATRIX])
def test_stage_matrix_258_queries(name, score, c, p, part, other, block, monkeypatch):
    _, k, _, _, _, stage = next(x for x in sbc.TOPK_CASES if x[0] == name)
    case = _many(name, score, c, p, part, other)
    nq = case.q.shape[0]
    assert nq == 258
    v, i, st = _check(case.q, case.g, k, c, score == "cross", block, monkeypatch)
    assert (i[:, 0] == case.target).all()
    _expect(st, k, 0 if stage == "first" else nq, nq if stage == "brute" else 0)


# mixed stages in one call: the aligned three-part mix, alone and with NaN rows; under the cross score every query part
# meets every gallery part, so NaN rows mix the stages instead
MIXED = ([("aligned", k, c, p, parts, nan_part, nan) for c, p, parts, nan_part in sbc.MIXED_PLACES for k in (1, 10)
          for nan in (False, True)]
         + [("cross", name, c, p, (a, b), (a + 1) % c, True) for c, p, a, b in (sbc.CROSS_PLACES[0], sbc.CROSS_PLACES[2])
            for name in ("k1_first", "k10_first", "k1_second", "k10_second")])


def _mixed_case(score, what, c, p, parts, nan_part, nan):
    """The case, and the rows the second pass and the brute-force path must see."""
    if score == "aligned":
        case = sbc.mixed_case(what, p, c, parts)
        stages = np.array(case.info["stages"])
    else:
        case = sbc.cross_embed(sbc.topk_case(what, p, False, scales=sbc.MANY_SCALES), c, *parts)
        stages = np.array([sbc.stage_of(what)] * case.q.shape[0])
    second, brute = set(np.nonzero(stages != "first")[0].tolist()), set(np.nonzero(stages == "brute")[0].tolist())
    if nan:
        rows = sbc.nan_rows(case.q.shape[0])
        case = sbc.with_nan(case, rows, nan_part)
        second |= set(rows.tolist())
        brute |= set(rows.tolist())
    return case, len(second), len(brute)


def _mixed_id(x):
    score, what, c, p, parts, nan_part, nan = x[:7]
    return f"{score}-{'k' + str(what) if score == 'aligned' else what}-C{c}-p{p}" + ("-nan" if nan else "") \
        + ("-block" if x[7:] and x[7] else "")


# the aligned form with the warp and the block re-score; the cross score always takes the block form
MIXED_FORMS = [(*x, block) for x in MIXED for block in ((False, True) if x[0] == "aligned" else (False,))]


@pytest.mark.parametrize("score,what,c,p,parts,nan_part,nan,block", MIXED_FORMS, ids=[_mixed_id(x) for x in MIXED_FORMS])
def test_mixed_stages_in_one_call(score, what, c, p, parts, nan_part, nan, block, monkeypatch):
    """The second-chance pass runs on a flagged subset spread over the three query tiles (qmap, thr_next), and the
    brute-force path over at least 33 queries: two batches or more."""
    case, n_second, n_flagged = _mixed_case(score, what, c, p, parts, nan_part, nan)
    k = what if score == "aligned" else int(what[1:what.index("_")])
    v, i, st = _check(case.q, case.g, k, c, score == "cross", block, monkeypatch)
    assert (i[:, 0] == case.target).all()
    assert n_flagged >= 33
    _expect(st, k, n_second, n_flagged)


@pytest.mark.parametrize("score,what,c,p,parts,nan_part,nan", [x for x in MIXED if x[-1]],
                         ids=[_mixed_id(x) for x in MIXED if x[-1]])
def test_answer_does_not_depend_on_the_batch(score, what, c, p, parts, nan_part, nan, monkeypatch):
    """The 258 queries reversed, then rows 130 and up alone: other query tiles, other flagged subsets, other brute-force
    batches; every row gets the indices and bits of the full run."""
    case, _, _ = _mixed_case(score, what, c, p, parts, nan_part, nan)
    k = what if score == "aligned" else int(what[1:what.index("_")])
    cross = score == "cross"
    v, i, _ = _topk(case.q, case.g, k, c, cross, False, monkeypatch)
    rv, ri, _ = _topk(np.ascontiguousarray(case.q[::-1]), case.g, k, c, cross, False, monkeypatch)
    assert np.array_equal(ri[::-1], i) and np.array_equal(rv[::-1].view(np.uint32), v.view(np.uint32))
    sv, si, st = _topk(np.ascontiguousarray(case.q[130:]), case.g, k, c, cross, False, monkeypatch)
    assert np.array_equal(si, i[130:]) and np.array_equal(sv.view(np.uint32), v[130:].view(np.uint32))


# the longest parts: the brute-force path at 12 (p = 4096) and 6 (p = 8192) queries per batch
LONG = [(score, c, p) for score in ("aligned", "cross") for c, p in ((2, 4096), (3, 8192))]


def _long_case(c, p):
    q, g = synthetic.descriptors(40, 1000, c * p, seed=c + p, planted=0.05)
    q, g = q.numpy(), g.numpy()
    rows = np.arange(0, 40, 2)   # 20 NaN rows: 2 batches of 12, 4 of 6
    q[rows, (c - 1) * p + 5] = np.nan
    return q, g, rows


@pytest.mark.parametrize("score,c,p", LONG, ids=[f"{s}-C{c}-p{p}" for s, c, p in LONG])
def test_longest_parts(score, c, p, monkeypatch):
    q, g, rows = _long_case(c, p)
    v, i, st = _check(q, g, 10, c, score == "cross", False, monkeypatch)
    assert st["n_flagged"] >= rows.size, st
    assert np.isfinite(v).all()


@pytest.mark.parametrize("c,p", [(2, 4096), (3, 8192)])
def test_longest_parts_range(c, p):
    """The aligned threshold search at the same shapes, tau at the 10th best split score of a query without NaN."""
    q, g, _ = _long_case(c, p)
    ov, _ = _split_topk(q, g, 10, c)
    tau = float(ov[1, -1])
    off, idx, val = (x.cpu().numpy() for x in similarity.sim_range_split(torch.from_numpy(q).cuda(),
                                                                         torch.from_numpy(g).cuda(), tau, c))
    ooff, oidx, oval = split_range(q, g, c, tau)
    assert np.array_equal(off, ooff) and np.array_equal(idx, oidx)
    assert np.array_equal(val.view(np.uint32), oval.view(np.uint32))
    assert off[2] - off[1] >= 10
