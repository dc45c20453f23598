"""GPU: dcr_sim_topk_split and dcr_sim_range_split on the split-score instances of tests/sim_bound_cases.py, whose bf16
error reaches the eps of split_row_bound in one descriptor part.  The instance sits in the first, second, last or 33rd
part, alone (quiet layout: eps comes from that part only) or with its competitors scoring in another part (cross).
Every output is compared with the fp64 oracle, indices equal and scores bitwise equal, and the top-k stage that decided
the queries is asserted from sim_topk_stats().  realized/eps (the target's emulated bf16 error over eps) is recorded per
case; the fp32 accumulation part of eps is not reached by these instances (their sums are exact)."""
import dataclasses
import functools

import numpy as np
import pytest
import torch

from dcr_b200 import dist as ddist
from dcr_b200 import similarity
from oracle import similarity as osim
from tests import sim_bound_cases as sbc
from tests.test_sim_range_split_cpu import split_range
from tests.test_sim_range_split_gpu import FakeWorld, Peer
from tests.test_sim_split_gpu import _rescore_every_row

pytestmark = pytest.mark.gpu


def _ratio(case):
    c, p = case.info["n_parts"], case.info["d"]
    op = sbc.split_operands(case.q, case.g, c)
    return op, float(np.min(sbc.split_realized(case, op) / sbc.split_eps(op, sbc.d_pad(p))))


def _topk(case, k, monkeypatch, block):
    if block:
        monkeypatch.setenv("DCR_B200_TUNING", "1")
        monkeypatch.setenv("DCR_SIM_RESCORE_BLOCK", "1")
    v, i = similarity.sim_topk_split(torch.from_numpy(case.q).cuda(), torch.from_numpy(case.g).cuda(), k,
                                     case.info["n_parts"])
    torch.cuda.synchronize()
    st = similarity.sim_topk_stats()
    monkeypatch.delenv("DCR_SIM_RESCORE_BLOCK", raising=False)
    monkeypatch.delenv("DCR_B200_TUNING", raising=False)
    return v.cpu().numpy(), i.cpu().numpy(), st


def _equal_oracle(q, g, c, k, v, i):
    ov, oi = osim.sim_topk_split(q, g, k, c)
    assert np.array_equal(i, oi), (i[:, :4], oi[:, :4])
    assert np.array_equal(v.view(np.uint32), ov.view(np.uint32))


def _label(c, p, layout, part, other):
    return f"C{c}-p{p}-{layout}{part}" + (f"-{other}" if other >= 0 else "")


# every TOPK_CASES instance at every placement of every shape; the warp- and block-form re-score on the quiet layout
TOPK = [(name, c, p, layout, part, other, block)
        for name, *_ in sbc.TOPK_CASES for c, p in sbc.SPLIT_SHAPES
        for layout, part, other in sbc.split_placements(c)
        for block in ((False, True) if layout == "quiet" else (False,))]


@functools.lru_cache(maxsize=1)
def _topk_case(name, c, p, layout, part, other):
    """The instance, its operands and realized/eps, shared by the warp and the block form."""
    case = sbc.split_case(name, p, c, part, layout, other)
    return (case, *_ratio(case))


@pytest.mark.parametrize("name,c,p,layout,part,other,block", TOPK,
                         ids=[f"{x[0]}-{_label(*x[1:6])}-{'block' if x[6] else 'warp'}" for x in TOPK])
def test_topk_stage_matrix(name, c, p, layout, part, other, block, monkeypatch, record_property):
    _, k, n_b, shared, tie, stage = next(x for x in sbc.TOPK_CASES if x[0] == name)
    case, op, ratio = _topk_case(name, c, p, layout, part, other)
    record_property("realized_over_eps", ratio)
    v, i, st = _topk(case, k, monkeypatch, block)
    _equal_oracle(case.q, case.g, c, k, v, i)
    rv, ri = _rescore_every_row(torch.from_numpy(case.q), torch.from_numpy(case.g), k, c)
    assert np.array_equal(i, ri) and np.array_equal(v.view(np.uint32), rv.view(np.uint32))
    nq = case.q.shape[0]
    assert st["kp"] == sbc.KP0[k]
    assert (i[:, 0] == case.target).all()
    if tie and k > 1:   # the exact tie: the lower index first, although its twin's bf16 score is eps above
        assert (i[:, 1] == case.twin).all()
    if stage == "first":
        assert st["n_second"] == 0 and st["n_flagged"] == 0, st
        ap = sbc.split_approx(op, c)
        for r in range(nq):   # the re-score inverted the bf16 order
            assert (ap[r, case.comps[r]] > ap[r, case.target[r]]).all()
    elif stage == "second":
        assert st["n_second"] == nq and st["n_flagged"] == 0, st
    else:
        assert st["n_second"] == (0 if k == 16 else nq) and st["n_flagged"] == nq, st


def _range_check(q, g, c, tau, res):
    off, idx, val = (x.cpu().numpy() for x in res)
    ooff, oidx, oval = split_range(q, g, c, tau)
    assert np.array_equal(off, ooff) and np.array_equal(idx, oidx)
    assert np.array_equal(val.view(np.uint32), oval.view(np.uint32))
    return off, idx


def _tau(case):
    """A's exact split score for query 0 as fp32 (query 1 meets the mirror instance at the same score)."""
    return float(np.float32(sbc.split_exact(case.q[:1], case.g, case.info["n_parts"])[0, case.target[0]]))


# the cross layout with the competitors in the other 64-column half of their tile than A: the running maxima of the two
# halves come from the two consumer warpgroups
RANGE = [(c, p, layout, part, other) for c, p in sbc.RANGE_SPLIT_SHAPES for layout, part, other in sbc.split_placements(c)]


@pytest.mark.parametrize("tie", [False, True], ids=["single", "tie"])
@pytest.mark.parametrize("c,p,layout,part,other", RANGE, ids=[_label(*x) for x in RANGE])
def test_range_reports_target_below_tau_in_bf16(c, p, layout, part, other, tie, record_property):
    """tau = A's fp32 split score: A is reported (inclusive) although its bf16 split score lies ~eps below tau; the
    competitors, whose bf16 split scores lie above tau and whose fp32 ones below it, are not.  The query tile stays
    resident up to d_pad = 512 (2 x 64, 4 x 64, 2 x 256) and is streamed beyond."""
    case = sbc.split_case("range", p, c, part, layout, other, tie=tie)
    if layout == "cross":
        case = sbc.second_half(case)
    op, ratio = _ratio(case)
    record_property("realized_over_eps", ratio)
    tau = _tau(case)
    ap = sbc.split_approx(op, c)
    assert ap[0, case.target[0]] < tau and (ap[0, case.comps[0]] >= tau).all()
    res = similarity.sim_range_split(torch.from_numpy(case.q).cuda(), torch.from_numpy(case.g).cuda(), tau, c)
    off, idx = _range_check(case.q, case.g, c, tau, res)
    for r in range(2):
        want = [case.target[r]] + ([case.twin[r]] if tie else [])
        assert idx[off[r]:off[r + 1]].tolist() == sorted(want)


@pytest.mark.parametrize("c,p,part", [(2, 256, 1), (197, 64, 33)], ids=["resident", "streamed"])
def test_range_many_queries_full_csr(c, p, part):
    """258 queries (pairs at scales 1, 2, 1/2) over 3 query tiles: the whole CSR equals the oracle's."""
    case = sbc.split_case("range", p, c, part, scales=(1.0, 2.0, 0.5) * 43)
    tau = _tau(case)
    res = similarity.sim_range_split(torch.from_numpy(case.q).cuda(), torch.from_numpy(case.g).cuda(), tau, c)
    off, idx = _range_check(case.q, case.g, c, tau, res)
    for r in range(0, case.q.shape[0], 6):   # scale 1: exactly A
        assert idx[off[r]:off[r + 1]].tolist() == [case.target[r]]


def _sharded_case(c, p, part):
    """Shard 0: A with 8 competitors beside it; shard 1: 20 more competitors, A's pair replaced by fillers.  Each shard
    is a +- gallery of its own, with the instance in part `part` (quiet layout), so each computes its own maxima."""
    a = sbc.build(p, 8, centred=False, seed=1)
    b = sbc.build(p, 20, centred=False, shared=True, seed=2)
    bg = b.g.copy()
    bg[b.target[0]] = a.g[300]
    bg[b.target[1]] = -a.g[300]
    s0 = sbc.split_embed(a, c, part)
    s1 = sbc.split_embed(dataclasses.replace(b, g=bg), c, part, seed=1)
    assert np.array_equal(s0.q, s1.q)
    return s0, s1


SHARDED = [(2, 64, 1), (4, 516, 3), (40, 64, 39), (197, 64, 33)]


@pytest.mark.parametrize("c,p,part", SHARDED, ids=[f"C{c}-p{p}-quiet{part}" for c, p, part in SHARDED])
def test_sharded_forms(c, p, part, record_property):
    s0, s1 = _sharded_case(c, p, part)
    record_property("realized_over_eps", _ratio(s0)[1])
    q = torch.from_numpy(s0.q).cuda()
    g0, g1 = torch.from_numpy(s0.g).cuda(), torch.from_numpy(s1.g).cuda()
    n0 = s0.g.shape[0]
    G = np.concatenate([s0.g, s1.g])
    # top-k: each shard on its own with its global index base, then the merge
    k = 10
    v0, i0 = similarity.sim_topk_split(q, g0, k, c)
    v1, i1 = similarity.sim_topk_split(q, g1, k, c, index_base=n0)
    v, i = similarity.topk_merge(torch.stack([v0, v1]), torch.stack([i0, i1]), k)
    torch.cuda.synchronize()
    v, i = v.cpu().numpy(), i.cpu().numpy()
    _equal_oracle(s0.q, G, c, k, v, i)
    assert (i[:, 0] == s0.target).all()
    # threshold search at A's fp32 score: A from this rank, nothing from the peer's competitors
    tau = _tau(s0)
    fake = FakeWorld(0, [Peer(q, g1, tau, c, n0, 1)])
    res = ddist.sharded_range(q, g0, tau, 0, allgather=fake, world=2, num_chunks=c)
    torch.cuda.synchronize()
    off, idx = _range_check(s0.q, G, c, tau, res)
    assert idx.tolist() == s0.target.tolist()
