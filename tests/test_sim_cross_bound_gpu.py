"""GPU: dcr_sim_range_cross on the cross split-score instances of tests/sim_bound_cases.py, whose winning pair's bf16
error reaches the eps of cross_row_bound; the sharded top-k merge on such an instance; and the cross re-score's staged
groups (cross_exact_scores stages the query cross_staged_parts parts at a time) in the top-k and the threshold search.
Every CSR is compared bit for bit with the dense fp64 oracle; realized/eps (the target's emulated bf16 error over eps)
is recorded per bound case."""
import numpy as np
import pytest
import torch

from dcr_b200 import similarity, synthetic
from tests import sim_bound_cases as sbc
from tests.test_sim_cross_cpu import cross_range, cross_topk
from tests.test_sim_cross_gpu import _rescore_cross

pytestmark = pytest.mark.gpu


def _ratio(case, op):
    p = case.info["p"]
    return float(np.min(sbc.cross_realized(case, op) / sbc.cross_eps(op, sbc.d_pad(p))))


def _tau(case):
    """A's exact cross score for query 0 as fp32 (query 1 meets the mirror instance at the same score)."""
    return float(np.float32(sbc.cross_exact(case.q[:1], case.g, case.info["n_parts"])[0, case.target[0]]))


def _range(q, g, tau, c):
    res = similarity.sim_range_split(torch.from_numpy(q).cuda(), torch.from_numpy(g).cuda(), tau, c, cross=True)
    return tuple(x.cpu().numpy() for x in res)


def _range_check(q, g, c, tau, got):
    off, idx, val = got
    ooff, oidx, oval = cross_range(q, g, c, tau)
    assert np.array_equal(off, ooff) and np.array_equal(idx, oidx)
    assert np.array_equal(val.view(np.uint32), oval.view(np.uint32))
    return off, idx


def _label(c, p, layout, part, other):
    return f"C{c}-p{p}-{layout}{part}" + (f"-{other}" if other >= 0 else "")


# every pair and split layout of every shape; resident query tile up to d_pad = 512, streamed beyond
RANGE = [(c, p, layout, part, other) for c, p in sbc.CROSS_RANGE_SHAPES for layout, part, other in sbc.cross_placements(c)]


@pytest.mark.parametrize("tie", [False, True], ids=["single", "tie"])
@pytest.mark.parametrize("c,p,layout,part,other", RANGE, ids=[_label(*x) for x in RANGE])
def test_range_reports_target_below_tau_in_bf16(c, p, layout, part, other, tie, record_property):
    """tau = A's fp32 cross score: A (and its twin) are reported, inclusive, although A's bf16 cross score lies ~eps
    below tau; the competitors, whose bf16 scores lie above tau and whose fp32 ones below it, are not.  Where A and its
    competitors score in different parts, the competitors sit in the other 64-column half of their tile."""
    case = sbc.cross_case("range", p, c, layout, part, other, tie=tie)
    if layout != "quiet":
        case = sbc.second_half(case)
    op = sbc.split_operands(case.q, case.g, c)
    record_property("realized_over_eps", _ratio(case, op))
    tau = _tau(case)
    ap = sbc.cross_approx(op, c)
    assert ap[0, case.target[0]] < tau and (ap[0, case.comps[0]] >= tau).all()
    off, idx = _range_check(case.q, case.g, c, tau, _range(case.q, case.g, tau, c))
    for r in range(2):
        want = [case.target[r]] + ([case.twin[r]] if tie else [])
        assert idx[off[r]:off[r + 1]].tolist() == sorted(want)


@pytest.mark.parametrize("c,p,a,b", [(2, 256, 0, 1), (40, 64, 33, 1)], ids=["resident", "streamed"])
def test_range_many_queries_full_csr(c, p, a, b, record_property):
    """258 queries (pairs at scales 1, 2, 1/2) over 3 query tiles: the whole CSR equals the oracle's."""
    case = sbc.cross_embed(sbc.build(p, 20, centred=False, scales=sbc.MANY_SCALES), c, a, b)
    record_property("realized_over_eps", _ratio(case, sbc.split_operands(case.q, case.g, c)))
    tau = _tau(case)
    off, idx = _range_check(case.q, case.g, c, tau, _range(case.q, case.g, tau, c))
    for r in range(0, case.q.shape[0], 6):   # scale 1: exactly A
        assert idx[off[r]:off[r + 1]].tolist() == [case.target[r]]


def _sharded_case(c, p, a, b):
    """Shard 0: A with 8 competitors beside it; shard 1: 20 more competitors, A's pair replaced by fillers.  Each shard
    is a +- gallery of its own with the instance in the pair (a, b), so each computes its own maxima."""
    s0 = sbc.build(p, 8, centred=False, seed=1)
    s1 = sbc.build(p, 20, centred=False, shared=True, seed=2)
    g1 = s1.g.copy()
    g1[s1.target[0]] = s0.g[300]
    g1[s1.target[1]] = -s0.g[300]
    s1.g = g1
    e0, e1 = sbc.cross_embed(s0, c, a, b), sbc.cross_embed(s1, c, a, b, seed=1)
    assert np.array_equal(e0.q, e1.q)
    return e0, e1


@pytest.mark.parametrize("c,p,a,b", sbc.CROSS_PLACES, ids=[f"C{x[0]}-p{x[1]}-q{x[2]}g{x[3]}" for x in sbc.CROSS_PLACES])
def test_sharded_topk_merge(c, p, a, b, record_property):
    """Each shard's top-k with its global index base, then topk_merge: the fp64 ranking of the whole gallery."""
    s0, s1 = _sharded_case(c, p, a, b)
    record_property("realized_over_eps", _ratio(s0, sbc.split_operands(s0.q, s0.g, c)))
    q = torch.from_numpy(s0.q).cuda()
    n0 = s0.g.shape[0]
    k = 10
    v0, i0 = similarity.sim_topk_split(q, torch.from_numpy(s0.g).cuda(), k, c, cross=True)
    v1, i1 = similarity.sim_topk_split(q, torch.from_numpy(s1.g).cuda(), k, c, cross=True, index_base=n0)
    v, i = similarity.topk_merge(torch.stack([v0, v1]), torch.stack([i0, i1]), k)
    torch.cuda.synchronize()
    v, i = v.cpu().numpy(), i.cpu().numpy()
    ov, oi = cross_topk(s0.q, np.concatenate([s0.g, s1.g]), k, c)
    assert np.array_equal(i, oi) and np.array_equal(v.view(np.uint32), ov.view(np.uint32))
    assert (i[:, 0] == s0.target).all()


# ------------------------------------------------------------------------------------------------------------------
# the staged groups of the cross re-score

STAGED = list(sbc.STAGED_SHAPES)


@pytest.mark.parametrize("c,p", STAGED, ids=[f"C{c}-p{p}-" + "+".join(map(str, sbc.STAGED_SHAPES[(c, p)])) for c, p in STAGED])
def test_staged_groups(c, p):
    """Random planted descriptors whose last query part is scaled by 4, so that every query's best pairs lie in the last
    staged group; the top-k and the threshold search at the 10th best cross score equal the dense oracle and
    dcr_split_rescore(cross = 1), which stages one part at a time, bit for bit."""
    assert sbc.cross_groups(c, p) == sbc.STAGED_SHAPES[(c, p)]
    nq, ng = (4, 600) if c > 3 else (8, 1000)
    q, g = synthetic.descriptors(nq, ng, c * p, seed=c + p, planted=0.05)
    q, g = q.numpy(), g.numpy()
    q[:, (c - 1) * p:] *= 4
    last = sum(sbc.STAGED_SHAPES[(c, p)][:-1])   # first query part of the last group
    k = 10
    ov, oi = cross_topk(q, g, k, c)
    # the winning query part of every reported pair lies in the last group
    q64, g64 = q.astype(np.float64).reshape(nq, c, p), g.astype(np.float64).reshape(ng, c, p)
    for r in range(nq):
        pairs = np.einsum("ap,jbp->jab", q64[r], g64[oi[r]]).reshape(k, -1)
        assert (pairs.argmax(axis=1) // c >= last).all()
    # top-k
    v, i = similarity.sim_topk_split(torch.from_numpy(q).cuda(), torch.from_numpy(g).cuda(), k, c, cross=True)
    v, i = v.cpu().numpy(), i.cpu().numpy()
    assert np.array_equal(i, oi) and np.array_equal(v.view(np.uint32), ov.view(np.uint32))
    rv, ri = _rescore_cross(torch.from_numpy(q), torch.from_numpy(g), 16, c, np.tile(np.arange(ng), (nq, 1)))
    assert np.array_equal(ri[:, :k], i) and np.array_equal(rv[:, :k].view(np.uint32), v.view(np.uint32))
    # threshold search at query 0's 10th best score
    tau = float(ov[0, -1])
    off, idx, val = _range(q, g, tau, c)
    _range_check(q, g, c, tau, (off, idx, val))
    for r in range(nq):   # the re-score's best 16 at or above tau are reported with their bits, and no other pair when
        keep = rv[r] >= np.float32(tau)   # the 16th lies below tau
        want = set(zip(ri[r][keep].tolist(), rv[r][keep].view(np.uint32).tolist()))
        got = set(zip(idx[off[r]:off[r + 1]].tolist(), val[off[r]:off[r + 1]].view(np.uint32).tolist()))
        assert want <= got and (keep[-1] or want == got)
    assert not (rv[0] >= np.float32(tau))[-1]
