"""GPU: dcr_sim_topk and dcr_sim_range on the instances of tests/sim_bound_cases.py, whose bf16 error reaches the eps of
row_bound.  Every output row is compared with the fp64 oracle, indices equal and scores bitwise equal, and the stage
that decided the queries is asserted from sim_topk_stats().  realized/eps (the target's emulated bf16 error over eps) is
recorded per case; the fp32 accumulation part of eps is not reached by these instances (their sums are exact)."""
import numpy as np
import pytest
import torch

from dcr_b200 import dist as ddist
from dcr_b200 import similarity
from oracle import similarity as osim
from tests import sim_bound_cases as sbc
from tests import sim_range_oracle as orange
from tests.test_sim_range_sharded_gpu import FakeWorld, Peer

pytestmark = pytest.mark.gpu


def _ratio(case, d):
    op = sbc.operands(case.q, case.g)
    return op, float(np.min(sbc.realized(case, op) / sbc.eps(op, d)))


def _topk(case, k, monkeypatch, block):
    if block:
        monkeypatch.setenv("DCR_B200_TUNING", "1")
        monkeypatch.setenv("DCR_SIM_RESCORE_BLOCK", "1")
    v, i = similarity.sim_topk(torch.from_numpy(case.q).cuda(), torch.from_numpy(case.g).cuda(), k)
    torch.cuda.synchronize()
    st = similarity.sim_topk_stats()
    monkeypatch.delenv("DCR_SIM_RESCORE_BLOCK", raising=False)
    monkeypatch.delenv("DCR_B200_TUNING", raising=False)
    return v.cpu().numpy(), i.cpu().numpy(), st


def _equal_oracle(case, k, v, i):
    ov, oi = osim.sim_topk(case.q, case.g, k)
    assert np.array_equal(i, oi), (i[:, :4], oi[:, :4])
    assert np.array_equal(v.view(np.uint32), ov.view(np.uint32))


@pytest.mark.parametrize("block", [False, True], ids=["warp", "block"])
@pytest.mark.parametrize("centred", [False, True], ids=["plain", "centred"])
@pytest.mark.parametrize("d", sbc.DIMS)
@pytest.mark.parametrize("name", [c[0] for c in sbc.TOPK_CASES])
def test_topk_stage_matrix(name, d, centred, block, monkeypatch, record_property):
    _, k, n_b, shared, tie, stage = next(c for c in sbc.TOPK_CASES if c[0] == name)
    case = sbc.topk_case(name, d, centred)
    op, ratio = _ratio(case, d)
    assert op.flag == centred
    record_property("realized_over_eps", ratio)
    v, i, st = _topk(case, k, monkeypatch, block)
    _equal_oracle(case, k, v, i)
    nq = case.q.shape[0]
    assert st["kp"] == sbc.KP0[k]
    assert (i[:, 0] == case.target).all()
    if tie and k > 1:   # the exact tie: the lower index first, although its twin's bf16 score is eps above
        assert (i[:, 1] == case.twin).all()
    if stage == "first":
        assert st["n_second"] == 0 and st["n_flagged"] == 0, st
        ap = sbc.approx(op)
        for r in range(nq):   # the re-score inverted the bf16 order
            assert (ap[r, case.comps[r]] > ap[r, case.target[r]]).all()
    elif stage == "second":
        assert st["n_second"] == nq and st["n_flagged"] == 0, st
    else:
        assert st["n_second"] == (0 if k == 16 else nq) and st["n_flagged"] == nq, st


def _range_check(case, tau, res):
    off, idx, val = (x.cpu().numpy() for x in res)
    ooff, oidx, oval = orange.sim_range(case.q, case.g, tau)
    assert np.array_equal(off, ooff) and np.array_equal(idx, oidx)
    assert np.array_equal(val.view(np.uint32), oval.view(np.uint32))
    return off, idx


@pytest.mark.parametrize("tie", [False, True], ids=["single", "tie"])
@pytest.mark.parametrize("centred", [False, True], ids=["plain", "centred"])
@pytest.mark.parametrize("d", sbc.DIMS)
def test_range_reports_target_below_tau_in_bf16(d, centred, tie, record_property):
    """tau = A's fp32 score: A is reported (inclusive) although its bf16 score lies ~eps below tau; the competitors,
    whose bf16 scores lie above tau and whose fp32 scores below it, are not."""
    case = sbc.build(d, 20, centred=centred, tie=tie)
    op, ratio = _ratio(case, d)
    record_property("realized_over_eps", ratio)
    tau = float(np.float32(sbc.exact(case.q[:1], case.g)[0, case.target[0]]))
    ap = sbc.approx(op)
    assert ap[0, case.target[0]] < tau and (ap[0, case.comps[0]] >= tau).all()
    res = similarity.sim_range(torch.from_numpy(case.q).cuda(), torch.from_numpy(case.g).cuda(), tau)
    off, idx = _range_check(case, tau, res)
    want = [case.target[0]] + ([case.twin[0]] if tie else [])
    assert idx[off[0]:off[1]].tolist() == sorted(want)
    assert idx[off[1]:off[2]].tolist() == sorted(case.target[1:2].tolist() + ([case.twin[1]] if tie else []))


@pytest.mark.parametrize("centred", [False, True], ids=["plain", "centred"])
@pytest.mark.parametrize("d", [512, 4096])
def test_range_many_queries_full_csr(d, centred):
    """258 queries (pairs at scales 1, 2, 1/2) over 3 query tiles: the whole CSR equals the oracle's."""
    case = sbc.build(d, 20, centred=centred, scales=(1.0, 2.0, 0.5) * 43)
    tau = float(np.float32(sbc.exact(case.q[:1], case.g)[0, case.target[0]]))
    res = similarity.sim_range(torch.from_numpy(case.q).cuda(), torch.from_numpy(case.g).cuda(), tau)
    off, idx = _range_check(case, tau, res)
    for r in range(0, case.q.shape[0], 6):   # scale 1: exactly A
        assert idx[off[r]:off[r + 1]].tolist() == [case.target[r]]


def _sharded_case(d, centred):
    """Shard 0: A with 8 competitors beside it; shard 1: 20 more competitors.  Each shard is a +- gallery of its own."""
    a = sbc.build(d, 8, centred=centred, seed=1)
    b = sbc.build(d, 20, centred=centred, shared=True, seed=2)
    n_x = a.g.shape[0] // 2
    # drop b's target pair so that shard 1 holds competitors and fillers only
    bg = b.g.copy()
    bg[b.target[0]] = a.g[300]
    bg[b.target[1]] = -a.g[300]
    return a, bg, n_x


@pytest.mark.parametrize("centred", [False, True], ids=["plain", "centred"])
@pytest.mark.parametrize("d", [64, 1024])
def test_sharded_forms(d, centred):
    a, bg, _ = _sharded_case(d, centred)
    q = torch.from_numpy(a.q).cuda()
    s0, s1 = torch.from_numpy(a.g).cuda(), torch.from_numpy(bg).cuda()
    G = np.concatenate([a.g, bg])
    full = sbc.Case(q=a.q, g=G, centred=centred, target=a.target, comps=a.comps, twin=a.twin)
    # top-k: this rank holds A's shard, the emulated peer the competitors' shard
    k = 10
    v1, i1 = similarity.sim_topk(q, s1, k, index_base=a.g.shape[0])
    peer = torch.cat([v1.contiguous().view(torch.uint8).reshape(-1), i1.contiguous().view(torch.uint8).reshape(-1)])

    def fake_allgather(send, recv, nbytes, stream):
        own = ddist.device_bytes(send, nbytes, q.device)
        out = ddist.device_bytes(recv, 2 * nbytes, q.device)
        out[:nbytes].copy_(own)
        out[nbytes:].copy_(peer)
        return 0

    v, i = ddist.sharded_topk_c(q, s0, k, 0, allgather=fake_allgather, world=2)
    torch.cuda.synchronize()
    v, i = v.cpu().numpy(), i.cpu().numpy()
    _equal_oracle(full, k, v, i)
    assert (i[:, 0] == a.target).all()
    # threshold search at A's fp32 score: A from this rank, nothing from the peer's competitors
    tau = float(np.float32(sbc.exact(a.q[:1], a.g)[0, a.target[0]]))
    fake = FakeWorld(0, [Peer(q, s1, tau, a.g.shape[0], 1)])
    res = ddist.sharded_range(q, s0, tau, 0, allgather=fake, world=2)
    torch.cuda.synchronize()
    off, idx = _range_check(full, tau, res)
    assert idx.tolist() == a.target.tolist()
