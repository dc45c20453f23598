"""GPU parity of the cross split score (a pair scores the best of every (query part, gallery part) dot product):
dcr_sim_topk_cross against the fp64 oracle and bit for bit against dcr_split_rescore(cross = 1), on shapes the per-part
composition refused, on operands that drive the winning pair's bf16 error to its bound, with NaN parts; the threshold
search dcr_sim_range_cross against the dense oracle; and the gallery-sharded top-k across two processes."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from dcr_b200 import _lib, similarity, synthetic
from dcr_b200 import dist as ddist
from oracle import similarity as osim
from tests import sim_bound_cases as sbc
from tests.test_sim_cross_cpu import cross_range, cross_topk

pytestmark = pytest.mark.gpu


def _cross(q, g, k, c, **kw):
    v, i = similarity.sim_topk_split(q.cuda(), g.cuda(), k, c, cross=True, **kw)
    torch.cuda.synchronize()
    return v.cpu().numpy(), i.cpu().numpy(), similarity.sim_topk_stats()


def _rescore_cross(q, g, k, c, cand):
    """dcr_split_rescore(cross = 1) on the given candidates [nq, n_cand]: the bits the fused search must report."""
    lib = _lib.load()
    qd, gd = q.cuda().contiguous(), g.cuda().contiguous()
    cand = torch.as_tensor(cand, dtype=torch.int64).cuda().contiguous()
    nq, d = qd.shape
    out_s = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    out_i = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    rc = lib.dcr_split_rescore(qd.data_ptr(), gd.data_ptr(), nq, d, c, 1, cand.data_ptr(), cand.shape[1], k,
                               out_s.data_ptr(), out_i.data_ptr(), torch.cuda.current_stream().cuda_stream)
    _lib.check(rc, "dcr_split_rescore")
    torch.cuda.synchronize()
    return out_s.cpu().numpy(), out_i.cpu().numpy()


def _check(q, g, k, c, exact_bits=True):
    """Indices equal to the fp64 ranking, values within 1e-6 of it, and every value bitwise what dcr_split_rescore
    reports for the returned rows (and, for galleries of <= 4096 rows, the same top-k from every row as a candidate)."""
    qn, gn = q.numpy(), g.numpy()
    v, i, st = _cross(q, g, k, c)
    ov, oi = cross_topk(qn, gn, k, c)
    bad = np.nonzero((i != oi).any(axis=1))[0]
    assert bad.size == 0, f"{bad.size} query rows differ, first {bad[:5]}: got {i[bad[:3]]} want {oi[bad[:3]]}"
    np.testing.assert_allclose(v, ov, rtol=0, atol=1e-6)
    rv, ri = _rescore_cross(q, g, k, c, i)
    assert np.array_equal(ri, i) and np.array_equal(v.view(np.uint32), rv.view(np.uint32))
    if exact_bits and g.shape[0] <= 4096:
        rv, ri = _rescore_cross(q, g, k, c, np.tile(np.arange(g.shape[0]), (q.shape[0], 1)))
        assert np.array_equal(i, ri) and np.array_equal(v.view(np.uint32), rv.view(np.uint32))
    return v, i, st


@pytest.mark.parametrize("nq,ng,c,p,k", [
    (64, 3000, 4, 128, 10),       # d_pad = 512: the widest resident query tile
    (33, 1000, 8, 4, 1),          # parts of 4, padded to one 64-column k-block each
    (20, 500, 3, 100, 16),        # p = 100 padded to 128
    (17, 700, 8, 64, 2),
    (25, 900, 8, 100, 10),        # d_pad = 1024: streamed query tile
    (40, 1300, 2, 64, 10),        # ng not a multiple of 128
    (1, 100, 2, 64, 10),          # nq = 1, ng < 128
    (9, 259, 2, 4, 3),
    (5, 16, 4, 64, 16),           # k = ng
])
def test_parity(nq, ng, c, p, k):
    q, g = synthetic.descriptors(nq, ng, c * p, seed=nq + ng + c, planted=0.05)
    _check(q, g, k, c)


@pytest.mark.parametrize("nq,ng,c,p,k", [
    (24, 1500, 32, 16, 10),       # C^2 k = 10240 > 4096: the composition refused this
    (10, 800, 64, 16, 5),
    (4, 600, 197, 64, 10),        # ViT token count at the default top-10
])
def test_shapes_the_composition_refused(nq, ng, c, p, k):
    q, g = synthetic.descriptors(nq, ng, c * p, seed=3 * c + k, planted=0.05)
    _check(q, g, k, c, exact_bits=ng <= 1000)


def test_matches_the_einsum_oracle():
    """oracle.similarity.sim_topk_split(cross=True), the restatement of einsum_in_chunks, on a small [chunk, G, C, C]."""
    q, g = synthetic.descriptors(12, 400, 256, seed=5, planted=0.05)
    v, i, _ = _cross(q, g, 10, 4)
    ov, oi = osim.sim_topk_split(q.numpy(), g.numpy(), 10, 4, cross=True, chunk=4)
    assert np.array_equal(i, oi)
    np.testing.assert_allclose(v, ov, rtol=0, atol=1e-6)


def test_duplicate_rows_lowest_index_wins():
    q, g = synthetic.descriptors(40, 1500, 256, seed=3, planted=0.05)
    g[100:110] = g[7]
    g[900] = 4 * q[3]            # query 3's best rows by far: every aligned pair scores 4 |q_a|^2
    g[300] = 4 * q[3]
    g[20] = g[100]
    v, i, _ = _check(q, g, 10, 4)
    assert i[3, 0] == 300 and i[3, 1] == 900 and v[3, 0] == v[3, 1]


def test_a_pair_equal_to_another_rows_best_pair():
    """Row b holds, in gallery part 0, what row a holds in the gallery part where its best pair lies: both rows score
    the same, and the lower index comes first."""
    c, p, k = 4, 64, 5
    q, g = synthetic.descriptors(16, 1200, c * p, seed=11, planted=0.05)
    _, oi = cross_topk(q.numpy(), g.numpy(), k, c)
    a = int(oi[0, 0])
    pairs = q[0].double().view(c, 1, p).mul(g[a].double().view(1, c, p)).sum(2)   # [query part, gallery part]
    bq, bg = divmod(int(pairs.argmax()), c)
    g2 = g.clone()
    b = 1199 if a != 1199 else 0
    g2[b] = 0
    g2[b, :p] = g[a, bg * p:(bg + 1) * p]
    v, i, _ = _check(q, g2, k, c)
    assert set(i[0, :2].tolist()) == {a, b} and i[0, 0] == min(a, b) and v[0, 0] == v[0, 1]


def test_one_part_gives_the_bits_of_sim_topk():
    q, g = synthetic.descriptors(100, 3000, 384, seed=2)
    v, i, _ = _cross(q, g, 10, 1)
    w, j = similarity.sim_topk(q.cuda(), g.cuda(), 10)
    assert np.array_equal(i, j.cpu().numpy())
    assert np.array_equal(v.view(np.uint32), w.cpu().numpy().view(np.uint32))


def test_index_base_and_stride():
    q, g = synthetic.descriptors(30, 800, 256, seed=4)
    v, i, _ = _cross(q, g, 7, 4)
    w, j, _ = _cross(q, g, 7, 4, index_base=5000, index_stride=3)
    assert np.array_equal(j, 5000 + 3 * i)
    assert np.array_equal(v.view(np.uint32), w.view(np.uint32))


def test_argument_errors_are_refused_with_a_message():
    q, g = synthetic.descriptors(4, 40, 64, seed=1)
    qc, gc = q.cuda(), g.cuda()
    for args, match in [((qc, gc, 3, 3), "parts"), ((qc, gc, 17, 2), "k="),
                        ((qc, gc[:5].contiguous(), 6, 2), "gallery size"), ((qc, gc, 3, 0), "n_parts")]:
        with pytest.raises(_lib.DcrError, match=match):
            similarity.sim_topk_split(*args, cross=True)


# ------------------------------------------------------------------------------------------------------------------
# the winning pair (query part a, gallery part b), a != b, at its bf16 error bound

CROSS_PLACES = sbc.CROSS_PLACES   # (C, p, a, b): the instance in the pair (a, b) (sbc.cross_embed)
ADVERSARIAL = [(name, *place) for name, *_ in sbc.TOPK_CASES for place in CROSS_PLACES]


@pytest.mark.parametrize("name,c,p,a,b", ADVERSARIAL, ids=[f"{x[0]}-C{x[1]}-p{x[2]}-q{x[3]}g{x[4]}" for x in ADVERSARIAL])
def test_pair_at_its_bf16_bound(name, c, p, a, b):
    """The bound instances of tests/sim_bound_cases.py (a near-tie whose bf16 order inverts the exact order, at the
    realized error of eps) in the pair (a, b): indices and score bits of the fp64 ranking, decided by the stage the
    instance is built for."""
    _, k, n_b, shared, tie, stage = next(x for x in sbc.TOPK_CASES if x[0] == name)
    case = sbc.topk_case(name, p, False)
    e = sbc.cross_embed(case, c, a, b)
    q, g = torch.from_numpy(e.q), torch.from_numpy(e.g)
    v, i, st = _check(q, g, k, c)
    nq = q.shape[0]
    assert (i[:, 0] == case.target).all()
    if tie and k > 1:
        assert (i[:, 1] == case.twin).all()
    assert st["kp"] == sbc.KP0[k]
    if stage == "first":
        assert st["n_second"] == 0 and st["n_flagged"] == 0, st
    elif stage == "second":
        assert st["n_second"] == nq and st["n_flagged"] == 0, st
    else:
        assert st["n_flagged"] == nq, st


# ------------------------------------------------------------------------------------------------------------------
# NaN parts

def test_nan_parts():
    """A NaN part in a query and in a gallery row is ignored; an all-NaN query scores -inf against every row (ties to
    the lowest rows); the NaN norms send the queries to the brute-force path, which still gives the oracle's answer."""
    c, p = 4, 64
    q, g = synthetic.descriptors(20, 700, c * p, seed=9, planted=0.05)
    q[2, p:2 * p] = float("nan")
    g[5, 2 * p:3 * p] = float("nan")
    q[7] = float("nan")
    v, i, st = _check(q, g, 10, c)
    assert st["n_flagged"] > 0, st
    assert np.all(v[7] == -np.inf) and np.array_equal(i[7], np.arange(10))
    # only the query holds a NaN part: that query alone is flagged
    q2, g2 = synthetic.descriptors(20, 700, c * p, seed=9, planted=0.05)
    q2[2, p:2 * p] = float("nan")
    _, _, st = _check(q2, g2, 10, c)
    assert st["n_flagged"] >= 1, st


# ------------------------------------------------------------------------------------------------------------------
# threshold search

def _range(q, g, tau, c, **kw):
    return tuple(x.cpu().numpy() for x in similarity.sim_range_split(q.cuda(), g.cuda(), tau, c, cross=True, **kw))


def _range_equal(got, want):
    off, idx, val = got
    ooff, oidx, oval = want
    assert np.array_equal(off, ooff) and np.array_equal(idx, oidx)
    assert np.array_equal(val.view(np.uint32), oval.view(np.uint32))


@pytest.mark.parametrize("nq,ng,c,p", [(40, 2000, 4, 128), (30, 1500, 8, 100), (9, 259, 2, 4), (6, 500, 32, 16)])
def test_range_matches_the_dense_oracle(nq, ng, c, p):
    """Resident (d_pad <= 512) and streamed (d_pad = 1024) query tiles; tau at the 10th best cross score of query 0."""
    q, g = synthetic.descriptors(nq, ng, c * p, seed=nq + c, planted=0.05)
    ov, _ = cross_topk(q.numpy(), g.numpy(), 10, c)
    tau = float(ov[0, -1])
    got = _range(q, g, tau, c)
    _range_equal(got, cross_range(q.numpy(), g.numpy(), c, tau))
    # every pair of the top-k at or above tau carries the top-k's bits
    v, i, _ = _cross(q, g, 10, c)
    off, idx, val = got
    for r in range(nq):
        row = dict(zip(idx[off[r]:off[r + 1]].tolist(), val[off[r]:off[r + 1]].view(np.uint32).tolist()))
        for s, j in zip(v[r], i[r]):
            if s >= np.float32(tau):
                assert row[int(j)] == np.float32(s).view(np.uint32)


def test_range_all_pairs_at_minus_inf():
    q, g = synthetic.descriptors(11, 300, 4 * 64, seed=13)
    off, idx, val = _range(q, g, float("-inf"), 4)
    assert off[-1] == 11 * 300 and np.array_equal(idx, np.tile(np.arange(300), 11))
    _range_equal((off, idx, val), cross_range(q.numpy(), g.numpy(), 4, float("-inf")))


def test_range_capacity_protocol_and_determinism():
    """DCR_ERR_CAPACITY with counts[1] the capacity the call needs, then the call with it succeeds; two calls, two
    workspace sizes and two query tilings give the same bits."""
    lib = _lib.load()
    c, p = 4, 64
    q, g = synthetic.descriptors(300, 1000, c * p, seed=21)
    qd, gd = q.cuda(), g.cuda()
    tau = 0.0
    nq, d = qd.shape
    ng = gd.shape[0]

    def call(cap, extra=0):
        counts = (C.c_int64 * 2)()
        nbytes = lib.dcr_sim_range_cross_workspace_size(nq, ng, d, c, cap)
        assert nbytes > 0
        ws = torch.empty(nbytes + extra + 256, dtype=torch.uint8, device="cuda")
        off = torch.empty(nq + 1, dtype=torch.int64, device="cuda")
        oi = torch.empty(max(cap, 1), dtype=torch.int64, device="cuda")
        os_ = torch.empty(max(cap, 1), dtype=torch.float32, device="cuda")
        rc = lib.dcr_sim_range_cross(qd.data_ptr(), nq, gd.data_ptr(), ng, d, c, tau, 0, 1, off.data_ptr(), oi.data_ptr(),
                                     os_.data_ptr(), cap, counts, (ws.data_ptr() + 255) // 256 * 256, nbytes + extra,
                                     torch.cuda.current_stream().cuda_stream)
        n = int(counts[0])
        return rc, int(counts[1]), (off.cpu().numpy(), oi[:n].cpu().numpy(), os_[:n].cpu().numpy())

    rc, need, _ = call(1000)
    assert rc == _lib.ERR_CAPACITY and need > 1000
    rc, need2, first = call(need)
    assert rc == 0 and need2 == need
    rc, _, second = call(4 * need, extra=1 << 20)
    assert rc == 0
    _range_equal(second, first)
    _range_equal(_range(q, g, tau, c), first)                          # the Python retry
    _range_equal(first, cross_range(q.numpy(), g.numpy(), c, tau))
    # queries 130.. alone: another query tiling and work split, the same rows
    off, idx, val = _range(q[130:].contiguous(), g, tau, c)
    o0 = first[0]
    assert np.array_equal(off, o0[130:] - o0[130])
    assert np.array_equal(idx, first[1][o0[130]:]) and np.array_equal(val.view(np.uint32), first[2][o0[130]:].view(np.uint32))


def test_range_one_part_gives_the_bits_of_sim_range():
    q, g = synthetic.descriptors(50, 2000, 256, seed=6)
    got = _range(q, g, 0.2, 1)
    want = tuple(x.cpu().numpy() for x in similarity.sim_range(q.cuda(), g.cuda(), 0.2))
    _range_equal(got, want)


def test_range_nan_parts():
    c, p = 4, 64
    q, g = synthetic.descriptors(12, 400, c * p, seed=19, planted=0.05)
    q[2, p:2 * p] = float("nan")
    g[5, 2 * p:3 * p] = float("nan")
    q[7] = float("nan")
    got = _range(q, g, float("-inf"), c)
    _range_equal(got, cross_range(q.numpy(), g.numpy(), c, float("-inf")))
    off, _, val = got
    assert np.all(val[off[7]:off[8]] == -np.inf)
    _range_equal(_range(q, g, 0.1, c), cross_range(q.numpy(), g.numpy(), c, 0.1))


# ------------------------------------------------------------------------------------------------------------------
# gallery-sharded across real processes, on a shape the per-part composition refused (C^2 k = 10240 > 4096)

_NQ, _NG, _D, _C = 45, 1301, 512, 32


def _worker(rank, world, port, out_dir):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    q, g = synthetic.descriptors(_NQ, _NG, _D, seed=8, planted=0.1)
    q, g = q.cuda(), g.cuda()
    qlo, qhi = ddist.shard_bounds(_NQ, rank, world)
    q_sizes = [b - a for a, b in (ddist.shard_bounds(_NQ, r, world) for r in range(world))]
    out = {}
    for name, ng, k in [("cross", _NG, 10), ("small", 13, 8)]:
        lo, hi = ddist.shard_bounds(ng, rank, world)
        s, i = ddist.sharded_topk(q[qlo:qhi], g[lo:hi], k, lo, ddist.split_local_topk(_C, cross=True), ddist.cuda_merge,
                                  query_sizes=q_sizes)
        out[f"{name}_s"], out[f"{name}_i"] = s.cpu().numpy(), i.cpu().numpy()
    np.savez(os.path.join(out_dir, f"rank{rank}.npz"), **out)
    dist.barrier()
    dist.destroy_process_group()


def test_sharded_two_processes_on_one_gpu_gloo(tmp_path):
    import torch.multiprocessing as mp
    mp.spawn(_worker, args=(2, 30500 + os.getpid() % 500, str(tmp_path)), nprocs=2, join=True)
    q, g = synthetic.descriptors(_NQ, _NG, _D, seed=8, planted=0.1)
    q, g = q.cuda(), g.cuda()
    want = {"cross": similarity.sim_topk_split(q, g, 10, _C, cross=True),
            "small": similarity.sim_topk_split(q, g[:13].contiguous(), 8, _C, cross=True)}   # shards of 7 and 6 < k
    for r in range(2):
        got = np.load(os.path.join(tmp_path, f"rank{r}.npz"))
        for name, (s, i) in want.items():
            assert np.array_equal(got[f"{name}_i"], i.cpu().numpy()), (r, name)
            assert np.array_equal(got[f"{name}_s"].view(np.uint32), s.cpu().numpy().view(np.uint32)), (r, name)
