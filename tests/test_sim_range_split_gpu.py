"""GPU: dcr_sim_range_split, the threshold search under the split score (max over the descriptor parts of the per-part dot
products), against the fp64 oracle, bit for bit against dcr_split_rescore and dcr_sim_topk_split, at the threshold's
edges, on a part at its bf16 error bound, on NaN parts, ties, capacity and argument errors, and gallery-sharded (emulated
ranks and two processes)."""
import ctypes as C
import os
import struct

import numpy as np
import pytest
import torch

from dcr_b200 import _lib, retrieval, similarity, synthetic
from dcr_b200 import dist as ddist
from tests import sim_bound_cases as sbc
from tests.test_sim_range_split_cpu import split_range, split_scores

pytestmark = pytest.mark.gpu

CUDA = torch.device("cuda")
MAGIC = int.from_bytes(b"DCRRNG1\0", "little")


def _srange(q, g, t, c, **kw):
    off, idx, val = similarity.sim_range_split(q.to(CUDA), g.to(CUDA), t, c, **kw)
    torch.cuda.synchronize()
    return off.cpu().numpy(), idx.cpu().numpy(), val.cpu().numpy()


def _np(x):
    return x.cpu().numpy() if isinstance(x, torch.Tensor) else x


def _dense_rescore(q, g, c):
    """[nq, ng] split scores from dcr_split_rescore with every gallery row a candidate (the bits the search must give)."""
    lib = _lib.load()
    qd, gd = q.to(CUDA).contiguous(), g.to(CUDA).contiguous()
    nq, d = qd.shape
    ng = gd.shape[0]
    assert ng <= 4096
    cand = torch.arange(ng, dtype=torch.int64, device=CUDA).repeat(nq, 1).contiguous()
    s = torch.empty((nq, ng), dtype=torch.float32, device=CUDA)
    i = torch.empty((nq, ng), dtype=torch.int64, device=CUDA)
    _lib.check(lib.dcr_split_rescore(qd.data_ptr(), gd.data_ptr(), nq, d, c, 0, cand.data_ptr(), ng, ng, s.data_ptr(),
                                     i.data_ptr(), torch.cuda.current_stream().cuda_stream), "dcr_split_rescore")
    out = torch.empty_like(s)
    out.scatter_(1, i, s)
    torch.cuda.synchronize()
    return out.cpu().numpy()


def _csr_of(dense, t):
    keep = dense >= np.float32(t)
    rows, cols = np.nonzero(keep)
    off = np.concatenate([[0], np.cumsum(keep.sum(axis=1))]).astype(np.int64)
    return off, cols.astype(np.int64), dense[rows, cols]


def _same_bits(a, b):
    return (np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
            and np.array_equal(np.asarray(a[2], np.float32).view(np.uint32), np.asarray(b[2], np.float32).view(np.uint32)))


def _tau(s, per_row):
    """A threshold about `per_row` pairs per query, in a gap of the oracle's scores (no pair within 1e-5 of it)."""
    v = np.unique(s[np.isfinite(s)].astype(np.float64))
    j = max(1, min(v.size - 1, v.size - per_row * s.shape[0]))
    while j < v.size - 1 and v[j] - v[j - 1] < 1e-5:
        j += 1
    return float((v[j] + v[j - 1]) / 2)


def _check(q, g, c, t=None, per_row=3):
    qn, gn = _np(q), _np(g)
    s = split_scores(qn, gn, c)
    if t is None:
        t = _tau(s, per_row)
    got = _srange(torch.as_tensor(qn), torch.as_tensor(gn), t, c)
    want = split_range(qn, gn, c, t)
    assert np.array_equal(got[0], want[0]), "row offsets differ"
    assert np.array_equal(got[1], want[1]), "indices differ"
    np.testing.assert_allclose(got[2], want[2], rtol=0, atol=2e-7)
    if gn.shape[0] <= 4096:
        assert _same_bits(got, _csr_of(_dense_rescore(torch.as_tensor(qn), torch.as_tensor(gn), c), t))
    return got, t


@pytest.mark.parametrize("nq,ng,d,c", [
    (64, 3000, 512, 4),              # resident query tile (d_pad = 512)
    (33, 1000, 96, 3),               # parts of 32: below one k-block; resident
    (20, 500, 512, 32),              # parts of 16
    (130, 777, 197 * 64, 197),       # ViT token count, one k-block per part; nq not a multiple of 128; streamed
    (3, 600, 197 * 384, 197),        # ViT-S/16 tokens
    (5, 700, 785 * 16, 785),         # ViT-B/8 token count, parts of 16
    (7, 1, 256, 4),                  # one gallery row
    (9, 5000, 197 * 64, 197),        # several gallery chunks
])
def test_oracle_parity(nq, ng, d, c):
    q, g = synthetic.descriptors(nq, ng, d, seed=nq + ng + c, planted=0.05)
    got, _ = _check(q, g, c, per_row=3 if ng > 1 else 1)
    assert got[0][-1] > 0


def test_all_pairs_are_the_bits_of_split_rescore_and_topk():
    q, g = synthetic.descriptors(50, 900, 256, seed=9, planted=0.1)
    dense = _dense_rescore(q, g, 4)
    got = _srange(q, g, -np.inf, 4)
    assert got[0][-1] == 50 * 900
    assert _same_bits(got, _csr_of(dense, -np.inf))
    # every top-10 entry at or above a threshold is in the CSR with the same bits
    v, i = similarity.sim_topk_split(q.cuda(), g.cuda(), 10, 4)
    v, i = v.cpu().numpy(), i.cpu().numpy()
    t = float(np.median(v[:, 4]))
    off, idx, val = _srange(q, g, t, 4)
    for r in range(50):
        row = dict(zip(idx[off[r]:off[r + 1]].tolist(), val[off[r]:off[r + 1]].view(np.uint32).tolist()))
        for s_, j in zip(v[r], i[r]):
            if s_ >= np.float32(t):
                assert row[int(j)] == np.float32(s_).view(np.uint32)


def test_threshold_edges():
    q, g = synthetic.descriptors(40, 1200, 384, seed=12, planted=0.1)
    off, idx, _ = _srange(q, g, np.inf, 6)
    assert off[-1] == 0 and np.all(off == 0) and idx.size == 0
    v, i = similarity.sim_topk_split(q.cuda(), g.cuda(), 1, 6)
    s0, j0 = np.float32(v[0, 0].item()), int(i[0, 0])
    off, idx, val = _srange(q, g, float(s0), 6)
    assert j0 in idx[off[0]:off[1]].tolist()
    assert np.all(val >= s0)
    nxt = float(np.nextafter(s0, np.float32(np.inf)))
    off, idx, val = _srange(q, g, nxt, 6)
    assert j0 not in idx[off[0]:off[1]].tolist() and np.all(val >= np.float32(nxt))


def test_a_part_at_its_bf16_bound_is_reported():
    """Part 0 holds the sim_bound_cases instance the split top-k test uses (a pair's bf16 error at the bound); the other
    parts score far lower.  At a threshold equal to a query's best exact score that pair is still reported."""
    case = sbc.build(64, 40, centred=False)
    nq, ng = case.q.shape[0], case.g.shape[0]
    rng = np.random.default_rng(5)
    c, p = 4, 64
    q = np.concatenate([case.q, 0.01 * rng.standard_normal((nq, (c - 1) * p))], axis=1).astype(np.float32)
    g = np.concatenate([case.g, 0.01 * rng.standard_normal((ng, (c - 1) * p))], axis=1).astype(np.float32)
    dense = _dense_rescore(torch.from_numpy(q), torch.from_numpy(g), c)
    for r in range(nq):
        t = float(dense[r].max())
        got = _srange(torch.from_numpy(q), torch.from_numpy(g), t, c)
        assert _same_bits(got, _csr_of(dense, t))
        assert int(np.argmax(dense[r])) in got[1][got[0][r]:got[0][r + 1]].tolist()


def test_nan_parts():
    c, p = 4, 64
    q, g = synthetic.descriptors(20, 700, c * p, seed=21, planted=0.1)
    g[3, :p] = float("nan")                  # one NaN part: ignored
    g[10] = float("nan")                     # every part NaN: -inf, reported only at -inf
    q[5, 2 * p:3 * p] = float("nan")         # a NaN query part: that row stays exact
    dense = _dense_rescore(q, g, c)
    assert np.all(dense[:, 10] == -np.inf) and np.all(np.isfinite(dense[:, 3]))
    for t in (-np.inf, -0.5, 0.0, 0.3):
        got = _srange(q, g, t, c)
        assert _same_bits(got, _csr_of(dense, t)), t
        want = split_range(q.numpy(), g.numpy(), c, t)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    off, idx, val = _srange(q, g, -np.inf, c)
    assert np.all(val[idx == 10] == -np.inf) and np.sum(idx == 10) == 20


def test_ties_and_duplicates():
    c = 8
    q, g = synthetic.descriptors(16, 1200, 512, seed=11, planted=0.05)
    g[100:110] = g[7]
    g[900] = q[3]
    g[300] = q[3]
    p = 512 // c
    dense = split_scores(q.numpy(), g.numpy(), c)
    a = int(np.argmax(dense[0]))
    parts = (q[0].double().view(c, p) * g[a].double().view(c, p)).sum(1)
    best = int(parts.argmax())
    b = a + 1 if a < 1199 else a - 1
    g[b] = 0
    g[b, best * p:(best + 1) * p] = g[a, best * p:(best + 1) * p]    # equal to row a only in its best part
    got, _ = _check(q, g, c, per_row=4)
    d2 = _dense_rescore(q, g, c)
    assert d2[0, a] == d2[0, b]
    got = _srange(q, g, float(d2[0, a]), c)
    assert {a, b} <= set(got[1][got[0][0]:got[0][1]].tolist())
    off, idx, _ = _srange(q, g, float(d2[1, 7]), c)                 # the eleven copies of row 7 tie for query 1
    assert set(range(100, 110)) | {7} <= set(idx[off[1]:off[2]].tolist())


def test_one_part_gives_the_bits_of_sim_range():
    q, g = synthetic.descriptors(100, 3000, 384, seed=2, planted=0.1)
    a = _srange(q, g, 0.3, 1)
    b = tuple(x.cpu().numpy() for x in similarity.sim_range(q.cuda(), g.cuda(), 0.3))
    assert b[0][-1] > 0 and _same_bits(a, b)


def test_index_base_stride_and_determinism():
    q, g = synthetic.descriptors(30, 800, 256, seed=4, planted=0.1)
    a = _srange(q, g, 0.2, 4)
    b = _srange(q, g, 0.2, 4, index_base=5000, index_stride=3)
    assert a[0][-1] > 0
    assert np.array_equal(a[0], b[0]) and np.array_equal(b[1], 5000 + 3 * a[1])
    assert np.array_equal(a[2].view(np.uint32), b[2].view(np.uint32))
    assert _same_bits(a, _srange(q, g, 0.2, 4))


def _c_call(q, g, t, c, cap):
    lib = _lib.load()
    nq, d = q.shape
    ng = g.shape[0]
    counts = (C.c_int64 * 2)()
    nbytes = lib.dcr_sim_range_split_workspace_size(nq, ng, d, c, cap)
    assert nbytes > 0
    ws = torch.empty(nbytes + 256, dtype=torch.uint8, device=CUDA)
    off = torch.empty(nq + 1, dtype=torch.int64, device=CUDA)
    idx = torch.empty(max(cap, 1), dtype=torch.int64, device=CUDA)
    val = torch.empty(max(cap, 1), dtype=torch.float32, device=CUDA)
    rc = lib.dcr_sim_range_split(q.data_ptr(), nq, g.data_ptr(), ng, d, c, t, 0, 1, off.data_ptr(), idx.data_ptr(),
                                 val.data_ptr(), cap, counts, similarity._aligned_ptr(ws), nbytes,
                                 torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return rc, (int(counts[0]), int(counts[1])), off, idx, val


def test_capacity_error_reports_the_exact_need():
    q, g = synthetic.descriptors(60, 2000, 256, seed=6, planted=0.2)
    q, g = q.cuda(), g.cuda()
    rc, (_, need), *_ = _c_call(q, g, 0.1, 4, 10)
    assert rc == _lib.ERR_CAPACITY and need > 10 and "sim_range_split" in _lib.last_error()
    rc, (pairs, need2), off, idx, val = _c_call(q, g, 0.1, 4, need)
    assert rc == 0 and need2 == need and 0 < pairs <= need
    want = similarity.sim_range_split(q, g, 0.1, 4)
    assert torch.equal(off, want[0]) and torch.equal(idx[:pairs], want[1]) and torch.equal(val[:pairs], want[2])


def test_argument_errors_are_refused_with_a_message():
    q, g = synthetic.descriptors(4, 40, 64, seed=1)
    qc, gc = q.cuda(), g.cuda()
    for args, match in [((qc, gc, 0.5, 3), "parts"),                                          # 64 into 3 parts
                        ((qc[:, :60].contiguous(), gc[:, :60].contiguous(), 0.5, 10), "multiple of 4"),
                        ((qc, gc, 0.5, 0), "n_parts"),
                        ((qc, gc, float("nan"), 2), "NaN"),
                        ((qc, gc[:, :32].contiguous(), 0.5, 2), "dims differ"),
                        ((q, g, 0.5, 2), "CUDA")]:
        with pytest.raises(_lib.DcrError, match=match):
            similarity.sim_range_split(*args)
    long_q = torch.zeros(2, 2 * 8196, device=CUDA)
    with pytest.raises(_lib.DcrError, match="8192"):
        similarity.sim_range_split(long_q, long_q, 0.5, 2)


# ------------------------------------------------------------------------------------------------------------------
# gallery-sharded

def _thr_bits(t):
    return struct.unpack("<I", struct.pack("<f", np.float32(t)))[0]


class Peer:
    """A rank played by the test: the header and message its library would send, from sim_range_split on its shard."""

    def __init__(self, q, shard, t, c, base, stride, **hdr):
        nq, d = q.shape
        if shard.shape[0] > 0:
            off, idx, val = similarity.sim_range_split(q, shard, t, c, index_base=base, index_stride=stride)
        else:
            off = torch.zeros(nq + 1, dtype=torch.int64, device=CUDA)
            idx = torch.zeros(0, dtype=torch.int64, device=CUDA)
            val = torch.zeros(0, dtype=torch.float32, device=CUDA)
        self.pairs = int(off[-1])
        self.payload = torch.cat([off.view(torch.uint8), idx.view(torch.uint8), val.view(torch.uint8)])
        h = dict(magic=MAGIC, status=0, pairs=self.pairs, cand=self.pairs, cap=1 << 20, max_pairs=1 << 30, nq=nq, d=d,
                 thr=_thr_bits(t), parts=c if c > 1 else 0)
        h.update(hdr)
        self.header = torch.tensor(list(h.values()), dtype=torch.int64, device=CUDA).view(torch.uint8)


class FakeWorld:
    """The all-gather callback of rank `me`: headers on the first call, messages on the second."""

    def __init__(self, me, peers):
        self.me, self.peers, self.calls = me, list(peers), []

    def __call__(self, send, recv, nbytes, stream):
        world = len(self.peers) + 1
        second = len(self.calls) > 0
        self.calls.append(nbytes)
        out = ddist.device_bytes(recv, nbytes * world, CUDA)
        own = ddist.device_bytes(send, nbytes, CUDA)
        ranks = self.peers[:self.me] + [None] + self.peers[self.me:]
        for r, p in enumerate(ranks):
            dst = out[r * nbytes:(r + 1) * nbytes]
            if p is None:
                dst.copy_(own)
                continue
            src = p.payload if second else p.header
            dst.fill_(0xA5)
            dst[:src.numel()].copy_(src)
        return 0


def _shards(g, world, layout):
    G = g.shape[0]
    if layout == "interleaved":
        return [g[r::world].contiguous() for r in range(world)], list(range(world)), world
    cuts = [0, G // 3, G // 3, G] if world == 3 else [0, 0, G]      # ragged, one shard empty
    return [g[cuts[r]:cuts[r + 1]].contiguous() for r in range(world)], cuts[:-1], 1


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("layout", ["contiguous", "interleaved"])
def test_emulated_ranks_equal_one_process(world, layout):
    c = 4
    q, g = synthetic.descriptors(130, 2500, 256, seed=world, planted=0.2)
    q, g = q.cuda(), g.cuda()
    t = 0.15                                       # planted rows reach it in their parts, random pairs do not
    want = similarity.sim_range_split(q, g, t, c)
    assert int(want[0][-1]) > 130
    shards, bases, stride = _shards(g, world, layout)
    for me in range(world):
        fake = FakeWorld(me, [Peer(q, shards[r], t, c, bases[r], stride) for r in range(world) if r != me])
        res = ddist.sharded_range(q, shards[me], t, bases[me], allgather=fake, world=world, index_stride=stride,
                                  num_chunks=c)
        torch.cuda.synchronize()
        assert len(fake.calls) == 2
        assert all(torch.equal(x, y) for x, y in zip(res, want)), (me, layout)


def test_peer_that_disagrees_on_n_parts():
    c = 4
    q, g = synthetic.descriptors(50, 1000, 256, seed=5, planted=0.2)
    q, g = q.cuda(), g.cuda()
    own, other = g[:600].contiguous(), g[600:].contiguous()
    for me, peer_parts in [(0, 0), (1, 8), (0, 2)]:
        fake = FakeWorld(me, [Peer(q, other, 0.3, c, 600, 1, parts=peer_parts)])
        with pytest.raises(_lib.DcrError, match="disagree"):
            ddist.sharded_range(q, own, 0.3, 0, allgather=fake, world=2, num_chunks=c)
        assert len(fake.calls) == 1
    # the dot-product entry still writes 0: a split peer disagrees with it, a dot-product peer does not
    fake = FakeWorld(0, [Peer(q, other, 0.3, c, 600, 1)])
    with pytest.raises(_lib.DcrError, match="disagree"):
        ddist.sharded_range(q, own, 0.3, 0, allgather=fake, world=2)


_NQ, _NG, _D, _C = 45, 1301, 256, 4


def _worker(rank, world, port, out_dir):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    q, g = synthetic.descriptors(_NQ, _NG, _D, seed=8, planted=0.1)
    q, g = q.cuda(), g.cuda()
    lo, hi = ddist.shard_bounds(_NG, rank, world)
    out = {}
    for name, t in [("match", 0.15), ("dense", -np.inf)]:
        o, i, v = ddist.sharded_range(q, g[lo:hi], t, lo, num_chunks=_C)
        out.update({f"{name}_o": o.cpu().numpy(), f"{name}_i": i.cpu().numpy(), f"{name}_v": v.cpu().numpy()})
    np.savez(os.path.join(out_dir, f"rank{rank}.npz"), **out)
    dist.barrier()
    dist.destroy_process_group()


def test_two_processes_on_one_gpu_gloo(tmp_path):
    import torch.multiprocessing as mp
    mp.spawn(_worker, args=(2, 28900 + os.getpid() % 500, str(tmp_path)), nprocs=2, join=True)
    q, g = synthetic.descriptors(_NQ, _NG, _D, seed=8, planted=0.1)
    q, g = q.cuda(), g.cuda()
    want = {"match": similarity.sim_range_split(q, g, 0.15, _C), "dense": similarity.sim_range_split(q, g, -np.inf, _C)}
    assert int(want["match"][0][-1]) > _NQ and int(want["dense"][0][-1]) == _NQ * _NG
    for r in range(2):
        got = np.load(os.path.join(tmp_path, f"rank{r}.npz"))
        for name, (o, i, v) in want.items():
            assert np.array_equal(got[f"{name}_o"], o.cpu().numpy()), (r, name)
            assert np.array_equal(got[f"{name}_i"], i.cpu().numpy()), (r, name)
            assert np.array_equal(got[f"{name}_v"].view(np.uint32), v.cpu().numpy().view(np.uint32)), (r, name)


# ------------------------------------------------------------------------------------------------------------------
# retrieval

def test_run_retrieval_threshold_with_parts(monkeypatch):
    """run_retrieval(threshold, num_loss_chunks = C) fills out["matches"] from sim_range_split; the cross form still
    refuses.  The network is stood in for by fixed descriptors (the wiring is under test, not the network)."""
    c = 4
    q, g = synthetic.descriptors(30, 500, 256, seed=14, planted=0.2)
    q_img = torch.zeros((30, 4, 4, 3), dtype=torch.uint8)
    g_img = torch.zeros((500, 4, 4, 3), dtype=torch.uint8)
    feats = {id(q_img): q, id(g_img): g}
    monkeypatch.setattr(retrieval, "extract_features", lambda net, images, bs=None: feats[id(images)].cuda().clone())
    out = retrieval.run_retrieval(None, q_img, g_img, k=1, num_loss_chunks=c, threshold=0.15)
    assert torch.equal(out["query_features"], similarity.l2_normalize_(q.cuda().clone()))
    want = similarity.sim_range_split(out["query_features"], out["gallery_features"], 0.15, c)
    assert int(want[0][-1]) > 0
    assert all(torch.equal(x, y) for x, y in zip(out["matches"], want))
    with pytest.raises(NotImplementedError):
        retrieval.run_retrieval(None, q_img, g_img, k=1, num_loss_chunks=c, cross=True, threshold=0.3)
