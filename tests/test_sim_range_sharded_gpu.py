"""GPU: the gallery-sharded threshold search (dcr_sim_range_sharded / dist.sharded_range) against the single-process
search and the fp64 oracle.

- Emulated ranks in one process: the test plays the peers.  Their headers and messages are built from sim_range on their
  shards in the layout include/dcr_b200.h documents, and the callback writes them around this rank's own block.
- The agreement rules: a peer's failure, capacity shortfall or different problem reaches this rank as the same outcome.
- Two real processes on one GPU over gloo through the default callback, and the same over NCCL with two GPUs.
"""
import ctypes as C
import os
import struct

import numpy as np
import pytest
import torch

from dcr_b200 import _lib, similarity, synthetic
from dcr_b200 import dist as ddist
from tests import sim_range_oracle as orange

pytestmark = pytest.mark.gpu

MAGIC = int.from_bytes(b"DCRRNG1\0", "little")
CUDA = torch.device("cuda")


def _thr_bits(t):
    return struct.unpack("<I", struct.pack("<f", np.float32(t)))[0]


class Peer:
    """A rank played by the test: the header and the message its library would send, from sim_range on its shard."""

    def __init__(self, q, shard, t, base, stride, **hdr):
        nq, d = q.shape
        if shard.shape[0] > 0:
            off, idx, val = similarity.sim_range(q, shard, t, index_base=base, index_stride=stride)
        else:
            off = torch.zeros(nq + 1, dtype=torch.int64, device=CUDA)
            idx = torch.zeros(0, dtype=torch.int64, device=CUDA)
            val = torch.zeros(0, dtype=torch.float32, device=CUDA)
        self.idx = idx
        self.pairs = int(off[-1])
        self.payload = torch.cat([off.view(torch.uint8), idx.view(torch.uint8), val.view(torch.uint8)])
        h = dict(magic=MAGIC, status=0, pairs=self.pairs, cand=self.pairs, cap=1 << 20, max_pairs=1 << 30, nq=nq, d=d,
                 thr=_thr_bits(t), reserved=0)
        h.update(hdr)
        self.header = torch.tensor(list(h.values()), dtype=torch.int64, device=CUDA).view(torch.uint8)


class FakeWorld:
    """The all-gather callback of rank `me`: [peers before me | own block | peers after me], headers on the first call,
    messages (padded to bytes_per_rank) on the second."""

    def __init__(self, me, peers):
        self.me, self.peers, self.calls = me, list(peers), []

    def __call__(self, send, recv, nbytes, stream):
        world = len(self.peers) + 1
        second = len(self.calls) > 0
        self.calls.append(nbytes)
        assert nbytes == 80 or second
        out = ddist.device_bytes(recv, nbytes * world, CUDA)
        own = ddist.device_bytes(send, nbytes, CUDA)
        ranks = self.peers[:self.me] + [None] + self.peers[self.me:]
        for r, p in enumerate(ranks):
            dst = out[r * nbytes:(r + 1) * nbytes]
            if p is None:
                dst.copy_(own)
                continue
            src = p.payload if second else p.header
            assert src.numel() <= nbytes
            dst.fill_(0xA5)                                         # padding is never read
            dst[:src.numel()].copy_(src)
        return 0


def _shards(g, world, layout):
    """(shards, bases, stride) for contiguous ragged shards with an empty one, or interleaved shards."""
    G = g.shape[0]
    if layout == "interleaved":
        return [g[r::world].contiguous() for r in range(world)], list(range(world)), world
    cuts = [0, G // 3, G // 3, G] if world == 3 else [0, 0, G]      # ragged, one shard empty
    return [g[cuts[r]:cuts[r + 1]].contiguous() for r in range(world)], cuts[:-1], 1


def _emulated(q, g, t, world, layout, me):
    shards, bases, stride = _shards(g, world, layout)
    peers = [Peer(q, shards[r], t, bases[r], stride) for r in range(world) if r != me]
    fake = FakeWorld(me, peers)
    res = ddist.sharded_range(q, shards[me], t, bases[me], allgather=fake, world=world, index_stride=stride)
    torch.cuda.synchronize()
    assert len(fake.calls) == 2
    return res, fake


def _equal(a, b):
    return all(torch.equal(x.cpu(), y.cpu()) for x, y in zip(a, b))


def _check_oracle(res, q, g, t):
    off, idx, val = (x.cpu().numpy() for x in res)
    ooff, oidx, oval = orange.sim_range(q.cpu().numpy(), g.cpu().numpy(), t)
    assert np.array_equal(off, ooff) and np.array_equal(idx, oidx)
    np.testing.assert_allclose(val, oval, rtol=0, atol=1.2e-7)


CASES = [("dense", 40, 300, 128, -np.inf), ("half", 130, 3000, 256, 0.5), ("none", 64, 2000, 512, 1.5)]


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("layout", ["contiguous", "interleaved"])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_emulated_ranks_equal_one_process(world, layout, case):
    _, nq, G, d, t = case
    q, g = synthetic.descriptors(nq, G, d, seed=G + world, planted=0.2)
    q, g = q.cuda(), g.cuda()
    want = similarity.sim_range(q, g, t)
    if case[0] == "dense":
        assert int(want[0][-1]) == nq * G
    elif case[0] == "half":
        assert int(want[0][-1]) > nq                                     # several pairs per row, spread over the ranks
    else:
        assert int(want[0][-1]) == 0
    for me in range(world):                                              # this rank at every position, the empty one too
        res, _ = _emulated(q, g, t, world, layout, me)
        assert _equal(res, want), (me, layout)
    _check_oracle(res, q, g, t)


def test_emulated_self_join_with_diagonal():
    _, g = synthetic.descriptors(16, 2500, 256, seed=5, planted=0.3)
    g = g.cuda()
    want = similarity.sim_range(g, g, 0.5)
    off, idx = want[0].cpu(), want[1].cpu()
    assert all(r in idx[off[r]:off[r + 1]] for r in range(2500))
    for layout in ("contiguous", "interleaved"):
        res, _ = _emulated(g, g, 0.5, 3, layout, 1)
        assert _equal(res, want)


def test_world_one_without_callback_or_process_group():
    import torch.distributed as dist
    assert not dist.is_initialized()
    q, g = synthetic.descriptors(100, 4000, 384, seed=9, planted=0.1)
    q, g = q.cuda(), g.cuda()
    for t in (0.5, -np.inf):
        want = similarity.sim_range(q, g[:500], t, index_base=7, index_stride=3)
        got = ddist.sharded_range(q, g[:500], t, 7, index_stride=3)
        assert _equal(got, want)
    empty = ddist.sharded_range(q, g[:0], 0.5, 0)
    assert torch.equal(empty[0].cpu(), torch.zeros(101, dtype=torch.int64)) and empty[1].numel() == 0


def test_shards_smaller_than_the_world():
    """G < world: shard_bounds leaves some ranks empty, and they take part all the same."""
    q, g = synthetic.descriptors(30, 2, 64, seed=3)
    q, g = q.cuda(), g.cuda()
    want = similarity.sim_range(q, g, -np.inf)
    world = 4
    bounds = [ddist.shard_bounds(2, r, world) for r in range(world)]
    assert [hi - lo for lo, hi in bounds].count(0) == 2
    shards = [g[lo:hi] for lo, hi in bounds]
    for me in range(world):
        peers = [Peer(q, shards[r], -np.inf, bounds[r][0], 1) for r in range(world) if r != me]
        got = ddist.sharded_range(q, shards[me], -np.inf, bounds[me][0], allgather=FakeWorld(me, peers), world=world)
        assert _equal(got, want)


# ------------------------------------------------------------------------------------------------------------------
# agreement, through the C entry


def _c_call(q, g, t, base, fake, world, max_pairs, local_cap, stride=1, workspace=True):
    """one dcr_sim_range_sharded call; outputs pre-filled with a sentinel so that 'nothing written' can be checked"""
    lib = _lib.load()
    nq, d = q.shape
    counts = (C.c_int64 * 3)()
    nbytes = lib.dcr_sim_range_sharded_workspace_size(nq, g.shape[0], d, world, local_cap)
    assert nbytes > 0
    ws = torch.empty(nbytes + 256, dtype=torch.uint8, device=CUDA)
    ws_ptr = similarity._aligned_ptr(ws) if workspace else None
    off = torch.full((nq + 1,), -7, dtype=torch.int64, device=CUDA)
    idx = torch.full((max(max_pairs, 1),), -7, dtype=torch.int64, device=CUDA)
    val = torch.full((max(max_pairs, 1),), -7.0, dtype=torch.float32, device=CUDA)
    cb = _lib.ALLGATHER_FN(lambda s, r, n, ctx, st: fake(s, r, n, st))
    rc = lib.dcr_sim_range_sharded(q.data_ptr(), nq, g.data_ptr() if g.shape[0] else None, g.shape[0], d, float(t),
                                   base, stride, world, C.cast(cb, C.c_void_p), None, off.data_ptr(), idx.data_ptr(),
                                   val.data_ptr(), max_pairs, local_cap, counts, ws_ptr, nbytes if workspace else 0,
                                   torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return rc, [int(c) for c in counts], off, idx, val


def _untouched(off, idx, val):
    return bool((off == -7).all() and (idx == -7).all() and (val == -7.0).all())


def _problem():
    q, g = synthetic.descriptors(120, 4000, 256, seed=31, planted=0.2)
    q, g = q.cuda(), g.cuda()
    return q, g, g[:1800].contiguous(), g[1800:].contiguous(), similarity.sim_range(q, g, 0.5)


def test_peer_capacity_status_and_retry():
    q, g, own, other, want = _problem()
    total = int(want[0][-1])
    need = 5_000_000
    fake = FakeWorld(0, [Peer(q, other, 0.5, 1800, 1, status=_lib.ERR_CAPACITY, pairs=0, cand=need)])
    rc, counts, off, idx, val = _c_call(q, own, 0.5, 0, fake, 2, 1 << 20, 1 << 20)
    assert rc == _lib.ERR_CAPACITY and "max_local_pairs" in _lib.last_error()
    assert len(fake.calls) == 1                                          # no second exchange
    own_pairs = int(similarity.sim_range(q, own, 0.5)[0][-1])
    # the peer's search did not finish: its candidates stand for its pairs in the total
    assert counts[0] == 0 and counts[1] == need and counts[2] == own_pairs + need
    assert _untouched(off, idx, val)
    # the retry with the stated needs, the peer now done
    fake = FakeWorld(0, [Peer(q, other, 0.5, 1800, 1)])
    rc, counts2, off, idx, val = _c_call(q, own, 0.5, 0, fake, 2, counts[2], counts[1])
    assert rc == 0 and counts2[0] == total, _lib.last_error()
    assert torch.equal(off, want[0]) and torch.equal(idx[:total], want[1]) and torch.equal(val[:total], want[2])


def test_own_capacities_too_small():
    q, g, own, other, want = _problem()
    total = int(want[0][-1])
    # max_pairs below the global total, here or on the peer: ERR_CAPACITY with the total, then success
    for mine, theirs in ((total - 1, 1 << 30), (1 << 30, total - 1)):
        fake = FakeWorld(0, [Peer(q, other, 0.5, 1800, 1, max_pairs=theirs)])
        rc, counts, off, idx, val = _c_call(q, own, 0.5, 0, fake, 2, mine, 1 << 20)
        assert rc == _lib.ERR_CAPACITY and counts[2] == total and _untouched(off, idx, val)
        assert len(fake.calls) == 1
    fake = FakeWorld(0, [Peer(q, other, 0.5, 1800, 1)])
    rc, counts, off, idx, val = _c_call(q, own, 0.5, 0, fake, 2, total, 1 << 20)
    assert rc == 0 and torch.equal(off, want[0]) and torch.equal(idx, want[1]) and torch.equal(val, want[2])
    # this rank's candidate capacity too small: its search stops after counting, and the retry with counts[1] succeeds
    fake = FakeWorld(0, [Peer(q, other, 0.5, 1800, 1)])
    rc, counts, off, idx, val = _c_call(q, own, 0.5, 0, fake, 2, 1 << 20, 3)
    assert rc == _lib.ERR_CAPACITY and counts[1] >= 3 and counts[2] >= total and _untouched(off, idx, val)
    fake = FakeWorld(0, [Peer(q, other, 0.5, 1800, 1)])
    rc, _, off, idx, val = _c_call(q, own, 0.5, 0, fake, 2, counts[2], counts[1])
    assert rc == 0 and torch.equal(off, want[0]) and torch.equal(idx[:total], want[1])
    # a peer whose receive buffer cannot hold this rank's message: its max_local_pairs fits its own pairs only
    small = Peer(q, g[3800:].contiguous(), 0.5, 3800, 1)
    big = g[:3800].contiguous()
    assert 0 < small.pairs < int(similarity.sim_range(q, big, 0.5)[0][-1])
    fake = FakeWorld(0, [Peer(q, g[3800:].contiguous(), 0.5, 3800, 1, cap=small.pairs)])
    rc, counts, off, idx, val = _c_call(q, big, 0.5, 0, fake, 2, 1 << 20, 1 << 20)
    assert rc == _lib.ERR_CAPACITY and counts[1] > small.pairs and counts[2] == total and _untouched(off, idx, val)
    fake = FakeWorld(0, [Peer(q, g[3800:].contiguous(), 0.5, 3800, 1, cap=counts[1])])
    rc, _, off, idx, val = _c_call(q, big, 0.5, 0, fake, 2, counts[2], counts[1])
    assert rc == 0 and torch.equal(off, want[0]) and torch.equal(idx, want[1]) and torch.equal(val, want[2])


@pytest.mark.parametrize("field,value,match", [
    ("nq", 121, "disagree"), ("d", 512, "disagree"), ("thr", _thr_bits(0.25), "disagree"),
    ("status", -1, "rank 1 failed"), ("magic", 0, "malformed header"),
])
def test_peer_header_errors(field, value, match):
    q, g, own, other, _ = _problem()
    fake = FakeWorld(0, [Peer(q, other, 0.5, 1800, 1, **{field: value})])
    rc, counts, off, idx, val = _c_call(q, own, 0.5, 0, fake, 2, 1 << 20, 1 << 20)
    assert rc != 0 and rc != _lib.ERR_CAPACITY and match in _lib.last_error(), _lib.last_error()
    assert len(fake.calls) == 1 and _untouched(off, idx, val)


def test_overlapping_shards_are_an_error():
    q, g, own, other, _ = _problem()
    for peer in (Peer(q, own, 0.5, 0, 1),                                 # the same shard twice
                 Peer(q, g[1000:2500].contiguous(), 0.5, 1000, 1)):       # a partial overlap
        fake = FakeWorld(0, [peer])
        rc, _, off, idx, val = _c_call(q, own, 0.5, 0, fake, 2, 1 << 20, 1 << 20)
        assert rc == -1 and "same gallery index" in _lib.last_error()
        assert len(fake.calls) == 2 and _untouched(off, idx, val)


def test_local_failure_still_exchanges():
    """A bad argument on this rank (NaN threshold) is reported in the header: the peers learn of it, nothing is
    written, and the callback ran once."""
    q, g, own, other, _ = _problem()
    fake = FakeWorld(0, [Peer(q, other, 0.5, 1800, 1)])
    rc, _, off, idx, val = _c_call(q, own, float("nan"), 0, fake, 2, 1 << 20, 1 << 20)
    assert rc == -1 and "rank 0 failed" in _lib.last_error() and "NaN" in _lib.last_error()
    assert len(fake.calls) == 1 and _untouched(off, idx, val)
    # no workspace at all: the header buffers come from the stream, and the error still goes round
    fake = FakeWorld(1, [Peer(q, other, 0.5, 1800, 1)])
    rc, _, off, idx, val = _c_call(q, own, 0.5, 0, fake, 2, 1 << 20, 1 << 20, workspace=False)
    assert rc == -1 and "rank 1 failed" in _lib.last_error() and "workspace too small" in _lib.last_error()
    assert len(fake.calls) == 1 and _untouched(off, idx, val)
    # a peer's failure reaches this rank the same way (and the Python entry raises on it)
    fake = FakeWorld(0, [Peer(q, other, 0.5, 1800, 1, status=-2)])
    with pytest.raises(_lib.DcrError, match="rank 1 failed"):
        ddist.sharded_range(q, own, 0.5, 0, allgather=fake, world=2)
    assert len(fake.calls) == 1


# ------------------------------------------------------------------------------------------------------------------
# real processes


def _worker(rank, world, backend, port, out_dir):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dev = torch.device("cuda", rank if backend == "nccl" else 0)
    torch.cuda.set_device(dev)
    dist.init_process_group(backend, rank=rank, world_size=world, device_id=dev if backend == "nccl" else None)
    q, g = synthetic.descriptors(700, 9001, 384, seed=41, planted=0.2, noise=0.03)
    q, g = q.to(dev), g.to(dev)
    lo, hi = ddist.shard_bounds(9001, rank, world)
    out = {}
    for name, (qq, t) in {"match": (q, 0.5), "self": (g, 0.5), "dense": (q[:50], -np.inf)}.items():
        o, i, v = ddist.sharded_range(qq, g[lo:hi], t, lo)
        out.update({f"{name}_o": o.cpu().numpy(), f"{name}_i": i.cpu().numpy(), f"{name}_v": v.cpu().numpy()})
    o, i, v = ddist.sharded_range(q, g[rank::world].contiguous(), 0.5, rank, index_stride=world)
    out.update({"inter_o": o.cpu().numpy(), "inter_i": i.cpu().numpy(), "inter_v": v.cpu().numpy()})
    lo1, hi1 = ddist.shard_bounds(1, rank, world)                         # one gallery row: rank 1 holds nothing
    o, i, v = ddist.sharded_range(q, g[lo1:hi1], -np.inf, lo1)
    out.update({"tiny_o": o.cpu().numpy(), "tiny_i": i.cpu().numpy(), "tiny_v": v.cpu().numpy()})
    np.savez(os.path.join(out_dir, f"rank{rank}.npz"), **out)
    dist.barrier()
    dist.destroy_process_group()


def _check_processes(tmp_path, backend, port):
    import torch.multiprocessing as mp
    mp.spawn(_worker, args=(2, backend, port, str(tmp_path)), nprocs=2, join=True)
    q, g = synthetic.descriptors(700, 9001, 384, seed=41, planted=0.2, noise=0.03)
    q, g = q.cuda(), g.cuda()
    want = {"match": similarity.sim_range(q, g, 0.5), "self": similarity.sim_range(g, g, 0.5),
            "dense": similarity.sim_range(q[:50], g, -np.inf), "inter": similarity.sim_range(q, g, 0.5),
            "tiny": similarity.sim_range(q, g[:1], -np.inf)}
    assert int(want["match"][0][-1]) > 700
    for r in range(2):
        got = np.load(os.path.join(tmp_path, f"rank{r}.npz"))
        for name, (o, i, v) in want.items():
            assert np.array_equal(got[f"{name}_o"], o.cpu().numpy()), (r, name)
            assert np.array_equal(got[f"{name}_i"], i.cpu().numpy()), (r, name)
            assert np.array_equal(got[f"{name}_v"].view(np.uint32), v.cpu().numpy().view(np.uint32)), (r, name)


def test_two_processes_on_one_gpu_gloo(tmp_path):
    _check_processes(tmp_path, "gloo", 29400 + os.getpid() % 500)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpus_nccl(tmp_path):
    _check_processes(tmp_path, "nccl", 29950 + os.getpid() % 40)
