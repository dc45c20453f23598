"""GPU: the gallery-sharded threshold search under the cross split score (dcr_sim_range_cross_sharded /
dist.sharded_range(cross=True)) against the one-process cross search, bit for bit.

- Emulated ranks in one process: the test plays the peers.  Their headers and messages are built from the search the
  peer would run on its shard (cross, aligned or dot product), with header word [9] as include/dcr_b200.h documents
  (0, n_parts or -n_parts), and the callback writes them around this rank's own block.
- The agreement on the score: a cross rank never merges with an aligned rank of the same n_parts, a dot-product rank or
  a cross rank of another n_parts; one part is the dot product and agrees with it.
- The capacity protocol and its one retry, determinism, and two real processes over gloo (and NCCL with two GPUs).
"""
import ctypes as C
import os
import struct

import numpy as np
import pytest
import torch

from dcr_b200 import _lib, similarity, synthetic
from dcr_b200 import dist as ddist

pytestmark = pytest.mark.gpu

CUDA = torch.device("cuda")
MAGIC = int.from_bytes(b"DCRRNG1\0", "little")
HEADER_BYTES = 80


def _thr_bits(t):
    return struct.unpack("<I", struct.pack("<f", np.float32(t)))[0]


def _search(q, g, t, c, form, base=0, stride=1):
    """The one-process search of a form: 'cross', 'aligned' (over c parts) or 'dot'."""
    if form == "dot":
        return similarity.sim_range(q, g, t, index_base=base, index_stride=stride)
    return similarity.sim_range_split(q, g, t, c, cross=form == "cross", index_base=base, index_stride=stride)


def _word(form, c):
    """Header word [9] of a form: 0 for the dot product and for one part, n_parts aligned, -n_parts cross."""
    if form == "dot" or c == 1:
        return 0
    return -c if form == "cross" else c


class Peer:
    """A rank played by the test: the message its library would send, from the search of `form` on its shard, and the
    header of each attempt (`first` overrides fields of the first attempt's header only)."""

    def __init__(self, q, shard, t, c, base, stride, form="cross", first=None, **hdr):
        nq, d = q.shape
        if shard.shape[0] > 0:
            off, idx, val = _search(q, shard, t, c, form, base, stride)
        else:
            off = torch.zeros(nq + 1, dtype=torch.int64, device=CUDA)
            idx = torch.zeros(0, dtype=torch.int64, device=CUDA)
            val = torch.zeros(0, dtype=torch.float32, device=CUDA)
        self.pairs = int(off[-1])
        self.payload = torch.cat([off.view(torch.uint8), idx.view(torch.uint8), val.view(torch.uint8)])
        h = dict(magic=MAGIC, status=0, pairs=self.pairs, cand=self.pairs, cap=1 << 20, max_pairs=1 << 30, nq=nq, d=d,
                 thr=_thr_bits(t), score=_word(form, c))
        h.update(hdr)
        self.headers = [self._pack(dict(h, **(first or {}))), self._pack(h)]

    @staticmethod
    def _pack(h):
        return torch.tensor(list(h.values()), dtype=torch.int64, device=CUDA).view(torch.uint8)


class FakeWorld:
    """The all-gather callback of rank `me`: [peers before me | own block | peers after me].  A call of 80 bytes per rank
    is a header exchange (attempt 0, 1, ... in call order); a longer one the message exchange, each padded to
    bytes_per_rank.  Every problem here has nq >= 10, so a message is longer than a header."""

    def __init__(self, me, peers):
        self.me, self.peers, self.calls = me, list(peers), []

    def __call__(self, send, recv, nbytes, stream):
        world = len(self.peers) + 1
        attempt = self.calls.count(HEADER_BYTES)                     # of a header call
        self.calls.append(nbytes)
        out = ddist.device_bytes(recv, nbytes * world, CUDA)
        own = ddist.device_bytes(send, nbytes, CUDA)
        ranks = self.peers[:self.me] + [None] + self.peers[self.me:]
        for r, p in enumerate(ranks):
            dst = out[r * nbytes:(r + 1) * nbytes]
            if p is None:
                dst.copy_(own)
                continue
            src = p.headers[min(attempt, 1)] if nbytes == HEADER_BYTES else p.payload
            assert src.numel() <= nbytes
            dst.fill_(0xA5)                                         # padding is never read
            dst[:src.numel()].copy_(src)
        return 0


def _same_bits(a, b):
    return (torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
            and torch.equal(a[2].contiguous().view(torch.int32), b[2].contiguous().view(torch.int32)))


def _tau(q, g, c):
    """The median over the queries of the third-best cross score: a few pairs per query."""
    v, _ = similarity.sim_topk_split(q, g, 3, c, cross=True)
    return float(v[:, 2].median())


def _shards(g, world, layout):
    """(shards, bases, stride) for contiguous ragged shards with an empty one, or interleaved shards."""
    G = g.shape[0]
    if layout == "interleaved":
        return [g[r::world].contiguous() for r in range(world)], list(range(world)), world
    cuts = [0, G // 3, G // 3, G] if world == 3 else [0, 0, G]      # ragged, one shard empty
    return [g[cuts[r]:cuts[r + 1]].contiguous() for r in range(world)], cuts[:-1], 1


C4 = 4


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("layout", ["contiguous", "interleaved"])
@pytest.mark.parametrize("case", ["match", "all"])
def test_emulated_ranks_equal_one_process(world, layout, case):
    q, g = synthetic.descriptors(130, 2500, 256, seed=world, planted=0.2)
    q, g = q.cuda(), g.cuda()
    if case == "all":
        q, t = q[:40].contiguous(), -np.inf
    else:
        t = _tau(q, g, C4)
    want = similarity.sim_range_split(q, g, t, C4, cross=True)
    pairs = int(want[0][-1])
    assert pairs == 40 * 2500 if case == "all" else pairs > q.shape[0]
    shards, bases, stride = _shards(g, world, layout)
    for me in range(world):                                              # this rank at every position, the empty one too
        fake = FakeWorld(me, [Peer(q, shards[r], t, C4, bases[r], stride) for r in range(world) if r != me])
        res = ddist.sharded_range(q, shards[me], t, bases[me], allgather=fake, world=world, index_stride=stride,
                                  num_chunks=C4, cross=True)
        torch.cuda.synchronize()
        assert len(fake.calls) == 2 and fake.calls[0] == HEADER_BYTES
        assert _same_bits(res, want), (me, layout, case)


def test_world_one_without_callback_or_process_group():
    import torch.distributed as dist
    assert not dist.is_initialized()
    q, g = synthetic.descriptors(100, 4000, 384, seed=9, planted=0.1)
    q, g = q.cuda(), g.cuda()
    shard = g[:500]
    for t in (_tau(q, shard, C4), -np.inf):
        want = similarity.sim_range_split(q, shard, t, C4, cross=True, index_base=7, index_stride=3)
        got = ddist.sharded_range(q, shard, t, 7, index_stride=3, num_chunks=C4, cross=True)
        assert int(want[0][-1]) > 100 and _same_bits(got, want), t
        # one part is the dot product: the bits of the dot-product sharded search
        dot = ddist.sharded_range(q, shard, t, 7, index_stride=3)
        assert _same_bits(ddist.sharded_range(q, shard, t, 7, index_stride=3, cross=True), dot)
        assert _same_bits(dot, similarity.sim_range(q, shard, t, index_base=7, index_stride=3))
    empty = ddist.sharded_range(q, g[:0], 0.5, 0, num_chunks=C4, cross=True)
    assert torch.equal(empty[0].cpu(), torch.zeros(101, dtype=torch.int64)) and empty[1].numel() == 0


def test_one_part_agrees_with_a_dot_product_peer():
    q, g = synthetic.descriptors(60, 1500, 256, seed=4, planted=0.2)
    q, g = q.cuda(), g.cuda()
    want = similarity.sim_range(q, g, 0.5)
    assert int(want[0][-1]) > 0
    fake = FakeWorld(1, [Peer(q, g[:700].contiguous(), 0.5, 1, 0, 1, form="dot")])
    got = ddist.sharded_range(q, g[700:].contiguous(), 0.5, 700, allgather=fake, world=2, num_chunks=1, cross=True)
    assert len(fake.calls) == 2 and _same_bits(got, want)


@pytest.mark.parametrize("mine,theirs,names", [
    (("cross", 4), ("aligned", 4), ("the cross score over 4 parts", "the aligned score over 4 parts")),
    (("aligned", 4), ("cross", 4), ("the aligned score over 4 parts", "the cross score over 4 parts")),
    (("cross", 4), ("dot", 1), ("the cross score over 4 parts", "the dot product")),
    (("cross", 4), ("cross", 8), ("the cross score over 4 parts", "the cross score over 8 parts")),
], ids=["cross-aligned", "aligned-cross", "cross-dot", "cross4-cross8"])
def test_peer_that_disagrees_on_the_score(mine, theirs, names):
    q, g = synthetic.descriptors(50, 1000, 256, seed=5, planted=0.2)
    q, g = q.cuda(), g.cuda()
    own, other = g[:600].contiguous(), g[600:].contiguous()
    for me in (0, 1):
        fake = FakeWorld(me, [Peer(q, other, 0.3, theirs[1], 600, 1, form=theirs[0])])
        with pytest.raises(_lib.DcrError, match="disagree") as e:
            ddist.sharded_range(q, own, 0.3, 0, allgather=fake, world=2, num_chunks=mine[1], cross=mine[0] == "cross")
        assert len(fake.calls) == 1
        assert all(n in str(e.value) for n in names), str(e.value)


def _c_call(q, g, t, base, fake, world, max_pairs, local_cap, c=C4):
    """one dcr_sim_range_cross_sharded call; outputs pre-filled with a sentinel so that 'nothing written' can be checked"""
    lib = _lib.load()
    nq, d = q.shape
    counts = (C.c_int64 * 3)()
    nbytes = lib.dcr_sim_range_cross_sharded_workspace_size(nq, g.shape[0], d, c, world, local_cap)
    assert nbytes > 0
    ws = torch.empty(nbytes + 256, dtype=torch.uint8, device=CUDA)
    off = torch.full((nq + 1,), -7, dtype=torch.int64, device=CUDA)
    idx = torch.full((max(max_pairs, 1),), -7, dtype=torch.int64, device=CUDA)
    val = torch.full((max(max_pairs, 1),), -7.0, dtype=torch.float32, device=CUDA)
    cb = _lib.ALLGATHER_FN(lambda s, r, n, ctx, st: fake(s, r, n, st))
    rc = lib.dcr_sim_range_cross_sharded(q.data_ptr(), nq, g.data_ptr(), g.shape[0], d, c, float(t), base, 1, world,
                                         C.cast(cb, C.c_void_p), None, off.data_ptr(), idx.data_ptr(), val.data_ptr(),
                                         max_pairs, local_cap, counts, similarity._aligned_ptr(ws), nbytes,
                                         torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return rc, [int(x) for x in counts], off, idx, val


def test_peer_capacity_status_and_retry():
    q, g = synthetic.descriptors(120, 4000, 256, seed=31, planted=0.2)
    q, g = q.cuda(), g.cuda()
    own, other = g[:1800].contiguous(), g[1800:].contiguous()
    t = _tau(q, g, C4)
    want = similarity.sim_range_split(q, g, t, C4, cross=True)
    own_pairs = int(similarity.sim_range_split(q, own, t, C4, cross=True)[0][-1])
    need = 2_000_000
    short = dict(status=_lib.ERR_CAPACITY, pairs=0, cand=need)
    # through the C entry: every rank learns the need, nothing is written, and there is no second exchange
    fake = FakeWorld(0, [Peer(q, other, t, C4, 1800, 1, **short)])
    rc, counts, off, idx, val = _c_call(q, own, t, 0, fake, 2, 1 << 20, 1 << 20)
    assert rc == _lib.ERR_CAPACITY and "max_local_pairs" in _lib.last_error()
    assert "sim_range_cross_sharded" in _lib.last_error()
    assert counts == [0, need, own_pairs + need] and len(fake.calls) == 1
    assert bool((off == -7).all() and (idx == -7).all() and (val == -7.0).all())
    # through sharded_range: the peer falls short on the first attempt only, and the one retry with the needs succeeds
    for me in (0, 1):
        fake = FakeWorld(me, [Peer(q, other, t, C4, 1800, 1, first=short)])
        got = ddist.sharded_range(q, own, t, 0, allgather=fake, world=2, num_chunks=C4, cross=True)
        assert fake.calls[:2] == [HEADER_BYTES, HEADER_BYTES] and len(fake.calls) == 3
        assert _same_bits(got, want)


def test_determinism():
    q, g = synthetic.descriptors(90, 3000, 384, seed=13, planted=0.2)
    q, g = q.cuda(), g.cuda()
    c = 6                                                                # parts of 64
    v, _ = similarity.sim_topk_split(q, g, 3, c, cross=True)
    t = float(v[:, 2].median())
    shards, bases, stride = _shards(g, 2, "interleaved")
    runs = []
    for _ in range(2):
        fake = FakeWorld(0, [Peer(q, shards[1], t, c, bases[1], stride)])
        runs.append(ddist.sharded_range(q, shards[0], t, bases[0], allgather=fake, world=2, index_stride=stride,
                                        num_chunks=c, cross=True))
    assert int(runs[0][0][-1]) > 90 and _same_bits(runs[0], runs[1])
    assert _same_bits(runs[0], similarity.sim_range_split(q, g, t, c, cross=True))


# ------------------------------------------------------------------------------------------------------------------
# real processes

_NQ, _NG, _D = 60, 1501, 256


def _data(dev):
    q, g = synthetic.descriptors(_NQ, _NG, _D, seed=17, planted=0.1)
    return q.to(dev), g.to(dev)


def _worker(rank, world, backend, port, tau, out_dir):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dev = torch.device("cuda", rank if backend == "nccl" else 0)
    torch.cuda.set_device(dev)
    dist.init_process_group(backend, rank=rank, world_size=world, device_id=dev if backend == "nccl" else None)
    q, g = _data(dev)
    lo, hi = ddist.shard_bounds(_NG, rank, world)
    out = {}
    for name, t in [("match", tau), ("dense", -np.inf)]:
        o, i, v = ddist.sharded_range(q, g[lo:hi], t, lo, num_chunks=C4, cross=True)
        out.update({f"{name}_o": o.cpu().numpy(), f"{name}_i": i.cpu().numpy(), f"{name}_v": v.cpu().numpy()})
    o, i, v = ddist.sharded_range(q, g[rank::world].contiguous(), tau, rank, index_stride=world, num_chunks=C4, cross=True)
    out.update({"inter_o": o.cpu().numpy(), "inter_i": i.cpu().numpy(), "inter_v": v.cpu().numpy()})
    np.savez(os.path.join(out_dir, f"rank{rank}.npz"), **out)
    dist.barrier()
    dist.destroy_process_group()


def _check_processes(tmp_path, backend, port):
    import torch.multiprocessing as mp
    q, g = _data(CUDA)
    tau = _tau(q, g, C4)
    mp.spawn(_worker, args=(2, backend, port, tau, str(tmp_path)), nprocs=2, join=True)
    want = {"match": similarity.sim_range_split(q, g, tau, C4, cross=True),
            "dense": similarity.sim_range_split(q, g, -np.inf, C4, cross=True)}
    want["inter"] = want["match"]
    assert int(want["match"][0][-1]) > _NQ and int(want["dense"][0][-1]) == _NQ * _NG
    for r in range(2):
        got = np.load(os.path.join(tmp_path, f"rank{r}.npz"))
        for name, (o, i, v) in want.items():
            assert np.array_equal(got[f"{name}_o"], o.cpu().numpy()), (r, name)
            assert np.array_equal(got[f"{name}_i"], i.cpu().numpy()), (r, name)
            assert np.array_equal(got[f"{name}_v"].view(np.uint32), v.cpu().numpy().view(np.uint32)), (r, name)


def test_two_processes_on_one_gpu_gloo(tmp_path):
    _check_processes(tmp_path, "gloo", 27400 + os.getpid() % 500)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpus_nccl(tmp_path):
    _check_processes(tmp_path, "nccl", 27950 + os.getpid() % 40)
