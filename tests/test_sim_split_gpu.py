"""GPU parity of dcr_sim_topk_split, the fused top-k under the split score (max over the descriptor parts of the per-part
dot products): against the fp64 oracle, bit for bit against dcr_split_rescore, on ties, per-token-like data, a part at
its bf16 error bound, argument errors, and gallery-sharded across two processes."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from dcr_b200 import _lib, similarity, synthetic
from dcr_b200 import dist as ddist
from oracle import similarity as osim
from tests import sim_bound_cases as sbc

pytestmark = pytest.mark.gpu


def _split(q, g, k, c, **kw):
    v, i = similarity.sim_topk_split(q.cuda(), g.cuda(), k, c, **kw)
    torch.cuda.synchronize()
    return v.cpu().numpy(), i.cpu().numpy(), similarity.sim_topk_stats()


def _rescore_every_row(q, g, k, c):
    """dcr_split_rescore with every gallery row as a candidate: the exact split score of all pairs, then top-k."""
    lib = _lib.load()
    qd, gd = q.cuda().contiguous(), g.cuda().contiguous()
    nq, d = qd.shape
    ng = gd.shape[0]
    cand = torch.arange(ng, dtype=torch.int64, device="cuda").repeat(nq, 1).contiguous()
    out_s = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    out_i = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    rc = lib.dcr_split_rescore(qd.data_ptr(), gd.data_ptr(), nq, d, c, 0, cand.data_ptr(), ng, k, out_s.data_ptr(),
                               out_i.data_ptr(), torch.cuda.current_stream().cuda_stream)
    _lib.check(rc, "dcr_split_rescore")
    torch.cuda.synchronize()
    return out_s.cpu().numpy(), out_i.cpu().numpy()


def _check(q, g, k, c):
    v, i, st = _split(q, g, k, c)
    ov, oi = osim.sim_topk_split(q.numpy(), g.numpy(), k, c)
    bad = np.nonzero((i != oi).any(axis=1))[0]
    assert bad.size == 0, f"{bad.size} query rows differ, first {bad[:5]}: got {i[bad[:3]]} want {oi[bad[:3]]}"
    np.testing.assert_allclose(v, ov, rtol=0, atol=1e-6)
    if g.shape[0] <= 4096:
        rv, ri = _rescore_every_row(q, g, k, c)
        assert np.array_equal(i, ri)
        assert np.array_equal(v.view(np.uint32), rv.view(np.uint32))
    return st


@pytest.mark.parametrize("nq,ng,d,c,k", [
    (64, 3000, 512, 4, 10),
    (33, 1000, 96, 3, 1),             # parts of 32: below one k-block
    (20, 500, 512, 32, 5),            # parts of 16
    (6, 300, 197 * 64, 197, 5),       # ViT token count, one k-block per part
    (5, 700, 785 * 16, 785, 10),      # C * k = 7850 candidates: beyond the per-part composition
    (3, 2048, 197 * 384, 197, 16),    # ViT-S/16 tokens, k = 16
    (5, 16, 128, 2, 16),              # k = ng
])
def test_parity(nq, ng, d, c, k):
    q, g = synthetic.descriptors(nq, ng, d, seed=nq + ng + c, planted=0.05)
    _check(q, g, k, c)


def test_exact_duplicate_rows_lowest_index_wins():
    q, g = synthetic.descriptors(40, 1500, 256, seed=3, planted=0.05)
    g[100:110] = g[7]
    g[900] = q[3]
    g[300] = q[3]
    _check(q, g, 10, 4)


def test_row_equal_only_in_its_best_part():
    """Row b copies only the part in which row a scores best for query 0 (its other parts are zero): both have the same
    split score, and the lower index of the two comes first."""
    c, k = 8, 5
    q, g = synthetic.descriptors(16, 1200, 512, seed=11, planted=0.05)
    p = 512 // c
    _, oi = osim.sim_topk_split(q.numpy(), g.numpy(), k, c)
    a = int(oi[0, 0])
    parts = (q[0].double().view(c, p) * g[a].double().view(c, p)).sum(1)
    best = int(parts.argmax())
    assert parts[best] > 0
    for b in (a - 1 if a > 0 else a + 1, 1199 if a != 1199 else 0):
        g2 = g.clone()
        g2[b] = 0
        g2[b, best * p:(best + 1) * p] = g[a, best * p:(best + 1) * p]
        v, i, _ = _split(q, g2, k, c)
        assert set(i[0, :2].tolist()) == {a, b} and i[0, 0] == min(a, b) and v[0, 0] == v[0, 1]
        _check(q, g2, k, c)


def test_per_token_data_never_needs_the_brute_force_path():
    """Every part is a shared direction plus noise of the same size, then the whole row is normalised (per-token ViT
    descriptors look like this): the part scores are about 1/C of a row score, and so must be the bound."""
    c, p, nq, ng = 197, 64, 24, 2000
    gen = torch.Generator().manual_seed(17)
    mean = torch.nn.functional.normalize(torch.randn(c, p, generator=gen), dim=1)

    def rows(n):
        x = mean + torch.nn.functional.normalize(torch.randn(n, c, p, generator=gen), dim=2)
        return torch.nn.functional.normalize(x.reshape(n, c * p), dim=1).contiguous()

    q, g = rows(nq), rows(ng)
    st = _check(q, g, 10, c)
    assert st["n_flagged"] == 0, st


def test_a_part_at_its_bf16_bound():
    """Part 0 holds an instance whose bf16 error reaches the bound with 40 competitors in one segment (more than either
    pass keeps); the other parts score far lower.  The certificate fails, the brute-force path answers, and the result is
    the oracle's."""
    case = sbc.build(64, 40, centred=False)
    nq, ng = case.q.shape[0], case.g.shape[0]
    rng = np.random.default_rng(5)
    c, p = 4, 64
    q = np.concatenate([case.q, 0.01 * rng.standard_normal((nq, (c - 1) * p))], axis=1).astype(np.float32)
    g = np.concatenate([case.g, 0.01 * rng.standard_normal((ng, (c - 1) * p))], axis=1).astype(np.float32)
    st = _check(torch.from_numpy(q), torch.from_numpy(g), 10, c)
    assert st["n_flagged"] > 0, st


def test_one_part_gives_the_bits_of_sim_topk():
    q, g = synthetic.descriptors(100, 3000, 384, seed=2)
    v, i, _ = _split(q, g, 10, 1)
    w, j = similarity.sim_topk(q.cuda(), g.cuda(), 10)
    assert np.array_equal(i, j.cpu().numpy())
    assert np.array_equal(v.view(np.uint32), w.cpu().numpy().view(np.uint32))


def test_index_base_and_stride():
    q, g = synthetic.descriptors(30, 800, 256, seed=4)
    v, i, _ = _split(q, g, 7, 4)
    w, j, _ = _split(q, g, 7, 4, index_base=5000, index_stride=3)
    assert np.array_equal(j, 5000 + 3 * i)
    assert np.array_equal(v.view(np.uint32), w.view(np.uint32))


def test_argument_errors_are_refused_with_a_message():
    q, g = synthetic.descriptors(4, 40, 64, seed=1)
    qc, gc = q.cuda(), g.cuda()
    for args, match in [((qc, gc, 3, 3), "parts"),                    # 64 does not split into 3
                        ((qc[:, :60].contiguous(), gc[:, :60].contiguous(), 3, 10), "multiple of 4"),   # parts of 6
                        ((qc, gc, 0, 2), "k="),
                        ((qc, gc, 17, 2), "k="),
                        ((qc, gc[:5].contiguous(), 6, 2), "gallery size"),
                        ((qc, gc, 3, 0), "n_parts"),
                        ((qc, gc[:, :32].contiguous(), 3, 2), "dims differ"),
                        ((q, g, 3, 2), "CUDA")]:
        with pytest.raises(_lib.DcrError, match=match):
            similarity.sim_topk_split(*args)
    long_q = torch.zeros(2, 2 * 8196, device="cuda")
    with pytest.raises(_lib.DcrError, match="8192"):
        similarity.sim_topk_split(long_q, long_q, 1, 2)


# ------------------------------------------------------------------------------------------------------------------
# gallery-sharded across real processes

_NQ, _NG, _D, _C = 45, 1301, 256, 4


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
    for name, ng, k, cross in [("aligned", _NG, 10, False), ("cross", _NG, 3, True), ("small", 13, 10, False),
                               ("small_cross", 13, 8, True)]:
        lo, hi = ddist.shard_bounds(ng, rank, world)
        s, i = ddist.sharded_topk(q[qlo:qhi], g[lo:hi], k, lo, ddist.split_local_topk(_C, cross), ddist.cuda_merge,
                                  query_sizes=q_sizes)
        out[f"{name}_s"], out[f"{name}_i"] = s.cpu().numpy(), i.cpu().numpy()
    np.savez(os.path.join(out_dir, f"rank{rank}.npz"), **out)
    dist.barrier()
    dist.destroy_process_group()


def test_two_processes_on_one_gpu_gloo(tmp_path):
    import torch.multiprocessing as mp
    mp.spawn(_worker, args=(2, 29900 + os.getpid() % 500, str(tmp_path)), nprocs=2, join=True)
    q, g = synthetic.descriptors(_NQ, _NG, _D, seed=8, planted=0.1)
    q, g = q.cuda(), g.cuda()
    assert ddist.shard_bounds(_NG, 0, 2) != (0, _NG // 2)        # ragged shards
    want = {"aligned": similarity.sim_topk_split(q, g, 10, _C),
            "cross": similarity.sim_topk_split(q, g, 3, _C, cross=True),
            "small": similarity.sim_topk_split(q, g[:13].contiguous(), 10, _C),     # shards of 7 and 6 rows < k
            "small_cross": similarity.sim_topk_split(q, g[:13].contiguous(), 8, _C, cross=True)}
    for r in range(2):
        got = np.load(os.path.join(tmp_path, f"rank{r}.npz"))
        for name, (s, i) in want.items():
            assert np.array_equal(got[f"{name}_i"], i.cpu().numpy()), (r, name)
            assert np.array_equal(got[f"{name}_s"].view(np.uint32), s.cpu().numpy().view(np.uint32)), (r, name)
