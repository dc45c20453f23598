"""GPU: the threshold search (dcr_sim_range) against the fp64 oracle -- offsets and indices exact, scores to fp32
rounding -- and against dcr_sim_topk, whose scores it must reproduce bit for bit."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from dcr_b200 import _lib, similarity, synthetic
from tests import sim_range_oracle as orange

pytestmark = pytest.mark.gpu


def _run(q, g, t, **kw):
    off, idx, val = similarity.sim_range(q.cuda(), g.cuda(), t, **kw)
    torch.cuda.synchronize()
    return off.cpu().numpy(), idx.cpu().numpy(), val.cpu().numpy()


def _check(q, g, t, rows=None):
    off, idx, val = _run(q, g, t)
    assert off[0] == 0 and off[-1] == idx.size == val.size and np.all(np.diff(off) >= 0)
    if rows is None:
        ooff, oidx, oval = orange.sim_range(q.numpy(), g.numpy(), t)
        assert np.array_equal(off, ooff)
        assert np.array_equal(idx, oidx)
        np.testing.assert_allclose(val, oval, rtol=0, atol=1.2e-7)
    else:
        ooff, oidx, oval = orange.sim_range(q.numpy()[rows], g.numpy(), t)
        for n, r in enumerate(rows):
            assert np.array_equal(idx[off[r]:off[r + 1]], oidx[ooff[n]:ooff[n + 1]]), r
            np.testing.assert_allclose(val[off[r]:off[r + 1]], oval[ooff[n]:ooff[n + 1]], rtol=0, atol=1.2e-7)
    return off, idx, val


def _quantile_threshold(q, g, per_row=30):
    """a score such that a query has about `per_row` results (the oracle's scores of a few rows)"""
    s = orange.dense_scores(q.numpy()[:64], g.numpy())
    return np.float32(np.quantile(s, max(0.0, 1.0 - per_row / g.shape[0])))


@pytest.mark.parametrize("nq,ng,d", [
    (256, 1000, 512), (1, 16, 64), (7, 300, 100), (130, 257, 384), (513, 4097, 512), (300, 20000, 512),
    (2000, 3000, 256), (300, 5000, 1024), (260, 3000, 768), (40, 700, 2048), (20, 900, 8192),
])
def test_parity_synthetic(nq, ng, d):
    """the shapes of the sim_topk parity grid (d = 64 .. 2048, d = 100, the streamed query tile at d > 512, ragged
    shapes) plus d = 8192"""
    q, g = synthetic.descriptors(nq, ng, d, seed=nq + ng)
    t = _quantile_threshold(q, g)
    off, _, _ = _check(q, g, t)
    assert off[-1] > 0


@pytest.mark.parametrize("nq,ng,d,k", [(300, 20000, 512, 10), (513, 4097, 384, 5), (100, 3000, 1024, 1)])
def test_agrees_with_sim_topk(nq, ng, d, k):
    """For every row with at least k results, its top-k by (score desc, index asc) is sim_topk's, scores bitwise."""
    q, g = synthetic.descriptors(nq, ng, d, seed=3 + d)
    g[11] = g[4]                                                   # an exact tie
    off, idx, val = _run(q, g, _quantile_threshold(q, g, per_row=40))
    tv, ti = similarity.sim_topk(q.cuda(), g.cuda(), k)
    tv, ti = tv.cpu().numpy(), ti.cpu().numpy()
    checked = 0
    for r in range(nq):
        i, v = idx[off[r]:off[r + 1]], val[off[r]:off[r + 1]]
        if i.size < k:
            continue
        order = np.lexsort((i, -v.astype(np.float64)))[:k]
        assert np.array_equal(i[order], ti[r]), r
        assert torch.equal(torch.from_numpy(v[order]), torch.from_numpy(tv[r])), r
        checked += 1
    assert checked > nq // 2


def test_edge_thresholds():
    q, g = synthetic.descriptors(50, 300, 128, seed=4)
    off, idx, val = _check(q, g, -np.inf)
    assert off[-1] == 50 * 300
    dense = orange.dense_scores(q.numpy(), g.numpy())
    np.testing.assert_allclose(val.reshape(50, 300), dense, rtol=0, atol=1.2e-7)
    off, idx, val = _run(q, g, np.inf)
    assert idx.size == 0 and np.all(off == 0)


def test_inclusive_boundary():
    q, g = synthetic.descriptors(64, 2000, 256, seed=6)
    off, idx, val = _run(q, g, 0.3)
    r = int(np.argmax(np.diff(off)))
    s = val[off[r]:off[r + 1]].min()
    j = idx[off[r]:off[r + 1]][np.argmin(val[off[r]:off[r + 1]])]
    o1, i1, _ = _run(q[r:r + 1], g, s)
    assert j in i1[o1[0]:o1[1]]
    o2, i2, _ = _run(q[r:r + 1], g, np.nextafter(np.float32(s), np.float32(np.inf)))
    assert j not in i2[o2[0]:o2[1]]
    # 3000 identical gallery rows, threshold = their score: all of them
    g3 = q[5:6].repeat(3000, 1).contiguous()
    t = _run(q[:1], g3[:1], -np.inf)[2][0]                        # their score, as the library computes it
    o3, i3, v3 = _run(q[:1], g3, t)
    assert o3[-1] == 3000 and np.array_equal(i3, np.arange(3000)) and np.all(v3 == t)


def test_centring_paths():
    """a large common offset (query centring switched on) and unnormalised data with negative scores"""
    gen = torch.Generator().manual_seed(21)
    common = torch.randn(1, 512, generator=gen)
    q = torch.nn.functional.normalize(common + 0.05 * torch.randn(300, 512, generator=gen), dim=1)
    g = torch.nn.functional.normalize(common + 0.05 * torch.randn(8000, 512, generator=gen), dim=1)
    _check(q, g, _quantile_threshold(q, g, per_row=20))
    q2 = torch.randn(200, 128, generator=gen).abs() * 3
    g2 = -torch.rand(5000, 128, generator=gen)
    t = _quantile_threshold(q2, g2, per_row=50)
    assert t < 0
    _check(q2, g2, t)


def test_capacity_through_the_c_abi():
    lib = _lib.load()
    q, g = synthetic.descriptors(100, 3000, 256, seed=8)
    t = float(_quantile_threshold(q, g, per_row=50))
    qd, gd = q.cuda(), g.cuda()
    off, idx, val = similarity.sim_range(qd, gd, t)
    counts = (C.c_int64 * 2)()
    st = torch.cuda.current_stream().cuda_stream

    def call(cap):
        nbytes = lib.dcr_sim_range_workspace_size(100, 3000, 256, cap)
        ws = torch.empty(nbytes + 256, dtype=torch.uint8, device="cuda")
        o = torch.empty(101, dtype=torch.int64, device="cuda")
        i = torch.empty(max(cap, 1), dtype=torch.int64, device="cuda")
        v = torch.empty(max(cap, 1), dtype=torch.float32, device="cuda")
        rc = lib.dcr_sim_range(qd.data_ptr(), 100, gd.data_ptr(), 3000, 256, t, 0, 1, o.data_ptr(), i.data_ptr(),
                               v.data_ptr(), cap, counts, similarity._aligned_ptr(ws), nbytes, st)
        return rc, o, i, v

    rc, *_ = call(10)
    assert rc == _lib.ERR_CAPACITY and counts[1] >= idx.numel() and "max_pairs" in _lib.last_error()
    need = int(counts[1])
    rc, o, i, v = call(need)
    assert rc == 0 and counts[0] == idx.numel() and counts[1] == need
    n = int(counts[0])
    assert torch.equal(o, off) and torch.equal(i[:n], idx) and torch.equal(v[:n], val)
    rc, o2, i2, v2 = call(need + 12345)                   # another capacity, another workspace size: same bits
    assert rc == 0 and torch.equal(o2, off) and torch.equal(i2[:n], idx) and torch.equal(v2[:n], val)


def test_determinism_and_index_mapping():
    q, g = synthetic.descriptors(700, 9000, 512, seed=10)
    t = _quantile_threshold(q, g, per_row=100)
    a = _run(q, g, t)
    b = _run(q, g, t)
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
    off, idx, val = _run(q, g, t, index_base=7, index_stride=3)
    assert np.array_equal(off, a[0]) and np.array_equal(idx, 7 + 3 * a[1]) and np.array_equal(val, a[2])


def test_scale_and_self_join():
    q, g = synthetic.descriptors(10000, 100000, 512, seed=2)
    rows = np.sort(np.random.default_rng(0).choice(10000, 256, replace=False))
    _check(q, g, 0.5, rows=rows)
    off, idx, val = _run(g[:20000], g[:20000], 0.5)
    for r in range(20000):
        assert r in idx[off[r]:off[r + 1]]


def test_argument_errors():
    q, g = synthetic.descriptors(4, 64, 64)
    with pytest.raises(_lib.DcrError):
        similarity.sim_range(q, g.cuda(), 0.5)                      # CPU tensor
    with pytest.raises(_lib.DcrError):
        similarity.sim_range(q.cuda(), g[:, :32].contiguous().cuda(), 0.5)   # dims differ
    with pytest.raises(_lib.DcrError):
        similarity.sim_range(q.cuda(), g.cuda(), float("nan"))


def test_cli_matches_end_to_end(tmp_path, monkeypatch):
    """matches.pth / matches_wtrain.pth equal sim_range on the CLI's own features; topk.pth and stats.json do not change."""
    from dcr_b200 import cli, data, retrieval
    from oracle import models as om
    from tests.test_cli_gpu import _write_images
    monkeypatch.chdir(tmp_path)
    q_dir, v_dir = str(tmp_path / "runs" / "exp" / "generations"), str(tmp_path / "train")
    _write_images(q_dir, 12, 1)
    _write_images(v_dir, 30, 2)
    wpath = str(tmp_path / "sscd.pt")
    torch.save(om.make_sscd_state_dict(7), wpath)
    common = ["--query_dir", q_dir, "--val_dir", v_dir, "--pt_style", "sscd", "--arch", "resnet50", "--weights", wpath,
              "--precision", "parity", "--topk", "5"]
    save = os.path.join("ret_plots", "runs", "exp", "generations", "images", "sscd_resnet50_dotproduct")
    assert cli.main(common) == 0
    topk0 = torch.load(os.path.join(save, "topk.pth"))
    stats0 = open(os.path.join(save, "stats.json")).read()
    assert not os.path.exists(os.path.join(save, "matches.pth"))
    assert cli.main(common + ["--sim_threshold=-inf"]) == 0
    topk1 = torch.load(os.path.join(save, "topk.pth"))
    assert torch.equal(topk0["indices"], topk1["indices"]) and torch.equal(topk0["values"], topk1["values"])
    assert open(os.path.join(save, "stats.json")).read() == stats0
    m = torch.load(os.path.join(save, "matches.pth"))
    mw = torch.load(os.path.join(save, "matches_wtrain.pth"))
    assert m["size"] == (12, 30) and mw["size"] == (30, 30) and m["threshold"] == -np.inf
    # the same features the command line computed
    args = cli.build_parser().parse_args(common)
    net = cli.build_model(args)
    qf = similarity.l2_normalize_(retrieval.extract_features(net, data.load_files_u8(data.list_images(q_dir), workers=1)))
    vf = similarity.l2_normalize_(retrieval.extract_features(net, data.load_files_u8(data.list_images(v_dir), workers=1)))
    for d, (qq, gg) in ((m, (qf, vf)), (mw, (vf, vf))):
        off, idx, val = similarity.sim_range(qq, gg, -np.inf)
        assert torch.equal(d["crow_indices"], off.cpu()) and torch.equal(d["col_indices"], idx.cpu())
        assert torch.equal(d["values"], val.cpu())
    dense = torch.sparse_csr_tensor(m["crow_indices"], m["col_indices"], m["values"], size=m["size"]).to_dense()
    assert torch.equal(dense.topk(5, dim=1).values, topk1["values"])
    assert torch.equal(torch.diagonal(torch.sparse_csr_tensor(mw["crow_indices"], mw["col_indices"], mw["values"],
                                                              size=mw["size"]).to_dense()) > 0.999, torch.ones(30, dtype=torch.bool))
