"""Improved precision & recall (metrics/ipr.py): oracle vs the reference's own functions (golden), CUDA path vs oracle."""
import os

import numpy as np
import pytest
import torch

from oracle import ipr as oipr

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _sets(seed=0):
    rng = np.random.default_rng(900 + seed)
    ref = (rng.standard_normal((300, 64)) * 3 + 1).astype(np.float32)
    sub = (rng.standard_normal((200, 64)) * 3.3 + 1.2).astype(np.float32)
    return ref, sub


def test_ipr_oracle_matches_reference_golden():
    g = np.load(os.path.join(GOLD, "ipr_seed0.npz"))
    ref, sub = _sets()
    r_ref = oipr.distances2radii(oipr.pairwise_distances(ref), 3)
    r_sub = oipr.distances2radii(oipr.pairwise_distances(sub), 3)
    np.testing.assert_allclose(r_ref, g["radii_ref"], rtol=0, atol=1e-12)
    np.testing.assert_allclose(r_sub, g["radii_sub"], rtol=0, atol=1e-12)
    assert oipr.compute_metric(ref, r_ref, sub) == float(g["precision"])
    assert oipr.compute_metric(sub, r_sub, ref) == float(g["recall"])
    real = [oipr.realism(ref, r_ref, sub[i:i + 1]) for i in range(8)]
    np.testing.assert_allclose(real, g["realism"], rtol=1e-12)


@pytest.mark.gpu
def test_ipr_cuda_metric_matches_reference_golden():
    from dcr_b200 import ipr
    g = np.load(os.path.join(GOLD, "ipr_seed0.npz"))
    ref, sub = _sets()
    r_ref, r_sub = ipr.kth_nn_radii(ref, 3), ipr.kth_nn_radii(sub, 3)
    np.testing.assert_allclose(r_ref, g["radii_ref"], rtol=0, atol=1e-9)
    np.testing.assert_allclose(r_sub, g["radii_sub"], rtol=0, atol=1e-9)
    assert ipr.compute_metric(ipr.Manifold(ref, r_ref), sub) == float(g["precision"])
    assert ipr.compute_metric(ipr.Manifold(sub, r_sub), ref) == float(g["recall"])
    real = [ipr.realism(ipr.Manifold(ref, r_ref), sub[i:i + 1]) for i in range(8)]
    # the reference takes these norms in float32 (numpy float32 inputs, ipr.py:256-258); here they are float64
    np.testing.assert_allclose(real, g["realism"], rtol=1e-6)


@pytest.mark.gpu
def test_ipr_cuda_metric_at_vgg_dim():
    """4096-d features (the real fc2 width), 3000 x 2000 rows, against the numpy oracle."""
    from dcr_b200 import ipr
    rng = np.random.default_rng(5)
    base = np.abs(rng.standard_normal((1, 4096))).astype(np.float32) * 2          # ReLU-network-like common offset
    ref = (base + np.abs(rng.standard_normal((3000, 4096))) * 1.5).astype(np.float32)
    sub = (base + np.abs(rng.standard_normal((2000, 4096))) * 1.6).astype(np.float32)
    r_ref = ipr.kth_nn_radii(ref, 3)
    o_ref = oipr.distances2radii(oipr.pairwise_distances(ref), 3)
    np.testing.assert_allclose(r_ref, o_ref, rtol=1e-10, atol=1e-9)
    got = ipr.compute_metric(ipr.Manifold(ref, r_ref), sub)
    want = oipr.compute_metric(ref, o_ref, sub)
    assert abs(got - want) < 1e-12, (got, want)


@pytest.mark.gpu
def test_vgg16_fc2_features_match_torchvision_module():
    from dcr_b200 import ipr, nets, synthetic
    sd = oipr.make_vgg16_state_dict(0)
    img = synthetic.images(3, seed=61, size=224)
    mean, std = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
    x = (img.permute(0, 3, 1, 2).float().div(255.0) - torch.tensor(mean).view(1, 3, 1, 1)) / torch.tensor(std).view(1, 3, 1, 1)
    ref = oipr.vgg16_fc2(sd, x)
    net = nets.build_vgg16_fc2(sd, max_batch=2, precision="exact")
    got = net(img.cuda()).cpu()
    assert (got - ref).abs().max().item() < 2e-5 * max(1.0, ref.abs().max().item())
    assert torch.equal(net(x.cuda()).cpu(), got)                     # the float32 NCHW entry, same kernels
    fast = nets.build_vgg16_fc2(sd, max_batch=4, precision="fast")
    gq = fast(img.cuda()).cpu()
    cos = torch.nn.functional.cosine_similarity(gq, ref, dim=1).min().item()
    assert cos > 0.999, cos
    # the IPR object end to end on tensors (uint8 path), against oracle features of the same network
    obj = ipr.IPR(batch_size=2, k=1, model=net)
    man = obj.compute_manifold(img)
    np.testing.assert_allclose(man.radii, oipr.distances2radii(oipr.pairwise_distances(man.features), 1), rtol=1e-9)


# ---- replication-shaped sets: clusters of near copies and groups of exact copies ----------------------------------------
# The data IPR is used on here: generated images that replicate training images have features within a hair of each other.
# Neighbours then sit far closer together than any float32 rounding of a float64 quantity, so the nearest-neighbour
# ranking has to be the float64 ranking of the features themselves.

K = 3


def _replicated(n, d, offset, jitter, clusters=(K + 1, K + 4, 25), dups=(K, K + 1, 20), seed=0):
    """n VGG-like rows (non-negative, a common offset of `offset` x ~2 per component), plus for every size in `clusters` a
    cluster of that many copies of one row jittered by N(0, jitter^2) per component, plus for every size in `dups` a group
    of that many identical rows.  Rows shuffled, float32."""
    rng = np.random.default_rng(seed)
    base = np.abs(rng.standard_normal((1, d))) * 2 * offset
    x = base + np.abs(rng.standard_normal((n, d))) * 1.5
    parts = [x]
    for j, m in enumerate(clusters):
        parts.append(x[j] + jitter * rng.standard_normal((m, d)))
    for j, m in enumerate(dups):
        parts.append(np.repeat(x[len(clusters) + j][None], m - 1, axis=0))   # the original row is the m-th copy
    out = np.vstack(parts).astype(np.float32)
    return out[rng.permutation(len(out))]


def _r2_tol(*sets):
    """float64 rounding of ||x||^2 - 2 x.y + ||y||^2 at the largest norm of the sets."""
    return 2.0 ** -46 * max(float((s.astype(np.float64) ** 2).sum(1).max()) for s in sets)


def _inside(ref, radii, sub):
    """The reference's per-subject answer (metrics/ipr.py:238-240) and the margin min_j |d^2 - r_j^2| in float64.
    `sub` keeps its dtype in the distances, as in the reference."""
    dist = oipr.pairwise_distances(ref, sub)
    d2 = oipr.pairwise_distances(ref, sub.astype(np.float64)) ** 2
    return (dist < radii[:, None]).any(0), np.abs(d2 - radii[:, None] ** 2).min(0)


def _fp64_ranked(q, g, kk):
    """What sim_topk returns for these operands: the kk largest float64 dot products, ties to the lowest index."""
    s = q.double().numpy() @ g.double().numpy().T
    return torch.from_numpy(np.argsort(-s, axis=1, kind="stable")[:, :kk])


@pytest.mark.parametrize("d", [64, 4096])
@pytest.mark.parametrize("jitter", [1e-3, 1e-4, 1e-5])
def test_ipr_operands_rank_replicated_sets_exactly(d, jitter):
    """The operands kth_nn_radii / compute_metric hand to sim_topk, ranked as sim_topk ranks them (float64 dot products of
    the float32 operands), keep every row the float64 answer needs: radii and ball membership match the reference."""
    from dcr_b200 import ipr
    x = _replicated(600, d, 1, jitter)
    x64 = torch.from_numpy(x).double()
    q, g = ipr._knn_operands(x64)
    assert q.dtype == g.dtype == torch.float32 and q.shape[1] % 4 == 0
    idx = _fp64_ranked(q, g, K + 1 + ipr._SPARE)
    cand = x64[idx]
    r2 = torch.sort(ipr._sq_dists(x64[:, None].expand_as(cand), cand), dim=1)[0][:, K].numpy()
    o = oipr.distances2radii(oipr.pairwise_distances(x), K)
    err = np.abs(r2 - o ** 2)
    assert err.max() <= _r2_tol(x), (int((err > _r2_tol(x)).sum()), err.max())

    # subjects: near copies of reference rows and fresh rows, against the reference's balls
    rng = np.random.default_rng(1)
    sub = np.vstack([x[:200] + jitter * rng.standard_normal((200, d)), _replicated(100, d, 1, jitter, (), (), seed=2)])
    sub = sub.astype(np.float32)
    sub64 = torch.from_numpy(sub).double()
    q, g = ipr._ball_operands(x64, torch.from_numpy(o), sub64)
    idx = _fp64_ranked(q, g, 1 + 2 * ipr._SPARE)
    cand = x64[idx]
    got = (torch.sqrt(ipr._sq_dists(cand, sub64[:, None].expand_as(cand))).numpy() < o[idx.numpy()]).any(1)
    want, margin = _inside(x, o, sub.astype(np.float64))
    clear = margin > 4 * _r2_tol(x, sub)
    assert clear.sum() >= 290 and 0 < want[clear].sum() < clear.sum()
    assert np.array_equal(got[clear], want[clear]), int((got != want)[clear].sum())


def test_ipr_rejects_k_and_n_the_reference_cannot_take():
    from dcr_b200 import _lib, ipr
    x = np.random.default_rng(3).standard_normal((40, 8)).astype(np.float32)
    for k in (1, 3, 12):
        with pytest.raises(ValueError):
            ipr.kth_nn_radii(x[:k + 1], k)        # np.argpartition(row, k + 1) is out of bounds at n == k + 1
    with pytest.raises(ValueError):
        ipr.kth_nn_radii(x, -1)
    for k in (13, 16, 20):
        with pytest.raises(_lib.DcrError, match="at most k = 12"):
            ipr.kth_nn_radii(x, k)


@pytest.mark.gpu
@pytest.mark.parametrize("d", [64, 4096])
@pytest.mark.parametrize("offset", [1, 30])
@pytest.mark.parametrize("jitter", [1e-3, 1e-4, 1e-5])
def test_ipr_cuda_radii_on_replicated_sets(d, offset, jitter):
    """Clusters of k+1, k+4 and 25 near copies and groups of k, k+1 and 20 exact copies.  r^2 is compared, not r: the
    reference's distance of two identical rows is the square root of float64 noise, not 0."""
    from dcr_b200 import ipr
    x = _replicated(1000, d, offset, jitter)
    r = ipr.kth_nn_radii(x, K)
    o = oipr.distances2radii(oipr.pairwise_distances(x), K)
    err = np.abs(r ** 2 - o ** 2)
    assert err.max() <= _r2_tol(x), (int((err > _r2_tol(x)).sum()), err.max())
    assert (r == 0).sum() >= 20 + K + 1          # the rows of the duplicate groups of more than k rows


def _near_copies_and_boundary(ref, radii, n_fresh, seed):
    """Subjects: fresh rows, exact copies of reference rows, jittered copies, and points at distance r_j (1 -/+ 1e-3) from
    reference row j (just inside / just outside its ball)."""
    rng = np.random.default_rng(seed)
    n, d = ref.shape
    fresh = _replicated(n_fresh, d, 1, 0.0, (), (), seed=seed + 1)
    j = rng.choice(n, 150, replace=False)
    u = rng.standard_normal((100, d))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    scale = np.where(np.arange(100) % 2 == 0, 1 - 1e-3, 1 + 1e-3)
    boundary = ref[j[50:]].astype(np.float64) + (radii[j[50:]] * scale)[:, None] * u
    copies = ref[j[:25]]
    jittered = ref[j[25:50]] + 1e-4 * rng.standard_normal((25, d))
    return np.vstack([fresh, copies, jittered, boundary]).astype(np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("d", [64, 4096])
def test_ipr_cuda_precision_recall_on_replicated_subjects(d):
    """compute_metric end to end in both directions, per subject: every subject clear of all ball boundaries by more than
    float64 rounding gets the float64 answer, and every subject clear of them by more than the reference's float32 rounding
    of ||subject||^2 (metrics/ipr.py:202) gets the reference's answer."""
    from dcr_b200 import ipr
    ref = _replicated(800, d, 1, 1e-4, seed=10)
    r_ref = ipr.kth_nn_radii(ref, K)
    o_ref = oipr.distances2radii(oipr.pairwise_distances(ref), K)
    sub = _near_copies_and_boundary(ref, o_ref, 300, seed=20)
    r_sub = ipr.kth_nn_radii(sub, K)
    o_sub = oipr.distances2radii(oipr.pairwise_distances(sub), K)
    for a, r_a, o_a, b in ((ref, r_ref, o_ref, sub), (sub, r_sub, o_sub, ref)):
        manifold = ipr.Manifold(a, r_a)
        truth, margin = _inside(a, o_a, b.astype(np.float64))
        faithful, _ = _inside(a, o_a, b)
        b2 = (b.astype(np.float64) ** 2).sum(1)
        for want, clear, min_cover in ((truth, margin > 4 * _r2_tol(a, b), 0.95),
                                       (faithful, margin > 2.0 ** -20 * b2, 0.9)):
            assert clear.sum() >= min_cover * len(b), (clear.sum(), len(b))
            inside, outside = b[clear & want], b[clear & ~want]
            assert len(inside) >= 20 and len(outside) >= 20
            assert ipr.compute_metric(manifold, inside) == 1.0
            assert ipr.compute_metric(manifold, outside) == 0.0


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 3, 7, 12])
@pytest.mark.parametrize("n", ["k+2", 50, 3000])
def test_ipr_cuda_k_and_n_edges(k, n):
    from dcr_b200 import ipr
    n = k + 2 if n == "k+2" else n
    x = _replicated(n, 64, 1, 1e-4, clusters=(k + 1,) if n > 2 * k + 2 else (), dups=(), seed=k)[:n]
    sub = _replicated(n, 64, 1, 0.0, (), (), seed=100 + k)
    r = ipr.kth_nn_radii(x, k)
    o = oipr.distances2radii(oipr.pairwise_distances(x), k)
    assert np.abs(r ** 2 - o ** 2).max() <= _r2_tol(x)
    assert ipr.compute_metric(ipr.Manifold(x, r), sub) == oipr.compute_metric(x, o, sub)
    o_sub = oipr.distances2radii(oipr.pairwise_distances(sub), k)
    assert ipr.compute_metric(ipr.Manifold(sub, o_sub), x) == oipr.compute_metric(sub, o_sub, x)


@pytest.mark.gpu
@pytest.mark.parametrize("d", [1, 2, 63, 100])
def test_ipr_cuda_odd_widths(d):
    """Feature widths that are not a multiple of 4 (the operands are padded for the kernel)."""
    from dcr_b200 import ipr
    x = _replicated(300, d, 1, 1e-4, seed=d)
    sub = _replicated(200, d, 1.1, 1e-4, seed=50 + d)
    r = ipr.kth_nn_radii(x, K)
    o = oipr.distances2radii(oipr.pairwise_distances(x), K)
    assert np.abs(r ** 2 - o ** 2).max() <= _r2_tol(x)
    o_sub = oipr.distances2radii(oipr.pairwise_distances(sub), K)
    assert ipr.compute_metric(ipr.Manifold(x, r), sub) == oipr.compute_metric(x, o, sub)
    assert ipr.compute_metric(ipr.Manifold(sub, ipr.kth_nn_radii(sub, K)), x) == oipr.compute_metric(sub, o_sub, x)


@pytest.mark.gpu
def test_ipr_cuda_realism_on_copies():
    """Exact copies (distance 0) and jittered copies (distance ~1e-4 sqrt(d)): the ratio r / (d + 1e-6) is then large and
    set by the radius and the tiny distance."""
    from dcr_b200 import ipr
    ref = _replicated(500, 4096, 1, 1e-5, seed=30)
    r = ipr.kth_nn_radii(ref, K)
    o = oipr.distances2radii(oipr.pairwise_distances(ref), K)
    rng = np.random.default_rng(31)
    subjects = [ref[i:i + 1] for i in range(0, 40, 5)]
    subjects += [(ref[i:i + 1] + 1e-4 * rng.standard_normal((1, 4096))).astype(np.float32) for i in range(1, 40, 5)]
    got = [ipr.realism(ipr.Manifold(ref, r), s) for s in subjects]
    want = [oipr.realism(ref, o, s) for s in subjects]
    assert min(got[:8]) > 1e6                           # distance 0: radius / 1e-6
    np.testing.assert_allclose(got, want, rtol=1e-6)
