"""GPU: FID statistics computed in shards and merged (dcr_fid_export / dcr_fid_merge, ActivationStatistics.merge_ /
all_reduce_, the distributed= argument of dcr_b200.fid and the CLI's sharded FID)."""
import json
import os

import numpy as np
import pytest
import torch

from dcr_b200 import _lib
from dcr_b200 import fid as dfid
from dcr_b200 import nets
from dcr_b200.retrieval import extract_features
from oracle import fid as ofid
from oracle import models as om

pytestmark = pytest.mark.gpu


def _imgs(n, seed):
    return torch.randint(0, 256, (n, 299, 299, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(seed))


def _acts(n, d, seed):
    # large mean against unit-scale spread: a merge that mixed up the per-state shifts would show at once
    return torch.randn(n, d, generator=torch.Generator().manual_seed(seed), dtype=torch.float64).float() * 0.7 + 3.0


def _ragged(n):
    """Shard bounds with an empty shard and a one-row shard among them."""
    cuts = [0, 0, 1, n // 3, n // 3, (2 * n) // 3 + 1, n]
    return list(zip(cuts[:-1], cuts[1:]))


def _states(x, bounds, batch=170):
    out = []
    for lo, hi in bounds:
        st = dfid.ActivationStatistics(x.shape[1])
        for s in range(lo, hi, batch):
            st.update(x[s:min(s + batch, hi)].cuda())
        out.append(st)
    return out


def _packed(states):
    return torch.stack([s.export() for s in states])


@pytest.mark.parametrize("d", [256, 2048])
def test_merge_equals_one_state(d):
    n = 1500
    x = _acts(n, d, 40 + d)
    bounds = _ragged(n)
    assert [hi - lo for lo, hi in bounds].count(0) >= 1 and 1 in [hi - lo for lo, hi in bounds]
    shards = _states(x, bounds)
    merged = dfid.ActivationStatistics(d).merge_(_packed(shards))
    assert merged.count == n
    mu, sig = merged.finalize()
    one = _states(x, [(0, n)])[0]
    mu1, sig1 = one.finalize()
    rmu, rsig = ofid.activation_statistics(x.numpy())
    for m, s in ((rmu, rsig), (mu1, sig1)):
        np.testing.assert_allclose(mu, m, rtol=0, atol=1e-12)
        np.testing.assert_allclose(sig, s, rtol=0, atol=1e-11)
    # folding into a state that already holds rows (its own shift is kept) gives the same statistics
    head = _states(x, bounds[2:3])[0]
    head.merge_(_packed(shards[:2] + shards[3:]))
    mu2, sig2 = head.finalize()
    np.testing.assert_allclose(mu2, rmu, rtol=0, atol=1e-12)
    np.testing.assert_allclose(sig2, rsig, rtol=0, atol=1e-11)


def test_merge_is_deterministic():
    x = _acts(900, 512, 7)
    packed = _packed(_states(x, _ragged(900)))
    a = dfid.ActivationStatistics(512).merge_(packed).finalize()
    b = dfid.ActivationStatistics(512).merge_(packed.clone()).finalize()
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


def test_accumulate_after_merge():
    x = _acts(1200, 256, 8)
    st = dfid.ActivationStatistics(256).merge_(_packed(_states(x[:700], _ragged(700))))
    for s in range(700, 1200, 130):
        st.update(x[s:s + 130].cuda())
    assert st.count == 1200
    mu, sig = st.finalize()
    rmu, rsig = ofid.activation_statistics(x.numpy())
    np.testing.assert_allclose(mu, rmu, rtol=0, atol=1e-12)
    np.testing.assert_allclose(sig, rsig, rtol=0, atol=1e-11)


def test_merge_errors():
    a = dfid.ActivationStatistics(256)
    a.update(_acts(10, 256, 1).cuda())
    other = dfid.ActivationStatistics(128)
    other.update(_acts(10, 128, 2).cuda())
    wrong_d = torch.zeros(a.packed_nbytes, dtype=torch.uint8, device="cuda")
    wrong_d[:other.packed_nbytes] = other.export()
    with pytest.raises(_lib.DcrError, match="d = 128"):
        a.merge_(wrong_d)
    with pytest.raises(_lib.DcrError, match="not an exported"):
        a.merge_(torch.zeros(a.packed_nbytes, dtype=torch.uint8, device="cuda"))
    with pytest.raises(_lib.DcrError):
        a.merge_(other.export())                        # a packed state of the wrong size
    assert a.count == 10                                # nothing was merged
    mu, _ = a.finalize()
    np.testing.assert_allclose(mu, _acts(10, 256, 1).double().mean(0).numpy(), rtol=0, atol=1e-12)
    empty = dfid.ActivationStatistics(256).merge_(_packed([dfid.ActivationStatistics(256) for _ in range(3)]))
    assert empty.count == 0
    with pytest.raises(_lib.DcrError, match="need at least 2 samples"):
        empty.finalize()
    assert _lib.load().dcr_fid_packed_size(0) == 0


def _stats_tol(act):
    """Check-1 tolerances (1e-12 on mu, 1e-11 on sigma for unit-scale data), scaled to the activations' magnitude."""
    scale = max(1.0, float(np.abs(act).max()))
    return 1e-12 * scale, 1e-11 * scale * scale


def test_fake_world_fid_exact_mode():
    """Each image set cut into 3 shards on one device, one state per shard, merged: the same statistics and FID as the
    whole sets through fid_from_images."""
    sd = om.make_inception_state_dict(4)
    net = nets.build_fid_inception(sd, max_batch=8, precision="exact")
    real, gen = _imgs(24, 50), _imgs(24, 51)
    merged = []
    for imgs in (real, gen):
        shards = []
        for lo, hi in ((0, 11), (11, 12), (12, 24)):
            st = dfid.ActivationStatistics(2048)
            st.update(extract_features(net, imgs[lo:hi], 8))
            shards.append(st)
        merged.append(dfid.ActivationStatistics(2048).merge_(_packed(shards)).finalize())
    whole = [dfid.statistics_of_images(net, imgs, 8) for imgs in (real, gen)]
    act = extract_features(net, real, 8).double().cpu().numpy()
    tol_mu, tol_sig = _stats_tol(act)
    for (m, s), (wm, ws) in zip(merged, whole):
        assert np.abs(m - wm).max() < tol_mu and np.abs(s - ws).max() < tol_sig
    got = dfid.frechet_distance(*merged[0], *merged[1])
    want = dfid.fid_from_images(net, real, gen, 8)
    tr = float(np.trace(whole[0][1]) + np.trace(whole[1][1]))
    # measured on an H100: difference 1.4e-8 against a bound of 3.2e-8; the statistics agree to rounding, the rest is the
    # Frechet step's square roots of the near-null eigenvalues of singular covariances (24 images, 2048 dimensions)
    print(f"fake-world fid: merged {got!r} whole {want!r} diff {abs(got - want):.3e} (Tr sum {tr:.3f})")
    assert abs(got - want) < 1e-9 * max(1.0, tr), (got, want)


def _write_pngs(folder, imgs):
    from PIL import Image
    os.makedirs(folder, exist_ok=True)
    for i, im in enumerate(imgs):
        Image.fromarray(im.numpy()).save(os.path.join(folder, f"{i}.png"))


def test_path_entry_unsharded_is_unchanged(tmp_path):
    """With sharding off the path-level entry streams the folder through `num_workers` decoding threads in the chunks
    statistics_of_images uses: the value is exactly what fid_from_images gives on the fully loaded folders."""
    sd = om.make_inception_state_dict(3)
    net = nets.build_fid_inception(sd, max_batch=8, precision="fast")
    ra, ga = str(tmp_path / "real"), str(tmp_path / "gen")
    _write_pngs(ra, _imgs(70, 60))                      # 64-image chunks: two of them
    _write_pngs(ga, _imgs(9, 61))
    want = dfid.fid_from_images(net, dfid.load_resized(ra), dfid.load_resized(ga), 8)
    for workers in (1, 3):
        assert dfid.calculate_fid_given_paths([ra, ga], 8, "cuda", 2048, workers, weights=net) == want
    m, s = dfid.statistics_of_images(net, dfid.load_resized(ra), 8)
    npz = str(tmp_path / "real.npz")
    dfid.save_fid_stats([ra, npz], 8, "cuda", 2048, 2, weights=net)
    with np.load(npz) as f:
        assert np.array_equal(f["mu"], m) and np.array_equal(f["sigma"], s)


# ------------------------------------------------------------------------------------------------------------------
# several ranks


def _path_worker(rank, world, backend, port, seed, dirs, out_dir):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dev = torch.device("cuda", rank if backend == "nccl" else 0)
    torch.cuda.set_device(dev)
    dist.init_process_group(backend, rank=rank, world_size=world, device_id=dev if backend == "nccl" else None)
    net = dfid._build_inception(om.make_inception_state_dict(seed), 8, "exact", _DIMS)
    stats = [dfid.compute_statistics_of_path(p, net, 8, num_workers=2, distributed=True) for p in dirs]
    val = dfid.calculate_fid_given_paths(list(dirs), 8, "cuda", _DIMS, 2, weights=net, distributed=True)
    dfid.save_fid_stats([dirs[0], os.path.join(out_dir, "real_stats.npz")], 8, "cuda", _DIMS, 2, weights=net,
                        distributed=True)
    np.savez(os.path.join(out_dir, f"rank{rank}.npz"), fid=val, mu1=stats[0][0], s1=stats[0][1], mu2=stats[1][0],
             s2=stats[1][1])
    dist.barrier()
    dist.destroy_process_group()


# The 64-wide pool1 block of the Inception, with more images than dimensions: full-rank covariances, so the Frechet step
# does not amplify last-bit differences of sigma.  With 2048 dimensions and a few images, the square roots of the
# covariance product's null eigenvalues do: for 13 vs 10 images, with statistics inside the tolerances below, the FID
# moved by 1.2e-7 (4e-9 relative), three times 1e-9 * (Tr sigma1 + Tr sigma2), measured on an H100.
_DIMS = 64


def _check_sharded_paths(tmp_path, world, backend, port):
    import torch.multiprocessing as mp
    dirs = (str(tmp_path / "real"), str(tmp_path / "gen"))
    _write_pngs(dirs[0], _imgs(71, 70))                 # odd count: ragged shards
    _write_pngs(dirs[1], _imgs(66, 71))
    out_dir = str(tmp_path / "out")
    os.makedirs(out_dir)
    mp.spawn(_path_worker, args=(world, backend, port, 5, dirs, out_dir), nprocs=world, join=True)
    net = dfid._build_inception(om.make_inception_state_dict(5), 8, "exact", _DIMS)
    single = [dfid.compute_statistics_of_path(p, net, 8) for p in dirs]
    want = dfid.frechet_distance(*single[0], *single[1])
    tr = float(np.trace(single[0][1]) + np.trace(single[1][1]))
    ranks = [np.load(os.path.join(out_dir, f"rank{r}.npz")) for r in range(world)]
    act = extract_features(net, dfid.load_resized(dirs[0]), 8).double().cpu().numpy()
    tol_mu, tol_sig = _stats_tol(act)
    for r, got in enumerate(ranks):
        for k in ("mu1", "s1", "mu2", "s2"):
            assert np.array_equal(got[k], ranks[0][k]), (r, k)          # bit-identical on every rank
        for (m, s), km, ks in zip(single, ("mu1", "mu2"), ("s1", "s2")):
            assert np.abs(got[km] - m).max() < tol_mu and np.abs(got[ks] - s).max() < tol_sig
        assert float(got["fid"]) == float(ranks[0]["fid"])
        print(f"rank {r}: sharded fid {float(got['fid'])!r} single {want!r} (Tr sum {tr:.3f})")
        assert abs(float(got["fid"]) - want) < 1e-9 * max(1.0, tr), (r, float(got["fid"]), want)
    with np.load(os.path.join(out_dir, "real_stats.npz")) as f:    # written by rank 0
        assert np.array_equal(f["mu"], ranks[0]["mu1"]) and np.array_equal(f["sigma"], ranks[0]["s1"])


def test_sharded_paths_two_ranks_on_one_gpu(tmp_path):
    """The sharded path entry with two ranks sharing one GPU (gloo all-gather of the device buffers)."""
    _check_sharded_paths(tmp_path, 2, "gloo", 29300 + os.getpid() % 600)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_sharded_paths_two_gpus_nccl(tmp_path):
    _check_sharded_paths(tmp_path, 2, "nccl", 29900 + os.getpid() % 600)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_cli_fid_multiprocessing_distributed(tmp_path, monkeypatch):
    """The distributed CLI with --fid_weights: every rank embeds its shard of both folders for FID; stats.json holds the
    single-process FID to the north-star tolerance (the CLI's Inception runs in fast mode)."""
    import subprocess
    import sys

    from tests.test_cli_gpu import _write_images
    monkeypatch.chdir(tmp_path)
    q_dir, v_dir = str(tmp_path / "runs" / "exp" / "generations"), str(tmp_path / "train")
    _write_images(q_dir, 11, 21)
    _write_images(v_dir, 37, 22)
    wpath, fpath = str(tmp_path / "sscd.pt"), str(tmp_path / "inception.pt")
    torch.save(om.make_sscd_state_dict(7), wpath)
    torch.save(om.make_inception_state_dict(6), fpath)
    from dcr_b200 import cli
    common = ["--query_dir", q_dir, "--val_dir", v_dir, "--pt_style", "sscd", "--arch", "resnet50", "--weights", wpath,
              "--precision", "parity", "--topk", "5", "--fid_weights", fpath]
    save = os.path.join("ret_plots", "runs", "exp", "generations", "images", "sscd_resnet50_dotproduct")
    assert cli.main(common) == 0
    single = json.load(open(os.path.join(save, "stats.json")))["fid"]
    os.remove(os.path.join(save, "stats.json"))
    port = 28500 + os.getpid() % 1000
    env = dict(os.environ, PYTHONPATH=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    r = subprocess.run([sys.executable, "-m", "dcr_b200.cli", *common, "--multiprocessing-distributed", "--world-size", "1",
                        "--rank", "0", "--dist-url", f"tcp://127.0.0.1:{port}"], env=env, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    multi = json.load(open(os.path.join(save, "stats.json")))["fid"]
    assert abs(multi - single) < 1e-4 * max(1.0, abs(single)), (multi, single)
