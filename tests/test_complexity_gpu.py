"""GPU: the match-complexity kernels (dcr_image_stats, dcr_jpeg_encode) against the cv2 goldens and the oracle, their
determinism over calls, chunkings and input placement, their error paths, and `--complexity` end to end."""
import ctypes as C
import hashlib
import json
import os

import numpy as np
import pytest
import torch

from dcr_b200 import _lib, cli, complexity, data, synthetic
from oracle import complexity as oc
from oracle import models as om

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "jpeg_cv2.npz")
# The GPU's log() and numpy's may differ in the last bit, so entropies are compared to 1e-12.  A pixel rounded into
# another grey bin changes the entropy by about |log p_a - log p_b| / N: ~1e-6 for the 224 x 224 images here, whose
# bins hold ~200 pixels each, so the tolerance still catches any difference in the grey rounding.
ENT_TOL = 1e-12


def _stack(imgs):
    return torch.from_numpy(np.stack(imgs))


def test_device_files_equal_the_cv2_goldens():
    g = np.load(GOLDEN)
    for si, (h, w) in enumerate(oc.GOLDEN_SIZES):
        batch = _stack([img for _, img in oc.golden_images(h, w)]).cuda()
        for qi, q in enumerate(oc.GOLDEN_QUALITIES):
            files = complexity.jpeg_encode(batch, q)
            sizes = complexity.jpeg_sizes(batch, q).cpu().numpy()
            assert sizes.tolist() == g["sizes"][si, :, qi].tolist(), (h, w, q)
            for k, b in enumerate(files):
                assert len(b) == sizes[k]
                assert hashlib.sha256(b).digest() == g["sha256"][si, k, qi].tobytes(), (h, w, q, g["kinds"][k])
            full = f"full_{h}x{w}_q{q}"
            if full in g.files:
                assert files[0] == g[full].tobytes()


def test_device_sizes_equal_the_oracle_on_seeded_images():
    rng = np.random.default_rng(11)
    crops = synthetic.images(4, seed=3)[:, 16:240, 16:240].contiguous()       # Resize(256)-sized images, centre 224
    imgs = [crops[i].numpy() for i in range(4)]
    imgs += [rng.integers(0, 256, (224, 224, 3), dtype=np.uint8) for _ in range(2)]
    base = rng.integers(0, 256, (4, 4, 3)).astype(np.float64)
    imgs.append(np.clip(np.kron(base, np.ones((56, 56, 1))) + rng.normal(0, 6, (224, 224, 3)), 0, 255).astype(np.uint8))
    batch = _stack(imgs).cuda()
    for q in (5, 50, 90, 100):
        got = complexity.jpeg_encode(batch, q)
        for i, img in enumerate(imgs):
            assert got[i] == oc.jpeg_encode(img, q), (i, q)
    other = rng.integers(0, 256, (3, 64, 160, 3), dtype=np.uint8)
    got = complexity.jpeg_encode(torch.from_numpy(other).cuda(), 75)
    assert [len(b) for b in got] == [len(oc.jpeg_encode(x, 75)) for x in other]


def test_entropy_and_total_variation_equal_the_oracle():
    rng = np.random.default_rng(12)
    imgs = [rng.integers(0, 256, (224, 224, 3), dtype=np.uint8) for _ in range(6)]   # ~5 near-.5 grey ties each
    imgs += [synthetic.images(2, seed=5)[i, :224, :224].numpy() for i in range(2)]
    imgs += [np.full((224, 224, 3), 77, np.uint8), rng.integers(0, 2, (37, 53, 3), dtype=np.uint8)]
    for img in imgs:
        ent, tv = complexity.image_stats(torch.from_numpy(np.ascontiguousarray(img))[None].cuda())
        assert abs(ent.item() - oc.entropy(oc.grey_u8(img))) <= ENT_TOL
        assert tuple(tv[0].tolist()) == oc.tv_sums(img)
    assert complexity.image_stats(torch.from_numpy(imgs[-2])[None].cuda())[0].item() == 0.0   # one grey level


def test_results_do_not_depend_on_call_chunking_or_placement():
    imgs = synthetic.images(15, seed=8, size=224)
    dev = imgs.cuda()
    ref_files = complexity.jpeg_encode(dev, 90)
    ref_sizes = complexity.jpeg_sizes(dev, 90)
    ref_ent, ref_tv = complexity.image_stats(dev)
    for chunk in (1, 7, 15):
        assert complexity.jpeg_encode(dev, 90, chunk=chunk) == ref_files
        assert torch.equal(complexity.jpeg_sizes(dev, 90, chunk=chunk), ref_sizes)
        e, t = complexity.image_stats(dev, chunk=chunk)
        assert torch.equal(e, ref_ent) and torch.equal(t, ref_tv)
    host = imgs.pin_memory()
    assert complexity.jpeg_encode(host, 90, chunk=7) == ref_files
    assert torch.equal(complexity.jpeg_sizes(imgs, 90).cpu(), ref_sizes.cpu())
    e, t = complexity.image_stats(host, chunk=4)
    assert torch.equal(e.cpu(), ref_ent.cpu()) and torch.equal(t.cpu(), ref_tv.cpu())
    assert torch.equal(complexity.jpeg_sizes(dev, 90), ref_sizes)          # a second call, same bits
    assert [len(b) for b in ref_files] == ref_sizes.tolist()


def test_empty_batch_and_error_paths_write_nothing():
    lib = _lib.load()
    empty = torch.empty((0, 32, 32, 3), dtype=torch.uint8, device="cuda")
    assert complexity.jpeg_sizes(empty).numel() == 0 and complexity.jpeg_encode(empty) == []
    assert complexity.image_stats(empty)[0].numel() == 0
    img = torch.from_numpy(np.random.default_rng(1).integers(0, 256, (2, 32, 32, 3), dtype=np.uint8)).cuda()
    ws_bytes = lib.dcr_jpeg_workspace_size(2, 32, 32)
    ws = torch.empty(ws_bytes + 256, dtype=torch.uint8, device="cuda")
    ws_ptr = (ws.data_ptr() + 255) // 256 * 256
    sizes = torch.full((2,), -7, dtype=torch.int64, device="cuda")
    stride = lib.dcr_jpeg_max_bytes(32, 32)
    out = torch.full((2, stride), 0xAB, dtype=torch.uint8, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    bad = [
        (img.data_ptr(), 2, 32, 32, 0, sizes.data_ptr(), out.data_ptr(), ws_ptr, ws_bytes, st),        # quality
        (img.data_ptr(), 2, 32, 32, 101, sizes.data_ptr(), out.data_ptr(), ws_ptr, ws_bytes, st),
        (img.data_ptr(), 2, 32, 40, 90, sizes.data_ptr(), out.data_ptr(), ws_ptr, ws_bytes, st),       # size
        (img.data_ptr(), 2, 32, 32, 90, sizes.data_ptr(), out.data_ptr(), ws_ptr, ws_bytes - 1, st),   # workspace
        (img.data_ptr(), 2, 32, 32, 90, sizes.data_ptr(), out.data_ptr(), ws_ptr + 16, ws_bytes, st),  # alignment
        (None, 2, 32, 32, 90, sizes.data_ptr(), out.data_ptr(), ws_ptr, ws_bytes, st),
        (img.data_ptr(), 2, 32, 32, 90, None, out.data_ptr(), ws_ptr, ws_bytes, st),
        (img.data_ptr(), -1, 32, 32, 90, sizes.data_ptr(), out.data_ptr(), ws_ptr, ws_bytes, st),
    ]
    for args in bad:
        assert lib.dcr_jpeg_encode(*args) < 0, args
        assert _lib.last_error() != ""
    ent = torch.full((2,), -3.0, dtype=torch.float64, device="cuda")
    tv = torch.full((2, 2), -5, dtype=torch.int64, device="cuda")
    for args in [(img.data_ptr(), 2, 0, 32, ent.data_ptr(), tv.data_ptr(), st),
                 (img.data_ptr(), 2, 32, 32, None, tv.data_ptr(), st),
                 (img.data_ptr(), -2, 32, 32, ent.data_ptr(), tv.data_ptr(), st)]:
        assert lib.dcr_image_stats(*args) < 0 and _lib.last_error() != ""
    torch.cuda.synchronize()
    assert (sizes == -7).all() and (out == 0xAB).all() and (ent == -3.0).all() and (tv == -5).all()
    with pytest.raises(_lib.DcrError, match="quality"):
        complexity.jpeg_sizes(img, 0)
    with pytest.raises(_lib.DcrError, match="multiples of 16"):
        complexity.jpeg_sizes(torch.zeros((1, 20, 32, 3), dtype=torch.uint8, device="cuda"))
    with pytest.raises(_lib.DcrError, match="uint8"):
        complexity.image_stats(torch.zeros((1, 16, 16, 3), device="cuda"))
    # a good call after the refused ones
    assert lib.dcr_jpeg_encode(img.data_ptr(), 2, 32, 32, 90, sizes.data_ptr(), out.data_ptr(), ws_ptr, ws_bytes, st) == 0
    torch.cuda.synchronize()
    assert [bytes(out[i, :sizes[i]].cpu().numpy()) for i in range(2)] == [oc.jpeg_encode(x, 90) for x in img.cpu().numpy()]


def _write_images(folder, n, seed):
    from PIL import Image
    os.makedirs(folder, exist_ok=True)
    rng = np.random.default_rng(seed)
    base = rng.integers(0, 256, (n, 8, 8, 3), dtype=np.uint8)
    imgs = np.stack([np.asarray(Image.fromarray(b).resize((256, 256), Image.BILINEAR)) for b in base])
    noise = rng.integers(-20, 21, imgs.shape) * (np.arange(n) % 3)[:, None, None, None]   # varied complexity
    imgs = np.clip(imgs.astype(np.int16) + noise, 0, 255).astype(np.uint8)
    for i in range(n):
        Image.fromarray(imgs[i]).save(os.path.join(folder, f"{i}.png"))
    return imgs


def test_cli_complexity_end_to_end(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    q_dir, v_dir = str(tmp_path / "runs" / "exp" / "generations"), str(tmp_path / "train")
    _write_images(q_dir, 10, 31)
    v_imgs = _write_images(v_dir, 9, 32)
    from PIL import Image
    for j, src in enumerate([2, 2, 5]):          # two generations share a match
        Image.fromarray(v_imgs[src]).save(os.path.join(q_dir, f"{j}.png"))
    sd = om.make_sscd_state_dict(7)
    wpath = str(tmp_path / "sscd.pt")
    torch.save(sd, wpath)
    rc = cli.main(["--query_dir", q_dir, "--val_dir", v_dir, "--pt_style", "sscd", "--arch", "resnet50",
                   "--weights", wpath, "--precision", "exact", "--topk", "3", "--complexity"])
    assert rc == 0
    save = os.path.join("ret_plots", "runs", "exp", "generations", "images", "sscd_resnet50_dotproduct")
    res = torch.load(os.path.join(save, "topk.pth"))
    stats = json.load(open(os.path.join(save, "stats.json")))
    got = {k: torch.load(os.path.join(save, f"{k}.pth"), weights_only=False)
           for k in ("entropies", "totvar", "compressions", "dbsims")}
    top1 = res["indices"][:, 0].numpy()
    assert top1[:3].tolist() == [2, 2, 5]
    vf = data.list_images(v_dir)
    matched = data.load_files_u8([vf[i] for i in top1], size=224, workers=1).numpy()   # dataset_simpl, per generation
    ref = oc.complexity_loop(matched, res["values"][:, 0].numpy())
    for k in ("entropies", "totvar", "compressions", "dbsims"):
        assert isinstance(got[k], np.ndarray) and got[k].shape == (10,), k
    np.testing.assert_array_equal(got["dbsims"], ref["dbsims"])
    np.testing.assert_array_equal(got["compressions"], ref["compressions"])
    assert np.abs(got["entropies"] - ref["entropies"]).max() <= ENT_TOL
    np.testing.assert_allclose(got["totvar"], ref["totvar"], rtol=1e-6)          # the reference sums in fp32
    exact = np.array([1e-4 * sum(oc.tv_sums(m)) for m in matched])
    np.testing.assert_array_equal(got["totvar"], exact)
    for k in oc.CORRELATION_KEYS:
        assert k in stats
        if np.isnan(ref[k]):
            assert np.isnan(stats[k]), k
        else:
            assert abs(stats[k] - ref[k]) <= 1e-5 * max(1.0, abs(ref[k])), (k, stats[k], ref[k])
