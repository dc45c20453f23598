"""No GPU: the match-complexity oracle (diff_retrieval.py:497-540) against cv2, sklearn and the reference's tv_loss, the
cv2 goldens, the host-only JPEG entry points and the --complexity flag."""
import hashlib
import os

import numpy as np
import pytest
import torch

from oracle import complexity as oc

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "jpeg_cv2.npz")


def _golden():
    return np.load(GOLDEN)


def test_golden_file_covers_the_stated_grid():
    g = _golden()
    assert tuple(g["qualities"]) == oc.GOLDEN_QUALITIES
    assert [tuple(x) for x in g["hw"]] == list(oc.GOLDEN_SIZES)
    assert g["sizes"].shape == (len(oc.GOLDEN_SIZES), len(oc.golden_images(16, 16)), len(oc.GOLDEN_QUALITIES))
    assert os.path.getsize(GOLDEN) < 1 << 20


@pytest.mark.parametrize("size_i", range(len(oc.GOLDEN_SIZES)))
def test_oracle_encoder_matches_the_cv2_goldens(size_i):
    g = _golden()
    h, w = oc.GOLDEN_SIZES[size_i]
    for k, (kind, img) in enumerate(oc.golden_images(h, w)):
        assert kind == g["kinds"][k]
        for qi, q in enumerate(oc.GOLDEN_QUALITIES):
            b = oc.jpeg_encode(img, q)
            assert len(b) == g["sizes"][size_i, k, qi], (h, w, kind, q)
            assert hashlib.sha256(b).digest() == g["sha256"][size_i, k, qi].tobytes(), (h, w, kind, q)
            full = f"full_{h}x{w}_q{q}"
            if kind == "noise" and full in g.files:
                assert b == g[full].tobytes()


def test_oracle_encoder_matches_cv2_on_random_images():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(5)
    for i in range(300):
        h, w = 16 * int(rng.integers(1, 5)), 16 * int(rng.integers(1, 5))
        q = int(rng.integers(1, 101))
        if i % 3 == 0:
            img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        else:   # smooth images with noise: the common, mostly-zero AC case
            base = rng.integers(0, 256, (2, 2, 3)).astype(np.float64)
            img = np.kron(base, np.ones((h // 2, w // 2, 1))) + rng.normal(0, 8 * (i % 4), (h, w, 3))
            img = np.clip(img, 0, 255).astype(np.uint8)
        ok, ref = cv2.imencode(".jpg", img, [int(cv2.IMWRITE_JPEG_QUALITY), q])
        assert ok and oc.jpeg_encode(img, q) == ref.tobytes(), (i, h, w, q)


def test_header_is_623_bytes_at_every_quality():
    for q in range(1, 101):
        hdr = oc.jpeg_header(224, 224, q)
        assert len(hdr) == 623 == oc.HEADER_BYTES
        assert oc.jpeg_encode(np.zeros((16, 16, 3), np.uint8), q)[:623] == oc.jpeg_header(16, 16, q)


def test_oracle_entropy_equals_sklearn():
    sk = pytest.importorskip("sklearn.metrics.cluster")
    rng = np.random.default_rng(2)
    for i in range(20):
        img = rng.integers(0, 256 if i % 2 else 8, (64, 48, 3), dtype=np.uint8)
        grey = oc.grey_u8(img)
        assert oc.entropy(grey) == sk.entropy(grey)
    assert oc.entropy(np.full((4, 4), 7, np.uint8)) == sk.entropy(np.full((4, 4), 7, np.uint8)) == 0.0


def test_grey_value_is_the_stated_fp64_order():
    c = np.arange(256, dtype=np.float64) * (1.0 / 255)
    assert oc.grey_u8(np.stack([np.arange(256)] * 3, -1).astype(np.uint8)).tolist() == list(range(256))
    # the half-to-even rounding of img_as_ubyte: rint, not floor(x + 0.5)
    assert np.rint(2.5) == 2.0 and c[1] == 1.0 / 255


def test_oracle_tv_equals_reference_tv_loss():
    rng = np.random.default_rng(3)
    for i in range(10):
        img = rng.integers(0, 256, (224, 224, 3), dtype=np.uint8)
        torchim = torch.from_numpy(img).permute(2, 0, 1).float().div(255) * 255   # ToTensor() * 255
        ref = oc.tv_loss(torchim)
        h, w = oc.tv_sums(img)
        exact = 1e-4 * (h + w)
        assert abs(ref - exact) <= 1e-6 * exact, (ref, exact)   # the reference sums in fp32


def test_max_bytes_bounds_the_noise_goldens_and_sizes_are_refused():
    from dcr_b200 import _lib
    lib = _lib.load()
    g = _golden()
    for si, (h, w) in enumerate(oc.GOLDEN_SIZES):
        bound = lib.dcr_jpeg_max_bytes(h, w)
        assert bound % 16 == 0 and g["sizes"][si].max() <= bound
        assert lib.dcr_jpeg_workspace_size(7, h, w) > lib.dcr_jpeg_workspace_size(1, h, w) > 0
    for h, w in [(0, 16), (16, 0), (15, 16), (16, 24), (4112, 16), (16, 4112), (-16, 16)]:
        assert lib.dcr_jpeg_max_bytes(h, w) < 0
        assert "multiples of 16" in _lib.last_error()
        assert lib.dcr_jpeg_workspace_size(1, h, w) == 0
    assert lib.dcr_jpeg_workspace_size(-1, 16, 16) == 0 and "bad n" in _lib.last_error()
    # argument checks run before anything touches a device, so they answer here too
    for q in (0, 101, -5):
        assert lib.dcr_jpeg_encode(None, 1, 16, 16, q, None, None, None, 0, None) < 0
        assert "quality" in _lib.last_error()
    assert lib.dcr_jpeg_encode(None, 1, 24, 16, 90, None, None, None, 0, None) < 0
    assert lib.dcr_jpeg_encode(None, 1, 16, 16, 90, None, None, None, 0, None) < 0
    assert "null pointer" in _lib.last_error()
    assert lib.dcr_jpeg_encode(None, 0, 16, 16, 90, None, None, None, 0, None) == 0
    assert lib.dcr_image_stats(None, 0, 16, 16, None, None, None) == 0
    assert lib.dcr_image_stats(None, 2, 16, 16, None, None, None) < 0
    assert lib.dcr_image_stats(None, 1, 0, 16, None, None, None) < 0


def test_oracle_correlations_follow_pearsonr_and_nan_for_degenerate_input():
    from scipy import stats
    from dcr_b200 import complexity
    rng = np.random.default_rng(4)
    e, c, t, s = (rng.random(50) for _ in range(4))
    got = complexity.complexity_correlations(e, c, t, s)
    assert set(got) == set(complexity.CORRELATION_KEYS) == set(oc.CORRELATION_KEYS)
    assert got == oc.correlations(e, c, t, s)
    r, p = stats.pearsonr(e * c ** 0.5, s)
    assert got["cc_mixed"] == r and got["pval_mixed"] == p
    for args in ((e[:1], c[:1], t[:1], s[:1]), (e, c, np.ones(50), s), (e, c, t, np.zeros(50))):
        got = complexity.complexity_correlations(*args)
        assert any(np.isnan(v) for v in got.values())
    got = complexity.complexity_correlations(e, c, np.ones(50), s)
    assert np.isnan(got["cc_tvl"]) and np.isnan(got["pval_tvl"]) and not np.isnan(got["cc_ent"])


def test_complexity_flag_parses_and_defaults_off():
    from dcr_b200 import cli
    p = cli.build_parser()
    assert p.parse_args(["--query_dir", "a", "--val_dir", "b"]).complexity is False
    assert p.parse_args(["--query_dir", "a", "--val_dir", "b", "--complexity"]).complexity is True
