"""FID on the H100 path: the host mirror of metrics/fid.py.

    get_activations / calculate_activation_statistics   metrics/fid.py:76-139, 199-221
        -> ActivationStatistics: Inception pool3 features computed by the dcr_net executor are folded, batch by batch,
           into a float64 (sum, X^T X) pair on the device (dcr_fid_*); the [N, 2048] float64 host array of the
           reference (:118) never exists.
    calculate_frechet_distance                          metrics/fid.py:142-196
        -> frechet_distance: same formula; Tr sqrtm(S1 S2) is evaluated as sum(sqrt(eig(S1^1/2 S2 S1^1/2))) with two
           symmetric eigendecompositions in float64 (torch.linalg.eigh on the GPU -- an O(d^3) library call outside the
           hot loop) instead of scipy's Schur-based sqrtm of the non-symmetric product; agrees to ~1e-9 relative.
    calculate_fid_given_paths                           metrics/fid.py:239-255
        -> fid_from_images(net, real_u8, gen_u8)  (the images are resized to 299 on the host with PIL exactly like
           metrics/fid.py:104-106; `load_resized` below does it for a directory)
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Tuple

import numpy as np
import torch

from . import _lib
from .nets import DcrNet
from .retrieval import extract_features


class ActivationStatistics:
    def __init__(self, dim: int = 2048, device: Optional[torch.device] = None):
        self.lib = _lib.load()
        if not torch.cuda.is_available():
            raise _lib.DcrError("ActivationStatistics needs a CUDA device")
        self.dim = dim
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        h = C.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(self.lib.dcr_fid_create(dim, C.byref(h)), "dcr_fid_create")
        self.handle = h
        self.count = 0

    def __del__(self):
        try:
            if getattr(self, "handle", None):
                self.lib.dcr_fid_destroy(self.handle)
                self.handle = None
        except Exception:
            pass

    def update(self, act: torch.Tensor) -> None:
        """act: CUDA float32 [n, dim]."""
        if not (act.is_cuda and act.dtype == torch.float32 and act.dim() == 2 and act.shape[1] == self.dim):
            raise _lib.DcrError(f"update expects CUDA float32 [n, {self.dim}]")
        act = act.contiguous()
        with torch.cuda.device(act.device):
            st = torch.cuda.current_stream().cuda_stream
            _lib.check(self.lib.dcr_fid_accumulate(self.handle, act.data_ptr(), act.shape[0], st), "dcr_fid_accumulate")
        self.count += act.shape[0]

    def finalize(self) -> Tuple[np.ndarray, np.ndarray]:
        mu = np.empty(self.dim, dtype=np.float64)
        sigma = np.empty((self.dim, self.dim), dtype=np.float64)
        n = C.c_int64(0)
        with torch.cuda.device(self.device):
            st = torch.cuda.current_stream().cuda_stream
            _lib.check(self.lib.dcr_fid_finalize(self.handle, mu.ctypes.data, sigma.ctypes.data, C.byref(n), st),
                       "dcr_fid_finalize")
        return mu, sigma


def frechet_distance(mu1, sigma1, mu2, sigma2, eps: float = 1e-6, device: Optional[torch.device] = None) -> float:
    """d^2 = ||mu1-mu2||^2 + Tr(s1) + Tr(s2) - 2 Tr(sqrt(s1 s2))   (metrics/fid.py:142-196)."""
    dev = torch.device("cuda") if (device is None and torch.cuda.is_available()) else (device or torch.device("cpu"))
    m1 = torch.as_tensor(np.atleast_1d(mu1), dtype=torch.float64, device=dev)
    m2 = torch.as_tensor(np.atleast_1d(mu2), dtype=torch.float64, device=dev)
    s1 = torch.as_tensor(np.atleast_2d(sigma1), dtype=torch.float64, device=dev)
    s2 = torch.as_tensor(np.atleast_2d(sigma2), dtype=torch.float64, device=dev)
    if m1.shape != m2.shape:
        raise ValueError("Training and test mean vectors have different lengths")          # fid.py:170-171
    if s1.shape != s2.shape:
        raise ValueError("Training and test covariances have different dimensions")        # fid.py:172-173

    def tr_sqrt_product(a, b):
        w, v = torch.linalg.eigh((a + a.T) * 0.5)
        ra = (v * torch.sqrt(w.clamp_min(0))) @ v.T            # a^(1/2)
        m = ra @ b @ ra
        ev = torch.linalg.eigvalsh((m + m.T) * 0.5)
        # sqrtm(s1 s2) has the spectrum sqrt(ev): a negative eigenvalue is an imaginary component of the reference's
        # covmean.  fid.py:187-191 tolerates |imag| <= 1e-3 on the diagonal and raises otherwise.
        neg = ev[ev < 0]
        if neg.numel() and torch.isfinite(neg).all():
            worst = float(torch.sqrt(-neg.min()))
            if worst > 1e-3:
                raise ValueError("Imaginary component {}".format(worst))
        return torch.sqrt(ev.clamp_min(0)).sum()

    tr = tr_sqrt_product(s1, s2)
    if not torch.isfinite(tr):                                                              # fid.py:179-184
        off = torch.eye(s1.shape[0], dtype=torch.float64, device=dev) * eps
        tr = tr_sqrt_product(s1 + off, s2 + off)
    diff = m1 - m2
    return float(diff.dot(diff) + torch.trace(s1) + torch.trace(s2) - 2 * tr)


def statistics_of_images(net: DcrNet, images_u8: torch.Tensor, batch_size: int = 50) -> Tuple[np.ndarray, np.ndarray]:
    """calculate_activation_statistics (metrics/fid.py:199-221) for uint8 [N,299,299,3] images (host or device)."""
    stats = ActivationStatistics(net.out_dim, net.device)
    n = images_u8.shape[0]
    chunk = max(batch_size, net.max_batch) * 8
    for s in range(0, n, chunk):
        stats.update(extract_features(net, images_u8[s:s + chunk], batch_size))
    return stats.finalize()


def fid_from_images(net: DcrNet, real_u8: torch.Tensor, gen_u8: torch.Tensor, batch_size: int = 50) -> float:
    """calculate_fid_given_paths (metrics/fid.py:239-255) on already decoded + resized images."""
    m1, s1 = statistics_of_images(net, real_u8, batch_size)
    m2, s2 = statistics_of_images(net, gen_u8, batch_size)
    return frechet_distance(m1, s1, m2, s2)


def load_resized(path: str, size: int = 299) -> torch.Tensor:
    """All **/*.JPEG|png|jpg under `path` (glob order of metrics/fid.py:231), PIL RGB, Resize(299) bilinear +
    CenterCrop(299) as metrics/fid.py:104-107 -> uint8 [N,299,299,3]."""
    import glob
    import os

    from PIL import Image
    from torchvision import transforms
    if not os.path.exists(path):
        raise RuntimeError("Invalid path: %s" % path)                                       # fid.py:243
    files = (list(glob.glob(os.path.join(path, "**/*.JPEG"), recursive=True)) +
             list(glob.glob(os.path.join(path, "**/*.png"), recursive=True)) +
             list(glob.glob(os.path.join(path, "**/*.jpg"), recursive=True)))
    tf = transforms.Compose([transforms.Resize(size), transforms.CenterCrop(size)])
    out = torch.empty((len(files), size, size, 3), dtype=torch.uint8)
    for i, f in enumerate(files):
        out[i] = torch.from_numpy(np.asarray(tf(Image.open(f).convert("RGB"))))
    return out


# ------------------------------------------------------------------------------------------------------------------
# the reference's call signatures (metrics/fid.py:224-275)
_FID_WEIGHTS_FILE = "pt_inception-2015-12-05-6726825d.pth"       # metrics/inception.py:13 (downloaded there; a local file here)


# InceptionV3.BLOCK_INDEX_BY_DIM (metrics/inception.py:22-28): the feature block each `dims` selects; blocks that end in
# a feature map are average pooled to 1x1 (metrics/fid.py:130-133), which the builder's GAP op does
_STOP_AFTER_BY_DIM = {64: "pool1", 192: "pool2", 768: "Mixed_6e", 2048: None}


def _build_inception(weights, max_batch: int, precision: str, dims: int = 2048) -> DcrNet:
    import os
    from . import nets
    if dims not in _STOP_AFTER_BY_DIM:
        raise KeyError(dims)                                   # InceptionV3.BLOCK_INDEX_BY_DIM[dims], fid.py:245
    if isinstance(weights, DcrNet):
        return weights
    if isinstance(weights, dict):
        sd = weights
    else:
        path = weights or os.environ.get("DCR_FID_WEIGHTS", _FID_WEIGHTS_FILE)
        if not os.path.exists(path):
            raise FileNotFoundError(f"FID Inception weights not found: {path} (there is no network access to fetch "
                                    f"{_FID_WEIGHTS_FILE}; pass weights= or set DCR_FID_WEIGHTS)")
        sd = torch.load(path, map_location="cpu")
    return nets.build_fid_inception(sd, max_batch=max_batch, precision=precision, stop_after=_STOP_AFTER_BY_DIM[dims])


def compute_statistics_of_path(path: str, net: DcrNet, batch_size: int = 50) -> Tuple[np.ndarray, np.ndarray]:
    """metrics/fid.py:224-236: a `.npz` with mu/sigma is loaded, anything else is globbed for images."""
    if path.endswith(".npz"):
        with np.load(path) as f:
            return f["mu"][:], f["sigma"][:]
    return statistics_of_images(net, load_resized(path), batch_size)


def calculate_fid_given_paths(paths, batch_size: int = 50, device=None, dims: int = 2048, num_workers: int = 1,
                              weights=None, precision: str = "fast") -> float:
    """metrics/fid.py:239-255.  `device` / `num_workers` are accepted for signature compatibility (the current CUDA
    device is used; image decoding is sequential).  dims in {64, 192, 768, 2048} select the feature block as
    InceptionV3.BLOCK_INDEX_BY_DIM does (metrics/inception.py:22-28); 2048 is what diff_retrieval.py:597-600 asks for."""
    import os
    for p in paths:
        if not os.path.exists(p):
            raise RuntimeError("Invalid path: %s" % p)                                       # fid.py:241-243
    print(dims)                                                                              # fid.py:244
    net = _build_inception(weights, batch_size, precision, dims)
    m1, s1 = compute_statistics_of_path(paths[0], net, batch_size)
    m2, s2 = compute_statistics_of_path(paths[1], net, batch_size)
    return frechet_distance(m1, s1, m2, s2)


def save_fid_stats(paths, batch_size: int = 50, device=None, dims: int = 2048, num_workers: int = 1, weights=None,
                   precision: str = "fast") -> None:
    """metrics/fid.py:258-275: statistics of paths[0] written to the .npz paths[1]."""
    import os
    if not os.path.exists(paths[0]):
        raise RuntimeError("Invalid path: %s" % paths[0])
    if os.path.exists(paths[1]):
        raise RuntimeError("Existing output file: %s" % paths[1])
    net = _build_inception(weights, batch_size, precision, dims)
    print(f"Saving statistics for {paths[0]}")
    m1, s1 = compute_statistics_of_path(paths[0], net, batch_size)
    np.savez_compressed(paths[1], mu=m1, sigma=s1)
