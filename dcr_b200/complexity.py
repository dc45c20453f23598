"""Match-complexity statistics on the GPU: the host side of diff_retrieval.py:497-540.

    entropy(img_as_ubyte(color.rgb2gray(rgbImg)))      :508       -> image_stats (dcr_image_stats)
    len(cv2.imencode('.jpg', rgbImg, q=90)[1]) / 1024  :513-515   -> jpeg_sizes / jpeg_encode (dcr_jpeg_encode)
    tv_loss(torchim)                                   :113-122   -> image_stats: exact int64 sums, 1e-4 * (h + w)
    stats.pearsonr(...) x 4                            :525-529   -> complexity_correlations (scipy, Q scalars)
    the loop over the top-1 matches                    :497-524   -> top1_complexity: decodes each matched training
                                                                     image once, however many generations share it
Images are uint8 [n, h, w, 3] (HWC), on the host (pinned for overlap) or on the device.  Host images are copied in
chunks; the JPEG workspace is sized per chunk, so a 10k batch never needs all its block data at once.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib

# device workspace the JPEG encoder may take per call (bit buffers for the worst-case file of every image in a chunk)
JPEG_WORKSPACE_BUDGET = 512 << 20
CORRELATION_KEYS = ("cc_ent", "pval_ent", "cc_comp", "pval_comp", "cc_tvl", "pval_tvl", "cc_mixed", "pval_mixed")


def _check_images(images: torch.Tensor) -> Tuple[int, int, int]:
    if not isinstance(images, torch.Tensor) or images.dtype != torch.uint8 or images.dim() != 4 or images.shape[3] != 3:
        raise _lib.DcrError(f"images must be a uint8 tensor [n, h, w, 3], got "
                            f"{getattr(images, 'dtype', type(images))} {tuple(getattr(images, 'shape', ()))}")
    if not torch.cuda.is_available():
        raise _lib.DcrError("the complexity statistics need a CUDA device (dcr_b200 has no CPU compute path)")
    return int(images.shape[0]), int(images.shape[1]), int(images.shape[2])


def _device(images: torch.Tensor) -> torch.device:
    return images.device if images.is_cuda else torch.device("cuda", torch.cuda.current_device())


def _chunks(images: torch.Tensor, chunk: int):
    """(start, device uint8 chunk) pairs; host chunks are copied on the current stream."""
    dev = _device(images)
    for s in range(0, images.shape[0], chunk):
        part = images[s:s + chunk]
        if not part.is_cuda:
            part = part.to(dev, non_blocking=part.is_pinned())
        yield s, part.contiguous()


def image_stats(images: torch.Tensor, chunk: Optional[int] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """(entropy float64 [n], tv int64 [n, 2] = (h, w) sums) on the images' device (the current one for host input)."""
    n, h, w = _check_images(images)
    lib = _lib.load()
    dev = _device(images)
    ent = torch.empty(n, dtype=torch.float64, device=dev)
    tv = torch.empty((n, 2), dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        st = torch.cuda.current_stream().cuda_stream
        if n == 0:
            _lib.check(lib.dcr_image_stats(None, 0, h, w, None, None, st), "dcr_image_stats")
        if chunk is None:
            chunk = max(n, 1) if images.is_cuda else 1024
        for s, part in _chunks(images, chunk):
            m = part.shape[0]
            _lib.check(lib.dcr_image_stats(part.data_ptr(), m, h, w, ent[s:].data_ptr(), tv[s:].data_ptr(), st),
                       "dcr_image_stats")
    return ent, tv


def jpeg_max_bytes(h: int, w: int) -> int:
    b = _lib.load().dcr_jpeg_max_bytes(h, w)
    if b < 0:
        raise _lib.DcrError(f"dcr_jpeg_max_bytes: {_lib.last_error()}")
    return int(b)


def _jpeg_chunk(h: int, w: int, with_bytes: bool) -> int:
    lib = _lib.load()
    one = lib.dcr_jpeg_workspace_size(1, h, w)
    if one == 0:
        raise _lib.DcrError(f"dcr_jpeg_workspace_size: {_lib.last_error()}")
    per = one + (jpeg_max_bytes(h, w) if with_bytes else 0)
    return max(1, JPEG_WORKSPACE_BUDGET // per)


def _jpeg(images: torch.Tensor, quality: int, with_bytes: bool, chunk: Optional[int]):
    n, h, w = _check_images(images)
    lib = _lib.load()
    dev = _device(images)
    chunk = chunk or _jpeg_chunk(h, w, with_bytes)
    sizes = torch.empty(n, dtype=torch.int64, device=dev)
    files: List[bytes] = []
    with torch.cuda.device(dev):
        st = torch.cuda.current_stream().cuda_stream
        if n == 0:       # still validates the size and the quality
            _lib.check(lib.dcr_jpeg_encode(None, 0, h, w, quality, None, None, None, 0, st), "dcr_jpeg_encode")
            return sizes, files
        m0 = min(chunk, n)
        ws_bytes = lib.dcr_jpeg_workspace_size(m0, h, w)
        if ws_bytes == 0:
            raise _lib.DcrError(f"dcr_jpeg_workspace_size: {_lib.last_error()}")
        ws = torch.empty(ws_bytes + 256, dtype=torch.uint8, device=dev)
        ws_ptr = (ws.data_ptr() + 255) // 256 * 256
        stride = jpeg_max_bytes(h, w)
        out = torch.empty((m0, stride), dtype=torch.uint8, device=dev) if with_bytes else None
        for s, part in _chunks(images, chunk):
            m = part.shape[0]
            _lib.check(lib.dcr_jpeg_encode(part.data_ptr(), m, h, w, quality, sizes[s:].data_ptr(),
                                           out.data_ptr() if with_bytes else None, ws_ptr, ws_bytes, st),
                       "dcr_jpeg_encode")
            if with_bytes:
                host = out[:m].cpu().numpy()
                sz = sizes[s:s + m].cpu().numpy()
                files.extend(host[i, :sz[i]].tobytes() for i in range(m))
    return sizes, files


def jpeg_sizes(images: torch.Tensor, quality: int = 90, chunk: Optional[int] = None) -> torch.Tensor:
    """int64 [n]: len(cv2.imencode('.jpg', img, [IMWRITE_JPEG_QUALITY, quality])[1]) of every image (h, w multiples
    of 16), on the images' device."""
    return _jpeg(images, quality, False, chunk)[0]


def jpeg_encode(images: torch.Tensor, quality: int = 90, chunk: Optional[int] = None) -> List[bytes]:
    """The files cv2.imencode('.jpg', img, [IMWRITE_JPEG_QUALITY, quality]) writes, one bytes object per image."""
    return _jpeg(images, quality, True, chunk)[1]


def match_complexity(images: torch.Tensor, quality: int = 90) -> Dict[str, np.ndarray]:
    """The per-image quantities of diff_retrieval.py:508-516 in the reference's units (float64 numpy arrays):
    entropies, compressions (KiB of the quality-90 JPEG) and totvar (1e-4 * (h + w))."""
    ent, tv = image_stats(images)
    sizes = jpeg_sizes(images, quality)
    tv = tv.cpu().numpy()
    return {"entropies": ent.cpu().numpy(), "compressions": sizes.cpu().numpy() / 1024,
            "totvar": 1e-4 * (tv[:, 0] + tv[:, 1]).astype(np.float64)}


def complexity_correlations(entropies, compressions, totvar, dbsims) -> Dict[str, float]:
    """diff_retrieval.py:525-529: Pearson r and p-value of entropy, JPEG size, TV and entropy * sqrt(size) against the
    top-1 similarity.  A key is NaN when there are fewer than two queries or either input is constant."""
    from scipy import stats
    e, c, t, s = (np.asarray(a, dtype=np.float64).ravel() for a in (entropies, compressions, totvar, dbsims))
    out = {}
    for name, x in (("ent", e), ("comp", c), ("tvl", t), ("mixed", e * c ** 0.5)):
        if len(s) < 2 or np.ptp(x) == 0 or np.ptp(s) == 0:
            r, p = float("nan"), float("nan")
        else:
            r, p = stats.pearsonr(x, s)
        out[f"cc_{name}"], out[f"pval_{name}"] = float(r), float(p)
    return out


def top1_complexity(gallery_files: Sequence[str], top1_idx, top1_sims, workers: int = 4) -> Dict:
    """The whole loop diff_retrieval.py:497-529: the matched training images are decoded once each (Resize(224) +
    CenterCrop(224), dataset_simpl :337-342), measured on the GPU and scattered back per generation.  Returns the four
    arrays the reference saves (entropies, compressions, totvar, dbsims) and the eight correlation keys."""
    from . import data
    idx = np.asarray(top1_idx, dtype=np.int64).ravel()
    sims = np.asarray(top1_sims).ravel()
    uniq, inverse = np.unique(idx, return_inverse=True)
    imgs = data.load_files_u8([gallery_files[i] for i in uniq], size=224, workers=workers)
    per = match_complexity(imgs)
    out = {k: v[inverse] for k, v in per.items()}
    out["dbsims"] = sims
    out.update(complexity_correlations(out["entropies"], out["compressions"], out["totvar"], sims))
    return out
