"""Improved Precision & Recall on the H100 path: the host mirror of metrics/ipr.py (imported by diff_retrieval.py:587).

    IPR(batch_size, k, num_samples, model)      metrics/ipr.py:33-181   same methods and return types
    compute_manifold -> Manifold(features, radii)           :80-122
    precision_and_recall -> PrecisionAndRecall              :49-64
    realism                                                 :71-77, 253-263

What changes underneath:
  * the VGG-16 fc2 features (:124-147) come from the dcr_net executor (nets.build_vgg16_fc2: wgmma implicit-GEMM convs);
  * the N x N (and N x M) float64 distance matrices of compute_pairwise_distances (:184-217) are never built.  Both uses of
    them are nearest-neighbour questions, answered by the fused similarity + top-k kernel on augmented vectors:
        -d(x,y)^2 / 2 + ||x||^2 / 2 = x.y - ||y||^2 / 2            = [x, 1] . [y, -||y||^2 / 2]              (k-th NN radius)
        (r_j^2 - d(y_j, x)^2) / 2 + ||x||^2 / 2 = x.y_j + (r_j^2 - ||y_j||^2) / 2                          (inside any ball?)
    Features are float32 (what the VGG-16 network produces), used uncentred, so the vector part of both operands is exact.
    The float64 norm term, divided by a power of two s, is carried as an error-free split into three float32 columns
    (hi + mid + lo == the float64 value) against s, s, s on the query side (_operands).  The kernel ranks by the float64
    dot product of its float32 operands, so its ranking is the float64 ranking of the features themselves: a few spare
    candidates absorb float64-level ties, and the final distances / comparisons are re-evaluated in float64 with the
    reference's own formula, so radii and the precision / recall counts agree with the reference to float64 rounding --
    also for sets of exact and near copies.
"""
from __future__ import annotations

import math
import os
from collections import namedtuple
from glob import glob
from typing import Optional

import numpy as np
import torch

from . import _lib
from .nets import DcrNet
from .retrieval import extract_features
from .similarity import sim_topk

Manifold = namedtuple("Manifold", ["features", "radii"])
PrecisionAndRecall = namedtuple("PrecisinoAndRecall", ["precision", "recall"])     # (sic) metrics/ipr.py:31

_SPARE = 3          # candidates kept beyond what the exact answer needs (float64-level ties)
_MAX_CANDIDATES = 16  # sim_topk keeps at most 16 rows per query


def _split3(a: torch.Tensor) -> torch.Tensor:
    """float64 [n] -> float32 [n, 3] (hi, mid, lo) with hi + mid + lo == a exactly (each step's remainder is exact)."""
    hi = a.float()
    r = a - hi.double()
    mid = r.float()
    lo = (r - mid.double()).float()
    return torch.stack([hi, mid, lo], dim=1)


def _augmented(x32: torch.Tensor, tail: torch.Tensor) -> torch.Tensor:
    """[x | tail | 0 ...] as float32, the width padded to a multiple of 4 (sim_topk's requirement)."""
    n, d = x32.shape
    out = torch.zeros((n, (d + 6) // 4 * 4), dtype=torch.float32, device=x32.device)
    out[:, :d] = x32
    out[:, d:d + 3] = tail
    return out


def _operands(queries: torch.Tensor, rows: torch.Tensor, term: torch.Tensor):
    """sim_topk operands whose float64 score is queries_i . rows_j + term_j with no rounding of either operand: the
    features as float32 (exact for float32 features), and term / s split over three columns against s, s, s.
    s is a power of two (the products are the same), 4x the largest feature norm rounded up: the constant query columns
    then dominate the queries' mean square, so sim_topk centres the queries, and term / s varies no more than the features
    do.  Both keep the kernel's bf16 error bound as tight as for centred features, so few queries need its float64
    brute-force path (with s = 1 every query of 4096-d VGG features does)."""
    q32, r32 = queries.float(), rows.float()
    top = max((q32.double() ** 2).sum(-1).max().item(), (r32.double() ** 2).sum(-1).max().item()) ** 0.5
    s = 2.0 ** (math.ceil(math.log2(max(top, 2.0 ** -60))) + 2)
    cols = torch.full((q32.shape[0], 3), s, dtype=torch.float32, device=q32.device)
    return _augmented(q32, cols), _augmented(r32, _split3(term / s))


def _knn_operands(x: torch.Tensor):
    """Score x_i . x_j - ||x_j||^2 / 2 = (||x_i||^2 - d(x_i, x_j)^2) / 2: nearest rows first."""
    x32 = x.float()
    return _operands(x32, x32, -0.5 * (x32.double() ** 2).sum(-1))


def _ball_operands(ref: torch.Tensor, radii: torch.Tensor, subjects: torch.Tensor):
    """Score s_i . r_j + (rad_j^2 - ||r_j||^2) / 2 = (rad_j^2 - d(s_i, r_j)^2 + ||s_i||^2) / 2: deepest ball first."""
    r32 = ref.float()
    return _operands(subjects, r32, 0.5 * (radii * radii - (r32.double() ** 2).sum(-1)))


def _sq_dists(a64: torch.Tensor, b64: torch.Tensor) -> torch.Tensor:
    """Row-wise ||a||^2 - 2 a.b + ||b||^2 in float64, clamped at 0 (metrics/ipr.py:198-214), for paired rows [n,d]."""
    d2 = (a64 * a64).sum(-1) - 2.0 * (a64 * b64).sum(-1) + (b64 * b64).sum(-1)
    return d2.clamp_min(0.0)


def kth_nn_radii(features, k: int = 3) -> np.ndarray:
    """distances2radii(compute_pairwise_distances(features), k) (metrics/ipr.py:119-121, 220-233): per row the distance to
    its k-th nearest OTHER row -- the (k+1)-th smallest entry of its distance row, the smallest being the row itself."""
    if k + 1 + _SPARE > _MAX_CANDIDATES:
        raise _lib.DcrError(f"k = {k}: at most k = {_MAX_CANDIDATES - 1 - _SPARE} (k + 1 + {_SPARE} spare candidates per "
                            f"row, sim_topk keeps at most {_MAX_CANDIDATES})")
    features = np.asarray(features)
    n = features.shape[0]
    if k < 0 or n < k + 2:
        raise ValueError(f"k = {k} needs k >= 0 and at least {k + 2} samples, got {n} "
                         f"(np.argpartition(row, k + 1) fails in the reference, too)")
    x = torch.as_tensor(features, dtype=torch.float64).cuda()
    kk = min(k + 1 + _SPARE, n)
    q, g = _knn_operands(x)
    _, idx = sim_topk(q, g, kk)                                            # nearest rows first (self among them)
    cand = x[idx.reshape(-1)].reshape(n, kk, -1)
    d = torch.sqrt(_sq_dists(x[:, None, :].expand_as(cand), cand))        # [n, kk] float64
    d_sorted, _ = torch.sort(d, dim=1)
    return d_sorted[:, k].cpu().numpy()                                   # (k+1)-th smallest, self included


def compute_metric(manifold_ref: Manifold, feats_subject, desc: str = "") -> float:
    """metrics/ipr.py:236-242: fraction of subjects lying inside at least one reference ball."""
    ref = torch.as_tensor(np.asarray(manifold_ref.features), dtype=torch.float64).cuda()
    rad = torch.as_tensor(np.asarray(manifold_ref.radii), dtype=torch.float64).cuda()
    sub = torch.as_tensor(np.asarray(feats_subject), dtype=torch.float64).cuda()
    ns, nr = sub.shape[0], ref.shape[0]
    kk = min(1 + 2 * _SPARE, nr)
    q, g = _ball_operands(ref, rad, sub)
    _, idx = sim_topk(q, g, kk)                                            # balls the subject is deepest inside, first
    cand = ref[idx.reshape(-1)].reshape(ns, kk, -1)
    d = torch.sqrt(_sq_dists(cand, sub[:, None, :].expand_as(cand)))      # dist[j, i] of the reference, selected pairs
    inside = (d < rad[idx]).any(dim=1)
    return float(inside.sum().item()) / ns


def realism(manifold_real: Manifold, feat_subject) -> float:
    """metrics/ipr.py:253-263."""
    real = torch.as_tensor(np.asarray(manifold_real.features), dtype=torch.float64).cuda()
    rad = torch.as_tensor(np.asarray(manifold_real.radii), dtype=torch.float64).cuda()
    f = torch.as_tensor(np.asarray(feat_subject), dtype=torch.float64).cuda().reshape(1, -1)
    dists = torch.linalg.norm(real - f, dim=1)
    return float((rad / (dists + 1e-6)).max().item())


def load_resized_224(files, size: int = 224) -> torch.Tensor:
    """get_custom_loader's decode + Resize([224, 224]) (metrics/ipr.py:300-303) -> uint8 [N,224,224,3]; ToTensor and the
    ImageNet Normalize (:304-306) are fused into the network's first kernel."""
    from PIL import Image
    from torchvision import transforms
    tf = transforms.Resize([size, size])
    out = torch.empty((len(files), size, size, 3), dtype=torch.uint8)
    for i, f in enumerate(files):
        out[i] = torch.from_numpy(np.asarray(tf(Image.open(f).convert("RGB"))).copy())
    return out


class IPR:
    """Same constructor and methods as metrics/ipr.IPR.  `model`: a DcrNet from nets.build_vgg16_fc2, or a torchvision
    VGG-16 state_dict (the reference downloads `models.vgg16(pretrained=True)`, :39 -- there is no network here)."""

    def __init__(self, batch_size: int = 50, k: int = 3, num_samples: int = 10000, model=None, precision: str = "fast"):
        self.manifold_ref = None
        self.batch_size = batch_size
        self.k = k
        self.num_samples = num_samples
        if model is None:
            raise _lib.DcrError("IPR needs the VGG-16 weights: pass model=<state_dict or DcrNet> (no download possible)")
        if isinstance(model, DcrNet):
            self.vgg16 = model
        else:
            from . import nets
            self.vgg16 = nets.build_vgg16_fc2(model, max_batch=batch_size, precision=precision)

    def __call__(self, subject):
        return self.precision_and_recall(subject)

    def precision_and_recall(self, subject):                                              # :49-64
        assert self.manifold_ref is not None, "call IPR.compute_manifold_ref() first"
        manifold_subject = self.compute_manifold(subject)
        precision = compute_metric(self.manifold_ref, manifold_subject.features, "computing precision...")
        recall = compute_metric(manifold_subject, self.manifold_ref.features, "computing recall...")
        return PrecisionAndRecall(precision, recall)

    def compute_manifold_ref(self, path):                                                 # :66-67
        self.manifold_ref = self.compute_manifold(path)

    def realism(self, image):                                                             # :69-77
        feat = self.extract_features(image)
        return realism(self.manifold_ref, feat)

    def compute_manifold(self, input):                                                    # :79-122
        if isinstance(input, str):
            if input.endswith(".npz"):
                print("loading", input)
                f = np.load(input)
                feats, radii = f["feature"], f["radii"]
                f.close()
                return Manifold(feats, radii)
            feats = self.extract_features_from_files(input)
        elif isinstance(input, torch.Tensor):
            feats = self.extract_features(input)
        elif isinstance(input, np.ndarray):
            feats = self.extract_features(torch.Tensor(input))
        elif isinstance(input, list):
            if isinstance(input[0], torch.Tensor):
                feats = self.extract_features(torch.cat(input, dim=0))
            elif isinstance(input[0], np.ndarray):
                feats = self.extract_features(torch.Tensor(np.concatenate(input, axis=0)))
            elif isinstance(input[0], str):
                feats = self.extract_features_from_files(input)
            else:
                raise TypeError
        else:
            print(type(input))
            raise TypeError
        radii = kth_nn_radii(feats, k=self.k)                                             # :119-121
        return Manifold(feats, radii)

    def extract_features(self, images: torch.Tensor) -> np.ndarray:                       # :124-147
        """images: N x C x H x W float (already normalised by the caller), or uint8 [N,224,224,3]."""
        if images.dtype == torch.uint8:
            return extract_features(self.vgg16, images, self.batch_size).cpu().numpy()
        _, _, height, width = images.shape
        if height != 224 or width != 224:
            print("IPR: resizing %s to (224, 224)" % str((height, width)))                # :135-137 (nearest, F.interpolate default)
        feats = []
        for s in range(0, images.shape[0], self.batch_size):
            batch = images[s:s + self.batch_size].cuda().float()
            if height != 224 or width != 224:
                batch = torch.nn.functional.interpolate(batch, size=(224, 224))
            feats.append(self.vgg16(batch.contiguous()).cpu())
        return torch.cat(feats, dim=0).numpy()

    def extract_features_from_files(self, path_or_fnames) -> np.ndarray:                   # :149-172
        if isinstance(path_or_fnames, list):
            fnames = path_or_fnames
        elif isinstance(path_or_fnames, str):
            fnames = glob(os.path.join(path_or_fnames, "**", "*.jpg"), recursive=True) + \
                glob(os.path.join(path_or_fnames, "**", "*.png"), recursive=True)          # :267-270
        else:
            raise TypeError
        if self.num_samples > 0:
            fnames = fnames[:self.num_samples]                                            # :318-319
        if len(fnames) < self.num_samples:
            print("WARNING: num_found_images(%d) < num_samples(%d)" % (len(fnames), self.num_samples))
        return extract_features(self.vgg16, load_resized_224(fnames), self.batch_size).cpu().numpy()

    def save_ref(self, fname):                                                            # :174-178
        print("saving manifold to", fname, "...")
        np.savez_compressed(fname, feature=self.manifold_ref.features, radii=self.manifold_ref.radii)
