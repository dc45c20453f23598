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
    several GPUs (no counterpart in the reference, which computes FID on rank 0 alone)
        -> distributed=True on the functions above: each rank embeds its share of the images, the states are exported,
           all-gathered and folded in rank order (ActivationStatistics.all_reduce_, dcr_fid_merge; DESIGN.md section 4)
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

    @property
    def packed_nbytes(self) -> int:
        """Bytes of one packed state (dcr_fid_packed_size; layout in include/dcr_b200.h)."""
        return int(self.lib.dcr_fid_packed_size(self.dim))

    def export(self) -> torch.Tensor:
        """This state as a packed CUDA uint8 tensor [packed_nbytes], written on the current stream."""
        with torch.cuda.device(self.device):
            out = torch.empty(self.packed_nbytes, dtype=torch.uint8, device=self.device)
            st = torch.cuda.current_stream().cuda_stream
            _lib.check(self.lib.dcr_fid_export(self.handle, out.data_ptr(), st), "dcr_fid_export")
        return out

    def merge_(self, packed: torch.Tensor) -> "ActivationStatistics":
        """Fold packed states (CUDA uint8 [W, packed_nbytes], or one [packed_nbytes]) into this one, in row order.
        Empty states are skipped; a state of another dim raises DcrError."""
        nb = self.packed_nbytes
        if not (packed.is_cuda and packed.dtype == torch.uint8 and packed.dim() in (1, 2) and packed.shape[-1] == nb):
            raise _lib.DcrError(f"merge_ expects CUDA uint8 [W, {nb}] packed states")
        packed = packed.reshape(-1, nb).contiguous()
        with torch.cuda.device(self.device):
            st = torch.cuda.current_stream().cuda_stream
            _lib.check(self.lib.dcr_fid_merge(self.handle, packed.data_ptr(), packed.shape[0], st), "dcr_fid_merge")
        self.count += int(packed[:, 16:24].cpu().contiguous().view(torch.int64).sum())   # header word 2: n
        return self

    def all_reduce_(self, group=None) -> "ActivationStatistics":
        """Replace this state by the statistics of the union of every rank's state in `group` (default: the default
        process group): one all_gather_into_tensor of the packed states, then all W states -- this rank's included --
        are folded into an empty state in rank order, so mu / sigma are bit-identical on every rank and from run to run
        for a given world size.  A no-op with world size 1."""
        import torch.distributed as dist
        world = dist.get_world_size(group)
        if world == 1:
            return self
        mine = self.export()
        gathered = torch.empty(world * mine.numel(), dtype=torch.uint8, device=self.device)   # rank-major
        dist.all_gather_into_tensor(gathered, mine, group=group)
        merged = ActivationStatistics(self.dim, self.device).merge_(gathered.view(world, -1))
        self.lib.dcr_fid_destroy(self.handle)
        self.handle, merged.handle = merged.handle, None
        self.count = merged.count
        return self


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


def _group_of(distributed):
    """The `distributed=` argument of the functions below -> (process group, world size).  False: this process computes
    everything (world 1); True: shard over the default process group; a ProcessGroup: shard over it."""
    if distributed is False or distributed is None:
        return None, 1
    import torch.distributed as dist
    if not dist.is_initialized():
        raise _lib.DcrError("distributed=... needs an initialized torch.distributed process group")
    group = None if distributed is True else distributed
    return group, dist.get_world_size(group)


def _chunk_rows(net: DcrNet, batch_size: int) -> int:
    """Images per accumulate call: the features of a chunk are folded into the statistics at once."""
    return max(batch_size, net.max_batch) * 8


def statistics_of_images(net: DcrNet, images_u8: torch.Tensor, batch_size: int = 50, *,
                         distributed=False) -> Tuple[np.ndarray, np.ndarray]:
    """calculate_activation_statistics (metrics/fid.py:199-221) for uint8 [N,299,299,3] images (host or device).
    distributed=True (or a process group): `images_u8` is this rank's share of the set and the statistics of the union
    over the ranks are returned on every rank (a collective: every rank of the group must call it)."""
    group, world = _group_of(distributed)
    stats = ActivationStatistics(net.out_dim, net.device)
    n = images_u8.shape[0]
    chunk = _chunk_rows(net, batch_size)
    for s in range(0, n, chunk):
        stats.update(extract_features(net, images_u8[s:s + chunk], batch_size))
    if world > 1:
        stats.all_reduce_(group)
    return stats.finalize()


def fid_from_images(net: DcrNet, real_u8: torch.Tensor, gen_u8: torch.Tensor, batch_size: int = 50, *,
                    distributed=False) -> float:
    """calculate_fid_given_paths (metrics/fid.py:239-255) on already decoded + resized images (with distributed=...:
    this rank's shares of both sets, see statistics_of_images)."""
    m1, s1 = statistics_of_images(net, real_u8, batch_size, distributed=distributed)
    m2, s2 = statistics_of_images(net, gen_u8, batch_size, distributed=distributed)
    return frechet_distance(m1, s1, m2, s2)


def image_files(path: str):
    """All **/*.JPEG|png|jpg under `path`, in the glob order of metrics/fid.py:231."""
    import glob
    import os
    if not os.path.exists(path):
        raise RuntimeError("Invalid path: %s" % path)                                       # fid.py:243
    return (list(glob.glob(os.path.join(path, "**/*.JPEG"), recursive=True)) +
            list(glob.glob(os.path.join(path, "**/*.png"), recursive=True)) +
            list(glob.glob(os.path.join(path, "**/*.jpg"), recursive=True)))


def _resize_transform(size: int):
    from torchvision import transforms
    return transforms.Compose([transforms.Resize(size), transforms.CenterCrop(size)])


def _decode(f: str, tf) -> torch.Tensor:
    from PIL import Image
    return torch.from_numpy(np.array(tf(Image.open(f).convert("RGB"))))


def load_resized(path: str, size: int = 299) -> torch.Tensor:
    """All **/*.JPEG|png|jpg under `path` (glob order of metrics/fid.py:231), PIL RGB, Resize(299) bilinear +
    CenterCrop(299) as metrics/fid.py:104-107 -> uint8 [N,299,299,3]."""
    files = image_files(path)
    tf = _resize_transform(size)
    out = torch.empty((len(files), size, size, 3), dtype=torch.uint8)
    for i, f in enumerate(files):
        out[i] = _decode(f, tf)
    return out


def statistics_of_files(net: DcrNet, files, batch_size: int = 50, num_workers: int = 1, size: int = 299
                        ) -> ActivationStatistics:
    """The activation statistics of image files (decoded and resized as load_resized does), streamed: `num_workers`
    threads decode chunk i+1 while the GPU embeds chunk i, so host memory holds about two chunks.  The chunks are those
    statistics_of_images cuts, so the result is bit-identical to statistics_of_images(net, load_resized(...))."""
    from concurrent.futures import ThreadPoolExecutor
    stats = ActivationStatistics(net.out_dim, net.device)
    chunk = _chunk_rows(net, batch_size)
    tf = _resize_transform(size)
    with ThreadPoolExecutor(max(1, num_workers)) as ex:
        nxt = [ex.submit(_decode, f, tf) for f in files[:chunk]]
        for s in range(0, len(files), chunk):
            cur, nxt = nxt, [ex.submit(_decode, f, tf) for f in files[s + chunk:s + 2 * chunk]]
            stats.update(extract_features(net, torch.stack([fut.result() for fut in cur]), batch_size))
    return stats


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


def compute_statistics_of_path(path: str, net: DcrNet, batch_size: int = 50, *, num_workers: int = 1,
                               distributed=False) -> Tuple[np.ndarray, np.ndarray]:
    """metrics/fid.py:224-236: a `.npz` with mu/sigma is loaded, anything else is globbed for images, which
    `num_workers` threads decode (statistics_of_files).  distributed=True (or a process group): every rank embeds its
    contiguous share of the file list (dist.shard_bounds) and the statistics of the whole folder are returned on every
    rank; every rank of the group must call it.  A `.npz` is read on every rank, without a collective."""
    if path.endswith(".npz"):
        with np.load(path) as f:
            return f["mu"][:], f["sigma"][:]
    group, world = _group_of(distributed)
    files = image_files(path)
    if world > 1:
        import torch.distributed as dist

        from .dist import shard_bounds
        lo, hi = shard_bounds(len(files), dist.get_rank(group), world)
        files = files[lo:hi]
    stats = statistics_of_files(net, files, batch_size, num_workers)
    if world > 1:
        stats.all_reduce_(group)
    return stats.finalize()


def _is_rank0(distributed) -> bool:
    group, world = _group_of(distributed)
    if world == 1:
        return True
    import torch.distributed as dist
    return dist.get_rank(group) == 0


def calculate_fid_given_paths(paths, batch_size: int = 50, device=None, dims: int = 2048, num_workers: int = 1,
                              weights=None, precision: str = "fast", *, distributed=False) -> float:
    """metrics/fid.py:239-255.  `device` is accepted for signature compatibility (the current CUDA device is used);
    `num_workers` threads decode the images.  dims in {64, 192, 768, 2048} select the feature block as
    InceptionV3.BLOCK_INDEX_BY_DIM does (metrics/inception.py:22-28); 2048 is what diff_retrieval.py:597-600 asks for.
    distributed=True (or a process group) shards both folders over the ranks (compute_statistics_of_path) and returns
    the same FID on every rank.  It is a collective: leave it off at a call site that only rank 0 reaches (the
    reference's `if args.rank == 0:` block, diff_retrieval.py:375), or that rank waits for the others forever.  The
    argument checks run on every rank before any collective, so a bad path raises everywhere."""
    import os
    for p in paths:
        if not os.path.exists(p):
            raise RuntimeError("Invalid path: %s" % p)                                       # fid.py:241-243
    if _is_rank0(distributed):
        print(dims)                                                                          # fid.py:244
    net = _build_inception(weights, batch_size, precision, dims)
    m1, s1 = compute_statistics_of_path(paths[0], net, batch_size, num_workers=num_workers, distributed=distributed)
    m2, s2 = compute_statistics_of_path(paths[1], net, batch_size, num_workers=num_workers, distributed=distributed)
    return frechet_distance(m1, s1, m2, s2)


def save_fid_stats(paths, batch_size: int = 50, device=None, dims: int = 2048, num_workers: int = 1, weights=None,
                   precision: str = "fast", *, distributed=False) -> None:
    """metrics/fid.py:258-275: statistics of paths[0] written to the .npz paths[1].  With distributed=True (or a process
    group) the ranks share the images and rank 0 writes the file; every rank returns once it exists."""
    import os
    if not os.path.exists(paths[0]):
        raise RuntimeError("Invalid path: %s" % paths[0])
    if os.path.exists(paths[1]):
        raise RuntimeError("Existing output file: %s" % paths[1])
    net = _build_inception(weights, batch_size, precision, dims)
    rank0 = _is_rank0(distributed)
    if rank0:
        print(f"Saving statistics for {paths[0]}")
    m1, s1 = compute_statistics_of_path(paths[0], net, batch_size, num_workers=num_workers, distributed=distributed)
    if rank0:
        np.savez_compressed(paths[1], mu=m1, sigma=s1)
    group, world = _group_of(distributed)
    if world > 1:
        import torch.distributed as dist
        dist.barrier(group)
