"""Descriptor networks on the dcr_net executor (libdcr_b200.so).

Host-side mirror of the reference's model zoo for the hot path:

    --pt_style sscd  --arch resnet50 | resnet50_im | resnet50_disc     diff_retrieval.py:277-285
        torch.jit.load(sscd_*.torchscript.pt): ResNet-50 trunk -> GeM(p=3) -> Linear(2048,512) -> L2
        (architecture from facebookresearch/sscd-copy-detection; not vendored in the reference -- SURVEY.md 8c)
    --pt_style dino  --arch vit_small  ->  dino_vits.dino_vits16           diff_retrieval.py:251-252, dino_vits.py:340
        VisionTransformer(patch 16, dim 384, depth 12, heads 6)            dino_vits.py:171-289

Each builder takes a state_dict (real weights when the user has them, seeded random weights in the tests), folds
BatchNorm into a per-channel affine, lays the weights out for the wgmma GEMM kernel and records the op list.
`forward` takes a uint8 NHWC image batch on the GPU and returns fp32 descriptors -- the resize/crop/ToTensor/
Normalize of diff_retrieval.py:325-330 is fused into the first op.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional, Sequence

import numpy as np
import torch

from . import _lib
from .ops import prepare_conv_weight

OP_IM2COL_U8, OP_CONV, OP_MAXPOOL, OP_AVGPOOL, OP_GEM, OP_GAP, OP_LAYERNORM, OP_VIT_TOKENS, OP_ATTENTION, \
    OP_L2NORM_OUT, OP_STEM_S2D, OP_EMBED, OP_STEM_ROWS, OP_STEM_CONV = range(14)

# fast/bf16: one bf16 plane, tensor cores.  parity/fp32: three planes (exact fp32 values), 6 tensor-core cross terms.
# exact: three planes, products accumulated in float64 on the CUDA cores (correctly rounded fp32 layer outputs).
# "s2d": 7x7/2 stem as a 4x4 window convolution over a space-to-depth tensor (conv_gemm.cu, every mode);
# "toeplitz": fused stem kernel with overlapping-window operand descriptors (stem_fused.cu, fast mode);
# "toeplitz_pool": the same with the 3x3/2 max pool taken in its epilogue (default of the fast mode: the stem activation
# never reaches HBM)
DEFAULT_STEM = "toeplitz_pool"
PRECISION_PLANES = {"fast": 1, "bf16": 1, "parity": 3, "fp32": 3, "bf16x3": 2, "exact": 3}


class DcrNet:
    """Thin owner of a dcr_net handle."""

    def __init__(self, max_batch: int, precision: str = "fast", device: Optional[torch.device] = None):
        self.lib = _lib.load()
        if not torch.cuda.is_available():
            raise _lib.DcrError("dcr_b200 networks need a CUDA (sm_90a) device; there is no CPU path")
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.max_batch = int(max_batch)
        self.planes = PRECISION_PLANES[precision]
        self.precision = precision
        self.out_dim = 0
        self.in_shape = None          # (IH, IW) expected uint8 input
        self.net_input = None         # (H, W) of the transformed fp32 input (after the centre crop)
        self.flops_per_image = 0.0
        self.meta = []                # one entry per op, in launch order (tools/layer_profile.py)
        h = C.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(self.lib.dcr_net_create(self.max_batch, self.planes, C.byref(h)), "dcr_net_create")
            if precision == "exact":
                _lib.check(self.lib.dcr_net_set_exact(h, 1), "dcr_net_set_exact")
        self.handle = h

    def __del__(self):
        try:
            if getattr(self, "handle", None):
                self.lib.dcr_net_destroy(self.handle)
                self.handle = None
        except Exception:
            pass

    def fork(self) -> "DcrNet":
        """A second executor of this (fully built) network: own activation buffers, the same device weights.  Two batches
        can then be in flight on two streams (retrieval.extract_features does that)."""
        import copy
        twin = copy.copy(self)
        twin.handle = None
        h = C.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(self.lib.dcr_net_fork(self.handle, C.byref(h)), "dcr_net_fork")
        twin.handle = h
        twin._twin = None
        return twin

    def twin(self) -> "DcrNet":
        """The cached fork extract_features alternates with."""
        if getattr(self, "_twin", None) is None:
            self._twin = self.fork()
        return self._twin

    # ---- graph construction -------------------------------------------------------------------------------------
    def tensor(self, rows_per_image: int, channels: int) -> int:
        with torch.cuda.device(self.device):
            r = self.lib.dcr_net_add_tensor(self.handle, rows_per_image, channels)
        if r < 0:
            raise _lib.DcrError(f"dcr_net_add_tensor: {_lib.last_error()}")
        return r

    def alias(self, src: int, rows_per_image: int, channels: int) -> int:
        r = self.lib.dcr_net_alias_tensor(self.handle, src, rows_per_image, channels)
        if r < 0:
            raise _lib.DcrError(f"dcr_net_alias_tensor: {_lib.last_error()}")
        return r

    def param(self, t: torch.Tensor) -> int:
        t = t.detach().contiguous().cpu()
        with torch.cuda.device(self.device):
            r = self.lib.dcr_net_add_param(self.handle, t.data_ptr(), t.numel() * t.element_size())
        if r < 0:
            raise _lib.DcrError(f"dcr_net_add_param: {_lib.last_error()}")
        return r

    def param_f32(self, t: torch.Tensor) -> int:
        return self.param(t.detach().float())

    def weight(self, w: torch.Tensor) -> int:
        """conv / linear weight -> prepared bf16 planes."""
        return self.param(prepare_conv_weight(w.detach().float().cpu(), self.planes))

    def op(self, kind: int, iargs: Sequence[int], fargs: Sequence[float] = ()) -> int:
        ia = (C.c_int * len(iargs))(*[int(v) for v in iargs])
        fa = (C.c_float * max(1, len(fargs)))(*[float(v) for v in fargs])
        r = self.lib.dcr_net_add_op(self.handle, kind, ia, len(iargs), fa, len(fargs))
        self.meta.append((kind, [int(v) for v in iargs]))
        if r < 0:
            raise _lib.DcrError(f"dcr_net_add_op(kind={kind}): {_lib.last_error()}")
        return r

    def set_output(self, dim: int) -> None:
        with torch.cuda.device(self.device):
            _lib.check(self.lib.dcr_net_set_output(self.handle, dim), "dcr_net_set_output")
        self.out_dim = dim

    def conv(self, in_t: int, out_t: int, h: int, w: int, c: int, weight: torch.Tensor, *, stride: int = 1,
             pad: Sequence[int] = (0, 0), scale: Optional[torch.Tensor] = None, bias: Optional[torch.Tensor] = None,
             residual: int = -1, act: int = 0, out_col_off: int = 0, to_output: bool = False,
             window: Optional[Sequence[int]] = None) -> None:
        if weight.dim() == 2:
            n, kh, kw = weight.shape[0], 1, 1
        else:
            n, _, kh, kw = weight.shape
        ho = (h + 2 * pad[0] - kh) // stride + 1
        wo = (w + 2 * pad[1] - kw) // stride + 1
        self.flops_per_image += 2.0 * ho * wo * n * c * kh * kw
        self.op(OP_CONV, [in_t, out_t, h, w, c, self.weight(weight), n, kh, kw, stride, pad[0], pad[1],
                          self.param_f32(scale) if scale is not None else -1,
                          self.param_f32(bias) if bias is not None else -1, residual, act, out_col_off,
                          1 if to_output else 0] + (list(window) if window else []))

    # ---- execution ----------------------------------------------------------------------------------------------
    @torch.no_grad()
    def forward(self, images: torch.Tensor) -> torch.Tensor:
        """Two input forms, same network and kernels:
          * CUDA uint8 [n, IH, IW, 3]: raw images; Resize/CenterCrop/ToTensor/Normalize (diff_retrieval.py:325-330) run
            fused in the first kernel (the fast path: 3 bytes per pixel cross PCIe / HBM instead of 12);
          * CUDA float32 [n, 3, H, W]: the tensor the reference's own loop passes to `model(samples)`
            (utils_ret.py:751, embedding_search/utils.py:101, metrics/fid.py:126) -- already transformed by the
            caller's torchvision pipeline; H x W must be the network's input size (self.net_input).
        Returns fp32 [n, out_dim] on the same device."""
        if not (isinstance(images, torch.Tensor) and images.is_cuda and images.dim() == 4):
            raise _lib.DcrError("forward expects a CUDA tensor: uint8 [n, H, W, 3] or float32 [n, 3, H, W]")
        f32 = images.dtype == torch.float32
        if f32:
            if images.shape[1] != 3:
                raise _lib.DcrError(f"float32 input must be NCHW with 3 channels, got {tuple(images.shape)}")
            if self.net_input is not None and tuple(images.shape[2:4]) != tuple(self.net_input):
                raise _lib.DcrError(f"network takes {self.net_input} transformed inputs, got {tuple(images.shape[2:4])}")
        elif images.dtype == torch.uint8:
            if images.shape[3] != 3:
                raise _lib.DcrError("uint8 input must be NHWC with 3 channels")
            if self.in_shape is not None and tuple(images.shape[1:3]) != tuple(self.in_shape):
                raise _lib.DcrError(f"network was built for {self.in_shape} inputs, got {tuple(images.shape[1:3])}")
        else:
            raise _lib.DcrError(f"forward expects uint8 or float32 input, got {images.dtype}")
        images = images.contiguous()
        n = images.shape[0]
        out = torch.empty((n, self.out_dim), dtype=torch.float32, device=images.device)
        fwd = self.lib.dcr_net_forward_f32 if f32 else self.lib.dcr_net_forward
        with torch.cuda.device(images.device):
            st = torch.cuda.current_stream().cuda_stream
            for s in range(0, n, self.max_batch):
                b = min(self.max_batch, n - s)
                rc = fwd(self.handle, images[s:s + b].data_ptr(), b, out[s:s + b].data_ptr(), st)
                _lib.check(rc, "dcr_net_forward")
        return out

    __call__ = forward

    @torch.no_grad()
    def forward_tokens(self, ids: torch.Tensor) -> torch.Tensor:
        """Text networks (first op EMBED): ids CUDA int32/int64 [n, T] -> fp32 [n, out_dim]."""
        if not (isinstance(ids, torch.Tensor) and ids.is_cuda and ids.dim() == 2):
            raise _lib.DcrError("forward_tokens expects a CUDA integer tensor [n, T]")
        ids = ids.to(torch.int32).contiguous()
        n = ids.shape[0]
        out = torch.empty((n, self.out_dim), dtype=torch.float32, device=ids.device)
        with torch.cuda.device(ids.device):
            st = torch.cuda.current_stream().cuda_stream
            for s in range(0, n, self.max_batch):
                b = min(self.max_batch, n - s)
                rc = self.lib.dcr_net_forward(self.handle, ids[s:s + b].data_ptr(), b, out[s:s + b].data_ptr(), st)
                _lib.check(rc, "dcr_net_forward")
        return out


def _fold_bn(sd: Dict[str, torch.Tensor], prefix: str, eps: float):
    g, b = sd[prefix + ".weight"].double(), sd[prefix + ".bias"].double()
    m, v = sd[prefix + ".running_mean"].double(), sd[prefix + ".running_var"].double()
    scale = g / torch.sqrt(v + eps)
    return scale.float(), (b - m * scale).float()


def _strip(sd: Dict[str, torch.Tensor], prefixes: Sequence[str]) -> Dict[str, torch.Tensor]:
    out = {}
    for k, v in sd.items():
        for p in prefixes:
            if k.startswith(p):
                k = k[len(p):]
                break
        out[k] = v
    return out


def _stem_s2d_weight(w: torch.Tensor) -> torch.Tensor:
    """[N,3,7,7] -> [N, 64, 4, 1]: tap a = filter row pair, channel c' = b*16 + (i*2+j)*3 + c holds w[n, c, 2a+i, 2b+j]
    (zero where 2a+i or 2b+j exceeds 6, and for the 4 padding channels of every stored pixel)."""
    n = w.shape[0]
    out = torch.zeros((n, 64, 4, 1), dtype=torch.float32)
    wf = w.detach().float()
    for a in range(4):
        for b in range(4):
            for i in range(2):
                for j in range(2):
                    r, s = 2 * a + i, 2 * b + j
                    if r < 7 and s < 7:
                        base = b * 16 + (i * 2 + j) * 3
                        out[:, base:base + 3, a, 0] = wf[:, :, r, s]
    return out


def _stem_toeplitz_weight(w: torch.Tensor) -> torch.Tensor:
    """[N,3,7,7] -> [N, 256] for csrc/stem_fused.cu: k = ((a*2 + e)*4 + b)*8 + i*3 + c holds w[n, c, 2a+i, 2b+e]
    (a, b: filter row / column pair, i, e: row / column parity; zero where 2a+i or 2b+e exceeds 6 and for the two
    padding channels of every 8-channel unit)."""
    n = w.shape[0]
    out = torch.zeros((n, 256), dtype=torch.float32)
    wf = w.detach().float()
    for a in range(4):
        for e in range(2):
            for b in range(4):
                for i in range(2):
                    r, s = 2 * a + i, 2 * b + e
                    if r < 7 and s < 7:
                        k0 = ((a * 2 + e) * 4 + b) * 8 + i * 3
                        out[:, k0:k0 + 3] = wf[:, :, r, s]
    return out


def first_conv_k_pad(kh: int, kw: int) -> int:
    """K of the im2col rows the IM2COL_U8 op emits: each filter row padded to ceil8(3*kw), total padded to 64."""
    rp = (3 * kw + 7) // 8 * 8
    return (kh * rp + 63) // 64 * 64


def _first_conv_weight(w: torch.Tensor, k_pad: int) -> torch.Tensor:
    """[N,3,kh,kw] -> [N, k_pad] in the layout im2col_u8 emits: k = r*RP + s*3 + c, RP = ceil8(3*kw), zero padded."""
    n, _, kh, kw = w.shape
    rp = (3 * kw + 7) // 8 * 8
    rows = torch.zeros((n, kh, rp), dtype=torch.float32)
    rows[:, :, :3 * kw] = w.detach().float().permute(0, 2, 3, 1).reshape(n, kh, 3 * kw)
    out = torch.zeros((n, k_pad), dtype=torch.float32)
    out[:, :kh * rp] = rows.reshape(n, kh * rp)
    return out


def _scaled_size(size: int, scale_factor: Optional[float]) -> int:
    """Output size of F.interpolate(scale_factor=s) (multi_scale, utils_ret.py:676-698); None or 1 = no resizing."""
    if scale_factor is None or scale_factor == 1:
        return size
    import math
    return int(math.floor(float(size) * float(scale_factor)))


def _input_op(net: DcrNet, kind: int, out_t: int, in_size: int, crop: int, mean: Sequence[float], std: Sequence[float],
              op_ints: Sequence[int] = (), post: Sequence[float] = (1.0, 0.0), scale_factor: Optional[float] = None) -> None:
    """An op that reads the image batch (IM2COL_U8, STEM_S2D, STEM_ROWS): the centre `crop` of the in_size x in_size
    image, ToTensor, Normalize(mean, std), the affine `post`, then the bilinear resize by `scale_factor`.
    ints [out_t, IH, IW, crop_y, crop_x, H, W] + op_ints (+ [RH, RW]), floats mean + std + post (+ [float(1 / s)])."""
    off = (in_size - crop) // 2
    iargs = [out_t, in_size, in_size, off, off, crop, crop, *op_ints]
    fargs = [*mean, *std, *post]
    if scale_factor is not None and scale_factor != 1:
        size = _scaled_size(crop, scale_factor)
        iargs += [size, size]
        fargs.append(float(np.float32(1.0 / float(scale_factor))))
    net.op(kind, iargs, fargs)


def _dense_from_grouped(w: torch.Tensor, c_in: int) -> torch.Tensor:
    """Grouped convolution weight [N, c_in/groups, kh, kw] -> the equivalent dense block-diagonal weight
    [N, c_in, kh, kw].  The tensor cores then run the grouped 3x3 convs of a ResNeXt trunk as ordinary dense
    implicit GEMMs (zeros included): `groups` times the arithmetic of the grouped form, but at the widths involved
    (128..1024 channels) that is still tensor-bound work at full tile efficiency, where per-group GEMMs with 4..32
    output channels would use a few percent of a wgmma tile."""
    n, cpg, kh, kw = w.shape
    if cpg == c_in:
        return w
    groups = c_in // cpg
    if cpg * groups != c_in or n % groups:
        raise _lib.DcrError(f"grouped conv weight {tuple(w.shape)} does not divide {c_in} input channels")
    npg = n // groups
    dense = torch.zeros((n, c_in, kh, kw), dtype=w.dtype)
    for g in range(groups):
        dense[g * npg:(g + 1) * npg, g * cpg:(g + 1) * cpg] = w[g * npg:(g + 1) * npg]
    return dense


# ------------------------------------------------------------------------------------------------------------------
# SSCD: ResNet / ResNeXt bottleneck trunk + GeM + Linear + L2
def build_sscd_resnet50(state_dict: Dict[str, torch.Tensor], max_batch: int = 64, precision: str = "fast",
                        mean: Sequence[float] = (0.5, 0.5, 0.5), std: Sequence[float] = (0.5, 0.5, 0.5),
                        in_size: int = 256, crop: int = 224, gem_p: float = 3.0, gem_eps: float = 1e-6,
                        l2_normalize: bool = True, scale_factor: Optional[float] = None,
                        stem: Optional[str] = None) -> DcrNet:
    """state_dict keys: torchvision ResNet names, optionally prefixed 'backbone.' / 'module.'; head Linear under
    'embeddings.1' (SSCD), 'fc' or 'head'.  mean/std: (0.5, 0.5) for diff_retrieval.py:329, ImageNet statistics for
    embedding_search/utils.py:37-39.
    The trunk is read off the state_dict: blocks per stage, bottleneck width and group count are whatever the tensors
    say, so the same builder serves sscd_disc_mixup / sscd_imagenet_mixup (ResNet-50, 512-d; `--arch resnet50`,
    `resnet50_im`, diff_retrieval.py:278-281) and sscd_disc_large (`--arch resnet50_disc`, :282-283 -- upstream a
    ResNeXt-101 with a 1024-d head [unverified]); grouped 3x3 convs run as dense block-diagonal GEMMs."""
    sd = _strip({k: v.detach().cpu() for k, v in state_dict.items()}, ["module.", "model."])
    sd = _strip(sd, ["backbone."])
    head_w = head_b = None
    for hp in ("embeddings.1", "embeddings.0", "fc", "head"):
        if hp + ".weight" in sd and sd[hp + ".weight"].dim() == 2:
            head_w, head_b = sd[hp + ".weight"], sd.get(hp + ".bias")
            break
    if head_w is None:
        raise _lib.DcrError("SSCD state_dict has no head Linear (embeddings.1 / fc / head)")
    net = DcrNet(max_batch, precision)
    net.in_shape = (in_size, in_size)
    net.net_input = (crop, crop)
    eps = 1e-5
    src_crop = crop
    # multi_scale (utils_ret.py:676-698): the transformed crop is bilinearly resized by `scale_factor` before the
    # network; fused into the stem's input kernel
    crop = _scaled_size(src_crop, scale_factor)
    if scale_factor not in (None, 1) and crop % 2:
        raise _lib.DcrError(f"scale_factor {scale_factor} gives an odd network input size {crop}")
    # stem: 7x7/2/pad-3 conv == 4x4/1 conv over the zero-padded 2x2 space-to-depth input (12 -> 16 channels); the
    # preprocessing (crop, ToTensor, Normalize) is fused into the space-to-depth kernel, and the GEMM kernel reads 4
    # horizontally adjacent 16-channel pixels as one 64-channel pixel through an overlapping-window tensor map
    s = (crop + 2 * 3 - 7) // 2 + 1   # 112
    u = (crop + 6) // 2               # 115 stored rows / pixels per row
    sc, bi = _fold_bn(sd, "bn1", eps)
    hw = (s + 2 - 3) // 2 + 1         # 56
    if stem is None:
        stem = DEFAULT_STEM if (net.planes == 1 and sd["conv1.weight"].shape[0] == 64) else "s2d"
    if stem in ("toeplitz", "toeplitz_pool"):
        # fused stem (csrc/stem_fused.cu): the input is stored once as two column-parity planes of 16-byte pixels and the
        # tensor cores read overlapping windows of it -- each pixel enters shared memory ~1.7 times instead of 16.
        # "toeplitz_pool" also takes the 3x3/2 max pool in the epilogue: the 112x112x64 activation never reaches HBM.
        if net.planes != 1 or sd["conv1.weight"].shape[0] != 64:
            raise _lib.DcrError("stem='toeplitz' needs the one-plane (fast) mode and a 64-channel stem")
        units = int(net.lib.dcr_stem_plane_units(s, s))
        t_rows = net.tensor(2 * units, 8)
        _input_op(net, OP_STEM_ROWS, t_rows, in_size, src_crop, mean, std, scale_factor=scale_factor)
        w_id = net.param(_stem_toeplitz_weight(sd["conv1.weight"]).to(torch.bfloat16))
        pooled = stem == "toeplitz_pool"
        t_stem = net.tensor(hw * hw if pooled else s * s, 64)
        net.op(OP_STEM_CONV, [t_rows, t_stem, s, s, w_id, net.param_f32(sc), net.param_f32(bi), 1 if pooled else 0])
        net.flops_per_image += 2.0 * s * s * 64 * 147
        if pooled:
            t = t_stem
        else:
            t = net.tensor(hw * hw, 64)
            net.op(OP_MAXPOOL, [t_stem, t, s, s, 64, 3, 2, 1, 0])
    else:
        t_stem = net.tensor(s * s, 64)
        t_z = net.tensor(u * u, 16)
        _input_op(net, OP_STEM_S2D, t_z, in_size, src_crop, mean, std, scale_factor=scale_factor)
        net.conv(t_z, t_stem, u, u - 3, 64, _stem_s2d_weight(sd["conv1.weight"]), scale=sc, bias=bi, act=1, window=(16, u))
        net.flops_per_image += 2.0 * s * s * 64 * (147 - 256)   # count the real 147-tap work, not the zero padding
        t = net.tensor(hw * hw, 64)
        net.op(OP_MAXPOOL, [t_stem, t, s, s, 64, 3, 2, 1, 0])
    c_in = 64
    for li, stride in enumerate([1, 2, 2, 2], start=1):
        blocks = 0
        while f"layer{li}.{blocks}.conv1.weight" in sd:
            blocks += 1
        if blocks == 0:
            raise _lib.DcrError(f"SSCD state_dict has no layer{li} blocks")
        for bi_ in range(blocks):
            pre = f"layer{li}.{bi_}"
            st = stride if bi_ == 0 else 1
            hw_out = (hw + 2 - 3) // st + 1
            width = sd[pre + ".conv1.weight"].shape[0]        # bottleneck width (64.. for ResNet-50, 128.. for 32x4d)
            c_out = sd[pre + ".conv3.weight"].shape[0]
            t1 = net.tensor(hw * hw, width)
            sc, bi = _fold_bn(sd, pre + ".bn1", eps)
            net.conv(t, t1, hw, hw, c_in, sd[pre + ".conv1.weight"], scale=sc, bias=bi, act=1)
            t2 = net.tensor(hw_out * hw_out, width)
            sc, bi = _fold_bn(sd, pre + ".bn2", eps)
            w2 = sd[pre + ".conv2.weight"]
            net.flops_per_image -= 2.0 * hw_out * hw_out * width * 9 * (width - w2.shape[1])   # zeros of the dense form
            net.conv(t1, t2, hw, hw, width, _dense_from_grouped(w2, width), stride=st, pad=(1, 1), scale=sc, bias=bi, act=1)
            ident = t
            if pre + ".downsample.0.weight" in sd:
                ident = net.tensor(hw_out * hw_out, c_out)
                sc, bi = _fold_bn(sd, pre + ".downsample.1", eps)
                net.conv(t, ident, hw, hw, c_in, sd[pre + ".downsample.0.weight"], stride=st, scale=sc, bias=bi)
            t3 = net.tensor(hw_out * hw_out, c_out)
            sc, bi = _fold_bn(sd, pre + ".bn3", eps)
            net.conv(t2, t3, hw_out, hw_out, width, sd[pre + ".conv3.weight"], scale=sc, bias=bi, residual=ident, act=1)
            t, c_in, hw = t3, c_out, hw_out
    d = head_w.shape[0]
    net.set_output(d)
    t_pool = net.tensor(1, c_in)
    net.op(OP_GEM, [t, t_pool, hw * hw, c_in, 0], [gem_p, gem_eps])
    net.conv(t_pool, -1, 1, 1, c_in, head_w, bias=head_b, to_output=True)
    if l2_normalize:     # SSCD's final L2Norm; off only for calibration / inspection of the raw embedding
        net.op(OP_L2NORM_OUT, [], [1e-12])
    return net


def interpolate_pos_embed(pos_embed: torch.Tensor, grid_h: int, grid_w: int) -> torch.Tensor:
    """Host-side parameter preparation for a ViT run at another input size: the reference resamples the patch position
    embeddings bicubically at every forward (dino_vits.py:213-233, including its `+ 0.1` on the target grid); here it
    happens once when the network is built.  pos_embed [1, 1 + n*n, dim] -> [1, 1 + grid_h * grid_w, dim]."""
    import math
    n = pos_embed.shape[1] - 1
    side = int(math.sqrt(n))
    if side * side != n:
        raise _lib.DcrError(f"pos_embed with {n} patch positions is not a square grid")
    if grid_h == side and grid_w == side:
        return pos_embed
    dim = pos_embed.shape[-1]
    pe = pos_embed.detach().float().cpu()
    patch_pos = pe[:, 1:].reshape(1, side, side, dim).permute(0, 3, 1, 2)
    patch_pos = torch.nn.functional.interpolate(patch_pos, scale_factor=((grid_h + 0.1) / side, (grid_w + 0.1) / side),
                                                mode="bicubic")
    if patch_pos.shape[-2] != grid_h or patch_pos.shape[-1] != grid_w:
        raise _lib.DcrError("position-embedding interpolation produced an unexpected grid")
    patch_pos = patch_pos.permute(0, 2, 3, 1).reshape(1, grid_h * grid_w, dim)
    return torch.cat((pe[:, :1], patch_pos), dim=1)


# ------------------------------------------------------------------------------------------------------------------
# DINO ViT (dino_vits.py:171-289)
def build_dino_vit(state_dict: Dict[str, torch.Tensor], max_batch: int = 64, precision: str = "fast",
                   mean: Sequence[float] = (0.5, 0.5, 0.5), std: Sequence[float] = (0.5, 0.5, 0.5),
                   in_size: int = 256, crop: int = 224, patch: Optional[int] = None,
                   heads: Optional[int] = None, scale_factor: Optional[float] = None, n_last_layers: int = 1,
                   global_pool: str = "token") -> DcrNet:
    """Width, depth, patch size and head count are read off the state_dict (64-dim heads, as every DINO ViT):
    vit_small/16 (`dino_vits16`, dino_vits.py:340-352; 384-d), vit_base/16 (`dino_vitb16`, :366-378; 768-d) and the
    patch-8 variants (`dino_vitb8`, :381-393: 785 tokens, streamed-KV attention kernel).
    scale_factor: `multi_scale` (utils_ret.py:676-698) -- the transformed crop is bilinearly resized before the patch
      embedding (fused into the first kernel) and the position embeddings are resampled as dino_vits.py:213-233 does.
    n_last_layers: `--layer n` (utils_ret.py:732,745): the normed output of block depth - n, i.e.
      `get_intermediate_layers(x, n)[0]` (dino_vits.py:267-275); 1 = the ordinary forward.
    global_pool: 'token' -> the CLS row [B, dim] (dino_vits.py:253-254); '' -> every token, flattened to
      [B, tokens * dim] as `rearrange(feats, 'b h w -> b (h w)')` does for --similarity_metric splitloss
      (dino_vits.py:255-256, utils_ret.py:728-737)."""
    sd =_strip({k: v.detach().cpu() for k, v in state_dict.items()}, ["module.", "backbone."])
    dim = sd["cls_token"].shape[-1]
    depth = 1 + max(int(k.split(".")[1]) for k in sd if k.startswith("blocks."))
    if not 1 <= n_last_layers <= depth:
        raise _lib.DcrError(f"--layer {n_last_layers} outside [1, {depth}]")
    if global_pool not in ("token", ""):
        raise _lib.DcrError(f"global_pool must be 'token' or '', got {global_pool!r}")
    depth_used = depth - n_last_layers + 1
    patch = int(sd["patch_embed.proj.weight"].shape[-1]) if patch is None else patch
    heads = dim // 64 if heads is None else heads
    net_in = _scaled_size(crop, scale_factor)
    grid = (net_in - patch) // patch + 1
    n_patch = grid * grid
    tokens = n_patch + 1
    if sd["pos_embed"].shape[1] != tokens:
        # another input size than the checkpoint's: resample the position embeddings as the reference does
        # (dino_vits.py:213-233)
        sd = dict(sd)
        sd["pos_embed"] = interpolate_pos_embed(sd["pos_embed"], grid, grid)
    net = DcrNet(max_batch, precision)
    net.in_shape = (in_size, in_size)
    net.net_input = (crop, crop)
    k_pad = first_conv_k_pad(patch, patch)
    t_cols = net.tensor(n_patch, k_pad)
    _input_op(net, OP_IM2COL_U8, t_cols, in_size, crop, mean, std, [patch, patch, patch, 0, k_pad], scale_factor=scale_factor)
    t_patch = net.tensor(n_patch, dim)
    net.conv(t_cols, t_patch, n_patch, 1, k_pad, _first_conv_weight(sd["patch_embed.proj.weight"], k_pad),
             bias=sd["patch_embed.proj.bias"])
    x = net.tensor(tokens, dim)
    net.op(OP_VIT_TOKENS, [t_patch, x, n_patch, dim, net.param_f32(sd["cls_token"].reshape(-1)),
                           net.param_f32(sd["pos_embed"].reshape(tokens, dim))])
    dh = dim // heads
    for i in range(depth_used):
        pre = f"blocks.{i}"
        t_ln = net.tensor(tokens, dim)
        net.op(OP_LAYERNORM, [x, t_ln, tokens, dim, net.param_f32(sd[pre + ".norm1.weight"]),
                              net.param_f32(sd[pre + ".norm1.bias"]), 1, 0], [1e-6])
        t_qkv = net.tensor(tokens, 3 * dim)
        net.conv(t_ln, t_qkv, tokens, 1, dim, sd[pre + ".attn.qkv.weight"], bias=sd.get(pre + ".attn.qkv.bias"))
        t_att = net.tensor(tokens, dim)
        net.op(OP_ATTENTION, [t_qkv, t_att, tokens, heads, dh], [dh ** -0.5])
        net.flops_per_image += 4.0 * heads * tokens * tokens * dh
        x2 = net.tensor(tokens, dim)
        net.conv(t_att, x2, tokens, 1, dim, sd[pre + ".attn.proj.weight"], bias=sd[pre + ".attn.proj.bias"], residual=x)
        t_ln2 = net.tensor(tokens, dim)
        net.op(OP_LAYERNORM, [x2, t_ln2, tokens, dim, net.param_f32(sd[pre + ".norm2.weight"]),
                              net.param_f32(sd[pre + ".norm2.bias"]), 1, 0], [1e-6])
        hid = sd[pre + ".mlp.fc1.weight"].shape[0]
        t_h = net.tensor(tokens, hid)
        net.conv(t_ln2, t_h, tokens, 1, dim, sd[pre + ".mlp.fc1.weight"], bias=sd[pre + ".mlp.fc1.bias"], act=2)
        x3 = net.tensor(tokens, dim)
        net.conv(t_h, x3, tokens, 1, hid, sd[pre + ".mlp.fc2.weight"], bias=sd[pre + ".mlp.fc2.bias"], residual=x2)
        x = x3
    gamma, beta = net.param_f32(sd["norm.weight"]), net.param_f32(sd["norm.bias"])
    if global_pool == "token":
        net.set_output(dim)
        # final LayerNorm on the CLS rows only (dino_vits.py:252-254: norm, then x[:, 0])
        net.op(OP_LAYERNORM, [x, -1, 1, dim, gamma, beta, tokens, 1], [1e-6])
    else:
        net.set_output(tokens * dim)
        net.op(OP_LAYERNORM, [x, -1, tokens, dim, gamma, beta, 1, 1], [1e-6])     # every token row, [B, tokens * dim]
    net.tokens = tokens
    return net


# ------------------------------------------------------------------------------------------------------------------
# CLIP ViT-B/16 towers for the CLIP score (utils_ret.py:1046-1066: clip.load("ViT-B/16"), encode_image / encode_text)
def _clip_blocks(net: DcrNet, sd, prefix: str, x: int, tokens: int, dim: int, causal: bool) -> int:
    """clip/model.py ResidualAttentionBlock x N: x += attn(ln_1(x)); x += c_proj(QuickGELU(c_fc(ln_2(x)))); LayerNorm eps
    1e-5, packed in_proj [q | k | v] (the same column order as the DINO qkv Linear), 64-dim heads."""
    heads = dim // 64
    i = 0
    while f"{prefix}resblocks.{i}.ln_1.weight" in sd:
        p = f"{prefix}resblocks.{i}."
        t_ln = net.tensor(tokens, dim)
        net.op(OP_LAYERNORM, [x, t_ln, tokens, dim, net.param_f32(sd[p + "ln_1.weight"]), net.param_f32(sd[p + "ln_1.bias"]), 1, 0], [1e-5])
        t_qkv = net.tensor(tokens, 3 * dim)
        net.conv(t_ln, t_qkv, tokens, 1, dim, sd[p + "attn.in_proj_weight"], bias=sd[p + "attn.in_proj_bias"])
        t_att = net.tensor(tokens, dim)
        net.op(OP_ATTENTION, [t_qkv, t_att, tokens, heads, 64, 1 if causal else 0], [64 ** -0.5])
        net.flops_per_image += 4.0 * heads * tokens * tokens * 64
        x2 = net.tensor(tokens, dim)
        net.conv(t_att, x2, tokens, 1, dim, sd[p + "attn.out_proj.weight"], bias=sd[p + "attn.out_proj.bias"], residual=x)
        t_ln2 = net.tensor(tokens, dim)
        net.op(OP_LAYERNORM, [x2, t_ln2, tokens, dim, net.param_f32(sd[p + "ln_2.weight"]), net.param_f32(sd[p + "ln_2.bias"]), 1, 0], [1e-5])
        hid = sd[p + "mlp.c_fc.weight"].shape[0]
        t_h = net.tensor(tokens, hid)
        net.conv(t_ln2, t_h, tokens, 1, dim, sd[p + "mlp.c_fc.weight"], bias=sd[p + "mlp.c_fc.bias"], act=3)
        x3 = net.tensor(tokens, dim)
        net.conv(t_h, x3, tokens, 1, hid, sd[p + "mlp.c_proj.weight"], bias=sd[p + "mlp.c_proj.bias"], residual=x2)
        x = x3
        i += 1
    return x


def build_clip_visual(state_dict: Dict[str, torch.Tensor], max_batch: int = 64, precision: str = "fast",
                      mean: Sequence[float] = (0.5, 0.5, 0.5), std: Sequence[float] = (0.5, 0.5, 0.5),
                      in_size: int = 256, crop: int = 224) -> DcrNet:
    """`model.encode_image` of clip.load("ViT-B/16") (utils_ret.py:1048, :1056): conv1 patch embedding (no bias),
    class + positional embeddings, ln_pre, the transformer, ln_post on the class token, @ proj -> [n, 512].
    gen_clipscore feeds the loader's tensors as they are, i.e. the 0.5/0.5-normalised 224 crop (diff_retrieval.py:325-330)
    -- hence the default mean/std; pass CLIP's own statistics when the caller preprocesses with clip's transform."""
    sd = {k: v.detach().cpu().float() for k, v in state_dict.items()}
    w = sd["visual.conv1.weight"]
    dim, patch = w.shape[0], w.shape[-1]
    grid = crop // patch
    n_patch, tokens = grid * grid, grid * grid + 1
    if sd["visual.positional_embedding"].shape[0] != tokens:
        raise _lib.DcrError("CLIP visual tower: positional embedding does not match the input size")
    net = DcrNet(max_batch, precision)
    net.in_shape, net.net_input = (in_size, in_size), (crop, crop)
    k_pad = first_conv_k_pad(patch, patch)
    t_cols = net.tensor(n_patch, k_pad)
    _input_op(net, OP_IM2COL_U8, t_cols, in_size, crop, mean, std, [patch, patch, patch, 0, k_pad])
    t_patch = net.tensor(n_patch, dim)
    net.conv(t_cols, t_patch, n_patch, 1, k_pad, _first_conv_weight(w, k_pad))
    x0 = net.tensor(tokens, dim)
    net.op(OP_VIT_TOKENS, [t_patch, x0, n_patch, dim, net.param_f32(sd["visual.class_embedding"].reshape(-1)),
                           net.param_f32(sd["visual.positional_embedding"].reshape(tokens, dim))])
    x = net.tensor(tokens, dim)
    net.op(OP_LAYERNORM, [x0, x, tokens, dim, net.param_f32(sd["visual.ln_pre.weight"]), net.param_f32(sd["visual.ln_pre.bias"]), 1, 0], [1e-5])
    x = _clip_blocks(net, sd, "visual.transformer.", x, tokens, dim, causal=False)
    t_cls = net.tensor(1, dim)
    net.op(OP_LAYERNORM, [x, t_cls, 1, dim, net.param_f32(sd["visual.ln_post.weight"]), net.param_f32(sd["visual.ln_post.bias"]), tokens, 0], [1e-5])
    proj = sd["visual.proj"]                                   # [dim, embed]: x @ proj == Linear with weight proj.T
    net.set_output(proj.shape[1])
    net.conv(t_cls, -1, 1, 1, dim, proj.T.contiguous(), to_output=True)
    net.tokens = tokens
    return net


def build_clip_text(state_dict: Dict[str, torch.Tensor], max_batch: int = 64, precision: str = "fast") -> DcrNet:
    """`model.encode_text` (utils_ret.py:1057) up to the per-token projection: token + positional embeddings, the causal
    transformer, ln_final on every token, @ text_projection -> float32 [n, 77 * 512]; the caller picks the row of the
    end-of-text token (`x[arange, text.argmax(-1)]`, clip/model.py).  Input: int32 token ids [n, 77] (DcrNet.forward_tokens)."""
    sd = {k: v.detach().cpu().float() for k, v in state_dict.items()}
    table = sd["token_embedding.weight"]
    vocab, dim = table.shape
    ctx = sd["positional_embedding"].shape[0]
    net = DcrNet(max_batch, precision)
    x = net.tensor(ctx, dim)
    net.op(OP_EMBED, [x, ctx, dim, net.param_f32(table), net.param_f32(sd["positional_embedding"]), vocab])
    x = _clip_blocks(net, sd, "transformer.", x, ctx, dim, causal=True)
    t_ln = net.tensor(ctx, dim)
    net.op(OP_LAYERNORM, [x, t_ln, ctx, dim, net.param_f32(sd["ln_final.weight"]), net.param_f32(sd["ln_final.bias"]), 1, 0], [1e-5])
    proj = sd["text_projection"]
    net.set_output(ctx * proj.shape[1])
    net.conv(t_ln, -1, ctx, 1, dim, proj.T.contiguous(), to_output=True)
    net.tokens, net.context_length, net.embed_dim = ctx, ctx, proj.shape[1]
    return net


# ------------------------------------------------------------------------------------------------------------------
# VGG-16 fc2 features for Improved Precision & Recall (metrics/ipr.py:37-41, 124-147)
_VGG16_CFG = (64, 64, "M", 128, 128, "M", 256, 256, 256, "M", 512, 512, 512, "M", 512, 512, 512, "M")


def build_vgg16_fc2(state_dict: Dict[str, torch.Tensor], max_batch: int = 50, precision: str = "fast",
                    mean: Sequence[float] = (0.485, 0.456, 0.406), std: Sequence[float] = (0.229, 0.224, 0.225)) -> DcrNet:
    """torchvision VGG-16 up to classifier[3] (the 4096-d `fc2` features of metrics/ipr.py:139-141:
    `vgg16.features(x)` -> view(-1, 7*7*512) -> `classifier[:4]` = Linear, ReLU, Dropout(eval: identity), Linear).
    Input: uint8 [n,224,224,3] (the caller resizes with PIL as get_custom_loader does, ipr.py:300-306; ToTensor +
    ImageNet Normalize are fused into the first kernel) or the already transformed float32 [n,3,224,224]."""
    sd = _strip({k: v.detach().cpu() for k, v in state_dict.items()}, ["module."])
    net = DcrNet(max_batch, precision)
    net.in_shape = (224, 224)
    net.net_input = (224, 224)
    h = 224
    k_pad = first_conv_k_pad(3, 3)
    t_cols = net.tensor(h * h, k_pad)
    _input_op(net, OP_IM2COL_U8, t_cols, 224, 224, mean, std, [3, 3, 1, 1, k_pad])
    w0 = sd["features.0.weight"]
    t = net.tensor(h * h, 64)
    net.conv(t_cols, t, h * h, 1, k_pad, _first_conv_weight(w0, k_pad), bias=sd["features.0.bias"], act=1)
    net.flops_per_image += 2.0 * h * h * 64 * (27 - k_pad)
    c, li = 64, 2                       # features.0 = conv, .1 = ReLU
    for v in _VGG16_CFG[1:]:
        if v == "M":
            ho = h // 2
            o = net.tensor(ho * ho, c)
            net.op(OP_MAXPOOL, [t, o, h, h, c, 2, 2, 0, 0])
            t, h = o, ho
            li += 1
        else:
            o = net.tensor(h * h, v)
            net.conv(t, o, h, h, c, sd[f"features.{li}.weight"], pad=(1, 1), bias=sd[f"features.{li}.bias"], act=1)
            t, c = o, v
            li += 2
    # before_fc.view(-1, 7*7*512) flattens NCHW as (c, h, w); the activation here is NHWC -> permute fc1's columns
    flat = net.alias(t, 1, h * h * c)
    w1 = sd["classifier.0.weight"].detach().float()
    w1 = w1.reshape(w1.shape[0], c, h * h).permute(0, 2, 1).reshape(w1.shape[0], h * h * c).contiguous()
    t_fc1 = net.tensor(1, w1.shape[0])
    net.conv(flat, t_fc1, 1, 1, h * h * c, w1, bias=sd["classifier.0.bias"], act=1)
    w2 = sd["classifier.3.weight"]
    net.set_output(w2.shape[0])
    net.conv(t_fc1, -1, 1, 1, w1.shape[0], w2, bias=sd["classifier.3.bias"], to_output=True)
    return net


# ------------------------------------------------------------------------------------------------------------------
# FID Inception-v3 (metrics/inception.py:16-341): pool3 features [N, 2048]
def build_fid_inception(state_dict: Dict[str, torch.Tensor], max_batch: int = 50, precision: str = "fast",
                        stop_after: Optional[str] = None) -> DcrNet:
    """Input: uint8 [n,299,299,3] -- the caller resizes with PIL exactly as metrics/fid.py:104-106 does
    (Resize(299) bilinear on uint8, CenterCrop(299)).  ToTensor, Normalize(0.5,0.5) (fid.py:108-109) and the SECOND
    `2*x-1` of InceptionV3.forward (inception.py:152-153) are fused into the first op."""
    sd = _strip({k: v.detach().cpu() for k, v in state_dict.items()}, ["module."])
    net = DcrNet(max_batch, precision)
    net.in_shape = (299, 299)
    net.net_input = (299, 299)
    eps = 1e-3

    def bconv(in_t, h, w, c, name, *, stride=1, pad=(0, 0), out_t=None, out_c=None, col_off=0):
        wt = sd[name + ".conv.weight"]
        n, _, kh, kw = wt.shape
        ho = (h + 2 * pad[0] - kh) // stride + 1
        wo = (w + 2 * pad[1] - kw) // stride + 1
        if out_t is None:
            out_t = net.tensor(ho * wo, n)
        sc, bi = _fold_bn(sd, name + ".bn", eps)
        net.conv(in_t, out_t, h, w, c, wt, stride=stride, pad=pad, scale=sc, bias=bi, act=1, out_col_off=col_off)
        return out_t, ho, wo, n

    def finish(t, hw, c):
        net.set_output(c)
        net.op(OP_GAP, [t, -1, hw, c, 1])
        return net

    # block 0
    k_pad = first_conv_k_pad(3, 3)
    s = (299 - 3) // 2 + 1   # 149
    t_cols = net.tensor(s * s, k_pad)
    _input_op(net, OP_IM2COL_U8, t_cols, 299, 299, [0.5] * 3, [0.5] * 3, [3, 3, 2, 0, k_pad], post=(2.0, -1.0))
    w1 = sd["Conv2d_1a_3x3.conv.weight"]
    sc, bi = _fold_bn(sd, "Conv2d_1a_3x3.bn", eps)
    t = net.tensor(s * s, 32)
    net.conv(t_cols, t, s * s, 1, k_pad, _first_conv_weight(w1, k_pad), scale=sc, bias=bi, act=1)
    net.flops_per_image += 2.0 * s * s * 32 * (27 - k_pad)
    h = w = s
    if stop_after == "Conv2d_1a_3x3":
        return finish(t, h * w, 32)
    t, h, w, c = bconv(t, h, w, 32, "Conv2d_2a_3x3")
    if stop_after == "Conv2d_2a_3x3":
        return finish(t, h * w, c)
    t, h, w, c = bconv(t, h, w, c, "Conv2d_2b_3x3", pad=(1, 1))
    if stop_after == "Conv2d_2b_3x3":
        return finish(t, h * w, c)

    def maxpool(in_t, h, w, c, k, stride, pad, out_t=None, out_c=None, col_off=0):
        ho = (h + 2 * pad - k) // stride + 1
        if out_t is None:
            out_t = net.tensor(ho * ho, c)
        net.op(OP_MAXPOOL, [in_t, out_t, h, w, c, k, stride, pad, col_off])
        return out_t, ho, ho

    t, h, w = maxpool(t, h, w, c, 3, 2, 0)
    if stop_after == "pool1":
        return finish(t, h * w, c)
    # block 1
    t, h, w, c = bconv(t, h, w, c, "Conv2d_3b_1x1")
    if stop_after == "Conv2d_3b_1x1":
        return finish(t, h * w, c)
    t, h, w, c = bconv(t, h, w, c, "Conv2d_4a_3x3")
    if stop_after == "Conv2d_4a_3x3":
        return finish(t, h * w, c)
    t, h, w = maxpool(t, h, w, c, 3, 2, 0)
    if stop_after == "pool2":
        return finish(t, h * w, c)

    def avgpool3(in_t, h, w, c):
        o = net.tensor(h * w, c)
        net.op(OP_AVGPOOL, [in_t, o, h, w, c, 3, 1, 1, 0])
        return o

    def inception_a(x, h, w, c, p):
        pool_c = sd[p + ".branch_pool.conv.weight"].shape[0]
        out_c = 64 + 64 + 96 + pool_c
        o = net.tensor(h * w, out_c)
        bconv(x, h, w, c, p + ".branch1x1", out_t=o, col_off=0)
        b, _, _, bc = bconv(x, h, w, c, p + ".branch5x5_1")
        bconv(b, h, w, bc, p + ".branch5x5_2", pad=(2, 2), out_t=o, col_off=64)
        b, _, _, bc = bconv(x, h, w, c, p + ".branch3x3dbl_1")
        b, _, _, bc = bconv(b, h, w, bc, p + ".branch3x3dbl_2", pad=(1, 1))
        bconv(b, h, w, bc, p + ".branch3x3dbl_3", pad=(1, 1), out_t=o, col_off=128)
        bconv(avgpool3(x, h, w, c), h, w, c, p + ".branch_pool", out_t=o, col_off=224)
        return o, out_c

    def inception_b(x, h, w, c, p):
        ho = (h - 3) // 2 + 1
        out_c = 384 + 96 + c
        o = net.tensor(ho * ho, out_c)
        bconv(x, h, w, c, p + ".branch3x3", stride=2, out_t=o, col_off=0)
        b, _, _, bc = bconv(x, h, w, c, p + ".branch3x3dbl_1")
        b, _, _, bc = bconv(b, h, w, bc, p + ".branch3x3dbl_2", pad=(1, 1))
        bconv(b, h, w, bc, p + ".branch3x3dbl_3", stride=2, out_t=o, col_off=384)
        net.op(OP_MAXPOOL, [x, o, h, w, c, 3, 2, 0, 480])
        return o, out_c, ho

    def inception_c(x, h, w, c, p):
        o = net.tensor(h * w, 768)
        bconv(x, h, w, c, p + ".branch1x1", out_t=o, col_off=0)
        b, _, _, bc = bconv(x, h, w, c, p + ".branch7x7_1")
        b, _, _, bc = bconv(b, h, w, bc, p + ".branch7x7_2", pad=(0, 3))
        bconv(b, h, w, bc, p + ".branch7x7_3", pad=(3, 0), out_t=o, col_off=192)
        b, _, _, bc = bconv(x, h, w, c, p + ".branch7x7dbl_1")
        b, _, _, bc = bconv(b, h, w, bc, p + ".branch7x7dbl_2", pad=(3, 0))
        b, _, _, bc = bconv(b, h, w, bc, p + ".branch7x7dbl_3", pad=(0, 3))
        b, _, _, bc = bconv(b, h, w, bc, p + ".branch7x7dbl_4", pad=(3, 0))
        bconv(b, h, w, bc, p + ".branch7x7dbl_5", pad=(0, 3), out_t=o, col_off=384)
        bconv(avgpool3(x, h, w, c), h, w, c, p + ".branch_pool", out_t=o, col_off=576)
        return o, 768

    def inception_d(x, h, w, c, p):
        ho = (h - 3) // 2 + 1
        out_c = 320 + 192 + c
        o = net.tensor(ho * ho, out_c)
        b, _, _, bc = bconv(x, h, w, c, p + ".branch3x3_1")
        bconv(b, h, w, bc, p + ".branch3x3_2", stride=2, out_t=o, col_off=0)
        b, _, _, bc = bconv(x, h, w, c, p + ".branch7x7x3_1")
        b, _, _, bc = bconv(b, h, w, bc, p + ".branch7x7x3_2", pad=(0, 3))
        b, _, _, bc = bconv(b, h, w, bc, p + ".branch7x7x3_3", pad=(3, 0))
        bconv(b, h, w, bc, p + ".branch7x7x3_4", stride=2, out_t=o, col_off=320)
        net.op(OP_MAXPOOL, [x, o, h, w, c, 3, 2, 0, 512])
        return o, out_c, ho

    def inception_e(x, h, w, c, p, max_pool):
        o = net.tensor(h * w, 2048)
        bconv(x, h, w, c, p + ".branch1x1", out_t=o, col_off=0)
        b, _, _, bc = bconv(x, h, w, c, p + ".branch3x3_1")
        bconv(b, h, w, bc, p + ".branch3x3_2a", pad=(0, 1), out_t=o, col_off=320)
        bconv(b, h, w, bc, p + ".branch3x3_2b", pad=(1, 0), out_t=o, col_off=704)
        b, _, _, bc = bconv(x, h, w, c, p + ".branch3x3dbl_1")
        b, _, _, bc = bconv(b, h, w, bc, p + ".branch3x3dbl_2", pad=(1, 1))
        bconv(b, h, w, bc, p + ".branch3x3dbl_3a", pad=(0, 1), out_t=o, col_off=1088)
        bconv(b, h, w, bc, p + ".branch3x3dbl_3b", pad=(1, 0), out_t=o, col_off=1472)
        pooled = net.tensor(h * w, c)
        net.op(OP_MAXPOOL if max_pool else OP_AVGPOOL, [x, pooled, h, w, c, 3, 1, 1, 0])   # E_2 uses MAX (:337)
        bconv(pooled, h, w, c, p + ".branch_pool", out_t=o, col_off=1856)
        return o, 2048

    for name in ("Mixed_5b", "Mixed_5c", "Mixed_5d"):
        t, c = inception_a(t, h, w, c, name)
        if stop_after == name:
            return finish(t, h * w, c)
    t, c, h = inception_b(t, h, w, c, "Mixed_6a")
    w = h
    if stop_after == "Mixed_6a":
        return finish(t, h * w, c)
    for name in ("Mixed_6b", "Mixed_6c", "Mixed_6d", "Mixed_6e"):
        t, c = inception_c(t, h, w, c, name)
        if stop_after == name:
            return finish(t, h * w, c)
    t, c, h = inception_d(t, h, w, c, "Mixed_7a")
    w = h
    if stop_after == "Mixed_7a":
        return finish(t, h * w, c)
    t, c = inception_e(t, h, w, c, "Mixed_7b", False)
    if stop_after == "Mixed_7b":
        return finish(t, h * w, c)
    t, c = inception_e(t, h, w, c, "Mixed_7c", True)
    net.set_output(2048)
    net.op(OP_GAP, [t, -1, h * w, c, 1])
    return net
