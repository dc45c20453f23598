"""GPU numerics: the wgmma implicit-GEMM convolution vs torch.nn.functional.conv2d (fp32, TF32 off)."""
import numpy as np
import pytest
import torch

from dcr_b200 import ops

pytestmark = pytest.mark.gpu

# (B, H, W, C, N, kh, kw, stride, pad_h, pad_w)
SHAPES = [
    (2, 56, 56, 64, 64, 1, 1, 1, 0, 0),      # resnet layer1 conv1 (plain GEMM path)
    (2, 56, 56, 64, 64, 3, 3, 1, 1, 1),      # resnet 3x3
    (3, 56, 56, 128, 128, 3, 3, 2, 1, 1),    # resnet strided 3x3
    (2, 56, 56, 256, 512, 1, 1, 2, 0, 0),    # strided 1x1 downsample
    (5, 14, 14, 256, 256, 3, 3, 1, 1, 1),    # tile spans several images
    (4, 7, 7, 512, 2048, 1, 1, 1, 0, 0),
    (2, 17, 17, 128, 192, 1, 7, 1, 0, 3),    # inception 1x7
    (2, 17, 17, 128, 192, 7, 1, 1, 3, 0),    # inception 7x1
    (2, 35, 35, 48, 64, 5, 5, 1, 2, 2),      # inception 5x5, C not a multiple of 64
    (2, 35, 35, 288, 384, 3, 3, 2, 0, 0),    # inception 3x3/2 no padding
    (300, 1, 1, 384, 1152, 1, 1, 1, 0, 0),   # ViT qkv Linear
    (1, 9, 9, 8, 8, 3, 3, 1, 1, 1),          # tiny
    (2, 56, 56, 64, 256, 1, 1, 1, 0, 0),     # resnet layer1 expansion: A-resident schedule (K = 64, 2 column blocks)
    (3, 28, 28, 128, 512, 1, 1, 1, 0, 0),    # layer2 expansion (K = 128, 4 column blocks)
    (5, 14, 14, 256, 1024, 1, 1, 1, 0, 0),   # layer3 expansion (K = 256, 8 column blocks, single output staging tile)
    (1, 10, 13, 192, 320, 1, 1, 1, 0, 0),    # ragged M and N with the A-resident schedule
]


def _ref(x, w, scale, bias, res, act, stride, pad):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    y = torch.nn.functional.conv2d(x.permute(0, 3, 1, 2).double(), w.double(), stride=stride, padding=pad)
    y = y.permute(0, 2, 3, 1)
    y = y * scale.double() + bias.double()
    if res is not None:
        y = y + res.double()
    if act == 1:
        y = torch.relu(y)
    elif act == 2:
        y = torch.nn.functional.gelu(y)
    elif act == 3:
        y = y * torch.sigmoid(1.702 * y)      # QuickGELU (CLIP)
    return y.float()


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("planes", [1, 2, 3])
def test_conv_matches_torch(shape, planes):
    b, h, w_, c, n, kh, kw, stride, ph, pw = shape
    gen = torch.Generator(device="cuda").manual_seed(b * 1000 + c + n + kh)
    x = torch.randn(b, h, w_, c, device="cuda", generator=gen)
    w = torch.randn(n, c, kh, kw, device="cuda", generator=gen) / (c * kh * kw) ** 0.5
    scale = 0.5 + torch.rand(n, device="cuda", generator=gen)
    bias = torch.randn(n, device="cuda", generator=gen) * 0.1
    ho = (h + 2 * ph - kh) // stride + 1
    wo = (w_ + 2 * pw - kw) // stride + 1
    res = torch.randn(b, ho, wo, n, device="cuda", generator=gen)
    # QuickGELU on the Inception-shaped filters: with one plane the TMA-store epilogue's own instantiation (kEpi = 4)
    act = 3 if (kh, kw) in ((1, 7), (7, 1), (5, 5)) else (1 if kh == 3 else (2 if h == 1 else 0))

    xp = ops.split_planes(x, planes)
    wp = ops.prepare_conv_weight(w, planes)
    rp = ops.split_planes(res, planes)
    out, out32 = ops.conv2d(xp, wp, n, kh, kw, stride, ph, pw, scale=scale, bias=bias, residual=rp, act=act,
                            want_f32=True)
    torch.cuda.synchronize()
    # reference on exactly the operands the kernel saw
    xm, wm = ops.merge_planes(xp), ops.merge_planes(wp).reshape(n, kh, kw, -1)[..., :c].permute(0, 3, 1, 2)
    ref = _ref(xm, wm, scale, bias, ops.merge_planes(rp), act, stride, (ph, pw))
    # one plane: bf16 x bf16 products are exact in fp32, only the accumulation order differs from the reference;
    # three planes (6 cross terms): fp32-level agreement, limited by the tensor core's fp32 accumulator rounding
    mx = max(1.0, ref.abs().max().item())
    tol = (3e-4 if planes == 1 else 5e-5) * mx   # the tensor core's fp32 accumulator truncates: ~1e-5 relative at K~2000
    if planes == 1 and act == 2:
        # single-plane (bf16) mode evaluates GELU in its tanh form with tanh.approx.f32: <= 4.7e-4 from the erf form plus
        # 2^-11 relative on 0.5 y (conv_gemm.cu gelu_tanh_fast); the split-bf16 modes keep the erf form
        tol += 1.2e-3 * mx
    if planes == 2:
        # bf16x3, hi.hi + hi.lo + lo.hi of the merged two-plane operands: the dropped lo.lo term is <= 2^-16 sum |x||w|
        # (a plane's rounding residual reaches half a bf16 ulp, 2^-8 of the value at the bottom of a binade); the fp32
        # accumulation of the 3K exact products adds <= 3K 2^-23 of the sum of their magnitudes (2 % above sum |x||w|);
        # fmaf and the two residual-plane adds round three times (4 u of the pre-activation magnitude).  The activation
        # is at most LIP = 1.13-Lipschitz and adds its own fp32 evaluation: GELU's erf polynomial 2e-7 absolute (1e-7 |y|),
        # QuickGELU 2 u 1.702 |y| + 2^-22 (argument and expf) + 2 u (sum and division) relative; the 2-plane store
        # keeps y - hi - lo <= 2^-16 |y|.
        K = kh * kw * c
        mag = _ref(xm.abs(), wm.abs(), scale.abs(), torch.zeros_like(bias), None, 0, stride, (ph, pw)).max().item()
        pre = mag + bias.abs().max().item() + ops.merge_planes(rp).abs().max().item()
        tol = 1.13 * ((2 ** -16 * 1.01 + 3 * K * 2 ** -23 * 1.02) * mag + 4 * 2 ** -24 * pre)
        tol += (2 ** -21 + 2 * 2 ** -24 * 1.702 * mx + 2 ** -22 + 2 * 2 ** -24) * mx
    err32 = (out32 - ref).abs().max().item()
    assert err32 < tol, f"fp32 out err {err32}"
    got = ops.merge_planes(out)
    errp = (got - ref).abs().max().item()
    ptol = {1: 2 ** -8, 2: 2 ** -16, 3: 2 ** -22}[planes] * mx + tol
    assert errp < ptol, f"plane out err {errp}"
    if planes == 1:
        # without the fp32 side output the kernel takes the shared-memory staged TMA-store epilogue (residual tile
        # fetched by TMA too); it must produce the same bf16 tensor bit for bit
        out2, _ = ops.conv2d(xp, wp, n, kh, kw, stride, ph, pw, scale=scale, bias=bias, residual=rp, act=act)
        torch.cuda.synchronize()
        assert torch.equal(out2, out), f"TMA-store epilogue differs: {(out2.float() - out.float()).abs().max().item()}"
        out3, _ = ops.conv2d(xp, wp, n, kh, kw, stride, ph, pw, scale=scale, bias=bias, act=act)
        ref3 = _ref(ops.merge_planes(xp), ops.merge_planes(wp).reshape(n, kh, kw, -1)[..., :c].permute(0, 3, 1, 2),
                    scale, bias, None, act, stride, (ph, pw))
        assert (ops.merge_planes(out3) - ref3).abs().max().item() < ptol


HALO_SHAPES = [   # (B, H, W, C, N): 3x3 / stride 1 / pad 1 without residual -> halo-reuse kernel (csrc/conv3x3_halo.cu)
    (2, 56, 56, 64, 64),       # resnet layer1: 2 output rows per tile
    (3, 28, 28, 128, 128),     # layer2: 4 rows per tile, two channel blocks
    (5, 14, 14, 128, 128),     # 8 rows per tile, last tile of every image half outside (14 = 8 + 6)
    (2, 14, 14, 64, 128),      # one channel block, two 64-column output slabs
    (1, 30, 62, 64, 64),       # widest supported row (62 + 2 = 64)
    (2, 9, 20, 128, 64),       # H not a multiple of the rows per tile (5)
    (1, 2, 8, 64, 64),         # smallest
]


def _halo_eligible(b, h, w_, c, n):
    """Mirror of conv3x3_halo_eligible (csrc/conv3x3_halo.cu) for what test_conv3x3_halo_path varies: a shape the
    kernel does not serve runs the generic kernel in both arms of the test, which then compares it with itself."""
    return c % 64 == 0 and n % 64 == 0 and n <= 128 and 8 <= w_ and w_ + 2 <= 64 and h >= 2 and b >= 1


assert all(_halo_eligible(*s) for s in HALO_SHAPES), \
    f"HALO_SHAPES the halo kernel does not serve: {[s for s in HALO_SHAPES if not _halo_eligible(*s)]}"


@pytest.mark.parametrize("shape", HALO_SHAPES)
@pytest.mark.parametrize("act", [0, 1])
def test_conv3x3_halo_path(shape, act, monkeypatch):
    b, h, w_, c, n = shape
    gen = torch.Generator(device="cuda").manual_seed(b * 100 + h + c + n)
    x = torch.randn(b, h, w_, c, device="cuda", generator=gen)
    w = torch.randn(n, c, 3, 3, device="cuda", generator=gen) / (c * 9) ** 0.5
    scale = 0.5 + torch.rand(n, device="cuda", generator=gen)
    bias = torch.randn(n, device="cuda", generator=gen) * 0.1
    xp, wp = ops.split_planes(x, 1), ops.prepare_conv_weight(w, 1)
    l0 = None
    out, _ = ops.conv2d(xp, wp, n, 3, 3, 1, 1, 1, scale=scale, bias=bias, act=act)
    torch.cuda.synchronize()
    monkeypatch.setenv("DCR_B200_TUNING", "1")
    monkeypatch.setenv("DCR_CONV_NO_HALO", "1")
    gen_out, _ = ops.conv2d(xp, wp, n, 3, 3, 1, 1, 1, scale=scale, bias=bias, act=act)
    torch.cuda.synchronize()
    monkeypatch.delenv("DCR_CONV_NO_HALO")
    ref = _ref(ops.merge_planes(xp), ops.merge_planes(wp).reshape(n, 3, 3, -1)[..., :c].permute(0, 3, 1, 2), scale, bias,
               None, act, 1, (1, 1))
    got, gen_got = ops.merge_planes(out), ops.merge_planes(gen_out)
    mx = max(1.0, ref.abs().max().item())
    err = (got - ref).abs().max().item()
    assert err < 2 ** -8 * mx + 3e-4 * mx, f"halo path err {err}"
    # same products, different accumulation order than the generic kernel: at most one bf16 ulp apart
    assert (got - gen_got).abs().max().item() <= 2 ** -7 * mx
    assert (got != gen_got).float().mean().item() < 0.02


@pytest.mark.parametrize("shape", [
    ((600, 1, 1), 1536, 384, 1, 1, 0, True, 0),     # plain GEMM, three column blocks, residual
    ((3, 28, 28), 128, 512, 3, 2, 1, False, 1),    # strided 3x3 through TMA im2col, four column blocks
    ((4, 14, 14), 1024, 512, 1, 1, 0, False, 1),   # two 256-wide column blocks
])
@pytest.mark.parametrize("direct", ["0", "1"])
def test_tile_order_does_not_change_results(shape, direct, monkeypatch):
    """n-fastest tile order (chosen when A is larger than L2: consecutive tiles share an m-tile's rows) against the default
    m-fastest order, with the TMA-store epilogue and with the direct epilogue: every tile computes the same thing, only who
    computes it and when changes."""
    (b, h, w_), c, n, k, stride, pad, with_res, act = shape
    gen = torch.Generator(device="cuda").manual_seed(c + n + k)
    x = torch.randn(b, h, w_, c, device="cuda", generator=gen)
    w = torch.randn(n, c, k, k, device="cuda", generator=gen) / (c * k * k) ** 0.5
    ho = (h + 2 * pad - k) // stride + 1
    wo = (w_ + 2 * pad - k) // stride + 1
    res = torch.randn(b, ho, wo, n, device="cuda", generator=gen) if with_res else None
    xp, wp = ops.split_planes(x, 1), ops.prepare_conv_weight(w, 1)
    rp = ops.split_planes(res, 1) if with_res else None
    monkeypatch.setenv("DCR_B200_TUNING", "1")
    if direct == "1":
        monkeypatch.setenv("DCR_GEMM_DIRECT_EPILOGUE", "1")
    outs = []
    for order in ("0", "1"):
        monkeypatch.setenv("DCR_GEMM_TILE_ORDER", order)
        o, _ = ops.conv2d(xp, wp, n, k, k, stride, pad, pad, residual=rp, act=act)
        torch.cuda.synchronize()
        outs.append(o)
    assert torch.equal(outs[0], outs[1])
    ref = _ref(ops.merge_planes(xp), ops.merge_planes(wp).reshape(n, k, k, -1)[..., :c].permute(0, 3, 1, 2),
               torch.ones(n, device="cuda"), torch.zeros(n, device="cuda"), ops.merge_planes(rp) if with_res else None, act,
               stride, (pad, pad))
    mx = max(1.0, ref.abs().max().item())
    assert (ops.merge_planes(outs[1]) - ref).abs().max().item() < (2 ** -8 + 3e-4) * mx
