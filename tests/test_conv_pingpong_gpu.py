"""GPU: the ping-pong schedule of the GEMM (BN <= 128) and 3x3 halo convolution kernels, where the CTA's tiles are dealt
alternately to the two consumer warpgroups.  Shapes are chosen by tile count per CTA (none / one / odd / even tiles for
warpgroup 1), ragged M and N, residual, concat column offsets and the A-resident schedule; every case is checked against
an fp64 torch reference at test_conv_matches_torch's single-plane tolerance, and bit for bit across tile orders and
between the TMA-store and direct epilogues (every output element keeps its k order and epilogue arithmetic)."""
import pytest
import torch

from dcr_b200 import _lib, ops

pytestmark = pytest.mark.gpu


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _ref(x, w, scale, bias, res, act, stride, pad):
    y = torch.nn.functional.conv2d(x.permute(0, 3, 1, 2).double(), w.double(), stride=stride, padding=pad)
    y = y.permute(0, 2, 3, 1) * scale.double() + bias.double()
    if res is not None:
        y = y + res.double()
    if act == 1:
        y = torch.relu(y)
    return y.float()


def _operands(b, h, w_, c, n, k, seed, with_res, stride=1, pad=0):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(b, h, w_, c, device="cuda", generator=gen)
    w = torch.randn(n, c, k, k, device="cuda", generator=gen) / (c * k * k) ** 0.5
    scale = 0.5 + torch.rand(n, device="cuda", generator=gen)
    bias = torch.randn(n, device="cuda", generator=gen) * 0.1
    ho, wo = (h + 2 * pad - k) // stride + 1, (w_ + 2 * pad - k) // stride + 1
    res = ops.split_planes(torch.randn(b, ho, wo, n, device="cuda", generator=gen), 1) if with_res else None
    return ops.split_planes(x, 1), ops.prepare_conv_weight(w, 1), scale, bias, res


def _check_ref(out, xp, wp, n, k, scale, bias, res, act, stride=1, pad=0):
    c = xp.shape[-1]
    ref = _ref(ops.merge_planes(xp), ops.merge_planes(wp).reshape(n, k, k, -1)[..., :c].permute(0, 3, 1, 2), scale, bias,
               ops.merge_planes(res) if res is not None else None, act, stride, (pad, pad))
    mx = max(1.0, ref.abs().max().item())
    err = (ops.merge_planes(out) - ref).abs().max().item()
    assert err < (2 ** -8 + 3e-4) * mx, f"err {err} (max |ref| {mx})"


def _gemm_cases():
    s = _sms() if torch.cuda.is_available() else 132
    # (name, B, H, W, C, N, with_res): 1x1 convolutions, M = B*H*W, tiles = ceil(M / 128) x ceil(N / BN)
    return [
        ("fewer_tiles_than_sms", 1, 3, 100, 64, 64, False),            # 3 tiles: warpgroup 1 of every CTA has none
        ("odd_per_cta_ragged_m", 1, 3 * s, 128 + 1, 64, 64, True),     # 3 tiles per CTA and more, M % 128 != 0
        ("even_per_cta", 2, s, 128, 128, 128, False),                  # 2 tiles per CTA
        ("n128_res", 1, 2 * s + 1, 64, 256, 128, True),
        ("n192_two_blocks", 1, 3 * s // 2, 128 + 7, 128, 192, True),   # second column block half outside N
        ("n192_no_res", 1, s + 3, 128, 192, 192, False),
        ("a_resident", 3, 56, 56, 64, 256, True),                      # K = 64, two column blocks, resident A rows
        ("a_resident_ragged", 1, 37, 61, 128, 512, False),            # four column blocks, M % 128 != 0
        # six and more tiles per CTA: ranges that start and end inside an m-tile (one warpgroup alone there), middle
        # m-tiles shared by both warpgroups, both a_full barriers through several phases, a_empty reused many times
        ("a_resident_long", 17, 56, 56, 64, 256, True),               # 417 m-tiles x 2 column blocks
        ("a_resident_long_4n", 1, 200, 130, 128, 512, False),         # 204 m-tiles x 4 column blocks
    ]


@pytest.mark.parametrize("case", _gemm_cases(), ids=lambda c: c[0])
def test_gemm_pingpong(case, monkeypatch):
    name, b, h, w_, c, n, with_res = case
    xp, wp, scale, bias, res = _operands(b, h, w_, c, n, 1, sum(map(ord, name)), with_res)
    monkeypatch.setenv("DCR_B200_TUNING", "1")
    outs = {}
    for direct in ("0", "1"):
        if direct == "1":
            monkeypatch.setenv("DCR_GEMM_DIRECT_EPILOGUE", "1")
        for order in ("0", "1"):
            monkeypatch.setenv("DCR_GEMM_TILE_ORDER", order)
            o, _ = ops.conv2d(xp, wp, n, 1, 1, scale=scale, bias=bias, residual=res, act=1)
            torch.cuda.synchronize()
            outs[(direct, order)] = o
    base = outs[("0", "0")]
    for key, o in outs.items():
        assert torch.equal(o, base), f"{key} differs from the TMA-store epilogue, m-fastest order"
    _check_ref(base, xp, wp, n, 1, scale, bias, res, 1)


def test_gemm_pingpong_im2col_odd_tiles():
    """strided 3x3 through TMA im2col at N = 128: a long k-loop (18 k-blocks) and an odd tile count per CTA"""
    b = max(1, (3 * _sms() * 128) // (28 * 28)) | 1
    xp, wp, scale, bias, res = _operands(b, 56, 56, 128, 128, 3, 11, True, stride=2, pad=1)
    o, _ = ops.conv2d(xp, wp, 128, 3, 3, 2, 1, 1, scale=scale, bias=bias, residual=res, act=1)
    torch.cuda.synchronize()
    _check_ref(o, xp, wp, 128, 3, scale, bias, res, 1, stride=2, pad=1)


def test_gemm_pingpong_split_planes():
    """the direct epilogue in the split-bf16 modes (two and three planes, fp32 side output) under the ping-pong schedule"""
    gen = torch.Generator(device="cuda").manual_seed(5)
    b, h, w_, c, n = 1, 2 * _sms() + 1, 128, 64, 128
    x = torch.randn(b, h, w_, c, device="cuda", generator=gen)
    w = torch.randn(n, c, 1, 1, device="cuda", generator=gen) / c ** 0.5
    scale = 0.5 + torch.rand(n, device="cuda", generator=gen)
    bias = torch.randn(n, device="cuda", generator=gen) * 0.1
    for planes in (2, 3):
        xp, wp = ops.split_planes(x, planes), ops.prepare_conv_weight(w, planes)
        _, out32 = ops.conv2d(xp, wp, n, 1, 1, scale=scale, bias=bias, act=1, want_f32=True)
        torch.cuda.synchronize()
        ref = _ref(ops.merge_planes(xp), ops.merge_planes(wp).reshape(n, 1, 1, -1)[..., :c].permute(0, 3, 1, 2), scale, bias,
                   None, 1, 1, (0, 0))
        mx = max(1.0, ref.abs().max().item())
        assert (out32 - ref).abs().max().item() < 5e-5 * mx, planes


@pytest.mark.parametrize("direct", ["0", "1"])
def test_gemm_pingpong_concat_offset(direct, monkeypatch):
    """output written into columns [off, off + N) of a wider tensor: the neighbours stay intact and the slice is the
    plain output bit for bit"""
    b, h, w_, c, n, off, width = 1, _sms() + 5, 128, 64, 128, 64, 320
    xp, wp, scale, bias, res = _operands(b, h, w_, c, n, 1, 21, True)
    monkeypatch.setenv("DCR_B200_TUNING", "1")
    if direct == "1":
        monkeypatch.setenv("DCR_GEMM_DIRECT_EPILOGUE", "1")
    plain, _ = ops.conv2d(xp, wp, n, 1, 1, scale=scale, bias=bias, residual=res, act=1)
    wide = torch.full((1, b, h, w_, width), 7.0, dtype=torch.bfloat16, device="cuda")
    lib = _lib.load()
    rc = lib.dcr_conv2d_bf16(xp.data_ptr(), 1, xp[0].numel(), b, h, w_, c, wp.data_ptr(), 1, wp[0].numel(), n, 1, 1, 1, 0, 0,
                             1, scale.data_ptr(), bias.data_ptr(), res.data_ptr(), 1, res[0].numel(), 1, wide.data_ptr(), 1,
                             wide[0].numel(), width, off, None, torch.cuda.current_stream().cuda_stream)
    _lib.check(rc, "dcr_conv2d_bf16")
    torch.cuda.synchronize()
    assert torch.equal(wide[..., off:off + n], plain)
    assert bool((wide[..., :off] == 7.0).all()) and bool((wide[..., off + n:] == 7.0).all())


def _halo_cases():
    s = _sms() if torch.cuda.is_available() else 132
    # (B, H, W, C, N): tiles = B * ceil(H / R), R = 128 // (W + 2) output rows per tile
    return [
        (14, 56, 56, 64, 64),                 # 392 tiles: 2 or 3 per CTA (resident weight taps)
        (3, 56, 56, 64, 128),                 # 84 tiles: fewer than SMs, warpgroup 1 idle
        (9, 28, 28, 128, 128),                # 63 tiles
        (57, 28, 28, 128, 128),               # 399 tiles: 3 or 4 per CTA
        ((3 * s) // 2 | 1, 14, 14, 256, 128),  # 2 tiles per image, odd image count, four channel blocks
        (67, 14, 14, 64, 64),
    ]


@pytest.mark.parametrize("shape", _halo_cases(), ids=lambda s: "x".join(map(str, s)))
def test_halo_pingpong(shape, monkeypatch):
    b, h, w_, c, n = shape
    xp, wp, scale, bias, _ = _operands(b, h, w_, c, n, 3, b * 7 + w_, False, pad=1)
    out, _ = ops.conv2d(xp, wp, n, 3, 3, 1, 1, 1, scale=scale, bias=bias, act=1)
    torch.cuda.synchronize()
    _check_ref(out, xp, wp, n, 3, scale, bias, None, 1, pad=1)
    # deterministic: a second launch gives the same bits
    again, _ = ops.conv2d(xp, wp, n, 3, 3, 1, 1, 1, scale=scale, bias=bias, act=1)
    torch.cuda.synchronize()
    assert torch.equal(out, again)
