"""GPU numerics of the network executor's own kernels, op by op: attention, the fused and space-to-depth ResNet stems, the
image input transform, LayerNorm, pooling, GeM / GAP, token assembly and embedding.

Each test builds a micro-network on nets.DcrNet around the one op under test, writes its input planes through
dcr_net_tensor, runs dcr_net_forward and compares the output planes with a float64 reference computed from the merged
input planes the kernel actually read.  Every bound is derived in a comment from the kernel's arithmetic; the measured
maximum error of each case is recorded as a test property (max_err, bound)."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from dcr_b200 import _lib, nets
from dcr_b200.dist import device_bytes
from dcr_b200.ops import split_planes
from oracle import models as om

pytestmark = pytest.mark.gpu

U = 2.0 ** -24                  # fp32 unit roundoff
FILL = 1.0e4                    # other images / unused batch slots: far from anything the op under test produces
SENTINEL = -7.75                # output planes the op must not touch


# ---- micro-network plumbing ---------------------------------------------------------------------------------------
class Micro:
    """A DcrNet with direct access to its activation tensors.  precision: a name of nets.PRECISION_PLANES, or a plane
    count (1: "fast", 3: "fp32")."""

    def __init__(self, max_batch: int, precision):
        if not isinstance(precision, str):
            precision = "fast" if precision == 1 else "fp32"
        self.net = nets.DcrNet(max_batch, precision)
        self.lib, self.mb, self.planes = self.net.lib, max_batch, self.net.planes
        self.shapes = {}

    def tensor(self, rows: int, ch: int) -> int:
        t = self.net.tensor(rows, ch)
        self.shapes[t] = (rows, ch)
        return t

    def view(self, t: int) -> torch.Tensor:
        """[planes, max_batch, rows, C] bf16 over the tensor's device buffer (valid while the net lives)."""
        ptr, ps = C.c_void_p(), C.c_int64()
        _lib.check(self.lib.dcr_net_tensor(self.net.handle, t, C.byref(ptr), C.byref(ps)), "dcr_net_tensor")
        rows, ch = self.shapes[t]
        assert ps.value == self.mb * rows * ch
        raw = device_bytes(ptr.value, self.planes * ps.value * 2, self.net.device)
        return raw.view(torch.bfloat16).view(self.planes, self.mb, rows, ch)

    def write(self, t: int, x: torch.Tensor) -> None:
        """x: fp32 [max_batch, rows, C] -> the tensor's planes (hi / mid / lo split with three planes)."""
        self.view(t).copy_(split_planes(x.cuda(), self.planes))

    def merged(self, t: int) -> torch.Tensor:
        return self.view(t).float().sum(0).cpu()

    def forward(self, B: int, inp=None, f32: bool = False) -> torch.Tensor:
        """Runs the op list on B images.  inp: the network input (uint8 NHWC images, fp32 NCHW crops or int32 ids);
        the other ops do not read it."""
        out = torch.zeros((self.mb, max(self.net.out_dim, 4)), dtype=torch.float32, device="cuda")
        src = (inp if inp is not None else out).contiguous()
        fn = self.lib.dcr_net_forward_f32 if f32 else self.lib.dcr_net_forward
        rc = fn(self.net.handle, src.data_ptr(), B, out.data_ptr(), torch.cuda.current_stream().cuda_stream)
        _lib.check(rc, "dcr_net_forward")
        torch.cuda.synchronize()
        return out[:B].cpu()


def _bf16_ulp(a: torch.Tensor) -> torch.Tensor:
    """Spacing of bf16 values at magnitude |a| (8 significant bits): 2^(e - 8) with |a| = m * 2^e, m in [0.5, 1)."""
    _, e = torch.frexp(a.abs().double().clamp_min(1e-30))
    return torch.ldexp(torch.ones_like(a, dtype=torch.float64), e - 8)


def _fp32_ulps(a: torch.Tensor, b: torch.Tensor) -> float:
    """max |a - b| in fp32 ulps of the larger magnitude."""
    sp = np.spacing(np.maximum(a.abs().numpy(), b.abs().numpy()).astype(np.float32)).astype(np.float64)
    return float(((a.double() - b.double()).abs().numpy() / sp).max())


def _check(record_property, err: torch.Tensor, bound: torch.Tensor, what: str) -> None:
    record_property("max_err", float(err.max()))
    record_property("max_err_over_bound", float((err / bound).max()))
    bad = err > bound
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} elements over the bound, worst err {float(err.max()):.3e} " \
                                f"(err / bound {float((err / bound).max()):.3f})"


# ---- attention (op 8) -----------------------------------------------------------------------------------------------
# (T, heads, B): T <= 128 (zeroed second key half), 128 < T <= 256 (K/V boxes reach into the next image or past the
# last row), T > 256 (streamed); every case runs with max_batch = B + 1
ATTN_CASES = [(1, 1, 3), (2, 6, 1), (77, 12, 3), (127, 6, 3), (128, 1, 3), (129, 12, 1), (197, 6, 3), (255, 12, 3),
              (256, 6, 1), (257, 6, 3), (785, 12, 1)]
SCALE = 64 ** -0.5


def _attn_image(gen, T: int, heads: int, causal: bool) -> torch.Tensor:
    """[T, 3 * heads * 64] fp32 q | k | v with the rows softmax gets wrong first: every 5th key a copy of key 0 (exact
    ties in every row), rows t = 1 mod 4 scaled so that their scaled scores span ~80 (the max subtraction matters),
    rows t = 2 mod 4 zero (all scores tie), rows t = 3 mod 4 aligned with key t // 2 (one dominant key)."""
    q, k, v = (torch.randn(T, heads, 64, generator=gen) for _ in range(3))
    k[::5] = k[0].clone()
    for t in range(T):
        if t % 4 == 1:
            keys = k[:t + 1] if causal else k
            s = torch.einsum("hd,jhd->hj", q[t], keys) * SCALE
            span = (s.max(1).values - s.min(1).values).clamp_min(1e-3)
            q[t] *= (80.0 / span)[:, None]
        elif t % 4 == 2:
            q[t] = 0
        elif t % 4 == 3:
            q[t] = 4 * k[t // 2]
    return torch.cat([q.reshape(T, -1), k.reshape(T, -1), v.reshape(T, -1)], 1)


def _attn_ref(x: torch.Tensor, heads: int, causal: bool, path: str, planes: int):
    """x: merged fp32 [B, T, 3*heads*64] -> (fp64 reference [B, T, heads*64], per-element bound) for `path`.

    The kernel's output is sum_j p~_j v_j / sum_j p~_j with p~_j = p_j (1 + e_j): any relative weight error |e_j| <= eps
    moves the normalised weights by at most 2 eps / (1 - eps) of themselves, so the output moves by at most
    2 eps / (1 - eps) * sum_j w_j |v_j - O| (the weights sum to one both ways).  eps per row:
      * scores: exact bf16 / fp32 products accumulated in fp32 over 64 terms: |ds_j| <= 64 * 2^-23 * scale * |q|.|k_j|,
        the maximum carries the same error: 2 max_j |ds_j|;
      * exponent argument (s - max) * log2(e) in fp32 and the exp itself: 8 u (max|s| + |max|) + 2^-20;
      * TC path only: P rounded to bf16 (8 significant bits) before P V: 2^-8.
    P V and the row sum accumulate T terms in fp32 (T 2^-23 of sum w |v| and of |O|; the streamed kernel rescales once per
    128-key tile: twice that), then 1 / sum and the product: 4 u |O|.  Store: bf16 (1 plane) rounds to 2^-8 |O|; three
    planes keep the fp32 value (2^-22 |O|)."""
    B, T, _ = x.shape
    xd = x.double().numpy().reshape(B, T, 3, heads, 64)
    q, k, v = xd[:, :, 0].transpose(0, 2, 1, 3), xd[:, :, 1].transpose(0, 2, 1, 3), xd[:, :, 2].transpose(0, 2, 1, 3)
    s = SCALE * q @ k.transpose(0, 1, 3, 2)                                   # [B, H, T, T]
    ds = 64 * 2.0 ** -23 * SCALE * (np.abs(q) @ np.abs(k).transpose(0, 1, 3, 2))
    if causal:
        mask = np.triu(np.ones((T, T), dtype=bool), 1)
        s = np.where(mask, -np.inf, s)
        ds = np.where(mask, 0.0, ds)
    m = s.max(-1, keepdims=True)
    w = np.exp(s - m)
    w /= w.sum(-1, keepdims=True)
    o = w @ v                                                                 # [B, H, T, 64]
    spread = np.empty_like(o)                                                 # sum_j w_j |v_j - O|, 16 query rows at a time
    for t0 in range(0, T, 16):
        d = np.abs(v[:, :, None, :, :] - o[:, :, t0:t0 + 16, None, :])
        spread[:, :, t0:t0 + 16] = np.einsum("bhtj,bhtjd->bhtd", w[:, :, t0:t0 + 16], d)
    wabs = w @ np.abs(v)
    smax = np.where(np.isinf(s), 0, np.abs(s)).max(-1, keepdims=True)
    eps = 2 * ds.max(-1, keepdims=True) + 8 * U * (smax + np.abs(m)) + 2.0 ** -20
    if path == "tc":
        eps = eps + 2.0 ** -8
    acc = (2 if path == "stream" else 1) * T * 2.0 ** -23
    bound = 2 * eps / (1 - eps) * spread + acc * (wabs + np.abs(o)) + 4 * U * np.abs(o)
    bound = bound + (2.0 ** -8 if planes == 1 else 2.0 ** -22) * (np.abs(o) + bound)
    o = torch.from_numpy(o.transpose(0, 2, 1, 3).reshape(B, T, heads * 64))
    bound = torch.from_numpy(bound.transpose(0, 2, 1, 3).reshape(B, T, heads * 64))
    return o, bound + 1e-30


def _attn_net(T: int, heads: int, mb: int, planes: int, causal: bool):
    m = Micro(mb, planes)
    t_qkv, t_out = m.tensor(T, 3 * heads * 64), m.tensor(T, heads * 64)
    m.net.op(nets.OP_ATTENTION, [t_qkv, t_out, T, heads, 64, int(causal)], [SCALE])
    m.net.set_output(4)
    return m, t_qkv, t_out


def _attn_run(m, t_qkv, t_out, imgs: torch.Tensor) -> torch.Tensor:
    """imgs: [B, T, 3*heads*64] in slots 0..B-1, FILL in the other slots; output planes of slots 0..B-1."""
    B = imgs.shape[0]
    x = torch.full((m.mb,) + tuple(imgs.shape[1:]), FILL)
    x[:B] = imgs
    m.write(t_qkv, x)
    m.view(t_out).fill_(SENTINEL)
    m.forward(B)
    out = m.view(t_out).cpu()
    assert bool((out[:, B:] == SENTINEL).all()), "attention wrote into an unused batch slot"
    return out[:, :B]


@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("case", ATTN_CASES, ids=lambda c: "T%d_h%d_B%d" % c)
@pytest.mark.parametrize("planes", [1, 3])
def test_attention_matches_fp64(case, causal, planes, monkeypatch, record_property):
    """Tensor-core kernel (1 plane, T <= 256), fp32 kernel (3 planes, T <= 256), streamed kernel (T > 256): output against
    the fp64 softmax per element; each image of the batch bit for bit equal to the same image run alone (neighbours and
    unused slots at 1e4, which would dominate any leaked key); the one-plane fp32 kernel (DCR_ATTN_FP32) against the
    reference and within the sum of both bounds of the tensor-core result."""
    T, heads, B = case
    gen = torch.Generator().manual_seed(T * 100 + heads * 10 + B + int(causal))
    imgs = torch.stack([_attn_image(gen, T, heads, causal) for _ in range(B)])
    if planes == 1:
        imgs = imgs.bfloat16().float()
    path = ("tc" if planes == 1 else "fp32") if T <= 256 else "stream"
    m, t_qkv, t_out = _attn_net(T, heads, B + 1, planes, causal)
    out = _attn_run(m, t_qkv, t_out, imgs)
    ref, bound = _attn_ref(imgs, heads, causal, path, planes)
    got = out.float().sum(0)
    err = (got.double() - ref).abs()
    _check(record_property, err, bound, path)
    for b in range(B):
        alone = _attn_run(m, t_qkv, t_out, imgs[b:b + 1])
        assert torch.equal(alone[:, 0], out[:, b]), f"image {b}: result depends on the rest of the batch"
    if planes == 1 and T <= 256:
        monkeypatch.setenv("DCR_B200_TUNING", "1")
        monkeypatch.setenv("DCR_ATTN_FP32", "1")
        fp = _attn_run(m, t_qkv, t_out, imgs)[0].float()
        _, bound_fp = _attn_ref(imgs, heads, causal, "fp32", 1)
        _check(record_property, (fp.double() - ref).abs(), bound_fp, "fp32 kernel, one plane")
        assert bool(((fp.double() - got.double()).abs() <= bound + bound_fp).all()), "TC and fp32 kernels disagree"


# ---- fused stem (STEM_ROWS + STEM_CONV) and the space-to-depth stem (STEM_S2D + CONV) -----------------------------
MEAN, STD = (0.5, 0.5, 0.5), (0.5, 0.5, 0.5)
IMNET_MEAN, IMNET_STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


def _transform(u8: torch.Tensor, cy: int, cx: int, h: int, w: int, mean, std, post=(1.0, 0.0)) -> torch.Tensor:
    """The arithmetic of oracle.models.preprocess (ToTensor u8 / 255, Normalize (x - mean) / std, fp32) on an
    arbitrary crop, then the post affine: uint8 [B, IH, IW, 3] -> fp32 [B, 3, h, w]."""
    x = u8[:, cy:cy + h, cx:cx + w, :].permute(0, 3, 1, 2).float().div(255.0)
    x = (x - torch.tensor(mean).view(1, 3, 1, 1)) / torch.tensor(std).view(1, 3, 1, 1)
    return x * post[0] + post[1] if tuple(post) != (1.0, 0.0) else x


def _images(gen, B: int, ih: int, iw: int) -> torch.Tensor:
    return torch.randint(0, 256, (B, ih, iw, 3), generator=gen, dtype=torch.uint8)


def _stem_params(gen):
    w = torch.randn(64, 3, 7, 7, generator=gen) / 147 ** 0.5
    return w, 0.5 + torch.rand(64, generator=gen), 0.1 * torch.randn(64, generator=gen)


def _stem_ref(x: torch.Tensor, w: torch.Tensor, sc: torch.Tensor, bi: torch.Tensor, exact_w: bool = False):
    """fp64 relu(sc * conv7x7/2/3(x, w) + bi) [B, OH, OW, 64] and the magnitude sc * conv(|x|, |w|) that bounds the
    fp32 accumulation error."""
    wd = w.double() if exact_w else w.bfloat16().double()
    y = F.conv2d(x.double(), wd, stride=2, padding=3)
    mag = F.conv2d(x.double().abs(), wd.abs(), stride=2, padding=3) * sc.double().view(1, 64, 1, 1)
    y = torch.relu(y * sc.double().view(1, 64, 1, 1) + bi.double().view(1, 64, 1, 1))
    return y.permute(0, 2, 3, 1), mag.permute(0, 2, 3, 1)


def _stem_bound_bf16(ref, mag):
    """Products of bf16 operands are exact in fp32; the 147 of them are summed in fp32 (|err| <= 147 * 2^-23 * mag with
    the tensor core's truncating accumulator), the BN affine adds 2 u; the bf16 store then rounds.  So the output is
    within one bf16 ulp of the reference plus the accumulation term."""
    slack = 147 * 2.0 ** -23 * mag + 4 * U * ref.abs()
    return _bf16_ulp(ref.abs() + slack) + slack


# (H, W, B): pooled-stem schedules of 4 / 2 / 1 parts per image (OHp = H/4 rounded up divisible by 4 / 2 / neither), the
# narrow widths whose MMA blocks span more conv rows than the old 8-row ring held, a rectangular crop and the widest
# crop stem_conv accepts.  B makes the pooled units (parts * B) exceed the 132 SMs: the persistent loop wraps.
STEM_CASES = [(224, 224, 40), (152, 152, 70), (146, 146, 140), (64, 64, 40), (40, 40, 70), (36, 36, 140),
              (34, 34, 140), (28, 28, 140), (64, 200, 40), (40, 262, 70)]


def _stem_net(B: int, ih: int, iw: int, cy: int, cx: int, H: int, W: int, w, sc, bi):
    m = Micro(B, 1)
    oh, ow = H // 2, W // 2
    units = int(m.lib.dcr_stem_plane_units(oh, ow))
    t_rows = m.tensor(2 * units, 8)
    m.net.op(nets.OP_STEM_ROWS, [t_rows, ih, iw, cy, cx, H, W], [*MEAN, *STD, 1.0, 0.0])
    w_id = m.net.param(nets._stem_toeplitz_weight(w).to(torch.bfloat16))
    sc_id, bi_id = m.net.param_f32(sc), m.net.param_f32(bi)
    t_full = m.tensor(oh * ow, 64)
    m.net.op(nets.OP_STEM_CONV, [t_rows, t_full, oh, ow, w_id, sc_id, bi_id, 0])
    t_pool = m.tensor(((oh - 1) // 2 + 1) * ((ow - 1) // 2 + 1), 64)
    m.net.op(nets.OP_STEM_CONV, [t_rows, t_pool, oh, ow, w_id, sc_id, bi_id, 1])
    m.net.set_output(4)
    return m, t_full, t_pool


@pytest.mark.parametrize("case", STEM_CASES, ids=lambda c: "%dx%d_B%d" % c)
def test_fused_stem_matches_fp64(case, record_property):
    """STEM_CONV without pooling against fp64 conv + BN + ReLU of the bf16-rounded transformed crop (one bf16 ulp); the
    pooled form bit for bit equal to F.max_pool2d(3, 2, 1) of the unpooled output.

    With the former fixed 8-row pooling ring, the 28- and 36-pixel crops failed here (28k and 55k pooled values
    wrong): a 128-position MMA block spans up to ceil(128 / PW) + 1 conv rows (PW = OW + 4), so on narrow images the
    block's ring stores land on rows that are still to be pooled, by a slower thread or by the next pooled row.  The
    ring depth now follows the width (stem_fused.cu, stem_ring_rows); images 96 pixels and wider keep 8 rows."""
    H, W, B = case
    gen = torch.Generator().manual_seed(H * 1000 + W)
    ih, iw, cy, cx = H + 6, W + 10, 3, 5
    u8 = _images(gen, B, ih, iw)
    w, sc, bi = _stem_params(gen)
    m, t_full, t_pool = _stem_net(B, ih, iw, cy, cx, H, W, w, sc, bi)
    m.forward(B, u8.cuda())
    oh, ow = H // 2, W // 2
    full = m.view(t_full)[0].float().cpu().view(B, oh, ow, 64)
    ref, mag = _stem_ref(_transform(u8, cy, cx, H, W, MEAN, STD).bfloat16().float(), w, sc, bi)
    _check(record_property, (full.double() - ref).abs(), _stem_bound_bf16(ref, mag), "fused stem")
    pooled = m.view(t_pool)[0].cpu().view(B, (oh - 1) // 2 + 1, (ow - 1) // 2 + 1, 64)
    want = F.max_pool2d(full.permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1).bfloat16()
    assert torch.equal(pooled, want), f"pooled stem differs from max_pool2d in {int((pooled != want).sum())} elements"


def test_fused_stem_refuses_too_wide_images():
    """The pooled stem keeps 8 conv rows of OW x 64 bf16 in shared memory next to the 32 KB of weights and one input
    window stage: 68352 + 1024 OW + 1024 ceil(32 ceil8(527 + 3 OW) / 1024) bytes within the 227 KB opt-in limit holds up
    to OW = 131 (a 262-pixel crop, run in test_fused_stem_matches_fp64).  OW = 132 must be refused by the host check
    before anything is launched."""
    m = Micro(1, 1)
    oh, ow = 20, 132
    t_rows = m.tensor(2 * int(m.lib.dcr_stem_plane_units(oh, ow)), 8)
    w, sc, bi = _stem_params(torch.Generator().manual_seed(0))
    t_pool = m.tensor(((oh - 1) // 2 + 1) * ((ow - 1) // 2 + 1), 64)
    m.net.op(nets.OP_STEM_CONV, [t_rows, t_pool, oh, ow, m.net.param(nets._stem_toeplitz_weight(w).to(torch.bfloat16)),
                                 m.net.param_f32(sc), m.net.param_f32(bi), 1])
    m.net.set_output(4)
    before = m.lib.dcr_kernel_launch_count()
    with pytest.raises(_lib.DcrError, match="too wide"):
        m.forward(1)
    assert m.lib.dcr_kernel_launch_count() == before


@pytest.mark.parametrize("planes", [1, 3])
@pytest.mark.parametrize("crop", [224, 64])
def test_s2d_stem_matches_fp64(crop, planes, record_property):
    """STEM_S2D + the 4x1-window CONV (the stem of the parity modes and of stem='s2d') against the same fp64 reference.
    One plane: one bf16 ulp as the fused stem.  Three planes: 6 cross terms of the split operands carry the fp32 input
    and weights; the dropped terms (lo x mid and smaller, ~2^-24 relative each) and the fp32 accumulation of 256 terms
    stay within 4e-5 of sc * conv(|x|, |w|), and the three output planes hold the fp32 result."""
    gen = torch.Generator().manual_seed(crop + planes)
    B = 6
    u8 = _images(gen, B, crop + 32, crop + 32)
    w, sc, bi = _stem_params(gen)
    m = Micro(B, planes)
    u = (crop + 6) // 2
    t_z, t_stem = m.tensor(u * u, 16), m.tensor((crop // 2) ** 2, 64)
    nets._input_op(m.net, nets.OP_STEM_S2D, t_z, crop + 32, crop, MEAN, STD)
    m.net.conv(t_z, t_stem, u, u - 3, 64, nets._stem_s2d_weight(w), scale=sc, bias=bi, act=1, window=(16, u))
    m.net.set_output(4)
    m.forward(B, u8.cuda())
    x = _transform(u8, 16, 16, crop, crop, MEAN, STD)
    got = m.merged(t_stem)[:B].view(B, crop // 2, crop // 2, 64)
    if planes == 1:
        ref, mag = _stem_ref(x.bfloat16().float(), w, sc, bi)
        bound = _stem_bound_bf16(ref, mag)
    else:
        ref, mag = _stem_ref(x, w, sc, bi, exact_w=True)
        bound = 4e-5 * mag + 2.0 ** -21 * ref.abs() + 1e-30
    _check(record_property, (got.double() - ref).abs(), bound, "s2d stem")


# ---- image input transform (IM2COL_U8, STEM_S2D, STEM_ROWS) ------------------------------------------------------------
def _im2col_ref(x: torch.Tensor, kh: int, kw: int, stride: int, pad: int, k_pad: int) -> torch.Tensor:
    """fp32 [B, 3, RH, RW] -> [B, OH * OW, k_pad] in im2col_u8's layout k = r * RP + s * 3 + c, RP = ceil8(3 kw), zero
    in the row padding, at padding taps and for k >= kh * RP."""
    B = x.shape[0]
    cols = F.unfold(F.pad(x, (pad, pad, pad, pad)), (kh, kw), stride=stride)          # [B, 3 * kh * kw, L], (c, r, s)
    L = cols.shape[-1]
    cols = cols.view(B, 3, kh, kw, L).permute(0, 4, 2, 3, 1).reshape(B, L, kh, 3 * kw)
    rp = (3 * kw + 7) // 8 * 8
    cols = F.pad(cols, (0, rp - 3 * kw)).reshape(B, L, kh * rp)
    return F.pad(cols, (0, k_pad - kh * rp))


# name: (kh, kw, stride, pad, IH, IW, crop_y, crop_x, H, W, mean, std, post, scale_factor)
IM2COL_CASES = {
    "vit16": (16, 16, 16, 0, 256, 256, 16, 16, 224, 224, MEAN, STD, (1.0, 0.0), None),
    "vit8": (8, 8, 8, 0, 80, 80, 8, 8, 64, 64, MEAN, STD, (1.0, 0.0), None),
    "vit14": (14, 14, 14, 0, 128, 128, 8, 8, 112, 112, IMNET_MEAN, IMNET_STD, (1.0, 0.0), None),
    "inception": (3, 3, 2, 0, 299, 299, 0, 0, 299, 299, MEAN, STD, (2.0, -1.0), None),
    "vgg": (3, 3, 1, 1, 64, 72, 5, 11, 56, 48, IMNET_MEAN, IMNET_STD, (1.0, 0.0), None),     # crop off centre
    "resnet7": (7, 7, 2, 3, 70, 70, 1, 4, 64, 64, MEAN, STD, (1.0, 0.0), None),
    "vit16_resize": (16, 16, 16, 0, 256, 256, 16, 16, 224, 224, MEAN, STD, (1.0, 0.0), 2 ** -0.5),
    "vgg_resize": (3, 3, 1, 1, 64, 64, 4, 4, 56, 56, IMNET_MEAN, IMNET_STD, (1.0, 0.0), 1.25),
}


def _resized(x: torch.Tensor, s):
    return x if s is None else F.interpolate(x, scale_factor=s, mode="bilinear", align_corners=False)


def _input_args(ih, iw, cy, cx, h, w, mean, std, post, s, op_ints=()):
    iargs = [ih, iw, cy, cx, h, w, *op_ints]
    fargs = [*mean, *std, *post]
    if s is not None:
        iargs += [nets._scaled_size(h, s), nets._scaled_size(w, s)]
        fargs.append(float(np.float32(1.0 / s)))
    return iargs, fargs


@pytest.mark.parametrize("name", list(IM2COL_CASES))
def test_im2col_matches_torch(name, record_property):
    """IM2COL_U8 on a 3-plane net (the merged planes hold the kernel's fp32 value) against an im2col built in torch from
    the same transform: bit for bit without resizing (same fp32 operations: u8 / 255, (x - mean) / std, post affine),
    within one fp32 ulp of F.interpolate(bilinear, align_corners=False) with it (the kernel evaluates torch's
    lerps as fma(h, a, l * b) where torch may round h * a first).  The fp32 NCHW input form must give the same planes
    bit for bit as the uint8 form."""
    kh, kw, stride, pad, ih, iw, cy, cx, h, w, mean, std, post, s = IM2COL_CASES[name]
    gen = torch.Generator().manual_seed(kh * 100 + ih)
    B = 2
    u8 = _images(gen, B, ih, iw)
    k_pad = nets.first_conv_k_pad(kh, kw)
    rh, rw = nets._scaled_size(h, s), nets._scaled_size(w, s)
    oh, ow = (rh + 2 * pad - kh) // stride + 1, (rw + 2 * pad - kw) // stride + 1
    m = Micro(B + 1, 3)
    t = m.tensor(oh * ow, k_pad)
    iargs, fargs = _input_args(ih, iw, cy, cx, h, w, mean, std, post, s, [kh, kw, stride, pad, k_pad])
    m.net.op(nets.OP_IM2COL_U8, [t] + iargs, fargs)
    m.net.set_output(4)
    m.write(t, torch.full((B + 1, oh * ow, k_pad), SENTINEL))
    m.forward(B, u8.cuda())
    got = m.merged(t)
    assert bool((got[B:] == SENTINEL).all())
    if name == "inception":     # FID: metrics/fid.py's transform, then InceptionV3's own 2x - 1
        x = om.fid_preprocess(u8) * 2.0 - 1.0
        assert torch.equal(x, _transform(u8, 0, 0, h, w, mean, std, post))
    else:
        x = _transform(u8, cy, cx, h, w, mean, std, post)
    ref = _im2col_ref(_resized(x, s), kh, kw, stride, pad, k_pad)
    if s is None:
        record_property("max_err", float((got[:B] - ref).abs().max()))
        assert torch.equal(got[:B], ref), f"{int((got[:B] != ref).sum())} elements differ"
    else:
        ulps = _fp32_ulps(got[:B], ref)
        record_property("max_err_fp32_ulps", ulps)
        assert ulps <= 1.0, f"resized im2col {ulps} fp32 ulps from F.interpolate"
    planes_u8 = m.view(t)[:, :B].clone()
    m.view(t).zero_()
    xf = _transform(u8, cy, cx, h, w, mean, std)     # the caller's transformed crop; the kernel applies the post affine
    m.forward(B, xf.cuda(), f32=True)
    assert torch.equal(m.view(t)[:, :B], planes_u8), "fp32 input form differs from the uint8 form"


@pytest.mark.parametrize("s", [None, 1.25])
def test_stem_s2d_layout(s, record_property):
    """STEM_S2D (3 planes): Z[b, u, v, (i*2+j)*3 + c] = x[c, 2u + i - 3, 2v + j - 3], zero outside the image and in
    channels 12..15, rebuilt in torch from the same transformed (and resized) crop; off-centre crop."""
    gen = torch.Generator().manual_seed(7)
    B, ih, iw, cy, cx, h, w = 2, 80, 90, 3, 17, 64, 64
    u8 = _images(gen, B, ih, iw)
    rh, rw = nets._scaled_size(h, s), nets._scaled_size(w, s)
    U, V = (rh + 6) // 2, (rw + 6) // 2
    m = Micro(B, 3)
    t = m.tensor(U * V, 16)
    iargs, fargs = _input_args(ih, iw, cy, cx, h, w, IMNET_MEAN, IMNET_STD, (1.0, 0.0), s)
    m.net.op(nets.OP_STEM_S2D, [t] + iargs, fargs)
    m.net.set_output(4)
    m.write(t, torch.full((B, U * V, 16), SENTINEL))
    m.forward(B, u8.cuda())
    x = _resized(_transform(u8, cy, cx, h, w, IMNET_MEAN, IMNET_STD), s)
    z = F.pad(x, (3, 3, 3, 3)).view(B, 3, U, 2, V, 2).permute(0, 2, 4, 3, 5, 1).reshape(B, U * V, 12)
    ref = F.pad(z, (0, 4))
    got = m.merged(t)
    if s is None:
        assert torch.equal(got, ref), f"{int((got != ref).sum())} elements differ"
    else:
        ulps = _fp32_ulps(got, ref)
        record_property("max_err_fp32_ulps", ulps)
        assert ulps <= 1.0
        assert bool((got[..., 12:] == 0).all())


@pytest.mark.parametrize("s", [None, 1.25])
def test_stem_rows_layout(s, record_property):
    """STEM_ROWS (one plane): plane_e[P * PW + u] = (x[2P + i - 3, 2u + e - 3, c] for i, c) + 2 zero channels, bf16,
    PW = OW + 4, P < OH + 3; the rest of each plane (read slack of the pooled schedule) stays zero.  Rebuilt in torch
    from the same transformed crop and rounded to bf16: bit for bit without resizing, one bf16 rounding of a value within
    one fp32 ulp with it."""
    gen = torch.Generator().manual_seed(8)
    B, ih, iw, cy, cx, h, w = 3, 70, 80, 2, 9, 40, 64
    u8 = _images(gen, B, ih, iw)
    rh, rw = nets._scaled_size(h, s), nets._scaled_size(w, s)
    oh, ow = rh // 2, rw // 2
    m = Micro(B, 1)
    units = int(m.lib.dcr_stem_plane_units(oh, ow))
    t = m.tensor(2 * units, 8)
    iargs, fargs = _input_args(ih, iw, cy, cx, h, w, MEAN, STD, (1.0, 0.0), s)
    m.net.op(nets.OP_STEM_ROWS, [t] + iargs, fargs)
    m.net.set_output(4)
    m.forward(B, u8.cuda())
    x = _resized(_transform(u8, cy, cx, h, w, MEAN, STD), s)
    pw = ow + 4
    xp = F.pad(x, (3, 2 * pw - rw - 3, 3, 3))                                           # [B, 3, 2 (OH + 3), 2 PW]
    rows = xp.view(B, 3, oh + 3, 2, pw, 2).permute(0, 5, 2, 4, 3, 1).reshape(B, 2, (oh + 3) * pw, 6)
    ref = torch.zeros(B, 2, units, 8)
    ref[:, :, :(oh + 3) * pw, :6] = rows
    got = m.view(t)[0].cpu().view(B, 2, units, 8)
    if s is None:
        want = ref.bfloat16()
        assert torch.equal(got, want), f"{int((got != want).sum())} elements differ"
    else:
        # the kernel's sample is within one fp32 ulp (2^-16 bf16 ulp) of torch's, then rounds to bf16 (half an ulp)
        err = (got.double() - ref.double()).abs()
        bound = _bf16_ulp(ref.abs() * (1 + 2.0 ** -22)) * (0.5 + 2.0 ** -15) + 1e-30
        _check(record_property, err, bound, "resized stem rows")
        assert bool((got[..., 6:] == 0).all())


# ---- LayerNorm (op 6) ---------------------------------------------------------------------------------------------------
def _ln_ref(x: torch.Tensor, g: torch.Tensor, b: torch.Tensor, eps: float, n_seq: int):
    """fp64 LayerNorm of the merged rows x [R, C] and the bound of the kernel's fp32 result.

    The mean is a fp32 sum of C values (n_seq sequential terms per lane, then <= 5 shuffle levels): |dmean| <= (n_seq +
    5) u mean|x|, which moves every output by |g| rstd |dmean| -- with a mean of 100 sigma this is the term that matters.
    The variance sums (x - mean)^2 the same way: relative (n_seq + 8) u, plus sqrt and division: the normalised value
    xhat carries (n_seq + 12) u of itself.  Then (xhat * g + b): 4 u of |g xhat| + |b|."""
    xd, gd, bd = x.double(), g.double(), b.double()
    mean = xd.mean(1, keepdim=True)
    rstd = 1.0 / torch.sqrt(((xd - mean) ** 2).mean(1, keepdim=True) + eps)
    xhat = (xd - mean) * rstd
    y = xhat * gd + bd
    dmean = (n_seq + 5) * U * xd.abs().mean(1, keepdim=True)
    bound = gd.abs() * rstd * dmean + gd.abs() * xhat.abs() * (n_seq + 12) * U + 4 * U * ((gd * xhat).abs() + bd.abs())
    return y, bound + 1e-30


# (C, rows per image, B): fast path for C in 384 / 512 / 768 / 1024 (one half-warp per row), generic path otherwise;
# rows 1 / 15 / 17 cover the half-warp tails
LN_CASES = [(384, 1, 1), (512, 15, 1), (768, 17, 1), (1024, 500, 2), (256, 17, 1), (640, 15, 1), (1000, 500, 2)]


@pytest.mark.parametrize("generic", [False, True])
@pytest.mark.parametrize("planes", [1, 3])
@pytest.mark.parametrize("case", LN_CASES, ids=lambda c: "C%d_r%d_B%d" % c)
def test_layernorm_matches_fp64(case, planes, generic, monkeypatch, record_property):
    """LAYERNORM on inputs with a mean of ~100 sigma: the bf16 / split planes and the fp32 rows written to the output
    buffer (to_output), against fp64; one plane with and without DCR_LN_GENERIC, three planes.  bf16 planes add one
    rounding (2^-8 of the value: 8 significant bits); three planes hold the fp32 result."""
    C_, rows, B = case
    if generic and planes == 3:
        pytest.skip("three planes always take the generic kernel")
    if generic:
        monkeypatch.setenv("DCR_B200_TUNING", "1")
        monkeypatch.setenv("DCR_LN_GENERIC", "1")
    gen = torch.Generator().manual_seed(C_ + rows)
    m = Micro(B + 1, planes)
    t_in, t_out = m.tensor(rows, C_), m.tensor(rows, C_)
    g, b = 1 + 0.5 * torch.randn(C_, generator=gen), 0.2 * torch.randn(C_, generator=gen)
    m.net.op(nets.OP_LAYERNORM, [t_in, t_out, rows, C_, m.net.param_f32(g), m.net.param_f32(b), 1, 1], [1e-6])
    m.net.set_output(rows * C_)
    x = 100 + torch.randn(B + 1, rows, C_, generator=gen)
    x[B:] = FILL
    m.write(t_in, x)
    m.write(t_out, torch.full((B + 1, rows, C_), SENTINEL))
    out32 = m.forward(B).view(B * rows, C_)
    xin = m.merged(t_in)[:B].reshape(B * rows, C_)
    n_seq = C_ // 16 if (planes == 1 and C_ in (384, 512, 768, 1024) and not generic) else C_ // 32 + 8
    ref, bound = _ln_ref(xin, g, b, 1e-6, n_seq)
    _check(record_property, (out32.double() - ref).abs(), bound, "fp32 rows")
    got = m.merged(t_out)
    assert bool((got[B:] == SENTINEL).all())
    pb = bound + (2.0 ** -8 if planes == 1 else 2.0 ** -22) * (ref.abs() + bound)
    _check(record_property, (got[:B].reshape(B * rows, C_).double() - ref).abs(), pb, "planes")


@pytest.mark.parametrize("generic", [False, True])
def test_layernorm_cls_rows(generic, monkeypatch, record_property):
    """The CLS-only form of the ViT / CLIP heads (in_row_stride = T rows: row b reads token 0 of image b)."""
    if generic:
        monkeypatch.setenv("DCR_B200_TUNING", "1")
        monkeypatch.setenv("DCR_LN_GENERIC", "1")
    T, C_, B = 197, 384, 3
    gen = torch.Generator().manual_seed(197)
    m = Micro(B, 1)
    t_in, t_out = m.tensor(T, C_), m.tensor(1, C_)
    g, b = 1 + 0.5 * torch.randn(C_, generator=gen), 0.2 * torch.randn(C_, generator=gen)
    m.net.op(nets.OP_LAYERNORM, [t_in, t_out, 1, C_, m.net.param_f32(g), m.net.param_f32(b), T, 1], [1e-6])
    m.net.set_output(C_)
    x = 100 + torch.randn(B, T, C_, generator=gen)
    x[:, 1:] = FILL
    m.write(t_in, x)
    out32 = m.forward(B)
    ref, bound = _ln_ref(m.merged(t_in)[:, 0], g, b, 1e-6, C_ // 16 if not generic else C_ // 32 + 8)
    _check(record_property, (out32.double() - ref).abs(), bound, "fp32 rows")
    got = m.merged(t_out)[:, 0]
    _check(record_property, (got.double() - ref).abs(), bound + 2.0 ** -8 * (ref.abs() + bound), "bf16 rows")


# ---- max / avg pooling (ops 2, 3) ---------------------------------------------------------------------------------------
# (H, W, C, k, stride, pad): odd output widths (7, 11, 17) for the two-outputs-per-thread max kernel; 2x2/2 (VGG) and
# 3x3/1/1 (Inception avg) shapes
POOL_CASES = [(13, 13, 64, 3, 2, 1), (9, 11, 16, 3, 1, 1), (35, 35, 24, 3, 2, 0), (14, 17, 32, 3, 2, 0),
              (8, 8, 64, 2, 2, 0), (12, 12, 40, 3, 1, 0)]


@pytest.mark.parametrize("generic", [False, True])
@pytest.mark.parametrize("is_max", [True, False])
@pytest.mark.parametrize("case", POOL_CASES, ids=lambda c: "%dx%dx%d_k%d_s%d_p%d" % c)
def test_pool_matches_torch(case, is_max, generic, monkeypatch, record_property):
    """MAXPOOL / AVGPOOL (count_include_pad=False), one plane, fast kernels and DCR_POOL_GENERIC, into the middle columns
    of a wider output (the Inception concat: ld_out = C + 24, out_col_off = 8): max bit for bit (a maximum of bf16
    values is one of them); avg an fp32 sum of <= 9 bf16 values (exact below 2^16 ulps of spread, here within 9 u)
    and one division, then the bf16 store: within one bf16 ulp.  Neighbouring columns and unused batch slots keep their
    sentinel."""
    H, W, C_, k, stride, pad = case
    if generic:
        monkeypatch.setenv("DCR_B200_TUNING", "1")
        monkeypatch.setenv("DCR_POOL_GENERIC", "1")
    B, off, ld = 3, 8, C_ + 24
    oh, ow = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    gen = torch.Generator().manual_seed(H * W + C_ + k)
    m = Micro(B + 1, 1)
    t_in, t_out = m.tensor(H * W, C_), m.tensor(oh * ow, ld)
    m.net.op(nets.OP_MAXPOOL if is_max else nets.OP_AVGPOOL, [t_in, t_out, H, W, C_, k, stride, pad, off])
    m.net.set_output(4)
    x = torch.randn(B + 1, H * W, C_, generator=gen)
    x[B:] = FILL
    m.write(t_in, x)
    m.write(t_out, torch.full((B + 1, oh * ow, ld), SENTINEL))
    m.forward(B)
    xin = m.merged(t_in)[:B].view(B, H, W, C_).permute(0, 3, 1, 2).double()
    got = m.merged(t_out)
    assert bool((got[B:] == SENTINEL).all()), "pool wrote into an unused batch slot"
    assert bool((got[:B, :, :off] == SENTINEL).all()) and bool((got[:B, :, off + C_:] == SENTINEL).all()), \
        "pool wrote outside its output columns"
    got = got[:B, :, off:off + C_].view(B, oh, ow, C_).permute(0, 3, 1, 2).double()
    if is_max:
        ref = F.max_pool2d(xin, k, stride, pad)
        record_property("max_err", float((got - ref).abs().max()))
        assert torch.equal(got, ref)
    else:
        ref = F.avg_pool2d(xin, k, stride, pad, count_include_pad=False)
        _check(record_property, (got - ref).abs(), _bf16_ulp(ref) + 1e-30, "avg pool")


# ---- GeM / GAP (ops 4, 5) ---------------------------------------------------------------------------------------------
# (HW, C): C = 8 (one group), 2048 (4 column blocks of 64 groups), 2056 (a fifth block with one group)
REDUCE_CASES = [(1, 8), (49, 2048), (3136, 2056), (49, 2056), (1, 2048), (3136, 8)]


@pytest.mark.parametrize("planes", [1, 3])
@pytest.mark.parametrize("kind", ["gem3", "gem2.5", "gap"])
@pytest.mark.parametrize("case", REDUCE_CASES, ids=lambda c: "HW%d_C%d" % c)
def test_gem_gap_matches_fp64(case, kind, planes, record_property):
    """GeM (p = 3: cube and cbrtf; p = 2.5: powf) and GAP over HW positions, inputs partly below eps and negative
    (clamped to eps by GeM).  Error of the fp32 result: the sum runs over HW / 4 sequential terms per slice and 4 slices,
    (HW / 4 + 8) u of the sum of |terms|; the power of each term 2 ulps (t t t, or powf), the division u; the 1/p root
    divides the relative error by p and adds 2 ulps, and 1/p rounded to fp32 moves it by u |ln mean| / p.  The
    planes add the bf16 store (one plane) or hold the fp32 value (three)."""
    HW, C_ = case
    p = {"gem3": 3.0, "gem2.5": 2.5, "gap": None}[kind]
    eps = 1e-6
    B = 3
    gen = torch.Generator().manual_seed(HW + C_)
    m = Micro(B + 1, planes)
    t_in, t_out = m.tensor(HW, C_), m.tensor(1, C_)
    if p is None:
        m.net.op(nets.OP_GAP, [t_in, t_out, HW, C_, 1])
    else:
        m.net.op(nets.OP_GEM, [t_in, t_out, HW, C_, 1], [p, eps])
    m.net.set_output(C_)
    x = torch.rand(B + 1, HW, C_, generator=gen) * 2
    x[:, ::3] = -torch.rand(B + 1, (HW + 2) // 3, C_, generator=gen)        # negative: clamped to eps
    x[:, 1::5] *= 1e-7                                                       # below eps
    x[0, :, :8] = -1.0                                                       # a whole channel group at eps
    x[B:] = FILL
    m.write(t_in, x)
    out32 = m.forward(B)
    xin = m.merged(t_in)[:B].double()
    if p is None:
        ref = xin.mean(1)
        bound = (HW / 4 + 8) * U * xin.abs().mean(1) + 2 * U * ref.abs()
    else:
        t = xin.clamp_min(eps) ** p
        mean = t.mean(1)
        ref = mean ** (1 / p)
        rel = ((HW / 4 + 8) * U + 3 * U) / p + 2 * U + U * mean.log().abs() / p
        bound = rel * ref
    bound = bound + 1e-30
    _check(record_property, (out32.double() - ref).abs(), bound, "fp32 output")
    got = m.merged(t_out)[:B, 0].double()
    pb = bound + (2.0 ** -8 if planes == 1 else 2.0 ** -22) * (ref.abs() + bound)
    _check(record_property, (got - ref).abs(), pb, "planes")


# ---- VIT_TOKENS (op 7), EMBED (op 11) --------------------------------------------------------------------------------
@pytest.mark.parametrize("planes", [1, 3])
def test_vit_tokens_bitwise(planes):
    """tokens[b, 0] = cls + pos[0], tokens[b, 1 + i] = patch[b, i] + pos[1 + i]: the same fp32 sums split into planes."""
    B, NP, C_ = 3, 196, 384
    gen = torch.Generator().manual_seed(196)
    m = Micro(B + 1, planes)
    t_patch, t_tok = m.tensor(NP, C_), m.tensor(NP + 1, C_)
    cls, pos = torch.randn(C_, generator=gen), torch.randn(NP + 1, C_, generator=gen)
    m.net.op(nets.OP_VIT_TOKENS, [t_patch, t_tok, NP, C_, m.net.param_f32(cls), m.net.param_f32(pos)])
    m.net.set_output(4)
    m.write(t_patch, torch.randn(B + 1, NP, C_, generator=gen))
    m.write(t_tok, torch.full((B + 1, NP + 1, C_), SENTINEL))
    m.forward(B)
    patch = m.merged(t_patch)[:B]
    want = torch.cat([cls.expand(B, 1, C_), patch], 1) + pos
    assert torch.equal(m.view(t_tok)[:, :B].cpu(), split_planes(want, planes))
    assert bool((m.merged(t_tok)[B:] == SENTINEL).all())


@pytest.mark.parametrize("planes", [1, 3])
def test_embed_bitwise_and_clamps_ids(planes):
    """rows table[id] + pos[t] as fp32 sums split into planes; ids below 0 or >= vocab clamp to [0, vocab - 1]."""
    B, T, C_, vocab = 3, 77, 512, 1000
    gen = torch.Generator().manual_seed(77)
    m = Micro(B, planes)
    t = m.tensor(T, C_)
    table, pos = torch.randn(vocab, C_, generator=gen), torch.randn(T, C_, generator=gen)
    m.net.op(nets.OP_EMBED, [t, T, C_, m.net.param_f32(table), m.net.param_f32(pos), vocab])
    m.net.set_output(4)
    ids = torch.randint(0, vocab, (B, T), generator=gen, dtype=torch.int32)
    ids[0, :4] = torch.tensor([-1, -(2 ** 31), vocab, 2 ** 31 - 1], dtype=torch.int32)
    ids[1, -1] = vocab - 1
    m.forward(B, ids.cuda())
    want = table[ids.long().clamp(0, vocab - 1)] + pos
    assert torch.equal(m.view(t).cpu(), split_planes(want, planes))
