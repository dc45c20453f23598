"""GPU numerics of the network executor's convolution op (OP_CONV) on the paths that only the executor reaches: the fused
bottleneck kernel (bottleneck_fuse.cu) at full-batch tile counts, the float64 path of the exact mode (conv_exact.cu),
Inception-style concat slices (out_col_off), fp32 heads (to_output), QuickGELU on both epilogues and the two-plane
bf16x3 mode.

Conventions of test_net_ops_gpu.py: a micro-network around the op, input planes written through dcr_net_tensor, FILL in
unused batch slots, SENTINEL in output tensors, a float64 reference computed from the merged planes the kernel read, every
bound derived in a comment, the measured error recorded as test properties (max_err, max_err_over_bound)."""
import math

import pytest
import torch
import torch.nn.functional as F

from dcr_b200 import _lib, nets, similarity
from dcr_b200.ops import split_planes
from tests.test_net_ops_gpu import FILL, SENTINEL, U, Micro, _bf16_ulp, _check

pytestmark = pytest.mark.gpu

LIP = 1.13                      # bound of |d act / dy| for GELU (max 1.129) and QuickGELU (max 1.0998)
MARGIN = 1.0001                 # second-order terms of the first-order activation bounds (relative errors < 1e-5)


def _gen(seed: int) -> torch.Generator:
    return torch.Generator(device="cuda").manual_seed(seed)


def _merged_w(w: torch.Tensor, planes: int) -> torch.Tensor:
    """The weight values the kernel multiplies by: the planes of prepare_conv_weight, summed (elementwise split)."""
    return split_planes(w.cuda(), planes).float().sum(0)


def _conv64(x: torch.Tensor, w: torch.Tensor, stride: int, pad) -> tuple:
    """NHWC x [B, H, W, C], w [N, C, kh, kw] -> fp64 (sum, sum of |x||w|) [B, P, Q, N] through an explicit im2col and a
    float64 matmul: every output is a K-term dot product, so its error is at most gamma_K = K 2^-53 of the second."""
    B, H, W, _ = x.shape
    N, _, kh, kw = w.shape
    P, Q = (H + 2 * pad[0] - kh) // stride + 1, (W + 2 * pad[1] - kw) // stride + 1
    cols = F.unfold(x.double().permute(0, 3, 1, 2), (kh, kw), padding=tuple(pad), stride=stride).transpose(1, 2)
    wm = w.double().reshape(N, -1).t()
    return (cols @ wm).view(B, P, Q, N), (cols.abs() @ wm.abs()).view(B, P, Q, N)


def _bits_equal(a: torch.Tensor, b: torch.Tensor) -> bool:
    iv = {torch.bfloat16: torch.int16, torch.float32: torch.int32}[a.dtype]
    return a.dtype == b.dtype and torch.equal(a.contiguous().view(iv), b.contiguous().view(iv))


# ---- A. fused bottleneck kernel at full-batch tile counts ------------------------------------------------------------
# (C, N1, N2, H, W); N2 = 0 is the expansion-only kernel.  With the 232448-byte opt-in, expand_reduce_impl plans
# (a_bufs, W stages, W tiles per column block): layer1 pair (2, 4, 1 + 2), layer1 -> layer2 pair (1, 4, 1 + 2), layer2
# pair (1, 3, 2 + 2), expand-only (1, 3, 4), one column block (1, 4, 3 + 2: nb = 1, so every residual prefetch crosses
# into the CTA's next m-tile).  These plans are derived from the host code.
FUSE_CASES = {
    "layer1_pair": (64, 256, 64, 56, 56),
    "layer1_to_layer2": (64, 256, 128, 56, 56),
    "layer2_pair": (128, 512, 128, 28, 28),
    "expand_only": (256, 1024, 0, 14, 14),
    "one_column_block": (192, 128, 64, 28, 28),
}


def _full_batch(hw: int, sms: int) -> int:
    """The smallest batch whose M = B * hw rows give at least 3 m-tiles of 128 rows per SM, a partial last tile and a
    tile count that is no multiple of the SM count (CTAs run unequal numbers of tiles)."""
    b = 1
    while True:
        m = b * hw
        tiles = -(-m // 128)
        if tiles >= 3 * sms and m % 128 and tiles % sms:
            return b
        b += 1


def _fused_bound(s: torch.Tensor, mag: torch.Tensor, sc, bi, r, K: int):
    """fp64 relu(sc * s + bi (+ r)) and the bound of the kernel's bf16 value.  The bf16 x bf16 products are exact in
    fp32; their fp32 accumulation over K terms moves s by at most K 2^-23 sum |a||w| (mag).  fmaf and the residual add
    round twice: 2 u of |sc s| + |bi| + |r| (3 u with the second-order terms).  ReLU is 1-Lipschitz; the bf16 store
    rounds to nearest: half a bf16 ulp at the stored magnitude, at most |ref| + slack."""
    pre = s * sc + bi
    mags = (s * sc).abs() + bi.abs()
    if r is not None:
        pre, mags = pre + r, mags + r.abs()
    ref = torch.relu(pre)
    slack = K * 2.0 ** -23 * sc.abs() * mag + 3 * U * mags
    return ref, 0.5 * _bf16_ulp(ref + slack) + slack + 1e-30


def _kernel_names(fn) -> list:
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events()]


@pytest.mark.parametrize("name", list(FUSE_CASES))
def test_fused_bottleneck_full_batch(name, monkeypatch, record_property):
    """conv(T2 -> Y, residual X, ReLU) followed by conv(Y -> T1, ReLU) -- or the expansion alone -- at a batch that gives
    every CTA of the persistent grid three or more m-tiles: the residual prefetch into the X buffer of two tiles back,
    the a_full / a_empty rotation, the T1 staging reuse and the W ring's phase across m-tiles all run.  The fused
    launch (one kernel for the pair, expand_reduce_kernel by name) must give Y and T1 bit for bit equal to the separate
    conv_gemm launches (DCR_NO_BLOCK_FUSION); Y within the bound of the fp64 reference from the T2, W3, X and BN
    tables the kernel read, T1 within the bound of the reference from the Y the kernel stored; slot B of Y and T1
    (rows past M: the partial last tile) keeps its sentinel."""
    C_, N1, N2, H, W = FUSE_CASES[name]
    hw = H * W
    B = _full_batch(hw, int(_lib.load().dcr_device_sm_count()))
    record_property("batch", B)
    g = _gen(C_ + N1 + N2)
    m = Micro(B + 1, "fast")
    t_t2, t_x, t_y = m.tensor(hw, C_), m.tensor(hw, N1), m.tensor(hw, N1)
    w3 = torch.randn(N1, C_, device="cuda", generator=g) / C_ ** 0.5
    sc3, bi3 = 0.5 + torch.rand(N1, device="cuda", generator=g), 0.1 * torch.randn(N1, device="cuda", generator=g)
    m.net.conv(t_t2, t_y, H, W, C_, w3.cpu(), scale=sc3.cpu(), bias=bi3.cpu(), residual=t_x, act=1)
    if N2:
        t_t1 = m.tensor(hw, N2)
        w1 = torch.randn(N2, N1, device="cuda", generator=g) / N1 ** 0.5
        sc1, bi1 = 0.5 + torch.rand(N2, device="cuda", generator=g), 0.1 * torch.randn(N2, device="cuda", generator=g)
        m.net.conv(t_y, t_t1, H, W, N1, w1.cpu(), scale=sc1.cpu(), bias=bi1.cpu(), act=1)
    m.net.set_output(4)
    # T2 >= 0 (a ReLU output) with all-zero rows; X rows at -1000 over a whole 128-column block: ReLU clamps the block
    t2 = torch.rand(B + 1, hw, C_, device="cuda", generator=g)
    t2[:, ::7] = 0
    x = torch.randn(B + 1, hw, N1, device="cuda", generator=g)
    x[:, 1::5, :128] = -1000.0
    x[:, 3::5, N1 - 128:] = -1000.0
    t2[B:], x[B:] = FILL, FILL
    m.write(t_t2, t2)
    m.write(t_x, x)
    outs = [t_y] + ([t_t1] if N2 else [])

    def run():
        for t in outs:
            m.view(t).fill_(SENTINEL)
        l0 = similarity.kernel_launch_count()
        m.forward(B)
        return similarity.kernel_launch_count() - l0, [m.view(t)[0].clone() for t in outs]

    res = {}
    names = _kernel_names(lambda: res.setdefault("fused", run()))
    n_fused, fused = res["fused"]
    assert n_fused == 1, f"{n_fused} launches: the layers did not run as one fused kernel"
    assert any("expand_reduce_kernel" in k for k in names), f"expand_reduce_kernel did not run: {sorted(set(names))}"
    monkeypatch.setenv("DCR_B200_TUNING", "1")
    monkeypatch.setenv("DCR_NO_BLOCK_FUSION", "1")
    n_plain, plain = run()
    assert n_plain == len(outs)
    for what, f, p in zip(("Y", "T1"), fused, plain):
        assert bool((f[B:] == SENTINEL).all()), f"fused kernel wrote {what} rows past M"
        if not _bits_equal(f, p):
            bad = (f.view(torch.int16) != p.view(torch.int16)).view(B + 1, -1).any(1)
            raise AssertionError(f"{what}: fused differs from the separate launches in images {bad.nonzero().flatten().tolist()}")
    # Y against fp64 from the operands the kernel read
    a = m.view(t_t2)[0, :B].reshape(-1, C_).double()
    w3m = _merged_w(w3, 1).double()
    xr = m.view(t_x)[0, :B].reshape(-1, N1).double()
    ref, bound = _fused_bound(a @ w3m.t(), a.abs() @ w3m.abs().t(), sc3.double(), bi3.double(), xr, C_)
    y = fused[0][:B].reshape(-1, N1).double()
    _check(record_property, (y - ref).abs(), bound, "Y")
    assert bool((ref == 0).view(B, hw, N1)[:, 1::5, :128].all())   # the clamped blocks are there
    if N2:
        w1m = _merged_w(w1, 1).double()
        ref1, bound1 = _fused_bound(y @ w1m.t(), y.abs() @ w1m.abs().t(), sc1.double(), bi1.double(), None, N1)
        _check(record_property, (fused[1][:B].reshape(-1, N2).double() - ref1).abs(), bound1, "T1")


# ---- B. float64 path (exact mode, conv_exact.cu) ---------------------------------------------------------------------
def _tie_neighbours(t: torch.Tensor):
    """t fp64 -> (RN fp32 value, its neighbour on t's side, t exactly halfway between the two)."""
    f = t.float()
    toward = torch.where(t > f.double(), torch.full_like(f, math.inf), torch.full_like(f, -math.inf))
    other = torch.nextafter(f, toward)
    tie = (f.double() != t) & ((f.double() + other.double()) * 0.5 == t)
    return f, other, tie


def _exact_pre(s32: torch.Tensor, sc, bi, r, upper: bool) -> torch.Tensor:
    """conv_exact's epilogue before the activation, in fp32: fmaf(s, scale, bias), then + residual.  fmaf is emulated
    as one fp64 operation (s * scale is exact in fp64) rounded to fp32: the same value unless the fp64 result is a tie
    of the fp32 rounding, where the lower (upper=False) or upper neighbour is taken."""
    f, other, tie = _tie_neighbours(s32.double() * sc.double() + bi.double())
    y = torch.where(tie, torch.minimum(f, other) if not upper else torch.maximum(f, other), f)
    return y + r if r is not None else y


def _exact_ref(s64, mag, K: int, sc, bi, r, act: int):
    """(lower, upper) fp32 outputs for act 0 / 1, or (fp64 reference, bound) for act 2 / 3.

    conv_exact sums the exact fp32 x fp32 products in fp64 (error <= gamma_K sum |x||w|, whatever the order), as does
    the reference: the kernel's sum lies within delta = 2 gamma_K mag of s64, and its fp32 rounding is a float between
    RN(s64 - delta) and RN(s64 + delta) -- one value unless that interval straddles a rounding boundary.  The epilogue
    is monotone in s (scale > 0), so the output lies between the emulations at both ends (ties of the fmaf rounding
    taken down / up); where the interval holds one float and no tie occurs both ends coincide: bit-identical.

    GELU (0.5 y (1 + erff(y c)), c = fp32(1/sqrt 2)) at the fp32 pre-activation y: y c carries 2 u, moving erf by at
    most 2/sqrt(pi) exp(-z^2) 2 u |z| (z = y / sqrt 2, smallest on the interval); erff is within 2 ulps (<= 2^-22 of
    |erf|, CUDA C Programming Guide, single-precision functions); 1 + erf rounds (u); 0.5 y is exact, the product
    rounds (u of the result).  QuickGELU (y / (1 + expf(-1.702f y))): the argument carries 2 u (the fp32 constant and
    the product), expf is within 2 ulps (2^-22 relative): e^a carries eps <= 2 u 1.702 |y| + 2^-22 of itself, which
    moves the quotient by eps e^a / (1 + e^a) = eps sigmoid(-1.702 y) of itself; the sum and the division round (2 u).
    An ambiguous pre-activation adds LIP times the width of its interval."""
    delta = 2 * (K + 2) * 2.0 ** -53 * mag * 1.01 + 2.0 ** -52 * s64.abs()
    lo = _exact_pre((s64 - delta).float(), sc, bi, r, False)
    hi = _exact_pre((s64 + delta).float(), sc, bi, r, True)
    if act == 0:
        return lo, hi
    if act == 1:
        return torch.relu(lo), torch.relu(hi)
    y = lo.double()
    if act == 2:
        z = y / math.sqrt(2.0)
        e = torch.erf(z)
        ref = 0.5 * y * (1 + e)
        d_erf = 2.0 ** -22 * e.abs() + 1.1284 * torch.exp(-(z.abs() * (1 - 4 * U)) ** 2) * 2 * U * z.abs() * (1 + 4 * U)
        d_sum = d_erf + U * ((1 + e).abs() + d_erf)
        bound = 0.5 * y.abs() * d_sum + U * (ref.abs() + 0.5 * y.abs() * d_sum)
    else:
        ref = y * torch.sigmoid(1.702 * y)
        eps = 2 * U * 1.702 * y.abs() + 2.0 ** -22
        bound = ref.abs() * (eps * torch.sigmoid(-1.702 * y) + 2 * U)
    bound = bound * MARGIN + LIP * (hi.double() - lo.double()) + 1e-40
    return ref, bound


def _check_exact(record_property, got: torch.Tensor, s64, mag, K, sc, bi, r, act, what: str) -> None:
    a, b = _exact_ref(s64, mag, K, sc, bi, r, act)
    if act <= 1:
        record_property("ambiguous", int((a != b).sum()))
        outside = (got < a) | (got > b)
        err = torch.maximum(a - got, got - b).clamp_min(0)
        record_property("max_err", float(err.max()))
        assert not bool(outside.any()), f"{what}: {int(outside.sum())} outputs differ from the fp32 emulation, worst " \
                                        f"by {float(err.max()):.3e}"
    else:
        _check(record_property, (got.double() - a).abs(), b, what)


# name: (B, H, W, C, N, kh, kw, stride, pad_h, pad_w, residual, col_off, to_output); the output tensor is at least 8
# columns wider than col_off + N, a multiple of 8 (sentinel columns on both sides when col_off > 0)
EXACT_CASES = {
    "1x1": (3, 10, 10, 64, 64, 1, 1, 1, 0, 0, True, 0, True),          # M = 300: not a multiple of 64
    "3x3_s1": (2, 9, 9, 64, 64, 3, 3, 1, 1, 1, False, 8, False),
    "3x3_s2": (2, 15, 15, 128, 64, 3, 3, 2, 1, 1, True, 16, True),
    "1x7": (2, 17, 17, 64, 96, 1, 7, 1, 0, 3, True, 0, False),
    "7x1": (2, 17, 17, 64, 96, 7, 1, 1, 3, 0, False, 24, True),
    "5x5_c48": (2, 11, 11, 48, 64, 5, 5, 1, 2, 2, True, 8, False),      # C not a multiple of the 16-channel chunk
    "c8_n8": (2, 9, 9, 8, 8, 3, 3, 1, 1, 1, True, 4, True),             # the smallest shape
    "n72": (2, 10, 10, 64, 72, 1, 1, 1, 0, 0, False, 8, True),          # N not a multiple of the 64-column tile
    "m63": (1, 7, 9, 128, 64, 1, 1, 1, 0, 0, True, 0, True),            # one partial 64-row tile
}


def _exact_outputs(m, B: int, t_out: int, rows: int, N: int, col_off: int, ld: int, to_output: bool, out32):
    """Sentinel checks; returns the merged fp32 output values [B, rows, N].  With to_output the planes must be the
    hi / mid / lo split of the fp32 row bit for bit (and sum to it)."""
    planes = m.view(t_out).cpu()
    merged = planes.float().sum(0)
    assert bool((merged[B:] == SENTINEL).all()), "wrote into an unused batch slot"
    assert bool((merged[:B, :, :col_off] == SENTINEL).all()) and bool((merged[:B, :, col_off + N:] == SENTINEL).all()), \
        "wrote outside the op's output columns"
    got = merged[:B, :, col_off:col_off + N]
    if to_output:
        o = out32.view(B, rows, N)
        assert _bits_equal(planes[:, :B, :, col_off:col_off + N], split_planes(o, 3).cpu()), \
            "output planes are not the split of the fp32 output"
        assert torch.equal(got, o)
    return got


@pytest.mark.parametrize("act", [0, 1, 2, 3])
@pytest.mark.parametrize("name", list(EXACT_CASES))
def test_exact_conv_matches_fp32_emulation(name, act, record_property):
    """The float64 path against its documented arithmetic: s = fp32(fp64 sum), fmaf(s, scale, bias), + the three-plane
    residual in fp32, the activation; ReLU / identity bit for bit, erff / expf within their documented ulp bounds
    (the build does not use fast math)."""
    B, H, W, C_, N, kh, kw, stride, ph, pw, with_res, col_off, to_output = EXACT_CASES[name]
    P, Q = (H + 2 * ph - kh) // stride + 1, (W + 2 * pw - kw) // stride + 1
    ld = (col_off + N + 15) // 8 * 8
    g = _gen(list(EXACT_CASES).index(name) * 4 + act)
    m = Micro(B + 1, "exact")
    t_x, t_out = m.tensor(H * W, C_), m.tensor(P * Q, ld)
    t_r = m.tensor(P * Q, N) if with_res else -1
    w = torch.randn(N, C_, kh, kw, device="cuda", generator=g) / (C_ * kh * kw) ** 0.5
    sc, bi = 0.5 + torch.rand(N, device="cuda", generator=g), 0.1 * torch.randn(N, device="cuda", generator=g)
    m.net.conv(t_x, t_out, H, W, C_, w.cpu(), stride=stride, pad=(ph, pw), scale=sc.cpu(), bias=bi.cpu(), residual=t_r,
               act=act, out_col_off=col_off, to_output=to_output)
    m.net.set_output(P * Q * N if to_output else 4)
    x = torch.randn(B + 1, H * W, C_, device="cuda", generator=g)
    x[B:] = FILL
    m.write(t_x, x)
    if with_res:
        r = torch.randn(B + 1, P * Q, N, device="cuda", generator=g)
        r[B:] = FILL
        m.write(t_r, r)
    m.write(t_out, torch.full((B + 1, P * Q, ld), SENTINEL))
    out32 = m.forward(B)
    got = _exact_outputs(m, B, t_out, P * Q, N, col_off, ld, to_output, out32).cuda()
    xm = m.merged(t_x)[:B].cuda().view(B, H, W, C_)
    s64, mag = _conv64(xm, _merged_w(w, 3), stride, (ph, pw))
    rm = m.merged(t_r)[:B].cuda().view(B, P, Q, N) if with_res else None
    _check_exact(record_property, got.reshape(B, P, Q, N), s64, mag, kh * kw * C_, sc, bi, rm, act, name)


@pytest.mark.parametrize("act", [0, 1, 2, 3])
def test_exact_windowed_stem(act, record_property):
    """The space-to-depth stem's 4x1 convolution over the overlapping-window view (window = (16, u): 4 adjacent
    16-channel pixels read as one 64-channel pixel), as in test_s2d_stem_matches_fp64, on the float64 path; the
    reference builds the same view from the merged STEM_S2D planes."""
    from tests.test_net_ops_gpu import MEAN, STD, _images, _stem_params
    crop, B = 64, 3
    gen = torch.Generator().manual_seed(64 + act)
    u8 = _images(gen, B, crop + 32, crop + 32)
    w, sc, bi = _stem_params(gen)
    m = Micro(B + 1, "exact")
    u, oh = (crop + 6) // 2, crop // 2
    t_z, t_stem = m.tensor(u * u, 16), m.tensor(oh * oh, 64)
    nets._input_op(m.net, nets.OP_STEM_S2D, t_z, crop + 32, crop, MEAN, STD)
    ws = nets._stem_s2d_weight(w)
    m.net.conv(t_z, t_stem, u, u - 3, 64, ws, scale=sc, bias=bi, act=act, window=(16, u), to_output=True)
    m.net.set_output(oh * oh * 64)
    m.write(t_stem, torch.full((B + 1, oh * oh, 64), SENTINEL))
    out32 = m.forward(B, u8.cuda())
    got = _exact_outputs(m, B, t_stem, oh * oh, 64, 0, 64, True, out32).cuda()
    z = m.merged(t_z)[:B].cuda().view(B, u, u, 16)
    view = torch.cat([z[:, :, j:j + u - 3] for j in range(4)], 3)                 # [B, u, u - 3, 64]
    s64, mag = _conv64(view, _merged_w(ws, 3), 1, (0, 0))
    _check_exact(record_property, got.reshape(B, oh, oh, 64), s64, mag, 4 * 64, sc.cuda(), bi.cuda(), None, act, "stem")


# ---- C. tensor-core convolution features reachable only through the executor -------------------------------------------
TC_MODES = ["fast", "bf16x3", "parity"]
N_TERMS = {1: 1, 2: 3, 3: 6}
# cross terms the mode drops, relative to sum |x||w| of the merged operands: a bf16 plane's rounding residual is at most
# 2^-8 of the value it splits (half an ulp of 8 significant bits), so two planes drop lo.lo <= 2^-16 (1 + 2^-7), three
# planes mid.lo + lo.mid + lo.lo <= 2^-23 (1 + 2^-7) + 2^-32 < 2^-22
DROPPED = {1: 0.0, 2: 2.0 ** -16 * 1.01, 3: 2.0 ** -22}


def _tc_ref(s, mag, K: int, planes: int, sc, bi, r, act: int, f32: bool = False):
    """(fp64 reference, bound) of a tensor-core convolution output.  Products of bf16 planes are exact in fp32; the
    N_TERMS * K of them are accumulated in fp32 (<= 2^-23 of the running sum of |terms| per add: N_TERMS K 2^-23 of
    mag, with 2 % for the cross terms' own magnitude), the mode drops DROPPED of mag; fmaf and one fp32 add per residual
    plane round once each.  ReLU is 1-Lipschitz; QuickGELU moves by LIP times the pre-activation error plus its own fp32
    evaluation (relative eps sigmoid(-1.702 y) + 2 u, as in _exact_ref).  The store: one plane rounds to nearest bf16
    (half an ulp), two planes keep y - hi - lo <= 2^-16 |y|, three planes and the fp32 output hold the fp32 value."""
    pre = s * sc + bi
    mags = (s * sc).abs() + bi.abs()
    n_add = 1
    if r is not None:
        pre, mags, n_add = pre + r, mags + r.abs(), 1 + planes
    e = sc.abs() * mag * (N_TERMS[planes] * K * 2.0 ** -23 * 1.02 + DROPPED[planes]) + (n_add + 1) * U * mags
    if act == 1:
        ref = torch.relu(pre)
    elif act == 3:
        ref = pre * torch.sigmoid(1.702 * pre)
        eps = 2 * U * 1.702 * (pre.abs() + e) + 2.0 ** -22
        e = LIP * e + (ref.abs() + LIP * e) * (eps * torch.sigmoid(-1.702 * (pre - e)) + 2 * U) * MARGIN
    else:
        ref = pre
    if f32 or planes == 3:
        bound = e
    elif planes == 2:
        bound = e + 2.0 ** -16 * (ref.abs() + e)
    else:
        bound = e + 0.5 * _bf16_ulp(ref.abs() + e)
    return ref, bound + 1e-30


@pytest.mark.parametrize("precision", TC_MODES)
def test_concat_slices_and_fp32_head(precision, record_property):
    """Two convolutions write adjacent column slices of one 240-wide tensor (the Inception concat): a 3x3 (N = 136, act
    3) at columns [80, 216) first, then a 1x1 with residual (N = 72, ReLU) at [8, 80).  Both leave a partial last 64-column
    slab -- in fast mode the TMA-store epilogue must clip it at the op's own columns, so the second op's slab must not
    spill into the first op's columns and the first op's must not reach the sentinel columns [216, 240); the split-bf16
    modes take the direct epilogue.  Plus an fp32 head (1x1, 256 -> 96, QuickGELU, to_output): the direct epilogue in
    every mode, its planes the split of its fp32 row bit for bit."""
    planes = nets.PRECISION_PLANES[precision]
    B, H, W, C_, ld = 3, 12, 12, 64, 240          # M = 432: a partial last m-tile
    hw = H * W
    g = _gen(TC_MODES.index(precision))
    m = Micro(B + 1, precision)
    t_x, t_r, t_cat = m.tensor(hw, C_), m.tensor(hw, 72), m.tensor(hw, ld)
    t_feat, t_head = m.tensor(1, 256), m.tensor(1, 96)
    wb = torch.randn(136, C_, 3, 3, device="cuda", generator=g) / (9 * C_) ** 0.5
    wa = torch.randn(72, C_, 1, 1, device="cuda", generator=g) / C_ ** 0.5
    wh = torch.randn(96, 256, 1, 1, device="cuda", generator=g) / 16
    scb, bib = 0.5 + torch.rand(136, device="cuda", generator=g), 0.1 * torch.randn(136, device="cuda", generator=g)
    sca, bia = 0.5 + torch.rand(72, device="cuda", generator=g), 0.1 * torch.randn(72, device="cuda", generator=g)
    sch, bih = 0.5 + torch.rand(96, device="cuda", generator=g), 0.1 * torch.randn(96, device="cuda", generator=g)
    m.net.conv(t_x, t_cat, H, W, C_, wb.cpu(), pad=(1, 1), scale=scb.cpu(), bias=bib.cpu(), act=3, out_col_off=80)
    m.net.conv(t_x, t_cat, H, W, C_, wa.cpu(), scale=sca.cpu(), bias=bia.cpu(), residual=t_r, act=1, out_col_off=8)
    m.net.conv(t_feat, t_head, 1, 1, 256, wh.cpu(), scale=sch.cpu(), bias=bih.cpu(), act=3, to_output=True)
    m.net.set_output(96)
    x = torch.randn(B + 1, hw, C_, device="cuda", generator=g)
    r = torch.randn(B + 1, hw, 72, device="cuda", generator=g)
    feat = torch.randn(B + 1, 1, 256, device="cuda", generator=g)
    x[B:], r[B:], feat[B:] = FILL, FILL, FILL
    m.write(t_x, x)
    m.write(t_r, r)
    m.write(t_feat, feat)
    m.write(t_cat, torch.full((B + 1, hw, ld), SENTINEL))
    m.write(t_head, torch.full((B + 1, 1, 96), SENTINEL))
    out32 = m.forward(B).cuda()
    cat = m.merged(t_cat).cuda()
    assert bool((cat[B:] == SENTINEL).all()), "a slice wrote into an unused batch slot"
    assert bool((cat[:B, :, :8] == SENTINEL).all()) and bool((cat[:B, :, 216:] == SENTINEL).all()), \
        "a slice wrote past its columns into the sentinel columns"
    xm = m.merged(t_x)[:B].cuda().view(B, H, W, C_)
    s, mag = _conv64(xm, _merged_w(wb, planes), 1, (1, 1))
    ref, bound = _tc_ref(s, mag, 9 * C_, planes, scb.double(), bib.double(), None, 3)
    _check(record_property, (cat[:B, :, 80:216].reshape(B, H, W, 136).double() - ref).abs(), bound, "3x3 slice [80, 216)")
    s, mag = _conv64(xm, _merged_w(wa, planes), 1, (0, 0))
    rm = m.merged(t_r)[:B].cuda().view(B, H, W, 72).double()
    ref, bound = _tc_ref(s, mag, C_, planes, sca.double(), bia.double(), rm, 1)
    _check(record_property, (cat[:B, :, 8:80].reshape(B, H, W, 72).double() - ref).abs(), bound, "1x1 slice [8, 80)")
    # the head
    fm = m.merged(t_feat)[:B].cuda().view(B, 1, 1, 256)
    s, mag = _conv64(fm, _merged_w(wh, planes), 1, (0, 0))
    ref, bound = _tc_ref(s.view(B, 96), mag.view(B, 96), 256, planes, sch.double(), bih.double(), None, 3, f32=True)
    _check(record_property, (out32.double() - ref).abs(), bound, "fp32 head")
    head = m.view(t_head).cpu()
    assert bool((head.float().sum(0)[B:] == SENTINEL).all())
    assert _bits_equal(head[:, :B, 0], split_planes(out32, planes).cpu()), "head planes are not the split of its fp32 row"
