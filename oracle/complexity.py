"""Oracle for the match-complexity statistics (test infrastructure only; see oracle/__init__.py).

  tv_loss            diff_retrieval.py:113-122   the reference's L1 total variation, literally, in torch fp32
  grey_u8            diff_retrieval.py:508       img_as_ubyte(color.rgb2gray(rgb)): skimage is not pinned by the
                                                 reference's env.yaml, so its definition is restated here and is the
                                                 contract: x = c * (1/255); g = (x0*0.2125 + x1*0.7154) + x2*0.0721;
                                                 u = rint(g * 255) (half to even), each step one fp64 rounding
  entropy            diff_retrieval.py:508       sklearn.metrics.cluster.entropy of the grey labels
  jpeg_encode        diff_retrieval.py:513-515   cv2.imencode('.jpg', rgb, [IMWRITE_JPEG_QUALITY, q]) as libjpeg(-turbo)
                                                 writes it: baseline, 4:2:0, islow DCT, Annex K Huffman tables, the
                                                 array read as BGR (channel 2 is red).  h and w multiples of 16.
  complexity_loop    diff_retrieval.py:497-540   entropies, compressions (KiB), totvar and the eight Pearson keys
"""
from __future__ import annotations

import numpy as np

# ---- grey level entropy and total variation ----------------------------------------------------------------------


def grey_u8(rgb: np.ndarray) -> np.ndarray:
    """[..., 3] uint8 -> uint8 grey levels, the fp64 operation order of the contract (no fused multiply-add)."""
    x = rgb.astype(np.float64) * (1.0 / 255)
    g = (x[..., 0] * 0.2125 + x[..., 1] * 0.7154) + x[..., 2] * 0.0721
    return np.clip(np.rint(g * 255), 0, 255).astype(np.uint8)


def entropy(labels: np.ndarray) -> float:
    """sklearn.metrics.cluster.entropy: -sum (p/N)(log p - log N) over the non-empty classes, 0 for one class."""
    labels = np.asarray(labels).ravel()
    if labels.size == 0:
        return 1.0
    pi = np.bincount(labels.astype(np.int64)).astype(np.float64)
    pi = pi[pi > 0]
    if pi.size == 1:
        return 0.0
    pi_sum = np.sum(pi)
    return float(-np.sum((pi / pi_sum) * (np.log(pi) - np.log(pi_sum))))


def tv_loss(img, tv_weight=1e-4):
    """diff_retrieval.py:113-122 (norm='l1') on the CHW float32 tensor `ToTensor()(img) * 255`."""
    w_variance = (img[:, :, :-1] - img[:, :, 1:]).abs().sum()
    h_variance = (img[:, :-1, :] - img[:, 1:, :]).abs().sum()
    return (tv_weight * (h_variance + w_variance)).item()


def tv_sums(rgb: np.ndarray):
    """The two exact integer sums of tv_loss for one HWC uint8 image: (h, w)."""
    a = rgb.astype(np.int64)
    return int(np.abs(a[1:] - a[:-1]).sum()), int(np.abs(a[:, 1:] - a[:, :-1]).sum())


# ---- baseline JPEG, as libjpeg writes it -------------------------------------------------------------------------

STD_LUMA_QT = np.array([
    16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56,
    14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
    49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99], dtype=np.int64)
STD_CHROMA_QT = np.array([
    17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99,
    47, 66, 99, 99, 99, 99, 99, 99] + [99] * 32, dtype=np.int64)

# zig-zag position k -> natural (row-major) index
ZIGZAG = np.array([
    0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21,
    28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61,
    54, 47, 55, 62, 63], dtype=np.int64)


def _runs(*spans):
    out = []
    for s in spans:
        out.extend(s if isinstance(s, list) else [s])
    return out


def _hexrange(lo, hi):
    return list(range(lo, hi + 1))


# Annex K.3 tables: (bits[1..16], values)
DC_LUMA = ([0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0], list(range(12)))
DC_CHROMA = ([0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0], list(range(12)))
AC_LUMA = ([0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d], _runs(
    [0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07,
     0x22, 0x71, 0x14, 0x32, 0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0,
     0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0a, 0x16, 0x17, 0x18, 0x19, 0x1a],
    _hexrange(0x25, 0x2a), _hexrange(0x34, 0x3a), _hexrange(0x43, 0x4a), _hexrange(0x53, 0x5a), _hexrange(0x63, 0x6a),
    _hexrange(0x73, 0x7a), _hexrange(0x83, 0x8a), _hexrange(0x92, 0x9a), _hexrange(0xa2, 0xaa), _hexrange(0xb2, 0xba),
    _hexrange(0xc2, 0xca), _hexrange(0xd2, 0xda), _hexrange(0xe1, 0xea), _hexrange(0xf1, 0xfa)))
AC_CHROMA = ([0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77], _runs(
    [0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71,
     0x13, 0x22, 0x32, 0x81, 0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0,
     0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16, 0x24, 0x34, 0xe1, 0x25, 0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26],
    _hexrange(0x27, 0x2a), _hexrange(0x35, 0x3a), _hexrange(0x43, 0x4a), _hexrange(0x53, 0x5a), _hexrange(0x63, 0x6a),
    _hexrange(0x73, 0x7a), _hexrange(0x82, 0x8a), _hexrange(0x92, 0x9a), _hexrange(0xa2, 0xaa), _hexrange(0xb2, 0xba),
    _hexrange(0xc2, 0xca), _hexrange(0xd2, 0xda), _hexrange(0xe2, 0xea), _hexrange(0xf2, 0xfa)))

HEADER_BYTES = 623


def quant_table(base: np.ndarray, quality: int) -> np.ndarray:
    """jpeg_quality_scaling + jpeg_add_quant_table (force_baseline): natural order, values in [1, 255]."""
    if not 1 <= quality <= 100:
        raise ValueError(f"quality {quality} outside 1..100")
    scale = 5000 // quality if quality < 50 else 200 - 2 * quality
    return np.clip((base * scale + 50) // 100, 1, 255)


def huff_codes(spec):
    """jpeg_make_c_derived_tbl: symbol -> (code, length), canonical codes from the bit counts."""
    bits, vals = spec
    codes, code, p = {}, 0, 0
    for length in range(1, 17):
        for _ in range(bits[length - 1]):
            codes[vals[p]] = (code, length)
            code += 1
            p += 1
        code <<= 1
    return codes


def jpeg_header(h: int, w: int, quality: int) -> bytes:
    """SOI, JFIF APP0, two DQT, SOF0, four DHT, SOS: 623 bytes."""
    out = bytearray(b"\xff\xd8")
    out += b"\xff\xe0\x00\x10JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00"
    for tid, base in enumerate((STD_LUMA_QT, STD_CHROMA_QT)):
        out += bytes([0xFF, 0xDB, 0x00, 0x43, tid]) + bytes(quant_table(base, quality)[ZIGZAG].astype(np.uint8))
    out += bytes([0xFF, 0xC0, 0x00, 0x11, 8, h >> 8, h & 255, w >> 8, w & 255, 3,
                  1, 0x22, 0, 2, 0x11, 1, 3, 0x11, 1])
    for cls_id, (bits, vals) in ((0x00, DC_LUMA), (0x10, AC_LUMA), (0x01, DC_CHROMA), (0x11, AC_CHROMA)):
        n = 2 + 1 + 16 + len(vals)
        out += bytes([0xFF, 0xC4, n >> 8, n & 255, cls_id]) + bytes(bits) + bytes(vals)
    out += bytes([0xFF, 0xDA, 0x00, 0x0C, 3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0])
    assert len(out) == HEADER_BYTES
    return bytes(out)


def _ycc(img: np.ndarray):
    """jccolor.c rgb_ycc_convert, 16-bit fixed point; cv2 hands the array over as BGR."""
    b, g, r = (img[..., c].astype(np.int64) for c in range(3))
    half, off = 1 << 15, 128 << 16
    y = (19595 * r + 38470 * g + 7471 * b + half) >> 16
    cb = (-11059 * r - 21709 * g + 32768 * b + off + half - 1) >> 16
    cr = (32768 * r - 27439 * g - 5329 * b + off + half - 1) >> 16
    return y, cb, cr


def _h2v2(c: np.ndarray) -> np.ndarray:
    """jcsample.c h2v2_downsample: 2x2 sum plus the bias 1, 2, 1, 2, ... along each output row, >> 2."""
    s = c[0::2, 0::2] + c[0::2, 1::2] + c[1::2, 0::2] + c[1::2, 1::2]
    bias = np.where(np.arange(s.shape[1]) % 2 == 0, 1, 2)
    return (s + bias[None, :]) >> 2


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def _fdct_pass(d, final: bool):
    """One pass of jfdctint.c jpeg_fdct_islow over the last axis (CONST_BITS 13, PASS1_BITS 2)."""
    cb, pb = 13, 2
    t0, t7 = d[..., 0] + d[..., 7], d[..., 0] - d[..., 7]
    t1, t6 = d[..., 1] + d[..., 6], d[..., 1] - d[..., 6]
    t2, t5 = d[..., 2] + d[..., 5], d[..., 2] - d[..., 5]
    t3, t4 = d[..., 3] + d[..., 4], d[..., 3] - d[..., 4]
    t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
    out = np.empty_like(d)
    sh = cb + pb if final else cb - pb
    if final:
        out[..., 0] = _descale(t10 + t11, pb)
        out[..., 4] = _descale(t10 - t11, pb)
    else:
        out[..., 0] = (t10 + t11) << pb
        out[..., 4] = (t10 - t11) << pb
    z1 = (t12 + t13) * 4433
    out[..., 2] = _descale(z1 + t13 * 6270, sh)
    out[..., 6] = _descale(z1 - t12 * 15137, sh)
    z1, z2, z3, z4 = t4 + t7, t5 + t6, t4 + t6, t5 + t7
    z5 = (z3 + z4) * 9633
    t4, t5, t6, t7 = t4 * 2446, t5 * 16819, t6 * 25172, t7 * 12299
    z1, z2, z3, z4 = z1 * -7373, z2 * -20995, z3 * -16069 + z5, z4 * -3196 + z5
    out[..., 7] = _descale(t4 + z1 + z3, sh)
    out[..., 5] = _descale(t5 + z2 + z4, sh)
    out[..., 3] = _descale(t6 + z2 + z3, sh)
    out[..., 1] = _descale(t7 + z1 + z4, sh)
    return out


def _blocks(plane: np.ndarray) -> np.ndarray:
    """[H, W] -> [H/8, W/8, 8, 8]"""
    h, w = plane.shape
    return plane.reshape(h // 8, 8, w // 8, 8).transpose(0, 2, 1, 3)


def _quantize(coef: np.ndarray, qt: np.ndarray) -> np.ndarray:
    """jcdctmgr.c: divisor = 8 * quantval, round to nearest with the sign handled as DIVIDE_BY."""
    q = (8 * qt).reshape(8, 8)
    a = np.abs(coef)
    return np.sign(coef) * ((a + (q >> 1)) // q)


def quantized_blocks(img: np.ndarray, quality: int):
    """[H, W, 3] uint8 -> (Y [H/8, W/8, 64], Cb, Cr [H/16, W/16, 64]) quantised coefficients in zig-zag order."""
    h, w = img.shape[:2]
    if h % 16 or w % 16 or not (16 <= h <= 4096 and 16 <= w <= 4096):
        raise ValueError(f"{h}x{w}: height and width must be multiples of 16 in 16..4096")
    y, cb, cr = _ycc(img)
    out = []
    for plane, base in ((y, STD_LUMA_QT), (_h2v2(cb), STD_CHROMA_QT), (_h2v2(cr), STD_CHROMA_QT)):
        blk = _blocks(plane - 128)
        coef = _fdct_pass(_fdct_pass(blk, False).swapaxes(-1, -2), True).swapaxes(-1, -2)
        qc = _quantize(coef, quant_table(base, quality))
        out.append(qc.reshape(*qc.shape[:2], 64)[..., ZIGZAG])
    return out


def _nbits(v: int) -> int:
    return int(abs(v)).bit_length()


def jpeg_encode(img: np.ndarray, quality: int = 90) -> bytes:
    """The bytes cv2.imencode('.jpg', img, [IMWRITE_JPEG_QUALITY, quality]) returns, for h, w multiples of 16."""
    img = np.ascontiguousarray(img, dtype=np.uint8)
    h, w = img.shape[:2]
    yq, cbq, crq = quantized_blocks(img, quality)
    tabs = [(huff_codes(DC_LUMA), huff_codes(AC_LUMA)), (huff_codes(DC_CHROMA), huff_codes(AC_CHROMA))]
    bits = []

    def put(code, length):
        if length:
            bits.append(format(code & ((1 << length) - 1), f"0{length}b"))

    def block(coefs, comp, pred):
        dc_tab, ac_tab = tabs[min(comp, 1)]
        diff = int(coefs[0]) - pred
        nb = _nbits(diff)
        put(*dc_tab[nb])
        put(diff if diff >= 0 else diff - 1, nb)
        run = 0
        for k in range(1, 64):
            v = int(coefs[k])
            if v == 0:
                run += 1
                continue
            while run > 15:
                put(*ac_tab[0xF0])
                run -= 16
            nb = _nbits(v)
            put(*ac_tab[(run << 4) + nb])
            put(v if v >= 0 else v - 1, nb)
            run = 0
        if run > 0:
            put(*ac_tab[0x00])
        return int(coefs[0])

    pred = [0, 0, 0]
    for my in range(h // 16):
        for mx in range(w // 16):
            for by, bx in ((0, 0), (0, 1), (1, 0), (1, 1)):
                pred[0] = block(yq[2 * my + by, 2 * mx + bx], 0, pred[0])
            pred[1] = block(cbq[my, mx], 1, pred[1])
            pred[2] = block(crq[my, mx], 2, pred[2])
    s = "".join(bits)
    s += "1" * (-len(s) % 8)
    scan = int(s, 2).to_bytes(len(s) // 8, "big") if s else b""
    return jpeg_header(h, w, quality) + scan.replace(b"\xff", b"\xff\x00") + b"\xff\xd9"


# ---- the images of tests/golden/jpeg_cv2.npz (rebuilt from seeds where cv2 is absent) ------------------------------

GOLDEN_QUALITIES = (1, 10, 50, 75, 90, 95, 100)
GOLDEN_SIZES = ((16, 16), (32, 48), (224, 224), (512, 256))


def golden_images(h: int, w: int):
    """[(kind, uint8 [h, w, 3])]: uniform noise (the largest Huffman categories at q = 100), the eight flat images with
    0 or 255 on each channel, gradients, checkerboards and a single hot pixel on black."""
    rng = np.random.default_rng(1000 * h + w)
    out = [("noise", rng.integers(0, 256, (h, w, 3), dtype=np.uint8))]
    for c in range(8):
        out.append((f"flat{c}", np.broadcast_to(np.array([255 * (c >> i & 1) for i in range(3)], np.uint8),
                                                (h, w, 3)).copy()))
    yy, xx = np.mgrid[0:h, 0:w]
    out.append(("gradient", np.stack([xx * 255 // max(w - 1, 1), yy * 255 // max(h - 1, 1),
                                      (xx + yy) % 256], -1).astype(np.uint8)))
    out.append(("checker1", np.repeat((((xx + yy) & 1) * 255).astype(np.uint8)[..., None], 3, -1)))
    out.append(("checker8", np.stack([((xx // 8 + yy // 8) & 1) * 255, ((xx // 8 + yy // 8) & 1) * 200,
                                      255 - ((xx // 8 + yy // 8) & 1) * 255], -1).astype(np.uint8)))
    hot = np.zeros((h, w, 3), np.uint8)
    hot[rng.integers(0, h), rng.integers(0, w)] = (255, 255, 255)
    out.append(("hotpixel", hot))
    return out


# ---- the reference loop ----------------------------------------------------------------------------------------------

CORRELATION_KEYS = ("cc_ent", "pval_ent", "cc_comp", "pval_comp", "cc_tvl", "pval_tvl", "cc_mixed", "pval_mixed")


def correlations(entropies, compressions, totvar, dbsims) -> dict:
    """diff_retrieval.py:525-529: Pearson r and p of each quantity, and of entropy * sqrt(size), with the top-1 sim."""
    from scipy import stats
    e, c, t, s = (np.asarray(a, dtype=np.float64) for a in (entropies, compressions, totvar, dbsims))
    out = {}
    for name, x in (("ent", e), ("comp", c), ("tvl", t), ("mixed", e * c ** 0.5)):
        if len(s) < 2 or np.ptp(x) == 0 or np.ptp(s) == 0:
            r, p = float("nan"), float("nan")
        else:
            r, p = stats.pearsonr(x, s)
        out[f"cc_{name}"], out[f"pval_{name}"] = float(r), float(p)
    return out


def complexity_loop(images_u8: np.ndarray, dbsims: np.ndarray, quality: int = 90) -> dict:
    """diff_retrieval.py:497-529 on the matched images [Q, H, W, 3] uint8 (one per generation)."""
    import torch
    ents, crs, tvls = [], [], []
    for rgb in images_u8:
        ents.append(entropy(grey_u8(rgb)))
        crs.append(len(jpeg_encode(rgb, quality)) / 1024)
        torchim = torch.from_numpy(np.ascontiguousarray(rgb)).permute(2, 0, 1).float().div(255) * 255
        tvls.append(tv_loss(torchim))
    out = {"entropies": np.array(ents), "compressions": np.array(crs), "totvar": np.array(tvls),
           "dbsims": np.asarray(dbsims)}
    out.update(correlations(out["entropies"], out["compressions"], out["totvar"], out["dbsims"]))
    return out
