"""Operands that drive the bf16 error of the fused similarity sweep to its bound (test infrastructure only).

dcr_sim_topk and dcr_sim_range both rank on a bf16 tensor-core score and trust one number per query, the `eps` of
row_bound (dcr_b200/csrc/sim_sweep.cuh), to bound |approximate score - exact centred score|.  Random descriptors keep that
error far below the bound.  The instances built here reach it, and they are built so that a CPU restatement of stage 1
reproduces the kernel's operands bit for bit:

- Few significant bits.  Gallery elements are 1 + x*2^-11 for a small integer x, or +-1; query elements are small
  multiples of 1/2.  Every fp32 partial sum of col_sum_kernel and of the tensor-core accumulation, and every fp64 dot
  product, is then exact: the centres, the approximate scores and the exact scores are known without rounding, and
  equal exact scores are real ties.
- Known centres.  The gallery comes in exact +- pairs, so its centre mu is 0.  The queries come in pairs c + w, c - w:
  with c = 0 the query centre is 0 and centring stays off; with c = 8 p (p = +1 on the first half of the dimensions,
  -1 on the second) the centre is exactly c, q - nu = +-w, and centre_decision_kernel switches centring on.
- The target A (every element 1 + 7*2^-11, just below the rounding midpoint 1 + 2^-8, so it rounds down to 1) loses
  ||w|| ||A - bf16(A)|| of its score to bf16 rounding: the Cauchy-Schwarz bound that eps is written for, attained.  It
  is the gallery's largest-residual row.
- The competitors B have a elements per half at 1 + 9*2^-11 (rounds up to 1 + 2^-7) and the rest at 1 - 3*2^-11 (rounds
  up to 1).  With 24 a < 10 d their exact score lies below A's, by as little as a few 2^-11 quanta, while their bf16
  score lies up to almost 2 eps above A's.  B rows (or the tie twin) are the gallery's largest-norm rows.
- Fillers are +-1 rows that score far below A for both queries.

For the query c - w the rows -A and -B play the roles of A and B, so both queries of a pair meet the same instance.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

U = 2.0 ** -11          # the gallery's quantum
SEG = 64                # the target and its competitors sit in the first 64 columns of a 128-row tile: one segment
                        # whether the fused sweep runs one epilogue set (128 columns) or two (64 each)
KP0 = {1: 4, 2: 4, 10: 12, 16: 32}   # candidates the first pass keeps per segment, by k (make_plan)
KP1 = 32                             # candidates of the second-chance pass


def bf16(x: np.ndarray) -> np.ndarray:
    """Round-to-nearest-even fp32 -> bf16, back in fp32, as __float2bfloat16_rn (finite values): add half a bf16 ulp
    less one, plus the kept lsb, to the bits and cut the low 16."""
    b = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    assert np.isfinite(x).all()
    return ((b + np.uint32(0x7FFF) + ((b >> 16) & np.uint32(1))) & np.uint32(0xFFFF0000)).view(np.float32)


def _levels(d: int):
    """Counts a of 1 + 9*2^-11 elements per half of a B row: exact score below A's (24 a < 10 d), bf16 score above A's
    fp32 score (32 a > 7 d).  Highest first (the closest to A, the largest bf16 lead)."""
    a_max = -(-10 * d // 24) - 1
    a_min = 7 * d // 32 + 1
    return list(range(a_max, a_min - 1, -1))


def _b_row(d: int, a: int, rng, bump: int = 0) -> np.ndarray:
    """x offsets of a B row: per half a entries 9, the rest -3; `bump` (even, < 24) is added to each half by raising
    -3 entries to 0 (+3) and one to -2 or -1, which still round up to 1."""
    x = np.empty(d, dtype=np.int64)
    h = d // 2
    for lo in (0, h):
        part = np.full(h, -3, dtype=np.int64)
        part[rng.permutation(h)[:a]] = 9
        rest = np.nonzero(part == -3)[0]
        b, j = bump, 0
        while b > 0:
            step = min(3, b)
            part[rest[j]] += step
            b -= step
            j += 1
        x[lo:lo + h] = part
    return x


def _filler(d: int, rng) -> np.ndarray:
    """+-1 row with d/4 + u_h ones in each half (u_h in -1..1, |u_1 - u_2| <= 1): sum 2(u_1 + u_2), p-sum 2(u_1 - u_2)."""
    h = d // 2
    u1 = int(rng.integers(-1, 2))
    u2 = int(np.clip(u1 + rng.integers(-1, 2), -1, 1))
    f = np.empty(d, dtype=np.float32)
    for lo, u in ((0, u1), (h, u2)):
        part = -np.ones(h, dtype=np.float32)
        part[rng.permutation(h)[:h // 2 + u]] = 1.0
        f[lo:lo + h] = part
    return f


@dataclass
class Case:
    """One instance.  Query i's target is target[i], its competitors comps[i], its tie twin twin[i] (-1: none)."""
    q: np.ndarray
    g: np.ndarray
    centred: bool
    target: np.ndarray
    comps: list
    twin: np.ndarray
    info: dict = field(default_factory=dict)


def build(d: int, n_b: int, *, centred: bool, shared: bool = False, tie: bool = False, tiles: int = 2,
          scales=(1.0,), seed: int = 0) -> Case:
    """The gallery X ++ (-X), X of 128 * tiles rows.  A sits in tile 0 (position 2 when it has competitors before it);
    the n_b competitors fill the rest of tile 0's first 64 rows, or of tile 1's when `shared` (A alone in its
    segment).  With `tie`, a twin row right after A has A's exact score and a bf16 score like the best B's.  Queries:
    for every scale s, the pair c + s w, c - s w."""
    assert d % 4 == 0 and d >= 64
    rng = np.random.default_rng(seed + 7919 * d + 31 * n_b + 3 * int(centred) + 5 * int(shared) + 11 * int(tie))
    n_x = 128 * tiles
    X = np.stack([_filler(d, rng) for _ in range(n_x)])
    lv = _levels(d)
    a_row = 1.0 + 7 * U
    b_rows = [(1.0 + _b_row(d, lv[j % len(lv)], rng) * U) for j in range(n_b)]
    pos_a = 0 if shared else min(2, n_b)
    X[pos_a] = a_row
    if shared:
        assert tiles >= 2 and n_b <= SEG
        b_pos = list(range(128, 128 + n_b))
    else:
        free = [p for p in range(SEG) if p != pos_a and not (tie and p == pos_a + 1)]
        assert n_b <= len(free)
        b_pos = free[:n_b]
    for p, r in zip(b_pos, b_rows):
        X[p] = r
    twin = -1
    if tie:
        a = lv[0]
        bump = 5 * d - 12 * a                       # per half: reach A's half sum 3.5 d exactly
        assert 0 < bump < 24 and bump % 2 == 0
        twin = pos_a + 1
        X[twin] = 1.0 + _b_row(d, a, rng, bump) * U
    X = X.astype(np.float32)
    g = np.concatenate([X, -X]).astype(np.float32)
    w = np.ones(d, dtype=np.float32)
    p = np.concatenate([np.ones(d // 2), -np.ones(d // 2)]).astype(np.float32)
    c = 8.0 * p if centred else np.zeros(d, dtype=np.float32)
    qs, target, comps, twins = [], [], [], []
    for s in scales:
        for sign in (1, -1):
            qs.append(c + sign * s * w)
            off = 0 if sign > 0 else n_x
            target.append(off + pos_a)
            comps.append(np.array(b_pos, dtype=np.int64) + off)
            twins.append(off + twin if tie else -1)
    q = np.stack(qs).astype(np.float32)
    return Case(q=q, g=g, centred=centred, target=np.array(target, dtype=np.int64), comps=comps,
                twin=np.array(twins, dtype=np.int64), info=dict(d=d, n_b=n_b, shared=shared, tie=tie))


# ---------------------------------------------------------------------------------------------------------------
# CPU restatement of stage 1 and of row_bound


def centre(x: np.ndarray):
    """col_sum_kernel + col_mean_finish_kernel (every partial sum exact here, so the order does not matter) and
    centre_decision_kernel: (mean as fp32, centring flag)."""
    x64 = x.astype(np.float64)
    n = x.shape[0]
    sums, sq = x64.sum(axis=0), (x64 * x64).sum(axis=0)
    m2 = float(np.sum(sq / n))
    nu2 = float(np.sum((sums / n) ** 2))
    return (sums / n).astype(np.float32), (m2 - nu2 < m2 / 16.0)


@dataclass
class Operands:
    mu: np.ndarray
    nu: np.ndarray          # the query centre in use (zeros when centring is off)
    flag: bool
    qh: np.ndarray          # bf16(q - nu), fp32 values
    gh: np.ndarray          # bf16(g - mu)
    qv: np.ndarray          # fp32(q - nu)
    gv: np.ndarray          # fp32(g - mu)
    qnh: np.ndarray         # to_bf16_rows_kernel's norms of the query rows
    qnr: np.ndarray
    qnx: np.ndarray
    g_norm: np.float32      # gmax[0], gmax[1]
    g_res: np.float32
    bias: np.ndarray        # fp32 nu.(g - mu) per gallery row (zeros when centring is off)


def _norm(v: np.ndarray) -> np.ndarray:
    """sqrtf of the row's sum of squares times 1.0001f, as to_bf16_rows_kernel stores it (the kernel's fp32 summation
    order is not restated: the sums agree to an ulp or two)."""
    s = np.sum(v.astype(np.float64) ** 2, axis=1).astype(np.float32)
    return (np.sqrt(s) * np.float32(1.0001)).astype(np.float32)


def operands(q: np.ndarray, g: np.ndarray) -> Operands:
    mu, _ = centre(g)
    nu, flag = centre(q)
    if not flag:
        nu = np.zeros_like(nu)
    qv = (q - nu[None, :]).astype(np.float32)
    gv = (g - mu[None, :]).astype(np.float32)
    qh, gh = bf16(qv), bf16(gv)
    bias = (gv.astype(np.float64) @ nu.astype(np.float64)).astype(np.float32) if flag else np.zeros(g.shape[0], np.float32)
    return Operands(mu=mu, nu=nu, flag=flag, qh=qh, gh=gh, qv=qv, gv=gv, qnh=_norm(qh), qnr=_norm(qv - qh),
                    qnx=_norm(qv), g_norm=_norm(gv).max(), g_res=_norm(gv - gh).max(), bias=bias)


def d_pad(d: int) -> int:
    return -(-d // 64) * 64


def eps(op: Operands, d: int) -> np.ndarray:
    """row_bound's eps per query row, in the kernel's fp32 order of operations."""
    f = np.float32
    qh, qr, qx = op.qnh, op.qnr, op.qnx
    e = f(1.001) * (qh * op.g_res + qr * op.g_norm) + f(d_pad(d)) * f(2.4e-7) * qh * (op.g_norm + op.g_res) + f(1e-30)
    nun = f(np.sqrt(np.float32(np.sum(op.nu.astype(np.float64) ** 2))) * f(1.001)) if op.flag else f(0)
    return (e + f(3e-7) * (qx + nun) * op.g_norm).astype(np.float32)


def bf16_terms(op: Operands) -> np.ndarray:
    """The bf16 part of eps, qh g_res + qr g_norm: what a row's bf16 rounding alone can cost."""
    return (op.qnh * op.g_res + op.qnr * op.g_norm).astype(np.float32)


def approx(op: Operands) -> np.ndarray:
    """The fused sweep's score: the tensor-core product of the bf16 operands (exact here) plus the column offset, one
    fp32 addition."""
    acc = (op.qh.astype(np.float64) @ op.gh.astype(np.float64).T).astype(np.float32)
    return (acc + op.bias[None, :]).astype(np.float32)


def exact(q: np.ndarray, g: np.ndarray) -> np.ndarray:
    return q.astype(np.float64) @ g.astype(np.float64).T


def realized(case: Case, op: Operands) -> np.ndarray:
    """Per query: how far the target's approximate score lies below its exact centred score q.(g - mu)."""
    ex_c = case.q.astype(np.float64) @ op.gv.astype(np.float64).T
    a = approx(op).astype(np.float64)
    rows = np.arange(case.q.shape[0])
    return ex_c[rows, case.target] - a[rows, case.target]


def as_integers(x: np.ndarray, quantum: float) -> np.ndarray:
    """x / quantum as int64, asserting that every entry is an integer multiple of the quantum."""
    y = x.astype(np.float64) / quantum
    assert np.array_equal(y, np.round(y)), "entries off the quantum grid"
    return y.astype(np.int64)


# ---------------------------------------------------------------------------------------------------------------
# The instances the tests run

DIMS = (64, 512, 516, 1024, 4096)   # resident query tile, padded d_pad, streamed query tile

# (name, k, competitors, competitors in another segment, tie twin, stage that must decide both queries)
#   first:  fewer than kp - 1 competitors share A's segment: A is a candidate of the first pass and the re-score puts it
#           above the competitors the bf16 scores rank first
#   second: at least kp of them (or, shared, in another segment whose threshold reaches A's unit): the first pass drops
#           A, the certificate fails, the second-chance pass keeps 32 per segment and finds it
#   brute:  more than 32: the brute-force path (k = 16 has no second pass)
TOPK_CASES = [
    ("k1_first", 1, 2, False, False, "first"),
    ("k2_first", 2, 2, False, False, "first"),
    ("k10_first", 10, 10, False, False, "first"),
    ("k16_first", 16, 20, False, False, "first"),
    ("k1_second", 1, 8, False, False, "second"),
    ("k2_second", 2, 30, False, False, "second"),
    ("k10_second", 10, 20, False, False, "second"),
    ("k1_brute", 1, 40, False, False, "brute"),
    ("k10_brute", 10, 40, False, False, "brute"),
    ("k16_brute", 16, 40, False, False, "brute"),
    ("k1_shared", 1, 8, True, False, "second"),
    ("k10_shared", 10, 20, True, False, "second"),
    ("k1_tie", 1, 1, False, True, "first"),
    ("k2_tie", 2, 1, False, True, "first"),
    ("k10_tie", 10, 9, False, True, "first"),
]


def topk_case(name: str, d: int, centred: bool, **build_kw) -> Case:
    _, k, n_b, shared, tie, _ = next(c for c in TOPK_CASES if c[0] == name)
    return build(d, n_b, centred=centred, shared=shared, tie=tie, **build_kw)


def stage_of(name: str) -> str:
    return next(c for c in TOPK_CASES if c[0] == name)[5]


# 258 queries, pairs at scales 1, 2, 1/2: query tiles of 128 + 128 + 2.  A power of two scales every score, norm and eps
# exactly, so every query is decided by the stage its instance is built for.  Query r has scale MANY_SCALES[r // 2].
MANY_SCALES = (1.0, 2.0, 0.5) * 43


# ---------------------------------------------------------------------------------------------------------------
# The split score: an instance in one descriptor part
#
# sim_topk_split and sim_range_split rank on the maximum over the parts of per-part bf16 scores and trust split_row_bound
# (sim_sweep.cuh): the largest over the parts of row_bound's expression, from each part's own query norms
# (q_norm_*[qrow * n_parts + c]) and gallery maxima (g_max[2c], g_max[2c + 1]).  The instances below put a build()
# instance (uncentred, its d becoming the part length p) into one part of n_parts:
#
# - quiet: every other part of the query is zero and every other part of the gallery holds tiny values x*2^-11
#   (|x| <= 3, bf16-exact).  Those parts score exactly 0 and contribute nothing to eps, so eps comes from the instance
#   part alone: a bound read from another part's norms or gallery maxima, or one that never visits the instance part,
#   collapses below A's realized error and lets the bf16 order through.
# - cross: A (and its twin) reach their scores in part `part`, the competitors in part `other`; the query holds +-w in
#   both, and a row's part that does not hold its instance holds a +-1 filler.  The running maximum over the parts then
#   decides every pair from a different part for A than for its competitors.

SPLIT_SHAPES = ((2, 64), (4, 516), (3, 1024), (40, 64), (197, 64))   # (n_parts, p); 516 pads to 576
RANGE_SPLIT_SHAPES = SPLIT_SHAPES + ((2, 256), (4, 64))              # d_pad <= 512: resident query tile


def split_placements(n_parts: int):
    """(layout, part, other) of every placement a shape is tested at.  quiet: the first part, the second, the last, and
    33 (the second lane round of split_row_bound's part loop) when there is one; cross: A in the first part and the
    competitors in the last, the reverse, and A in part 33 against competitors in part 1."""
    quiet = sorted({0, 1, n_parts - 1} | ({33} if n_parts > 33 else set()))
    cross = [(0, n_parts - 1), (n_parts - 1, 0)] + ([(33, 1)] if n_parts > 33 else [])
    return [("quiet", c, -1) for c in quiet] + [("cross", c, o) for c, o in cross]


def _mirror_set(g: np.ndarray, cols: slice, rows, rng):
    """Fresh +-1 fillers in part `cols` of rows `rows` of X and, negated, of their mirrors in -X."""
    n_x = g.shape[0] // 2
    for r in sorted({int(r) % n_x for r in rows}):
        f = _filler(cols.stop - cols.start, rng)
        g[r, cols], g[r + n_x, cols] = f, -f


def split_embed(case: Case, n_parts: int, part: int, layout: str = "quiet", other: int = -1, seed: int = 0) -> Case:
    """`case` (uncentred, of dimension p) put into part `part` of n_parts; see above for the layouts."""
    assert not case.centred and 0 <= part < n_parts
    nq, p = case.q.shape
    ng = case.g.shape[0]
    rng = np.random.default_rng(seed + 1009 * n_parts + 17 * part)
    q = np.zeros((nq, n_parts * p), np.float32)
    g = (rng.integers(-3, 4, size=(ng, n_parts * p)) * U).astype(np.float32)
    at = slice(part * p, (part + 1) * p)
    q[:, at] = case.q
    g[:, at] = case.g
    if layout == "cross":
        assert 0 <= other < n_parts and other != part
        to = slice(other * p, (other + 1) * p)
        q[:, to] = case.q
        g[:, to] = case.g
        _mirror_set(g, at, np.concatenate(case.comps), rng)                                    # B scores in `other` only
        _mirror_set(g, to, np.concatenate([case.target, case.twin[case.twin >= 0]]), rng)     # A, twin in `part` only
    else:
        assert layout == "quiet"
    return Case(q=q, g=g, centred=False, target=case.target, comps=case.comps, twin=case.twin,
                info=dict(case.info, n_parts=n_parts, p=p, part=part, layout=layout, other=other))


def split_case(name: str, p: int, n_parts: int, part: int, layout: str = "quiet", other: int = -1, **build_kw) -> Case:
    """A TOPK_CASES instance (by name), or with name "range" the threshold-search instance build(p, 20, **build_kw)
    (tie=, scales=), in part `part` of n_parts."""
    base = build(p, 20, centred=False, **build_kw) if name == "range" else topk_case(name, p, False, **build_kw)
    return split_embed(base, n_parts, part, layout, other)


def second_half(case: Case) -> Case:
    """The competitors moved from columns 0-63 of their 128-row tile to columns 64-127 (swapped with fillers), in X and
    -X alike: the two column halves of a tile are swept by different consumer warpgroups."""
    ng = case.g.shape[0]
    n_x = ng // 2
    perm = np.arange(ng)
    for b in sorted({int(b) % n_x for b in np.concatenate(case.comps)}):
        assert b % 128 < 64
        for off in (0, n_x):
            perm[off + b], perm[off + b + 64] = off + b + 64, off + b
    inv = np.argsort(perm)   # new position of old row j: inv[j]
    return Case(q=case.q, g=case.g[perm], centred=False, target=inv[case.target], comps=[inv[c] for c in case.comps],
                twin=np.where(case.twin >= 0, inv[np.maximum(case.twin, 0)], -1), info=dict(case.info, second_half=True))


@dataclass
class SplitOperands:
    qh: np.ndarray          # bf16(q), fp32 values [nq, d]
    gh: np.ndarray          # bf16(g)
    qnh: np.ndarray         # to_bf16_parts_kernel's norms of the query parts [nq, n_parts]
    qnr: np.ndarray
    qnx: np.ndarray
    g_norm: np.ndarray      # gmax[2c], gmax[2c + 1]: the gallery maxima of every part [n_parts]
    g_res: np.ndarray


def _part_norm(v: np.ndarray, n_parts: int) -> np.ndarray:
    """_norm of every part of every row: [n, n_parts]."""
    v3 = v.astype(np.float64).reshape(v.shape[0], n_parts, -1)
    s = np.sum(v3 ** 2, axis=2).astype(np.float32)
    return (np.sqrt(s) * np.float32(1.0001)).astype(np.float32)


def split_operands(q: np.ndarray, g: np.ndarray, n_parts: int) -> SplitOperands:
    """to_bf16_parts_kernel per part: no centring, bf16 RNE, norms x 1.0001f, gallery maxima per part (the zero padding
    of a part to p_pad adds nothing to any of them)."""
    qh, gh = bf16(q), bf16(g)
    return SplitOperands(qh=qh, gh=gh, qnh=_part_norm(qh, n_parts), qnr=_part_norm(q - qh, n_parts),
                         qnx=_part_norm(q, n_parts), g_norm=_part_norm(g, n_parts).max(axis=0),
                         g_res=_part_norm(g - gh, n_parts).max(axis=0))


def split_part_eps(op: SplitOperands, p_pad: int) -> np.ndarray:
    """split_row_bound's term of every part, in the kernel's fp32 order of operations: [nq, n_parts]."""
    f = np.float32
    qh, qr, qx, gn, gr = op.qnh, op.qnr, op.qnx, op.g_norm[None, :], op.g_res[None, :]
    e = f(1.001) * (qh * gr + qr * gn) + f(p_pad) * f(2.4e-7) * qh * (gn + gr) + f(3e-7) * qx * gn + f(1e-30)
    return e.astype(np.float32)


def split_eps(op: SplitOperands, p_pad: int) -> np.ndarray:
    """split_row_bound's eps per query row: the largest part term."""
    return split_part_eps(op, p_pad).max(axis=1)


def split_bf16_terms(op: SplitOperands) -> np.ndarray:
    """The bf16 part of every part's term, qh g_res + qr g_norm: [nq, n_parts]."""
    return (op.qnh * op.g_res[None, :] + op.qnr * op.g_norm[None, :]).astype(np.float32)


def part_products(q: np.ndarray, g: np.ndarray, n_parts: int) -> np.ndarray:
    """The fp64 dot products of every part: [n_parts, nq, ng]."""
    qp = q.astype(np.float64).reshape(q.shape[0], n_parts, -1).transpose(1, 0, 2)
    gp = g.astype(np.float64).reshape(g.shape[0], n_parts, -1).transpose(1, 2, 0)
    return np.matmul(qp, gp)


def split_approx(op: SplitOperands, n_parts: int) -> np.ndarray:
    """The fused sweep's split score: per part the tensor-core product of the bf16 operands (exact here) as fp32, then
    the maximum over the parts."""
    return part_products(op.qh, op.gh, n_parts).astype(np.float32).max(axis=0)


def split_exact(q: np.ndarray, g: np.ndarray, n_parts: int) -> np.ndarray:
    """The fp64 split score: the maximum over the parts of the fp64 part dot products."""
    return part_products(q, g, n_parts).max(axis=0)


def split_realized(case: Case, op: SplitOperands) -> np.ndarray:
    """Per query: how far the target's approximate split score lies below its exact split score."""
    c = case.info["n_parts"]
    rows = np.arange(case.q.shape[0])
    return split_exact(case.q, case.g, c)[rows, case.target] - split_approx(op, c)[rows, case.target].astype(np.float64)


# ---------------------------------------------------------------------------------------------------------------
# Mixed stages in one call (the aligned split score)
#
# The first, second and brute-force instances of one k in three parts of one gallery (build() always gives 512 rows):
# query r is of type r % 3 and holds instance (r % 3)'s query r in that instance's part, zeros elsewhere.  Its zero parts
# score 0 and give terms of 1e-30, so its candidates, its eps and its stage are those of its own instance; the flagged
# queries of a pass are then no prefix of the batch and span every query tile.

MIXED = {1: ("k1_first", "k1_second", "k1_brute"), 10: ("k10_first", "k10_second", "k10_brute")}


def mixed_case(k: int, p: int, n_parts: int, parts, scales=MANY_SCALES, seed: int = 0) -> Case:
    assert len(set(parts)) == 3 and all(0 <= c < n_parts for c in parts)
    cases = [topk_case(name, p, False, scales=scales) for name in MIXED[k]]
    nq, ng = cases[0].q.shape[0], cases[0].g.shape[0]
    rng = np.random.default_rng(seed + 1009 * n_parts + 17 * parts[0] + 5 * parts[1] + parts[2])
    q = np.zeros((nq, n_parts * p), np.float32)
    g = (rng.integers(-3, 4, size=(ng, n_parts * p)) * U).astype(np.float32)
    for case, c in zip(cases, parts):
        assert case.g.shape[0] == ng
        g[:, c * p:(c + 1) * p] = case.g
    types = np.arange(nq) % 3
    for r in range(nq):
        c = parts[types[r]]
        q[r, c * p:(c + 1) * p] = cases[types[r]].q[r]
    return Case(q=q, g=g, centred=False, target=np.array([cases[t].target[r] for r, t in enumerate(types)]),
                comps=[cases[t].comps[r] for r, t in enumerate(types)], twin=np.full(nq, -1, np.int64),
                info=dict(d=p, n_parts=n_parts, p=p, parts=tuple(parts), types=types, layout="mixed",
                          stages=[stage_of(MIXED[k][t]) for t in types]))


def nan_rows(nq: int) -> np.ndarray:
    """Every 7th query, and the last row of the first query tile, the first of the second and the last of the batch."""
    return np.array(sorted(set(range(0, nq, 7)) | {r for r in (127, 128, nq - 1) if 0 <= r < nq}), dtype=np.int64)


def with_nan(case: Case, rows, part: int) -> Case:
    """A NaN in the first value of query part `part` (a zero part of these queries) of every row in `rows`.  Its part
    norms are NaN, so eps is NaN and the certificate fails in both passes: such a query is answered by the brute-force
    path.  The pairs of the NaN part are ignored by the score, so the answer is the query's answer without it."""
    p = case.info["p"]
    q = case.q.copy()
    assert not q[rows, part * p:(part + 1) * p].any()
    q[rows, part * p] = np.nan
    return Case(q=q, g=case.g, centred=False, target=case.target, comps=case.comps, twin=case.twin,
                info=dict(case.info, nan_rows=np.asarray(rows), nan_part=part))


# ---------------------------------------------------------------------------------------------------------------
# The cross split score: an instance in one (query part, gallery part) pair
#
# sim_topk_split(cross=True) and sim_range_split(cross=True) rank on the maximum over every (query part a, gallery part
# b) of the bf16 dot product and trust cross_row_bound (sim_sweep.cuh): the largest over the pairs of row_bound's
# expression, from query part a's norms (q_norm_*[qrow * n_parts + a]) and gallery part b's maxima (g_max[2b],
# g_max[2b + 1]).  The operands are those of the split score (to_bf16_parts_kernel: split_operands).
#
# cross_embed puts a build() instance into the pair (a, b), a != b: the queries in query part a, the gallery in gallery
# part b; the other query parts are zero and the other gallery parts hold tiny exact fillers x*2^-11 (|x| <= 3).  Every
# other pair scores near 0 and has a term of at most 1e-3 of (a, b)'s, so eps comes from (a, b) alone: a bound read from
# the aligned pairs (split_row_bound), from another query part's norms or from another gallery part's maxima collapses
# below A's realized error.  The split layouts (split_embed) hold under the cross score too: their instance pairs are
# the aligned ones, and a pair across two parts meets a filler.

CROSS_PLACES = [(2, 64, 0, 1), (4, 516, 3, 0), (40, 64, 33, 1), (197, 64, 196, 0)]   # (C, p, a, b); 516 pads to 576
# the threshold search's shapes: resident query tile (d_pad <= 512) and streamed
CROSS_RANGE_SHAPES = ((2, 256), (4, 64), (8, 64), (4, 516), (40, 64), (197, 64))


def cross_embed(case: Case, n_parts: int, a: int, b: int, seed: int = 0) -> Case:
    """`case` (uncentred, dimension p): its queries in query part a, its gallery in gallery part b (see above)."""
    assert not case.centred and a != b and 0 <= a < n_parts and 0 <= b < n_parts
    nq, p = case.q.shape
    ng = case.g.shape[0]
    rng = np.random.default_rng(seed + 1009 * n_parts + 17 * a + b)
    q = np.zeros((nq, n_parts * p), np.float32)
    g = (rng.integers(-3, 4, size=(ng, n_parts * p)) * U).astype(np.float32)
    q[:, a * p:(a + 1) * p] = case.q
    g[:, b * p:(b + 1) * p] = case.g
    return Case(q=q, g=g, centred=False, target=case.target, comps=case.comps, twin=case.twin,
                info=dict(case.info, n_parts=n_parts, p=p, part=a, other=b, layout="pair"))


def cross_pairs(n_parts: int):
    """(a, b) of every pair a shape is tested at: the first query part against the last gallery part, the reverse, and
    query part 33 against gallery part 1 and 196 against 0 when there are such parts (the second and the seventh lane
    round of cross_row_bound's loop over a)."""
    pairs = [(0, n_parts - 1), (n_parts - 1, 0)] + ([(33, 1)] if n_parts > 33 else []) + ([(196, 0)] if n_parts > 196 else [])
    return list(dict.fromkeys(pairs))


def cross_placements(n_parts: int):
    """(layout, part, other): the pairs of cross_pairs, then the split layouts of split_placements."""
    return [("pair", a, b) for a, b in cross_pairs(n_parts)] + split_placements(n_parts)


def cross_case(name: str, p: int, n_parts: int, layout: str, part: int, other: int, **build_kw) -> Case:
    """A TOPK_CASES instance (or with name "range" build(p, 20, **build_kw)) at a placement of cross_placements."""
    if layout != "pair":
        return split_case(name, p, n_parts, part, layout, other, **build_kw)
    base = build(p, 20, centred=False, **build_kw) if name == "range" else topk_case(name, p, False, **build_kw)
    return cross_embed(base, n_parts, part, other)


def instance_pair(case: Case):
    """(query part, gallery part) where A reaches its score."""
    return (case.info["part"], case.info["other"]) if case.info["layout"] == "pair" else (case.info["part"],) * 2


def cross_part_eps(op: SplitOperands, p_pad: int) -> np.ndarray:
    """cross_row_bound's term of every (query part a, gallery part b), in the kernel's fp32 order of operations: query
    part a's norms, gallery part b's maxima, split_part_eps's expression: [nq, C, C]."""
    f = np.float32
    qh, qr, qx = op.qnh[:, :, None], op.qnr[:, :, None], op.qnx[:, :, None]
    gn, gr = op.g_norm[None, None, :], op.g_res[None, None, :]
    e = f(1.001) * (qh * gr + qr * gn) + f(p_pad) * f(2.4e-7) * qh * (gn + gr) + f(3e-7) * qx * gn + f(1e-30)
    return e.astype(np.float32)


def cross_eps(op: SplitOperands, p_pad: int) -> np.ndarray:
    """cross_row_bound's eps per query row: the largest pair term."""
    return cross_part_eps(op, p_pad).max(axis=(1, 2))


def cross_bf16_terms(op: SplitOperands) -> np.ndarray:
    """The bf16 part of every pair's term, qh_a g_res_b + qr_a g_norm_b: [nq, C, C]."""
    return (op.qnh[:, :, None] * op.g_res[None, None, :] + op.qnr[:, :, None] * op.g_norm[None, None, :]).astype(np.float32)


def _cross_fold(q: np.ndarray, g: np.ndarray, n_parts: int, as_f32: bool) -> np.ndarray:
    """max over every (query part, gallery part) of the fp64 dot product (rounded to fp32 first when as_f32), folded
    with fmax (a NaN pair is ignored), a few query parts at a time: memory about max(nq * ng * C, 2^23) values."""
    nq, d = q.shape
    ng, p = g.shape[0], d // n_parts
    q64 = q.astype(np.float64).reshape(nq, n_parts, p)
    g64 = g.astype(np.float64).reshape(ng * n_parts, p)
    best = np.full((nq, ng), -np.inf, np.float32 if as_f32 else np.float64)
    step = max(1, 2 ** 23 // (nq * ng * n_parts))
    for a in range(0, n_parts, step):
        na = min(step, n_parts - a)
        s = (q64[:, a:a + na].reshape(nq * na, p) @ g64.T).reshape(nq, na, ng, n_parts)
        s = np.fmax.reduce(np.fmax.reduce(s.astype(np.float32) if as_f32 else s, axis=3), axis=1)
        best = np.fmax(best, s)
    return best


def cross_approx(op: SplitOperands, n_parts: int) -> np.ndarray:
    """The fused sweep's cross score: per pair the tensor-core product of the bf16 operands (exact here) as fp32, then
    the maximum over the pairs."""
    return _cross_fold(op.qh, op.gh, n_parts, True)


def cross_exact(q: np.ndarray, g: np.ndarray, n_parts: int) -> np.ndarray:
    """The fp64 cross score."""
    return _cross_fold(q, g, n_parts, False)


def cross_realized(case: Case, op: SplitOperands) -> np.ndarray:
    """Per query: how far the target's approximate cross score lies below its exact cross score."""
    c = case.info["n_parts"]
    rows = np.arange(case.q.shape[0])
    return cross_exact(case.q, case.g, c)[rows, case.target] - cross_approx(op, c)[rows, case.target].astype(np.float64)


# The cross re-score (cross_exact_scores) stages the query `staged` parts at a time in kCrossStageBytes of shared
# memory, (pl + 8) fp64 values per part: the restatement of cross_staged_parts.
CROSS_STAGE_BYTES = 44 * 1024


def cross_staged_parts(n_parts: int, pl: int) -> int:
    return max(1, min(n_parts, CROSS_STAGE_BYTES // ((pl + 8) * 8)))


def cross_groups(n_parts: int, pl: int):
    """The sizes of the staged groups, in order."""
    s = cross_staged_parts(n_parts, pl)
    return [min(s, n_parts - a0) for a0 in range(0, n_parts, s)]


# (C, p): the shapes whose groups the staged-group tests walk, with those groups
STAGED_SHAPES = {(79, 64): [78, 1], (156, 64): [78, 78], (197, 64): [78, 78, 41], (3, 2808): [2, 1], (2, 4096): [1, 1],
                 (3, 8192): [1, 1, 1]}

# (C, p, parts of the first / second / brute instance, a part that is zero for every query): the mixed-stage shapes
MIXED_PLACES = [(4, 64, (0, 1, 3), 2), (40, 64, (1, 33, 39), 0)]
