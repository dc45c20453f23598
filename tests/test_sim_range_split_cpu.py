"""The threshold search under the split score without a GPU: the host-only planners of
dcr_sim_range_split_workspace_size and dcr_sim_range_split_sharded_workspace_size, and the dense fp64 split-score oracle
the GPU tests compare against."""
import itertools

import numpy as np

from oracle import similarity as osim


def _lib():
    from dcr_b200 import _lib
    return _lib.load()


def split_scores(q: np.ndarray, g: np.ndarray, n_parts: int) -> np.ndarray:
    """Dense [nq, ng] split scores: per part the fp64 dot product, folded with fmax from -inf in part order (a NaN part is
    ignored, all-NaN parts give -inf), rounded to fp32 once."""
    nq, d = q.shape
    p = d // n_parts
    q64 = q.astype(np.float64).reshape(nq, n_parts, p)
    g64 = g.astype(np.float64).reshape(g.shape[0], n_parts, p)
    best = np.full((nq, g.shape[0]), -np.inf)
    for c in range(n_parts):
        best = np.fmax(best, q64[:, c] @ g64[:, c].T)
    return best.astype(np.float32)


def split_range(q: np.ndarray, g: np.ndarray, n_parts: int, threshold: float):
    """The CSR dcr_sim_range_split returns: (offsets, local gallery rows ascending, fp32 scores)."""
    s = split_scores(q, g, n_parts)
    keep = s >= np.float32(threshold)
    off = np.concatenate([[0], np.cumsum(keep.sum(axis=1))]).astype(np.int64)
    rows, cols = np.nonzero(keep)
    return off, cols.astype(np.int64), s[rows, cols]


def test_oracle_agrees_with_the_einsum_max():
    rng = np.random.default_rng(3)
    for nq, ng, d, c in [(9, 40, 64, 4), (5, 33, 96, 3), (4, 17, 48, 1)]:
        q = rng.standard_normal((nq, d)).astype(np.float32)
        g = rng.standard_normal((ng, d)).astype(np.float32)
        s = split_scores(q, g, c)
        v, i = osim.sim_topk_split(q, g, ng, c)          # every row, ranked: the einsum max of diff_retrieval.py:399
        assert np.array_equal(np.take_along_axis(s, i, axis=1), v)
        off, idx, val = split_range(q, g, c, -np.inf)
        assert off[-1] == nq * ng and np.array_equal(val, s.reshape(-1))


def test_oracle_nan_parts():
    q = np.ones((2, 8), np.float32)
    g = np.ones((3, 8), np.float32)
    g[0, :4] = np.nan                                     # one NaN part: ignored
    g[1] = np.nan                                         # every part NaN: -inf
    s = split_scores(q, g, 2)
    assert s[0, 0] == 4 and s[0, 1] == -np.inf and s[0, 2] == 4
    off, idx, _ = split_range(q, g, 2, 0.0)
    assert off.tolist() == [0, 2, 4] and idx.tolist() == [0, 2, 0, 2]
    off, idx, val = split_range(q, g, 2, -np.inf)
    assert off[-1] == 6 and val[1] == -np.inf


def test_planner_accepts_the_supported_range():
    lib = _lib()
    for nq, ng, (p, c), cap in itertools.product([1, 130, 10000], [1, 100000, 5000000],
                                                 [(4, 2), (16, 785), (64, 197), (384, 197), (128, 4), (8192, 3)],
                                                 [0, 1 << 20, 1 << 40]):
        assert lib.dcr_sim_range_split_workspace_size(nq, ng, p * c, c, cap) > 0, (
            nq, ng, p, c, cap, lib.dcr_last_error().decode())


def test_planner_refusals():
    lib = _lib()
    for nq, ng, d, c, cap, match in [(10, 10, 64, 3, 100, "parts"),          # d % n_parts
                                     (10, 10, 66, 2, 100, "multiple of 4"),  # p = 33
                                     (10, 10, 8196 * 2, 2, 100, "8192"),     # p > 8192
                                     (10, 10, 64, 0, 100, "n_parts"),
                                     (10, 10, 64, -3, 100, "n_parts"),
                                     (10, 10, 64, 2, -1, "max_pairs"),
                                     (10, 10, 64, 2, (1 << 40) + 1, "max_pairs"),
                                     (0, 10, 64, 2, 100, "empty"),
                                     (10, 0, 64, 2, 100, "empty")]:
        assert lib.dcr_sim_range_split_workspace_size(nq, ng, d, c, cap) == 0, (nq, ng, d, c, cap)
        msg = lib.dcr_last_error().decode()
        assert match in msg and "sim_range_split" in msg, msg


def test_one_part_plans_the_dot_product_search():
    lib = _lib()
    for nq, ng, d, cap in [(1, 1, 4, 0), (130, 3000, 512, 1 << 20), (10000, 100000, 384, 1 << 30), (7, 300, 8192, 5)]:
        assert lib.dcr_sim_range_split_workspace_size(nq, ng, d, 1, cap) == lib.dcr_sim_range_workspace_size(nq, ng, d, cap)
        assert (lib.dcr_sim_range_split_sharded_workspace_size(nq, ng, d, 1, 3, cap)
                == lib.dcr_sim_range_sharded_workspace_size(nq, ng, d, 3, cap))


def test_workspace_does_not_grow_with_nq_times_ng():
    """Beyond the bf16 copies of both sides and the candidate capacity, the workspace grows at most linearly when nq and
    ng both grow 4x (16x the pairs)."""
    lib = _lib()
    d, c, cap = 197 * 64, 197, 1 << 20                    # p = 64: no part padding

    def extra(nq, ng):
        ws = lib.dcr_sim_range_split_workspace_size(nq, ng, d, c, cap)
        assert ws > 0
        pad = lambda n: -(-n // 128) * 128
        return ws - 2 * (pad(nq) + pad(ng)) * d

    small, big = extra(10000, 100000), extra(40000, 400000)
    assert 0 < small and big < 4.5 * small
    # one candidate more: its index and score, and at most a piece's bookkeeping
    grow = lib.dcr_sim_range_split_workspace_size(1000, 5000, 512, 4, 10 ** 6 + cap) - \
        lib.dcr_sim_range_split_workspace_size(1000, 5000, 512, 4, cap)
    assert 8 * 10 ** 6 <= grow < 8 * 10 ** 6 + 10 ** 5


def _round(n):
    return -(-n // 256) * 256


def test_sharded_workspace_equals_its_layout():
    """header, inner search, send, world x receive, row counts, flag -- each cut at a 256-byte boundary."""
    lib = _lib()
    for nq, ng, d, c, world, cap in [(7, 300, 512, 4, 2, 1000), (130, 0, 197 * 64, 197, 3, 1 << 20),
                                     (1, 1, 8, 2, 1, 0), (10000, 100000, 512, 4, 8, 1 << 24)]:
        inner = lib.dcr_sim_range_split_workspace_size(nq, max(ng, 1), d, c, cap) if ng > 0 else 0
        msg = (8 * (nq + 1) + 12 * cap + 15) // 16 * 16
        want = (_round(80 * (world + 1)) + _round(inner) + _round(msg) + _round(msg * world) + _round(8 * nq)
                + _round(4))
        assert lib.dcr_sim_range_split_sharded_workspace_size(nq, ng, d, c, world, cap) == want, (nq, ng, d, c, world)


def test_sharded_planner_refusals():
    lib = _lib()
    for nq, ng, d, c, world, cap in [(10, 10, 64, 0, 2, 100), (10, 10, 64, 3, 2, 100), (10, 10, 66, 2, 2, 100),
                                     (10, 10, 64, 2, 0, 100), (10, 10, 64, 2, 65536, 100), (10, 10, 64, 2, 2, -1),
                                     (0, 10, 64, 2, 2, 100), (10, -1, 64, 2, 2, 100)]:
        assert lib.dcr_sim_range_split_sharded_workspace_size(nq, ng, d, c, world, cap) == 0, (nq, ng, d, c, world, cap)
        assert "sim_range_split" in lib.dcr_last_error().decode()
