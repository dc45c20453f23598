"""The cross split score without a GPU: the host-only planners of dcr_sim_topk_cross_workspace_size and
dcr_sim_range_cross_workspace_size, and the dense fp64 cross-score oracle the GPU tests compare against.

The cross score of a pair is the maximum over every (query part a, gallery part b) of <q_a, g_b> (--stype cross,
einsum_in_chunks)."""
import numpy as np

from oracle import similarity as osim


def _lib():
    from dcr_b200 import _lib
    return _lib.load()


def cross_scores64(q: np.ndarray, g: np.ndarray, n_parts: int) -> np.ndarray:
    """Dense [nq, ng] cross scores in fp64: the fp64 dot product of every (query part, gallery part) pair, folded with
    fmax from -inf (a NaN pair is ignored, all-NaN pairs give -inf).  One [nq, ng, C] product per query part, so the
    memory is nq * ng * C, never nq * ng * C^2."""
    nq, d = q.shape
    ng = g.shape[0]
    p = d // n_parts
    q64 = q.astype(np.float64).reshape(nq, n_parts, p)
    g64 = g.astype(np.float64).reshape(ng * n_parts, p)
    best = np.full((nq, ng), -np.inf)
    for a in range(n_parts):
        s = (q64[:, a] @ g64.T).reshape(nq, ng, n_parts)
        best = np.fmax(best, np.fmax.reduce(s, axis=2))
    return best


def cross_topk(q: np.ndarray, g: np.ndarray, k: int, n_parts: int):
    """(values f32[Q,k], indices i64[Q,k]) ranked on the fp64 cross score, ties to the lowest gallery index."""
    s = cross_scores64(q, g, n_parts)
    idx = np.stack([osim._rank_row(row, k) for row in s])
    return np.take_along_axis(s, idx, axis=1).astype(np.float32), idx


def cross_range(q: np.ndarray, g: np.ndarray, n_parts: int, threshold: float):
    """The CSR dcr_sim_range_cross returns: (offsets, local gallery rows ascending, fp32 scores)."""
    s = cross_scores64(q, g, n_parts).astype(np.float32)
    keep = s >= np.float32(threshold)
    off = np.concatenate([[0], np.cumsum(keep.sum(axis=1))]).astype(np.int64)
    rows, cols = np.nonzero(keep)
    return off, cols.astype(np.int64), s[rows, cols]


def test_planner_accepts_per_token_shapes():
    lib = _lib()
    for nq, ng, d, c, k in [(10000, 100000, 197 * 384, 197, 10),     # ViT-S/16 tokens
                            (1000, 5000, 785 * 768, 785, 10),        # ViT-B/8 tokens: 785^2 * 12 k-blocks per tile
                            (10000, 100000, 512, 4, 10),
                            (1000, 10000, 197 * 384, 197, 1),
                            (5, 700, 785 * 16, 785, 16),             # parts shorter than one 64-column k-block
                            (1, 1, 8192 * 3, 3, 1),                  # the longest part
                            (7, 300, 100, 1, 3)]:                    # one part: the dot-product planner
        assert lib.dcr_sim_topk_cross_workspace_size(nq, ng, d, c, k) > 0, (nq, ng, d, c, k, lib.dcr_last_error())
    for nq, ng, d, c in [(10000, 100000, 197 * 384, 197), (1000, 5000, 785 * 768, 785), (10000, 100000, 512, 4),
                         (1, 1, 8192 * 3, 3), (7, 300, 100, 1)]:
        assert lib.dcr_sim_range_cross_workspace_size(nq, ng, d, c, 1 << 20) > 0, (nq, ng, d, c, lib.dcr_last_error())


def test_cross_and_aligned_plan_the_same_workspace():
    """The cross schedule changes the sweep's k-loop, not what the search keeps: the same bytes as the aligned form."""
    lib = _lib()
    for nq, ng, d, c, k in [(10000, 100000, 197 * 384, 197, 10), (300, 4000, 512, 4, 3)]:
        assert lib.dcr_sim_topk_cross_workspace_size(nq, ng, d, c, k) == lib.dcr_sim_topk_split_workspace_size(nq, ng, d, c, k)
        assert (lib.dcr_sim_range_cross_workspace_size(nq, ng, d, c, 12345)
                == lib.dcr_sim_range_split_workspace_size(nq, ng, d, c, 12345))


def test_bad_arguments_return_zero_with_a_message():
    lib = _lib()
    for nq, ng, d, c, k, what in [(10, 10, 66, 2, 1, "multiple of 4"),     # part length 33
                                  (10, 10, 64, 3, 1, "split into"),        # d not divisible into 3 parts
                                  (10, 10, 8196 * 2, 2, 1, "8192"),        # part length above 8192
                                  (10, 10, 64, 0, 1, "n_parts"),
                                  (10, 40, 64, 2, 17, "k="),
                                  (10, 40, 64, 2, 0, "k="),
                                  (10, 5, 64, 2, 6, "gallery size"),       # k > ng
                                  (0, 10, 64, 2, 1, "empty")]:
        assert lib.dcr_sim_topk_cross_workspace_size(nq, ng, d, c, k) == 0, (nq, ng, d, c, k)
        msg = lib.dcr_last_error().decode()
        assert what in msg and "sim_topk" in msg, (what, msg)
    for nq, ng, d, c, what in [(10, 10, 66, 2, "multiple of 4"), (10, 10, 64, 3, "split into"),
                               (10, 10, 8196 * 2, 2, "8192"), (10, 10, 64, 0, "n_parts"), (0, 10, 64, 2, "empty")]:
        assert lib.dcr_sim_range_cross_workspace_size(nq, ng, d, c, 100) == 0, (nq, ng, d, c)
        msg = lib.dcr_last_error().decode()
        assert what in msg and "sim_range" in msg, (what, msg)
    assert lib.dcr_sim_topk_cross_workspace_size(10, 10, 64, 2, 1) > 0   # the message of a refusal names the cross form
    lib.dcr_sim_topk_cross_workspace_size(10, 10, 66, 2, 1)
    assert "sim_topk_cross" in lib.dcr_last_error().decode()
    lib.dcr_sim_range_cross_workspace_size(10, 10, 66, 2, 1)
    assert "sim_range_cross" in lib.dcr_last_error().decode()


def test_oracle_with_one_part_is_the_dot_product():
    rng = np.random.default_rng(1)
    q = rng.standard_normal((7, 48)).astype(np.float32)
    g = rng.standard_normal((30, 48)).astype(np.float32)
    np.testing.assert_array_equal(cross_scores64(q, g, 1), q.astype(np.float64) @ g.astype(np.float64).T)


def test_cross_score_is_at_least_the_aligned_score():
    rng = np.random.default_rng(2)
    for c in (2, 3, 8):
        q = rng.standard_normal((9, 24 * c)).astype(np.float32)
        g = rng.standard_normal((40, 24 * c)).astype(np.float32)
        p = 24
        aligned = np.max(np.einsum("nap,map->nma", q.astype(np.float64).reshape(9, c, p),
                                   g.astype(np.float64).reshape(40, c, p)), axis=2)
        # the aligned pairs are among the cross pairs (up to the association of two fp64 matrix products)
        assert np.all(cross_scores64(q, g, c) >= aligned - 1e-12 * np.abs(aligned).max())


def test_oracles_agree():
    """The dense cross oracle, its top-k and its threshold CSR agree with oracle.similarity.sim_topk_split(cross=True)."""
    rng = np.random.default_rng(4)
    for nq, ng, d, c, k in [(9, 40, 64, 4, 5), (5, 33, 96, 3, 1), (4, 17, 48, 1, 3)]:
        q = rng.standard_normal((nq, d)).astype(np.float32)
        g = rng.standard_normal((ng, d)).astype(np.float32)
        g[5] = g[2]
        ov, oi = osim.sim_topk_split(q, g, k, c, cross=True, chunk=4)
        v, i = cross_topk(q, g, k, c)
        np.testing.assert_array_equal(i, oi)
        np.testing.assert_array_equal(v, ov)
        # every pair above the k-th score of its row is in the CSR at that threshold
        s = cross_scores64(q, g, c).astype(np.float32)
        for r in range(nq):
            off, cols, sc = cross_range(q[r:r + 1], g, c, float(ov[r, -1]))
            assert set(oi[r].tolist()) <= set(cols.tolist())
            np.testing.assert_array_equal(sc, s[r, cols])
            assert np.all(np.diff(cols) > 0) and off[-1] == cols.size
        off, cols, _ = cross_range(q, g, c, float("-inf"))
        assert off[-1] == nq * ng
