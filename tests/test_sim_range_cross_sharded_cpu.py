"""Gallery-sharded threshold search under the cross split score without a GPU: the planner of
dcr_sim_range_cross_sharded_workspace_size, its refusals, the bytes sharding adds around the local search, and the only
refusals that may come before the first exchange."""
import ctypes as C
import itertools


def _lib():
    from dcr_b200 import _lib
    return _lib.load()


def test_planner_accepts_the_supported_shape_range():
    """The shapes the dot-product planner test accepts, with d = p * C for parts of those lengths."""
    lib = _lib()
    for nq, ng, p, c, world, cap in itertools.product([1, 7, 10000, 1000000], [0, 1, 100000, 5000000], [4, 100, 512, 8192],
                                                      [2, 4, 197], [1, 2, 8, 1024], [0, 1 << 20, 1 << 40]):
        assert lib.dcr_sim_range_cross_sharded_workspace_size(nq, ng, p * c, c, world, cap) > 0, (
            nq, ng, p, c, world, cap, lib.dcr_last_error().decode())


def test_planner_refusals():
    lib = _lib()
    for nq, ng, d, c, world, cap, match in [(10, 10, 64, 0, 2, 100, "n_parts"),
                                            (10, 10, 64, -4, 2, 100, "n_parts"),
                                            (10, 10, 64, 3, 2, 100, "parts"),            # d % n_parts
                                            (10, 10, 66, 2, 2, 100, "multiple of 4"),    # p = 33
                                            (10, 10, 8196 * 2, 2, 2, 100, "8192"),       # p > 8192
                                            (10, 10, 64, 2, 0, 100, "world"),
                                            (10, 10, 64, 2, 65536, 100, "world"),
                                            (10, 10, 64, 2, 2, -1, "max_local_pairs"),
                                            (10, 10, 64, 2, 2, (1 << 40) + 1, "max_local_pairs"),
                                            (0, 10, 64, 2, 2, 100, "nq"),
                                            (10, -1, 64, 2, 2, 100, "ng_local")]:
        assert lib.dcr_sim_range_cross_sharded_workspace_size(nq, ng, d, c, world, cap) == 0, (nq, ng, d, c, world, cap)
        msg = lib.dcr_last_error().decode()
        assert match in msg and "sim_range_cross" in msg, msg


def test_sharding_adds_the_same_bytes_around_either_local_search():
    """header, send, world x receive, row counts and flag around the local search: the same for the aligned and the
    cross split score."""
    lib = _lib()
    for nq, ng, d, c, world, cap in [(7, 300, 512, 4, 2, 1000), (130, 5, 197 * 64, 197, 3, 1 << 20),
                                     (1, 1, 8, 2, 1, 0), (10000, 100000, 512, 4, 8, 1 << 24),
                                     (1000, 10000, 197 * 384, 197, 2, 1 << 20)]:
        cross = lib.dcr_sim_range_cross_sharded_workspace_size(nq, ng, d, c, world, cap)
        split = lib.dcr_sim_range_split_sharded_workspace_size(nq, ng, d, c, world, cap)
        inner_cross = lib.dcr_sim_range_cross_workspace_size(nq, ng, d, c, cap)
        inner_split = lib.dcr_sim_range_split_workspace_size(nq, ng, d, c, cap)
        assert min(cross, split, inner_cross, inner_split) > 0, (nq, ng, d, c, world, cap)
        assert cross - inner_cross == split - inner_split, (nq, ng, d, c, world, cap)


def test_one_part_plans_the_dot_product_search():
    lib = _lib()
    for nq, ng, d, world, cap in [(1, 1, 4, 1, 0), (130, 3000, 512, 2, 1 << 20), (10000, 0, 384, 8, 1 << 30)]:
        assert (lib.dcr_sim_range_cross_sharded_workspace_size(nq, ng, d, 1, world, cap)
                == lib.dcr_sim_range_sharded_workspace_size(nq, ng, d, world, cap))


def test_refusals_before_the_exchange():
    """world < 1 and a missing callback with world > 1 are the only outcomes decided alone: there is nobody to agree with."""
    lib = _lib()
    counts = (C.c_int64 * 3)()
    args = lambda world: (None, 4, None, 0, 64, 4, 0.5, 0, 1, world, None, None, None, None, None, 0, 0, counts, None, 0,
                          None)
    assert lib.dcr_sim_range_cross_sharded(*args(2)) == -1
    msg = lib.dcr_last_error().decode()
    assert "all-gather callback" in msg and "sim_range_cross_sharded" in msg
    assert lib.dcr_sim_range_cross_sharded(*args(0)) == -1
    assert "world=0" in lib.dcr_last_error().decode()
