"""Gallery-sharded threshold search without a GPU: the planner of dcr_sim_range_sharded_workspace_size and the only
refusals that may come before the first exchange."""
import ctypes as C
import itertools


def test_planner_accepts_the_supported_shape_range():
    from dcr_b200 import _lib
    lib = _lib.load()
    for nq, ng, d, world, cap in itertools.product([1, 7, 10000, 1000000], [0, 1, 100000, 5000000], [4, 100, 512, 8192],
                                                   [1, 2, 8, 1024], [0, 1 << 20, 1 << 40]):
        assert lib.dcr_sim_range_sharded_workspace_size(nq, ng, d, world, cap) > 0, (
            nq, ng, d, world, cap, lib.dcr_last_error().decode())


def test_planner_growth():
    """The workspace grows with the candidate capacity times the world size (the receive buffer) and with ng_local, never
    with nq * ng."""
    from dcr_b200 import _lib
    ws = _lib.load().dcr_sim_range_sharded_workspace_size
    base = ws(10000, 100000, 512, 4, 0)
    assert base < 10000 * 100000 // 4
    # one candidate more per rank costs the local search (8 B) plus a send and world receive slots (12 B each)
    grow = ws(10000, 100000, 512, 4, 10 ** 6) - base
    assert 10 ** 6 * (8 + 12 * 5) <= grow < 10 ** 6 * (8 + 12 * 5) + 10 ** 6
    assert ws(10000, 100000, 512, 8, 10 ** 6) - ws(10000, 100000, 512, 4, 10 ** 6) >= 4 * 10 ** 6 * 12
    assert ws(10000, 0, 512, 4, 10 ** 6) < ws(10000, 100000, 512, 4, 10 ** 6)   # an empty shard runs no search
    # 10x the gallery and 10x the queries: far from 100x
    assert ws(100000, 1000000, 512, 4, 0) < 12 * ws(10000, 100000, 512, 4, 0)


def test_planner_refusals():
    from dcr_b200 import _lib
    lib = _lib.load()
    for nq, ng, d, world, cap in [(0, 10, 64, 2, 100), (10, -1, 64, 2, 100), (10, 10, 8200, 2, 100), (10, 10, 66, 2, 100),
                                  (10, 10, 64, 0, 100), (10, 10, 64, 65536, 100), (10, 10, 64, 2, -1),
                                  (10, 10, 64, 2, (1 << 40) + 1), (10, 0, 0, 2, 100)]:
        assert lib.dcr_sim_range_sharded_workspace_size(nq, ng, d, world, cap) == 0, (nq, ng, d, world, cap)
        assert lib.dcr_last_error().decode() != ""


def test_refusals_before_the_exchange():
    """world < 1 and a missing callback with world > 1 are the only outcomes decided alone: there is nobody to agree with."""
    from dcr_b200 import _lib
    lib = _lib.load()
    counts = (C.c_int64 * 3)()
    args = lambda world: (None, 4, None, 0, 64, 0.5, 0, 1, world, None, None, None, None, None, 0, 0, counts, None, 0, None)
    assert lib.dcr_sim_range_sharded(*args(2)) == -1
    assert "all-gather callback" in lib.dcr_last_error().decode()
    assert lib.dcr_sim_range_sharded(*args(0)) == -1
    assert "world=0" in lib.dcr_last_error().decode()
