"""Workspace sizes that are planned on the host, pinned to their layouts: a caller (dist.sharded_topk,
complexity._jpeg_chunk) sizes its allocations and chunks from them, so a change of layout must not change them."""
import itertools


def _up(x):
    return (x + 255) // 256 * 256


def test_sim_topk_sharded_workspace_size(lib):
    # the local search's workspace, this rank's list, world gathered lists, their scores and their indices
    for nq, ng, d, k, world in itertools.product([1, 7, 256, 10000], [1, 3, 16, 1000, 100000], [4, 64, 512, 2048],
                                                 [1, 5, 10, 16, 32], [1, 2, 8]):
        inner = lib.dcr_sim_topk_workspace_size(nq, ng, d, min(k, ng))
        L = nq * k
        want = _up(inner) + _up(12 * L) + _up(12 * L * world) + _up(4 * L * world) + _up(8 * L * world) if inner else 0
        assert lib.dcr_sim_topk_sharded_workspace_size(nq, ng, d, k, world) == want, (nq, ng, d, k, world)
    assert lib.dcr_sim_topk_sharded_workspace_size(10, 3, 64, 32, 2) > 0   # a shard smaller than k plans top-3
    for nq, ng, d, k, world in [(0, 10, 64, 1, 1), (10, 10, 64, 0, 1), (10, 10, 64, 1, 0), (10, 0, 64, 1, 2),
                                (10, 10, 8200, 1, 2), (10, 100, 64, 17, 1)]:
        assert lib.dcr_sim_topk_sharded_workspace_size(nq, ng, d, k, world) == 0, (nq, ng, d, k, world)


def test_jpeg_workspace_size(lib):
    # DC coefficients (int16) and AC bit counts (uint32) per block, total bits per image, the header, then the bit buffer
    for n, h, w in itertools.product([0, 1, 3, 64, 1000], [16, 48, 256, 4096], [16, 32, 512, 4096]):
        nb = 6 * (h // 16) * (w // 16)
        words = -(-nb * 1660 // 32)
        want = _up(2 * n * nb) + _up(4 * n * nb) + _up(4 * n) + _up(623) + 4 * n * words
        assert lib.dcr_jpeg_workspace_size(n, h, w) == want, (n, h, w)
    for n, h, w in [(-1, 16, 16), (1, 8, 16), (1, 16, 24), (1, 4112, 16)]:
        assert lib.dcr_jpeg_workspace_size(n, h, w) == 0, (n, h, w)
