"""Host-side parts of the sharded FID statistics that need no GPU: the packed-state size, the `distributed=` argument,
and the block sharding of tools/fid_scaling.py."""
import pytest

from dcr_b200 import _lib
from dcr_b200 import fid as dfid


def test_packed_size_is_header_plus_shift_sum_and_square():
    lib = _lib.load()
    for d in (1, 64, 256, 2048, 16384):
        assert lib.dcr_fid_packed_size(d) == 32 + 8 * (2 * d + d * d)
    for d in (0, -3, 16385):
        assert lib.dcr_fid_packed_size(d) == 0
        assert "bad dim" in _lib.last_error()


def test_sharding_is_opt_in_and_needs_a_process_group():
    import torch.distributed as dist
    assert dfid._group_of(False) == (None, 1) and dfid._group_of(None) == (None, 1)
    if not dist.is_initialized():
        with pytest.raises(_lib.DcrError, match="process group"):
            dfid._group_of(True)


@pytest.mark.parametrize("total,block", [(50000, 500), (4001, 500), (7, 3)])
def test_scaling_blocks_cover_the_same_set_for_every_world_size(total, block):
    """tools/fid_scaling.py deals whole seeded blocks to the ranks: for every N the ranks' blocks, in rank order, are the
    global blocks 0..B-1 with the same sizes, so the union is the same image set."""
    import importlib.util
    import os
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools", "fid_scaling.py")
    spec = importlib.util.spec_from_file_location("fid_scaling", path)
    tool = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tool)
    whole = tool.rank_blocks(total, block, 0, 1)
    assert sum(n for _, n in whole) == total
    for world in (2, 3, 8):
        got = [blk for rank in range(world) for blk in tool.rank_blocks(total, block, rank, world)]
        assert got == whole
