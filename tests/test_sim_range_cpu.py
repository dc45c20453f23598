"""Threshold search without a GPU: the planner of dcr_sim_range_workspace_size, the command-line flag and the
combinations it refuses, and the oracle the GPU tests compare against."""
import itertools

import numpy as np
import pytest

from tests import sim_range_oracle as orange


def test_planner_accepts_the_supported_shape_range():
    """Host-only planning: every shape of the supported range plans, and the workspace grows with the capacity but not
    with nq * ng."""
    from dcr_b200 import _lib
    lib = _lib.load()
    for nq, ng, d, cap in itertools.product([1, 7, 256, 10000, 1000000], [1, 16, 100000, 5000000],
                                            [4, 64, 100, 512, 1024, 8192], [0, 1 << 20, 10 ** 9, 1 << 40]):
        assert lib.dcr_sim_range_workspace_size(nq, ng, d, cap) > 0, (nq, ng, d, cap, lib.dcr_last_error().decode())
    small = lib.dcr_sim_range_workspace_size(10000, 100000, 512, 0)
    assert lib.dcr_sim_range_workspace_size(10000, 100000, 512, 10 ** 6) - small < 10 ** 6 * 9
    assert small < 10000 * 100000 // 4               # nothing proportional to nq * ng
    for nq, ng, d, cap in [(0, 10, 64, 100), (10, 0, 64, 100), (10, 10, 8200, 100), (10, 10, 66, 100),
                           (10, 10, 64, -1), (10, 10, 64, (1 << 40) + 1)]:
        assert lib.dcr_sim_range_workspace_size(nq, ng, d, cap) == 0
        assert lib.dcr_last_error().decode() != ""


def test_cli_flag_and_refused_combinations(tmp_path):
    from dcr_b200 import cli
    p = cli.build_parser()
    assert p.parse_args(["--query_dir", "a", "--val_dir", "b"]).sim_threshold is None
    assert p.parse_args(["--query_dir", "a", "--val_dir", "b", "--sim_threshold", "0.5"]).sim_threshold == 0.5
    assert p.parse_args(["--query_dir", "a", "--val_dir", "b", "--sim_threshold=-inf"]).sim_threshold == -np.inf
    common = ["--query_dir", str(tmp_path), "--val_dir", str(tmp_path), "--sim_threshold", "0.5"]
    with pytest.raises(NotImplementedError):
        cli.main(common + ["--similarity_metric", "splitloss", "--num_loss_chunks", "2"])
    with pytest.raises(NotImplementedError):
        cli.main(common + ["--world-size", "2", "--rank", "0"])
    with pytest.raises(NotImplementedError):
        cli.main(common + ["--multiprocessing-distributed"])


def test_oracle_is_a_dense_threshold():
    rng = np.random.default_rng(0)
    q = rng.standard_normal((37, 24)).astype(np.float32)
    g = rng.standard_normal((90, 24)).astype(np.float32)
    g[5] = np.nan
    dense = (q.astype(np.float64) @ g.astype(np.float64).T).astype(np.float32)
    for t in (-np.inf, -1.0, 0.0, 2.5, np.inf):
        off, idx, val = orange.sim_range(q, g, t, chunk=8)
        assert off[0] == 0 and off[-1] == idx.size == val.size
        for r in range(q.shape[0]):
            cols = np.nonzero(dense[r] >= np.float32(t))[0]
            assert np.array_equal(idx[off[r]:off[r + 1]], cols)
            assert np.array_equal(val[off[r]:off[r + 1]], dense[r, cols])
            assert 5 not in cols                       # NaN scores are never reported
    off, idx, _ = orange.sim_range(q, g, -np.inf)
    assert idx.size == 37 * 89
