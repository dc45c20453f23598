"""The split-score top-k without a GPU: the host-only planner of dcr_sim_topk_split_workspace_size."""


def _lib():
    from dcr_b200 import _lib
    return _lib.load()


def test_planner_accepts_per_token_shapes():
    lib = _lib()
    for nq, ng, d, c, k in [(10000, 100000, 197 * 384, 197, 10),     # ViT-S/16 tokens
                            (1000, 5000, 785 * 768, 785, 10),        # ViT-B/8 tokens, C * k > 4096
                            (10000, 100000, 512, 4, 10),
                            (3, 2048, 197 * 384, 197, 16),
                            (5, 700, 785 * 16, 785, 10),             # parts shorter than one 64-column k-block
                            (1, 1, 8192 * 3, 3, 1),                  # the longest part
                            (7, 300, 100, 1, 3)]:                    # one part: the dot-product planner
        assert lib.dcr_sim_topk_split_workspace_size(nq, ng, d, c, k) > 0, (nq, ng, d, c, k, lib.dcr_last_error())


def test_workspace_does_not_grow_with_nq_times_ng():
    """Beyond the bf16 copies of both sides, the workspace grows at most linearly when nq and ng both grow 4x (16x the
    pairs)."""
    lib = _lib()
    d, c = 197 * 64, 197                                  # p = 64: no part padding

    def extra(nq, ng):
        ws = lib.dcr_sim_topk_split_workspace_size(nq, ng, d, c, 10)
        assert ws > 0
        pad = lambda n: -(-n // 128) * 128
        return ws - 2 * (pad(nq) + pad(ng)) * d

    small, big = extra(10000, 100000), extra(40000, 400000)
    assert 0 < small and big < 4.5 * small


def test_bad_arguments_return_zero_with_a_message():
    lib = _lib()
    for nq, ng, d, c, k in [(10, 10, 66, 2, 1),           # part length 33: not a multiple of 4
                            (10, 10, 64, 3, 1),           # d not divisible into 3 parts
                            (10, 10, 8196 * 2, 2, 1),     # part length above 8192
                            (10, 10, 64, 0, 1),           # no parts
                            (10, 10, 64, -2, 1),
                            (10, 10, 64, 2, 0),           # k outside [1, 16]
                            (10, 40, 64, 2, 17),
                            (10, 5, 64, 2, 6),            # k > ng
                            (0, 10, 64, 2, 1),            # empty
                            (10, 0, 64, 2, 1)]:
        assert lib.dcr_sim_topk_split_workspace_size(nq, ng, d, c, k) == 0, (nq, ng, d, c, k)
        assert lib.dcr_last_error().decode() != ""
