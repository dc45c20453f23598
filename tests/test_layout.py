"""Repository contract checks that need no GPU: the C-ABI library loads and exports every symbol the header declares,
the ctypes table mirrors the header, and nothing under dcr_b200/ touches the oracle or /root/reference."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_functions():
    src = open(os.path.join(ROOT, "include", "dcr_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(dcr_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from dcr_b200 import _lib
    lib = _lib.load()
    names = _header_functions()
    assert len(names) >= 15
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/dcr_b200.h but not exported"
    assert set(_lib.SIGNATURES) == set(names), set(_lib.SIGNATURES) ^ set(names)
    assert lib.dcr_version() == 100


def test_compute_calls_fail_loudly_without_gpu():
    import torch
    from dcr_b200 import _lib
    lib = _lib.load()
    if torch.cuda.is_available():
        return
    assert lib.dcr_device_sm_count() < 0
    assert lib.dcr_sim_topk_workspace_size(10, 10, 64, 1) in (0, lib.dcr_sim_topk_workspace_size(10, 10, 64, 1))
    import pytest
    from dcr_b200 import similarity
    with pytest.raises(_lib.DcrError):
        similarity.sim_topk(torch.zeros(4, 64), torch.zeros(8, 64), 1)


def test_product_never_imports_oracle_or_reference():
    bad = []
    for dirpath, _, files in os.walk(os.path.join(ROOT, "dcr_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dirpath, f)).read()
                if re.search(r"^\s*(from|import)\s+oracle\b", txt, flags=re.M) or "/root/reference" in txt:
                    bad.append(os.path.join(dirpath, f))
    assert not bad, bad


def test_similarity_planner_accepts_the_supported_shape_range():
    """dcr_sim_topk_workspace_size is host-only (launch planning: tiles, chunks, shared-memory budget, candidate slots):
    every shape of the supported range must plan -- the BASELINE configs, single rows, 1M+ galleries, descriptor dims up
    to 8192, every k <= 16 -- and out-of-range arguments must be refused with a message."""
    import itertools
    from dcr_b200 import _lib
    lib = _lib.load()
    for nq, ng, d, k in itertools.product([1, 7, 256, 10000, 50000, 1000000], [16, 1000, 100000, 1000000, 5000000],
                                          [4, 64, 100, 384, 512, 768, 1024, 2048, 8192], [1, 2, 5, 10, 16]):
        if k > ng:
            continue
        assert lib.dcr_sim_topk_workspace_size(nq, ng, d, k) > 0, (nq, ng, d, k, lib.dcr_last_error().decode())
    for nq, ng, d, k in [(0, 10, 64, 1), (10, 10, 64, 17), (10, 5, 64, 8), (10, 10, 8200, 1), (10, 0, 64, 1)]:
        assert lib.dcr_sim_topk_workspace_size(nq, ng, d, k) == 0
        assert lib.dcr_last_error().decode() != ""


def test_hopper_scaffolding_has_one_definition():
    """The opt-in to large dynamic shared memory, the kernel launch, the TMA bulk-store group and the 1024-byte alignment
    of dynamic shared memory are each written once (host_util, ptx.cuh); kernels and launch sites use those instead of a
    private copy."""
    csrc = os.path.join(ROOT, "dcr_b200", "csrc")
    texts = {f: open(os.path.join(csrc, f)).read() for f in sorted(os.listdir(csrc)) if f.endswith((".cu", ".cuh", ".h"))}
    for needle, home in [("cudaFuncSetAttribute", "host_util.cu"), ("cp.async.bulk.commit_group", "ptx.cuh"),
                         ("cp.async.bulk.wait_group", "ptx.cuh"), ("~uintptr_t(1023)", "ptx.cuh")]:
        assert [f for f, t in texts.items() if needle in t] == [home], needle
    # every kernel is launched through host_util's launch(): counted, error-checked under its caller's name, smem opted in
    sources = [f for f in texts if f.endswith((".cu", ".cuh"))]
    assert "sim_sweep.cu" in sources and "pool_norm.cu" in sources
    assert [f for f in sources if "<<<" in texts[f]] == ["host_util.cuh"]
    assert [f for f in texts if "count_launch(" in texts[f]] == ["host_util.cu", "host_util.cuh"]
    # workspaces are laid out with Carve, not with private round-up helpers
    assert [f for f in texts if "up256" in texts[f]] == []
