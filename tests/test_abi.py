"""CPU: the C-ABI library loads and exports exactly the symbols include/b200rec.h declares (no compute)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def built_lib():
    from rechorus_b200 import build
    return build.build()


def _declared():
    src = open(os.path.join(ROOT, "include", "b200rec.h")).read()
    return sorted(set(re.findall(r"B2R_API[^;(]*?\b(b2r_\w+)\s*\(", src)))


def test_header_declares_entry_points():
    names = _declared()
    assert "b2r_rowdot_fwd" in names and "b2r_segment_apply" in names and len(names) >= 12


def test_library_exports_every_declared_symbol(built_lib):
    lib = ctypes.CDLL(built_lib)
    for name in _declared():
        assert hasattr(lib, name), f"{name} declared in include/b200rec.h but not exported"


def test_binding_table_matches_header_at_abi_version_102(built_lib):
    from rechorus_b200 import lib as L
    assert sorted(L.SIGNATURES) == _declared()
    handle = L.load()
    assert handle.b2r_version() == 102
    assert ctypes.sizeof(L.GradSource) == 40 and ctypes.sizeof(L.Optim) == 48      # b2r_optim: 9 x 4 bytes, pad, clock pointer


def test_bad_arguments_are_rejected_without_a_gpu(built_lib):
    from rechorus_b200 import lib as L
    handle = L.load()
    rc = handle.b2r_rowdot_fwd(None, None, 0, None, None, 0, None, 4, 4, 64, None, None)
    assert rc == -1 and b"null pointer" in handle.b2r_last_error()
    rc = handle.b2r_bpr_loss(None, None, None, None, 1, 1, None)
    assert rc == -1
    assert handle.b2r_plan_workspace_bytes(0, 10) == 0


def test_no_cpu_fallback():
    import torch
    from rechorus_b200 import ops
    from rechorus_b200.lib import B200RecError
    with pytest.raises(B200RecError):
        ops.rowdot(torch.zeros(2, 8), None, torch.zeros(4, 8), torch.zeros(2, 3, dtype=torch.int64))


def test_header_with_its_public_structs_is_plain_c99(tmp_path):
    """the boundary is a C ABI: the header must compile as C (no C++-isms, no torch/CUDA types)"""
    import shutil
    import subprocess
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    src = tmp_path / "use_header.c"
    src.write_text('#include "b200rec.h"\nint main(void) { b2r_grad_source g; b2r_optim o; b2r_bprmf_tables t; (void)g; (void)o; (void)t; return 0; }\n')
    r = subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-fsyntax-only",
                        "-I", os.path.join(ROOT, "include"), str(src)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def test_eval_and_direct_plan_entry_points_reject_bad_arguments(built_lib):
    from rechorus_b200 import lib as L
    h = L.load()
    assert h.b2r_gt_rank(None, 4, 4, 4, None, None) == -1 and b"null pointer" in h.b2r_last_error()
    assert h.b2r_rank_histogram(None, 4, 10, None, None) == -1
    assert h.b2r_rank_all_items(None, 64, None, None, 4, 100, 64, None, None, 0, None, None, None, None) == -1
    assert h.b2r_direct_plan_apply(None, 100, 1000, 64, None, None, 2, None, None, None, None, None, None) == -1
    assert h.b2r_direct_plan_workspace_bytes(0, 10) == 0 and h.b2r_direct_plan_workspace_bytes(100, 1000) > 100 * 24


def test_step_workspace_is_sized_from_the_direct_plans(built_lib):
    """b2r_bprmf_step_workspace_bytes covers the benchmarked shapes and is 0 where the step's index plans cannot be
    sized (B*C > 2^30 - 1); the plugin then trains through the autograd route."""
    from rechorus_b200 import lib as L
    h = L.load()
    assert h.b2r_bprmf_step_workspace_bytes(4096, 100, 64, 1_000_000, 1_000_000) > 0            # c2
    assert h.b2r_bprmf_step_workspace_bytes(4096, 256, 128, 1_000_000, 25_000_000) > 0          # c5 on one GPU
    assert h.b2r_direct_plan_workspace_bytes(2 ** 21 * 513, 1_000_000) == 0
    assert h.b2r_bprmf_step_workspace_bytes(2 ** 21, 513, 64, 1_000_000, 1_000_000) == 0
