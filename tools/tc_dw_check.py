#!/usr/bin/env python
"""Time the wgmma weight-gradient kernel (csrc/linear_dw_tc.cu) against the CUDA-core kernel, with a coarse error check
against fp64 on the side.  The accuracy criteria live in tests/test_gpu_linear_tc.py."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from rechorus_b200 import lib as _lib, ops  # noqa: E402


def run(M, N, K, relu, bias, ldpad=0):
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    x = torch.randn(M, K + ldpad, device="cuda", generator=g)[:, :K] * 0.7
    dy = torch.randn(M, N, device="cuda", generator=g) * 0.3
    y = torch.randn(M, N, device="cuda", generator=g) if relu else None
    L = _lib.load()
    dW = torch.empty(N, K, device="cuda")
    db = torch.empty(N, device="cuda") if bias else None
    ws = torch.empty(L.b2r_linear_bwd_weight_tc_workspace_bytes(M, N, K), dtype=torch.uint8, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    ldx = x.stride(0)

    def tc():
        _lib.check(L.b2r_linear_bwd_weight_tc(dy.data_ptr(), N, y.data_ptr() if relu else None, x.data_ptr(), ldx, dW.data_ptr(),
                                              db.data_ptr() if bias else None, M, N, K, ws.data_ptr(), ws.numel(), st), "dw_tc")
    tc()
    torch.cuda.synchronize()
    dym = dy.double() * ((y > 0).double() if relu else 1.0)
    ref = dym.t() @ x.double()
    scale = float(ref.abs().max())
    err = float((dW.double() - ref).abs().max()) / scale
    berr = float((db.double() - dym.sum(0)).abs().max()) / float(dym.sum(0).abs().max()) if bias else 0.0
    # CUDA-core kernel on the same problem
    dW2 = torch.empty_like(dW)
    db2 = torch.empty(N, device="cuda") if bias else None
    ws2 = torch.empty(max(16, L.b2r_linear_bwd_weight_workspace_bytes(M, N, K)), dtype=torch.uint8, device="cuda")

    def cc():
        _lib.check(L.b2r_linear_bwd_weight(dy.data_ptr(), N, y.data_ptr() if relu else None, x.data_ptr(), ldx, dW2.data_ptr(),
                                           db2.data_ptr() if bias else None, M, N, K, ws2.data_ptr(), ws2.numel(), st), "dw")
    cc()
    err2 = float((dW2.double() - ref).abs().max()) / scale
    tc(); dW_a = dW.clone(); tc()
    assert torch.equal(dW, dW_a), "tensor-core dW not bit-reproducible"

    def timeit(fn):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(20):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / 20 * 1e3
    print(f"M={M} N={N} K={K} relu={relu} bias={bias}: tc rel err {err:.2e} (bias {berr:.2e}), cuda-core rel err {err2:.2e}; "
          f"tc {timeit(tc):.1f} us, cuda-core {timeit(cc):.1f} us", flush=True)
    # the tensor core accumulates in fp32 with its own rounding: ~6e-6 of the largest entry over 204,800 rows (north-star
    # bar for gradients: 1e-5)
    assert err <= 1e-5 and berr <= 1e-5, (err, berr)


if __name__ == "__main__":
    run(204800, 64, 64, False, True)
    run(204800, 64, 64, True, True)
    run(20480, 32, 64, True, True)
    run(20481, 16, 32, False, False)         # ragged tail, narrow
    run(20480, 64, 128, False, True, ldpad=64)   # wide input read from a column block of a wider matrix
    run(5000, 128, 64, False, True)
    run(20480, 64, 192, True, True)          # K > 143: the widest (n = 256) accumulator
    ops.check_ids()
    print("tc dw ok")
