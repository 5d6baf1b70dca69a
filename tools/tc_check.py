#!/usr/bin/env python
"""Check + time b2r_linear_fwd_tc (wgmma TF32 hi/lo-split Linear) against fp64 and against the CUDA-core SGEMM.
Run in its own process (a descriptor mistake faults the kernel and poisons the CUDA context)."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from rechorus_b200 import ops  # noqa: E402


def main():
    torch.manual_seed(0)
    out = []
    worst = 0.0
    for (M, K, N, relu, bias) in [(128, 64, 64, False, True), (300, 64, 64, True, True), (1000, 32, 16, False, False),
                                  (4096 * 50, 64, 64, False, True), (20480, 128, 64, True, True), (5000, 64, 192, False, True),
                                  (777, 96, 32, True, True), (8192, 64, 256, True, True)]:
        x = (torch.randn(M, K) * 2).cuda()
        W = torch.randn(N, K).cuda()
        b = torch.randn(N).cuda() if bias else None
        ref = x.double() @ W.double().t()
        if bias:
            ref = ref + b.double()
        if relu:
            ref = ref.relu()
        y = ops.linear_fwd_tc(x, W, b, relu)
        torch.cuda.synchronize()
        scale = float(ref.abs().max())
        err = float((y.double() - ref).abs().max()) / scale
        y2 = ops.linear_fwd(x, W, b, relu)
        err2 = float((y2.double() - ref).abs().max()) / scale
        # timing
        def t(fn):
            for _ in range(3):
                fn()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(10):
                fn()
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / 10
        ms_tc = t(lambda: ops.linear_fwd_tc(x, W, b, relu))
        ms_cc = t(lambda: ops.linear_fwd(x, W, b, relu))
        gb = (M * K + M * N) * 4 / 1e9
        out.append(dict(M=M, K=K, N=N, rel_err_tc=err, rel_err_fma=err2, ms_tc=round(ms_tc, 4), ms_fma=round(ms_cc, 4),
                        GBps_tc=round(gb / ms_tc * 1e3, 1), TFLOPs_tc=round(2 * M * N * K / ms_tc / 1e9, 2)))
        worst = max(worst, err)
    # masked form (dX of a ReLU layer): Y = (X o (mask > 0)) W^T through b2r_linear_tc
    from rechorus_b200 import lib as _lib
    L = _lib.load()
    for (M, K, N) in [(300, 64, 64), (5000, 32, 48), (4096 * 50, 64, 64), (1111, 128, 64)]:
        x = torch.randn(M, K).cuda()
        mk = torch.randn(M, K).cuda()
        W = torch.randn(N, K).cuda()
        y = torch.empty(M, N).cuda()
        _lib.check(L.b2r_linear_tc(x.data_ptr(), K, mk.data_ptr(), W.data_ptr(), None, y.data_ptr(), N, M, N, K, 0,
                                   torch.cuda.current_stream().cuda_stream), "b2r_linear_tc")
        ref = (x.double() * (mk > 0)) @ W.double().t()
        err = float((y.double() - ref).abs().max()) / float(ref.abs().max())
        out.append(dict(M=M, K=K, N=N, masked=True, rel_err_tc=err))
        worst = max(worst, err)
    for o in out:
        print(json.dumps(o))
    assert worst <= 2.5e-6, worst   # tensor-core internal accumulation: ~1-2e-6 relative (fp32 FMA path: 2-6e-7)
    print("tc linear ok, worst relative error %.2e" % worst)


if __name__ == "__main__":
    main()
