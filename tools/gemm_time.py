"""time the Linear kernels at the SASRec config-4 shape (M = B*L = 204800, N = K = 64): SGEMM (dense.cu) vs the wgmma
kernels (linear_tc.cu, linear_dw_tc.cu), forward / dX / dW"""
import os, sys, subprocess
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
code = r'''
import sys, torch
sys.path.insert(0, %r)
from rechorus_b200 import ops
M, N, K = 204800, 64, 64
g = torch.Generator().manual_seed(1)
x = torch.randn(M, K, generator=g).cuda(); W = (torch.randn(N, K, generator=g) * 0.1).cuda(); b = torch.randn(N, generator=g).cuda()
dy = torch.randn(M, N, generator=g).cuda()
flush = torch.empty(64 << 20, device="cuda")
def t(fn, n=20):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    tot = 0.0
    for _ in range(n):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); torch.cuda.synchronize(); tot += e0.elapsed_time(e1)
    return tot / n * 1e3
y0 = ops.linear_fwd(x, W, b, True)
y1 = ops.linear_fwd_tc(x, W, b, True)
ref = torch.relu(x.double() @ W.double().t() + b.double())
print("fwd  sgemm %%.1f us (err %%.2e)  tc %%.1f us (err %%.2e)" %% (t(lambda: ops.linear_fwd(x, W, b, True)), float((y0 - ref).abs().max() / ref.abs().max()),
      t(lambda: ops.linear_fwd_tc(x, W, b, True)), float((y1 - ref).abs().max() / ref.abs().max())))
for flag in (False, True):
    ops._TC_LINEAR = flag
    dx, _, _ = ops.linear_bwd(dy, x, W, y0, True, False, False)
    refdx = ((dy.double() * (y0 > 0)) @ W.double())
    print("dX   tc=%%s %%.1f us (err %%.2e)" %% (flag, t(lambda: ops.linear_bwd(dy, x, W, y0, True, False, False)), float((dx - refdx).abs().max() / refdx.abs().max())))
for flag in (False, True):
    ops._TC_DW = flag
    print("dW   tc=%%s %%.1f us" %% (flag, t(lambda: ops.linear_bwd(dy, x, W, None, False, True, True))))
''' % ROOT
r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600)
print(r.stdout.strip(), r.stderr.strip()[-800:])
