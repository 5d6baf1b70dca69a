"""diagnostic: which configuration invalidates the CUDA-graph capture of the contract-route step?"""
import os, sys, subprocess
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
code = r'''
import sys, os
sys.path.insert(0, %r)
import torch, bench
from rechorus_b200.graph import GraphedStep
w = dict(bench.WORKLOADS[sys.argv[1]])
if len(sys.argv) > 2: w["B"] = int(sys.argv[2])
dev = torch.device("cuda", 0)
model, _ = bench.build_model(w, dev)
feeds = [bench.to_feed(f, dev, w["B"]) for f in bench.make_batches(w, seed=1, pool=2)]
if os.environ.get("EAGER_FIRST"):
    for f in feeds:
        model.optimizer.zero_grad(); model.loss(model(f)).backward(); model.optimizer.step()
try:
    g = GraphedStep(model, feeds[0], warmup=2)
    l = g(feeds[1]); torch.cuda.synchronize()
    print("OK", sys.argv[1:], float(l))
except Exception as e:
    import traceback; traceback.print_exc()
    print("FAIL", sys.argv[1:], repr(e)[:300])
''' % ROOT
for env, argv in (({"EAGER_FIRST": "1"}, ["c3"]), ({"EAGER_FIRST": "1"}, ["c4"]), ({"B2R_TC_DW": "0"}, ["c3"]), ({}, ["c3"]), ({}, ["c3", "512"]),
                  ({"B2R_TC_DW": "0"}, ["c4"]), ({}, ["c4"]), ({"B2R_SASREC_LIVE": "0", "B2R_TC_DW": "0"}, ["c4"])):
    if os.environ.get("DIAG_ONLY") and "EAGER_FIRST" not in env:
        continue
    r = subprocess.run([sys.executable, "-c", code] + argv, env=dict(os.environ, **env), capture_output=True, text=True, timeout=600)
    print(env, (r.stdout.strip().splitlines() or ["<no output>"])[-1][:400])
    if "FAIL" in r.stdout or r.returncode != 0:
        print("   stderr tail:", r.stderr.strip()[-3000:].replace("\n", " | "))
