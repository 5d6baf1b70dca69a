"""Where the time of the c2 training step goes (BPRMF d=64, 1M x 1M, B=4096, K=99), measured on the GPU it runs on.

    python tools/c2_breakdown.py [--steps 400] [--json OUT] [--rmw build/rmw_bench]

Reports, next to the card name and its power limit (both are part of every number):
  step_ms        steady-state step: model.train_step(feed, next_feed) as bench.py times it, the next batch's index plan
                 built on the library's side stream underneath the step;
  in_step        the tagged kernels inside those steps (b2r_profile_arm brackets: flash, apply, the whole plan), and
                 every kernel's mean device time from torch.profiler;
  alone          flash and apply with nothing else on the GPU: a step whose plan was prefetched by the step before and
                 that prefetches nothing itself, after a synchronize; the plan alone: b2r_direct_plan_build for the
                 item and the user table (single-table launches; the step carries both tables in one launch);
  rmw            the ceiling of the apply's row read-modify-write traffic (tools/rmw_bench.cu), when built;
  sweep          (--sweep) the steady-state step at each plan grid size (CTAs per plan launch, 0 = sized to the work)
                 and side-stream priority (b2r_bprmf_ctx_plan_launch), best of --sweep_reps runs each.
step_over_flash_plus_apply_pct = (step_ms - flash alone - apply alone) / (flash alone + apply alone): what the step
loses to running the plan underneath its kernels (and to the gaps between them).  alone_ms.step is that no-plan step
timed from an idle GPU, launch latency included: not comparable with step_ms.
"""
import argparse
import collections
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def card():
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm,clocks.max.mem",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        out["power_limit"], out["max_sm_clock"], out["max_mem_clock"] = [x.strip() for x in q.split(",")]
    except Exception as e:                                  # the numbers stay usable, the card line says why it is short
        out["power_limit"] = f"unknown ({e})"
    return out


def mean_events(pairs):
    return statistics.mean(a.elapsed_time(b) for a, b in pairs)


def kernel_table(prof, n_steps):
    """mean device microseconds per step and launches per step of every kernel in the capture"""
    tot, cnt = collections.defaultdict(float), collections.defaultdict(int)
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and e.device_time_total > 0:
            name = e.name.split("(")[0].replace("void ", "")
            tot[name] += e.device_time_total
            cnt[name] += 1
    return {k: {"us_per_step": round(tot[k] / n_steps, 2), "launches_per_step": round(cnt[k] / n_steps, 2)}
            for k in sorted(tot, key=lambda k: -tot[k])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=400)
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--json", default=None)
    ap.add_argument("--rmw", default=os.path.join(ROOT, "build", "rmw_bench"))
    ap.add_argument("--sweep", action="store_true")
    ap.add_argument("--sweep_ctas", default="0,33,66,132,264,528")
    ap.add_argument("--sweep_reps", type=int, default=3)
    a = ap.parse_args()

    import bench
    from rechorus_b200 import lib as L, ops
    dev = torch.device("cuda", 0)
    w = bench.WORKLOADS["c2"]
    B = w["B"]
    model, _ = bench.build_model(w, dev)
    lib = L.load()
    feeds = [bench.to_feed(f, dev, B) for f in bench.make_batches(w, seed=1000)]
    P = len(feeds)
    res = {"card": card(), "workload": "c2", "steps": a.steps}

    def step(k, prefetch=True):
        return model.train_step(feeds[k % P], feeds[(k + 1) % P] if prefetch else None)

    ev = lambda: (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))   # noqa: E731

    # ---- steady state, as bench.py times it -------------------------------------------------------------------
    for k in range(a.warmup):
        step(k)
    torch.cuda.synchronize()
    t0, t1 = ev()
    t0.record()
    for k in range(a.steps):
        step(k)
    t1.record()
    torch.cuda.synchronize()
    res["step_ms"] = t0.elapsed_time(t1) / a.steps

    # ---- the tagged kernels inside the steady-state step ------------------------------------------------------
    tags = {"flash": L.PROF_SCORE_FWD, "apply": L.PROF_SEGMENT_I, "plan": L.PROF_PLAN_I}
    samples = {name: [] for name in tags}
    for k in range(a.steps):
        if k % 4 == 0:
            for name, tag in tags.items():
                e = ev()
                e[0].record(); e[1].record()                # created before the library records into them
                samples[name].append(e)
                lib.b2r_profile_arm(tag, e[0].cuda_event, e[1].cuda_event)
        step(k)
    torch.cuda.synchronize()
    for tag in tags.values():
        lib.b2r_profile_arm(tag, None, None)
    res["in_step_ms"] = {name: mean_events(samples[name]) for name in tags}

    n_prof = 40
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for k in range(n_prof):
            step(k)
        torch.cuda.synchronize()
    res["in_step_kernels"] = kernel_table(prof, n_prof)

    # ---- alone: flash + apply of a step whose plan was prefetched, nothing else running ----------------------
    alone = {"flash": [], "apply": [], "step": []}
    for k in range(0, 2 * 64, 2):
        step(k)                                             # builds plan(k + 1) ...
        torch.cuda.synchronize()                            # ... and lets it finish
        ef, ea, es = ev(), ev(), ev()
        for e in (ef, ea):
            e[0].record(); e[1].record()
        torch.cuda.synchronize()
        lib.b2r_profile_arm(L.PROF_SCORE_FWD, ef[0].cuda_event, ef[1].cuda_event)
        lib.b2r_profile_arm(L.PROF_SEGMENT_I, ea[0].cuda_event, ea[1].cuda_event)
        es[0].record()
        step(k + 1, prefetch=False)                         # no plan work in this step
        es[1].record()
        torch.cuda.synchronize()
        alone["flash"].append(ef); alone["apply"].append(ea); alone["step"].append(es)
    lib.b2r_profile_arm(L.PROF_SCORE_FWD, None, None)
    lib.b2r_profile_arm(L.PROF_SEGMENT_I, None, None)
    res["alone_ms"] = {name: mean_events(v) for name, v in alone.items()}

    # ---- the plan alone (both tables, one build each) ---------------------------------------------------------
    ops.bprmf_step_reset()
    n_i, n_u = w["n_items"], w["n_users"]
    plans = []
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for k in range(32):
            f = feeds[k % P]
            plans.append(ops.DirectPlan(f["item_id"], n_i))
            plans.append(ops.DirectPlan(f["user_id"], n_u))
            torch.cuda.synchronize()
    res["plan_alone_kernels"] = kernel_table(prof, 32)
    es = []
    for k in range(32):
        f = feeds[k % P]
        e = ev()
        e[0].record()
        ops.DirectPlan(f["item_id"], n_i)
        ops.DirectPlan(f["user_id"], n_u)
        e[1].record()
        torch.cuda.synchronize()
        es.append(e)
    res["alone_ms"]["plan_both_tables"] = mean_events(es)

    if a.sweep:
        if not hasattr(lib, "b2r_bprmf_ctx_plan_launch"):
            res["sweep"] = "this build has no b2r_bprmf_ctx_plan_launch"
        else:
            (ctx,) = list(ops._step_ctx.values())
            sweep = {}
            for high in (1, 0):
                for ctas in [int(x) for x in a.sweep_ctas.split(",")]:
                    L.check(lib.b2r_bprmf_ctx_plan_launch(ctx.handle, ctas, high), "b2r_bprmf_ctx_plan_launch")
                    best = None
                    for _ in range(a.sweep_reps):
                        for k in range(20):
                            step(k)
                        t0, t1 = ev()
                        t0.record()
                        for k in range(a.steps):
                            step(k)
                        t1.record()
                        torch.cuda.synchronize()
                        ms = t0.elapsed_time(t1) / a.steps
                        best = ms if best is None else min(best, ms)
                    sweep[f"{'high' if high else 'default'}_prio ctas={ctas}"] = round(best, 5)
            res["sweep_step_ms"] = sweep
            ops.bprmf_step_reset()

    fa = res["alone_ms"]["flash"] + res["alone_ms"]["apply"]
    res["flash_plus_apply_alone_ms"] = fa
    res["step_over_flash_plus_apply_pct"] = 100.0 * (res["step_ms"] - fa) / fa

    if os.path.exists(a.rmw):
        res["rmw"] = subprocess.run([a.rmw], capture_output=True, text=True, timeout=300).stdout.strip().splitlines()

    ops.check_ids(dev)
    print(json.dumps(res, indent=1))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
