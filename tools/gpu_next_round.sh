#!/bin/bash
# First GPU call of the next round: validate and A/B the candidates that were written without a GPU (DESIGN.md §8).
#   B2R_NEXT bit 0 = counting-sort k_bucket_sort, bit 1 = warp-per-sample fused kernel (d=64, C<=104).
# For each setting: the parity tests that exercise the changed kernel, then the bench line; then ncu times alone.
mkdir -p gpurun_out
B2R_NEXT=0 timeout 600 python -m pytest tests/test_gpu_zz_fit_golden.py -q > gpurun_out/n_pytest_zz.log 2>&1; echo "zz tests (default kernels) rc=$?"; tail -3 gpurun_out/n_pytest_zz.log
B2R_NEXT=0 timeout 300 python -m pytest tests/test_gpu_zz_next_round.py -q > gpurun_out/n_pytest_next.log 2>&1; echo "next-round groundwork tests rc=$?"; tail -3 gpurun_out/n_pytest_next.log
for NX in 0 1 2 3; do
  B2R_NEXT=$NX timeout 600 python -m pytest tests/test_gpu_bprmf.py tests/test_gpu_fullsize.py tests/test_gpu_shard.py tests/test_gpu_runner_fit.py -x -q > gpurun_out/n_pytest_$NX.log 2>&1
  echo "B2R_NEXT=$NX pytest rc=$? $(tail -1 gpurun_out/n_pytest_$NX.log)"
  B2R_NEXT=$NX timeout 300 python bench.py --steps 1000 --warmup 20 --no_cpu_baseline > gpurun_out/n_bench_$NX.json 2> gpurun_out/n_bench_$NX.err
  tail -1 gpurun_out/n_bench_$NX.json | python -c "
import sys,json; d=json.loads(sys.stdin.read()); print('B2R_NEXT=$NX: ms %.4f e2e %.4f apply %.4f plan %.4f fused %.4f'%(d['ms_per_step'], d['e2e']['ms_per_step'], d['roofline']['kernel_ms'], d['kernels']['plan_items']['ms'], d['kernels']['fused_score_loss_bwd']['ms']))"
done
B2R_NEXT=3 timeout 300 ncu --metrics gpu__time_duration.sum --clock-control none -s 100 -c 200 --csv --log-file gpurun_out/n_launches_3.csv \
    python bench.py --steps 12 --warmup 8 --no_cpu_baseline > /dev/null 2>&1
python - <<'PY'
import csv,collections
rows=[r for r in csv.reader(open('gpurun_out/n_launches_3.csv')) if len(r)>10]
hdr=rows[0]; ki=hdr.index('Kernel Name'); vi=hdr.index('Metric Value')
agg=collections.OrderedDict()
for r in rows[1:]:
    try: agg.setdefault(r[ki][:60],[]).append(float(r[vi].replace(',','')))
    except: pass
for k,v in agg.items(): print(f"  n={len(v):3d} avg={sum(v)/len(v)/1000:8.2f} us  {k}")
PY
# SASRec / NeuMF with every Linear forward on the tcgen05 kernel: parity, step time, tensor-pipe activity
B2R_TC_LINEAR=1 timeout 600 python -m pytest tests/test_gpu_models.py tests/test_gpu_dense.py -x -q > gpurun_out/n_pytest_tc.log 2>&1; echo "B2R_TC_LINEAR=1 pytest rc=$? $(tail -1 gpurun_out/n_pytest_tc.log)"
B2R_TC_LINEAR=1 timeout 400 python tools/model_bench.py 2>/dev/null | grep -E '^\{' | cut -c1-200
timeout 400 ncu --metrics gpu__time_duration.sum,sm__inst_executed_pipe_tensor.sum,sm__pipe_tensor_op_umma_cycles_active.avg.pct_of_peak_sustained_active --clock-control none -k regex:k_linear_fwd_tc -c 6 --csv --log-file gpurun_out/n_tc_pipe.csv env B2R_TC_LINEAR=1 python tools/model_bench.py > /dev/null 2>&1; tail -8 gpurun_out/n_tc_pipe.csv | cut -d, -f5,13-
# SASRec with the last block computed for one query per sequence (exact; DESIGN.md §8): parity on the fixtures, step time
B2R_SASREC_LASTQ=1 timeout 600 python -m pytest tests/test_gpu_models.py tests/test_gpu_fullsize.py -x -q > gpurun_out/n_pytest_lastq.log 2>&1; echo "B2R_SASREC_LASTQ=1 pytest rc=$? $(tail -1 gpurun_out/n_pytest_lastq.log)"
B2R_SASREC_LASTQ=1 timeout 400 python tools/model_bench.py 2>/dev/null | grep -E '^\{' | grep -i sasrec | cut -c1-200
# Multi-GPU candidate (separate call, charged 2x):  gpurun --gpus 2 -- 'B2R_SHARD_P2P=1 bash tools/gpu_shard.sh 2 nobench'
# -> the --check line must stay <= 1e-5 / update_ok, then compare the c5 ms_per_step with the NCCL-only run.
