#!/bin/bash
mkdir -p gpurun_out
timeout 300 python tools/tc_dw_check.py 2>&1 | tail -12
timeout 900 python -m pytest tests/test_gpu_tc.py tests/test_gpu_dense.py tests/test_gpu_models.py tests/test_gpu_fullsize.py tests/test_gpu_optin_modes.py tests/test_gpu_listwise.py tests/test_gpu_shard.py tests/test_gpu_bprmf.py -q > gpurun_out/r2g_pytest.log 2>&1; echo "pytest rc=$? $(tail -1 gpurun_out/r2g_pytest.log)"
grep -E "^FAILED|^ERROR|^E  " gpurun_out/r2g_pytest.log | head -20
for T in 1 0; do
B2R_TC_DW=$T timeout 600 python bench.py --workload c4 --steps 20 --warmup 3 --no_cpu_baseline 2>/dev/null | tail -1 | python -c "
import sys,json
d=json.loads(sys.stdin.read()); print('c4 TC_DW=$T ms %.4f e2e %.4f loss %s tensor %s'%(d['ms_per_step'], d['e2e']['ms_per_step'], d['final_loss'], d['tensor_roofline']['achieved']))"
done
B2R_TC_DW=1 timeout 600 python bench.py --workload c3 --steps 40 --warmup 3 --no_cpu_baseline 2>/dev/null | tail -1 | python -c "
import sys,json
d=json.loads(sys.stdin.read()); print('c3 ms %.4f e2e %.4f'%(d['ms_per_step'], d['e2e']['ms_per_step']))"
timeout 300 ncu --metrics gpu__time_duration.sum,sm__inst_executed_pipe_tensor.sum,sm__pipe_tensor_op_umma_cycles_active.avg.pct_of_peak_sustained_active --clock-control none -k regex:k_linear_dw_tc -c 4 --csv --log-file gpurun_out/r2g_dw_tc_pipe.csv python bench.py --workload c4 --steps 3 --warmup 3 --no_cpu_baseline > /dev/null 2>&1; tail -13 gpurun_out/r2g_dw_tc_pipe.csv | cut -d, -f5,13-
timeout 600 python tools/shard_bench.py --n_items 100000000 --n_users 1000000 --emb 128 --B 4096 --K 255 --steps 20 --warmup 5 2>/dev/null | grep -E "^\{" | cut -c1-160
timeout 300 python bench.py --steps 300 --warmup 10 --no_cpu_baseline --headline_only 2>/dev/null | tail -1 | python -c "
import sys,json
d=json.loads(sys.stdin.read()); print('contract route with direct plan', d['contract_route']['ms_per_step'], 'c2 ms', d['ms_per_step'])"
