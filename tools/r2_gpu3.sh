#!/bin/bash
mkdir -p gpurun_out
python -m pytest tests/test_gpu_pf.py tests/test_gpu_metrics.py tests/test_gpu_wl.py -x -q -m gpu 2>&1 | tail -25 > gpurun_out/r2c_pytest_pf.log
cat gpurun_out/r2c_pytest_pf.log
{
python tools/r2_stages.py --win2 1
python tools/r2_stages.py --win2 1 --frames 64
} 2>&1 | tee gpurun_out/r2c_stages.log
timeout 300 ncu --set full --clock-control none --import-source on -k regex:k_pf_win_medians -s 1 -c 1 -o gpurun_out/prof_wmed_r2c -f python tools/prof_pf.py 1 512 > gpurun_out/r2c_ncu1.log 2>&1
timeout 300 ncu --set full --clock-control none --import-source on -k regex:k_pf_win_fwxm -s 1 -c 1 -o gpurun_out/prof_wfwxm_r2c -f python tools/prof_pf.py 1 512 > gpurun_out/r2c_ncu2.log 2>&1
tail -n 3 gpurun_out/r2c_ncu1.log gpurun_out/r2c_ncu2.log
python -m pytest tests -x -q -m gpu 2>&1 | tail -8 | tee gpurun_out/r2c_pytest_all.log
python bench.py --steps 10 --warmup 3 > gpurun_out/r2c_bench.json 2> gpurun_out/r2c_bench.err; tail -c 3000 gpurun_out/r2c_bench.json; tail -5 gpurun_out/r2c_bench.err
python tools/r2_stages.py --win2 1 --mixed 5 | tee -a gpurun_out/r2c_stages.log
