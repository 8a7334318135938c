#!/bin/bash
# second GPU call of round 2: parity, stage timings of the loader variants, ncu captures of the two window kernels
mkdir -p gpurun_out
python -m pytest tests/test_gpu_pf.py -x -q -m gpu 2>&1 | tail -5 > gpurun_out/r2b_pytest_pf.log
cat gpurun_out/r2b_pytest_pf.log
{
python tools/r2_stages.py --win2 0
python tools/r2_stages.py --win2 1
python tools/r2_stages.py --win2 1 --mixed 5
} 2>&1 | tee gpurun_out/r2b_stages.log
timeout 300 ncu --set full --clock-control none --import-source on -k regex:k_pf_win_medians -s 1 -c 1 -o gpurun_out/prof_wmed_r2b -f python tools/prof_pf.py 1 512 > gpurun_out/r2b_ncu1.log 2>&1
timeout 300 ncu --set full --clock-control none --import-source on -k regex:k_pf_win_fwxm -s 1 -c 1 -o gpurun_out/prof_wfwxm_r2b -f python tools/prof_pf.py 1 512 > gpurun_out/r2b_ncu2.log 2>&1
tail -3 gpurun_out/r2b_ncu1.log gpurun_out/r2b_ncu2.log
python -m pytest tests -x -q -m gpu 2>&1 | tail -8 | tee gpurun_out/r2b_pytest_all.log
