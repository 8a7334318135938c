#!/bin/bash
mkdir -p gpurun_out
python -m pytest tests/test_gpu_pf.py -x -q -m gpu 2>&1 | tail -5 | tee gpurun_out/r2d_pytest_pf.log
{
python tools/r2_stages.py --win2 1
python tools/r2_stages.py --win2 1 --mixed 5
} 2>&1 | tee gpurun_out/r2d_stages.log
timeout 300 ncu --set full --clock-control none --import-source on -k regex:k_pf_win_medians -s 1 -c 1 -o gpurun_out/prof_wmed_r2d -f python tools/prof_pf.py 1 512 > gpurun_out/r2d_ncu1.log 2>&1
timeout 300 ncu --set full --clock-control none --import-source on -k regex:"k_pf_tail|k_pf_finalize|k_pf_pilot" -s 3 -c 3 -o gpurun_out/prof_lat_r2d -f python tools/prof_pf.py 1 512 > gpurun_out/r2d_ncu2.log 2>&1
tail -n 2 gpurun_out/r2d_ncu1.log gpurun_out/r2d_ncu2.log
