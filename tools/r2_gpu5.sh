#!/bin/bash
mkdir -p gpurun_out
python -m pytest tests/test_gpu_pf.py -x -q -m gpu 2>&1 | tail -5 | tee gpurun_out/r2e_pytest_pf.log
{
python tools/r2_stages.py --win2 1
python tools/r2_stages.py --win2 1 --mixed 5
python tools/r2_stages.py --win2 1 --frames 64
} 2>&1 | tee gpurun_out/r2e_stages.log
