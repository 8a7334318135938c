#!/bin/bash
# first GPU call of round 2: parity of the new window path / per-frame fallback, then stage timings of the variants
mkdir -p gpurun_out
python -m pytest tests/test_gpu_pf.py -x -q -m gpu 2>&1 | tail -15 > gpurun_out/r2a_pytest_pf.log
cat gpurun_out/r2a_pytest_pf.log
{
python tools/r2_stages.py --win2 0
python tools/r2_stages.py --win2 1
python tools/r2_stages.py --win2 1 --mixed 5
python tools/r2_stages.py --win2 1 --frames 64
} 2>&1 | tee gpurun_out/r2a_stages.log
python -m pytest tests -x -q -m gpu 2>&1 | tail -8 | tee gpurun_out/r2a_pytest_all.log
