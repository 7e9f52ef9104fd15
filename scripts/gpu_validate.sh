#!/bin/bash
# Validation on one H100: smoke, the whole GPU test suite, the default bench line.
cd ${GRAFT_REPO_ROOT:-.}
mkdir -p gpurun_out
timeout 300 python __graft_entry__.py smoke 2>&1 | tail -3
timeout 1500 python -m pytest tests/ -x -q -m gpu 2>&1 | tail -4
timeout 1500 python bench.py > gpurun_out/bench_final.json 2> gpurun_out/bench_final.err; tail -2 gpurun_out/bench_final.err; grep '^{' gpurun_out/bench_final.json | cut -c1-400
