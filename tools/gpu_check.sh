#!/bin/bash
# One GPU: full parity suite, render timings per plane layout (single-pass and importance), sampler, SR accuracy, smoke, default bench.
#   bash tools/gpu_check.sh
mkdir -p gpurun_out
timeout 1200 python -m pytest tests -m gpu -q -rf --timeout 600 2>&1 | tail -30 > gpurun_out/check_pytest.log
timeout 300 python tools/bench_render.py > gpurun_out/check_render.log 2>&1
timeout 300 python tools/bench_render.py --fine 48 > gpurun_out/check_render_fine.log 2>&1
timeout 300 python tools/bench_ops.py --op sample > gpurun_out/check_sample.log 2>&1
timeout 300 python tools/sr_accuracy.py > gpurun_out/check_sr_accuracy.log 2>&1
timeout 600 python __graft_entry__.py smoke > gpurun_out/check_smoke.log 2>&1
timeout 900 python bench.py > gpurun_out/check_bench.json 2> gpurun_out/check_bench.err
tail -8 gpurun_out/check_pytest.log; cat gpurun_out/check_render.log gpurun_out/check_render_fine.log gpurun_out/check_sample.log gpurun_out/check_sr_accuracy.log; tail -3 gpurun_out/check_smoke.log; tail -c 600 gpurun_out/check_bench.err; head -c 600 gpurun_out/check_bench.json
