#!/bin/bash
# quick TSDF-only loop: parity tests + bench (no CPU arm, no seg, no ncu)
TAG=${1:-q}
OUT=gpurun_out; mkdir -p $OUT
timeout 600 python -m pytest tests/test_tsdf_gpu.py -x -q 2>&1 | tail -5
for B in ${BATCHES:-8 16}; do timeout 600 python bench.py --no-cpu --no-seg --batch $B > $OUT/bench_q${B}_$TAG.json 2>$OUT/bench_q${B}_$TAG.err; python -c "
import json,sys; d=json.load(open('$OUT/bench_q${B}_$TAG.json')); r=d['roofline']; print('batch $B value', round(d['value']), 'e2e', round(d['e2e']['value']), 'integ_ms/launch', round(r['avg_launch_ms'],4), 'alloc_total_ms', round(r['alloc_kernel_ms_total'],2), 'integ_total_ms', round(r['integrate_kernel_ms_total'],2), 'ms_per_step', round(d['ms_per_step'],3))" || tail -3 $OUT/bench_q${B}_$TAG.err; done
