#!/bin/bash
mkdir -p gpurun_out
timeout 1500 python -m pytest tests -m gpu -x -q --no-header -p no:cacheprovider 2>&1 | tail -5
timeout 1500 python bench.py --steps 2 --warmup 3 2> gpurun_out/bench.err > gpurun_out/bench.json; tail -2 gpurun_out/bench.err
python - <<PY
import json
d=json.load(open('gpurun_out/bench.json'))
print({k:d[k] for k in ('value','ms_per_step','unet_step_ms','whole_path_tflops','gpu_launches')}, d['roofline'], d['e2e'], d['cpu_baseline'])
PY
for w in main fused; do
timeout 900 ncu --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum --clock-control none --nvtx --nvtx-include "unet_forward/" --csv --log-file gpurun_out/launches_$w.csv python scripts/profile_fused.py $w > gpurun_out/prof_$w.log 2>&1
tail -1 gpurun_out/prof_$w.log
done
# --set full, one launch each: tall-tile GEMM (ff2 at c=1280, 256x160 tiles), the qkv GEMM at c=1280
timeout 600 ncu --set full --import-source on --clock-control none -k regex:gemm_tc --launch-skip 2 --launch-count 1 -o gpurun_out/r01_gemm_tall_ff2 -f python scripts/gemm_one.py 4096 1280 5120 > gpurun_out/ncu_g1.log 2>&1; tail -1 gpurun_out/ncu_g1.log
timeout 600 ncu --set full --import-source on --clock-control none -k regex:gemm_tc --launch-skip 2 --launch-count 1 -o gpurun_out/r01_gemm_pair_qkv -f python scripts/gemm_one.py 4096 3840 1280 > gpurun_out/ncu_g2.log 2>&1; tail -1 gpurun_out/ncu_g2.log
