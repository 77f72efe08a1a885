#!/bin/bash
# A/B timing pass: tools/prof_pv.py for the given kinds with the product library and every
# experiment build under build_variants/ (tools/build_variants.sh), two rounds.
#   tools/gpu_r2_ab.sh TAG "wind pv" "small big"
TAG=${1:-r2ab}; KINDS=${2:-wind}; SIZES=${3:-small big}
mkdir -p gpurun_out
nvidia-smi --query-gpu=clocks.sm,clocks.max.sm,power.draw,temperature.gpu --format=csv > gpurun_out/gpu_$TAG.txt
for rep in 1 2; do
for lib in default build_variants/*.so; do for k in $KINDS; do for s in $SIZES; do
  if [ $lib = default ]; then timeout 120 python tools/prof_pv.py $k $s 9
  else ATL_LIB_PATH=$lib timeout 120 python tools/prof_pv.py $k $s 9; fi
done; done; done
if [ -n "$ATL_AB_ENV" ]; then for k in $KINDS; do for s in $SIZES; do env $ATL_AB_ENV timeout 120 python tools/prof_pv.py $k $s 9 | sed "s/\"lib\": \"default\"/\"lib\": \"default $ATL_AB_ENV\"/"; done; done; fi
done > gpurun_out/prof_$TAG.jsonl 2>gpurun_out/prof_$TAG.err
python - <<PY
import json
for l in open("gpurun_out/prof_$TAG.jsonl"):
    j=json.loads(l); print(j["lib"][:34].ljust(34), j["kind"], j["size"].ljust(6), j["ms"], j["frac_of_hbm_peak"])
PY
tail -3 gpurun_out/prof_$TAG.err
