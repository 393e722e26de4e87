#!/bin/bash
# On an H100: for every build/variants/libb200pose_<name>.so a parity subset and one bench line.
# Usage: bash tools/run_variants.sh [name ...]      (results: build/variants/<name>.{json,log})
mkdir -p build/variants
names="$@"
[ -z "$names" ] && names=$(ls build/variants/libb200pose_*.so | sed 's/.*libb200pose_\(.*\)\.so/\1/')
for v in $names; do
  lib=$PWD/build/variants/libb200pose_$v.so
  [ -f "$lib" ] || { echo "$v: missing $lib"; continue; }
  B200POSE_LIB=$lib timeout 300 python -m pytest tests/test_gpu.py -x -q -m gpu \
      -k "post_kernels or net_368 or batch_rows or fused_engine" > build/variants/$v.log 2>&1
  echo "$v parity rc=$? $(tail -1 build/variants/$v.log)"
  B200POSE_LIB=$lib timeout 200 python bench.py --steps 20 --warmup 5 --no-cpu-baseline \
      > build/variants/$v.json 2>> build/variants/$v.log
done
python tools/variants.py report
