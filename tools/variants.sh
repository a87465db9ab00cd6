#!/bin/bash
# Kernel variants side by side on ONE box (compile-time switches of binder_b200/csrc):
#   tools/variants.sh build            here (no GPU): builds binder_b200/variants/lib_<name>.so for every variant
#   tools/variants.sh run              on the GPU box: for each variant - quick parity subset, bench (value, serial,
#                                      graph-replay launch time), 1M-batch span; the default build first and last
# Variants: "base" (default flags), "mb8" (-DBB_MIN_BLOCKS=8: 64 registers).  Add a line to VARIANTS to try another define.
set -u
cd "$(dirname "$0")/.."
VARIANTS=("base:" "mb8:-DBB_MIN_BLOCKS=8")
FLAGS="-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC,-Wall,-Wno-unused-function -shared -cudart static"
SRCS="binder_b200/csrc/engine.cu binder_b200/csrc/zone_build.cpp binder_b200/csrc/balancer_frames.cpp"
case "${1:-}" in
build)
    mkdir -p binder_b200/variants
    for v in "${VARIANTS[@]}"; do
        name="${v%%:*}"; defs="${v#*:}"
        echo "== $name ($defs)"
        /usr/local/cuda/bin/nvcc $FLAGS $defs -Xptxas -v -o binder_b200/variants/lib_$name.so $SRCS 2>&1 | grep -E "resolve_kernelILb0ELb0|spill" | paste - - | grep -A0 "ILb0ELb0" | head -2
    done ;;
run)
    cp binder_b200/libbinder_b200.so /tmp/lib_default.so
    bench() { timeout 300 python bench.py --no-cpu --no-e2e --steps 8000 > gpurun_out/v.json 2> gpurun_out/v.err; python -c "
import json,sys; d=json.load(open('gpurun_out/v.json')); print(sys.argv[1], 'value Gq/s', round(d['value']/1e9,2), 'serial us', round(d['config']['serial_ms_per_step']*1e3,2), 'graph us', round(d['config']['graph_replay_ms_per_step']*1e3,2), 'frac', round(d['roofline']['frac'],3))" "$1" || tail -3 gpurun_out/v.err; }
    for v in "${VARIANTS[@]}" "base:"; do
        name="${v%%:*}"
        cp binder_b200/variants/lib_$name.so binder_b200/libbinder_b200.so
        timeout 300 python -m pytest tests/test_gpu_parity.py -x -q -m gpu 2>&1 | tail -1
        bench "$name"
        python tools/stage_times.py 1048576 2>&1 | grep "kernel span" | tail -1
    done
    cp /tmp/lib_default.so binder_b200/libbinder_b200.so ;;
*) echo "usage: tools/variants.sh build|run" ;;
esac
