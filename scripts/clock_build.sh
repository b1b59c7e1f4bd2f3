#!/bin/bash
# builds boxmot_b200/libboxmot_b200_clocks.so: the product library with -DBMB_TC_CLOCKS (in-kernel clock64 phase prints of
# the tensor-core ReID kernels).  On the GPU box: cp it over libboxmot_b200.so and run scripts/tc_clock_run.py.
set -e
cd "$(dirname "$0")/.."
python -m boxmot_b200.build >/dev/null
F="-gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC,-fvisibility=hidden"
nvcc $F -DBMB_TC_CLOCKS -c boxmot_b200/csrc/reid_model.cu -o /tmp/reid_model_clocks.o
nvcc $F -shared -o boxmot_b200/libboxmot_b200_clocks.so boxmot_b200/csrc/_obj/tracker_engine.o boxmot_b200/csrc/_obj/ss_kernels.o boxmot_b200/csrc/_obj/capi.o /tmp/reid_model_clocks.o -lcudart
ls -la boxmot_b200/libboxmot_b200_clocks.so
