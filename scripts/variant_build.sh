#!/bin/bash
# scripts/variant_build.sh NAME "-DFOO=... -DBAR=..."  -> boxmot_b200/libboxmot_b200_NAME.so (reid_model.cu rebuilt with the flags)
set -e
cd "$(dirname "$0")/.."
F="-gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC,-fvisibility=hidden"
nvcc $F $2 -c boxmot_b200/csrc/reid_model.cu -o /tmp/reid_model_$1.o 2>/dev/null
nvcc $F -shared -o boxmot_b200/libboxmot_b200_$1.so boxmot_b200/csrc/_obj/tracker_engine.o boxmot_b200/csrc/_obj/ss_kernels.o boxmot_b200/csrc/_obj/capi.o /tmp/reid_model_$1.o -lcudart
echo built $1
