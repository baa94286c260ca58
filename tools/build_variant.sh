#!/bin/bash
# Build a kernel variant of libnsb.so with extra nvcc flags for nsb_field.cu (A/B runs: NSB_LIB=tools/_variants/NAME.so).
# usage: tools/build_variant.sh NAME "-DNSB_FOO=1 ..."        (tools/_variants/ is git-ignored)
set -e
cd "$(dirname "$0")/../nersemble_b200/csrc"
NAME=$1; FLAGS=$2
OUT=../../tools/_variants
mkdir -p $OUT
/usr/local/cuda/bin/nvcc -O3 -std=c++17 -lineinfo -Xcompiler -fPIC -I../../include -gencode arch=compute_90a,code=sm_90a -Xptxas -v \
    $FLAGS -c nsb_field.cu -o $OUT/$NAME.field.o 2> $OUT/$NAME.ptxas.log || (cat $OUT/$NAME.ptxas.log; false)
/usr/local/cuda/bin/nvcc -shared -gencode arch=compute_90a,code=sm_90a -o $OUT/$NAME.so $OUT/$NAME.field.o \
    nsb_api.o nsb_render.o nsb_backward.o nsb_deform_bwd.o nsb_optim.o nsb_losses.o nsb_rays.o nsb_normals.o -lcudart
python ../../tools/spill_report.py $OUT/$NAME.field.o kernel_tc
