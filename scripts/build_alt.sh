#!/bin/bash
# Builds trajopt_b200/csrc/libtb200_alt.so: the product library with the 7-joint SQP kernel compiled with extra
# defines (kernel experiments: TB200_LIB=<path> selects it).  usage: scripts/build_alt.sh -DTB200_PROFILE
set -e
cd "$(dirname "$0")/../trajopt_b200/csrc"
FLAGS="-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -ccbin /usr/bin/g++"
nvcc $FLAGS "$@" -c -o solve_inst_7_0.alt.o solve_inst_7_0.cu
OBJS=$(ls *.o | grep -v '\.alt\.o$' | grep -v '\.prof\.o$' | grep -v '^solve_inst_7_0\.o$')
nvcc -shared -gencode arch=compute_90a,code=sm_90a -ccbin /usr/bin/g++ -o libtb200_alt.so $OBJS solve_inst_7_0.alt.o
rm -f solve_inst_7_0.alt.o
echo built libtb200_alt.so "$@"
