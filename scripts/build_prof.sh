#!/bin/bash
# Builds trajopt_b200/csrc/libtb200_prof.so: the product library with the phase counters (TB200_PROFILE) compiled into
# the 7-joint instances of the persistent SQP kernel and the cycle stamps (TB200_EVAL_PROFILE) into the 7-joint instance
# of the evaluation kernel.  Used by scripts/prof_phases.py and scripts/eval_phases.py through TB200_LIB=<path>.
set -e
cd "$(dirname "$0")/../trajopt_b200/csrc"
FLAGS="-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -ccbin /usr/bin/g++"
nvcc $FLAGS -DTB200_PROFILE $PROF_EXTRA -c -o solve_inst_7_0.prof.o solve_inst_7_0.cu &
nvcc $FLAGS -DTB200_PROFILE -c -o solve_inst_7_1.prof.o solve_inst_7_1.cu &
nvcc $FLAGS -DTB200_EVAL_PROFILE -c -o eval_inst_7.prof.o eval_inst_7.cu &
wait
OBJS=$(ls *.o | grep -v '\.prof\.o$' | grep -v '^solve_inst_7_[01]\.o$' | grep -v '^eval_inst_7\.o$')
nvcc -shared -gencode arch=compute_90a,code=sm_90a -ccbin /usr/bin/g++ -o libtb200_prof.so $OBJS solve_inst_7_0.prof.o solve_inst_7_1.prof.o eval_inst_7.prof.o
rm -f solve_inst_7_0.prof.o solve_inst_7_1.prof.o eval_inst_7.prof.o
echo built libtb200_prof.so
