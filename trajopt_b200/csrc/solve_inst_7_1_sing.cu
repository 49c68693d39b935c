#define TB200_INST_D 7
#define TB200_INST_PAIR 1
#define TB200_INST_SING 1
#include "solve_inst.cuh"
