#define TB200_INST_D 15
#define TB200_INST_PAIR 0
#define TB200_INST_SING 1
#include "solve_inst.cuh"
