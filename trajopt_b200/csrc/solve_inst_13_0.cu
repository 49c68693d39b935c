#define TB200_INST_D 13
#define TB200_INST_PAIR 0
#include "solve_inst.cuh"
