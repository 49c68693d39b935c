#define TB200_INST_D 4
#define TB200_INST_SING 1
#include "eval_inst.cuh"
