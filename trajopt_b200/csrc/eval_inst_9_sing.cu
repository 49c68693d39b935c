#define TB200_INST_D 9
#define TB200_INST_SING 1
#include "eval_inst.cuh"
