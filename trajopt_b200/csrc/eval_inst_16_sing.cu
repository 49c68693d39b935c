#define TB200_INST_D 16
#define TB200_INST_SING 1
#include "eval_inst.cuh"
