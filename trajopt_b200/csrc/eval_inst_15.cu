#define TB200_INST_D 15
#include "eval_inst.cuh"
