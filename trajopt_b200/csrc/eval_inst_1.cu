#define TB200_INST_D 1
#include "eval_inst.cuh"
