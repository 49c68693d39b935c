#define TB200_INST_D 2
#include "eval_inst.cuh"
