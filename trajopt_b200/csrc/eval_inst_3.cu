#define TB200_INST_D 3
#include "eval_inst.cuh"
