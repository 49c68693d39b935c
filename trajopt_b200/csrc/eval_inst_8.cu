#define TB200_INST_D 8
#include "eval_inst.cuh"
