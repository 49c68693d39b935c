#define TB200_INST_D 10
#include "eval_inst.cuh"
