#define TB200_INST_D 11
#include "eval_inst.cuh"
