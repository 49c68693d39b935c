#define TB200_INST_D 7
#include "eval_inst.cuh"
