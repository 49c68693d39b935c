#define TB200_INST_D 14
#include "eval_inst.cuh"
