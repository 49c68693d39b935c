#define TB200_INST_D 6
#include "eval_inst.cuh"
