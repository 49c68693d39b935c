#define TB200_INST_D 4
#include "eval_inst.cuh"
