#define TB200_INST_D 13
#include "eval_inst.cuh"
