#define TB200_INST_D 5
#include "eval_inst.cuh"
