#define TB200_INST_D 9
#include "eval_inst.cuh"
