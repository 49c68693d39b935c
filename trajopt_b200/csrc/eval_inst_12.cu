#define TB200_INST_D 12
#include "eval_inst.cuh"
