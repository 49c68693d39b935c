#define TB200_INST_D 16
#include "eval_inst.cuh"
