// slu_cond_z.cu -- the doublecomplex build of the condition-estimation step kernels: slu_cond.cu compiled with SLU_COMPLEX
// (zlacn2), launched by slu_b200_z_gscon / slu_b200_z_batch_gscon.
#define SLU_COMPLEX 1
#include "slu_cond.cu"
