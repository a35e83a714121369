// slu_refine_z.cu -- the doublecomplex build of the iterative-refinement kernels: slu_refine.cu compiled with SLU_COMPLEX
// (pzgsrfs, zgerfs: |.| is cabs1), launched by slu_b200_z_gsrfs / slu_b200_z_batch_gsrfs.
#define SLU_COMPLEX 1
#include "slu_refine.cu"
