// slu_schur_z.cu -- the doublecomplex build of the Schur-complement gather: slu_schur.cu compiled with SLU_COMPLEX,
// launched by slu_b200_z_schur_get.
#define SLU_COMPLEX 1
#include "slu_schur.cu"
