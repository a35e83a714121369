// slu_solve_z.cu -- the doublecomplex build of the triangular solves and the device-side distribution: slu_solve.cu
// compiled with SLU_COMPLEX (pzgstrs3d, SRC/complex16/pzgstrs3d.c), launched by slu_b200_z_solve / slu_b200_z_fill_csr.
#define SLU_COMPLEX 1
#include "slu_solve.cu"
