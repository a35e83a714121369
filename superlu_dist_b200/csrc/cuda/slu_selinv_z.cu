// slu_selinv_z.cu -- the doublecomplex build of the selected-inversion kernels: slu_selinv.cu compiled with SLU_COMPLEX,
// launched by slu_b200_z_selinv / slu_b200_z_selinv_get / slu_b200_z_logdet.
#define SLU_COMPLEX 1
#include "slu_selinv.cu"
