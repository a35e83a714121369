// slu_grad_z.cu -- the doublecomplex build of the gradient kernels: slu_grad.cu compiled with SLU_COMPLEX (conj(x) in the
// solve gradient, conj(H) in the log-determinant gradient), launched by the slu_b200_z_ gradient calls.
#define SLU_COMPLEX 1
#include "slu_grad.cu"
