// slu_scalar.cuh -- element arithmetic of val_t shared by the kernels of both precisions (slu_kernels_z.cu and
// slu_solve.cu / slu_solve_z.cu).  The doublecomplex helpers (z*) work on the reference's (re, im) pairs; the val_t
// helpers (v*) let one kernel source serve both builds: in the double build each is exactly the double expression it
// stands for, so the real kernels compile to the same instructions as when written out.  Compiled into namespace
// SLU_NS (slu_device.cuh).
#pragma once
#include "slu_device.cuh"

namespace SLU_NS {

#ifdef SLU_COMPLEX
typedef double2 zd;
__device__ __forceinline__ zd zmake(double r, double i) { return make_double2(r, i); }
__device__ __forceinline__ zd zmul(zd a, zd b) { return zmake(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }
__device__ __forceinline__ void zsubmul(zd &acc, zd a, zd b)  // acc -= a * b
{
    acc.x -= a.x * b.x - a.y * b.y;
    acc.y -= a.x * b.y + a.y * b.x;
}
__device__ __forceinline__ void zaddmul(zd &acc, zd a, zd b)  // acc += a * b
{
    acc.x += a.x * b.x - a.y * b.y;
    acc.y += a.x * b.y + a.y * b.x;
}
__device__ __forceinline__ bool zzero(zd a) { return a.x == 0.0 && a.y == 0.0; }
// 1 / a by Smith's scaling (no overflow of |a|^2); the reference's slud_z_div(&t, &one, &a), dcomplex.c
__device__ __forceinline__ zd zrecip(zd a)
{
    if (fabs(a.x) >= fabs(a.y)) {
        const double r = a.y / a.x, den = a.x + a.y * r;
        return zmake(1.0 / den, -r / den);
    }
    const double r = a.x / a.y, den = a.y + a.x * r;
    return zmake(r / den, -1.0 / den);
}

__device__ __forceinline__ val_t vzero() { return zmake(0.0, 0.0); }
__device__ __forceinline__ val_t vadd(val_t a, val_t b) { return zmake(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ val_t vsub(val_t a, val_t b) { return zmake(a.x - b.x, a.y - b.y); }
__device__ __forceinline__ void vaddmul(val_t &acc, val_t a, val_t b) { zaddmul(acc, a, b); }
__device__ __forceinline__ void vsubmul(val_t &acc, val_t a, val_t b) { zsubmul(acc, a, b); }
__device__ __forceinline__ val_t vdiv(val_t a, val_t piv) { return zmul(a, zrecip(piv)); }   // a / piv
__device__ __forceinline__ val_t vshfl(unsigned mask, val_t v, int lane)
{
    return zmake(__shfl_sync(mask, v.x, lane), __shfl_sync(mask, v.y, lane));
}
// *p -= v: there is no double2 atomic; the real and imaginary parts are two independent sums
__device__ __forceinline__ void vatomic_sub(val_t *p, val_t v)
{
    atomicAdd(&p->x, -v.x);
    atomicAdd(&p->y, -v.y);
}
__device__ __forceinline__ val_t vmul(val_t a, val_t b) { return zmul(a, b); }
__device__ __forceinline__ val_t vrecip(val_t a) { return zrecip(a); }
// conj(a) for CONJ = true (the conjugate-transposed solve reads every factor entry conjugated), a otherwise
template <bool CONJ>
__device__ __forceinline__ val_t vconj(val_t a) { return CONJ ? zmake(a.x, -a.y) : a; }
__device__ __forceinline__ val_t vnan() { return zmake(NAN, NAN); }
// acc + a * b and acc - a * b as values (one fused multiply-add each in double)
__device__ __forceinline__ val_t vfma(val_t a, val_t b, val_t acc) { zaddmul(acc, a, b); return acc; }
__device__ __forceinline__ val_t vfnma(val_t a, val_t b, val_t acc) { zsubmul(acc, a, b); return acc; }
#else
__device__ __forceinline__ val_t vzero() { return 0.0; }
__device__ __forceinline__ val_t vadd(val_t a, val_t b) { return a + b; }
__device__ __forceinline__ val_t vsub(val_t a, val_t b) { return a - b; }
__device__ __forceinline__ void vaddmul(val_t &acc, val_t a, val_t b) { acc += a * b; }
__device__ __forceinline__ void vsubmul(val_t &acc, val_t a, val_t b) { acc -= a * b; }
__device__ __forceinline__ val_t vdiv(val_t a, val_t piv) { return a / piv; }
__device__ __forceinline__ val_t vshfl(unsigned mask, val_t v, int lane) { return __shfl_sync(mask, v, lane); }
__device__ __forceinline__ void vatomic_sub(val_t *p, val_t v) { atomicAdd(p, -v); }
__device__ __forceinline__ val_t vmul(val_t a, val_t b) { return a * b; }
__device__ __forceinline__ val_t vrecip(val_t a) { return 1.0 / a; }
template <bool CONJ>
__device__ __forceinline__ val_t vconj(val_t a) { return a; }   // a real entry is its own conjugate
__device__ __forceinline__ val_t vnan() { return NAN; }
__device__ __forceinline__ val_t vfma(val_t a, val_t b, val_t acc) { return fma(a, b, acc); }
__device__ __forceinline__ val_t vfnma(val_t a, val_t b, val_t acc) { return fma(-a, b, acc); }
#endif

}  // namespace SLU_NS
