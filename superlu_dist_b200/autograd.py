"""torch.autograd through the device-resident factors: differentiable solves and log-determinants of a sparse A(theta) whose
values live in a torch CUDA tensor.

    h = capi.Handle(prob)                        # or capi.BatchHandle(prob, B)
    h.fill_csr_scaled(rp, ci, v0, perm, perm_r, R, C)   # the pattern, the matching and the scalings, once
    f = autograd.factorize(h, val)               # refill + factor_device on the current stream; val may require grad
    x = f.solve(b)                               # differentiable in val and b
    sign, logabs = f.slogdet()                   # logabs differentiable in val (and the sign in complex)

Every step, forward and backward, is enqueued on the current CUDA stream without a host wait, so a whole step can be captured
into a CUDA graph.  The backward of a solve is one transposed solve (lambda = A^-T dL/dx, A^-H in complex) and the sampled
product -lambda x^T on A's pattern (slu_b200_solve_grad_device); the backward of slogdet is a selected inversion of the
factors (slu_b200_selinv_device, once per Factors) and the gather coef * A^-T on the pattern (slu_b200_logdet_grad_device).
The row matching, R, C and perm of the scaled fill are constants: no gradient flows into them.  Where the factorization
replaced tiny pivots, the gradients describe L U as factored.  A member whose factorization found an exact zero pivot gets
NaN results and gradients.

One live graph per handle: a Factors is valid until the handle's values or factors are written again (another factorize,
refill, fill or factor); a backward after that raises RuntimeError naming the call.  No double backward.
"""
import math
import weakref

import numpy as np
import torch
from torch.autograd.function import once_differentiable

from . import capi

__all__ = ["Factors", "factorize"]

# per handle: (fill generation, shift, parity) with log |det F| = log |det A| + shift_j and sign(det F) = parity sign(det A)
# for F = Pr Dr A Dc: shift_j = sum log R_j + sum log C_j (a CUDA tensor per member), parity = sign(det Pr)
_SCALE = weakref.WeakKeyDictionary()


def _parity(perm):
    """sign of the permutation perm (None: the identity)"""
    if perm is None:
        return 1.0
    p, seen, sign = np.asarray(perm), np.zeros(len(perm), bool), 1.0
    for i in range(len(p)):
        if not seen[i]:
            j, length = i, 0
            while not seen[j]:
                seen[j] = True
                j = p[j]
                length += 1
            if length % 2 == 0:
                sign = -sign
    return sign


def _scale_of(h, device):
    """the (shift, parity) of h's last scaled fill; read from the handle once per fill (a host wait, outside any capture)"""
    hit = _SCALE.get(h)
    if hit is not None and hit[0] == h.fill_generation:
        return hit[1], hit[2]
    if isinstance(h, capi.BatchHandle):
        rc = [h.scaling(j) for j in range(h.batch)]
    else:
        rc = [h.scaling()[1:]]
    shift = torch.tensor([math.fsum(np.log(R)) + math.fsum(np.log(C)) for R, C in rc], dtype=torch.float64, device=device)
    if not isinstance(h, capi.BatchHandle):
        shift = shift.reshape(())
    par = _parity(h.fill_perm_r)
    _SCALE[h] = (h.fill_generation, shift, par)
    return shift, par


class Factors:
    """The factors of one factorize(h, val): solve(b) and slogdet(), differentiable in val."""

    def __init__(self, h, val, info):
        self.h, self.val, self.info = h, val, info
        self.generation = h.generation
        self.complex_ = h.z_
        self._inverse = False          # selinv_device has run on these factors

    def _check(self, what):
        if self.h.generation != self.generation:
            raise RuntimeError(f"{what}: the handle's factors were replaced by {type(self.h).__name__}.{self.h.moved_by}() after "
                               "factorize(); a handle holds one factorization at a time, so finish its backward first")

    def solve(self, b):
        """x = A^-1 b in A's own ordering: b of shape (n,) or (nrhs, n) on a Handle, (B, n) or (B, nrhs, n) on a BatchHandle"""
        return _Solve.apply(self.val, b, self)

    def slogdet(self):
        """(sign, log |det A|) as torch.linalg.slogdet: 0-d tensors on a Handle, (B,) on a BatchHandle"""
        return _Slogdet.apply(self.val, self)


def factorize(h, val):
    """Refill h with val and factor it on the current stream (refill + factor_device) -> Factors.  h: a capi.Handle or
    capi.BatchHandle after one fill_csr_scaled of the pattern (pass no perm_r, R or C and equil=False for no scaling).  val: a
    CUDA tensor (nnz,) or (B, nnz), float64 or complex128 as the handle, in that fill's CSR entry order; it may require grad."""
    if not isinstance(h, (capi.Handle, capi.BatchHandle)):
        raise TypeError(f"h must be a capi.Handle or capi.BatchHandle, not {type(h).__name__}")
    if not isinstance(val, torch.Tensor):
        raise TypeError("val must be a torch CUDA tensor")
    shift, parity = _scale_of(h, val.device)
    h.refill(val.detach())
    info = h.factor_device()
    f = Factors(h, val, info)
    f._shift, f._parity = shift, parity
    return f


class _Solve(torch.autograd.Function):
    @staticmethod
    def forward(ctx, val, b, f):
        f._check("Factors.solve")
        x = f.h.solve_scaled(b)
        ctx.f = f
        ctx.save_for_backward(val, x)
        return x

    @staticmethod
    @once_differentiable
    def backward(ctx, gx):
        f = ctx.f
        _, x = ctx.saved_tensors
        f._check("backward of Factors.solve")
        lam = f.h.solve_scaled(gx.contiguous(), "H" if f.complex_ else "T")
        gval = f.h.solve_grad(lam, x) if ctx.needs_input_grad[0] else None
        return gval, (lam if ctx.needs_input_grad[1] else None), None


class _Slogdet(torch.autograd.Function):
    @staticmethod
    def forward(ctx, val, f):
        f._check("Factors.slogdet")
        sign, logabs = f.h.logdet_device()     # of F = Pr Dr A Dc
        sign, logabs = sign * f._parity, logabs - f._shift
        ctx.f = f
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(val, sign)
        if not f.complex_:
            ctx.mark_non_differentiable(sign)   # piecewise constant
        return sign, logabs

    @staticmethod
    @once_differentiable
    def backward(ctx, gsign, glogabs):
        f = ctx.f
        _, sign = ctx.saved_tensors
        f._check("backward of Factors.slogdet")
        coef = torch.zeros_like(sign, dtype=torch.float64) if glogabs is None else glogabs
        if f.complex_:
            # torch.linalg.slogdet's backward: g_A = (g_logabs + i Im(conj(sign) g_sign)) A^-H
            coef = coef.to(torch.complex128)
            if gsign is not None:
                coef = coef + 1j * (sign.conj() * gsign).imag
        if not f._inverse:
            f.h.selinv_device()
            f._inverse = True
        gval = f.h.logdet_grad(coef.contiguous())
        return gval.reshape(f.val.shape), None
