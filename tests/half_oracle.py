"""The error bound of the sparse conv's half entry points, for the GPU tests.

Half tensors are widened to fp32, convolved by the BF16x3 kernels with fp32 accumulation and narrowed once, so each
result should sit within one fp16 rounding of the float64 conv of the half-rounded inputs, plus the error of the fp32
computation:

    |got - ref| <= ulp(ref) + C_BF16X3 * absref

  * ulp(ref): the spacing of the result's dtype at |ref| (the smallest subnormal below the normal range).  One
    rounding to nearest is at most half of it; the other half covers a result that crosses into the next binade.
  * absref: the same float64 conv of |features| and |weights| (and |out_grad| for the backward): it bounds every
    product's size, so it bounds the accumulated error even where the sum cancels.
  * C_BF16X3 = 3 * 2^-16, the error per product of the BF16x3 split: a = a_hi + a_lo + e_a with a_hi = bf16(a),
    a_lo = bf16(a - a_hi) and |e_a| <= 2^-8 * 2^-8 |a|, the same for b, and the kernel drops a_lo * b_lo (at most
    2^-16 |ab|): |ab - (a_hi b_hi + a_hi b_lo + a_lo b_hi)| <= 3 * 2^-16 |ab| to first order.  The fp32 sums add
    about 2^-24 per addition, far inside the half ulp of slack.  (Single-pass TF32 errs by up to 2^-10 |ab| per
    product, and single-pass bf16 by 2^-7: a result where the sum cancels breaks the bound at once.)

Results of magnitude at least 65520 round to inf in fp16; `check` asks for inf with the sign of ref where the whole
error band lies beyond that, and accepts 65504 or inf inside the band."""
import torch

C_BF16X3 = 3 * 2.0 ** -16
FP16_INF_FROM = 65520.0          # the smallest magnitude that rounds to inf (65504 + half its ulp)


def ulp(ref, dtype):
    """spacing of `dtype` (float16 / float32) at |ref| (float64), the smallest subnormal below the normal range"""
    mant, emin = {torch.float16: (10, -14), torch.float32: (23, -126)}[dtype]
    _, e = torch.frexp(ref.abs().clamp_min(2.0 ** emin))       # |ref| in [2^(e-1), 2^e)
    return torch.ldexp(torch.ones_like(ref), e - 1 - mant)


def check(got, ref, absref, what, c=C_BF16X3):
    """Asserts the bound on every element of `got` (the device result, fp16 or fp32) against float64 `ref` and
    `absref`, and that fp16 results past the range are inf with the sign of ref.  Returns the worst ratio
    |got - ref| / (ulp(ref) + c * absref) over the finite results."""
    assert got.shape == ref.shape, what
    assert bool(torch.isfinite(ref).all()), "%s: the float64 reference itself is not finite" % what
    g = got.double()
    slack = c * absref
    if got.dtype == torch.float16:
        must_inf = ref.abs() - slack >= FP16_INF_FROM
        may_inf = ref.abs() + slack >= FP16_INF_FROM
    else:
        must_inf = may_inf = torch.zeros_like(ref, dtype=torch.bool)
    signed_inf = torch.isinf(g) & (torch.sign(g) == torch.sign(ref))
    assert bool(signed_inf[must_inf].all()), "%s: %d results past the fp16 range are not inf of the right sign" % (
        what, int((~signed_inf[must_inf]).sum()))
    finite = ~(may_inf & signed_inf)
    assert bool(torch.isfinite(g[finite]).all()), "%s: %d non-finite results where float64 is in range" % (
        what, int((~torch.isfinite(g[finite])).sum()))
    ratio = (g - ref).abs()[finite] / (ulp(ref, got.dtype) + slack)[finite]
    worst = float(ratio.max()) if ratio.numel() else 0.0
    assert worst <= 1.0, "%s: |got - ref| reaches %.3f of ulp(ref) + %.2e * absref" % (what, worst, c)
    return worst
