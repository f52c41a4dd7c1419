"""Helpers shared by the bit-exact kernel tests (test_conv_exact.py, test_elementwise_exact.py).

Importing this module does not touch CUDA: tensors are only made when a helper is called.
"""
from __future__ import annotations

import math

import pytest
import torch

DEV = "cuda"
U = 2.0 ** -24   # fp32 unit round-off
POISON_U8 = 0xA5  # prefill of uint8 outputs (masks, argmax indices): a value no kernel writes by accident


def tern(shape, gen, density=0.6, hi=1):
    """fp32 tensor of {-1, 0, 1}; with ``hi > 1`` a quarter of the non-zeros are +-hi instead."""
    v = (torch.randint(0, 2, shape, device=DEV, generator=gen) * 2 - 1).float()
    v *= (torch.rand(shape, device=DEV, generator=gen) < density).float()
    if hi > 1:
        v *= torch.where(torch.rand(shape, device=DEV, generator=gen) < 0.25, float(hi), 1.0)
    return v


class Guarded:
    """``t``: a tensor of ``shape`` inside a larger allocation whose ``guard`` elements before and after it are NaN
    (0xA5 for uint8).  ``fill`` is the prefill of ``t`` itself (None: the same poison as the guards)."""

    def __init__(self, shape, dtype, fill=None, guard=4096):
        n = math.prod(shape)
        self.guard = guard
        poison = POISON_U8 if dtype == torch.uint8 else float("nan")
        self.buf = torch.full((n + 2 * guard,), poison, dtype=dtype, device=DEV)
        self.t = self.buf[guard:guard + n].view(shape)
        self.t.fill_(poison if fill is None else fill)
        self._bits = self._as_int(self.buf).clone()

    @staticmethod
    def _as_int(t):
        return t.view({1: torch.uint8, 2: torch.int16, 4: torch.int32}[t.element_size()])

    def check_guards(self, name):
        b = self._as_int(self.buf)
        g = self.guard
        for side, a, ref in (("before", b[:g], self._bits[:g]), ("after", b[-g:], self._bits[-g:])):
            bad = (a != ref).nonzero().flatten()
            if bad.numel():
                pytest.fail(f"{name}: {bad.numel()} guard elements {side} the output were written (first at offset "
                            f"{int(bad[0]) - (g if side == 'before' else 0)})")

    def untouched(self):
        """bool tensor shaped like ``t``: the element still holds its prefill bit pattern."""
        g = self.guard
        return (self._as_int(self.buf)[g:-g] == self._bits[g:-g]).view(self.t.shape)


def check_equal(name, out, exp, locate=None):
    """Exact comparison (NaN, i.e. an element never written, is a mismatch); reports the first mismatches with the
    kernel coordinates ``locate(*index)`` returns."""
    if out.dtype == exp.dtype and out.shape == exp.shape and bool((out == exp).all()):
        return
    o, e = out.double(), exp.double()
    bad = ~(o == e)
    n = int(bad.sum())
    if n == 0:
        return
    lines = []
    for ix in bad.nonzero()[:8].tolist():
        where = locate(*ix) if locate is not None else ""
        lines.append(f"  at {tuple(ix)}: got {o[tuple(ix)].item()} want {e[tuple(ix)].item()} {where}")
    pytest.fail(f"{name}: {n} of {o.numel()} elements differ\n" + "\n".join(lines))


def check_sum(name, got, ref, ref_abs, depth):
    """Per-channel fp32 sums of integer terms.  ``ref_abs`` = sum of |terms| (float64).  Below 2^24 every partial sum,
    in any order, is an integer that fp32 holds exactly: equality is demanded.  Above, each fp32 addition on a term's
    path to the result errs by at most u * |partial| <= u * sum|terms|, and no term passes more than ``depth`` additions,
    so |error| <= depth * u * sum|terms| (first order in u)."""
    got = got.double()
    if float(ref_abs.max()) < 2.0 ** 24:
        check_equal(name, got, ref)
        return "exact"
    bound = depth * U * ref_abs * (1 + 1e-6)
    err = (got - ref).abs()
    if not bool((err <= bound).all()):
        c = int((err - bound).argmax())
        pytest.fail(f"{name}: channel {c} got {got[c].item()} want {ref[c].item()} (error {err[c].item():.3e} > bound "
                    f"{bound[c].item():.3e}, sum|terms| {ref_abs[c].item():.3e}, depth {depth})")
    return "bounded"


def bf16_half_ulp(x):
    """Half a bf16 ulp of |x| (float64 tensor; 0 where x == 0): the largest error of rounding x to bf16 (nearest even)."""
    _, e = torch.frexp(x.abs())
    return torch.where(x != 0, torch.ldexp(torch.ones_like(x), e - 9), torch.zeros_like(x))


def bf16_bound(ref, err):
    """Bound on |bf16(a) - ref| for an fp32 value a with |a - ref| <= err: a's own rounding plus err."""
    return bf16_half_ulp(ref.abs() + err) + err


def to_bf16_exact(ref):
    """bf16 of a float64 tensor holding values exact in fp32 (round to nearest even, like __floats2bfloat162_rn)."""
    assert bool((ref.float().double() == ref).all()), "reference is not exact in fp32"
    return ref.float().to(torch.bfloat16)


def pack_mask(mask_bool):
    """[M, C] bool -> uint8 [M * C / 8]; bit k of byte j = channel 8 j + k (the layout bn_apply writes)."""
    M, C_ = mask_bool.shape
    bits = mask_bool.reshape(M, C_ // 8, 8).to(torch.int32)
    w = 2 ** torch.arange(8, device=mask_bool.device, dtype=torch.int32)
    return (bits * w).sum(-1).to(torch.uint8).view(-1).contiguous()
