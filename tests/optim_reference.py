"""Reference of the AdamW and RMSprop steps (wb_adamw_step / wb_rmsprop_step) and of MultiviewStep's learning-rate schedule
(TEST INFRASTRUCTURE, NOT PRODUCT CODE), beside composite_reference.py's Adam functions and built from the same parts.

For each rule
  *_fp32   the kernel's fp32 chain bit for bit, as wb_optim.cu's comment states it: every product, quotient and square root
           rounded once, the moment updates and the parameter update single fmas.  The kernels spell every operation out
           (fmaf / __fmul_rn / __fdiv_rn / __fsqrt_rn / __fadd_rn), so unlike Adam's last line there is one admissible result.
  the interval function: centre and radius of one step from the fp32 state before it, one rounding per operation
           (composite_reference._I); exact=True turns the roundings off and gives the float64 operation.

lr and weight_decay are the fp32 values the segment carries; AdamW's decay factor is fl32(1 - lr * wd) formed in double from them.
"""
from __future__ import annotations

import numpy as np

from composite_reference import _I, bias_corrections, f32, fma32

GOLDEN_GROUPS = ("decoder", "grid", "rest")          # column order of the golden's learning rates: init_optimizer's group order


def adamw_decay(lr, wd, exact: bool = False):
    """The factor p is multiplied by: double arithmetic on the segment's fp32 lr and wd, rounded to fp32 (exact: float64 values)."""
    return 1.0 - float(lr) * float(wd) if exact else float(f32(1.0 - float(f32(lr)) * float(f32(wd))))


def adamw_fp32(p, g, m, v, lr, wd, b1, b2, eps, step: int, grad_scale: float = 1.0):
    """wb_rule_kernel<AdamW>'s chain -> (p, m, v) as float32 arrays."""
    bc1, bc2s = (f32(x) for x in bias_corrections(b1, b2, step))
    p, g, m, v = (np.asarray(a, f32) for a in (p, g, m, v))
    decay = f32(adamw_decay(lr, wd))
    b1, b2, eps, lr, gs = (f32(x) for x in (b1, b2, eps, lr, grad_scale))
    pd = p * decay
    gg = g * gs
    m1 = fma32(b1, m, (f32(1) - b1) * gg).astype(f32)
    v1 = fma32(b2, v, ((f32(1) - b2) * gg) * gg).astype(f32)
    ss = lr / bc1
    q = m1 / (np.sqrt(v1) / bc2s + eps)
    return fma32(-ss, q, pd).astype(f32), m1, v1


def rmsprop_fp32(p, g, sq, buf, lr, wd, alpha, eps, momentum, grad_scale: float = 1.0):
    """wb_rule_kernel<RMSprop>'s chain -> (p, square_avg, momentum_buffer) as float32 arrays; buf is ignored and None comes back
    when momentum == 0."""
    p, g, sq = (np.asarray(a, f32) for a in (p, g, sq))
    lr, wd, alpha, eps, mom, gs = (f32(x) for x in (lr, wd, alpha, eps, momentum, grad_scale))
    gg = g * gs
    if wd != 0:
        gg = fma32(wd, p, gg).astype(f32)
    sq1 = fma32(alpha, sq, ((f32(1) - alpha) * gg) * gg).astype(f32)
    q = gg / (np.sqrt(sq1) + eps)
    if mom == 0:
        return fma32(-lr, q, p).astype(f32), sq1, None
    buf1 = fma32(mom, np.asarray(buf, f32), q).astype(f32)
    return fma32(-lr, buf1, p).astype(f32), sq1, buf1


def _consts(exact):
    k = lambda x: _I(x, np.zeros_like(np.asarray(x, np.float64)), exact)
    arr = (lambda a: k(np.asarray(a, np.float64))) if exact else (lambda a: k(np.asarray(a, f32).astype(np.float64)))
    cst = (lambda x: k(float(x))) if exact else (lambda x: k(float(f32(x))))
    return k, arr, cst


def adamw(p, g, m, v, lr, wd, b1, b2, eps, step: int, grad_scale: float = 1.0, exact: bool = False):
    """One wb_adamw_step over one segment from its fp32 state -> (p, m, v) each (centre, radius)."""
    bc1, bc2s = bias_corrections(b1, b2, step, exact)
    k, arr, cst = _consts(exact)
    P, G, M, V = (arr(a) for a in (p, g, m, v))
    B1, B2, one = cst(b1), cst(b2), k(1.0)
    PD = P * k(adamw_decay(lr, wd, exact))
    gg = G * cst(grad_scale)
    M1 = B1.fma(M, (one - B1) * gg)
    V1 = B2.fma(V, ((one - B2) * gg) * gg)
    q = M1 / (V1.sqrt() / k(bc2s) + cst(eps))
    P1 = (k(0.0) - cst(lr) / k(bc1)).fma(q, PD)
    return (P1.c, P1.r), (M1.c, M1.r), (V1.c, V1.r)


def rmsprop(p, g, sq, buf, lr, wd, alpha, eps, momentum, grad_scale: float = 1.0, exact: bool = False):
    """One wb_rmsprop_step over one segment -> (p, square_avg, momentum_buffer) each (centre, radius); buffer None at momentum 0."""
    k, arr, cst = _consts(exact)
    P, G, S = (arr(a) for a in (p, g, sq))
    AL, one, nlr = cst(alpha), k(1.0), k(0.0) - cst(lr)
    gg = G * cst(grad_scale)
    if wd != 0.0:
        gg = cst(wd).fma(P, gg)
    S1 = AL.fma(S, ((one - AL) * gg) * gg)
    q = gg / (S1.sqrt() + cst(eps))
    if momentum == 0.0:
        P1 = nlr.fma(q, P)
        return (P1.c, P1.r), (S1.c, S1.r), None
    B1 = cst(momentum).fma(arr(buf), q)
    P1 = nlr.fma(B1, P)
    return (P1.c, P1.r), (S1.c, S1.r), (B1.c, B1.r)


def multistep_lrs(lr0: float, milestones, gamma: float, steps: int):
    """Learning rate of optimiser steps 1..steps: lr0 * gamma^k, k = the milestones <= t - 1 with multiplicity, the factor
    multiplied up in double (MultiviewStep's rule, written out independently of the package)."""
    out = []
    for t in range(1, steps + 1):
        f = 1.0
        for _ in range(sum(1 for m in milestones if m <= t - 1)):
            f *= gamma
        out.append(lr0 * f)
    return out


def golden_groups(names, lrs_row, weight_decay):
    """(lr, weight_decay) of every named parameter under init_optimizer's groups, from one row of the golden's recorded rates."""
    col = {n: i for i, n in enumerate(GOLDEN_GROUPS)}
    grp = lambda n: "decoder" if "decoder" in n else "grid" if "grid" in n else "rest"
    return {n: (float(lrs_row[col[grp(n)]]), weight_decay if grp(n) == "decoder" else 0.0) for n in names}
