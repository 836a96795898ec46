"""Error bound of the Poisson solve of ``blend_cheby_kernel`` (fresco_blend_poisson, blend.cu) against the exact
least-squares solution, and a CPU emulation of the iteration it runs.

CHECKER ONLY (see ``oracle/__init__``).

The system
----------
Per Lab channel with gradient weight w, poisson_fusion solves [w Gx; w Gy; I] u ~ [w gx; w gy; im] in least squares.
Gx (Gy) takes forward differences along rows (columns), with an empty last row (column), so G = [Gx; Gy] is the
incidence matrix of the h x w grid graph and the normal equations are

    M u = b,   M = I + w^2 G^T G = I + w^2 (L_h (x) I + I (x) L_w),   b = im + w^2 G^T g,

L_n the path-graph (Neumann) Laplacian.  Its eigenvalues 4 sin^2(pi k / 2n), k = 0 .. n-1, give M's spectrum in closed
form: lambda = 1 + w^2 (4 sin^2(pi k / 2h) + 4 sin^2(pi l / 2w)), in [1, lambda_max] with
lambda_max = 1 + w^2 (4 sin^2(pi (h-1) / 2h) + 4 sin^2(pi (w-1) / 2w)) < 1 + 8 w^2.  (M 1 = 1, so the reference's mean
subtraction, which only helps lsqr's conditioning, does not change the solution.)

The iteration
-------------
Chebyshev iteration on [1, lambda_max] from y_0 = im: theta = (lambda_max + 1) / 2, sigma = (lambda_max + 1) /
(lambda_max - 1), y_1 = y_0 + (b - M y_0) / theta, y_{k+1} = omega_{k+1} (y_k - y_{k-1} + (b - M y_k) / theta) + y_{k-1}
with omega_{k+1} = 2 sigma T_k(sigma) / T_{k+1}(sigma).  The error after k steps is p_k(M) e_0 with
p_k(lambda) = T_k((theta - lambda) / delta) / T_k(sigma), |p_k| <= 1 / T_k(sigma) on the spectrum, so

    max_p |u_k - u*| <= ||u_k - u*||_2 <= ||e_0||_2 / T_k(sigma).

It needs no dot products (no grid-wide reductions) and is deterministic.  A DCT-II solve is exact too, but would need
mixed-radix transforms (896 = 7 * 128) for one solve per plane; the iteration is a 5-point stencil per step.

The initial error.  u* - im = M^-1 (b - M im) = w^2 M^-1 G^T (g - G im).  |g| <= 100 (clipped) and |G im| <= 255 per
edge, so ||g - G im||_2 <= 355 sqrt(E), E = (h-1) w + h (w-1) edges.  The singular values of w^2 M^-1 G^T are
w^2 sqrt(mu) / (1 + w^2 mu) over the eigenvalues mu of G^T G, at most |w| / 2 (1 + w^2 mu >= 2 |w| sqrt(mu)).  Hence
||e_0||_2 <= E0 = (|w| / 2) 355 sqrt(E).

The count.  k is the least integer with E0 / T_k(sigma) <= TRUNC = 5e-4, T_k(sigma) = cosh(k acosh sigma).  At 512 x 896
this is 76 steps for w = 2.5 (lambda_max ~ 51, rho = (sqrt(kappa) - 1) / (sqrt(kappa) + 1) ~ 0.75) and 15 for w = 0.5
(lambda_max ~ 3); at 64 x 64, 67 and 14.  A rougher estimate of ~65 for w = 2.5 assumes a smaller initial error than
the a-priori E0 (4.3e5 at 512 x 896) guarantees.  The count is computed, never an option.

Rounding.  The kernel runs in fp64 and nvcc may contract its multiply-adds.  Each step's rounding is at most a few ulp
of |y| + |b| + w^2 |L y| <= (1 + 8 w^2) 2 max|y|, about 1e-12 at w = 2.5 for values ~ 300, and the Chebyshev recurrence
propagates a local error through polynomials bounded by 1 on the spectrum (times at most k), so after 76 steps it is
below 1e-9, far inside the ROUND = 5e-4 left for it.  TOL = TRUNC + ROUND = 1e-3 is the elementwise bound the tests hold
the kernel's fp64 solution to.
"""
from __future__ import annotations

import math

import numpy as np

TRUNC = 5e-4
ROUND = 5e-4
TOL = TRUNC + ROUND
GRAD_EDGE = 100.0 + 255.0     # |g - G im| per edge


def lambda_max(h, w, weight):
    sh = math.sin(math.pi * (h - 1) / (2.0 * h))
    sw = math.sin(math.pi * (w - 1) / (2.0 * w))
    return 1.0 + weight * weight * (4.0 * sh * sh + 4.0 * sw * sw)


def initial_error(h, w, weight):
    """E0 >= ||u* - im||_2."""
    edges = (h - 1) * w + h * (w - 1)
    return 0.5 * abs(weight) * GRAD_EDGE * math.sqrt(edges)


def truncation_bound(h, w, weight, k, lam_max=None):
    lmax = lambda_max(h, w, weight) if lam_max is None else lam_max
    e0 = initial_error(h, w, weight)
    if e0 == 0.0 or lmax <= 1.0:
        return 0.0
    return e0 / math.cosh(k * math.acosh((lmax + 1.0) / (lmax - 1.0)))


def cheby_iterations(h, w, weight):
    """The step count fresco_blend_cheby_iterations returns: least k with truncation_bound <= TRUNC."""
    e0 = initial_error(h, w, weight)
    lmax = lambda_max(h, w, weight)
    if e0 == 0.0 or lmax <= 1.0:
        return 0
    return max(0, math.ceil(math.acosh(e0 / TRUNC) / math.acosh((lmax + 1.0) / (lmax - 1.0))))


def apply_m(y, weight):
    """M y on one [h, w] plane (Neumann 5-point stencil), in the kernel's association."""
    lap = np.zeros_like(y)
    lap[1:] += y[1:] - y[:-1]
    lap[:-1] += y[:-1] - y[1:]
    lap[:, 1:] += y[:, 1:] - y[:, :-1]
    lap[:, :-1] += y[:, :-1] - y[:, 1:]
    return y + weight * weight * lap


def cheby_emulate(rhs, im, weight, iters, lam_max=None, apply=apply_m):
    """CPU emulation of blend_cheby_kernel on one plane: ``iters`` steps from y_0 = im."""
    h, w = rhs.shape
    lmax = lambda_max(h, w, weight) if lam_max is None else lam_max
    inv_theta = 2.0 / (lmax + 1.0)
    sigma = (lmax + 1.0) / (lmax - 1.0) if lmax > 1.0 else 1.0
    t_prev, t_cur = 1.0, sigma
    cur, prev = im.astype(np.float64).copy(), im.astype(np.float64).copy()
    for k in range(iters):
        if k == 0:
            omega = 1.0
        else:
            t_next = 2.0 * sigma * t_cur - t_prev
            omega = 2.0 * sigma * t_cur / t_next
            t_prev, t_cur = t_cur, t_next
        nxt = omega * (cur - prev + inv_theta * (rhs - apply(cur, weight))) + prev
        prev, cur = cur, nxt
    return cur
