"""fp64 references of the per-step elementwise kernels in hbm_kernels.cu -- Adam (O4: ``adam_kernel``), AdaIN (O5:
``adain_kernel<half|float>``), classifier-free guidance and the DDPM step (S1: ``cfg_pred_x0_kernel``,
``ddpm_prev_kernel``) and the dilation (W2: ``dilate_kernel``) -- with an elementwise bound on each kernel's error and
input families built to break them.

CHECKER ONLY (see ``oracle/__init__``).  Every reference is evaluated in fp64 on the operands the kernel reads: fp16
operands as their fp16 values, fp32 constants as the launcher rounds them.  u = 2^-24, F = 2 (``SAFETY``) on every
rounding term, TINY = 2^-150 (half the fp32 subnormal spacing: the absolute error of one rounding below the normal
range).  "Any contraction" means: nvcc may fuse a product into the following add (fma) or not; each bound below counts
the roundings of the unfused form, which is never fewer than the fused form's.  An fp16 output adds half an fp16 ulp of
|ref| + E (2^-11 relative) in the normal range and half the subnormal spacing (2^-25) below it; a value the fp32 result
rounds past 65504 must be +-inf exactly where |ref| - E >= 65520 and finite where |ref| + E < 65520 (``ratio16``).

Adam, one step (hbm_kernels.cu ``adam_kernel``; ``fresco_adam_step`` derives the constants)
----------------------------------------------------------------------------------------------
The launcher folds beta^step in double, rounds c1 = 1 - beta1, b2, c2 = 1 - beta2, lr / bc1, 1 / sqrt(bc2) and eps to
fp32 one by one -- the values torch.optim.Adam's python scalars become.  The reference uses those fp32 values except
for 1 / sqrt(bc2), which it keeps exact: the kernel multiplies by fl(1 / sqrt(bc2)) (one rounding, u) where torch divides
by fl(sqrt(bc2)) or multiplies by its fp32 reciprocal (two roundings); the bound charges 3u on that term so it holds
for both, and that 3u is the whole cost of the kernel's multiplication.

* m' = m + (g - m) c1: the subtraction, the product and the add, any contraction:
  E_m = F (u |m'| + 2u c1 |g - m| + 3 TINY).  (torch's lerp at weight >= 0.5 computes g - (g - m)(1 - c1); with
  c1 = 0.5 the same terms bound it.)
* v' = v b2 + (g g) c2: two products on one side, one on the other, one add: E_v = F (u |v'| + u b2 |v| + 2u c2 g^2
  + 4 TINY).
* s = sqrt(v'): the error of v' moves s by at most min(sqrt(E_v), E_v / s) (|sqrt a - sqrt b| <= |a - b| / (sqrt a
  + sqrt b)), the sqrtf rounds once: E_s = that + F u s.
* D = s / sqrt(bc2) + eps: E_D = E_s / sqrt(bc2) + F (3u s / sqrt(bc2) + u D).
* q = m' / D: E_q = (E_m + |q| E_D) / (D - E_D) + F u |q|.
* p' = p - (lr / bc1) q: E_p = (lr/bc1) E_q + F (2u (lr/bc1) |q| + u |p'| + 2 TINY) (the product, the subtraction and
  slack for the launcher's fold of beta^step against torch's pow).
Elements with g = m = v = 0 are exact: m' = v' = 0, q = 0 and p' = p bit for bit.

AdaIN (``adain_kernel``: one CTA of 256 threads per plane)
---------------------------------------------------------
Each thread sums ceil(hw / 256) terms in order, a 5-level warp butterfly and a second one over the 8 warp sums follow:
every term passes through at most d = ceil(hw / 256) + 10 roundings, so a sum errs by at most d u sum |x|.
* mean: E_mu = F (d u sum|x| / hw + u |mu|).
* the two-pass sum of squares around the kernel's mean mu~ is Q + hw (mu~ - mu)^2 (the first-order term vanishes:
  sum (x - mu) = 0), and each term carries the subtraction and the square: E_Q = hw E_mu^2 + F (d + 3) u (Q + hw E_mu^2).
* var = Q / (hw - 1) (unbiased): E_var = E_Q / (hw - 1) + F u var;  sigma = sqrt(var + eps) with content eps fp32(1e-5)
  and style eps 1 (the reference's quirk: ``calc_mean_std(style_feat, chunk)`` passes chunk = 1 as eps):
  E_sigma = (E_var + F u (var + eps)) / sigma + F u sigma.
* out = (c - mu_c) / sigma_c * sigma_s + mu_s, any contraction: with r = |c - mu_c| / sigma_c,
  E_o = (F u |c - mu_c| + E_mu_c) sigma_s / sigma_c + r sigma_s (E_sigma_c / sigma_c + E_sigma_s / sigma_s + 2F u)
  + F u |o| + E_mu_s.
On the fp16 path the content is rounded to fp16 first (``cs.data.to(sample.dtype)``), so the reference reads it so.

Guidance and x0 (``cfg_pred_x0_kernel``)
----------------------------------------
e = u + g (t - u) (e = u without the text half): the subtraction and the product act on g |t - u|, the add on |e|:
E_e = F (2u g |t - u| + u |e|) -- cancellation-aware: at g = 7.5 or 30, e is far smaller than g |t - u|.
x0 = (s - sqrt(1 - a) e) / sqrt(a).  The launcher rounds 1 - a, its sqrt, sqrt(a) and 1 / sqrt(a) in fp32 (2.5u on
sqrt(1 - a), 2u on 1 / sqrt(a)); the reference keeps them exact.  y = s - sqrt(1 - a) e: E_y = sqrt(1 - a) E_e
+ F (3u sqrt(1 - a) |e| + u |y|) (the subtraction rounds |y| <= |s| + sqrt(1 - a)|e|, never |x0|); then the
1 / sqrt(a) amplification (up to 14.6 at t = 999) and its two roundings plus the product:
E_x0 = E_y / sqrt(a) + F 3u |x0|.

DDPM step (``ddpm_prev_kernel``)
--------------------------------
prev = c_x0 x0 + c_xt s + sigma z with the launcher's fp32 coefficients (exact operands); z = noise[i mod per_frame]
under repeat_noise.  Three products and two adds in any association and contraction: every term passes through at most
three roundings: E = F (3u sum |terms| + 3 TINY).

Dilation (``dilate_kernel``)
----------------------------
The fp64 reference is the k x k box sum over the replicate-padded plane (clamped indices), clamped to [0, 1].  The kernel
sums the k^2 values in order from 0: E = F k^2 u sum |x| over the box, and the clamp is 1-Lipschitz.  Binary masks and
inputs on a coarse dyadic grid have box sums that are exact in fp32: those families must match bit for bit.
"""
from __future__ import annotations

import math

import numpy as np
import torch

U = 2.0 ** -24
SAFETY = 2.0
TINY = 2.0 ** -150
HALF_ULP = 2.0 ** -11
HALF_SUB = 2.0 ** -25
F16_INF_EDGE = 65520.0          # the smallest magnitude fp16 rounds to inf

ADAM_FAMILIES = ("zero-grad", "tiny-grad", "subnormal-v", "steps", "hyper")
ADAIN_FAMILIES = ("planes", "offset", "constant", "fp16-range")
STEP_FAMILIES = ("schedule", "no-text", "repeat", "overflow")
DILATE_FAMILIES = ("binary", "dyadic", "unit", "signed", "large")
DILATE_EXACT = ("binary", "dyadic")
TIMESTEPS = (999, 981, 501, 21, 1, 0)
GUIDANCE = (1.0, 7.5, 30.0)


def f32(x) -> float:
    return float(np.float32(x))


# ------------------------------------------------------------------------------------------------ common
def out_tol(ref, tol, dtype):
    """The bound of the fp32 value widened by the final store to ``dtype``."""
    if dtype == torch.float16:
        return tol + HALF_ULP * (ref.abs() + tol) + HALF_SUB
    return tol


def ratio(out, ref, tol):
    """|out - ref| / tol elementwise (0 where out == ref, also where tol is 0; NaN counts as infinitely wrong)."""
    err = (out.double() - ref).abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / tol)
    return torch.nan_to_num(r, nan=float("inf"))


def ratio16(out, ref, tol):
    """``ratio`` for an fp16 output whose fp32 value may round past 65504: where |ref| - tol >= 65520 the output must be
    the infinity of ref's sign (ratio 0, else inf), where |ref| + tol < 65520 it must be finite and within tol; in
    between either is right."""
    o = out.double()
    must_inf = ref.abs() - tol >= F16_INF_EDGE
    may_inf = ref.abs() + tol >= F16_INF_EDGE
    is_inf = torch.isinf(o)
    good_inf = is_inf & (torch.sign(o) == torch.sign(ref)) & may_inf
    r = ratio(torch.where(is_inf, torch.zeros_like(o), o), ref, tol)
    r = torch.where(is_inf, torch.where(good_inf, torch.zeros_like(r), torch.full_like(r, float("inf"))), r)
    return torch.where(must_inf & ~is_inf, torch.full_like(r, float("inf")), r)


# ------------------------------------------------------------------------------------------------ Adam
def adam_constants(step, lr=0.2, beta1=0.9, beta2=0.999, eps=1e-8):
    """What fresco_adam_step passes to the kernel (fp32 values as python floats) and the exact sqrt(bc2)."""
    p1 = p2 = 1.0
    for _ in range(step):
        p1 *= beta1
        p2 *= beta2
    bc1, bc2 = 1.0 - p1, 1.0 - p2
    return {"c1": f32(1.0 - beta1), "b2": f32(beta2), "c2": f32(1.0 - beta2), "step_size": f32(lr / bc1),
            "inv_sqrt_bc2": f32(1.0 / math.sqrt(bc2)), "eps": f32(eps), "sqrt_bc2": math.sqrt(bc2)}


def adam_reference_and_bound(p, g, m, v, step, lr=0.2, beta1=0.9, beta2=0.999, eps=1e-8):
    """One Adam step in fp64 on fp32 operands -> dict of (ref, tol) for "p", "m", "v"."""
    k = adam_constants(step, lr, beta1, beta2, eps)
    p, g, m, v = (t.double() for t in (p, g, m, v))
    c1, b2, c2, ss, sq, e = k["c1"], k["b2"], k["c2"], k["step_size"], k["sqrt_bc2"], k["eps"]
    m1 = m + (g - m) * c1
    v1 = v * b2 + g * g * c2
    E_m = SAFETY * (U * m1.abs() + 2 * U * c1 * (g - m).abs() + 3 * TINY)
    E_v = SAFETY * (U * v1.abs() + U * b2 * v.abs() + 2 * U * c2 * g * g + 4 * TINY)
    s = v1.sqrt()
    ds = torch.where(s > 0, torch.minimum(E_v.sqrt(), E_v / s.clamp_min(1e-300)), E_v.sqrt())
    E_s = ds + SAFETY * U * s
    D = s / sq + e
    E_D = E_s / sq + SAFETY * (3 * U * s / sq + U * D)
    q = m1 / D
    E_q = (E_m + q.abs() * E_D) / (D - E_D).clamp_min(0.5 * e) + SAFETY * U * q.abs()
    p1 = p - ss * q
    E_p = ss * E_q + SAFETY * (2 * U * ss * q.abs() + U * p1.abs() + 2 * TINY)
    return {"p": (p1, E_p), "m": (m1, E_m), "v": (v1, E_v)}


ADAM_CONFIGS = {
    # family -> [(step, lr, beta1, beta2, eps)]
    "zero-grad": [(1, 0.2, 0.9, 0.999, 1e-8), (10, 0.2, 0.9, 0.999, 1e-8)],
    "tiny-grad": [(1, 0.2, 0.9, 0.999, 1e-8), (2, 0.2, 0.9, 0.999, 1e-8), (1000, 0.2, 0.9, 0.999, 1e-8)],
    "subnormal-v": [(1, 0.2, 0.9, 0.999, 1e-8), (10, 0.2, 0.9, 0.999, 1e-8)],
    "steps": [(s, 0.2, 0.9, 0.999, 1e-8) for s in (1, 2, 10, 1000)],
    "hyper": [(1, 1e-3, 0.5, 0.99, 1e-6), (2, 0.2, 0.5, 0.99, 1e-8), (10, 1e-3, 0.9, 0.999, 1e-6),
              (1000, 0.2, 0.5, 0.99, 1e-6)],
}


def adam_family(name, n, seed=0, device="cpu"):
    """(p, g, m, v) fp32 [n] of one family; ``ADAM_CONFIGS[name]`` lists the steps and hyper-parameters to run them at.
    Returns a dict that also holds ``exact``: the elements whose p, m and v must come back bit-identical."""
    gen = torch.Generator().manual_seed(seed * 7919 + sum(map(ord, name)) + n)
    p = torch.randn(n, generator=gen)
    g = torch.randn(n, generator=gen) * 1e-2
    m = torch.randn(n, generator=gen) * 1e-2
    v = torch.rand(n, generator=gen) * 1e-4
    exact = torch.zeros(n, dtype=torch.bool)
    if name == "zero-grad":
        exact = torch.rand(n, generator=gen) < 0.5          # masked features: no gradient, no history
        g, m, v = (torch.where(exact, torch.zeros_like(t), t) for t in (g, m, v))
    elif name == "tiny-grad":
        # |g| around eps: sqrt(v') / sqrt(bc2) and eps are of one size in the denominator
        mag = torch.where(torch.rand(n, generator=gen) < 0.5, torch.tensor(1e-8), torch.tensor(1e-9))
        g = torch.randn(n, generator=gen) * mag
        m = torch.randn(n, generator=gen) * mag * 0.3
        v = torch.rand(n, generator=gen) * mag * mag
    elif name == "subnormal-v":
        # v and g^2 (1 - beta2) below fp32's normal range (1.18e-38)
        v = torch.rand(n, generator=gen) * 1e-39
        g = torch.randn(n, generator=gen) * 1e-20
        m = torch.randn(n, generator=gen) * 1e-20
        assert ((v > 0) & (v < 1.1754944e-38)).float().mean() > 0.9
    elif name == "steps":
        g = torch.randn(n, generator=gen) * torch.logspace(-6, 0, 7)[torch.randint(0, 7, (n,), generator=gen)]
        m = 0.3 * g + torch.randn(n, generator=gen) * 1e-3
        v = g * g * torch.rand(n, generator=gen) * 2 + 1e-10
    elif name == "hyper":
        g = torch.randn(n, generator=gen) * 1e-3
        m = torch.randn(n, generator=gen) * 1e-3
        v = torch.rand(n, generator=gen) * 1e-5
    else:
        raise ValueError(name)
    dev = torch.device(device)
    return {"p": p.float().to(dev), "g": g.float().to(dev), "m": m.float().to(dev), "v": v.float().to(dev),
            "exact": exact.to(dev)}


# ------------------------------------------------------------------------------------------------ AdaIN
CONTENT_EPS = f32(1e-5)
STYLE_EPS = 1.0


def _stats(x, hw):
    d = math.ceil(hw / 256) + 10
    mu = x.mean(-1, keepdim=True)
    E_mu = SAFETY * (d * U * x.abs().sum(-1, keepdim=True) / hw + U * mu.abs())
    Q = ((x - mu) ** 2).sum(-1, keepdim=True)
    E_Q = hw * E_mu ** 2 + SAFETY * (d + 3) * U * (Q + hw * E_mu ** 2)
    var = Q / (hw - 1)
    E_var = E_Q / (hw - 1) + SAFETY * U * var
    return mu, E_mu, var, E_var


def adain_reference_and_bound(content, style):
    """content fp32 [P, hw] (the kernel rounds it to fp16 when style is fp16), style fp16 / fp32 [P, hw] ->
    (ref fp64, tol) [P, hw], tol including the output rounding."""
    hw = content.shape[-1]
    c = (content.half() if style.dtype == torch.float16 else content.float()).double()
    s = style.double()
    mu_c, E_mu_c, var_c, E_var_c = _stats(c, hw)
    mu_s, E_mu_s, var_s, E_var_s = _stats(s, hw)
    sig_c, sig_s = (var_c + CONTENT_EPS).sqrt(), (var_s + STYLE_EPS).sqrt()
    E_sig_c = (E_var_c + SAFETY * U * (var_c + CONTENT_EPS)) / sig_c + SAFETY * U * sig_c
    E_sig_s = (E_var_s + SAFETY * U * (var_s + STYLE_EPS)) / sig_s + SAFETY * U * sig_s
    dc = (c - mu_c).abs()
    o = (c - mu_c) / sig_c * sig_s + mu_s
    E_o = ((SAFETY * U * dc + E_mu_c) * sig_s / sig_c
           + dc / sig_c * sig_s * (E_sig_c / sig_c + E_sig_s / sig_s + 2 * SAFETY * U)
           + SAFETY * U * o.abs() + E_mu_s)
    return o, out_tol(o, E_o, style.dtype)


ADAIN_HW = (2, 3, 7, 100, 255, 256, 257, 1000, 4096, 9216)


def adain_family(name, planes, hw, dtype, seed=0, device="cpu"):
    """(content fp32 [planes, hw], style ``dtype`` [planes, hw])."""
    gen = torch.Generator().manual_seed(seed * 7919 + sum(map(ord, name)) + planes * 31 + hw)
    scale_c = torch.logspace(-2, 2, planes)[torch.randperm(planes, generator=gen)][:, None]
    c = torch.randn(planes, hw, generator=gen) * scale_c + torch.randn(planes, 1, generator=gen) * scale_c
    s = torch.randn(planes, hw, generator=gen) * 2 + torch.randn(planes, 1, generator=gen)
    if name == "planes":
        pass
    elif name == "offset":
        # |mean| / std up to 1e3 on both sides: the two-pass variance must not cancel
        ratio_ = torch.logspace(0, 3, planes)[torch.randperm(planes, generator=gen)][:, None]
        c = torch.randn(planes, hw, generator=gen) + ratio_ * torch.sign(torch.randn(planes, 1, generator=gen))
        s = torch.randn(planes, hw, generator=gen) * 3 + 3 * ratio_
    elif name == "constant":
        # constant content planes (var 0: sigma_c = sqrt(1e-5)) and constant style planes (sigma_s = 1)
        cc = torch.rand(planes, 1, generator=gen) < 0.5
        c = torch.where(cc, torch.randn(planes, 1, generator=gen).expand(planes, hw), c)
        c[0::4] = 0.1                       # its fp32 sum is not exact: the mean's rounding is all there is
        sc = ~cc
        s = torch.where(sc, torch.randn(planes, 1, generator=gen).expand(planes, hw) * 10, s)
    elif name == "fp16-range":
        # styles near the top of fp16 (mean 6e4, spread 2e3) and in its subnormal range (|s| < 6.1e-5)
        top = torch.arange(planes)[:, None] % 2 == 0
        c = torch.rand(planes, hw, generator=gen) * 2 - 1
        s_top = 6e4 + (torch.rand(planes, hw, generator=gen) * 2 - 1) * 2e3
        s_sub = (torch.rand(planes, hw, generator=gen) * 2 - 1) * 6e-5
        s = torch.where(top, s_top, s_sub)
    else:
        raise ValueError(name)
    dev = torch.device(device)
    return c.float().contiguous().to(dev), s.to(dtype).contiguous().to(dev)


# ------------------------------------------------------------------------------------------------ CFG + DDPM
def sd15_alphas_cumprod():
    """SD-1.5's scaled-linear schedule as diffusers builds it in fp32: betas = linspace(sqrt(0.00085), sqrt(0.012),
    1000)^2, alphas_cumprod = cumprod(1 - betas)."""
    betas = torch.linspace(0.00085 ** 0.5, 0.012 ** 0.5, 1000, dtype=torch.float32) ** 2
    return torch.cumprod(1.0 - betas, dim=0)


def cfg_reference_and_bound(uncond, text, sample, guidance, alpha_prod_t):
    """x0 of cfg_pred_x0 in fp64 (text None: no guidance) -> (ref, tol) shaped like sample, before the output
    rounding."""
    u, s = uncond.reshape(-1).double(), sample.reshape(-1).double()
    a = f32(alpha_prod_t)
    if text is None:
        e, E_e = u, torch.zeros_like(u)
    else:
        d = text.reshape(-1).double() - u
        e = u + f32(guidance) * d
        E_e = SAFETY * (2 * U * abs(f32(guidance)) * d.abs() + U * e.abs())
    sb, isa = math.sqrt(1.0 - a), 1.0 / math.sqrt(a)
    y = s - sb * e
    E_y = sb * E_e + SAFETY * (3 * U * sb * e.abs() + U * y.abs())
    x0 = y * isa
    tol = E_y * isa + SAFETY * 3 * U * x0.abs()
    return x0.reshape(sample.shape), tol.reshape(sample.shape)


def ddpm_noise(noise, n, per_frame, repeat):
    z = noise.reshape(-1)
    return z[:per_frame].repeat(n // per_frame) if repeat else z[:n]


def ddpm_reference_and_bound(x0, sample, noise, c_x0, c_xt, sigma, per_frame, repeat):
    """prev of ddpm_prev in fp64 -> (ref, tol) before the output rounding; x0 / sample / noise flat or shaped."""
    n = sample.numel()
    x, s = x0.reshape(-1).double(), sample.reshape(-1).double()
    z = ddpm_noise(noise, n, per_frame, repeat).double()
    t = (f32(c_x0) * x, f32(c_xt) * s, f32(sigma) * z)
    ref = t[0] + t[1] + t[2]
    tol = SAFETY * (3 * U * (t[0].abs() + t[1].abs() + t[2].abs()) + 3 * TINY)
    return ref.reshape(sample.shape), tol.reshape(sample.shape)


def step_coefficients(alphas_cumprod, t, prev_t):
    """(alpha_prod_t, c_x0, c_xt, sigma) as src/pipe_FRESCO.py:22-31,51-58 computes them: 0-dim fp32 tensor arithmetic,
    returned as python floats."""
    a = alphas_cumprod[t]
    a_prev = alphas_cumprod[prev_t] if prev_t >= 0 else torch.tensor(1.0)
    b, b_prev = 1 - a, 1 - a_prev
    cur_a = a / a_prev
    cur_b = 1 - cur_a
    c_x0 = (a_prev ** 0.5 * cur_b) / b
    c_xt = cur_a ** 0.5 * b_prev / b
    var = torch.clamp(torch.as_tensor(b_prev / b * cur_b), min=1e-20)
    return float(a), float(c_x0), float(c_xt), float(var ** 0.5)


def step_family(name, frames, per_frame, dtype, t, seed=0, device="cpu"):
    """Operands of one guided step at timestep t: dict of noise_pred [2 frames, per_frame] (uncond | text), sample,
    noise [frames, per_frame] in ``dtype``.  ``overflow`` (fp16) builds x0 and prev past 65504 for about half the
    elements at every timestep; for fp32 it is the same operands at full size."""
    gen = torch.Generator().manual_seed(seed * 7919 + sum(map(ord, name)) + t + frames * per_frame)
    shape = (frames, per_frame)
    u = torch.randn(shape, generator=gen)
    txt = u + torch.randn(shape, generator=gen) * 0.1       # text and uncond predictions close: guidance cancels
    s = torch.randn(shape, generator=gen) * 1.5
    z = torch.randn(shape, generator=gen)
    if name == "overflow":
        a = f32(sd15_alphas_cumprod()[t])
        lim = 65504.0
        s = (torch.rand(shape, generator=gen) * 0.5 + 0.75) * min(lim, F16_INF_EDGE * math.sqrt(a))
        s = s.clamp(max=65504.0) * torch.sign(torch.randn(shape, generator=gen))
        u = torch.randn(shape, generator=gen) * 0.5
        txt = u + torch.randn(shape, generator=gen) * 0.01
    elif name not in ("schedule", "no-text", "repeat"):
        raise ValueError(name)
    dev = torch.device(device)
    cast = lambda x: x.to(dtype).contiguous().to(dev)          # noqa: E731
    return {"noise_pred": cast(torch.cat([u, txt])), "sample": cast(s), "noise": cast(z)}


# ------------------------------------------------------------------------------------------------ dilation
def dilate_reference_and_bound(x, k):
    """x fp32 [P, h, w] -> (clamped replicate-padded k x k box sum in fp64, tol), both [P, h, w]."""
    P, h, w = x.shape
    r = (k - 1) // 2
    dev = x.device
    off = torch.arange(-r, r + 1, device=dev)
    yy = (torch.arange(h, device=dev)[:, None] + off[None]).clamp(0, h - 1)        # [h, k]
    xx = (torch.arange(w, device=dev)[:, None] + off[None]).clamp(0, w - 1)        # [w, k]
    xd = x.double()
    rows = xd[:, yy].sum(2)                     # [P, h, w]: column sums over the k clamped rows
    rows_abs = xd.abs()[:, yy].sum(2)
    S = rows[:, :, xx].sum(3)
    A = rows_abs[:, :, xx].sum(3)
    return S.clamp(0, 1), SAFETY * k * k * U * A


def dilate_family(name, P, h, w, seed=0, device="cpu"):
    gen = torch.Generator().manual_seed(seed * 7919 + sum(map(ord, name)) + P * h * w)
    if name == "binary":
        x = (torch.rand(P, h, w, generator=gen) < 0.03).float()
        x[0::3] = 0
        if P > 1:
            x[1::3, h // 2, w // 2] = 1                          # a single pixel: the radius shows
    elif name == "dyadic":
        x = torch.randint(-512, 1024, (P, h, w), generator=gen).float() / 512       # box sums exact in fp32
    elif name == "unit":
        # sparse values in [0, 1]: box sums straddle 1, so the border's replicated pixels count
        x = torch.rand(P, h, w, generator=gen) * (torch.rand(P, h, w, generator=gen) < 0.3)
        x[:, 0] = torch.rand(P, w, generator=gen) * 0.2                            # border rows and columns
        x[:, :, -1] = torch.rand(P, h, generator=gen) * 0.2
    elif name == "signed":
        x = torch.randn(P, h, w, generator=gen) * 0.3
    elif name == "large":
        x = torch.rand(P, h, w, generator=gen) * 3 - torch.rand(P, h, w, generator=gen) * 2.9
    else:
        raise ValueError(name)
    return x.float().contiguous().to(torch.device(device))
