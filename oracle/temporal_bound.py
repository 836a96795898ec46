"""fp64 reference of fresco_temporal_attn_fwd[_strided], an elementwise bound on the error of both temporal-guided
attention kernels, and adversarial input families.

CHECKER ONLY (see ``oracle/__init__``).  Layout as the C ABI's: q, k, v [chunks*N, tokens, heads*d] fp16 (views into a
wider row, such as the packed q | k | v row of the trajectory exchange, are fine: ``unpack`` makes them), fwd_map int64
[N, tokens] (trajectory p visits token fwd_map[f, p] of frame f), mask [tokens, N, N] (mask[p, f, g]: frame f of
trajectory p attends to frame g).  ``scale`` is rounded to fp32 first, since the C ABI passes it as a float; everything
else is evaluated in fp64 from the fp16 operands exactly as the kernels read them:

    x_fg = fp32(scale) q_f . k_g  (masked keys -inf)      w_fg = softmax_g(x_fg)      y_f = sum_g w_fg v_g

gathered along the trajectory and scattered back to token fwd_map[f, p] of frame f.

The bound
---------
For one output row (trajectory p, frame f, head h) and channel c, with m = max_g x_g over the unmasked keys,
l = sum_g exp(x_g - m), u = 2^-24, n = the number of unmasked keys of the row, D the head dim:

    A_c = sum_g w_g |v_gc|          Q_g = sum_c |q_fc k_gc|

    tol = F * ( (2^-11 + n u) |ref| + 2^-25 + (n + 1) u A + sum_g w_g rho_g (|v_gc| + |ref_c|) + N 2^-126 max_g|v_gc| / l )

Each term, in the order the kernels do the work:

* ``rho_g`` -- the relative error of the unnormalised weight p_g = exp(x_g - m).  A relative perturbation rho_g of
  each numerator moves sum_g p_g v_g / sum_g p_g by at most sum_g w_g |rho_g| (|v_g| + |ref|) (first order); a
  perturbation common to the whole row, such as the error in m, cancels.  Its parts:

  - the dot product.  Products of fp16 operands are exact in fp32, so an FMA chain of k terms errs by (k - 1) u times
    the sum of the |products|.  ``temporal_attn_rows_kernel`` runs two interleaved chains of D/2 terms and adds them,
    (D/2 - 1) u Q_g + u Q_g = (D/2) u Q_g; ``temporal_attn_kernel`` runs one chain of D terms, (D - 1) u Q_g.  In
    logit units both are multiplied by fp32(scale).
  - the logit.  The row kernel multiplies by c2 = fl(fp32(scale) fl(log2 e)), computed on the host: two roundings,
    then fl(fl(a0 + a1) c2) a third, 3 u |x_g| (log2 units times ln 2 = nats).  The round-1 kernel rounds
    fl(acc scale) once, u |x_g|.
  - the subtraction fl(x_g - m) (either kernel), u |x_g - m|.
  - the exponential.  Row kernel: ex2.approx.ftz.f32, within 2 ulp, EPS_EX2 = 2^-22.  Round-1 kernel: __expf, whose
    documented error is 2 + floor(1.173 |x|) ulp (CUDA C++ Programming Guide, intrinsic functions); taken as
    (2 + 1.173 |x_g - m|) 2^-23 relative.  That figure is the guide's, not a measurement; the CPU emulation
    (``tests/test_temporal_attention_numerics_model.py``) and the GPU runs check it.

  rows:    rho_g = fp32(scale) (D/2) u Q_g + 3 u |x_g| + u |x_g - m| + 2^-22
  round-1: rho_g = fp32(scale) (D - 1) u Q_g + u |x_g| + u |x_g - m| + (2 + 1.173 |x_g - m|) 2^-23

* ``N 2^-126 max|v| / l`` -- ftz: a p_g below 2^-126 is flushed to zero, which moves the numerator by at most
  2^-126 |v_gc| per key.  Negligible, but it makes the bound complete.
* ``(n - 1) u |ref|`` -- l, a sequential fp32 sum of the N exponentials (masked keys and the row kernel's g >= N slots
  are exact zeros, so only n - 1 additions round).  A relative error of l scales the whole output row.
* ``u |ref|`` -- ``1.f / l``, IEEE (the library is built with --use_fast_math=false).
* ``u A`` -- pw = fl(p_g inv), one rounding per key that does not cancel between numerator and denominator.
* ``n u A`` -- O accumulated per channel by N sequential fp32 FMAs (a masked key's pw is 0 and its FMA exact; the
  first unmasked one rounds the product).
* ``2^-11 |ref| + 2^-25`` -- the output rounded to fp16: relative 2^-11, absolute 2^-25 below the normal range.

The terms are first order.  F = 2 is the one safety factor: it covers the products of first-order errors.  Nothing
else is widened.

Exact answers
-------------
Three families have exactly known outputs, which both kernels must reproduce bit for bit: ``self-only`` (only the
diagonal unmasked: p = 1, l = 1, y_f = v_f), ``dominant`` (one key > 150 nats above every other: the others flush to
zero under ftz, so y_f = v_g*) and ``uniform`` (all k rows of a trajectory equal, N a power of two, small dyadic v:
every p is exactly 1, 1/N is exact and so is the mean).
"""
from __future__ import annotations

import math
from typing import NamedTuple

import numpy as np
import torch

U = 2.0 ** -24
SAFETY = 2.0
EPS_EX2 = 2.0 ** -22          # ex2.approx.ftz.f32
EXPF_ULP = 2.0 ** -23         # one ulp of a normal fp32 result, relative
FLT_MIN = 2.0 ** -126
KERNELS = ("rows", "round1")


def _f32(x: float) -> float:
    return float(np.float32(x))


def unpack(buf: torch.Tensor, C: int, offsets=None):
    """q, k, v views [B, tokens, C] of a strided buffer [B, tokens, stride] at column offsets (default q | k | v)."""
    offsets = (0, C, 2 * C) if offsets is None else offsets
    return tuple(buf[..., o:o + C] for o in offsets)


def gather(t: torch.Tensor, fwd_map: torch.Tensor, chunks: int, heads: int) -> torch.Tensor:
    """[chunks*N, tokens, C] (any strides) -> fp64 [chunks, tokens (trajectory), heads, N, d] along the trajectories."""
    B, L, C = t.shape
    N, d = B // chunks, C // heads
    fr = torch.arange(N, device=t.device)[:, None]
    x = t.reshape(chunks, N, L, C)[:, fr, fwd_map.to(t.device)]           # [chunks, N, p, C]
    return x.double().reshape(chunks, N, L, heads, d).permute(0, 2, 3, 1, 4)


def scatter(y: torch.Tensor, fwd_map: torch.Tensor) -> torch.Tensor:
    """Inverse of ``gather``: [chunks, tokens, heads, N, d] -> [chunks*N, tokens, heads*d], row fwd_map[f, p] of frame
    f taking trajectory p."""
    c, L, H, N, d = y.shape
    fr = torch.arange(N, device=y.device)[:, None]
    out = torch.empty(c, N, L, H * d, dtype=y.dtype, device=y.device)
    out[:, fr, fwd_map.to(y.device)] = y.permute(0, 3, 1, 2, 4).reshape(c, N, L, H * d)
    return out.reshape(c * N, L, H * d)


def logits(qg, kg, mask, scale):
    """fp64 logits [chunks, tokens, heads, N, N] (nats; masked keys -inf) from gathered operands."""
    x = (qg @ kg.transpose(-1, -2)) * _f32(scale)
    return x.masked_fill(~mask.bool().to(x.device)[None, :, None], float("-inf"))


def ref_and_bound(q, k, v, fwd_map, mask, chunks, heads, scale, kernel="rows", gathered=False):
    """(reference, tolerance), fp64 [chunks*N, tokens, C] in the output layout.  ``kernel`` "rows" bounds
    temporal_attn_rows_kernel, "round1" temporal_attn_kernel.  gathered=True returns both in the gathered layout
    [chunks, tokens, heads, N, d] instead."""
    if kernel not in KERNELS:
        raise ValueError(kernel)
    qg, kg, vg = (gather(t, fwd_map, chunks, heads) for t in (q, k, v))
    N, d = qg.shape[-2], qg.shape[-1]
    keep = mask.bool().to(qg.device)[None, :, None]                       # [1, L, 1, N, N]
    x = logits(qg, kg, mask, scale)
    m = x.amax(-1, keepdim=True)
    e = torch.exp(x - m)
    l = e.sum(-1, keepdim=True)
    w = e / l
    ref = w @ vg
    va = vg.abs()
    A = w @ va
    n = keep.sum(-1, keepdim=True).double()                               # unmasked keys per row
    Q = qg.abs() @ kg.abs().transpose(-1, -2)
    xf = torch.where(keep, x, 0.0).abs()
    dm = torch.where(keep, x - m, 0.0).abs()
    if kernel == "rows":
        rho = _f32(scale) * (d / 2) * U * Q + 3 * U * xf + U * dm + EPS_EX2
    else:
        rho = _f32(scale) * (d - 1) * U * Q + U * xf + U * dm + (2 + 1.173 * dm) * EXPF_ULP
    wr = torch.where(keep, w * rho, 0.0)
    tol = SAFETY * ((2.0 ** -11 + n * U) * ref.abs() + 2.0 ** -25 + (n + 1) * U * A
                    + wr @ va + wr.sum(-1, keepdim=True) * ref.abs()
                    + N * FLT_MIN * va.amax(-2, keepdim=True) / l)
    if gathered:
        return ref, tol
    return scatter(ref, fwd_map), scatter(tol, fwd_map)


def ratio(out: torch.Tensor, ref: torch.Tensor, tol: torch.Tensor) -> torch.Tensor:
    """|out - ref| / tol elementwise; an output that is NaN or infinite counts as infinitely wrong."""
    r = (out.double() - ref).abs() / tol
    return torch.nan_to_num(r, nan=float("inf"))


# ============================================================================================== adversarial families
class Case(NamedTuple):
    family: str
    q: torch.Tensor            # [chunks*N, tokens, C] fp16
    k: torch.Tensor
    v: torch.Tensor
    fwd_map: torch.Tensor      # int64 [N, tokens]
    mask: torch.Tensor         # bool [tokens, N, N]
    chunks: int
    heads: int
    scale: float
    exact: torch.Tensor = None   # the exactly known output (fp16 [chunks*N, tokens, C]) of the exact families


FAMILIES = ("self-only", "dominant", "uniform", "masked-max", "huge", "floor", "staircase-rising",
            "staircase-falling", "asymmetric", "reference")
EXACT = ("self-only", "dominant", "uniform")


def _perms(N, L, g, identity_first=False):
    """Per-frame token permutations, none the identity (frame 0's too unless identity_first)."""
    rows = []
    for f in range(N):
        if f == 0 and identity_first:
            rows.append(torch.arange(L))
            continue
        p = torch.randperm(L, generator=g)
        if L > 1 and torch.equal(p, torch.arange(L)):
            p = p.roll(1)
        rows.append(p)
    return torch.stack(rows)


def _case(family, qg, kg, vg, fwd, mask, heads, scale, exact=None):
    """Gathered fp32 [chunks, L, H, N, d] operands -> a Case in the token layout (fp16)."""
    def tok(t):
        return scatter(t.double(), fwd).half() if t is not None else None
    return Case(family, tok(qg), tok(kg), tok(vg), fwd, mask, qg.shape[0], heads, scale, tok(exact))


def _layernorm(t, gain):
    return gain * (t - t.mean(-1, keepdim=True)) / t.std(-1, keepdim=True, unbiased=False)


def _diag_kept_random_mask(L, N, g, p_keep=0.6):
    m = torch.rand(L, N, N, generator=g) < p_keep
    m |= torch.eye(N, dtype=torch.bool)
    return m


def reference_mask(N, L, g, cut_prob=0.3, self_only=0.05):
    """The structure of the reference's get_mapping_ind (flow_utils.py:126-133): per trajectory a set of cuts between
    frames <= i and > i, every cut position i used by some trajectory; plus self_only of the trajectories attending
    only to their own frame."""
    mask = torch.ones(L, N, N, dtype=torch.bool)
    for i in range(N - 1):
        cut = torch.ones(N, N, dtype=torch.bool)
        cut[:i + 1, i + 1:] = False
        cut[i + 1:, :i + 1] = False
        sel = torch.rand(L, generator=g) < cut_prob
        sel[i % L] = True
        mask[sel] &= cut
    mask[torch.rand(L, generator=g) < self_only] = torch.eye(N, dtype=torch.bool)
    return mask


def make_case(family, N, L, heads, d, chunks=2, seed=0):
    """One case of ``family`` on CPU tensors (move them with .cuda() for the GPU)."""
    g = torch.Generator().manual_seed(seed * 1009 + N * 31 + d)
    scale = 1.0 / math.sqrt(d)
    shape = (chunks, L, heads, N, d)
    randn = lambda *s: torch.randn(*s, generator=g)
    fwd = _perms(N, L, g)
    ones = torch.ones(L, N, N, dtype=torch.bool)
    eye = torch.eye(N, dtype=torch.bool)
    if family == "self-only":
        qg, kg, vg = randn(*shape), randn(*shape), randn(*shape)
        return _case(family, qg, kg, vg, fwd, eye.expand(L, N, N).clone(), heads, scale, exact=vg)
    if family == "dominant":
        # hot key of row (p, f): frame 0, N - 1 or 8 (past the NMAX = 8 slots), rotating over (p, f); the row's q is a
        # multiple of the hot key's k, > 150 nats above every other key
        cand = [c for c in (0, N - 1, 8) if c < N]
        p = torch.arange(L)[:, None, None]
        f = torch.arange(N)[None, None, :]
        hot = torch.tensor(cand)[(p + f) % len(cand)].expand(L, heads, N)              # [L, H, N]
        kg = randn(*shape)
        kg = (kg * (math.sqrt(d) / kg.norm(dim=-1, keepdim=True))).half().float()       # equal norms: k_h . k_h leads
        vg = randn(*shape)
        kh = torch.gather(kg, 3, hot[None, ..., None].expand(chunks, L, heads, N, d))   # k of the hot key per row
        dots = kh @ kg.transpose(-1, -2)                                                # [c, L, H, N(f), N(g)]
        self_dot = dots.gather(-1, hot[None, ..., None].expand(chunks, -1, -1, -1, 1))
        others = dots.scatter(-1, hot[None, ..., None].expand(chunks, -1, -1, -1, 1), float("-inf")).amax(-1, True)
        gap = (self_dot - others).clamp(min=0.1) if N > 1 else self_dot
        qg = kh * (200.0 / (scale * gap))
        exact = torch.gather(vg.half().float(), 3, hot[None, ..., None].expand(chunks, L, heads, N, d))
        return _case(family, qg, kg, vg, fwd, ones, heads, scale, exact=exact)
    if family == "uniform":
        qg = randn(*shape)
        kg = randn(chunks, L, heads, 1, d).expand(*shape).contiguous()
        vg = torch.randint(-32, 33, shape, generator=g).float() / 8
        return _case(family, qg, kg, vg, fwd, ones, heads, scale, exact=vg.mean(3, keepdim=True).expand(*shape))
    if family == "masked-max":
        # keys of odd frames score hundreds of nats above the even ones and are masked for every other row
        qg, kg, vg = randn(*shape), 0.3 * randn(*shape), randn(*shape)
        fr = torch.arange(N, dtype=torch.float32)
        odd = fr.remainder(2) == 1
        qg[..., 0] = 4.0
        kg[..., 0] = torch.where(odd, (300.0 + 20.0 * fr) / (4.0 * scale), 0.0)
        mask = ~odd[None, None, :].expand(L, N, N) | eye
        return _case(family, qg, kg, vg, fwd, mask.clone(), heads, scale)
    if family == "huge":
        s = math.sqrt(1000.0 / (scale * math.sqrt(d)))             # logits ~ N(0, 1000^2) nats
        qg, kg, vg = s * randn(*shape), s * randn(*shape), randn(*shape)
        return _case(family, qg, kg, vg, fwd, _diag_kept_random_mask(L, N, g), heads, scale)
    if family == "floor":
        # shared direction: every logit about -100 nats
        qg, kg, vg = 0.3 * randn(*shape), randn(*shape), 1.0 + 0.1 * randn(*shape)
        qg[..., 0] = -10.0
        kg[..., 0] = (100.0 + 2.0 * torch.rand(chunks, L, heads, N, generator=g)) / (10.0 * scale)
        return _case(family, qg, kg, vg, fwd, _diag_kept_random_mask(L, N, g), heads, scale)
    if family.startswith("staircase"):
        # logit of key g rises (falls) by 1-4 nats per frame: several frames mix, frames >= 8 matter
        fr = torch.arange(N, dtype=torch.float32)
        if family.endswith("falling"):
            fr = N - 1 - fr
        qg, kg, vg = 0.02 * randn(*shape), randn(*shape), randn(*shape)
        qg[..., 0] = 1.0 + 3.0 * torch.rand(chunks, L, heads, N, generator=g)
        kg[..., 0] = fr / scale
        return _case(family, qg, kg, vg, fwd, ones, heads, scale)
    if family == "asymmetric":
        qg, kg, vg = 2.0 * randn(*shape), 2.0 * randn(*shape), randn(*shape)
        mask = _diag_kept_random_mask(L, N, g, 0.5)
        if N > 1:
            asym = (mask == mask.transpose(1, 2)).all(-1).all(-1)
            mask[asym, 0, 1] = True
            mask[asym, 1, 0] = False
        return _case(family, qg, kg, vg, fwd, mask, heads, scale)
    if family == "reference":
        gain = 1.0 + 2.0 * torch.rand(chunks, L, heads, 1, 1, generator=g)
        qg, kg = _layernorm(randn(*shape), gain), _layernorm(randn(*shape), gain)
        vg = randn(*shape)
        return _case(family, qg, kg, vg, fwd, reference_mask(N, L, g), heads, scale)
    raise ValueError(family)


def families_for(N):
    """The families that are defined at N frames (masked-max, staircase and asymmetric need two; uniform a power of
    two)."""
    fams = list(FAMILIES)
    if N & (N - 1):
        fams.remove("uniform")
    if N == 1:
        fams = [f for f in fams if f not in ("masked-max", "staircase-rising", "staircase-falling", "asymmetric")]
    return fams


# ---------------------------------------------------------------------------------------------- family properties
def family_property(case: Case) -> None:
    """Assert, on the fp64 logits, the property that makes the family sensitive; a change to a generator that made it
    harmless fails here."""
    qg, kg = (gather(t, case.fwd_map, case.chunks, case.heads) for t in (case.q, case.k))
    x = logits(qg, kg, case.mask, case.scale)
    keep = case.mask.bool()[None, :, None].expand_as(x)
    N = x.shape[-1]
    fam = case.family
    m = x.amax(-1, keepdim=True)
    if fam == "self-only":
        assert torch.equal(case.mask.bool(), torch.eye(N, dtype=torch.bool).expand_as(case.mask)), fam
    elif fam == "dominant":
        if N > 1:
            second = x.topk(2, -1).values
            gap = (second[..., 0] - second[..., 1]).min().item()
            assert gap > 150, f"{fam}: hot key only {gap:.1f} nats above the rest"
            hot = x.argmax(-1)
            for c in (0, N - 1, 8):
                if c < N:
                    assert (hot == c).any(), f"{fam}: no row's hot key is frame {c}"
    elif fam == "uniform":
        assert N & (N - 1) == 0, f"{fam}: N = {N} is not a power of two, 1/N is not exact"
        assert (x == x[..., :1]).all(), f"{fam}: logits of a row differ"
    elif fam == "masked-max":
        xm = torch.where(keep, float("-inf"), logits(qg, kg, torch.ones_like(case.mask), case.scale))
        lead = (xm.amax(-1) - x.amax(-1))[..., 0::2]                       # even rows: every odd key is masked
        assert lead.min().item() >= 100, f"{fam}: a masked key leads by only {lead.min().item():.1f} nats"
    elif fam == "huge":
        spread = (m.squeeze(-1) - torch.where(keep, x, m).amin(-1)).max().item()
        assert x[keep].abs().max().item() >= 1000 and (N == 1 or spread >= 1000), \
            f"{fam}: logits not spread over > 1000 nats"
        for t in (case.q, case.k):
            assert torch.isfinite(t).all(), f"{fam}: fp16 operands overflow"
    elif fam == "floor":
        xk = x[keep]
        assert xk.max().item() <= -90 and xk.min().item() >= -110, f"{fam}: logits in [{xk.min():.1f}, {xk.max():.1f}]"
    elif fam.startswith("staircase"):
        step = x[..., 1:] - x[..., :-1]
        step = -step if fam.endswith("falling") else step
        assert step.min().item() >= 0.8 and step.max().item() <= 4.5, \
            f"{fam}: per-frame step in [{step.min().item():.2f}, {step.max().item():.2f}] nats"
        if N > 8:
            w = torch.softmax(x, -1)
            late = w[..., 8:].sum(-1) if fam.endswith("rising") else w[..., :8].sum(-1)
            assert late.min().item() >= 0.5, f"{fam}: frames past 8 hold only {late.min().item():.2f} of a row"
    elif fam == "asymmetric":
        assert (case.mask.diagonal(dim1=1, dim2=2)).all(), f"{fam}: a diagonal entry is masked"
        if N > 1:
            asym = (case.mask != case.mask.transpose(1, 2)).flatten(1).any(-1)
            assert asym.all(), f"{fam}: {(~asym).sum().item()} trajectories with a symmetric mask"
    elif fam == "reference":
        assert (case.mask.diagonal(dim1=1, dim2=2)).all(), f"{fam}: a diagonal entry is masked"
        if case.fwd_map.shape[1] > 1:
            ident = (case.fwd_map == torch.arange(case.fwd_map.shape[1], device=case.fwd_map.device)).all(-1)
            assert not ident.any(), f"{fam}: a frame's map is the identity"
        if N > 1:
            cuts = [(~case.mask[:, :i + 1, i + 1:]).flatten(1).all(-1).any().item() for i in range(N - 1)]
            assert all(cuts), f"{fam}: cuts at {[i for i, c in enumerate(cuts) if not c]} never used"
        spread = (m.squeeze(-1) - torch.where(keep, x, m).amin(-1)).amax().item()
        assert N == 1 or spread >= 10, f"{fam}: logits spread over only {spread:.1f} nats"
    else:
        raise ValueError(fam)
