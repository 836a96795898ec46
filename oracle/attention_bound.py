"""fp64 reference of fresco_attn_fwd, an elementwise bound on the fp16 kernel's error, and adversarial input families.

CHECKER ONLY (see ``oracle/__init__``).  Layout as the kernel's: q [B, Lq, H*d], k / v [B / q_per_kv, Lk, H*d], fp16,
token-major.  ``scale`` and ``diag_bias`` are rounded to fp32 first, since the C ABI passes them as floats; everything
else is evaluated in fp64 from the fp16 operands exactly as the kernel reads them.

The bound
---------
For one row i and channel c of one head, with raw scores s_ij = q_i . k_j, logits x_ij = scale s_ij + bias [i == j],
m_i = max_j x_ij, exact weights w_ij = exp(x_ij - m_i) / l_i, l_i = sum_j exp(x_ij - m_i), and u = 2^-24:

    A_ic = sum_j w_ij |v_jc|       Z_ic = (sum_j |v_jc| + [ROWSUM] Lk |ref_ic|) / l_i

    tol = F * ( (2^-11 + (Lk/4 + 5) u) |ref| + 2^-25
              + (2^-10 + 2 eps_i + 2 sigma_i + (Lk/16 + 2 n_tiles) u) A
              + 2^-25 Z )

Each term, in the order the kernel does the work:

* ``2 sigma_i A`` -- fp32 S.  The products of fp16 operands are exact in fp32; accumulating d of them errs by at most
  d u sum_k |q_ik k_jk| in raw units, so every logit of row i by at most
  sigma_i = scale d u max_j sum_k |q_ik k_jk| + u |bias| (the second part: diag_bias / softmax_scale rounded to fp32).
  A relative perturbation rho_j of each weight's numerator moves sum_j w_j v_j / sum_j w_j by at most
  max|rho| (A + |ref|) <= 2 max|rho| A, hence the factor 2 (a perturbation common to the whole row, such as an error
  in m, cancels).
* ``2 eps_i A`` -- the exponential.  p = exp2(fma(s, c, -m c)) with c = fp32(scale log2 e).  The argument carries the
  rounding of the FFMA (u |x|), of m c (u |m c|), of c itself (u |x|) and of the biased score s + bias (u |s + bias|),
  all in log2 units; |x| <= 2 X_i and |m c|, |s + bias| <= X_i with X_i = max_j |x_ij| log2 e, so the relative error
  of p is at most ln 2 * 5 u X_i = 5 u max_j |x_ij|.  On top comes the exponential itself: ex2.approx.ftz.f32 is
  within 2 ulp (2^-22); the POLY variants' exp2_poly within 7.5e-5, taken as 1e-4.
  eps_i = (2^-22 or 1e-4) + 5 u max_j |x_ij|.  alpha needs no term: the same fp32 alpha scales O and l.
* ``2^-10 A`` -- P rounded to fp16 (relative 2^-11 while P is a normal fp16) enters the numerator; the denominator
  sums the fp32 p (2^-11 |ref| <= 2^-11 A from the mismatch) or, under ROWSUM, the same fp16 P (2^-11 A through l).
* ``2^-25 Z`` -- P below the fp16 normal range 2^-14 is rounded with an absolute error of at most 2^-25 per key
  (also P flushed or rounded to zero), which moves the numerator by 2^-25 sum_j |v_jc| and, under ROWSUM, l by
  2^-25 Lk; both over l_i.
* ``(Lk/16 + 2 n_tiles) u A`` -- O accumulated in fp32: one accumulator add per 16-key wgmma step, and per key tile one
  rescale by alpha and one add of the tile's P V.  n_tiles = ceil(Lk / 64), the most tiles any variant makes.
* ``(Lk/4 + 5) u |ref|`` -- l in fp32: each lane of a quad sums Lk/4 exponentials in sequence, then two quad shuffles
  add the four partial sums; __fdividef(1, l) within 2 ulp and O * (1 / l) one more rounding.
* ``2^-11 |ref| + 2^-25`` -- the output rounded to fp16: relative 2^-11, absolute 2^-25 below the normal range.

The terms are first order.  F = 2 is the one safety factor: it covers the products of first-order errors and the
accumulation order inside the tensor core, which is not documented.  Nothing else is widened.
"""
from __future__ import annotations

import math
from typing import NamedTuple

import numpy as np
import torch

U = 2.0 ** -24
SAFETY = 2.0
EPS_EX2 = 2.0 ** -22          # ex2.approx.ftz.f32
EPS_POLY = 1e-4               # exp2_poly of the POLY variants (7.5e-5 measured in test_attention_numerics_model)


def _f32(x: float) -> float:
    return float(np.float32(x))


def _heads(t: torch.Tensor, heads: int) -> torch.Tensor:
    """[B, L, H*d] -> [B, H, L, d] fp64."""
    B, L, C = t.shape
    return t.double().reshape(B, L, heads, C // heads).transpose(1, 2)


def _logits(q, k, heads, q_per_kv, scale, diag_bias, rows=None):
    """fp64 logits [B, H, Lq, Lk] (nats) and raw |q| . |k| row maxima, from the fp16 operands.  ``rows`` (int64 [Lq]):
    the absolute query index of each row of ``q`` when it is a subset of the rows, which the diagonal bias follows."""
    qh, kh = _heads(q, heads), _heads(k, heads).repeat_interleave(q_per_kv, 0)
    x = (qh @ kh.transpose(-1, -2)) * _f32(scale)
    bias = _f32(diag_bias)
    if bias != 0.0:
        if rows is None:
            diag = torch.eye(q.shape[1], k.shape[1], dtype=torch.float64, device=q.device)
        else:
            diag = (rows.to(q.device)[:, None] == torch.arange(k.shape[1], device=q.device)[None]).double()
        x = x + diag * bias
    return x, qh, kh


def ref_and_bound(q, k, v, heads, q_per_kv=1, scale=None, diag_bias=0.0, poly=0, rowsum=False, rows=None):
    """(attention_ref, attention_bound) in one pass, fp64 [B, Lq, H*d].  ``rows``: see ``_logits``."""
    B, Lq, C = q.shape
    d, Lk = C // heads, k.shape[1]
    scale = 1.0 / math.sqrt(d) if scale is None else scale
    x, qh, kh = _logits(q, k, heads, q_per_kv, scale, diag_bias, rows)
    vh = _heads(v, heads).repeat_interleave(q_per_kv, 0)
    m = x.amax(-1, keepdim=True)
    e = torch.exp(x - m)
    l = e.sum(-1, keepdim=True)
    w = e / l
    ref = w @ vh
    A = w @ vh.abs()
    Z = vh.abs().sum(-2, keepdim=True) / l
    if rowsum:
        Z = Z + Lk * ref.abs() / l
    sigma = _f32(scale) * d * U * (qh.abs() @ kh.abs().transpose(-1, -2)).amax(-1, keepdim=True) + U * abs(_f32(diag_bias))
    eps = (EPS_POLY if poly else EPS_EX2) + 5 * U * x.abs().amax(-1, keepdim=True)
    n_tiles = (Lk + 63) // 64
    tol = SAFETY * ((2.0 ** -11 + (Lk / 4 + 5) * U) * ref.abs() + 2.0 ** -25
                    + (2.0 ** -10 + 2 * eps + 2 * sigma + (Lk / 16 + 2 * n_tiles) * U) * A
                    + 2.0 ** -25 * Z)

    def tok(t):
        return t.transpose(1, 2).reshape(B, Lq, C)
    return tok(ref), tok(tol)


def attention_ref(q, k, v, heads, q_per_kv=1, scale=None, diag_bias=0.0):
    """softmax(scale q k^T + diag_bias eye(Lq, Lk)) v in fp64, token-major [B, Lq, H*d]."""
    return ref_and_bound(q, k, v, heads, q_per_kv, scale, diag_bias)[0]


def attention_bound(q, k, v, heads, q_per_kv=1, scale=None, diag_bias=0.0, poly=0, rowsum=False):
    """Elementwise tolerance of the fp16 kernel against attention_ref (module docstring)."""
    return ref_and_bound(q, k, v, heads, q_per_kv, scale, diag_bias, poly, rowsum)[1]


# ============================================================================================== adversarial families
class Case(NamedTuple):
    family: str
    q: torch.Tensor
    k: torch.Tensor
    v: torch.Tensor
    heads: int
    q_per_kv: int
    scale: float
    diag_bias: float


def _tok(t):
    """[B, H, L, d] fp32 -> token-major [B, L, H*d] fp16."""
    B, H, L, d = t.shape
    return t.transpose(1, 2).reshape(B, L, H * d).half().contiguous()


def _gen(seed, device):
    return torch.Generator(device=device).manual_seed(seed)


def _randn(shape, g, device):
    return torch.randn(*shape, generator=g, device=device)


def staircase(d, Lq, Lk, kind="rising", kn=64, heads=1, seed=0, device="cpu"):
    """Head-dim coordinate 0 is a ramp over the keys: row i's logits rise by rise_i in [0.2, 0.4) nat per 64 keys
    (rise_i differs between rows i and i + 8, the two rows a thread holds), plus ~0.03 nat of noise.  kind "falling"
    reverses the ramp (the max is set in the first tile); "sawtooth" drops every odd kn-key tile by two tiles' worth, so
    the max rises every other tile.  V channel 0 is the key's 64-key block index (exact in fp16)."""
    g = _gen(seed, device)
    scale = 1.0 / math.sqrt(d)
    j = torch.arange(Lk, device=device, dtype=torch.float32)
    if kind == "rising":
        level = j / 64
    elif kind == "falling":
        level = (Lk - 1 - j) / 64
    elif kind == "sawtooth":
        level = j / 64 - torch.where((j // kn) % 2 == 1, 2.0 * kn / 64, 0.0)
    else:
        raise ValueError(kind)
    i = torch.arange(Lq, device=device)
    a = 1.0 + ((7 * i) % 16).float() / 16                     # rise_i = 0.2 a_i
    q = 0.03 * _randn((1, heads, Lq, d), g, device)
    k = _randn((1, heads, Lk, d), g, device)
    v = _randn((1, heads, Lk, d), g, device)
    q[..., 0] = a
    k[..., 0] = level * (0.2 / scale)
    v[..., 0] = torch.div(j, 64, rounding_mode="floor")
    return Case("staircase-" + kind, _tok(q), _tok(k), _tok(v), heads, 1, scale, 0.0)


def hot_keys(Lq, Lk, kn):
    """Row i's hot key: first tile, last full tile, the ragged last key, both sides of 16-key k-step boundaries."""
    cand = [0, Lk - 1, 15, 16, 31, 32, kn - 1, kn, (Lk // kn - 1) * kn + 7, Lk - 17, Lk - 16, Lk // 2]
    cand = [c for c in cand if 0 <= c < Lk]
    return torch.tensor([cand[i % len(cand)] for i in range(Lq)])


def one_hot(d, Lq, Lk, kn=64, heads=1, seed=0, device="cpu"):
    """q_i = lambda_i k_h(i): the hot key scores >= 35 nats above every other key of the row.  V channel 0 is
    key mod 2048, channel 1 key // 2048, so output row i reads back which key it used."""
    g = _gen(seed, device)
    scale = 1.0 / math.sqrt(d)
    k = _randn((1, heads, Lk, d), g, device)
    v = _randn((1, heads, Lk, d), g, device)
    j = torch.arange(Lk, device=device, dtype=torch.float32)
    v[..., 0] = j % 2048
    v[..., 1] = torch.div(j, 2048, rounding_mode="floor")
    hot = hot_keys(Lq, Lk, kn).to(device)
    kh = k.half().float()
    kq = kh[:, :, hot]                                           # [1, H, Lq, d]
    dots = kq @ kh.transpose(-1, -2)                             # [1, H, Lq, Lk]
    self_dot = dots.gather(-1, hot.view(1, 1, -1, 1).expand(1, heads, -1, 1))
    others = dots.scatter(-1, hot.view(1, 1, -1, 1).expand(1, heads, -1, 1), float("-inf")).amax(-1, keepdim=True)
    gap = (self_dot - others).clamp(min=1.0) if Lk > 1 else self_dot
    lam = 40.0 / (scale * gap)
    return Case("one-hot", _tok(kq * lam), _tok(k), _tok(v), heads, 1, scale, 0.0)


def negative_floor(d, Lq, Lk, heads=1, seed=0, device="cpu"):
    """Every logit in [-31, -24] nats; V = 1 + noise.  A zero-filled key past kv_len (logit 0, V = 0) would take
    the row."""
    g = _gen(seed, device)
    scale = 1.0 / math.sqrt(d)
    q = 0.3 * _randn((1, heads, Lq, d), g, device) / math.sqrt(d)
    k = _randn((1, heads, Lk, d), g, device)
    q[..., 0] = -25.0 / (10.0 * scale)
    k[..., 0] = 10.0 + 2.0 * torch.rand(1, heads, Lk, generator=g, device=device)
    v = 1.0 + 0.1 * _randn((1, heads, Lk, d), g, device)
    return Case("negative-floor", _tok(q), _tok(k), _tok(v), heads, 1, scale, 0.0)


def flat(d, Lq, Lk, heads=1, seed=0, device="cpu"):
    """intraattn_scale_factor 0.2 and small q: every logit within a few hundredths of a nat, the output the mean
    of V = 1 + noise, so an error in l shows in full."""
    g = _gen(seed, device)
    q = 0.05 * _randn((1, heads, Lq, d), g, device)
    k = _randn((1, heads, Lk, d), g, device)
    v = 1.0 + 0.25 * _randn((1, heads, Lk, d), g, device)
    return Case("flat", _tok(q), _tok(k), _tok(v), heads, 1, 0.2 / math.sqrt(d), 0.0)


def diagonal(d, Lq, Lk, bias, heads=1, seed=0, device="cpu"):
    """Spatial-guided attention: softmax_scale 0.2 / sqrt(d) and diag_bias on key == query."""
    g = _gen(seed, device)
    q = _randn((1, heads, Lq, d), g, device)
    k = _randn((1, heads, Lk, d), g, device)
    v = _randn((1, heads, Lk, d), g, device)
    return Case("diagonal%+g" % bias, _tok(q), _tok(k), _tok(v), heads, 1, 0.2 / math.sqrt(d), float(bias))


def peaky(d, Lq, Lk, heads=1, seed=0, device="cpu"):
    """Logits with a spread of ~20 nats: most of P is subnormal or zero in fp16."""
    g = _gen(seed, device)
    q = 5.0 * _randn((1, heads, Lq, d), g, device)
    k = 4.0 * _randn((1, heads, Lk, d), g, device)
    v = _randn((1, heads, Lk, d), g, device)
    return Case("peaky", _tok(q), _tok(k), _tok(v), heads, 1, 1.0 / math.sqrt(d), 0.0)


# ---------------------------------------------------------------------------------------------- family properties
def family_property(case: Case, kn: int = 64) -> None:
    """Assert, on the fp64 logits, the property that makes the family sensitive; a change to a generator that made it
    harmless fails here."""
    x, _, _ = _logits(case.q, case.k, case.heads, case.q_per_kv, case.scale, case.diag_bias)
    x = x.flatten(0, 1)                                          # [B*H, Lq, Lk]
    Lq, Lk = x.shape[-2:]
    fam = case.family
    if fam.startswith("staircase"):
        nb = Lk // 64
        assert nb >= 9, f"{fam}: {nb} full 64-key blocks, want >= 9"
        bm = x[..., :nb * 64].unflatten(-1, (nb, 64)).amax(-1)    # block maxima [., Lq, nb]
        w = torch.softmax(x, -1)[..., :nb * 64].unflatten(-1, (nb, 64)).sum(-1)
        run = torch.cummax(bm, -1).values
        if fam == "staircase-rising":
            rise = bm[..., 1:] - run[..., :-1]
            assert rise.min() >= 0.1, f"{fam}: the row max rises by only {rise.min().item():.3f} nat in some block"
            assert w[..., -8:].min() >= 0.005, f"{fam}: a late block holds {w[..., -8:].min().item():.2e} of a row"
        elif fam == "staircase-falling":
            assert (bm[..., 0] >= bm.amax(-1)).all(), f"{fam}: the row max is not in the first block"
        else:
            tiles = Lk // kn
            assert tiles >= 4, f"{fam}: {tiles} full tiles"
            tm = x[..., :tiles * kn].unflatten(-1, (tiles, kn)).amax(-1)
            trun = torch.cummax(tm, -1).values
            for u in range(1, tiles):
                step = (tm[..., u] - trun[..., u - 1]) * (1 if u % 2 == 0 else -1)
                assert step.min() >= 0.1, f"{fam}: tile {u} does not {'raise' if u % 2 == 0 else 'stay below'} the max"
    elif fam == "one-hot":
        top2 = x.topk(min(2, Lk), -1).values
        hot = x.argmax(-1)
        want = hot_keys(Lq, Lk, kn).to(hot.device)
        assert (hot == want).all(), f"{fam}: a row's largest logit is not its hot key"
        if Lk > 1:
            gap = (top2[..., 0] - top2[..., 1]).min().item()
            assert gap >= 30, f"{fam}: hot key only {gap:.1f} nats above the rest"
    elif fam == "negative-floor":
        assert x.amax().item() <= -20, f"{fam}: a logit of {x.amax().item():.1f} nats, want <= -20"
    elif fam == "flat":
        spread = (x.amax(-1) - x.amin(-1)).max().item()
        assert spread <= 0.5, f"{fam}: logits spread over {spread:.2f} nats"
    elif fam.startswith("diagonal"):
        n = min(Lq, Lk)
        wd = torch.softmax(x, -1).diagonal(dim1=-2, dim2=-1)[..., :n]
        if case.diag_bias >= 8:
            assert wd.min() >= 0.5, f"{fam}: the diagonal key holds only {wd.min().item():.2f} of a row"
        elif case.diag_bias <= -8:
            assert wd.max() <= 1e-3 / Lk, f"{fam}: the diagonal key keeps {wd.max().item():.2e} of a row"
        else:
            assert (wd * Lk).median() >= 2.0, f"{fam}: the diagonal key is not favoured"
    elif fam == "peaky":
        p = torch.exp(x - x.amax(-1, keepdim=True))             # P before normalisation, as the kernel rounds it
        sub = (p < 2.0 ** -14).double().mean().item()
        spread = (x.amax(-1) - x.amin(-1)).min().item()
        assert sub >= 0.8 and spread >= 60, f"{fam}: {sub:.2f} of P subnormal, spread {spread:.0f} nats"
    else:
        raise ValueError(fam)
