"""The arithmetic of the attention kernel (fresco_attn_kernel, attn_wgmma.cu), restated in torch on the CPU.

* exp2_poly: the FMA-pipe exponential of the POLY variants -- clamp, round-to-nearest by the 1.5 * 2^23 trick, degree-3
  minimax on [-0.5, 0.5], exponent patched in with an integer add.  Its error must stay inside the fp16 rounding of P,
  and very negative arguments (masked keys) must give ~0.
* ``emulate``: the online softmax tile by tile -- KN-key tiles, fp32 S from the fp16 operands, the row max on raw
  scores, alpha and p as exp2(fma(s, c, -m c)) in fp32 (exp2_poly on the pairs the POLY variants give it), P rounded to
  fp16, O accumulated in fp32 and rescaled after each tile, l from the fp32 p (or from the fp16 P under ROWSUM), the
  output rounded to fp16.  It checks the error model of ``oracle.attention_bound`` without a GPU: the emulator stays
  inside the bound on every adversarial input family, and five one-line mistakes a schedule change could make
  (``MUTANTS``) each leave it on at least one family.
"""
import math

import numpy as np
import pytest
import torch

from oracle import attention_bound as AB


def exp2_poly(t):
    """exp2_poly of attn_wgmma.cu in fp32."""
    t = torch.clamp(t, min=-126.0)
    magic = torch.tensor(12582912.0)
    r = t + magic
    n = r - magic
    f = t - n
    q = torch.tensor(0.05517164617776871) * f + torch.tensor(0.2426111251115799)
    q = q * f + torch.tensor(0.6932609677314758)
    q = q * f + torch.tensor(0.9999280571937561)
    bits = q.view(torch.int32) + (r.view(torch.int32) << 23)
    return bits.view(torch.float32)


def test_polynomial_exp2_error_and_range():
    t = torch.linspace(-100.0, 9.0, 200001)                         # (P is fp16: anything below 2^-25 rounds to zero anyway)
    ref = torch.exp2(t.double())
    rel = ((exp2_poly(t).double() - ref) / ref).abs().max().item()
    assert rel < 1e-4, rel                                          # 7.5e-5 by design: inside the fp16 rounding of P
    edge = exp2_poly(torch.tensor([-1e30, -140.0, -126.0, 0.0, 8.0]))
    assert torch.isfinite(edge).all() and (edge[:3] < 2e-38).all() and abs(edge[3].item() - 1.0) < 1e-4


# ------------------------------------------------------------------------------------------------ the kernel, emulated
MUTANTS = {
    "M1": "tail mask off by one: col > kv_len, so the zero-filled key at kv_len joins the row",
    "M2": "diagonal-tile test with one warpgroup's rows: q0 + 64 > col0",
    "M3": "O rescaled with the first row's alpha for both rows a thread holds",
    "M4": "l *= alpha after the tile's exponentials are added to l",
    "M5": "ROWSUM: l rescaled with the first row's alpha for both rows a thread holds",
}


def _f32(x):
    return float(np.float32(x))


def emulate(case, kn, nwg=2, poly=0, rowsum=False, mutant=None):
    """fresco_attn_kernel<d, kn, nwg, poly, rowsum> on the CPU (q_per_kv = 1), optionally with one of MUTANTS."""
    B, Lq, C = case.q.shape
    H = case.heads
    d, Lk = C // H, case.k.shape[1]
    tile_m = 64 * nwg
    scale = _f32(case.scale)
    c = torch.tensor(scale, dtype=torch.float32) * torch.tensor(1.4426950408889634, dtype=torch.float32)
    bias_raw = torch.tensor(_f32(case.diag_bias), dtype=torch.float32) / torch.tensor(scale, dtype=torch.float32)
    rows = torch.arange(Lq)
    second = (rows % 16) >= 8                                     # the thread's row + 8 (alpha[1], l_run[1])
    partner = torch.where(second, rows - 8, rows)                 # the row whose alpha[0] that thread holds
    out = torch.empty(B, Lq, C, dtype=torch.float16)
    for b in range(B):
        for h in range(H):
            sl = slice(h * d, (h + 1) * d)
            qh = case.q[b, :, sl].float().cpu()
            kh = case.k[b // case.q_per_kv, :, sl].float().cpu()
            vh = case.v[b // case.q_per_kv, :, sl].float().cpu()
            kv_len = Lk
            if mutant == "M1" and Lk % kn:                        # TMA zero-fills the key at kv_len
                kh = torch.cat([kh, torch.zeros(1, d)])
                vh = torch.cat([vh, torch.zeros(1, d)])
                kv_len = Lk + 1
            n_tiles = (Lk + kn - 1) // kn
            s = torch.full((Lq, n_tiles * kn), float("-inf"))
            s[:, :kv_len] = qh @ kh.T
            vp = torch.zeros(n_tiles * kn, d)
            vp[:kv_len] = vh
            if case.diag_bias != 0.0:
                for i in range(min(Lq, kv_len)):
                    col0, q0 = i // kn * kn, i // tile_m * tile_m
                    if mutant == "M2" and not (col0 + kn > Lk or (q0 < col0 + kn and q0 + 64 > col0)):
                        continue
                    s[i, i] = s[i, i] + bias_raw
            col = torch.arange(kn)
            pair = 2 * (col // 8)[None, :] + second[:, None].long()
            use_poly = (pair % poly == poly - 1) if poly else torch.zeros(Lq, kn, dtype=torch.bool)
            m = torch.full((Lq,), float("-inf"))
            l = torch.zeros(Lq)
            o = torch.zeros(Lq, d)
            for t in range(n_tiles):
                st = s[:, t * kn:(t + 1) * kn]
                m_new = torch.maximum(m, st.amax(1))
                alpha = torch.exp2((m - m_new) * c)
                neg_ms = -(m_new * c)
                m = m_new
                x = (st.double() * c.double() + neg_ms.double()[:, None]).float()   # one FFMA
                p = torch.exp2(x)
                p = torch.where(p < 2.0 ** -126, torch.zeros(()), p)             # ex2.approx.ftz
                if poly:
                    p = torch.where(use_poly, exp2_poly(x), p)
                p16 = p.half().float()
                a_o = alpha[partner] if mutant == "M3" else alpha
                if rowsum:
                    a_l = alpha[partner] if mutant == "M5" else alpha
                    l = l * a_l + p16.sum(1)
                elif mutant == "M4":
                    l = (l + p.sum(1)) * alpha
                else:
                    l = l * alpha + p.sum(1)
                o = o * a_o[:, None] + p16 @ vp[t * kn:(t + 1) * kn]
            out[b, :, sl] = (o * (1.0 / l)[:, None]).half()
    return out


def cpu_families(kn):
    """Every input family of tests/test_gpu_attention_edges.py at CPU sizes (d = 40, 136 query rows: two CTAs of
    128 rows, a warpgroup of 64 that is partly past q_len)."""
    d, Lq = 40, 136
    out = [AB.staircase(d, Lq, 9 * 128 + 37, kind, kn=kn, seed=1) for kind in ("rising", "falling", "sawtooth")]
    out.append(AB.one_hot(d, Lq, 4 * kn + 1, kn=kn, seed=2))
    out.append(AB.negative_floor(d, Lq, 3 * kn + 5, seed=3))
    out.append(AB.flat(d, Lq, 2000, seed=4))
    for bias in (8.0, -8.0, 1.5):
        out.append(AB.diagonal(d, 193, 193, bias, seed=5))
    out.append(AB.diagonal(d, 193, 2 * 193 - 5, 8.0, seed=6))
    out.append(AB.diagonal(d, 193, 193 // 2 + 3, 8.0, seed=7))
    out.append(AB.peaky(d, Lq, 500, seed=8))
    return out


def _ratio(case, got, poly, rowsum):
    ref, tol = AB.ref_and_bound(case.q, case.k, case.v, case.heads, case.q_per_kv, case.scale, case.diag_bias, poly,
                                rowsum)
    return ((got.double() - ref).abs() / tol).nan_to_num(nan=float("inf"))


@pytest.mark.parametrize("kn", [64, 128])
def test_families_have_their_property(kn):
    for case in cpu_families(kn):
        AB.family_property(case, kn)


@pytest.mark.parametrize("kn", [64, 128])
@pytest.mark.parametrize("poly", [0, 4, 8])
@pytest.mark.parametrize("rowsum", [False, True])
def test_emulated_kernel_within_bound(kn, poly, rowsum):
    """The error model: the kernel's arithmetic, restated, stays inside attention_bound on every family."""
    for case in cpu_families(kn):
        r = _ratio(case, emulate(case, kn, poly=poly, rowsum=rowsum), poly, rowsum)
        assert r.max().item() <= 1.0, f"{case.family}: emulated err / bound {r.max().item():.3g}"


# mutant -> (variant, the family that must catch it)
MUTANT_CASES = {
    "M1": (dict(kn=64), "negative-floor"),
    "M2": (dict(kn=64), "diagonal+8"),
    "M3": (dict(kn=128), "staircase-rising"),
    "M4": (dict(kn=64), "staircase-rising"),
    "M5": (dict(kn=64, rowsum=True), "staircase-rising"),
}


@pytest.mark.parametrize("mutant", sorted(MUTANTS))
def test_emulated_mutants_leave_the_bound(mutant):
    """Each mutant breaks the bound on the family built to expose it, so the families are sensitive to it."""
    cfg, family = MUTANT_CASES[mutant]
    caught = []
    for case in cpu_families(cfg["kn"]):
        r = _ratio(case, emulate(case, mutant=mutant, **cfg), 0, cfg.get("rowsum", False))
        if r.max().item() > 1.0:
            caught.append(case.family)
    assert family in caught, f"{mutant} ({MUTANTS[mutant]}) is caught only by {caught}"
