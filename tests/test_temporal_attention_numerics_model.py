"""Both temporal-guided attention kernels (A5, hbm_kernels.cu), restated in torch fp32 on the CPU.

``emulate`` follows each kernel's arithmetic operation by operation:

* fp16 x fp16 products are exact in fp32, so each FMA of the dot product is one fp32 add of the exact product;
  ``temporal_attn_rows_kernel`` runs two interleaved chains (even and odd channels) and adds them, the round-1
  ``temporal_attn_kernel`` one chain over the channels in order;
* rows: sc = fl(fl(a0 + a1) c2) with c2 = fl(fp32(scale) fl(log2 e)) from the host, p = exp2(fl(sc - mx));
  round-1: r = fl(acc scale), p = exp2(fl(fl(r - m) log2 e)) for __expf.  torch's fp32 exp2 stands in for the
  hardware exponentials, whose error the bound already carries; results below 2^-126 are flushed to zero (ftz);
* l a sequential fp32 sum over the frames, inv = 1 / l, pw = fl(p inv);
* per channel N sequential FMAs fma(pw, v, acc): the product of an fp32 and an fp16 value is exact in fp64, so the
  FMA is evaluated in fp64 and rounded to fp32 once (double rounding can differ from the hardware's single rounding in
  the last bit, well inside the bound);
* the output rounded to fp16.

The tests check that the emulation stays inside ``oracle.temporal_bound`` on every input family, that the exact
families come out bit for bit, and that seven one-line mutants of the kernels' arithmetic each leave the bound on a
named family -- the bound is tight enough to see them.
"""
import math

import numpy as np
import pytest
import torch

from oracle import temporal_bound as TB

LOG2E = float(np.float32(1.4426950408889634))
FLT_MIN = 2.0 ** -126
MUTANTS = {
    # mutant: the families that must catch it
    "mask-after-max": ("masked-max",),
    "no-max-subtraction": ("huge", "floor"),
    "scale-without-log2e": ("staircase-rising", "staircase-falling", "asymmetric", "reference"),
    "transposed-mask": ("asymmetric",),
    "last-frame-not-in-l": ("staircase-rising",),
    "q-through-fwd0": ("reference",),
    "fp16-dot": ("staircase-rising", "reference"),
}
ROUND1_MUTANTS = [m for m in MUTANTS if m != "scale-without-log2e"]   # the round-1 kernel has no log2 scaling


def _f32(x):
    return float(np.float32(x))


def emulate(case, kernel="rows", mutant=None):
    """fp16 output of the kernel on ``case`` in the gathered layout [chunks, tokens, heads, N, d] (fp64 values)."""
    qmap = case.fwd_map[:1].expand_as(case.fwd_map) if mutant == "q-through-fwd0" else case.fwd_map
    qg = TB.gather(case.q, qmap, case.chunks, case.heads).float()
    kg, vg = (TB.gather(t, case.fwd_map, case.chunks, case.heads).float() for t in (case.k, case.v))
    N, d = qg.shape[-2:]
    keep = case.mask.bool()[None, :, None]                                 # [1, L, 1, f, g]
    if mutant == "transposed-mask":
        keep = keep.transpose(-1, -2)
    prods = lambda c: qg[..., :, None, c] * kg[..., None, :, c]          # exact in fp32: [c, L, H, f, g]
    fp16_dot = mutant == "fp16-dot"

    def add(a, b):
        s = a + b
        return s.half().float() if fp16_dot else s
    if kernel == "rows":
        a0 = torch.zeros(qg.shape[:-1] + (N,))
        a1 = torch.zeros_like(a0)
        for c in range(0, d, 2):
            a0, a1 = add(a0, prods(c)), add(a1, prods(c + 1))
        c2 = _f32(case.scale) if mutant == "scale-without-log2e" else _f32(_f32(case.scale) * LOG2E)
        sc = (a0 + a1) * c2
    else:
        acc = torch.zeros(qg.shape[:-1] + (N,))
        for c in range(d):
            acc = add(acc, prods(c))
        sc = acc * _f32(case.scale)
    if mutant == "mask-after-max":
        mx = sc.amax(-1, keepdim=True)
        sc = sc.masked_fill(~keep, float("-inf"))
    else:
        sc = sc.masked_fill(~keep, float("-inf"))
        mx = sc.amax(-1, keepdim=True)
    if mutant == "no-max-subtraction":
        mx = torch.zeros_like(mx)
    if kernel == "rows":
        p = torch.exp2(sc - mx)
    else:
        p = torch.exp2((sc - mx) * LOG2E)
    p = torch.where(p < FLT_MIN, 0.0, p)                                   # ftz
    l = torch.zeros(p.shape[:-1])
    for g in range(N - 1 if mutant == "last-frame-not-in-l" else N):
        l = l + p[..., g]
    inv = 1.0 / l
    pw = p * inv[..., None]
    out = torch.zeros(qg.shape)
    for g in range(N):
        out = (pw[..., g, None].double() * vg[..., g, None, :].double() + out.double()).float()
    return out.half().double()


def _cases(kernel):
    """(N, heads, d) shapes per kernel: the row kernel's NMAX = 8 and 16 slots, a ragged N, N = 1; the round-1 kernel
    past 16 and 32 frames and at head dims the row kernel has no instantiation for."""
    if kernel == "rows":
        return [(1, 2, 40), (2, 2, 40), (5, 2, 64), (8, 1, 80), (12, 2, 40), (16, 1, 40)]
    return [(4, 1, 8), (8, 2, 24), (17, 1, 40), (33, 1, 16)]


def _case(fam, N, heads, d, seed=0):
    return TB.make_case(fam, N, L=24, heads=heads, d=d, chunks=2, seed=seed)


@pytest.mark.parametrize("kernel", TB.KERNELS)
def test_family_properties(kernel):
    for N, heads, d in _cases(kernel):
        for fam in TB.families_for(N):
            TB.family_property(_case(fam, N, heads, d))


@pytest.mark.parametrize("kernel", TB.KERNELS)
def test_emulation_within_bound(kernel):
    """Every family at every shape: the emulated kernel inside the bound; the exact families bit for bit."""
    worst = {}
    for N, heads, d in _cases(kernel):
        for fam in TB.families_for(N):
            case = _case(fam, N, heads, d)
            out = emulate(case, kernel)
            ref, tol = TB.ref_and_bound(case.q, case.k, case.v, case.fwd_map, case.mask, case.chunks, case.heads,
                                        case.scale, kernel, gathered=True)
            r = TB.ratio(out, ref, tol)
            worst[fam] = max(worst.get(fam, 0.0), r.max().item())
            assert r.max().item() <= 1, f"{kernel} {fam} N={N} d={d}: err/tol {r.max().item():.3g}"
            if fam in TB.EXACT:
                want = TB.gather(case.exact, case.fwd_map, case.chunks, case.heads)
                assert torch.equal(out, want), f"{kernel} {fam} N={N} d={d}: not bit-exact"
    print(kernel, {f: round(v, 3) for f, v in worst.items()})


@pytest.mark.parametrize("kernel,mutant", [("rows", m) for m in MUTANTS] + [("round1", m) for m in ROUND1_MUTANTS])
def test_mutant_caught(kernel, mutant):
    """Each mutant leaves the bound on every family named for it, at a shape with frames past slot 8."""
    N, heads, d = (12, 2, 40) if kernel == "rows" else (17, 1, 40)
    for fam in MUTANTS[mutant]:
        case = _case(fam, N, heads, d)
        ref, tol = TB.ref_and_bound(case.q, case.k, case.v, case.fwd_map, case.mask, case.chunks, case.heads,
                                    case.scale, kernel, gathered=True)
        assert TB.ratio(emulate(case, kernel), ref, tol).max().item() <= 1, f"{fam}: the kernel itself fails"
        r = TB.ratio(emulate(case, kernel, mutant), ref, tol).max().item()
        assert r > 1, f"{kernel} mutant {mutant} stays inside the bound on {fam} (err/tol {r:.3g})"


def test_bound_is_not_loose():
    """On the mixing families the emulated error reaches a visible share of the bound: a bound many orders above the
    kernel's error would catch nothing."""
    for fam in ("reference", "staircase-rising"):
        case = _case(fam, 12, 2, 40)
        ref, tol = TB.ref_and_bound(case.q, case.k, case.v, case.fwd_map, case.mask, case.chunks, case.heads,
                                    case.scale, "rows", gathered=True)
        r = TB.ratio(emulate(case, "rows"), ref, tol).max().item()
        assert 0.05 < r <= 1, (fam, r)
        assert math.isfinite(r)
