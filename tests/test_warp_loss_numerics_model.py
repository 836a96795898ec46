"""The temporal-consistency loss kernels (O2, hbm_kernels.cu), restated in torch fp32 on the CPU.

``emulate`` runs the arithmetic of warp_loss_quad_kernel and warp_loss_group_kernel as they schedule it: make_taps in
fp32 (``oracle.warp_loss_bound.taps32``, the same function warp_taps_kernel evaluates); the residuals as four rounded
products summed left to right; the signs sgn(r) m in fp16 (exact); the adjoint ELL packed by ``ops._pack_adjoint`` and
walked slot by slot -- the group kernel skips a slot whose weight field is 0, the quad kernel stops a 32-lane warp at the
first slot that is 0 in all of its live lanes; the overflow runs summed in list order and added to ga before the ELL
slots (bwd) or to the carry after them (fwd); fl(fl(ga k) + fl(carry k)); the wrap-around add to frame 0, or the halo
plane of the open chain.  It checks the error model of ``oracle.warp_loss_bound`` without a GPU: the emulator stays
inside the bound on every input family, matches the integer family bit for bit, and each of ``MUTANTS`` -- a one-line
mistake a change to the kernels or the packing could make -- leaves the bound or the exact answer on at least one
family.  The packing's invariant (used slots first, a 0 weight field ends the row) is checked on every family.
"""
import pytest
import torch

from fresco_b200 import ops
from oracle import warp_loss_bound as WB

MUTANTS = {
    "early-exit": "the quad kernel's early exit over a packing that keeps taps whose weight field rounds to 0",
    "truncate": "floor instead of round when the packing quantises a weight",
    "no-overflow": "the overflow lists are never read",
    "sign0": "sgn(0) = +1",
    "mask-swap": "keep_f and keep_b swapped",
    "no-wrap": "the carry of the last pair never reaches frame 0 of the ring",
    "halo-mean": "the open chain takes k from its local frame count instead of the ring's",
}

CHUNKS, C = 2, 4
SHAPES = [(16, 16), (12, 20)]
# (frames, open chain, total frames, accumulate)
CONFIGS = [(3, False, 3, False), (2, True, 5, True)]
INV = torch.tensor(WB.INV65535, dtype=torch.float32)


def _fma(a, b, c):
    """fp32 fma: the product of two fp32 values is exact in fp64, one rounding to fp32 after the add."""
    return (a.double() * b.double() + c.double()).float()


def _pack(T, h, w, mutant):
    dest = torch.where(T["w"] != 0, T["idx"], torch.full_like(T["idx"], -1))[None]
    wgt = T["w"][None]
    if mutant == "early-exit":
        return ops._pack_ell(dest.reshape(1, -1), wgt.reshape(1, -1), h, w)
    if mutant == "truncate":
        wgt = (wgt * 65535.0).floor() * INV
    return ops._pack_adjoint(dest, wgt, h, w)


def _decode(packed):
    e = packed[0].long() & 0xffffffff                                        # [hw, 8] uint32
    return (e >> 16).float() * INV, e & 0xffff, (e >> 16) != 0


def _runs(adj, s, hw):
    """Overflow runs, each summed in list order from 0: -> [P, hw] fp32 (0 where no run ends)."""
    out = torch.zeros(s.shape[0], hw)
    o = adj["ovf"][0]
    for e in range(adj["n_ovf"]):
        d, src, wb = int(o[e, 0]), int(o[e, 1]), o[e, 2:3].view(torch.float32)
        out[:, d] = _fma(-wb, s[:, src], out[:, d])
    return out


def _gather(acc, adj, s, hw, quad, mutant):
    """acc -= sum over the ELL slots of w s[src], slot by slot (quad: a warp of 32 destinations stops together)."""
    wq, src, used = _decode(adj["ell_packed"])
    if quad:
        lanes = torch.arange(hw)
        live = torch.zeros((hw + 31) // 32 * 32, 8, dtype=torch.bool)
        live[:hw] = used
        alive = live.view(-1, 32, 8).any(1)                                    # [warps, 8]
        stop = torch.where(~alive, torch.arange(8), torch.full_like(alive, 8, dtype=torch.long)).amin(1)
        run = torch.arange(8)[None] < stop[lanes // 32][:, None]
    else:
        run = used
    for j in range(8):
        upd = _fma(-wq[:, j], s[:, src[:, j]], acc)
        acc = torch.where(run[:, j][None], upd, acc)
    return acc


def emulate(d, quad=True, mutant=None, total_frames=None, accumulate=False, prefill=None):
    cs, ff, bf, kf, kb, halo_cs = d["cs"], d["ff"], d["bf"], d["kf"], d["kb"], d["halo_cs"]
    chunks, N, Cc, h, w = cs.shape
    hw, Pl = h * w, chunks * Cc
    total = N if (total_frames is None or mutant == "halo-mean") else total_frames
    k = torch.tensor(WB.loss_scale(chunks, total, Cc, h, w), dtype=torch.float32)
    planes = cs.permute(1, 0, 2, 3, 4).reshape(N, Pl, hw)
    grad = (torch.zeros(N, Pl, hw) if prefill is None else prefill.permute(1, 0, 2, 3, 4).reshape(N, Pl, hw).clone())
    carry = torch.zeros(Pl, hw)
    loss = torch.zeros((), dtype=torch.float32)
    halo = None
    for f in range(N):
        c1 = planes[f]
        c2 = halo_cs.reshape(Pl, hw) if (f + 1 == N and halo_cs is not None) else planes[(f + 1) % N]
        mb, mf = kb[f].reshape(1, hw), kf[f].reshape(1, hw)
        if mutant == "mask-swap":
            mb, mf = mf, mb
        res = []
        for flow, own, src, m in ((bf[f], c2, c1, mb), (ff[f], c1, c2, mf)):
            T = WB.taps32(flow)
            smp = T["w"][:, 0] * src[:, T["idx"][:, 0]]
            for t in range(1, 4):
                smp = smp + T["w"][:, t] * src[:, T["idx"][:, t]]
            r = own - smp
            sg = torch.sign(r)
            if mutant == "sign0":
                sg = torch.where(r == 0, torch.ones_like(sg), sg)
            loss = loss + (r.abs() * m).sum()
            res.append((sg * m, _pack(T, h, w, mutant)))
        (s1, adj_b), (s2, adj_f) = res
        ga = s2.clone()
        if adj_b["n_ovf"] > 0 and mutant != "no-overflow":
            ga = ga + _runs(adj_b, s1, hw)
        ga = _gather(ga, adj_b, s1, hw, quad, mutant)
        gb = _gather(s1.clone(), adj_f, s2, hw, quad, mutant)
        if adj_f["n_ovf"] > 0 and mutant != "no-overflow":
            gb = gb + _runs(adj_f, s2, hw)
        v = ga * k + carry * k
        grad[f] = grad[f] + v if accumulate else v
        carry = gb
    if halo_cs is not None:
        halo = (carry * k).reshape(chunks, Cc, h, w)
    elif mutant != "no-wrap":
        grad[0] = grad[0] + carry * k
    return {"loss": (loss * k).item(), "grad": grad.reshape(N, chunks, Cc, h, w).permute(1, 0, 2, 3, 4), "halo": halo}


def _case(fam, shape, cfg, seed=0):
    N, open_, total, acc = cfg
    h, w = shape
    d = WB.family(fam, CHUNKS, N, C, h, w, seed=seed, halo=open_)
    prefill = torch.randn(d["cs"].shape, generator=torch.Generator().manual_seed(seed + 1)) if acc else None
    ref = WB.reference_and_bound(d["cs"], d["ff"], d["bf"], d["kf"], d["kb"], halo_cs=d["halo_cs"],
                                 total_frames=total if open_ else None, prefill=prefill)
    return d, ref, dict(total_frames=total if open_ else None, accumulate=acc, prefill=prefill)


def _violations(out, ref):
    """Worst err / tol over gradient, halo plane and loss (> 1: outside the bound)."""
    worst = WB.ratio(out["grad"], ref["grad"], ref["grad_tol"]).max().item()
    if ref["halo"] is not None:
        worst = max(worst, WB.ratio(out["halo"], ref["halo"], ref["halo_tol"]).max().item())
    return max(worst, abs(out["loss"] - ref["loss"]) / ref["loss_tol"])


def _exact_mismatch(out, ref, kw, open_):
    want, halo = WB.exact_grad(ref, accumulate=kw["accumulate"], prefill=kw["prefill"], ring=not open_)
    bad = not torch.equal(out["grad"], want)
    return bad or (halo is not None and not torch.equal(out["halo"], halo))


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "%dx%d" % s)
@pytest.mark.parametrize("cfg", CONFIGS, ids=["ring3", "open2of5-acc"])
@pytest.mark.parametrize("fam", WB.FAMILIES)
def test_emulation_within_bound(fam, cfg, shape):
    d, ref, kw = _case(fam, shape, cfg)
    if fam not in ("near-tie", "integer"):
        # (near-tie is built to sit in the band; the integer family's exact zeros are in it by construction)
        assert ref["in_band"] < 0.01, f"{fam}: {ref['in_band']:.3f} of the residuals inside their band"
    for quad in (True, False):
        out = emulate(d, quad=quad, **kw)
        r = _violations(out, ref)
        assert r <= 1.0, f"{fam} quad={quad}: err/tol {r:.3g}"
        if fam == "integer":
            assert not _exact_mismatch(out, ref, kw, cfg[1]), f"integer family not bit-exact (quad={quad})"


def _caught(mutant, fam):
    for shape in SHAPES:
        for cfg in CONFIGS:
            d, ref, kw = _case(fam, shape, cfg)
            out = emulate(d, quad=True, mutant=mutant, **kw)
            if _violations(out, ref) > 1.0:
                return True
            if fam == "integer" and _exact_mismatch(out, ref, kw, cfg[1]):
                return True
    return False


@pytest.mark.parametrize("mutant", sorted(MUTANTS))
def test_mutant_caught(mutant):
    fams = ["subthreshold"] if mutant == "early-exit" else WB.FAMILIES
    assert any(_caught(mutant, fam) for fam in fams), f"{mutant} ({MUTANTS[mutant]}) passes every family"


@pytest.mark.parametrize("fam", WB.FAMILIES)
def test_packing_invariant(fam):
    """Every tap with a nonzero weight field is packed exactly once (ELL or overflow), a row's used slots come first,
    and a slot whose weight field is 0 ends the row -- what the quad kernel's early exit relies on."""
    h, w = SHAPES[0]
    d = WB.family(fam, CHUNKS, 3, C, h, w, seed=0)
    for flow in list(d["bf"]) + list(d["ff"]):
        T = WB.taps32(flow)
        adj = _pack(T, h, w, None)
        _, src, used = _decode(adj["ell_packed"])
        after_empty = (~used).int().cummax(1).values.bool() & used
        assert not after_empty.any(), f"{fam}: {int(after_empty.any(1).sum())} rows hold a used slot after a 0 field"
        keep = (T["w"] * 65535.0).round() > 0
        want = torch.zeros(h * w, dtype=torch.long).index_add_(0, T["idx"][keep], torch.ones(int(keep.sum()), dtype=torch.long))
        got = used.sum(1)
        o = adj["ovf"][0][: adj["n_ovf"]]
        if adj["n_ovf"] > 0:
            got = got.index_add(0, o[:, 0].long(), torch.ones(adj["n_ovf"], dtype=torch.long))
        assert torch.equal(got, want), f"{fam}: taps lost or duplicated by the packing"


def test_bound_not_vacuous():
    """On the smooth family, dropping any single tap of weight >= 2^-12 from the adjoint leaves the bound."""
    h, w = SHAPES[0]
    d, ref, kw = _case("smooth", (h, w), CONFIGS[0])
    out = emulate(d, quad=True, **kw)
    err = (out["grad"].double() - ref["grad"]).abs()
    k = ref["k"]
    checked = 0
    for f in range(d["cs"].shape[1]):
        # taps of pair f's bwd warp carry s1 (mask kb[f]) into frame f's gradient
        T = WB.taps64(d["bf"][f])
        c1 = d["cs"][:, f].reshape(CHUNKS * C, -1).double()
        c2 = d["cs"][:, (f + 1) % d["cs"].shape[1]].reshape(CHUNKS * C, -1).double()
        s1 = torch.sign(c2 - WB._warp(c1, T)) * d["kb"][f].reshape(1, -1).double()
        e = err[:, f].reshape(CHUNKS * C, -1)
        tol = ref["grad_tol"][:, f].reshape(CHUNKS * C, -1)
        big = T["w"] >= 2.0 ** -12                                             # [hw, 4]
        p, t = torch.nonzero(big, as_tuple=True)
        q = T["idx"][p, t]
        shift = k * T["w"][p, t][None] * s1[:, p].abs()                        # what dropping the tap moves
        live = s1[:, p] != 0
        assert ((shift - e[:, q] > tol[:, q]) | ~live).all(), "a dropped tap stays inside the bound"
        checked += int(live.sum())
    assert checked > 1000, checked
