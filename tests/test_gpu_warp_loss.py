"""The temporal-consistency loss (O2) through the C ABI, at shapes that select every kernel, against fp64 references.

``fresco_warp_loss_fwd_bwd_halo`` runs one of three kernels, and the launch name is asserted for every case:

* warp_loss_quad_kernel<P,NQ> for (1,4), (2,2) and (4,1);
* warp_loss_group_kernel<P,KT> with G > 1 sub-groups (planes of fewer than 512 pixels), KT = 1, 2, 4 and P = 18;
* warp_loss_kernel, one CTA per plane, for plane sizes no group instantiation takes.

Every family of ``oracle.warp_loss_bound`` runs on every kernel: the closed ring at 2, 3 and 8 frames and the open
chain at 1 and 3 frames (halo_grad checked elementwise), with accumulate 0 and 1 (a random prefill for 1).  grad and
halo_grad are filled with NaN first (under accumulate=1 grad holds the prefill instead), so an element the kernel never
writes fails.  The loss and every gradient element must lie within the bound; the integer family must match the
exactly known gradient bit for bit on the quad and group kernels (the one-CTA kernel sums the k-scaled terms, whose
multiples of k round, so it is held to the bound there).  ``fresco_warp_taps`` is checked bit for bit against the fp32
restatement of make_taps the bound is built on.

``test_report_worst_ratios`` prints the largest err / tol per kernel and family (-s to see it).
"""
import pytest
import torch
import torch.nn.functional as F

from oracle import warp_loss_bound as WB

pytestmark = pytest.mark.gpu

# kernel -> (chunks, C, h, w) that select it on a 132-SM H100
SHAPES = {
    "warp_loss_quad_kernel<1,4>": (2, 1056, 32, 32),
    "warp_loss_quad_kernel<2,2>": (2, 536, 32, 32),
    "warp_loss_quad_kernel<4,1>": (2, 12, 64, 64),
    "warp_loss_group_kernel<1,1>": (2, 6, 16, 16),          # G = 2
    "warp_loss_group_kernel<1,4>": (2, 1190, 16, 16),       # G = 2
    "warp_loss_group_kernel<2,2>": (2, 450, 32, 32),
    "warp_loss_group_kernel<3,1>": (2, 6, 36, 36),
    "warp_loss_group_kernel<18,1>": (2, 6, 96, 96),
    "warp_loss_kernel": (2, 6, 56, 56),
}
# (id, frames, open chain, accumulate); every family runs one ring and one open-chain case per kernel, the frame count
# and accumulate rotating with the family
RING = [(2, False), (3, True), (8, False)]
OPEN = [(1, True), (3, False)]
RATIOS = {}     # (kernel, family, case) -> worst err / tol


@pytest.fixture(scope="module")
def fb():
    if not torch.cuda.is_available():
        pytest.skip("GPU tests need a CUDA device")
    from fresco_b200 import _lib, ops
    _lib.lib()      # fails loudly if the extension is missing

    class NS:
        pass
    ns = NS()
    ns.lib, ns.ops, ns.c = _lib, ops, _lib.lib()
    return ns


def P(t):
    return t.data_ptr() if t is not None else None


def _worst_tile(ratio, rows=128, cols=256):
    """Where err / tol is largest, by rows x cols tile of the [planes, pixels] matrix (NaN counts as infinitely wrong)."""
    ratio = torch.nan_to_num(ratio.double(), nan=float("inf"))
    R, C = ratio.shape
    t = F.pad(ratio, (0, (-C) % cols, 0, (-R) % rows)).view((R + rows - 1) // rows, rows, (C + cols - 1) // cols, cols)
    t = t.amax((1, 3))
    i, j = divmod(int(t.argmax().item()), t.shape[1])
    return (f"worst {rows}x{cols} tile planes [{i * rows}, {(i + 1) * rows}) pixels [{j * cols}, {(j + 1) * cols}): "
            f"max err/tol {t[i, j].item():.3g}; {(t > 1).sum().item()} of {t.numel()} tiles fail")


def _cases():
    out = []
    for kname in SHAPES:
        for i, fam in enumerate(WB.FAMILIES):
            N, acc = RING[i % 3]
            out.append(pytest.param(kname, fam, N, False, acc, id=f"{kname}-{fam}-ring{N}-acc{int(acc)}"))
            N, acc = OPEN[i % 2]
            out.append(pytest.param(kname, fam, N, True, acc, id=f"{kname}-{fam}-open{N}-acc{int(acc)}"))
    return out


@pytest.mark.parametrize("kname,fam,N,open_,acc", _cases())
def test_warp_loss_family(fb, kname, fam, N, open_, acc):
    chunks, C, h, w = SHAPES[kname]
    total = N + 2 if open_ else N
    seed = sum(map(ord, kname + fam)) + 10 * N + int(open_)
    d = WB.family(fam, chunks, N, C, h, w, seed=seed, halo=open_, device="cuda")
    adj = fb.ops.warp_adjoint_pair(d["bf"], d["ff"])
    g = torch.Generator(device="cuda").manual_seed(seed)
    prefill = torch.randn(d["cs"].shape, device="cuda", generator=g) if acc else None
    grad = prefill.clone() if acc else torch.full_like(d["cs"], float("nan"))
    halo_grad = torch.full_like(d["halo_cs"], float("nan")) if open_ else None
    loss = torch.zeros(1, device="cuda")
    rc = fb.c.fresco_warp_loss_fwd_bwd_halo(
        P(d["cs"]), P(d["ff"]), P(d["bf"]), P(d["kf"]), P(d["kb"]), P(adj.bwd["ell_packed"]), P(adj.fwd["ell_packed"]),
        P(adj.ovf), int(adj.n_ovf), P(grad), P(loss), int(acc), chunks, N, C, h, w, P(d["halo_cs"]), P(halo_grad), total,
        fb.lib.stream())
    fb.lib.check(rc, "fresco_warp_loss_fwd_bwd_halo")
    assert fb.lib.last_kernel() == kname, f"launched {fb.lib.last_kernel()}"
    ref = WB.reference_and_bound(d["cs"], d["ff"], d["bf"], d["kf"], d["kb"], halo_cs=d["halo_cs"],
                                 total_frames=total if open_ else None, prefill=prefill)
    if fam not in ("near-tie", "integer"):
        assert ref["in_band"] < 0.01, f"{fam}: {ref['in_band']:.3f} of the residuals inside their band"
    ratio = WB.ratio(grad, ref["grad"], ref["grad_tol"])
    worst = ratio.max().item()
    msg = "grad: " + _worst_tile(ratio.reshape(-1, h * w))
    if open_:
        hr = WB.ratio(halo_grad, ref["halo"], ref["halo_tol"])
        if hr.max().item() > worst:
            msg = "halo_grad: " + _worst_tile(hr.reshape(-1, h * w))
        worst = max(worst, hr.max().item())
    lr = abs(loss.item() - ref["loss"]) / ref["loss_tol"] if ref["loss_tol"] > 0 else float(loss.item() != 0)
    worst = max(worst, lr)
    RATIOS[(kname, fam, ("open%d" if open_ else "ring%d") % N + "-acc%d" % int(acc))] = worst
    assert lr <= 1.0, f"loss {loss.item()!r} vs {ref['loss']!r}: err/tol {lr:.3g}"
    assert worst <= 1.0, f"{kname} {fam}: {msg}"
    if fam == "integer" and kname != "warp_loss_kernel":
        want, halo_want = WB.exact_grad(ref, accumulate=acc, prefill=prefill, ring=not open_)
        assert torch.equal(grad, want), f"integer family: {(grad != want).sum().item()} elements not bit-exact"
        if open_:
            assert torch.equal(halo_grad, halo_want), "integer family: halo_grad not bit-exact"


@pytest.mark.parametrize("fam", WB.FAMILIES)
def test_warp_taps_bit_exact(fb, fam):
    """fresco_warp_taps (warp_taps_kernel) equals make_taps restated in torch fp32, the taps the bound is built on."""
    h, w = 36, 44
    d = WB.family(fam, 1, 3, 1, h, w, seed=5, device="cuda")
    for flow in (d["bf"], d["ff"]):
        dest = torch.full((3, h * w, 4), -7, dtype=torch.int32, device="cuda")
        wgt = torch.full((3, h * w, 4), float("nan"), device="cuda")
        fb.lib.check(fb.c.fresco_warp_taps(P(flow), P(dest), P(wgt), 3, h, w, fb.lib.stream()), "fresco_warp_taps")
        for f in range(3):
            T = WB.taps32(flow[f])
            assert torch.equal(wgt[f], T["w"]), f"{fam}: weights differ"
            want = torch.where(T["w"] != 0, T["idx"], torch.full_like(T["idx"], -1)).to(torch.int32)
            assert torch.equal(dest[f], want), f"{fam}: destinations differ"


def test_report_worst_ratios():
    """Prints the largest err / tol seen per kernel and family (-s to see it)."""
    if not RATIOS:
        pytest.skip("no temporal-loss case ran")
    print("\nworst err/tol per kernel, family and case")
    for (kn, fam, case), r in sorted(RATIOS.items()):
        print(f"  {kn:30s} {fam:13s} {case:12s} {r:.3g}")
    for fam in WB.FAMILIES:
        rs = [r for k, r in RATIOS.items() if k[1] == fam]
        if rs:
            print(f"  max {fam:13s} {max(rs):.3g}")
    for kn in SHAPES:
        rs = [r for k, r in RATIOS.items() if k[0] == kn]
        if rs:
            print(f"  max {kn:30s} {max(rs):.3g}")
