"""warp_tensor's frame-chain kernels (W1, hbm_kernels.cu), restated in torch fp32 on the CPU.

``emulate`` runs the arithmetic every chain kernel shares, in their order of work: make_taps in fp32
(``oracle.warp_loss_bound.taps32``); ``sample_taps`` as four products summed left to right, either rounded one by one or
contracted into an fmul and three fmas; ``chain_blend`` z (1 - m) + warped m rounded term by term or contracted either
way (fma(z, 1 - m, warped m) or fma(warped, m, z (1 - m))); the chain carried in fp32 between frames; the closing blend
of the chained frame N - 1 with frame 0 warped through ``fwd_flow_last``; one rounding to the output type per stored
element.  The group and quad kernels do exactly this per element (float and float4 paths of the same helpers), so the
contraction modes are the freedom nvcc has between them.

It checks the error model of ``oracle.warp_chain_bound`` without a GPU: every contraction mode stays inside the bound
on every family, at fp32 and fp16, and matches the exact families bit for bit; each of ``MUTANTS`` -- a one-line mistake
a change to the kernels could make -- leaves the bound or the exact answer on the family named with it.
"""
import pytest
import torch

from oracle import warp_chain_bound as CB
from oracle import warp_loss_bound as WB

MUTANTS = {
    # name: (what it does, the family that must catch it)
    "mask-off-by-one": ("step i blends with the weights of frame i + 1", "identity"),
    "closing-bwd": ("the closing blend warps frame 0 through bwd_flow[N-1] instead of fwd_flow_last", "realistic"),
    "closing-unchained": ("the closing blend starts from sample frame N-1 instead of its chained value", "identity"),
    "xy-swap": ("the x and y components of the flow swapped", "realistic"),
    "clamp": ("clamp padding: taps past the border read the edge pixel with their weight", "edges"),
    "trunc": ("truncation instead of floor for the cell corner", "edges"),
    "fp16-chain": ("the chain carried in fp16 between frames", "realistic"),
}
MODES = ("none", "fma-z", "fma-w")
# (chunks, frames, C, h, w)
CASES = [(2, 3, 3, 12, 16), (1, 8, 2, 9, 7), (1, 16, 2, 6, 5), (2, 2, 2, 1, 13), (1, 3, 2, 11, 1)]


def _fma(a, b, c):
    """fp32 fma: the product of two fp32 values is exact in fp64, one rounding to fp32 after the add."""
    return (a.double() * b.double() + c.double()).float()


def _taps(flow, mutant):
    if mutant == "xy-swap":
        flow = flow.flip(0)
    _, h, w = flow.shape
    if mutant not in ("clamp", "trunc"):
        return WB.taps32(flow)
    xs, ys = WB._grid(h, w, flow.device, torch.float32)
    X, Y = xs + flow[0].reshape(-1), ys + flow[1].reshape(-1)
    fl = torch.trunc if mutant == "trunc" else torch.floor
    xf, yf = fl(X), fl(Y)
    ax, ay = X - xf, Y - yf
    x0, y0 = xf.long(), yf.long()
    x1, y1 = x0 + 1, y0 + 1
    cx0, cx1, cy0, cy1 = x0.clamp(0, w - 1), x1.clamp(0, w - 1), y0.clamp(0, h - 1), y1.clamp(0, h - 1)
    idx = torch.stack([cy0 * w + cx0, cy0 * w + cx1, cy1 * w + cx0, cy1 * w + cx1], -1)
    wt = torch.stack([(1 - ax) * (1 - ay), ax * (1 - ay), (1 - ax) * ay, ax * ay], -1)
    if mutant == "trunc":
        valid = torch.stack([(x0 >= 0) & (x0 < w) & (y0 >= 0) & (y0 < h), (x1 >= 0) & (x1 < w) & (y0 >= 0) & (y0 < h),
                             (x0 >= 0) & (x0 < w) & (y1 >= 0) & (y1 < h), (x1 >= 0) & (x1 < w) & (y1 >= 0) & (y1 < h)], -1)
        wt = torch.where(valid, wt, torch.zeros_like(wt))
    far = ~((X.abs() < 1e9) & (Y.abs() < 1e9))
    wt = torch.where(far[:, None], torch.zeros_like(wt), wt)
    return {"idx": idx, "w": wt}


def _sample(plane, T, mode):
    acc = T["w"][:, 0] * plane[:, T["idx"][:, 0]]
    for t in range(1, 4):
        wv, v = T["w"][:, t].expand_as(acc), plane[:, T["idx"][:, t]]
        acc = acc + wv * v if mode == "none" else _fma(wv, v, acc)
    return acc


def _blend(z, warped, m, mode):
    om = 1 - m
    if mode == "none":
        return z * om + warped * m
    if mode == "fma-z":
        return _fma(z, om.expand_as(z), warped * m)
    return _fma(warped, m.expand_as(z), z * om)


def emulate(d, chunks, mode="none", mutant=None):
    sample, bwd, fwd_last, blend = d["sample"], d["bwd"], d["fwd_last"], d["blend"]
    B, C, h, w = sample.shape
    N, hw = B // chunks, h * w
    x = sample.float().reshape(chunks, N, C, hw).permute(1, 0, 2, 3).reshape(N, chunks * C, hw)
    m = blend.reshape(N, 1, hw)
    carry = (lambda t: t.half().float()) if mutant == "fp16-chain" else (lambda t: t)
    z = [x[0]]
    for i in range(N - 1):
        mi = m[min(i + 1, N - 1)] if mutant == "mask-off-by-one" else m[i]
        z.append(carry(_blend(x[i + 1], _sample(z[-1], _taps(bwd[i], mutant), mode), mi, mode)))
    last_flow = bwd[N - 1] if mutant == "closing-bwd" else fwd_last
    own = x[N - 1] if mutant == "closing-unchained" else z[-1]
    z[-1] = _blend(own, _sample(x[0], _taps(last_flow, mutant), mode), m[N - 1], mode)
    out = torch.stack(z).reshape(N, chunks, C, h, w).transpose(0, 1).reshape(B, C, h, w)
    return out.to(sample.dtype)


def _case(fam, case, dtype, seed=0):
    chunks, N, C, h, w = case
    d = CB.family(fam, chunks, N, C, h, w, dtype=dtype, seed=seed)
    ref, tol = CB.chain_reference_and_bound(d["sample"], d["bwd"], d["fwd_last"], d["blend"], chunks)
    return d, ref, tol


def _fails(out, ref, tol, fam, dtype):
    if CB.ratio(out, ref, tol).max().item() > 1.0:
        return True
    return fam in CB.EXACT and not torch.equal(out, CB.exact_output(ref, dtype))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16], ids=["float", "half"])
@pytest.mark.parametrize("case", CASES, ids=lambda c: "c%dn%dC%d-%dx%d" % c)
@pytest.mark.parametrize("fam", CB.FAMILIES)
def test_emulation_within_bound(fam, case, dtype):
    if fam in ("near-integer", "realistic") and min(case[3], case[4]) == 1:
        # the floor needs cells to cross; the reference's flow_warp normalises by (w - 1) and is undefined there
        pytest.skip("one-pixel axis")
    d, ref, tol = _case(fam, case, dtype)
    for mode in MODES:
        out = emulate(d, case[0], mode)
        r = CB.ratio(out, ref, tol).max().item()
        assert r <= 1.0, f"{fam} {mode}: err/tol {r:.3g}"
        if fam in CB.EXACT:
            assert torch.equal(out, CB.exact_output(ref, dtype)), f"{fam} {mode}: not bit-exact"


def test_exact_families_are_exact_in_fp64():
    """The exact families' fp64 references are fp32 values, so 'bit-exact' is a statement about the kernel alone."""
    for fam in CB.EXACT:
        for case in CASES:
            _, ref, _ = _case(fam, case, torch.float32)
            CB.exact_output(ref, torch.float32)


@pytest.mark.parametrize("mutant", sorted(MUTANTS))
def test_mutant_caught(mutant):
    what, fam = MUTANTS[mutant]
    caught = []
    for dtype in (torch.float32, torch.float16):
        for case in CASES[:3]:
            d, ref, tol = _case(fam, case, dtype)
            out = emulate(d, case[0], "none", mutant)
            caught.append(_fails(out, ref, tol, fam, dtype))
    assert any(caught), f"{mutant} ({what}) passes the {fam} family"

