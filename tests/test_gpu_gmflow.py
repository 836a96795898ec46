"""GMFlow's kernels through the C ABI, at the feature grids FRESCO's frames give, against fp64 references.

FRESCO calls GMFlow at the frame resolution, so the 1/8-resolution token count L = (H/8)(W/8) is a multiple of 64 but
not always of 128 (576 x 576 -> 72 x 72, L = 5184 = 40.5 key tiles), and frames are often not square.

* ``gmflow_global_corr_softmax`` (to_token_major_f16_kernel twice, then tile_gemm_kernel<EPI_GMFLOW,0> once per
  direction) and ``gmflow_flow_attention`` (the same GEMM with V = a flow field): every output is prefilled with NaN,
  the launch count and name are asserted, and every element is checked against ``oracle.gmflow_bound`` (fp64 on the
  operands the kernel reads, elementwise bound derived from its arithmetic).  The input families of
  ``gmflow_bound.family``:
  - uniform: every score equal, p = 1, l and the coordinate sums are integers -- the flow is ((w-1)/2 - x, (h-1)/2 - y)
    up to the rounding of 1.f / l and of the multiply-subtract (fused or not; ``gmflow_bound.exact_out``): checked
    bit for bit;
  - translated: distinct sign patterns rolled by (3, -5); every other key >= 150 log2 units below the match, so every
    other p and every alpha flushes to 0, l = 1 and the flow is the shift (wrapped at the border): bit for bit, which
    pins orientation, sign and the [fwd(B), bwd(B)] order;
  - bimodal: every pattern twice, half a grid apart: the midpoint of two keys in different tiles (the ragged last one
    included), l = 2, bit for bit;
  - late / early: the only strong match in the last (ragged) tile -- everything before it rescaled to 0 -- or in the
    first, every later tile >= 100 nats lower;
  - negative-floor: every logit in about [-125, -100] nats, so a zero-filled column entering the max or the sums shows;
  - peaky1..3: LayerNorm-scale features at gains 1-3, logits of tens to about a hundred nats.
* The same kernel against the reference on the fp32 features (``oracle.fresco_oracle.global_correlation_softmax`` in
  fp64), with the operand-rounding term of ``gmflow_bound``: fp16 operands are adequate by a checked bound.
* ``single_head_split_window_attention`` with and without shift on non-square grids whose windows and shifted regions
  are not multiples of 128 tokens: every token against a dense fp64 reference with the reference's additive -100 mask,
  within attention_bound of its block plus the measured contribution of the masked keys (asserted < 2^-30 max|y|).
* Both against the reference's own outputs on a 24 x 40 grid (tests/golden/gmflow_rect*.npz).

``test_report_worst_ratios`` prints the largest err / tol per check, family and grid (-s to see it).
"""
import math

import numpy as np
import pytest
import torch

from oracle import attention_bound as AB
from oracle import fresco_oracle as O
from oracle import gmflow_bound as GB

pytestmark = pytest.mark.gpu

GEMM = "tile_gemm_kernel<EPI_GMFLOW,0>"
# 512^2, 512x640 both ways, 768^2 (config 5), 576^2 (ragged), 576x704 (ragged), 512x896
GRIDS = [(64, 64), (64, 80), (80, 64), (96, 96), (72, 72), (72, 88), (64, 112)]
RATIOS = {}     # (check, family, grid) -> worst err / tol


@pytest.fixture(scope="module")
def fb():
    if not torch.cuda.is_available():
        pytest.skip("GPU tests need a CUDA device")
    from fresco_b200 import _lib
    _lib.lib()      # fails loudly if the extension is missing
    torch.backends.cuda.matmul.allow_tf32 = False

    class NS:
        pass
    ns = NS()
    ns.lib, ns.c = _lib, _lib.lib()
    return ns


def _gid(g):
    return "%dx%d" % g


def _nan(shape):
    return torch.full(shape, float("nan"), dtype=torch.float32, device="cuda")


def corr(fb, f0, f1, bidir):
    """gmflow_global_corr_softmax on NaN-prefilled output; asserts the launches."""
    B, C, h, w = f0.shape
    out = _nan((B * (2 if bidir else 1), 2, h, w))
    nbytes = int(fb.c.fresco_gmflow_corr_workspace_bytes(B, C, h, w))
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    n0 = fb.lib.launch_count()
    fb.lib.check(fb.c.gmflow_global_corr_softmax(f0.data_ptr(), f1.data_ptr(), out.data_ptr(), B, C, h, w, int(bidir),
                                                 ws.data_ptr(), nbytes, fb.lib.stream()), "gmflow_global_corr_softmax")
    assert fb.lib.last_kernel() == GEMM, fb.lib.last_kernel()
    assert fb.lib.launch_count() - n0 == 3 + int(bidir), "two to_token_major_f16_kernel launches, one GEMM per direction"
    return out


def flow_attn(fb, q, k, vals, scale):
    B, L, C = q.shape
    out = _nan((B, 2, L))
    n0 = fb.lib.launch_count()
    fb.lib.check(fb.c.gmflow_flow_attention(q.data_ptr(), k.data_ptr(), vals.data_ptr(), out.data_ptr(), B, L, C, scale,
                                            fb.lib.stream()), "gmflow_flow_attention")
    assert fb.lib.last_kernel() == GEMM and fb.lib.launch_count() - n0 == 1
    return out


def _worst_tile(ratio):
    """Where err / tol is largest: flow index, channel and 128-query row tile (ratio [n, 2, L])."""
    n, _, L = ratio.shape
    r = torch.nn.functional.pad(ratio, (0, (-L) % 128)).view(n, 2, -1, 128).amax(-1)
    i, c, t = (int(x) for x in torch.unravel_index(r.argmax(), r.shape))
    return (f"worst at flow {i} channel {'xy'[c]} query tile [{t * 128}, {min(L, (t + 1) * 128)}): err/tol "
            f"{r[i, c, t].item():.3g}; {(r > 1).sum().item()} of {r.numel()} tiles fail")


def check(what, family, grid, out, ref, tol):
    """|out - ref| <= tol everywhere; NaN (never written) fails."""
    out, ref, tol = (t.reshape(t.shape[0], 2, -1) for t in (out, ref, tol))
    ratio = ((out.double() - ref).abs() / tol).nan_to_num(nan=float("inf"))
    worst = ratio.max().item()
    key = (what, family, grid)
    RATIOS[key] = max(RATIOS.get(key, 0.0), worst)
    assert worst <= 1.0, f"{what} {family} {grid}: " + _worst_tile(ratio)


def check_exact(what, family, out, want):
    """out bit-exact: either rounding of the last multiply-subtract (gmflow_bound.exact_out)."""
    out = out.reshape(want.shape[1:])
    bad = ~GB.matches_exact(out, want)
    if bad.any():
        i = tuple(bad.nonzero()[0].tolist())
        raise AssertionError(f"{what} {family}: {bad.sum().item()} of {bad.numel()} outputs not bit-exact; first at "
                             f"{list(i)}: {out[i].item()!r} want {want[0][i].item()!r} or {want[1][i].item()!r}")


def _corr_case(fb, name, B, C, grid, seed, bidir=True):
    h, w = grid
    fam = GB.family(name, B, C, h, w, seed=seed, device="cuda")
    GB.family_property(fam)
    out = corr(fb, fam.f0, fam.f1, bidir)
    ref, tol = GB.corr_ref_and_bound(fam.f0, fam.f1, bidir)
    check("corr", name, _gid(grid) + f" B{B} C{C}", out, ref, tol)
    if fam.exact:
        check_exact("corr", name, out, GB.corr_exact(fam.f0, fam.f1, bidir))
    return fam, out


# ================================================================================================ global correlation
@pytest.mark.parametrize("grid", GRIDS, ids=_gid)
def test_corr_families(fb, grid):
    """B = 8 pairs in both directions (16 flows) at C = 128, every family."""
    for i, name in enumerate(GB.FAMILIES):
        _corr_case(fb, name, 8, 128, grid, seed=11 * i + grid[0] + grid[1])
        torch.cuda.empty_cache()


@pytest.mark.parametrize("B", [3, 4])
@pytest.mark.parametrize("grid", [(72, 72), (72, 88)], ids=_gid)
def test_corr_pair_shares(fb, grid, B):
    """The pair shares of N = 7 frames over 2 GPUs (dist.frame_range), both directions and one: the one-direction call
    gives the forward half of the two-direction call bit for bit."""
    for name in ("translated", "peaky2", "late"):
        fam, both = _corr_case(fb, name, B, 128, grid, seed=B)
        one = corr(fb, fam.f0, fam.f1, False)
        assert torch.equal(one.view(torch.int32), both[:B].view(torch.int32)), name


def test_corr_small_channels(fb):
    """C = 24: the K tail of the 64-wide TMA atom, on the 24 x 40 grid (7.5 key tiles)."""
    for i, name in enumerate(GB.FAMILIES):
        _corr_case(fb, name, 2, 24, (24, 40), seed=i)


@pytest.mark.parametrize("grid", [(64, 64), (72, 88)], ids=_gid)
def test_corr_against_fp32_features(fb, grid):
    """Reference contract: on LayerNorm-scale fp32 features (not fp16-representable), the kernel is within its bound
    plus the operand-rounding term of the fp32-feature reference, oracle.global_correlation_softmax in fp64."""
    h, w = grid
    C, B = 128, 4
    for gain in (1.0, 2.0, 3.0):
        gen = torch.Generator(device="cuda").manual_seed(int(gain) + h)
        ln = lambda t: (t - t.mean(1, keepdim=True)) / t.std(1, keepdim=True, unbiased=False)
        f0 = ln(torch.randn(B, C, h, w, device="cuda", generator=gen))
        f1 = ln(torch.roll(f0, (2, -3), (2, 3)) + 0.5 * torch.randn(B, C, h, w, device="cuda", generator=gen))
        f0, f1 = (gain * f0).contiguous(), (gain * f1).contiguous()
        out = corr(fb, f0, f1, True)
        ref32, term = GB.operand_rounding_term(f0, f1, True)
        oracle64, _ = O.global_correlation_softmax(f0.double(), f1.double(), True)
        assert (oracle64 - ref32).abs().max().item() < 1e-9
        _, tol = GB.corr_ref_and_bound(f0, f1, True)
        check("corr-vs-fp32-features", f"gain{gain:g}", _gid(grid), out, ref32, tol + term)
        err = (out.double() - ref32).abs().max().item()
        print(f"\nfp32-feature reference {_gid(grid)} gain {gain:g}: max err {err:.3g} px, max tol "
              f"{(tol + term).max().item():.3g} px, worst err/tol {RATIOS[('corr-vs-fp32-features', f'gain{gain:g}', _gid(grid))]:.3g}")


# ================================================================================================ flow attention
def _flow_field(B, L, seed):
    """A smooth-ish flow field in quarter pixels, |v| <= 40: sums of any L of them are exact in fp32."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    v = torch.randn(B, L, 2, device="cuda", generator=g).cumsum(1) * 0.5
    v = v - v.mean(1, keepdim=True)
    return (v.clamp(-40, 40) * 4).round() / 4


def _flow_attn_case(fb, name, B, C, grid, seed):
    h, w = grid
    fam = GB.family(name, B, C, h, w, seed=seed, device="cuda")
    q = GB.to_tokens(fam.f0).half().contiguous()
    k = GB.to_tokens(fam.f1).half().contiguous()
    vals = _flow_field(B, h * w, seed).contiguous()
    scale = 1.0 / math.sqrt(C)
    out = flow_attn(fb, q, k, vals, scale)
    ref, tol = GB.flow_attn_ref_and_bound(q, k, vals, scale)
    check("flow-attn", name, _gid(grid) + f" B{B}", out, ref, tol)
    if fam.exact:
        check_exact("flow-attn", name, out, GB.flow_attn_exact(q, k, vals))


@pytest.mark.parametrize("grid", GRIDS, ids=_gid)
def test_flow_attention_families(fb, grid):
    for i, name in enumerate(GB.FAMILIES):
        _flow_attn_case(fb, name, 8, 128, grid, seed=7 * i + grid[1])
        torch.cuda.empty_cache()


@pytest.mark.parametrize("B", [3, 4])
def test_flow_attention_pair_shares(fb, B):
    for name in ("bimodal", "peaky3", "negative-floor"):
        _flow_attn_case(fb, name, B, 128, (72, 88), seed=B)


# ================================================================================================ window attention
def _nan_empty(monkeypatch):
    """torch.empty that fills floating-point tensors with NaN, so an output row nothing writes is caught."""
    real = torch.empty

    def empty(*a, **k):
        t = real(*a, **k)
        if t.is_floating_point():
            t.fill_(float("nan"))
        return t
    monkeypatch.setattr(torch, "empty", empty)


def _region_labels(h, w, wh, ww, sh, sw):
    """The labels generate_shift_window_attn_mask gives the ROLLED grid: three row bands x three column bands."""
    lab = torch.zeros(h, w, dtype=torch.long)
    cnt = 0
    for hs in (slice(0, -wh), slice(-wh, -sh), slice(-sh, None)):
        for ws in (slice(0, -ww), slice(-ww, -sw), slice(-sw, None)):
            lab[hs, ws] = cnt
            cnt += 1
    return lab


def window_ref_and_bound(q, k, v, h, w, with_shift, num_splits=2):
    """Dense fp64 reference of the reference's split-window attention (additive -100 between regions, on the rolled
    grid), and per token attention_bound of its block plus |dense - block-exact|.  All [b, L, c] in ORIGINAL token
    order; also returns the masked keys' contribution |dense - block-exact|."""
    b, L, c = q.shape
    wh, ww = h // num_splits, w // num_splits
    sh, sw = (wh // 2, ww // 2) if with_shift else (0, 0)
    roll = lambda t: torch.roll(t.view(b, h, w, -1), (-sh, -sw), (1, 2))
    qr, kr, vr = roll(q), roll(k), roll(v)
    lab = _region_labels(h, w, wh, ww, sh, sw).to(q.device) if with_shift else torch.zeros(h, w, dtype=torch.long,
                                                                                          device=q.device)
    dense = torch.empty(b, h, w, c, dtype=torch.float64, device=q.device)
    exact = torch.empty_like(dense)
    tol = torch.empty_like(dense)
    for i in range(num_splits):
        for j in range(num_splits):
            sl = (slice(None), slice(i * wh, (i + 1) * wh), slice(j * ww, (j + 1) * ww))
            qw, kw, vw = (t[sl].reshape(b, wh * ww, -1) for t in (qr, kr, vr))
            lw = lab[sl[1:]].reshape(-1)
            same = lw[:, None] == lw[None, :]
            # the scale rounded to fp32 as the C ABI passes it, as attention_bound does: the dense - block-exact
            # difference is then the masked keys' contribution alone
            s = (qw.double() @ kw.double().transpose(1, 2)) * AB._f32(1.0 / math.sqrt(c))
            dense[sl] = (torch.softmax(s + (~same) * -100.0, -1) @ vw.double()).view(b, wh, ww, c)
            ex = torch.empty(b, wh * ww, c, dtype=torch.float64, device=q.device)
            tw = torch.empty_like(ex)
            for r in lw.unique():
                idx = (lw == r).nonzero()[:, 0]
                rr, tt = AB.ref_and_bound(qw[:, idx], kw[:, idx], vw[:, idx], heads=1)
                ex[:, idx], tw[:, idx] = rr, tt
            exact[sl], tol[sl] = ex.view(b, wh, ww, c), tw.view(b, wh, ww, c)
    back = lambda t: torch.roll(t, (sh, sw), (1, 2)).reshape(b, L, c)
    dense, exact, tol = back(dense), back(exact), back(tol)
    masked = (dense - exact).abs()
    return dense, tol + masked, masked


WINDOW_GRIDS = [(64, 88), (72, 72), (80, 64), (64, 112)]


@pytest.mark.parametrize("with_shift", [False, True], ids=["plain", "shift"])
@pytest.mark.parametrize("grid", WINDOW_GRIDS, ids=_gid)
def test_split_window_attention_every_token(fb, monkeypatch, grid, with_shift):
    from fresco_b200 import gmflow_transformer as gt
    assert fb.c.fresco_attn_variant(128).decode() == "fresco_attn_kernel<128,keys128,wg2,poly0> (wgmma)"
    h, w = grid
    gen = torch.Generator(device="cuda").manual_seed(h * w + with_shift)
    q = (1.5 * torch.randn(2, h * w, 128, device="cuda", generator=gen)).half()
    k, v = (torch.randn(2, h * w, 128, device="cuda", generator=gen).half() for _ in range(2))
    _nan_empty(monkeypatch)
    out = gt.single_head_split_window_attention(q.float(), k.float(), v.float(), num_splits=2, with_shift=with_shift,
                                                h=h, w=w)
    monkeypatch.undo()
    assert fb.lib.last_kernel() == "rows_scatter_kernel"
    ref, tol, masked = window_ref_and_bound(q, k, v, h, w, with_shift)
    ymax = ref.abs().max().item()
    assert masked.max().item() < 2.0 ** -30 * ymax, f"masked keys contribute {masked.max().item():.3g}"
    ratio = ((out.double() - ref).abs() / tol).nan_to_num(nan=float("inf"))
    worst = ratio.max().item()
    key = ("window", "shift" if with_shift else "plain", _gid(grid))
    RATIOS[key] = worst
    if worst > 1:
        bb, tok = (int(x) for x in (ratio.amax(-1) > 1).nonzero()[0])
        raise AssertionError(f"window {key}: {(ratio.amax(-1) > 1).sum().item()} tokens over the bound, worst "
                             f"{worst:.3g}; first batch {bb} token {tok} (y {tok // w}, x {tok % w})")


# ================================================================================================ reference fixture
def test_rect_golden_through_the_kernels(fb, golden):
    """The reference's own outputs on a 24 x 40 grid: the kernel within its bound plus the fixture's measured fp32
    error (|fixture - fp64 oracle|), and the window decomposition within attention_bound plus the same."""
    from fresco_b200 import gmflow_transformer as gt
    g = golden("gmflow_rect")
    f0, f1 = (torch.from_numpy(np.asarray(g[n])).float().cuda().contiguous() for n in ("f0", "f1"))
    for bidir, key in ((True, "flow_bidir"), (False, "flow_uni")):
        fix = torch.from_numpy(g[key]).double().cuda()
        out = corr(fb, f0, f1, bidir)
        ref, tol = GB.corr_ref_and_bound(f0, f1, bidir)
        own = (fix - ref).abs()
        assert own.max().item() < 1e-4
        check("golden-corr", key, "24x40", out, fix, tol + own)
    q, k, v = (torch.from_numpy(np.asarray(g[n])).cuda() for n in "qkv")
    h, w = int(g["h"]), int(g["w"])
    for with_shift, key in ((False, "out_split"), (True, "out_shift")):
        fix = torch.from_numpy(g[key]).double().cuda()
        ref, tol, masked = window_ref_and_bound(q, k, v, h, w, with_shift)
        own = (fix - ref).abs()
        assert own.max().item() < 1e-5 * ref.abs().max().item()
        out = gt.single_head_split_window_attention(q.float(), k.float(), v.float(), num_splits=2,
                                                    with_shift=with_shift, h=h, w=w)
        ratio = ((out.double() - fix).abs() / (tol + own)).nan_to_num(nan=float("inf"))
        RATIOS[("golden-window", key, "24x40")] = ratio.max().item()
        assert ratio.max().item() <= 1.0, (key, ratio.max().item())


def test_report_worst_ratios():
    """Prints the largest err / tol seen per check, family and grid (-s to see it)."""
    if not RATIOS:
        pytest.skip("no GMFlow case ran")
    print("\nworst err/tol per check, family and grid")
    for (what, fam, grid), r in sorted(RATIOS.items()):
        print(f"  {what:22s} {fam:15s} {grid:16s} {r:.3g}")
    for what in sorted({k[0] for k in RATIOS}):
        for fam in sorted({k[1] for k in RATIOS if k[0] == what}):
            print(f"  max {what:18s} {fam:15s} {max(r for k, r in RATIOS.items() if k[:2] == (what, fam)):.3g}")
