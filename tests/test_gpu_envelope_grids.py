"""The pieces of the keyframe path that already accept the web UI's frame sizes below 512 (256..448 at 1:1, 4:3,
3:4, 16:9 and 9:16; see tests/test_gpu_gram_ragged.py), checked at those sizes' grids:

* get_flow_and_interframe_paras with a stand-in flow model: masks and trajectories bit-exact against the CPU oracle,
* the cross-frame K/V selection bit-exact,
* GMFlow's split-window attention against a dense fp64 reference within oracle/attention_bound.py, at the 1/8 feature
  grids 40x56, 40x72, 48x88 and 56x96,
* temporal-guided attention within oracle/temporal_bound.py at the trajectory lengths (s/8)(l/8) and (s/16)(l/16).
"""
import math

import numpy as np
import pytest
import torch

from oracle import attention_bound as AB
from oracle import fresco_oracle as O
from oracle import temporal_bound as TB

pytestmark = pytest.mark.gpu


def resize_dims(h, w, resolution):
    """(H, W) of src/utils.py resize_image: the short side scaled to ``resolution``, both sides rounded to 64."""
    k = float(resolution) / min(h, w)
    return int(np.round(h * k / 64.0)) * 64, int(np.round(w * k / 64.0)) * 64


ASPECTS = [(512, 512), (480, 640), (640, 480), (1080, 1920), (1920, 1080)]
ENVELOPE = sorted({resize_dims(h, w, s) for s in range(256, 512, 64) for h, w in ASPECTS})


def _gid(hw):
    return "%dx%d" % hw


@pytest.fixture(scope="module")
def fb():
    if not torch.cuda.is_available():
        pytest.skip("GPU tests need a CUDA device")
    from fresco_b200 import _lib, diffusion_hacked, flow_utils, ops
    _lib.lib()      # fails loudly if the extension is missing
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False

    class NS:
        pass
    ns = NS()
    ns.lib, ns.c, ns.ops, ns.dh, ns.fu = _lib, _lib.lib(), ops, diffusion_hacked, flow_utils
    return ns


@pytest.mark.parametrize("hw", ENVELOPE, ids=_gid)
def test_flow_and_interframe_paras(fb, hw):
    """Per-batch preparation (src/diffusion_hacked.py:905-957) with a stand-in flow model that returns smooth flows:
    occlusions, the K/V masks at 3 scales and the trajectories at 2 scales equal the oracle's on the same flows."""
    H, W = hw
    N = 3
    flows, _ = O.synth_flows(N, H, W, seed=H + W, mag=10.0)

    class StubFlow(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.p = torch.nn.Parameter(torch.zeros(1))

        def forward(self, a, b, **kw):
            return {"flow_preds": [torch.cat([flows[0], flows[1]]).to(a.device)]}

    g = torch.Generator().manual_seed(H * W)
    imgs = [(torch.rand(H, W, 3, generator=g) * 255).to(torch.uint8).numpy() for _ in range(N)]
    fl, oc, masks, paras = fb.dh.get_flow_and_interframe_paras(StubFlow().cuda(), imgs)
    images = torch.stack([torch.from_numpy(im).permute(2, 0, 1).float() for im in imgs])
    resh = list(range(1, N)) + [0]
    fo, bo = O.forward_backward_consistency_check(flows[0], flows[1])
    bo = torch.clamp(bo + ((images[resh] - O.flow_warp(images, flows[1])).abs().mean(1) > 255 * 0.25).float(), 0, 1)
    assert (oc[1].cpu() != bo).float().mean().item() < 2e-3
    ref_masks = O.cross_frame_masks(oc[1].cpu())
    assert [tuple(m.shape) for m in masks] == [(N, (H // s) * (W // s)) for s in (8, 16, 32)]
    assert all(torch.equal(a.cpu(), b) for a, b in zip(masks, ref_masks))
    for i, s in enumerate((8.0, 16.0)):
        fm, bm, im = O.mapping_ind(fl[1].cpu(), oc[1].cpu(), images / 127.5 - 1.0, s)
        assert torch.equal(paras["fwd_mappings"][i].cpu(), fm), s
        assert torch.equal(paras["bwd_mappings"][i].cpu(), bm), s
        assert torch.equal(paras["interattn_masks"][i].cpu(), im), s


@pytest.mark.parametrize("hw", ENVELOPE, ids=_gid)
def test_kv_selection(fb, hw):
    """Cross-frame K/V of the two FRESCO decoder levels (1/8 and 1/16 of the frame) bit-exact against the oracle's
    ``key[:, attn_mask]``."""
    H, W = hw
    N, chunks, C = 4, 2, 320
    flows, occs = O.synth_flows(N, H, W, seed=H * 3 + W, mag=12.0)
    masks = O.cross_frame_masks(occs[1])
    for s, m in zip((8, 16), masks[:2]):
        L = (H // s) * (W // s)
        g = torch.Generator(device="cuda").manual_seed(L)
        k = torch.randn(chunks * N, L, C, device="cuda", generator=g).half()
        v = torch.randn(chunks * N, L, C, device="cuda", generator=g).half()
        ctrl = fb.dh.AttentionControl()
        ctrl.enable_cfattn([mm.cuda() for mm in masks])
        idx = ctrl.kv_indices(L)
        ks, vs = fb.ops.kv_compact(k, v, idx, chunks)
        ref_idx = O.kv_select_indices(m).cuda()
        assert torch.equal(idx.long(), ref_idx)
        assert torch.equal(ks, k.view(chunks, N * L, C)[:, ref_idx])
        assert torch.equal(vs, v.view(chunks, N * L, C)[:, ref_idx])


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
    """Dense fp64 reference of the reference's split-window attention (additive -100 between the regions of the
    rolled grid) and, per token, attention_bound of its region plus the masked keys' contribution."""
    b, L, c = q.shape
    wh, ww = h // num_splits, w // num_splits
    sh, sw = (wh // 2, ww // 2) if with_shift else (0, 0)
    roll = lambda t: torch.roll(t.view(b, h, w, -1), (-sh, -sw), (1, 2))
    qr, kr, vr = roll(q), roll(k), roll(v)
    lab = (_region_labels(h, w, wh, ww, sh, sw) if with_shift else torch.zeros(h, w, dtype=torch.long)).to(q.device)
    dense = torch.empty(b, h, w, c, dtype=torch.float64, device=q.device)
    exact, tol = torch.empty_like(dense), torch.empty_like(dense)
    for i in range(num_splits):
        for j in range(num_splits):
            sl = (slice(None), slice(i * wh, (i + 1) * wh), slice(j * ww, (j + 1) * ww))
            qw, kw, vw = (t[sl].reshape(b, wh * ww, -1) for t in (qr, kr, vr))
            lw = lab[sl[1:]].reshape(-1)
            same = lw[:, None] == lw[None, :]
            s = (qw.double() @ kw.double().transpose(1, 2)) * AB._f32(1.0 / math.sqrt(c))
            dense[sl] = (torch.softmax(s + (~same) * -100.0, -1) @ vw.double()).view(b, wh, ww, c)
            ex = torch.empty(b, wh * ww, c, dtype=torch.float64, device=q.device)
            tw = torch.empty_like(ex)
            for r in lw.unique():
                idx = (lw == r).nonzero()[:, 0]
                ex[:, idx], tw[:, idx] = AB.ref_and_bound(qw[:, idx], kw[:, idx], vw[:, idx], heads=1)
            exact[sl], tol[sl] = ex.view(b, wh, ww, c), tw.view(b, wh, ww, c)
    back = lambda t: torch.roll(t, (sh, sw), (1, 2)).reshape(b, L, c)
    dense, exact, tol = back(dense), back(exact), back(tol)
    masked = (dense - exact).abs()
    return dense, tol + masked


@pytest.mark.parametrize("with_shift", [False, True], ids=["plain", "shift"])
@pytest.mark.parametrize("grid", [(40, 56), (40, 72), (48, 88), (56, 96)], ids=_gid)
def test_split_window_attention(fb, monkeypatch, grid, with_shift):
    """GMFlow's split-window self-attention (2 x 2 windows, with and without the shift) at the 1/8 feature grids of
    the envelope: every token within the bound of the dense reference; outputs prefilled with NaN."""
    from fresco_b200 import gmflow_transformer as gt
    h, w = grid
    gen = torch.Generator(device="cuda").manual_seed(h * w + with_shift)
    q = (1.5 * torch.randn(2, h * w, 128, device="cuda", generator=gen)).half()
    k, v = (torch.randn(2, h * w, 128, device="cuda", generator=gen).half() for _ in range(2))
    real = torch.empty

    def empty(*a, **kw):
        t = real(*a, **kw)
        if t.is_floating_point():
            t.fill_(float("nan"))
        return t
    monkeypatch.setattr(torch, "empty", empty)
    out = gt.single_head_split_window_attention(q.float(), k.float(), v.float(), num_splits=2, with_shift=with_shift,
                                                h=h, w=w)
    monkeypatch.undo()
    ref, tol = window_ref_and_bound(q, k, v, h, w, with_shift)
    ratio = ((out.double() - ref).abs() / tol).nan_to_num(nan=float("inf"))
    assert ratio.max().item() <= 1, f"{(ratio.amax(-1) > 1).sum().item()} tokens over the bound, worst {ratio.max():.3g}"


TRAJ = sorted({(H // s) * (W // s) for H, W in ENVELOPE for s in (8, 16)})


@pytest.mark.parametrize("L", TRAJ)
def test_temporal_attention_trajectory_lengths(fb, L):
    """Temporal-guided attention at every trajectory length of the envelope (8 frames, 8 heads, d = 40 and 80, the
    decoder levels' head dims), on the reference-structured family and the huge family, within the bound."""
    for d, fam in ((40, "reference"), (80, "reference"), (40, "huge")):
        case = TB.make_case(fam, 8, L, 8, d, 2, seed=L + d)
        case = case._replace(q=case.q.cuda(), k=case.k.cuda(), v=case.v.cuda(), fwd_map=case.fwd_map.cuda(),
                             mask=case.mask.cuda())
        out = fb.ops.temporal_attn_fwd(case.q, case.k, case.v, case.fwd_map, case.mask.to(torch.uint8).contiguous(),
                                       case.chunks, case.heads, case.scale)
        ref, tol = TB.ref_and_bound(case.q, case.k, case.v, case.fwd_map, case.mask, case.chunks, case.heads,
                                    case.scale, "rows")
        r = TB.ratio(out, ref, tol)
        assert r.max().item() <= 1, (fam, d, r.max().item(), (r > 1).sum().item())
