"""GPU parity tests added in round 2: the shapes the bench actually executes (VERDICT r1, "parity gaps").

* every attention variant (key-tile width, consumer warpgroups, FMA-pipe exponentials, tensor-core row sums) at every head_dim,
* golden set B (N = 3, 64 x 96 plane, head_dim 80 -- odd frame count, non-square) through the kernels,
* temporal-guided attention at the bench shapes (N = 8, 8 heads, d = 40, L = 4096 and d = 80, L = 1024),
* teacher-forced single-iteration optimize_feature pieces at [16,1280,32,32] and [16,640,64,64], and the
  overflow path of the warp adjoint (destinations hit by more than 8 taps),
* the processor against the reference's outputs at the stated 2e-3 tolerance with fp32 Linear layers,
* per-batch caches across two keyframe batches, fp16 image-resolution warp_tensor.

Everything goes through the C ABI.  References are the CPU oracle, the golden vectors generated from the reference,
or -- at sizes the CPU oracle would take minutes for -- the oracle's own torch code evaluated in fp32 on the GPU
(same formulas, TF32 off)."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import attention_bound as AB  # noqa: E402  (checker only)
from oracle import fresco_oracle as O  # noqa: E402  (checker only)
from oracle import temporal_bound as TB  # noqa: E402  (checker only)
from oracle import warp_chain_bound as CB  # noqa: E402  (checker only)


def T(a, device="cuda"):
    return torch.from_numpy(np.asarray(a)).to(device)


def _warp_tensor_within_bound(fb, sample, flows, occs, sal, chunks):
    """warp_tensor, held to oracle.warp_chain_bound of the fp64 chain on the operands its own preparation made
    (flow_utils.chain_operands).  Returns (out, the fp64 reference)."""
    out = fb.fu.warp_tensor(sample, flows, occs, sal, chunks)
    n, (h, w) = sample.shape[0] // chunks, sample.shape[2:]
    bwd, fwd_last, blend = fb.fu.chain_operands(flows, occs, sal, n, h, w)
    chain_in = sample if 2 * h * w * 4 <= 200 * 1024 else sample.float()         # image planes: the fp32 per-step kernel
    ref, tol = CB.chain_reference_and_bound(chain_in, bwd, fwd_last, blend, chunks, out_dtype=sample.dtype)
    ratio = CB.ratio(out, ref, tol)
    assert out.dtype == sample.dtype and not (ratio > 1).any(), f"warp_tensor: err/tol {ratio.max().item():.3g}"
    return out, ref


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
    ns.ops, ns.dh, ns.fu, ns.lib = ops, diffusion_hacked, flow_utils, _lib
    return ns


def sdpa_ref(q, k, v, heads, q_per_kv=1, scale=None, diag_bias=0.0):
    q, k, v = q.float(), k.float(), v.float()
    B, Lq, C = q.shape
    d = C // heads
    scale = scale if scale is not None else 1 / math.sqrt(d)
    k = k.repeat_interleave(q_per_kv, 0)
    v = v.repeat_interleave(q_per_kv, 0)
    qh = q.view(B, Lq, heads, d).transpose(1, 2)
    kh = k.view(B, -1, heads, d).transpose(1, 2)
    vh = v.view(B, -1, heads, d).transpose(1, 2)
    s = qh @ kh.transpose(-1, -2) * scale
    if diag_bias != 0.0:
        s = s + torch.eye(Lq, kh.shape[2], device=q.device) * diag_bias
    return (torch.softmax(s, -1) @ vh).transpose(1, 2).reshape(B, Lq, C)


ATTN_OPTS = ("FRESCO_ATTN_WIDE", "FRESCO_ATTN_POLY", "FRESCO_ATTN_ROWSUM")


@pytest.fixture
def attn_opts(fb):
    def set_(**kw):
        for name in ATTN_OPTS:
            fb.lib.set_option(name, kw.get(name, -1))
    yield set_
    for name in ATTN_OPTS:
        fb.lib.set_option(name, -1)


VARIANTS = [
    dict(),                                                              # the defaults (per head_dim)
    dict(FRESCO_ATTN_WIDE=1, FRESCO_ATTN_POLY=0),                        # 128-key tiles, two consumer warpgroups
    dict(FRESCO_ATTN_WIDE=1, FRESCO_ATTN_POLY=4),
    dict(FRESCO_ATTN_WIDE=1, FRESCO_ATTN_POLY=8),
    dict(FRESCO_ATTN_WIDE=2, FRESCO_ATTN_POLY=0),                        # 128-key tiles, three consumer warpgroups
    dict(FRESCO_ATTN_WIDE=2, FRESCO_ATTN_POLY=4),
    dict(FRESCO_ATTN_WIDE=2, FRESCO_ATTN_POLY=8),
    dict(FRESCO_ATTN_WIDE=0, FRESCO_ATTN_POLY=0, FRESCO_ATTN_ROWSUM=0),  # 64-key tiles (ROWSUM: row sums by wgmma)
    dict(FRESCO_ATTN_WIDE=0, FRESCO_ATTN_POLY=0, FRESCO_ATTN_ROWSUM=1),
    dict(FRESCO_ATTN_WIDE=0, FRESCO_ATTN_POLY=4, FRESCO_ATTN_ROWSUM=1),
    dict(FRESCO_ATTN_WIDE=0, FRESCO_ATTN_POLY=8, FRESCO_ATTN_ROWSUM=0),
]


@pytest.mark.parametrize("variant", VARIANTS, ids=lambda v: "-".join(f"{k[12:]}{x}" for k, x in v.items()) or "default")
@pytest.mark.parametrize("d", [40, 64, 80, 128])
def test_attention_variants_all_head_dims(fb, attn_opts, variant, d):
    """every attention variant (key-tile width, consumer warpgroups, FMA-pipe exponentials, tensor-core row sums):
    ragged q / kv tails, shared K/V, a peaky softmax (gain 4 / 8: the running max moves), kv lengths that leave most of
    the last key tile masked (20, 33, 77), the diagonal bias + k-scale of spatial-guided attention.
    (Three warpgroups stop at head_dim 64: WIDE=2 is the WIDE=1 launch at 80 and 128.)"""
    attn_opts(**variant)
    heads = 2
    poly = variant.get("FRESCO_ATTN_POLY", 0)
    rowsum = variant.get("FRESCO_ATTN_WIDE", 1) == 0 and variant.get("FRESCO_ATTN_ROWSUM", 0) == 1

    def check(out, q, k, v, qpk, scale=None, bias=0.0, what=""):
        # elementwise against the fp64 reference, within the kernel's error bound (oracle/attention_bound.py)
        ref, tol = AB.ref_and_bound(q, k, v, heads, qpk, scale, bias, poly, rowsum)
        ratio = ((out.double() - ref).abs() / tol).nan_to_num(nan=float("inf"))
        assert ratio.max().item() <= 1.0, (what, ratio.max().item(), (ratio > 1).sum().item())

    g = torch.Generator(device="cuda").manual_seed(17 + d)
    for (B, Lq, Lk, qpk, gain) in [(4, 300, 1000, 2, 4.0), (2, 130, 77, 1, 8.0), (2, 64, 20, 1, 1.0), (2, 128, 33, 2, 1.0),
                                   (2, 256, 4096 + 64, 1, 1.0)]:
        q = (torch.randn(B, Lq, heads * d, device="cuda", generator=g) * gain).half()
        k = torch.randn(B // qpk, Lk, heads * d, device="cuda", generator=g).half()
        v = torch.randn(B // qpk, Lk, heads * d, device="cuda", generator=g).half()
        out = fb.ops.attn_fwd(q, k, v, heads, qpk)
        check(out, q, k, v, qpk, what=(B, Lq, Lk, qpk, gain))
    qs = (torch.randn(2, 256, heads * d, device="cuda", generator=g) * 4.0).half()
    ks = torch.randn(2, 256, heads * d, device="cuda", generator=g).half()
    vs = torch.randn(2, 256, heads * d, device="cuda", generator=g).half()
    out = fb.ops.attn_fwd(qs, ks, vs, heads, 1, softmax_scale=0.2 / math.sqrt(d), diag_bias=1.5)
    check(out, qs, ks, vs, 1, 0.2 / math.sqrt(d), 1.5, "diagonal bias")


def test_attention_level_a_full_size(fb):
    """BASELINE level A (B = 16, L = 1024, d = 80, Lk = 2963): spot rows against fp32 + rows sum to one."""
    g = torch.Generator(device="cuda").manual_seed(12)
    N, chunks, L, heads, d, Lk = 8, 2, 1024, 8, 80, 2963
    C = heads * d
    q = torch.randn(chunks * N, L, C, device="cuda", generator=g).half()
    k = torch.randn(chunks, Lk, C, device="cuda", generator=g).half()
    v = torch.randn(chunks, Lk, C, device="cuda", generator=g).half()
    o = fb.ops.attn_fwd(q, k, v, heads, N).float()
    oc = fb.ops.attn_fwd(q, k, torch.full_like(v, 0.75), heads, N).float()
    assert (oc - 0.75).abs().max().item() < 1e-3
    rows = torch.randint(0, L, (32,), generator=torch.Generator().manual_seed(2)).tolist()
    for b in (0, 9, 15):
        ref = sdpa_ref(q[b:b + 1, rows], k[b // N:b // N + 1], v[b // N:b // N + 1], heads)
        assert (o[b, rows] - ref[0]).abs().max().item() < 2e-3 * ref.abs().max().item()


# ------------------------------------------------------------------------------------------------ golden set B
class FakeAttn(torch.nn.Module):
    def __init__(self, g):
        super().__init__()
        c = g["wq"].shape[0]
        self.heads = int(g["heads"])
        self.spatial_norm = self.group_norm = None
        self.norm_cross = self.residual_connection = False
        self.rescale_output_factor = 1.0
        self.to_q, self.to_k, self.to_v = (torch.nn.Linear(c, c, bias=False) for _ in range(3))
        self.to_out = torch.nn.ModuleList([torch.nn.Linear(c, c), torch.nn.Dropout(0.0)])
        with torch.no_grad():
            for lin, key in ((self.to_q, "wq"), (self.to_k, "wk"), (self.to_v, "wv"), (self.to_out[0], "wo")):
                lin.weight.copy_(T(g[key], "cpu"))
            self.to_out[0].bias.copy_(T(g["bo"], "cpu"))


def _run_processor(fb, attn, x, ref_hidden, masks, paras, flags):
    ctrl = fb.dh.AttentionControl()
    proc = fb.dh.FRESCOAttnProcessor2_0(2, ctrl)
    if flags & 2:
        ctrl.stored_attn["decoder_attn"] = [ref_hidden.clone()]
        ctrl.enable_intraattn()
    if flags & 4:
        ctrl.enable_interattn(paras)
    if flags & 1:
        ctrl.enable_cfattn(masks)
    with torch.no_grad():
        return proc(attn, x.clone()).float().cpu()


@pytest.mark.parametrize("fixture", ["attention", "set_b"])
def test_processor_reference_outputs_at_stated_tolerance(fb, golden, fixture):
    """The reference's own fp32 outputs for the on/off combinations of the three attention modes.  The Linear layers
    are kept in fp32 here (the processor casts q/k/v to fp16 for the kernels and the result back), so what is compared
    is the kernels' arithmetic: 2e-3 * max|y|, the tolerance stated for fp16 attention."""
    g = golden(fixture)
    attn = FakeAttn(g).cuda()                                   # fp32 weights
    x, ref_hidden = T(g["x"]).float(), T(g["ref_hidden"]).float()
    masks = [T(g[f"attn_mask{i}"]) for i in range(3)]
    paras = {"fwd_mappings": [T(g["fwd_map"])], "bwd_mappings": [T(g["bwd_map"])], "interattn_masks": [T(g["inter_mask"])]}
    for flags in (range(8) if fixture == "attention" else (0, 1, 6, 7)):
        out = _run_processor(fb, attn, x, ref_hidden, masks, paras, flags)
        ref = T(g[f"out_{flags}"], "cpu")
        err = (out - ref).abs().max().item()
        assert err < 2e-3 * ref.abs().max().item(), (fixture, flags, err, ref.abs().max().item())


def test_set_b_through_the_kernels(fb, golden):
    """golden set B (generated from the reference): mapping / trajectory mask bit-exact, fp16 processor, warp_tensor on
    a non-square plane (feature and image resolution), optimize_feature loss curves."""
    g = golden("set_b")
    fm, bm, mask = fb.fu.get_mapping_ind(T(g["bwd"]), T(g["bwd_occ"]), T(g["imgs"]), scale=8.0)
    assert torch.equal(fm.cpu(), T(g["fwd_map"], "cpu")) and torch.equal(bm.cpu(), T(g["bwd_map"], "cpu"))
    assert torch.equal(mask.cpu(), T(g["inter_mask"], "cpu"))
    attn = FakeAttn(g).cuda().half()
    x, ref_hidden = T(g["x"]).half(), T(g["ref_hidden"]).half()
    masks = [T(g[f"attn_mask{i}"]) for i in range(3)]
    paras = {"fwd_mappings": [T(g["fwd_map"])], "bwd_mappings": [T(g["bwd_map"])], "interattn_masks": [T(g["inter_mask"])]}
    for flags in (0, 1, 6, 7):
        out = _run_processor(fb, attn, x, ref_hidden, masks, paras, flags)
        ref = T(g[f"out_{flags}"], "cpu")
        # fp16 weights and activations through the 4 Linear layers (torch / cuBLAS) dominate this error, not the kernels
        assert (out - ref).abs().max().item() < 1e-2 * ref.abs().max().item(), flags
    flows, occs, sal = [T(g["fwd"]), T(g["bwd"])], [T(g["fwd_occ"]), T(g["bwd_occ"])], T(g["saliency"])
    _, ref = _warp_tensor_within_bound(fb, T(g["sample_feat"]), flows, occs, sal, 2)
    assert (ref - T(g["out_feat"]).double()).abs().max().item() < 2e-5         # the reference's fp32 arithmetic
    _, ref = _warp_tensor_within_bound(fb, T(g["sample_img"]), flows, occs, sal, 1)
    assert (ref - T(g["out_img"]).double()).abs().max().item() < 2e-5
    for tag, iters in (("full1", 1), ("full3", 3)):
        tr = fb.dh.OptimizeTrace()
        out = fb.dh.optimize_feature(T(g["opt_sample"]), flows, occs, correlation_matrix=[T(g["opt_target"])],
                                     intra_weight=1e2, iters=iters, trace=tr)
        assert np.allclose(np.array(tr.losses), g[f"opt_{tag}_losses"], rtol=1e-2), (tag, tr.losses)
        diff = (out.cpu() - T(g[f"opt_{tag}_out"], "cpu")).abs()
        if iters == 1:
            # Adam's first step moves every element by exactly +-lr: an element whose tiny gradient changes sign under the
            # fp16 Gram operands lands 2*lr away, all the others agree closely (4 % of them flip on this fixture)
            assert (diff > 2e-3).float().mean().item() < 0.06
            assert diff.median().item() < 1e-4
        else:
            assert (diff.mean() / T(g[f"opt_{tag}_out"], "cpu").abs().mean()).item() < 0.1


# ------------------------------------------------------------------------------------------------ temporal attention
def _trajectory_case(N, L, seed):
    """random per-frame permutations (a trajectory visits an arbitrary token of every frame) and trajectory masks with
    the reference's structure: block-diagonal cuts between frames <= i and > i (flow_utils.py:126-133)."""
    g = torch.Generator().manual_seed(seed)
    fwd = torch.stack([torch.arange(L)] + [torch.randperm(L, generator=g) for _ in range(N - 1)])
    mask = torch.ones(L, N, N, dtype=torch.bool)
    for i in range(N - 1):
        cut = torch.ones(N, N, dtype=torch.bool)
        cut[:i + 1, i + 1:] = False
        cut[i + 1:, :i + 1] = False
        sel = torch.rand(L, generator=g) < 0.15
        mask[sel] = mask[sel] & cut
    return fwd, mask


@pytest.mark.parametrize("N,L,heads,d", [(8, 4096, 8, 40), (8, 1024, 8, 80), (3, 96, 2, 80), (5, 200, 4, 64)])
def test_temporal_attention_bench_shapes(fb, N, L, heads, d):
    """A5 at the shapes bench.py runs (level B: N=8, 8 heads, d=40, L=4096; level A: d=80, L=1024) + odd sizes:
    every trajectory within oracle.temporal_bound of the fp64 formula, and every output row written (NaN prefill)."""
    chunks, C = 2, heads * d
    g = torch.Generator(device="cuda").manual_seed(N * 1000 + L)
    q = torch.randn(chunks * N, L, C, device="cuda", generator=g).half()
    k = (torch.randn(chunks * N, L, C, device="cuda", generator=g) * 2.0).half()
    a = torch.randn(chunks * N, L, C, device="cuda", generator=g).half()
    fwd, mask = _trajectory_case(N, L, seed=L + N)
    fwd, mask = fwd.cuda().contiguous(), mask.to(torch.uint8).cuda().contiguous()
    scale = 0.2 / math.sqrt(d)
    out = torch.full_like(a, float("nan"))
    fb.lib.check(fb.lib.lib().fresco_temporal_attn_fwd(q.data_ptr(), k.data_ptr(), a.data_ptr(), out.data_ptr(),
                                                       fwd.data_ptr(), mask.data_ptr(), chunks, N, L, heads, d, scale,
                                                       fb.lib.stream()), "fresco_temporal_attn_fwd")
    ref, tol = TB.ref_and_bound(q, k, a, fwd, mask, chunks, heads, scale)
    ratio = TB.ratio(out, ref, tol)
    assert not (ratio > 1).any(), f"err/tol {ratio.max().item():.3g}; {(ratio > 1).sum().item()} elements outside"


# ------------------------------------------------------------------------------------------------ optimize_feature
def _layer_case(N, C, h, seed, res=512, mag=12.0):
    flows, occs = O.synth_flows(N, res, res, seed=seed, mag=mag)
    g = torch.Generator().manual_seed(seed + 50)
    base = torch.randn(2, 1, C, h, h, generator=g)
    cs = (base + 0.5 * torch.randn(2, N, C, h, h, generator=g)).contiguous()          # frames correlated, like features
    return flows, occs, cs


@pytest.mark.parametrize("N,C,h", [(8, 1280, 32), (8, 640, 64), (8, 1280, 16), (8, 1280, 8)])
def test_temporal_loss_teacher_forced_layer_shapes(fb, N, C, h):
    """O2 at the decoder shapes of BASELINE config 3 ([16,1280,8..32,..], [16,640,64,64]): loss and gradient of one
    evaluation against the oracle's formulas in fp32 (torch on the GPU; autograd adjoint of grid_sample)."""
    flows, occs, cs = _layer_case(N, C, h, seed=h)
    ff, bf, fo, bo = O._resize_flow_occ(flows, occs, h / flows[0].shape[2])
    dev = "cuda"
    csd = cs.to(dev)
    loss_ref, grad_ref = O.temporal_loss_and_grad(csd, ff.to(dev).repeat(2, 1, 1, 1), bf.to(dev).repeat(2, 1, 1, 1),
                                                  (1 - fo).to(dev).repeat(2, 1, 1, 1), (1 - bo).to(dev).repeat(2, 1, 1, 1))
    grad = torch.full_like(csd, 3.0)
    loss = torch.zeros(1, device=dev)
    fb.ops.warp_loss_fwd_bwd(csd, ff.to(dev).contiguous(), bf.to(dev).contiguous(), (1 - fo).reshape(N, h, h).to(dev).contiguous(),
                             (1 - bo).reshape(N, h, h).to(dev).contiguous(), grad, loss, accumulate=False)
    assert abs(loss.item() - float(loss_ref)) < 1e-4 * abs(float(loss_ref))
    gmax = grad_ref.abs().max().item()
    # the gradient is a sum of +-k and bilinear weights of +-k: elements where a residual is within rounding of zero may
    # flip a sign, everything else agrees to the 16-bit weights of the adjoint
    bad = ((grad - grad_ref).abs() > 1e-3 * gmax).float().mean().item()
    assert bad < 1e-4, bad
    cos = torch.nn.functional.cosine_similarity(grad.flatten(), grad_ref.flatten(), dim=0).item()
    assert cos > 0.9999, cos


def test_temporal_loss_adjoint_overflow_path(fb):
    """A contracting flow sends ~16 source pixels to every destination pixel: the 8-slot ELL rows overflow and the
    remaining taps go through the overflow list (n_ovf > 0)."""
    N, C, h = 3, 8, 32
    g = torch.Generator().manual_seed(3)
    ys, xs = torch.meshgrid(torch.arange(h, dtype=torch.float32), torch.arange(h, dtype=torch.float32), indexing="ij")
    contract = torch.stack([(h / 2 - xs) * 0.75 + 0.3, (h / 2 - ys) * 0.75 - 0.2])                # sample near the centre
    bf = torch.randn(N, 2, h, h, generator=g) * 1.5
    ff = torch.randn(N, 2, h, h, generator=g) * 1.5
    bf[0] = contract
    ff[1] = contract
    keep_f = (torch.rand(N, 1, h, h, generator=g) > 0.2).float()
    keep_b = (torch.rand(N, 1, h, h, generator=g) > 0.2).float()
    cs = torch.randn(2, N, C, h, h, generator=g)
    adj = fb.ops.warp_adjoint_pair(bf.cuda().contiguous(), ff.cuda().contiguous())
    assert adj.n_ovf > 0, "fixture must overflow the ELL rows"
    loss_ref, grad_ref = O.temporal_loss_and_grad(cs, ff.repeat(2, 1, 1, 1), bf.repeat(2, 1, 1, 1), keep_f.repeat(2, 1, 1, 1),
                                                  keep_b.repeat(2, 1, 1, 1))
    grad = torch.empty_like(cs).cuda()
    loss = torch.zeros(1, device="cuda")
    fb.ops.warp_loss_fwd_bwd(cs.cuda(), ff.cuda().contiguous(), bf.cuda().contiguous(), keep_f.reshape(N, h, h).cuda().contiguous(),
                             keep_b.reshape(N, h, h).cuda().contiguous(), grad, loss, accumulate=False, adjoint=adj)
    assert abs(loss.item() - float(loss_ref)) < 1e-5 * abs(float(loss_ref))
    assert (grad.cpu() - grad_ref).abs().max().item() < 1e-6 + 2e-4 * grad_ref.abs().max().item()
    # the generic kernels (planes the quad kernel does not take: channels % 4 != 0) through the same entry point
    cs3 = cs[:, :, :6].contiguous()
    loss_ref3, grad_ref3 = O.temporal_loss_and_grad(cs3, ff.repeat(2, 1, 1, 1), bf.repeat(2, 1, 1, 1), keep_f.repeat(2, 1, 1, 1),
                                                    keep_b.repeat(2, 1, 1, 1))
    grad3 = torch.empty_like(cs3).cuda()
    loss3 = torch.zeros(1, device="cuda")
    fb.ops.warp_loss_fwd_bwd(cs3.cuda(), ff.cuda().contiguous(), bf.cuda().contiguous(), keep_f.reshape(N, h, h).cuda().contiguous(),
                             keep_b.reshape(N, h, h).cuda().contiguous(), grad3, loss3, accumulate=False, adjoint=adj)
    assert abs(loss3.item() - float(loss_ref3)) < 1e-5 * abs(float(loss_ref3))
    assert (grad3.cpu() - grad_ref3).abs().max().item() < 1e-6 + 2e-4 * grad_ref3.abs().max().item()


@pytest.mark.parametrize("N,C,h,world", [(8, 640, 64, 2), (8, 1280, 16, 4), (8, 1280, 8, 8), (6, 6, 24, 3), (8, 6, 32, 2),
                                         (4, 4, 100, 2), (8, 640, 96, 2)])
def test_temporal_loss_open_chain_equals_ring(fb, N, C, h, world):
    """Exchange 3 of the frame partition (SURVEY 8e): every "rank" evaluates its own pairs with the following rank's first
    frame as halo (fresco_warp_loss_fwd_bwd_halo) and hands the halo gradient on; the assembled gradient must be
    BIT-identical to the closed ring over all N frames, ELL overflow lists included (they are summed in list order, no
    atomics) -- quad kernel, channel-grouped kernel (C = 6 / 24; config 5's 96 x 96 planes: P = 18) and the
    one-plane-per-CTA kernel (100 x 100 planes; that one associates the overflow terms differently, so it is
    bit-identical only when no ELL row overflows)."""
    flows, occs, cs = _layer_case(N, C, h, seed=7 * h + world, res={100: 800, 96: 768}.get(h, 512))
    ff, bf, fo, bo = O._resize_flow_occ(flows, occs, h / flows[0].shape[2])
    dev = "cuda"
    cs = cs.to(dev)
    ff, bf = ff.to(dev).contiguous(), bf.to(dev).contiguous()
    kf, kb = (1 - fo).reshape(N, h, h).to(dev).contiguous(), (1 - bo).reshape(N, h, h).to(dev).contiguous()
    adj = fb.ops.warp_adjoint_pair(bf, ff)
    ring = torch.empty_like(cs)
    loss_ring = torch.zeros(1, device=dev)
    fb.ops.warp_loss_fwd_bwd(cs, ff, bf, kf, kb, ring, loss_ring, adjoint=adj)
    grads, halos = [], []
    loss = torch.zeros(1, device=dev)
    n = N // world
    for r in range(world):
        lo, hi = r * n, (r + 1) * n
        mine = cs[:, lo:hi].contiguous()
        halo_cs = cs[:, hi % N].contiguous()
        g = torch.full_like(mine, 7.0)
        hg = torch.full_like(halo_cs, 9.0)
        fb.ops.warp_loss_fwd_bwd(mine, ff[lo:hi], bf[lo:hi], kf[lo:hi], kb[lo:hi], g, loss,
                                 adjoint=fb.ops.WarpAdjointSlice(adj, lo, hi), halo_cs=halo_cs, halo_grad=hg, total_frames=N)
        grads.append(g)
        halos.append(hg)
    for r in range(world):                                   # rank r's halo gradient belongs to rank r+1's first frame
        grads[(r + 1) % world][:, 0] += halos[r]
    got = torch.cat(grads, 1)
    if h * h > 9216 and adj.n_ovf > 0:
        assert (got - ring).abs().max().item() < 1e-6 * ring.abs().max().item()
    else:
        assert torch.equal(got, ring), (adj.n_ovf, (got - ring).abs().max().item())
    assert abs(loss.item() - loss_ring.item()) < 1e-5 * abs(loss_ring.item())


class _LockstepRing:
    """Ring communicator for `world` ranks emulated by threads of ONE process on one GPU: a rank holds the lock while it
    issues work and gives it up only inside an exchange, so the ranks' kernel sequences interleave exactly at the halo
    exchanges (all on the same stream: program order is execution order)."""

    def __init__(self, world):
        import threading
        self.world = world
        self.lock = threading.Lock()
        self.barrier = threading.Barrier(world)
        self.slots = [None] * world

    class _Comm:
        def __init__(self, ring, rank):
            self.ring, self.rank = ring, rank

        def _publish(self, t):
            r = self.ring
            r.slots[self.rank] = t
            r.lock.release()
            r.barrier.wait()
            r.lock.acquire()

        def _done(self):
            r = self.ring
            r.lock.release()
            r.barrier.wait()
            r.lock.acquire()

        def shift(self, send, recv, direction):
            self._publish(send)
            recv.copy_(self.ring.slots[(self.rank - direction) % self.ring.world])
            self._done()

        def all_reduce_sum(self, t):
            self._publish(t.clone())
            total = sum(self.ring.slots[1:], self.ring.slots[0].clone())
            self._done()
            t.copy_(total)

    def comm(self, rank):
        return self._Comm(self, rank)


@pytest.mark.parametrize("N,C,h,world", [(8, 640, 64, 2), (8, 1280, 16, 4)])
def test_optimize_feature_ring_halo_bit_identical(fb, N, C, h, world):
    """optimize_feature on a frame-sharded batch (the ranks emulated by threads in lock step, real kernels): temporal +
    Gram-L1 terms, Adam, AdaIN -- the ranks' outputs together are BIT-identical to the unsharded call."""
    import threading
    flows, occs, cs = _layer_case(N, C, h, seed=31 + h)
    flows = [f.cuda() for f in flows]
    occs = [o.cuda() for o in occs]
    sample = cs.reshape(2 * N, C, h, h).half().cuda()
    g = torch.Generator(device="cuda").manual_seed(5)
    ref = (sample.float() + 0.5 * torch.randn(sample.shape, device="cuda", generator=g)).half()
    target = fb.dh.gram_targets([ref])[0]
    full = fb.dh.optimize_feature(sample, flows, occs, correlation_matrix=[target], iters=6)
    ring = _LockstepRing(world)
    n = N // world
    outs, errs = [None] * world, []

    def run(rank):
        ring.lock.acquire()
        try:
            sel = torch.cat([torch.arange(c * N + rank * n, c * N + (rank + 1) * n) for c in range(2)]).cuda()
            tgt = fb.dh.GramTarget(target.yhat[sel].contiguous())
            outs[rank] = (sel, fb.dh.optimize_feature(sample[sel].contiguous(), flows, occs, correlation_matrix=[tgt], iters=6,
                                                      shard=(world, rank, ring.comm(rank))))
        except Exception as e:                                  # noqa: BLE001 (reported below; a dead rank must not hang the others)
            errs.append(e)
            ring.barrier.abort()
        finally:
            ring.lock.release()
    threads = [threading.Thread(target=run, args=(r,)) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(300)
    assert not errs, errs
    for sel, out in outs:
        assert torch.equal(out, full[sel])


@pytest.mark.parametrize("N,C,h", [(8, 1280, 32), (8, 640, 64)])
def test_spatial_loss_teacher_forced_layer_shapes(fb, N, C, h):
    """O3 at layers 2 and 3 of config 3 ([16,1280,32,32], [16,640,64,64]): loss, sign matrix exact outside the fp16
    error band, gradient (fp32 torch on the GPU as the reference of the same formulas)."""
    B, L = 2 * N, h * h
    _, _, cs = _layer_case(N, C, h, seed=7 + h)
    cs = cs.cuda()
    ref_feat = (cs + 0.7 * torch.randn(cs.shape, device="cuda", generator=torch.Generator(device="cuda").manual_seed(h))).half()
    target = fb.dh.gram_targets([ref_feat.reshape(B, C, h, h)])[0]                   # GramTarget: normalised features
    dense = target.dense()                                                           # the reference's fp16-bmm -> fp32 store
    assert tuple(target.shape) == (B, L, L) and dense.shape == (B, L, L) and dense.dtype == torch.float32
    loss_ref, grad_ref = O.spatial_loss_and_grad(cs, dense, 100.0)
    # one evaluation of optimize_feature's spatial branch (the function optimize_feature itself calls)
    grad = torch.zeros(B, C, L, device="cuda")
    loss = torch.zeros(1, device="cuda")
    fb.dh.spatial_loss_grad(cs.view(B, C, L), target, 100.0, grad, loss)
    assert abs(loss.item() - float(loss_ref)) < 2e-3 * float(loss_ref)
    gr = grad_ref.reshape(B, C, L)
    rel = ((grad - gr).abs().mean() / gr.abs().mean()).item()
    cos = torch.nn.functional.cosine_similarity(grad.flatten(), gr.flatten(), dim=0).item()
    assert rel < 3e-2 and cos > 0.999, (rel, cos)
    # the dense-target entry point (what a caller holding the reference's own correlation_matrix uses) agrees
    grad2 = torch.zeros(B, C, L, device="cuda")
    loss2 = torch.zeros(1, device="cuda")
    fb.dh.spatial_loss_grad(cs.view(B, C, L), dense, 100.0, grad2, loss2)
    assert abs(loss2.item() - float(loss_ref)) < 2e-3 * float(loss_ref)
    assert torch.nn.functional.cosine_similarity(grad2.flatten(), gr.flatten(), dim=0).item() > 0.999


def test_optimize_feature_full_layer3_loss_curve(fb):
    """20 Adam iterations at layer 3 ([16,640,64,64], temporal + spatial): the loss curve against the oracle's formulas
    run in fp32 on the GPU (the optimisation is chaotic elementwise, SURVEY 9: curves within 1e-2, AdaIN statistics)."""
    N, C, h = 8, 640, 64
    flows, occs, cs = _layer_case(N, C, h, seed=21)
    sample = cs.reshape(2 * N, C, h, h).cuda().half()
    ref_feat = (sample.float() + 0.7 * torch.randn(sample.shape, device="cuda",
                                                   generator=torch.Generator(device="cuda").manual_seed(5))).half()
    target = fb.dh.gram_targets([ref_feat])[0]
    fl, oc = [f.cuda() for f in flows], [o.cuda() for o in occs]
    tr = fb.dh.OptimizeTrace()
    out = fb.dh.optimize_feature(sample, fl, oc, correlation_matrix=[target], intra_weight=1e2, iters=20, trace=tr)
    ref_out, ref_trace = O.optimize_feature(sample, fl, oc, correlation_matrix=[target.dense()], intra_weight=1e2, iters=20,
                                            return_trace=True)
    ref_losses = [t["loss"] for t in ref_trace]
    del ref_trace
    assert out.shape == sample.shape and out.dtype == torch.float16
    # AdaIN pins the per-(sample, channel) statistics of the output to those of the input (eps quirk aside)
    m_in, m_out = sample.float().mean((2, 3)), out.float().mean((2, 3))
    assert (m_in - m_out).abs().max().item() < 2e-2
    m_ref = ref_out.float().mean((2, 3))
    assert (m_ref - m_out).abs().max().item() < 2e-2
    losses = np.array(tr.losses)
    assert losses[-1] < losses[0]
    assert np.allclose(losses, np.array(ref_losses), rtol=1e-2), (losses, ref_losses)


@pytest.mark.parametrize("B,C,h,w", [(4, 64, 8, 8), (2, 320, 16, 24), (2, 16, 24, 24), (2, 640, 32, 32), (2, 1280, 16, 16)])
def test_gram_sign_recomputed_target(fb, B, C, h, w):
    """O3 with the target recomputed in the kernel (fresco_gram_sign_ref) + the 128 x 256 T Xh product: sign matrix exact
    outside the fp16 error band, loss, gradient -- incl. plane sizes that are not multiples of the tile (576, 384)."""
    L = h * w
    g = torch.Generator().manual_seed(C + h)
    cs = torch.randn(B, C, L, generator=g)
    ref = (cs + 0.7 * torch.randn(B, C, L, generator=g)).half().cuda()
    target = fb.dh.gram_targets([ref.reshape(B, C, h, w)])[0]
    assert isinstance(target, fb.dh.GramTarget)
    dense = target.dense().cpu()
    loss_ref, grad_ref = O.spatial_loss_and_grad(cs.reshape(1, B, C, h, w), dense, 100.0)
    X = cs.transpose(1, 2)
    Xh = X / (X ** 2).sum(2, keepdim=True) ** 0.5
    D = torch.bmm(Xh, Xh.transpose(1, 2)) - dense
    T_ref = torch.sign(D) + torch.sign(D.transpose(1, 2))
    xhat, norms = fb.ops.gram_normalize(cs.cuda())
    loss = torch.zeros(1, device="cuda")
    tsign = fb.ops.gram_sign_ref(xhat, target.yhat, 100.0, loss)
    safe = (D.abs() > 2e-3) & (D.transpose(1, 2).abs() > 2e-3)
    assert safe.float().mean() > 0.8
    assert torch.equal(tsign.float().cpu()[safe], T_ref[safe])
    assert abs(loss.item() - float(loss_ref)) < 2e-3 * float(loss_ref)
    grad = torch.zeros(B, C, L, device="cuda")
    fb.ops.gram_grad(tsign, xhat, norms, grad, 100.0)
    gr = grad_ref.reshape(B, C, L)
    rel = ((grad.cpu() - gr).abs().mean() / gr.abs().mean()).item()
    cos = torch.nn.functional.cosine_similarity(grad.cpu().flatten(), gr.flatten(), dim=0).item()
    assert rel < 3e-2 and cos > 0.999, (rel, cos)
    # the round-1 128 x 128 product behind the same entry point gives the same gradient
    fb.lib.set_option("FRESCO_GRAM_V", 1)
    try:
        grad1 = torch.zeros(B, C, L, device="cuda")
        fb.ops.gram_grad(tsign, xhat, norms, grad1, 100.0)
    finally:
        fb.lib.set_option("FRESCO_GRAM_V", -1)
    assert (grad1 - grad).abs().max().item() < 1e-5 * grad.abs().max().item() + 1e-12


# ------------------------------------------------------------------------------------------------ caches, dtypes
def test_two_keyframe_batches_do_not_share_prepared_flows(fb):
    """ADVICE r1 (high): same-shape flows of a second batch must not hit the first batch's cached preparation."""
    outs, refs = [], []
    for seed in (1, 2, 3, 4):
        flows, occs = O.synth_flows(3, 128, 128, seed=seed, mag=6.0)
        sal = torch.rand(3, 1, 64, 64, generator=torch.Generator().manual_seed(seed))
        feat = torch.randn(6, 8, 16, 16, generator=torch.Generator().manual_seed(100 + seed))
        fl, oc, sl = [f.cuda() for f in flows], [o.cuda() for o in occs], sal.cuda()
        outs.append(fb.fu.warp_tensor(feat.cuda(), fl, oc, sl, 2).cpu())
        outs.append(fb.fu.warp_tensor(feat.cuda(), fl, oc, sl, 2).cpu())
        r = O.warp_tensor(feat, flows, occs, sal, 2)
        refs += [r, r]
        del fl, oc, sl
    for o, r in zip(outs, refs):
        assert (o - r).abs().max().item() < 5e-5


def test_warp_tensor_fp16_image_resolution(fb):
    """ADVICE r1 (medium): the background-smoothing call warps the fp16 VAE image at 512 x 512 (pipe_FRESCO.py:46)."""
    N, H, W = 3, 256, 320
    flows, occs = O.synth_flows(N, H, W, seed=4, mag=6.0)
    sal = torch.rand(N, 1, H // 2, W // 2, generator=torch.Generator().manual_seed(0))
    img = torch.randn(N, 3, H, W, generator=torch.Generator().manual_seed(1)).half()
    _, ref = _warp_tensor_within_bound(fb, img.cuda(), [f.cuda() for f in flows], [o.cuda() for o in occs], sal.cuda(), 1)
    assert (ref.cpu() - O.warp_tensor(img.float(), flows, occs, sal, 1).double()).abs().max().item() < 5e-5


# ------------------------------------------------------------------------------------------------ GMFlow transformer rows
def test_gmflow_transformer_attention_golden(fb, golden):
    """SURVEY 8(f)-1 through the kernels: full / 2 x 2 windows / shifted windows (d = 128, one head) and the
    flow-propagation attention (V = flow) against the reference's outputs."""
    from fresco_b200 import gmflow_transformer as gt
    g = golden("gmflow_attn")
    q, k, v = (T(g[n]).float() for n in "qkv")
    h, w = int(g["h"]), int(g["w"])
    tol = 2e-3 * float(abs(g["out_full"]).max())
    assert (gt.single_head_full_attention(q, k, v).cpu() - T(g["out_full"], "cpu")).abs().max().item() < tol
    o = gt.single_head_split_window_attention(q, k, v, num_splits=2, with_shift=False, h=h, w=w)
    assert (o.cpu() - T(g["out_split"], "cpu")).abs().max().item() < tol
    o = gt.single_head_split_window_attention(q, k, v, num_splits=2, with_shift=True, h=h, w=w)
    assert (o.cpu() - T(g["out_shift"], "cpu")).abs().max().item() < tol

    class FFA(torch.nn.Module):
        def __init__(self):
            super().__init__()
            c = g["ffa_wq"].shape[0]
            self.q_proj, self.k_proj = torch.nn.Linear(c, c), torch.nn.Linear(c, c)
            with torch.no_grad():
                self.q_proj.weight.copy_(T(g["ffa_wq"], "cpu")), self.q_proj.bias.copy_(T(g["ffa_bq"], "cpu"))
                self.k_proj.weight.copy_(T(g["ffa_wk"], "cpu")), self.k_proj.bias.copy_(T(g["ffa_bk"], "cpu"))
    out = gt.feature_flow_attention(FFA().cuda(), T(g["ffa_f0"]).float(), T(g["ffa_flow"]))
    assert (out.cpu() - T(g["ffa_out"], "cpu")).abs().max().item() < 2e-2            # pixels
    # GMFlow's real shape at 512 x 512: 64 x 64 tokens, 8 pairs bidirectional -> 16 x 4 windows of 1024 tokens
    gen = torch.Generator(device="cuda").manual_seed(3)
    qq, kk, vv = (torch.randn(4, 4096, 128, device="cuda", generator=gen) for _ in range(3))
    o = gt.single_head_split_window_attention(qq, kk, vv, num_splits=2, with_shift=True, h=64, w=64)
    rows = [0, 31 * 64 + 31, 32 * 64 + 5, 47 * 64 + 50, 63 * 64 + 63]              # one token of each region type
    sh = 16
    yy, xx = torch.meshgrid(torch.arange(64), torch.arange(64), indexing="ij")
    ry, rx = (yy - sh) % 64, (xx - sh) % 64                                           # rolled coordinates of every token
    cls = lambda t: (t >= 32).long() * 2 + ((t >= 32) & (t >= 48)).long()             # window half + seam class
    key_all = (cls(ry) * 4 + cls(rx)).reshape(-1).cuda()
    for r in rows:
        allowed = key_all == key_all[r]
        s = (qq[:, r].half().float()[:, None] * kk.half().float()).sum(-1) / math.sqrt(128)
        s = s.masked_fill(~allowed[None], float("-inf"))
        ref = torch.einsum("bl,blc->bc", torch.softmax(s, -1), vv.half().float())
        assert (o[:, r] - ref).abs().max().item() < 2e-3 * ref.abs().max().item()


# ------------------------------------------------------------------------------------------------ step epilogue, dilation
def test_ddpm_step_kernels_and_dilate_golden(fb, golden):
    """fresco_cfg_pred_x0 / fresco_ddpm_prev through fresco_b200.pipe_FRESCO.step vs the reference's step()
    (src/pipe_FRESCO.py:14-77, guidance :212-215), fp32 to 1e-5 and fp16 to 3 fp16 ulps of the largest value; Dilate exact."""
    from fresco_b200 import pipe_FRESCO as pf
    g = golden("ddpm_step")

    class Sched:
        alphas_cumprod = T(g["alphas_cumprod"], "cpu")
        one = torch.tensor(1.0)

        @staticmethod
        def previous_timestep(t):
            return t - 50

    class Pipe:
        scheduler = Sched()
    raw, sample = T(g["raw"]), T(g["sample"])
    for tag in "abc":
        ts, rep = int(g[f"{tag}_t"]), bool(g[f"{tag}_repeat"])
        prev, x0 = pf.step(Pipe, raw, ts, sample, None, repeat_noise=rep, guidance_scale=7.5, noise=T(g[f"{tag}_noise"]))
        for got, want in ((prev, T(g[f"{tag}_prev"], "cpu")), (x0, T(g[f"{tag}_x0"], "cpu"))):
            assert (got.cpu() - want).abs().max().item() < 2e-6 * want.abs().max().item() + 1e-6     # fp32, values up to ~40
        prev16, _ = pf.step(Pipe, raw.half(), ts, sample.half(), None, repeat_noise=rep, guidance_scale=7.5,
                            noise=T(g[f"{tag}_noise"]).half())
        ref = T(g[f"{tag}_prev"], "cpu")
        assert prev16.dtype == torch.float16
        assert (prev16.float().cpu() - ref).abs().max().item() < 4e-3 * ref.abs().max().item()
    m = T(g["dil_in"])
    assert torch.equal(fb.ops.dilate(m, 5).cpu(), T(g["dil5"], "cpu"))
    assert torch.equal(fb.ops.dilate(m, 13).cpu(), T(g["dil13"], "cpu"))


# ------------------------------------------------------------------------------------------------ NCCL, world size 2
def _nccl_worker(rank, world, port, ret):
    import os
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    from fresco_b200 import diffusion_hacked as dh
    from fresco_b200.dist import ShardedFRESCOAttention, frame_range
    dev = torch.device("cuda", rank)
    ok = True
    for (N, L, heads, d) in [(4, 256, 2, 40), (8, 1024, 8, 80)]:
        C, chunks = heads * d, 2
        g = torch.Generator().manual_seed(N * 7 + L)
        q, k, v, rq, rk = (torch.randn(chunks * N, L, C, generator=g).half().to(dev) for _ in range(5))
        mask = torch.rand(N, L, generator=g) > 0.6
        mask[0] = True
        fwd, tmask = _trajectory_case(N, L, seed=3)
        paras = {"fwd_mappings": [fwd[:, None].to(dev)], "bwd_mappings": [torch.argsort(fwd, 1)[:, None].to(dev)],
                 "interattn_masks": [tmask[:, None].to(dev)]}
        for flags in range(8):
            ctrl = dh.AttentionControl()
            if flags & 2:
                ctrl.stored_attn["decoder_attn"] = [q]
                ctrl.enable_intraattn()
            if flags & 4:
                ctrl.enable_interattn(paras)
            if flags & 1:
                ctrl.enable_cfattn([mask.to(dev)])
            full = ShardedFRESCOAttention(ctrl, 1, 0, chunks)(q, k, v, heads, ref_q=rq, ref_k=rk)
            lo, hi = frame_range(N, world, rank)
            sel = torch.cat([torch.arange(c * N + lo, c * N + hi) for c in range(chunks)]).to(dev)
            mine = ShardedFRESCOAttention(ctrl, world, rank, chunks)(q[sel].contiguous(), k[sel].contiguous(), v[sel].contiguous(),
                                                                   heads, ref_q=rq[sel].contiguous(), ref_k=rk[sel].contiguous())
            ok = ok and bool(torch.equal(mine, full[sel]))
    # warp_tensor on the frame shard (chain re-sharded by channel: two all-to-alls) == unsharded, bit for bit
    from fresco_b200 import flow_utils as fu
    N, chunks = 8, 2
    flows, occs = O.synth_flows(N, 256, 256, seed=5, mag=6.0)
    flows, occs = [f.to(dev) for f in flows], [o.to(dev) for o in occs]
    sal = torch.rand(N, 1, 128, 128, generator=torch.Generator().manual_seed(2)).to(dev)
    feat = torch.randn(chunks * N, 64, 32, 32, generator=torch.Generator().manual_seed(3)).half().to(dev)
    full = fu.warp_tensor(feat, flows, occs, sal, chunks)
    lo, hi = frame_range(N, world, rank)
    sel = torch.cat([torch.arange(c * N + lo, c * N + hi) for c in range(chunks)]).to(dev)
    mine = fu.warp_tensor(feat[sel].contiguous(), flows, occs, sal, chunks, shard=(world, rank, None))
    ok = ok and bool(torch.equal(mine, full[sel]))
    # optimize_feature on the frame shard (ring halo of one boundary frame per Adam iteration over NCCL send/recv)
    feat32 = torch.randn(chunks * N, 64, 32, 32, generator=torch.Generator().manual_seed(4)).half().to(dev)
    ref32 = (feat32.float() + 0.5 * torch.randn(feat32.shape, generator=torch.Generator().manual_seed(5)).to(dev)).half()
    target = dh.gram_targets([ref32])[0]
    full = dh.optimize_feature(feat32, flows, occs, correlation_matrix=[target], iters=5)
    mine = dh.optimize_feature(feat32[sel].contiguous(), flows, occs, correlation_matrix=[dh.GramTarget(target.yhat[sel].contiguous())],
                               iters=5, shard=(world, rank, None))
    ok_opt = bool(torch.equal(mine, full[sel]))
    if not ok_opt:
        print("rank %d: sharded optimize_feature differs: max |d| = %g" % (rank, (mine.float() - full[sel].float()).abs().max().item()),
              flush=True)
    ok = ok and ok_opt
    t = torch.tensor([1 if ok else 0], device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MIN)
    if rank == 0:
        ret.put(int(t.item()))
    dist.destroy_process_group()


def test_sharded_attention_nccl_world2_bit_identical(fb):
    """frame-sharded FRESCO attention over NCCL on two GPUs (K/V all-gather, trajectory all-to-alls), the channel-resharded
    warp chain and the ring-halo optimize_feature == unsharded, bit for bit.  Needs two devices (gpurun --gpus 2);
    skipped on a one-GPU box."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import socket
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    ret = ctx.Queue()
    procs = [ctx.Process(target=_nccl_worker, args=(r, 2, port, ret)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(300)
        assert p.exitcode == 0
    assert ret.get(timeout=5) == 1
