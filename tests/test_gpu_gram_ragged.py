"""The spatial-consistency (Gram-L1) loss at token counts that are not multiples of 8, the ones the reference's web UI
produces below its 512 resolution setting.

The web UI's "Frame resolution" slider runs from 256 to 512 in steps of 64; ``resize_image`` makes the short side the
slider value and rounds the long side to a multiple of 64.  Decoder layer 0 then has (s/64)(l/64) tokens and layer 1
four times as many, e.g. 25 / 100 at 320 x 320 or 84 / 336 at 448 x 768.  At such counts T [B, L, L] fp16 has a row
stride that is not a multiple of 16 bytes, so the launchers pick the ragged instantiations (DESIGN §3.2).

* padding invariance: zero-padding X^, Y^ and the dense target to roundup(L, 8) and running the aligned call gives the
  same T, g^ and gradient bit for bit, and the same loss up to the order of the cross-CTA sum, on every entry point,
  both products FRESCO_GRAM_V selects and the _scaled forms;
* every output against fp64 within ``oracle.gram_bound`` (``tests/test_gpu_gram.py`` runs its input families);
* NaN-prefilled outputs between NaN guard rows: every element written, no guard touched;
* the launch names: the parent instantiations at aligned counts, the ragged ones otherwise;
* optimize_feature at every failing (resolution, aspect ratio) setting: one iteration within the composed bound of
  oracle/optimize_bound.py, 20-iteration loss curves against the CPU oracle, and one harness-UNet denoise step with
  every FRESCO flag at three of them.
"""
import math
import os
import re
import types

import numpy as np
import pytest
import torch

from oracle import fresco_oracle as O
from oracle import gram_bound as GB
from oracle import layer_bound as LB
from oracle import optimize_bound as OB
from oracle.gram_bound import Run, launched

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "fresco_b200", "csrc")

RAGGED_NAMES = {"gram2_kernel<G2_SIGN,ragged>", "gram2_kernel<G2_GRAD,ragged>", "tile_gemm_kernel<EPI_STORE,1,ragged>"}


# ------------------------------------------------------------------------------------------------ the web UI envelope
def resize_dims(h, w, resolution):
    """(H, W) of src/utils.py resize_image: the short side scaled to ``resolution``, both sides rounded to 64."""
    k = float(resolution) / min(h, w)
    return int(np.round(h * k / 64.0)) * 64, int(np.round(w * k / 64.0)) * 64


ASPECTS = {"1:1": (512, 512), "4:3": (480, 640), "3:4": (640, 480), "16:9": (1080, 1920), "9:16": (1920, 1080)}
SLIDER = range(256, 512, 64)                                          # 512 runs today at every aspect ratio


def envelope():
    """{(H, W)} of every slider value below 512 at every aspect ratio."""
    return sorted({resize_dims(h, w, s) for s in SLIDER for h, w in ASPECTS.values()})


def layer_tokens(H, W):
    return (H // 64) * (W // 64), (H // 32) * (W // 32)


EDGE_TOKENS = [1, 7, 9, 127, 129, 255, 257]                          # the 128- and 256-token tile edges
TOKENS = sorted({t for H, W in envelope() for t in layer_tokens(H, W)} | set(EDGE_TOKENS))
FAILING = [(H, W) for H, W in envelope() if any(t % 8 for t in layer_tokens(H, W))]


def test_envelope_matches_the_issue_table():
    """The rule gives the 1:1 / 4:3 / 16:9 table of the web UI: ten of the twelve settings below 512 have a ragged
    layer-0 or layer-1 token count.  (Needs no GPU.)"""
    land = [resize_dims(h, w, s) for s in SLIDER for h, w in (ASPECTS["1:1"], ASPECTS["4:3"], ASPECTS["16:9"])]
    assert land == [(256, 256), (256, 320), (256, 448), (320, 320), (320, 448), (320, 576), (384, 384), (384, 512),
                    (384, 704), (448, 448), (448, 576), (448, 768)]
    assert sum(any(t % 8 for t in layer_tokens(H, W)) for H, W in land) == 10
    assert layer_tokens(448, 768) == (84, 336) and layer_tokens(320, 320) == (25, 100)
    assert all(t % 16 == 0 for H, W in envelope() for t in ((H // 16) * (W // 16), (H // 8) * (W // 8)))


def test_ragged_launch_names_in_source():
    """The ragged instantiations the launchers can name are exactly the ones this file asserts.  (Needs no GPU.)"""
    names = set()
    for f in ("gram_wgmma.cu", "gemm_wgmma.cu"):
        names.update(re.findall(r"\"(\w+<[\w,]*ragged>)\"", open(os.path.join(CSRC, f)).read()))
    assert names == RAGGED_NAMES


# ------------------------------------------------------------------------------------------------ C ABI helpers
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


def P(t):
    return t.data_ptr()


def same_bits(a, b, what):
    assert a.shape == b.shape, (what, a.shape, b.shape)
    ai = a.contiguous().view(torch.int16 if a.element_size() == 2 else torch.int32)
    bi = b.contiguous().view(torch.int16 if b.element_size() == 2 else torch.int32)
    bad = (ai != bi).sum().item()
    assert bad == 0, f"{what}: {bad} of {a.numel()} elements differ from the padded call"


def atomic_tol(loss):
    """The loss is a sum of per-warp partials added with atomicAdd in whatever order the CTAs finish: each of at most
    8 * SMs additions rounds once."""
    n = 8 * torch.cuda.get_device_properties(0).multi_processor_count
    return n * 2.0 ** -24 * abs(loss) + 1e-30


def operands(B, L, C, seed):
    """cs, cs_ref [B, C, L] fp32 with the statistics of the gram rows (D changes sign), a dense target close to
    X^ X^T and a finite gradient accumulator."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    base = torch.randn(B, C, 1, device="cuda", generator=g)
    cs = (base + torch.randn(B, C, L, device="cuda", generator=g)).contiguous()
    cs_ref = (base + torch.randn(B, C, L, device="cuda", generator=g)).contiguous()
    grad0 = torch.randn(B, C, L, device="cuda", generator=g)
    return cs, cs_ref, grad0, g


def normalize(fb, src):
    B, C, L = src.shape
    xhat = torch.full((B, L, C), float("nan"), dtype=torch.float16, device="cuda")
    norms = torch.full((B, L), float("nan"), dtype=torch.float32, device="cuda")
    launched(fb, "fresco_gram_normalize", fb.c.fresco_gram_normalize(P(src), P(xhat), P(norms), B, C, L,
                                                                     fb.lib.stream()), "gram_normalize_kernel")
    GB.check_normalize(src, xhat, norms)
    return xhat, norms


def pad_tokens(t, Lp, dims):
    """zero-pad ``t`` to Lp along each of ``dims``"""
    for d in dims:
        shape = list(t.shape)
        shape[d] = Lp - t.shape[d]
        t = torch.cat([t, torch.zeros(shape, dtype=t.dtype, device=t.device)], d)
    return t.contiguous()


# ------------------------------------------------------------------------------------------------ the kernels
@pytest.mark.gpu
@pytest.mark.parametrize("N", [3, 8])
@pytest.mark.parametrize("C", [1280, 640])
@pytest.mark.parametrize("L", TOKENS)
def test_gram_entry_points(fb, L, C, N):
    B, weight = 2 * N, 100.0
    Lp = (L + 7) // 8 * 8
    scale = weight / (B * L * L)
    cs, cs_ref, grad0, g = operands(B, L, C, seed=L * 7 + C + N)
    xhat, norms = normalize(fb, cs)
    yhat, _ = normalize(fb, cs_ref)
    target = torch.empty(B, L, L, device="cuda")
    for b in range(B):
        target[b] = (xhat[b].double() @ xhat[b].double().T
                     + 0.05 * torch.randn(L, L, device="cuda", generator=g, dtype=torch.float64)).float()
    run = Run(fb, xhat, yhat, norms, target, grad0, weight, scale)
    run.hygiene()
    # the weight form divides in double and rounds once: the same fp32 scale, so the same bits
    same_bits(run.tsign1, run.tsign, "T (weight form)")
    assert abs(run.loss1.item() - run.loss.item()) <= atomic_tol(run.loss.item())
    for v in (2, 1):
        same_bits(run.grads[(v, "weight")], run.grads[(v, "scaled")], f"grad V={v} (weight form)")
    GB.check_run(run, xhat, yhat, norms, target, grad0, scale, torch.cuda.get_device_properties(0).multi_processor_count)
    if Lp == L:
        return
    # padding invariance: the aligned instantiations on operands zero-padded to Lp, with the same fp32 scale
    xp, yp = pad_tokens(xhat, Lp, [1]), pad_tokens(yhat, Lp, [1])
    np_ = pad_tokens(norms, Lp, [1])
    np_[:, L:] = 1.0
    tp = pad_tokens(target, Lp, [1, 2])
    gp = pad_tokens(grad0, Lp, [2])
    pad = types.SimpleNamespace()
    st = fb.lib.stream()
    pad.tsign = torch.empty(B, Lp, Lp, dtype=torch.float16, device="cuda")
    pad.loss = torch.zeros(1, device="cuda")
    launched(fb, "padded sign_ref", fb.c.fresco_gram_sign_ref_scaled(P(xp), P(yp), P(pad.tsign), P(pad.loss), B, Lp, C,
                                                                     scale, st), "gram2_kernel<G2_SIGN>")
    tsign_d = torch.empty(B, Lp, Lp, dtype=torch.float16, device="cuda")
    loss_d = torch.zeros(1, device="cuda")
    launched(fb, "padded sign", fb.c.fresco_gram_sign_scaled(P(xp), P(tp), P(tsign_d), P(loss_d), B, Lp, C, scale, st),
             "tile_gemm_kernel<EPI_GRAM_SIGN,0>")
    ghat = torch.empty(B, Lp, C, device="cuda")
    launched(fb, "padded tx", fb.c.fresco_gram_tx(P(pad.tsign), P(xp), P(ghat), B, Lp, C, scale, st),
             "gram2_kernel<G2_GRAD>")
    nbytes = int(fb.c.fresco_gram_grad_workspace_bytes(B, Lp, C))
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    grads = {}
    try:
        for v in (2, 1):
            fb.lib.set_option("FRESCO_GRAM_V", v)
            gr = gp.clone()
            launched(fb, f"padded grad V={v}", fb.c.fresco_gram_grad_scaled(P(pad.tsign), P(xp), P(np_), P(gr), B, Lp, C,
                                                                            scale, P(ws), nbytes, st),
                     "gram_project_kernel")
            grads[v] = gr
    finally:
        fb.lib.set_option("FRESCO_GRAM_V", -1)
    torch.cuda.synchronize()
    same_bits(run.tsign, pad.tsign[:, :L, :L], "T")
    assert (pad.tsign[:, L:] == 0).all() and (pad.tsign[:, :, L:] == 0).all()
    assert abs(run.loss.item() - pad.loss.item()) <= atomic_tol(pad.loss.item()), (run.loss.item(), pad.loss.item())
    same_bits(run.tsign_d, tsign_d[:, :L, :L], "T (dense target)")
    assert abs(run.loss_d.item() - loss_d.item()) <= atomic_tol(loss_d.item()), (run.loss_d.item(), loss_d.item())
    same_bits(run.ghat, ghat[:, :L], "g^")
    for v in (2, 1):
        same_bits(run.grads[(v, "scaled")], grads[v][:, :, :L], f"grad (FRESCO_GRAM_V={v})")


@pytest.mark.gpu
@pytest.mark.parametrize("L", [84, 88, 336])
def test_gram_grad_product_instantiation(fb, L):
    """fresco_gram_grad under FRESCO_GRAM_V=1 ends with gram_project_kernel, so the product it launches first is read
    from the profiler: the parent's tile_gemm_kernel<EPI_STORE,1> at an aligned count, the ragged one otherwise."""
    B, C = 16, 1280
    cs, _, _, _ = operands(B, L, C, seed=L)
    xhat, norms = fb.ops.gram_normalize(cs)
    tsign = (2 * torch.sign(torch.randn(B, L, L, device="cuda"))).half()
    grad = torch.zeros(B, C, L, device="cuda")
    fb.lib.set_option("FRESCO_GRAM_V", 1)
    try:
        fb.ops.gram_grad(tsign, xhat, norms, grad, 100.0)                         # warm-up
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            fb.ops.gram_grad(tsign, xhat, norms, grad, 100.0)
            torch.cuda.synchronize()
    finally:
        fb.lib.set_option("FRESCO_GRAM_V", -1)
    kernels = [e.name for e in prof.events() if "tile_gemm_kernel" in e.name]
    want = "tile_gemm_kernel<0, true, true>" if L % 8 else "tile_gemm_kernel<0, true, false>"
    assert kernels and all(want in k for k in kernels), kernels


# ------------------------------------------------------------------------------------------------ optimize_feature
def _setting_id(hw):
    return "%dx%d" % hw


def _layer_case(N, H, W, layer, seed):
    """flows / occlusions of an H x W batch and decoder features of layer 0 or 1 ([2, N, 1280, H/64, W/64] or /32),
    frames correlated like features; the target is the Gram of perturbed features (as get_intraframe_paras gives)."""
    flows, occs = O.synth_flows(N, H, W, seed=seed, mag=12.0)
    h, w = (H // 64, W // 64) if layer == 0 else (H // 32, W // 32)
    g = torch.Generator().manual_seed(seed + 50)
    base = torch.randn(2, 1, 1280, h, w, generator=g)
    cs = (base + 0.5 * torch.randn(2, N, 1280, h, w, generator=g)).contiguous()
    ref = (cs + 0.7 * torch.randn(cs.shape, generator=g)).reshape(2 * N, 1280, h, w)
    return flows, occs, cs, ref


@pytest.mark.gpu
@pytest.mark.parametrize("layer", [0, 1])
@pytest.mark.parametrize("hw", FAILING, ids=_setting_id)
def test_optimize_feature_teacher_forced(fb, monkeypatch, hw, layer):
    """One Adam iteration of optimize_feature within the bound composed from its kernels' bounds
    (oracle/optimize_bound.py), checked by a spy on ``ops`` on the state the GPU held: the temporal gradient, the
    Gram-L1 term's normalisation, sign matrix (exact outside the derived band) and gradient, Adam's p, m and v, the
    trace's loss and AdaIN."""
    H, W = hw
    N = 8
    flows, occs, cs, ref = _layer_case(N, H, W, layer, seed=H + W + layer)
    B, C, h, w = 2 * N, 1280, cs.shape[3], cs.shape[4]
    target = fb.dh.gram_targets([ref.half().cuda()])[0]
    sample = cs.reshape(B, C, h, w).cuda()
    fl, oc = [f.cuda() for f in flows], [o.cuda() for o in occs]
    g = OB.glue(sample, fl, oc, [target], 1e2, 2)
    spy = OB.OpsSpy(fb.ops, fb.lib.last_kernel, g, sample, torch.cuda.get_device_properties(0).multi_processor_count)
    spy.install(monkeypatch)
    tr = fb.dh.OptimizeTrace()
    out = fb.dh.optimize_feature(sample, fl, oc, correlation_matrix=[target], intra_weight=1e2, iters=1, trace=tr)
    assert out.shape == sample.shape and torch.isfinite(out).all()
    assert [t for t, _ in spy.saturated] == [1] and spy.adain_ratio is not None and tr.losses == spy.losses


@pytest.mark.gpu
@pytest.mark.parametrize("layer", [0, 1])
@pytest.mark.parametrize("hw", [(320, 448), (448, 768)], ids=_setting_id)
def test_optimize_feature_loss_curve(fb, hw, layer):
    """20 Adam iterations (temporal + Gram-L1): the loss curve within 1e-2 of the oracle's, AdaIN statistics pinned."""
    H, W = hw
    N = 8
    flows, occs, cs, ref = _layer_case(N, H, W, layer, seed=3 * H + W + layer)
    sample = cs.reshape(2 * N, 1280, cs.shape[3], cs.shape[4]).half()
    target = fb.dh.gram_targets([ref.half().cuda()])[0]
    tr = fb.dh.OptimizeTrace()
    fl, oc = [f.cuda() for f in flows], [o.cuda() for o in occs]
    out = fb.dh.optimize_feature(sample.cuda(), fl, oc, correlation_matrix=[target], intra_weight=1e2, iters=20, trace=tr)
    ref_out, ref_trace = O.optimize_feature(sample, flows, occs, correlation_matrix=[target.dense().cpu()],
                                            intra_weight=1e2, iters=20, return_trace=True)
    losses, ref_losses = np.array(tr.losses), np.array([t["loss"] for t in ref_trace])
    assert out.dtype == torch.float16 and torch.isfinite(out).all()
    assert losses[-1] < losses[0]
    assert np.allclose(losses, ref_losses, rtol=1e-2), (losses, ref_losses)
    m_out, m_ref = out.float().mean((2, 3)).cpu(), ref_out.float().mean((2, 3))
    assert (m_out - m_ref).abs().max().item() < 2e-2


# ------------------------------------------------------------------------------------------------ one denoise step
class _Sched:
    timesteps = torch.arange(950, -1, -50)

    def __init__(self):
        self.ac = torch.linspace(0.999, 0.01, 1000)

    def add_noise(self, x0, noise, t):
        a = self.ac[int(t)].item()
        return (math.sqrt(a) * x0.float() + math.sqrt(1 - a) * noise.float()).to(x0.dtype)


class _VAE:
    class config:
        scaling_factor = 0.18215

    class _Dist:
        def __init__(self, x):
            self.latent_dist = self
            self.x = x

        def sample(self):
            return torch.nn.functional.avg_pool2d(self.x, 8)[:, :1].repeat(1, 4, 1, 1)

    def encode(self, x):
        return self._Dist(x)


@pytest.mark.gpu
@pytest.mark.parametrize("hw", [(320, 320), (320, 448), (448, 768)], ids=_setting_id)
def test_harness_denoise_step(fb, hw):
    """One denoise step of the SD-1.5-shaped harness UNet with every FRESCO flag on: get_intraframe_paras targets,
    cross-frame, spatial- and temporal-guided attention, and apply_FRESCO_opt on all four decoder layers.  The output
    is finite and each FRESCO self-attention call is within the bound composed from its kernels' bounds
    (oracle/layer_bound.py), evaluated on the fp16 projections of the call's own hidden states (all frames' rows of
    512 sampled trajectories at the larger token counts), each stage's own bound on the operands its kernel received
    (recorded by a spy on ``ops``)."""
    from fresco_b200.harness import synth
    from fresco_b200.harness.sd15_unet import FakePipe, SD15UNet
    H, W = hw
    N, dev = 2, torch.device("cuda")
    dh, fu = fb.dh, fb.fu
    torch.manual_seed(0)
    pipe = FakePipe(SD15UNet().to(device=dev).eval())
    pipe.scheduler, pipe.vae, pipe._execution_device = _Sched(), _VAE(), dev
    pipe.prepare_latents = lambda B, C, h, w, dtype, device, generator, latents=None: torch.randn(
        B, C, h // 8, w // 8, generator=generator, dtype=dtype, device=device)
    proc = dh.apply_FRESCO_attn(pipe)
    imgs = synth.frames(N, H, W, dev, seed=H + W)
    pe = 0.5 * torch.randn(2 * N, 77, 768, device=dev)
    corr = dh.get_intraframe_paras(pipe, imgs, proc, pe, seed=3)
    assert [tuple(c.shape) for c in corr] == [(2 * N, t, t) for t in
                                              ((H // 64) * (W // 64), (H // 32) * (W // 32), (H // 16) * (W // 16),
                                               (H // 8) * (W // 8))]
    flows, occs = synth.smooth_flows(N, H, W, dev, seed=H * W)
    sal = torch.rand(N, 1, H, W, generator=torch.Generator().manual_seed(1)).to(dev)
    attn_mask = dh.cross_frame_attn_masks(occs[1])
    fm, bm, im = [], [], []
    for s in (8.0, 16.0):
        f, b, m = fu.get_mapping_ind(flows[1], occs[1], imgs, scale=s)
        fm.append(f), bm.append(b), im.append(m)
    paras = {"fwd_mappings": fm, "bwd_mappings": bm, "interattn_masks": im}
    t = 700
    dh.apply_FRESCO_opt(pipe, steps=[t], layers=[0, 1, 2, 3], flows=flows, occs=occs, correlation_matrix=corr,
                        intra_weight=1e2, iters=20, optimize_temporal=True, saliency=sal)
    proc.controller.enable_controller(interattn_paras=paras, attn_mask=attn_mask)
    calls, launches = [], []
    real = dh.FRESCOAttnProcessor2_0._fresco_self_attention
    real_ops = {name: getattr(fb.ops, name) for name in ("attn_fwd", "temporal_attn_fwd")}

    def spy(self, attn, query, key, value, hidden_states, heads, head_dim):
        ctrl = self.controller
        ref = ctrl.stored_attn["decoder_attn"][ctrl.index] if ctrl.use_intraattn else None
        start = len(launches)
        out = real(self, attn, query, key, value, hidden_states, heads, head_dim)
        calls.append((hidden_states.detach().clone(), ref.detach().clone(), attn, heads, out.float(), launches[start:]))
        return out

    def spy_op(name):
        def call(*a, **kw):
            launches.append((name, a))
            return real_ops[name](*a, **kw)
        return call

    lat = torch.randn(N, 4, H // 8, W // 8, generator=torch.Generator().manual_seed(2)).to(dev)
    dh.FRESCOAttnProcessor2_0._fresco_self_attention = spy
    for name in real_ops:
        setattr(fb.ops, name, spy_op(name))
    try:
        with torch.no_grad():
            out = pipe.unet(torch.cat([lat] * 2), t, encoder_hidden_states=pe, return_dict=False)[0]
        torch.cuda.synchronize()
    finally:
        dh.FRESCOAttnProcessor2_0._fresco_self_attention = real
        for name, fn in real_ops.items():
            setattr(fb.ops, name, fn)
    assert out.shape == (2 * N, 4, H // 8, W // 8) and torch.isfinite(out).all()
    assert len(calls) == 6, len(calls)
    for i, (x, ref, attn, heads, got, ops_calls) in enumerate(calls):
        B, L, C = x.shape
        d = C // heads
        rowsum = ",rowsum" in fb.lib.lib().fresco_attn_variant(d).decode()
        poly = int(re.search(r"poly(\d+)", fb.lib.lib().fresco_attn_variant(d).decode()).group(1))
        with torch.no_grad():
            ops = LB.Operands(attn.to_q(x).half(), attn.to_k(x).half(), attn.to_v(x).half(), attn.to_q(ref).half(),
                              attn.to_k(ref).half(), heads, 2)
        ctl = LB.Control(True, True, True, attn_mask, fm, bm, im)
        assert [n for n, _ in ops_calls] == ["attn_fwd", "attn_fwd", "temporal_attn_fwd"], ops_calls
        (_, spatial), (_, cross), (_, temporal) = ops_calls
        assert all(torch.equal(a, b) for a, b in zip(spatial[:3], (ops.q_ref, ops.k_ref, ops.q))), i
        assert torch.equal(temporal[0], ops.q) and torch.equal(temporal[1], ops.k), i
        received = {"cross_q": cross[0], "temporal_v": temporal[2]}
        sample = torch.randperm(L, generator=torch.Generator().manual_seed(i))[:512] if L >= 2304 else None
        lay = LB.evaluate(ops, ctl, sample, received, poly=poly, rowsum=rowsum, device=dev)
        want, tol = LB.attention_result(lay)
        rows = lay.rows.to(dev)[..., None].expand(-1, -1, C)
        r = LB.ratio(torch.gather(got, 1, rows), want, tol)
        assert not (r > 1).any(), (i, L, r.max().item())
