"""Keyframe batches with fewer frames than ranks, sharded over the two CFG halves as well as the frames
(``dist.shard_layout``): the layout for G <= 8 and N <= 32, the loss scales of the half layout, and gloo runs of every
sharded call with the torch stand-ins of test_dist_uneven_cpu.py.  Each rank compares its rows -- one CFG half of its
frames -- with the unsharded call on the whole batch."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from test_dist_batch_cpu import _finish, _init, _run  # noqa: E402


class _NoGroups:
    """stands in for the shard's process group so the layout can be enumerated without creating groups"""

    def half_comm(self, world, rank):
        return ("half", rank // (world // 2))


def _half_rows(N, layout):
    base = layout.half * N
    return torch.arange(base + layout.lo, base + layout.hi)


# ------------------------------------------------------------------------------------------------ the layout
def test_shard_layout_enumerated():
    from fresco_b200.dist import frame_range, shard_layout
    for G in range(1, 9):
        for N in range(1, 33):
            if N >= G:
                for r in range(G):
                    lay = shard_layout(N, (G, r, None))
                    assert (lay.lo, lay.hi) == frame_range(N, G, r) and lay.halves == (0, 2)
                    assert (lay.world, lay.rank, lay.group, lay.partner) == (G, r, None, None)
                continue
            if G % 2 or 2 * N < G:
                with pytest.raises(ValueError, match="G <= 2N") as e:
                    shard_layout(N, (G, 0, _NoGroups()))
                assert "process group of %d ranks" % N in str(e.value)
                continue
            owned = {}
            lays = [shard_layout(N, (G, r, _NoGroups())) for r in range(G)]
            for r, lay in enumerate(lays):
                assert lay.split_halves and lay.halves == (r // (G // 2), r // (G // 2) + 1)
                assert (lay.world, lay.rank) == (G // 2, r % (G // 2))
                assert (lay.lo, lay.hi) == frame_range(N, G // 2, r % (G // 2))
                assert lay.group == ("half", lay.half)
                partner = lays[lay.partner]
                assert partner.partner == r and partner.half == 1 - lay.half
                assert (partner.lo, partner.hi) == (lay.lo, lay.hi)                     # partners hold the same frames
                for f in range(lay.lo, lay.hi):
                    assert (lay.half, f) not in owned
                    owned[(lay.half, f)] = r
            assert sorted(owned) == [(h, f) for h in range(2) for f in range(N)]          # every sample exactly once
    with pytest.raises(ValueError, match="both"):
        shard_layout(3, (4, 0, _NoGroups())).chunks(1)


def test_half_layout_loss_scales_equal_unsharded():
    """In every half layout the fp32 Gram scale of a rank (its share n / 2N of the weight, divided by its own batch of
    n samples in double, rounded once) is the unsharded one.  (The temporal mean's element count is checked on what
    optimize_feature passes, in the gloo runs.)"""
    from fresco_b200.dist import frame_range
    from fresco_b200.ops import _gram_scale
    from test_dist_uneven_cpu import _level_tokens
    f32 = np.float32
    cases = 0
    for intra_weight in (1.0, 10.0, 50.0, 100.0, 200.0):
        for L in _level_tokens():
            for G in (2, 4, 6, 8):
                for N in range(G // 2, G):
                    want = f32(float(f32(intra_weight)) / (2 * N * L * L))
                    for r in range(G // 2):
                        lo, hi = frame_range(N, G // 2, r)
                        n = hi - lo
                        weight = intra_weight * (float(n) / float(2 * N))         # optimize_feature's share
                        assert f32(_gram_scale(weight, n, L)) == want, (intra_weight, L, N, G, r)
                        cases += 1
    assert cases > 0


# ------------------------------------------------------------------------------------------------ gloo: every sharded call
def _attention(N, lay, rank):
    from fresco_b200 import diffusion_hacked as dh
    from fresco_b200.dist import ShardedFRESCOAttention
    from oracle import fresco_oracle as O
    from test_dist_cpu import TorchBackend
    torch.manual_seed(N)
    chunks, L, heads, C = 2, 64, 2, 16
    x = torch.randn(chunks * N, L, C)
    ref = torch.randn(chunks * N, L, C)
    w = [torch.randn(C, C) * 0.3 for _ in range(4)]
    bo = torch.randn(C) * 0.1
    masks = [torch.rand(N, L) > 0.6]
    masks[0][0] = True
    masks[0][-1] = False
    perm = torch.stack([torch.randperm(L) for _ in range(N)])
    perm[0] = torch.arange(L)
    fm, bm = perm[:, None, :], torch.argsort(perm, dim=1)[:, None, :]
    im = (torch.rand(L, 1, N, N) > 0.3) | torch.eye(N, dtype=torch.bool)[None, None]
    sel = _half_rows(N, lay)
    xl, rl = x[sel], ref[sel]
    proj = lambda t, i: t @ w[i].t()
    bad = []
    for flags in range(8):
        cf, intra, inter = bool(flags & 1), bool(flags & 2), bool(flags & 4)
        want = O.fresco_attention(x, w[0], w[1], w[2], w[3], bo, heads, use_cfattn=cf, attn_masks=masks,
                                  use_intraattn=intra, ref_hidden=ref, use_interattn=inter, fwd_mappings=[fm],
                                  bwd_mappings=[bm], interattn_masks=[im])
        for no_mask in (False, True):
            if no_mask and not cf:
                continue
            ctrl = dh.AttentionControl()
            if intra:
                ctrl.stored_attn["decoder_attn"] = [ref]
                ctrl.enable_intraattn()
            if inter:
                ctrl.enable_interattn({"fwd_mappings": [fm], "bwd_mappings": [bm], "interattn_masks": [im]})
            if cf:
                ctrl.enable_cfattn(masks)
                if no_mask:
                    ctrl.attn_mask = [torch.ones(N, 16, dtype=torch.bool)]     # no mask at 64 tokens: frame 0 only
            full = ShardedFRESCOAttention(ctrl, 1, 0, chunks, backend=TorchBackend())(
                proj(x, 0), proj(x, 1), proj(x, 2), heads, ref_q=proj(ref, 0), ref_k=proj(ref, 1))
            mine = ShardedFRESCOAttention(ctrl, lay.world, lay.rank, 1, lay.group, backend=TorchBackend())(
                proj(xl, 0), proj(xl, 1), proj(xl, 2), heads, ref_q=proj(rl, 0), ref_k=proj(rl, 1))
            if not torch.equal(mine, full[sel]):
                bad.append("attention flags %d no_mask %s" % (flags, no_mask))
            if not no_mask and (mine @ w[3].t() + bo - want[sel]).abs().max().item() >= 1e-4:
                bad.append("attention flags %d against the oracle" % flags)
    # the processor takes the same layout from the batch frame count
    proc = dh.FRESCOAttnProcessor2_0(2, dh.AttentionControl(), shard=lay.shard)
    proc.set_batch_frames(N)
    assert proc._layout.split_halves and proc._layout.half == lay.half
    return bad


def _warp(N, lay, rank):
    from fresco_b200 import flow_utils as fu
    from oracle import fresco_oracle as O
    from test_cpu_host import _TorchWarpOps
    fu.ops = _TorchWarpOps
    flows, occs = O.synth_flows(N, 64, 64, seed=5 + N, mag=5.0)
    sal = torch.rand(N, 1, 32, 32, generator=torch.Generator().manual_seed(2))
    bad = []
    # decoder features of both CFG chunks (4 channels: re-shard by channel; 3: gather path), then a decoded image batch
    for chunks, C, h in ((2, 4, 8), (2, 3, 8), (1, 3, 64)):
        feat = torch.randn(chunks * N, C, h, h, generator=torch.Generator().manual_seed(3 + h + C))
        sel = _half_rows(N, lay) if chunks == 2 else torch.arange(lay.lo, lay.hi)
        full = fu.warp_tensor(feat, flows, occs, sal, chunks)
        mine = fu.warp_tensor(feat[sel].contiguous(), flows, occs, sal, chunks, shard=lay.shard)
        if not torch.equal(mine, full[sel]):
            bad.append("warp_tensor chunks %d C %d h %d" % (chunks, C, h))
    return bad


def _optimize(N, lay, rank):
    from fresco_b200 import diffusion_hacked as dh
    from oracle import fresco_oracle as O
    from test_dist_cpu import TorchOptBackend
    chunks, C, h = 2, 6, 8
    flows, occs = O.synth_flows(N, 64, 64, seed=11, mag=5.0)
    g = torch.Generator().manual_seed(4)
    base = torch.randn(chunks, 1, C, h, h, generator=g)
    feat = (base + 0.5 * torch.randn(chunks, N, C, h, h, generator=g)).reshape(chunks * N, C, h, h)
    ref = feat + 0.3 * torch.randn(feat.shape, generator=g)
    X = ref.reshape(chunks * N, C, h * h).transpose(1, 2)
    Xh = X / (X ** 2).sum(2, keepdim=True) ** 0.5
    target = torch.bmm(Xh, Xh.transpose(1, 2))
    sel = _half_rows(N, lay)
    counts = []

    class Recording(TorchOptBackend):
        def temporal(self, cs, prep, grad, loss_acc, halo_cs=None, halo_grad=None, total_frames=None):
            counts.append(cs.shape[0] * (total_frames if total_frames is not None else cs.shape[1]))
            super().temporal(cs, prep, grad, loss_acc, halo_cs, halo_grad, total_frames)
    be = Recording(O)
    bad = []
    for temporal, spatial in ((True, True), (True, False), (False, True)):
        if temporal and N < 2:
            continue
        corr, corr_l = ([target], [target[sel]]) if spatial else ([], [])
        tr_full, tr_mine = dh.OptimizeTrace(), dh.OptimizeTrace()
        full = dh.optimize_feature(feat, flows, occs, corr, iters=6, optimize_temporal=temporal, trace=tr_full, backend=be)
        mine = dh.optimize_feature(feat[sel].contiguous(), flows, occs, corr_l, iters=6, optimize_temporal=temporal,
                                   trace=tr_mine, shard=lay.shard, backend=be)
        # the stand-ins evaluate the open chain in another order than the ring: the tolerance of test_dist_uneven_cpu
        if (mine - full[sel]).abs().max().item() >= 1e-4:
            bad.append("optimize_feature temporal %s spatial %s" % (temporal, spatial))
        if len(tr_full.losses) != 6 or not all(abs(a - b) < 1e-4 * abs(a) for a, b in zip(tr_full.losses, tr_mine.losses)):
            bad.append("optimize_feature loss curve temporal %s spatial %s" % (temporal, spatial))
    # the temporal mean's element count, chunks * total_frames (times C*h*w), is the unsharded call's 2N on every rank
    if not counts or set(counts) != {2 * N}:
        bad.append("temporal element counts %s, want %d" % (sorted(set(counts)), 2 * N))
    full = dh.optimize_feature(feat, None, None, [target], iters=3, backend=be)
    mine = dh.optimize_feature(feat[sel].contiguous(), None, None, [target[sel]], iters=3, shard=lay.shard, backend=be)
    if (mine - full[sel]).abs().max().item() >= 1e-4:
        bad.append("optimize_feature without flows")
    return bad


class _NoisyVAE:
    """the per-frame stub VAE of test_dist_batch_cpu whose posterior sample adds noise from the process's global
    generator, as a diffusers VAE does (and the reference leaves unseeded)"""

    def __init__(self):
        from test_dist_batch_cpu import _StubVAE
        self.inner = _StubVAE()
        self.config = self.inner.config

    def encode(self, x):
        d = self.inner.encode(x)
        v = d.v + 0.1 * torch.randn(d.v.shape)
        d.v = v
        return d

    def decode(self, z):
        return self.inner.decode(z)


def _inference(N, lay, rank):
    from fresco_b200 import flow_utils as fu
    from fresco_b200 import pipe_FRESCO as pf
    from oracle import fresco_oracle as O
    from test_cpu_host import _TorchStepOps, _TorchWarpOps
    from test_dist_batch_cpu import _StubVAE
    from test_dist_cpu import _Ctrl, _StubPipe
    pf.ops = _TorchStepOps
    fu.ops = _TorchWarpOps
    ac = torch.from_numpy(np.load(os.path.join(ROOT, "tests", "golden", "ddpm_step.npz"))["alphas_cumprod"])
    g = torch.Generator().manual_seed(1)
    imgs = torch.rand(N, 3, 64, 64, generator=g)
    pe = torch.randn(2 * N, 5, 8, generator=g)
    flows, occs = O.synth_flows(N, 64, 64, seed=9, mag=6.0)
    sal = (torch.rand(N, 1, 64, 64, generator=g) > 0.4).float()
    timesteps = [950 - 50 * i for i in range(20)]

    def pipe(vae=_StubVAE):
        p = _StubPipe(ac)
        p.vae = vae()
        return p
    bad = []
    for repeat in (False, True):
        rec_full, rec_sh = [], []
        for propagation in (False, True):
            kw = dict(num_warmup_steps=14, use_controlnet=False, seed=3, repeat_noise=repeat, bg_smoothing_steps=[16, 17],
                      propagation_mode=propagation, flows=flows, occs=occs, saliency=sal)
            full = pf.inference(pipe(), None, _Ctrl, imgs, pe, None, timesteps, record_latents=rec_full, **kw)
            mine = pf.inference(pipe(), None, _Ctrl, imgs, pe, None, timesteps, record_latents=rec_sh, shard=lay.shard,
                                **kw)
            if not (torch.equal(mine, full[lay.lo:lay.hi]) and len(rec_full) == len(rec_sh)
                    and all(torch.equal(a, b) for a, b in zip(rec_full, rec_sh))):
                bad.append("inference repeat %s propagation %s" % (repeat, propagation))
    # partners hold the same latents although the VAE draws its posterior noise from an unseeded generator; a mutant in
    # which the upper partner draws its own sample breaks that
    kw = dict(num_warmup_steps=14, use_controlnet=False, seed=3, bg_smoothing_steps=[16, 17], flows=flows, occs=occs,
              saliency=sal)
    torch.manual_seed(100 + rank)
    if not _partners_agree(lay, pf.inference(pipe(_NoisyVAE), None, _Ctrl, imgs, pe, None, timesteps, record_latents=[],
                                             shard=lay.shard, **kw)):
        bad.append("partners differ with a noisy VAE")
    real = pf.partner_share
    pf.partner_share = lambda layout, make, like: make()
    try:
        if _partners_agree(lay, pf.inference(pipe(_NoisyVAE), None, _Ctrl, imgs, pe, None, timesteps, record_latents=[],
                                             shard=lay.shard, **kw)):
            bad.append("a VAE sample drawn on both partners went unnoticed")
    finally:
        pf.partner_share = real
    return bad


def _partners_agree(lay, latents):
    """True iff this rank and its partner ended with the same latents"""
    mine = latents.contiguous()
    theirs = torch.empty_like(mine)
    for r in dist.batch_isend_irecv([dist.P2POp(dist.isend, mine, lay.partner), dist.P2POp(dist.irecv, theirs, lay.partner)]):
        r.wait()
    return torch.equal(mine, theirs)


def _flow(N, lay, rank):
    from fresco_b200 import diffusion_hacked as dh
    from fresco_b200 import flow_utils as fu
    from test_cpu_host import _TorchWarpOps
    from test_dist_batch_cpu import _flow_paras_equal, _frames, _StubFlow
    fu.ops = _TorchWarpOps
    imgs = _frames(N, 64, 64, seed=4)
    model = _StubFlow()
    calls = []
    model.register_forward_pre_hook(lambda m, a: calls.append(a[0].shape[0]))
    full = dh.get_flow_and_interframe_paras(model, imgs)
    calls.clear()
    mine = dh.get_flow_and_interframe_paras(model, imgs, shard=lay.shard)
    bad = [] if _flow_paras_equal(mine, full) else ["get_flow_and_interframe_paras"]
    if calls != ([lay.hi - lay.lo] if lay.half == 0 else []):                       # every pair once, on half 0
        bad.append("flow model calls %s" % calls)
    return bad


def _intraframe(N, lay, rank):
    from fresco_b200 import diffusion_hacked as dh
    from fresco_b200.dist import ShardedFRESCOAttention
    from fresco_b200.harness.sd15_unet import FakePipe, SD15UNet
    from test_cpu_host import _Sched, _TorchOps
    from test_dist_batch_cpu import _close, _StandInBackend, _StubVAE
    dh.ops = _TorchOps
    torch.manual_seed(1)
    unet = SD15UNet(block_out=(32, 64, 128, 128), heads=8, cross_dim=24)
    pipe = FakePipe(unet)

    class Sched(_Sched):
        timesteps = torch.arange(950, -1, -50)

    pipe.scheduler, pipe.vae, pipe._execution_device = Sched(torch.linspace(0.999, 0.01, 1000)), _StubVAE(), torch.device("cpu")
    pipe.prepare_latents = lambda B, C, H, W, dtype, device, generator, latents=None: torch.randn(
        B, C, H // 8, W // 8, generator=generator, dtype=dtype)
    seen = []
    unet.register_forward_pre_hook(lambda m, a: seen.append(a[0].clone()))
    g = torch.Generator().manual_seed(5)
    imgs = torch.rand(N, 3, 128, 128, generator=g) * 2 - 1
    pe = torch.randn(2 * N, 7, 24, generator=g)
    sel = _half_rows(N, lay)
    proc = dh.apply_FRESCO_attn(pipe)
    corr_full = dh.get_intraframe_paras(pipe, imgs, proc, pe, seed=3)
    in_full = seen[-1]
    proc = dh.apply_FRESCO_attn(pipe, shard=lay.shard)
    proc.set_batch_frames(N)
    proc._sharded = ShardedFRESCOAttention(proc.controller, lay.world, lay.rank, 1, lay.group, backend=_StandInBackend())
    corr = dh.get_intraframe_paras(pipe, imgs, proc, pe, seed=3, shard=lay.shard)
    bad = []
    if not torch.equal(seen[-1], in_full[sel]):                                          # this half's rows only
        bad.append("get_intraframe_paras UNet input")
    if not (len(corr) == len(corr_full) == 4 and all(_close(a, b[sel]) for a, b in zip(corr, corr_full))):
        bad.append("get_intraframe_paras targets")
    return bad


def _halves_worker(rank, world, port, ret, N, parts):
    _init(rank, world, port)
    from fresco_b200.dist import shard_layout
    lay = shard_layout(N, (world, rank, None))
    assert lay.split_halves
    bad = []
    for part in parts:
        bad += globals()[part](N, lay, rank)
    for b in bad:
        print("rank %d of %d, N %d: %s" % (rank, world, N, b), flush=True)
    _finish(rank, not bad, ret)


def _subgroup_worker(rank, world, port, ret, N, G, parts):
    """a shard on the process group of ranks 1..G of the world; ranks 0 and G+1.. take no part after creating it"""
    _init(rank, world, port)
    from fresco_b200 import dist as fd
    members = list(range(1, G + 1))
    bad = []
    for attempt in range(2):                     # the second shard group object over the same ranks finds the cache
        group = dist.new_group(members)
        if rank in members:
            lay = fd.shard_layout(N, (G, rank - 1, group))
            if not lay.split_halves or lay.partner != 1 + (lay.rank + (1 - lay.half) * (G // 2)):
                bad.append("layout %r" % lay)
            for part in parts if attempt == 0 else ("_attention",):
                bad += globals()[part](N, lay, rank)
    if rank in members and len(fd._HALF_GROUPS) != 1:
        bad.append("%d half groups cached" % len(fd._HALF_GROUPS))
    for b in bad:
        print("rank %d of %d, N %d on a sub-group of %d: %s" % (rank, world, N, G, b), flush=True)
    _finish(rank, not bad, ret)


_ALL = ("_attention", "_warp", "_optimize", "_inference", "_flow", "_intraframe")


@pytest.mark.parametrize("N,world,parts", [
    (3, 4, _ALL),
    (5, 8, ("_attention", "_warp", "_optimize", "_inference", "_flow")),
    (2, 4, ("_attention", "_warp", "_optimize")),
    (7, 8, ("_attention", "_warp")),
    (3, 6, ("_attention", "_flow")),
])
def test_half_layout_matches_unsharded_gloo(N, world, parts):
    """Every sharded call in the half layout against the unsharded call on the whole batch, each rank on its rows:
    attention (8 flag combinations, and the no-mask frame-0 broadcast within a half), warp_tensor (channel re-shard,
    gather path, image resolution), optimize_feature (output and loss curve, with and without flows), inference with
    background smoothing, propagation_mode and repeat_noise (bit for bit, record_latents included; partners agree under
    a VAE with unseeded posterior noise, and a mutant drawing it on both partners is caught), the flow parameters
    (every pair computed once, on half 0) and the intra-frame parameters (this half's rows)."""
    _run(_halves_worker, world, N, parts, timeout=600)


def test_half_layout_on_a_shard_subgroup_gloo():
    """The half layout of a shard on a process sub-group (ranks 1..4 of 6): the half groups are created by the shard's
    ranks alone (ranks 0 and 5 never reach that point), the exchanges and partner transfers address global ranks
    through the group, and a second group object over the same ranks reuses the cached half groups."""
    _run(_subgroup_worker, 6, 3, 4, ("_attention", "_optimize", "_inference"), timeout=600)
