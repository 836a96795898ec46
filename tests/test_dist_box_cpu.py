"""Keyframe batches of any frame count on any number of ranks through ``dist.Box``: the layout ``dist.shard_layout``
picks for a Box (G <= 8, N <= 32), and gloo runs of every sharded call with the torch stand-ins of
test_dist_uneven_cpu.py at worlds 3, 5 and 7 (frame, unequal-halves and idle layouts) and 8.  Each active rank compares
its rows with the unsharded call on the whole batch; an idle rank must return empty results without touching its
process group or any collective."""
import copy
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
    """stands in for the Box's process group so the layout can be enumerated without creating groups"""

    def __init__(self, tag=()):
        self.tag = tag

    def __eq__(self, other):
        return isinstance(other, _NoGroups) and other.tag == self.tag

    def __hash__(self):
        return hash(self.tag)

    def half_comm(self, world, rank):
        return ("half", self.tag, 0 if rank < world - world // 2 else 1)

    def sub_comm(self, active, rank):
        return _NoGroups(("active", active))


def _rows(N, lay):
    """this rank's rows of a (chunk, frame)-major batch of both CFG chunks"""
    halves = range(*lay.halves)
    return torch.cat([torch.arange(h * N + lay.lo, h * N + lay.hi) for h in halves]).long()


# ------------------------------------------------------------------------------------------------ the layout
def test_box_layout_enumerated():
    from fresco_b200.dist import Box, frame_range, shard_layout
    for G in range(1, 9):
        for N in range(1, 33):
            lays = [shard_layout(N, Box(G, r, _NoGroups())) for r in range(G)]       # never raises
            idle = [r for r, lay in enumerate(lays) if lay.idle]
            assert len(idle) == max(0, G - 2 * N) and idle == list(range(G - len(idle), G))
            owned = {}
            for r, lay in enumerate(lays):
                for h in range(*lay.halves):
                    for f in range(lay.lo, lay.hi):
                        assert (h, f) not in owned
                        owned[(h, f)] = r
            assert sorted(owned) == [(h, f) for h in range(2) for f in range(N)]      # every row exactly once
            active = min(G, 2 * N)
            if N >= G or (G % 2 == 0 and 2 * N >= G) or G > 2 * N:
                # the frame and half layouts of the tuple (on the first 2N ranks when G > 2N)
                for r in range(active):
                    want = shard_layout(N, (active, r, _NoGroups(() if G <= 2 * N else ("active", active))))
                    got = lays[r]
                    assert (got.halves, got.lo, got.hi, got.world, got.rank, got.group, got.partner) == (
                        want.halves, want.lo, want.hi, want.world, want.rank, want.group, want.partner), (G, N, r)
                    assert got.peers == want.peers
                continue
            # G odd, N < G <= 2N: ceil(G/2) ranks on the unconditional half, floor(G/2) on the text half
            G0, G1 = G - G // 2, G // 2
            for r, lay in enumerate(lays):
                h, s, size = (0, r, G0) if r < G0 else (1, r - G0, G1)
                assert lay.halves == (h, h + 1) and (lay.world, lay.rank) == (size, s) and lay.partner is None
                assert (lay.lo, lay.hi) == frame_range(N, size, s) and lay.group == ("half", (), h)
                # the peers: the other half's ranks overlapping my frames, in frame order, covering them exactly
                assert lay.peers and lay.peers[0][1] == lay.lo and lay.peers[-1][2] == lay.hi
                assert all(a[2] == b[1] for a, b in zip(lay.peers, lay.peers[1:]))
                for p, a, b in lay.peers:
                    assert lays[p].half == 1 - h and (r, a, b) in lays[p].peers
    with pytest.raises(ValueError, match="both"):
        shard_layout(4, Box(7, 0, _NoGroups())).chunks(1)
    with pytest.raises(ValueError, match="G <= 2N"):                              # the tuple still raises
        shard_layout(4, (7, 0, _NoGroups()))


def test_box_unequal_halves_loss_scales_equal_unsharded():
    """The fp32 Gram scale of every rank of every unequal-halves layout (its share n / 2N of the weight, divided by its
    own batch of n samples in double, rounded once) is the unsharded one."""
    from fresco_b200.dist import frame_range
    from fresco_b200.ops import _gram_scale
    from test_dist_uneven_cpu import _level_tokens
    f32 = np.float32
    cases = 0
    for intra_weight in (1.0, 10.0, 50.0, 100.0, 200.0):
        for L in _level_tokens():
            for G in (3, 5, 7):
                for N in range((G + 1) // 2, G):
                    want = f32(float(f32(intra_weight)) / (2 * N * L * L))
                    for size in (G - G // 2, G // 2):
                        for r in range(size):
                            lo, hi = frame_range(N, size, r)
                            weight = intra_weight * (float(hi - lo) / float(2 * N))
                            assert f32(_gram_scale(weight, hi - lo, L)) == want, (intra_weight, L, N, G, r)
                            cases += 1
    assert cases > 0


def test_box_propagation_frames_held_by_ranks_of_the_first_batch():
    """In propagation mode the ranks holding frame 0 or 1 of a later batch restore them from the first batch's
    record_latents, which only the first batch's active ranks hold.  With a first batch of at least 3 frames (the web
    UI's smallest) on up to 8 ranks, every such rank was active in it."""
    from fresco_b200.dist import Box, shard_layout
    for G in range(1, 9):
        for N0 in range(3, 17):
            active = [not shard_layout(N0, Box(G, r, _NoGroups())).idle for r in range(G)]
            for N1 in range(3, 19):
                for r in range(G):
                    lay = shard_layout(N1, Box(G, r, _NoGroups()))
                    if not lay.idle and lay.lo < 2:
                        assert active[r], (G, N0, N1, r)


# ------------------------------------------------------------------------------------------------ gloo: every sharded call
def _attention(N, lay, box, rank):
    from fresco_b200 import diffusion_hacked as dh
    from fresco_b200.dist import ShardedFRESCOAttention
    from oracle import fresco_oracle as O
    from test_dist_cpu import TorchBackend
    torch.manual_seed(N)
    L, heads, C = 64, 2, 16
    x = torch.randn(2 * N, L, C)
    ref = torch.randn(2 * N, L, C)
    w = [torch.randn(C, C) * 0.3 for _ in range(4)]
    bo = torch.randn(C) * 0.1
    masks = [torch.rand(N, L) > 0.6]
    masks[0][0] = True
    masks[0][-1] = False
    perm = torch.stack([torch.randperm(L) for _ in range(N)])
    perm[0] = torch.arange(L)
    fm, bm = perm[:, None, :], torch.argsort(perm, dim=1)[:, None, :]
    im = (torch.rand(L, 1, N, N) > 0.3) | torch.eye(N, dtype=torch.bool)[None, None]
    sel = _rows(N, lay)
    xl, rl = x[sel], ref[sel]
    proj = lambda t, i: t @ w[i].t()
    # the layer the processor builds from the Box and the batch's frame count
    proc = dh.FRESCOAttnProcessor2_0(2, dh.AttentionControl(), shard=box)
    proc.set_batch_frames(N)
    chunks = proc._layout.chunks(2)
    bad = [] if (proc._layout.halves, proc._layout.lo, proc._layout.hi) == (lay.halves, lay.lo, lay.hi) else ["layout"]
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
            full = ShardedFRESCOAttention(ctrl, 1, 0, 2, backend=TorchBackend())(
                proj(x, 0), proj(x, 1), proj(x, 2), heads, ref_q=proj(ref, 0), ref_k=proj(ref, 1))
            mine = ShardedFRESCOAttention(ctrl, lay.world, lay.rank, chunks, lay.group, backend=TorchBackend())(
                proj(xl, 0), proj(xl, 1), proj(xl, 2), heads, ref_q=proj(rl, 0), ref_k=proj(rl, 1))
            if not torch.equal(mine, full[sel]):
                bad.append("attention flags %d no_mask %s" % (flags, no_mask))
            if not no_mask and (mine @ w[3].t() + bo - want[sel]).abs().max().item() >= 1e-4:
                bad.append("attention flags %d against the oracle" % flags)
    return bad


def _warp(N, lay, box, rank):
    from fresco_b200 import flow_utils as fu
    from oracle import fresco_oracle as O
    from test_cpu_host import _TorchWarpOps
    fu.ops = _TorchWarpOps
    flows, occs = O.synth_flows(N, 64, 64, seed=5 + N, mag=5.0)
    sal = torch.rand(N, 1, 32, 32, generator=torch.Generator().manual_seed(2))
    bad = []
    # decoder features of both CFG chunks at feature resolution (4 channels: re-shard by channel, 3: gather path), then
    # a decoded image batch at image resolution (one chunk: what background smoothing warps on the ranks of half 0)
    for chunks, C, h in ((2, 4, 8), (2, 3, 8), (1, 3, 64)):
        if chunks == 1 and lay.half != 0:
            continue
        feat = torch.randn(chunks * N, C, h, h, generator=torch.Generator().manual_seed(3 + h + C))
        sel = _rows(N, lay) if chunks == 2 else torch.arange(lay.lo, lay.hi)
        full = fu.warp_tensor(feat, flows, occs, sal, chunks)
        mine = fu.warp_tensor(feat[sel].contiguous(), flows, occs, sal, chunks, shard=box)
        if not torch.equal(mine, full[sel]):
            bad.append("warp_tensor chunks %d C %d h %d" % (chunks, C, h))
    return bad


def _optimize(N, lay, box, rank):
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
    sel = _rows(N, lay)
    counts = []

    class Recording(TorchOptBackend):
        def temporal(self, cs, prep, grad, loss_acc, halo_cs=None, halo_grad=None, total_frames=None):
            counts.append(cs.shape[0] * (total_frames if total_frames is not None else cs.shape[1]))
            if halo_cs is None and total_frames is not None and total_frames != cs.shape[1]:
                # a CFG half on one rank (the unequal layout's text half on 3 ranks): the closed ring of its frames,
                # averaged over the whole batch; the stand-in averages over its own frames, so rescale
                part = torch.zeros(1) if loss_acc is not None else None
                super().temporal(cs, prep, grad, part)
                grad.mul_(cs.shape[1] / total_frames)
                if loss_acc is not None:
                    loss_acc += part * (cs.shape[1] / total_frames)
                return
            super().temporal(cs, prep, grad, loss_acc, halo_cs, halo_grad, total_frames)
    be = Recording(O)
    bad = []
    for temporal, spatial in ((True, True), (True, False), (False, True)):
        corr, corr_l = ([target], [target[sel]]) if spatial else ([], [])
        tr_full, tr_mine = dh.OptimizeTrace(), dh.OptimizeTrace()
        full = dh.optimize_feature(feat, flows, occs, corr, iters=6, optimize_temporal=temporal, trace=tr_full, backend=be)
        mine = dh.optimize_feature(feat[sel].contiguous(), flows, occs, corr_l, iters=6, optimize_temporal=temporal,
                                   trace=tr_mine, shard=box, backend=be)
        # the stand-ins evaluate the open chain in another order than the ring: the tolerance of test_dist_uneven_cpu
        if (mine - full[sel]).abs().max().item() >= 1e-4:
            bad.append("optimize_feature temporal %s spatial %s" % (temporal, spatial))
        if len(tr_full.losses) != 6 or not all(abs(a - b) < 1e-4 * abs(a) for a, b in zip(tr_full.losses, tr_mine.losses)):
            bad.append("optimize_feature loss curve temporal %s spatial %s" % (temporal, spatial))
    # the temporal mean's element count is the unsharded call's 2N on every rank
    if not counts or set(counts) != {2 * N}:
        bad.append("temporal element counts %s, want %d" % (sorted(set(counts)), 2 * N))
    with pytest.raises(ValueError, match="flows"):                              # a Box takes N from the flows
        dh.optimize_feature(feat[sel].contiguous(), None, None, [target[sel]], iters=3, shard=box, backend=be)
    return bad


def _step(N, lay, box, rank):
    """pipe_FRESCO.step with guidance and background smoothing, given the Box (it has flows) and given the layout"""
    from fresco_b200 import flow_utils as fu
    from fresco_b200 import pipe_FRESCO as pf
    from fresco_b200.dist import shard_layout
    from oracle import fresco_oracle as O
    from test_cpu_host import _TorchStepOps, _TorchWarpOps
    from test_dist_batch_cpu import _StubVAE
    from test_dist_cpu import _StubPipe
    pf.ops = _TorchStepOps
    fu.ops = _TorchWarpOps
    ac = torch.from_numpy(np.load(os.path.join(ROOT, "tests", "golden", "ddpm_step.npz"))["alphas_cumprod"])
    pipe = _StubPipe(ac)
    pipe.vae = _StubVAE()
    g = torch.Generator().manual_seed(6)
    eps = torch.randn(2 * N, 4, 8, 8, generator=g)
    x = torch.randn(N, 4, 8, 8, generator=g)
    noise = torch.randn(N, 4, 8, 8, generator=g)
    flows, occs = O.synth_flows(N, 64, 64, seed=9, mag=6.0)
    sal = (torch.rand(N, 1, 64, 64, generator=g) > 0.4).float()
    lo, hi = lay.lo, lay.hi
    eps_mine = eps[_rows(N, lay)]
    bad = []
    for smooth in (False, True):
        kw = dict(flows=flows, occs=occs, saliency=sal) if smooth else {}
        full = pf.step(pipe, eps, 700, x, None, guidance_scale=7.5, noise=noise, **kw)
        for spec in ([box, shard_layout(N, box)] if smooth else [shard_layout(N, box)]):
            mine = pf.step(pipe, eps_mine, 700, x[lo:hi].contiguous(), None, guidance_scale=7.5,
                           noise=noise[lo:hi].contiguous(), shard=spec, **kw)
            if not all(torch.equal(a, b[lo:hi]) for a, b in zip(mine, full)):
                bad.append("step smoothing %s shard %r" % (smooth, type(spec).__name__))
    return bad


def _inference(N, lay, box, rank):
    from fresco_b200 import flow_utils as fu
    from fresco_b200 import pipe_FRESCO as pf
    from fresco_b200.dist import partner_swap
    from oracle import fresco_oracle as O
    from test_cpu_host import _TorchStepOps, _TorchWarpOps
    from test_dist_batch_cpu import _StubVAE
    from test_dist_cpu import _Ctrl, _StubPipe
    from test_dist_halves_cpu import _NoisyVAE
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
    rec_full, rec_sh = [], []
    for propagation in (False, True):
        kw = dict(num_warmup_steps=14, use_controlnet=False, seed=3, bg_smoothing_steps=[16, 17],
                  propagation_mode=propagation, flows=flows, occs=occs, saliency=sal)
        full = pf.inference(pipe(), None, _Ctrl, imgs, pe, None, timesteps, record_latents=rec_full, **kw)
        mine = pf.inference(pipe(), None, _Ctrl, imgs, pe, None, timesteps, record_latents=rec_sh, shard=box, **kw)
        if not (torch.equal(mine, full[lay.lo:lay.hi]) and len(rec_full) == len(rec_sh)
                and all(torch.equal(a, b) for a, b in zip(rec_full, rec_sh))):
            bad.append("inference propagation %s" % propagation)
    if lay.split_halves:
        # the two halves' ranks of the same frames agree although the VAE draws its posterior noise from an unseeded
        # generator: it is drawn on half 0 only
        torch.manual_seed(100 + rank)
        out = pf.inference(pipe(_NoisyVAE), None, _Ctrl, imgs, pe, None, timesteps, record_latents=[], shard=box,
                           num_warmup_steps=14, use_controlnet=False, seed=3, bg_smoothing_steps=[16, 17], flows=flows,
                           occs=occs, saliency=sal)
        if not torch.equal(partner_swap(lay, out), out):
            bad.append("the halves differ with a noisy VAE")
    return bad


def _flow(N, lay, box, rank):
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
    mine = dh.get_flow_and_interframe_paras(model, imgs, shard=box)
    bad = [] if _flow_paras_equal(mine, full) else ["get_flow_and_interframe_paras"]
    if calls != ([lay.hi - lay.lo] if lay.halves[0] == 0 else []):                   # every pair once, on half 0
        bad.append("flow model calls %s" % calls)
    return bad


def _intraframe(N, lay, box, rank):
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
    sel = _rows(N, lay)
    proc = dh.apply_FRESCO_attn(pipe)
    corr_full = dh.get_intraframe_paras(pipe, imgs, proc, pe, seed=3)
    in_full = seen[-1]
    proc = dh.apply_FRESCO_attn(pipe, shard=box)
    proc.set_batch_frames(N)
    proc._sharded = ShardedFRESCOAttention(proc.controller, lay.world, lay.rank, proc._layout.chunks(2), lay.group,
                                           backend=_StandInBackend())
    corr = dh.get_intraframe_paras(pipe, imgs, proc, pe, seed=3, shard=box)
    bad = []
    if not torch.equal(seen[-1], in_full[sel]):
        bad.append("get_intraframe_paras UNet input")
    if not (len(corr) == len(corr_full) == 4 and all(_close(a, b[sel]) for a, b in zip(corr, corr_full))):
        bad.append("get_intraframe_paras targets")
    return bad


# ------------------------------------------------------------------------------------------------ idle ranks, misuse
_COLLECTIVES = ("all_gather_into_tensor", "all_gather", "all_to_all_single", "all_reduce", "broadcast",
                "batch_isend_irecv", "isend", "irecv", "send", "recv", "barrier", "new_group", "split_group",
                "get_global_rank", "get_backend")


class _Untouchable:
    """an idle rank's process group: fails on any use"""

    def __getattr__(self, name):
        raise AssertionError("an idle rank used its process group (.%s)" % name)


class _NoCollectives:
    """replaces every collective and group call of torch.distributed by one that fails"""

    def __enter__(self):
        self.saved = {n: getattr(dist, n) for n in _COLLECTIVES}
        for n in _COLLECTIVES:
            setattr(dist, n, self._fail(n))
        return self

    @staticmethod
    def _fail(name):
        def f(*a, **k):
            raise AssertionError("torch.distributed.%s called" % name)
        return f

    def __exit__(self, *exc):
        for n, f in self.saved.items():
            setattr(dist, n, f)
        return False


def _idle(N, world, rank):
    """every entry point on an idle rank, its group and every collective failing on use"""
    from fresco_b200 import diffusion_hacked as dh
    from fresco_b200 import flow_utils as fu
    from fresco_b200 import pipe_FRESCO as pf
    from fresco_b200.dist import Box, shard_layout
    from oracle import fresco_oracle as O
    from test_cpu_host import _TorchStepOps, _TorchWarpOps
    from test_dist_batch_cpu import _frames, _StubFlow, _StubVAE
    from test_dist_cpu import _Ctrl, _StubPipe
    from fresco_b200.harness.sd15_unet import FakePipe, SD15UNet
    pf.ops = _TorchStepOps
    fu.ops = _TorchWarpOps
    box = Box(world, rank, _Untouchable())
    ac = torch.from_numpy(np.load(os.path.join(ROOT, "tests", "golden", "ddpm_step.npz"))["alphas_cumprod"])
    flows, occs = O.synth_flows(N, 64, 64, seed=9, mag=6.0)
    sal = torch.ones(N, 1, 64, 64)
    pe = torch.randn(2 * N, 5, 8)
    bad = []
    with _NoCollectives():
        lay = shard_layout(N, box)
        if not lay.idle:
            return ["rank %d not idle: %r" % (rank, lay)]
        fl, oc, masks, paras = dh.get_flow_and_interframe_paras(_StubFlow(), _frames(N, 64, 64, seed=4), shard=box)
        if fl[0].shape[0] or oc[0].shape[0] or masks or paras["fwd_mappings"]:
            bad.append("get_flow_and_interframe_paras returned frames")
        unet_pipe = FakePipe(SD15UNet(block_out=(32, 64, 128, 128), heads=8, cross_dim=24))
        unet_pipe.vae, unet_pipe._execution_device = _StubVAE(), torch.device("cpu")
        proc = dh.apply_FRESCO_attn(unet_pipe, shard=box)
        if dh.get_intraframe_paras(unet_pipe, torch.rand(N, 3, 64, 64), proc, pe, shard=box) != []:
            bad.append("get_intraframe_paras returned targets")
        dh.apply_FRESCO_opt(unet_pipe, steps=[700], flows=flows, occs=occs, saliency=sal, shard=box)
        none = torch.empty(0, 6, 8, 8)
        if dh.optimize_feature(none, flows, occs, [], shard=box) is not none:
            bad.append("optimize_feature")
        if fu.warp_tensor(none, flows, occs, sal, 2, shard=box) is not none:
            bad.append("warp_tensor")
        pipe = _StubPipe(ac)
        pipe.vae = _StubVAE()
        x = torch.empty(0, 4, 8, 8)
        if pf.step(pipe, x, 700, x, None, guidance_scale=7.5, flows=flows, occs=occs, saliency=sal, shard=box)[0] is not x:
            bad.append("step")
        rec = []
        out = pf.inference(pipe, None, _Ctrl, torch.rand(N, 3, 64, 64), pe, None, [950 - 50 * i for i in range(20)],
                           num_warmup_steps=14, use_controlnet=False, record_latents=rec, flows=flows, occs=occs,
                           saliency=sal, shard=box)
        if tuple(out.shape) != (0, 4, 8, 8) or rec:
            bad.append("inference returned %s" % (tuple(out.shape),))
    return bad


def _misuse(N, lay, box, rank):
    """a batch without classifier-free guidance cannot shard over its halves: ValueError on every rank, before any
    collective (the groups exist already: they were created by the calls above)"""
    from fresco_b200 import diffusion_hacked as dh
    from fresco_b200 import pipe_FRESCO as pf
    from oracle import fresco_oracle as O
    from test_dist_cpu import TorchOptBackend, _Ctrl, _StubPipe
    from test_dist_batch_cpu import _StubVAE
    ac = torch.from_numpy(np.load(os.path.join(ROOT, "tests", "golden", "ddpm_step.npz"))["alphas_cumprod"])
    pipe = _StubPipe(ac)
    pipe.vae = _StubVAE()
    flows, occs = O.synth_flows(N, 64, 64, seed=9, mag=6.0)
    n = lay.hi - lay.lo
    calls = {
        "inference": lambda: pf.inference(pipe, None, _Ctrl, torch.rand(N, 3, 64, 64), torch.randn(N, 5, 8), None,
                                          [950 - 50 * i for i in range(20)], num_warmup_steps=14, use_controlnet=False,
                                          do_classifier_free_guidance=False, record_latents=[], shard=box),
        "step": lambda: pf.step(pipe, torch.randn(n, 4, 8, 8), 700, torch.randn(n, 4, 8, 8), None, shard=lay),
        "optimize_feature": lambda: dh.optimize_feature(torch.randn(n, 6, 8, 8), flows, occs, [], iters=2,
                                                        unet_chunk_size=1, shard=box, backend=TorchOptBackend(O)),
    }
    bad = []
    with _NoCollectives():
        for name, call in calls.items():
            try:
                call()
                bad.append("%s without guidance did not raise" % name)
            except ValueError:
                pass
    return bad


def _box_worker(rank, world, port, ret, N, parts):
    _init(rank, world, port)
    from fresco_b200.dist import Box, shard_layout
    idle = rank >= 2 * N
    bad = []
    if idle:
        bad += _idle(N, world, rank)
    else:
        box = Box(world, rank)
        lay = shard_layout(N, box)
        for part in parts:
            bad += globals()[part](N, lay, box, rank)
    for b in bad:
        print("rank %d of %d, N %d: %s" % (rank, world, N, b), flush=True)
    _finish(rank, not bad, ret)


_ALL = ("_attention", "_warp", "_optimize", "_step", "_inference", "_flow")


@pytest.mark.parametrize("N,world", [(2, 3), (3, 3), (4, 3), (6, 3), (2, 5), (3, 5), (4, 5), (6, 5),
                                     (2, 7), (3, 7), (4, 7), (6, 7), (3, 8)])
def test_box_matches_unsharded_gloo(N, world):
    """Every sharded call under a Box against the unsharded call on the whole batch, each active rank on its rows, bit
    for bit (optimize_feature to the stand-ins' tolerance, as in test_dist_halves_cpu): the processor's layer at all 8
    flag combinations and the no-mask frame-0 broadcast, warp_tensor (channel re-shard, gather path, image resolution),
    optimize_feature with both losses, step with guidance and smoothing, inference in normal and propagation mode with
    record_latents, and the flow parameters.  Worlds 3, 5, 7 cover the frame, unequal-halves and idle layouts; at
    (2, 5), (2, 7), (3, 7) and (3, 8) the ranks beyond 2N are idle and must not touch a group or collective."""
    _run(_box_worker, world, N, _ALL, timeout=900)


@pytest.mark.parametrize("N,world", [(2, 3), (3, 7)])
def test_box_intraframe_paras_gloo(N, world):
    """get_intraframe_paras under a Box: the UNet input is this rank's rows of the unsharded call's, the targets equal
    its slices to the CPU UNet's batch-size round-off (test_dist_batch_cpu); idle ranks return none"""
    _run(_box_worker, world, N, ("_intraframe",), timeout=600)


@pytest.mark.parametrize("N,world", [(2, 3), (4, 7)])
def test_box_without_guidance_raises_on_every_rank_gloo(N, world):
    """A Box in the unequal-halves layout on a batch without classifier-free guidance raises ValueError on every rank
    before any collective, so no rank waits for another"""
    _run(_box_worker, world, N, ("_flow", "_misuse"), timeout=300)
