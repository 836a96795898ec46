"""Frame-sharded batches whose frame count G does not divide: the partition ``dist.frame_range``, the fp32 loss scale of
the Gram kernels on every rank, and gloo runs of every sharded call at uneven (N, G) with the torch stand-ins of
test_dist_cpu.py / test_cpu_host.py / test_dist_batch_cpu.py.  Each rank compares its share with the unsharded call on
the whole batch."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from test_dist_batch_cpu import _finish, _init, _rows, _run  # noqa: E402


# ------------------------------------------------------------------------------------------------ the partition
def test_frame_range_partition():
    from fresco_b200.dist import block_sizes, frame_range
    for G in range(1, 9):
        for N in range(1, 33):
            if N < G:
                with pytest.raises(ValueError, match="process group of %d ranks" % N):
                    frame_range(N, G, 0)
                continue
            ranges = [frame_range(N, G, r) for r in range(G)]
            assert ranges[0][0] == 0 and ranges[-1][1] == N
            assert all(ranges[r][1] == ranges[r + 1][0] for r in range(G - 1))          # contiguous, in rank order
            shares = [hi - lo for lo, hi in ranges]
            assert min(shares) >= 1 and max(shares) - min(shares) <= 1
            assert block_sizes(N, G) == shares
            if N % G == 0:
                per = N // G
                assert ranges == [(r * per, (r + 1) * per) for r in range(G)]               # the even split as before


# ------------------------------------------------------------------------------------------------ Gram loss scale
def _level_tokens():
    """L of the four SD decoder levels (latent / 8, / 4, / 2, / 1) for square frames 256..1024 in steps of 64 and for
    640 x 512"""
    sizes = [(r, r) for r in range(256, 1025, 64)] + [(640, 512)]
    return [(w // 8 // f) * (h // 8 // f) for w, h in sizes for f in (8, 4, 2, 1)]


def test_sharded_gram_loss_scale_equals_unsharded():
    """Every rank's fp32 Gram loss scale equals the unsharded one: the unsharded launcher rounds
    fp32(intra_weight) / (2N L^2) once; a rank passes its share of the weight, intra_weight * n / N (optimize_feature),
    and ops divides it by its own batch 2n L^2 in double before the one rounding.  Rounding the share to fp32 first (the
    weight entry points) gives a different scale in some of these cases."""
    from fresco_b200.dist import frame_range
    from fresco_b200.ops import _gram_scale
    f32 = np.float32
    cases = rounded_share_differs = 0
    for intra_weight in (1.0, 10.0, 50.0, 100.0, 200.0):
        for L in _level_tokens():
            for N in range(1, 33):
                want = f32(float(f32(intra_weight)) / (2 * N * L * L))
                for G in range(1, min(N, 8) + 1):
                    for rank in range(G):
                        lo, hi = frame_range(N, G, rank)
                        n = hi - lo
                        weight = intra_weight * (float(n) / float(N))            # optimize_feature's share
                        got = f32(_gram_scale(weight, 2 * n, L))
                        assert got == want, (intra_weight, L, N, G, rank, got, want)
                        rounded_share_differs += f32(float(f32(weight)) / (2 * n * L * L)) != want
                        cases += 1
    assert cases == 5 * len(_level_tokens()) * sum(G * (33 - G) for G in range(1, 9))
    assert rounded_share_differs > 0


# ------------------------------------------------------------------------------------------------ attention
def _attention_worker(rank, world, port, ret, N):
    _init(rank, world, port)
    from fresco_b200 import diffusion_hacked as dh
    from fresco_b200.dist import ShardedFRESCOAttention, frame_range
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
    masks[0][-1] = False                                  # a rank may select no row of its own frames
    perm = torch.stack([torch.randperm(L) for _ in range(N)])
    perm[0] = torch.arange(L)
    fm, bm = perm[:, None, :], torch.argsort(perm, dim=1)[:, None, :]
    im = (torch.rand(L, 1, N, N) > 0.3) | torch.eye(N, dtype=torch.bool)[None, None]
    lo, hi = frame_range(N, world, rank)
    sel = _rows(N, lo, hi, chunks)
    xl, rl = x[sel], ref[sel]
    proj = lambda t, i: t @ w[i].t()
    ok = True
    for flags in range(8):
        cf, intra, inter = bool(flags & 1), bool(flags & 2), bool(flags & 4)
        want = O.fresco_attention(x, w[0], w[1], w[2], w[3], bo, heads, use_cfattn=cf, attn_masks=masks,
                                  use_intraattn=intra, ref_hidden=ref, use_interattn=inter, fwd_mappings=[fm],
                                  bwd_mappings=[bm], interattn_masks=[im])
        ctrl = dh.AttentionControl()
        if intra:
            ctrl.stored_attn["decoder_attn"] = [ref]
            ctrl.enable_intraattn()
        if inter:
            ctrl.enable_interattn({"fwd_mappings": [fm], "bwd_mappings": [bm], "interattn_masks": [im]})
        if cf:
            ctrl.enable_cfattn(masks)
        full = ShardedFRESCOAttention(ctrl, 1, 0, chunks, backend=TorchBackend())(
            proj(x, 0), proj(x, 1), proj(x, 2), heads, ref_q=proj(ref, 0), ref_k=proj(ref, 1))
        mine = ShardedFRESCOAttention(ctrl, world, rank, chunks, backend=TorchBackend())(
            proj(xl, 0), proj(xl, 1), proj(xl, 2), heads, ref_q=proj(rl, 0), ref_k=proj(rl, 1))
        err = (mine @ w[3].t() + bo - want[sel]).abs().max().item()
        close = (mine - full[sel]).abs().max().item()
        if not (err < 1e-4 and close == 0):
            print("rank %d of %d, N %d, flags %d: oracle err %g, world-1 err %g" % (rank, world, N, flags, err, close),
                  flush=True)
            ok = False
    _finish(rank, ok, ret)


@pytest.mark.parametrize("N,world", [(5, 2), (7, 2), (7, 3), (5, 4)])
def test_sharded_attention_uneven_gloo(N, world):
    """ShardedFRESCOAttention, all 8 guidance flag combinations, on uneven frame blocks; L = 64 trajectories split
    unevenly over 3 ranks.  Every rank's share equals the oracle on the whole batch and the world-1 call."""
    _run(_attention_worker, world, N)


# ------------------------------------------------------------------------------------------------ warp_tensor
def _warp_worker(rank, world, port, ret, N, C):
    _init(rank, world, port)
    from fresco_b200 import flow_utils as fu
    from fresco_b200.dist import frame_range
    from oracle import fresco_oracle as O
    from test_cpu_host import _TorchWarpOps
    fu.ops = _TorchWarpOps
    flows, occs = O.synth_flows(N, 64, 64, seed=5 + N, mag=5.0)
    sal = torch.rand(N, 1, 32, 32, generator=torch.Generator().manual_seed(2))
    lo, hi = frame_range(N, world, rank)
    ok = True
    for chunks, h in ((2, 8), (1, 64)):
        feat = torch.randn(chunks * N, C, h, h, generator=torch.Generator().manual_seed(3 + h))
        sel = _rows(N, lo, hi, chunks)
        full = fu.warp_tensor(feat, flows, occs, sal, chunks)
        mine = fu.warp_tensor(feat[sel].contiguous(), flows, occs, sal, chunks, shard=(world, rank, None))
        ok = ok and torch.equal(mine, full[sel])
        ok = ok and (mine - O.warp_tensor(feat, flows, occs, sal, chunks)[sel]).abs().max().item() < 1e-5
    _finish(rank, ok, ret)


@pytest.mark.parametrize("N,world,C", [(5, 2, 4), (7, 2, 4), (5, 2, 3), (7, 3, 3)])
def test_sharded_warp_tensor_uneven_gloo(N, world, C):
    """warp_tensor on uneven frame blocks: the channel re-shard (C = 4 over 2 ranks, all-to-alls with per-rank frame
    counts) and the gather path (3 channels over 2 or 3 ranks, blocks padded to the largest share).  Bit-identical to
    the unsharded call."""
    _run(_warp_worker, world, N, C)


# ------------------------------------------------------------------------------------------------ optimize_feature
def _optimize_worker(rank, world, port, ret, N):
    _init(rank, world, port)
    from fresco_b200 import diffusion_hacked as dh
    from fresco_b200.dist import frame_range
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
    lo, hi = frame_range(N, world, rank)
    sel = _rows(N, lo, hi, chunks)
    be = TorchOptBackend(O)
    ok = True
    for temporal, spatial in ((True, True), (True, False), (False, True)):
        corr, corr_l = ([target], [target[sel]]) if spatial else ([], [])
        tr_full, tr_mine = dh.OptimizeTrace(), dh.OptimizeTrace()
        full = dh.optimize_feature(feat, flows, occs, corr, iters=6, optimize_temporal=temporal, trace=tr_full, backend=be)
        want = O.optimize_feature(feat, flows, occs, corr, iters=6, optimize_temporal=temporal)
        mine = dh.optimize_feature(feat[sel].contiguous(), flows, occs, corr_l, iters=6, optimize_temporal=temporal,
                                   trace=tr_mine, shard=(world, rank, None), backend=be)
        ok = ok and (full - want).abs().max().item() < 1e-4
        ok = ok and (mine - full[sel]).abs().max().item() < 1e-4
        ok = ok and all(abs(a - b) < 1e-4 * abs(a) for a, b in zip(tr_full.losses, tr_mine.losses))
    # without flows the batch frame count comes from an all-reduce of the local counts
    full = dh.optimize_feature(feat, None, None, [target], iters=3, backend=be)
    mine = dh.optimize_feature(feat[sel].contiguous(), None, None, [target[sel]], iters=3, shard=(world, rank, None),
                               backend=be)
    ok = ok and (mine - full[sel]).abs().max().item() < 1e-4
    _finish(rank, ok, ret)


@pytest.mark.parametrize("N,world", [(7, 2), (6, 3)])
def test_sharded_optimize_feature_uneven_gloo(N, world):
    """the ring-halo optimize_feature on frame blocks of 4 / 3 and of 2 / 2 / 2 frames: all ranks together == the
    unsharded call == the oracle, loss curves included, at the tolerances of test_sharded_optimize_feature_gloo"""
    _run(_optimize_worker, world, N)


# ------------------------------------------------------------------------------------------------ per-batch preparation
def _inference_worker(rank, world, port, ret, N):
    _init(rank, world, port)
    from fresco_b200 import flow_utils as fu
    from fresco_b200 import pipe_FRESCO as pf
    from fresco_b200.dist import frame_range
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

    def pipe():
        p = _StubPipe(ac)
        p.vae = _StubVAE()
        return p
    lo, hi = frame_range(N, world, rank)
    ok = True
    for repeat in (False, True):
        rec_full, rec_sh = [], []
        for propagation in (False, True):
            kw = dict(num_warmup_steps=14, use_controlnet=False, seed=3, repeat_noise=repeat, bg_smoothing_steps=[16, 17],
                      propagation_mode=propagation, flows=flows, occs=occs, saliency=sal)
            full = pf.inference(pipe(), None, _Ctrl, imgs, pe, None, timesteps, record_latents=rec_full, **kw)
            mine = pf.inference(pipe(), None, _Ctrl, imgs, pe, None, timesteps, record_latents=rec_sh,
                                shard=(world, rank, None), **kw)
            ok = ok and torch.equal(mine, full[lo:hi]) and len(rec_full) == len(rec_sh)
            ok = ok and all(torch.equal(a, b) for a, b in zip(rec_full, rec_sh))
    _finish(rank, ok, ret)


def _flow_worker(rank, world, port, ret, N):
    _init(rank, world, port)
    from fresco_b200 import diffusion_hacked as dh
    from fresco_b200 import flow_utils as fu
    from test_cpu_host import _TorchWarpOps
    from test_dist_batch_cpu import _flow_paras_equal, _frames, _StubFlow
    fu.ops = _TorchWarpOps
    imgs = _frames(N, 64, 64, seed=4)
    model = _StubFlow()
    full = dh.get_flow_and_interframe_paras(model, imgs)
    mine = dh.get_flow_and_interframe_paras(model, imgs, shard=(world, rank, None))
    _finish(rank, _flow_paras_equal(mine, full), ret)


def _intraframe_worker(rank, world, port, ret, N):
    _init(rank, world, port)
    from fresco_b200 import diffusion_hacked as dh
    from fresco_b200.dist import ShardedFRESCOAttention, frame_range
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
    lo, hi = frame_range(N, world, rank)
    sel = _rows(N, lo, hi, 2)
    proc = dh.apply_FRESCO_attn(pipe)
    corr_full = dh.get_intraframe_paras(pipe, imgs, proc, pe, seed=3)
    in_full = seen[-1]
    proc = dh.apply_FRESCO_attn(pipe, shard=(world, rank, None))
    proc._sharded = ShardedFRESCOAttention(proc.controller, world, rank, 2, None, backend=_StandInBackend())
    corr = dh.get_intraframe_paras(pipe, imgs, proc, pe, seed=3, shard=(world, rank, None))
    ok = torch.equal(seen[-1], in_full[sel])                                      # same noise, same encoded frames
    ok = ok and len(corr) == len(corr_full) == 4 and all(_close(a, b[sel]) for a, b in zip(corr, corr_full))
    _finish(rank, ok, ret)


@pytest.mark.parametrize("N,world", [(5, 2), (7, 2), (5, 3), (7, 3)])
def test_sharded_batch_preparation_uneven_gloo(N, world):
    """inference with background smoothing (bit-identical latents and record_latents, first-batch and propagation mode,
    with and without repeat_noise) and get_flow_and_interframe_paras (flows gathered from uneven pair blocks,
    bit-identical) on uneven frame blocks"""
    _run(_inference_worker, world, N)
    _run(_flow_worker, world, N)


@pytest.mark.parametrize("N,world", [(5, 2), (7, 3)])
def test_sharded_get_intraframe_paras_uneven_gloo(N, world):
    """get_intraframe_paras on uneven frame blocks: the latents entering the UNet are bit-identical to this rank's
    frames of the unsharded call, the Gram targets equal the unsharded slices to the round-off bound of
    test_dist_batch_cpu (the CPU UNet pass runs at a different batch size)"""
    _run(_intraframe_worker, world, N)
