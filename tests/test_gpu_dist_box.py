"""GPU tests of keyframe batches sharded through ``dist.Box`` with the real kernels: the unequal-halves layout at world 3
(N = 2: two ranks on the unconditional half, one on the text half) and idle ranks at world 4 (N = 1).  Every active
rank's rows must equal the one-GPU call bit for bit: the FRESCO layer, optimize_feature with the ring halo, and a
denoise step with guidance and background smoothing; an idle rank returns empty results without a collective.  gloo:
the ranks share one GPU (transfers staged through host memory); nccl: one GPU each, skipped on a box with fewer, and
there one step is also captured in a CUDA graph and replayed."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from dist_harness import ROOT, Ctrl, NoCollectives, StubPipe, fb, finish, gpu_layer, init, rows, run  # noqa: F401

pytestmark = pytest.mark.gpu


class _FrameVAE:
    """a per-pixel VAE stand-in (nearest up-sampling to decode, average pooling to encode): every output frame depends on
    its own input frame only, so its bits do not depend on the batch size"""

    class config:
        scaling_factor = 0.18215

    class _Dist:
        def __init__(self, x):
            self.latent_dist = self
            self.x = x

        def sample(self):
            return F.avg_pool2d(self.x, 8).repeat(1, 2, 1, 1)[:, :4].contiguous()

    def encode(self, x):
        return self._Dist(x)

    def decode(self, z):
        class Out:
            sample = F.interpolate(z[:, :3].float(), scale_factor=8, mode="nearest").contiguous()
        return Out


def _optimize(N, lay, box, dev):
    from fresco_b200 import diffusion_hacked as dh
    from test_gpu_parity_r2 import _layer_case
    C, h = 640, 64
    flows, occs, cs = _layer_case(N, C, h, seed=31 + h)
    flows, occs = [f.to(dev) for f in flows], [o.to(dev) for o in occs]
    sample = cs.reshape(2 * N, C, h, h).half().to(dev)
    g = torch.Generator(device=dev).manual_seed(5)
    ref = (sample.float() + 0.5 * torch.randn(sample.shape, device=dev, generator=g)).half()
    target = dh.gram_targets([ref])[0]
    tr_full, tr_mine = dh.OptimizeTrace(), dh.OptimizeTrace()
    full = dh.optimize_feature(sample, flows, occs, correlation_matrix=[target], iters=6, trace=tr_full)
    sel = rows(N, lay, dev)
    mine = dh.optimize_feature(sample[sel].contiguous(), flows, occs, iters=6, trace=tr_mine, shard=box,
                               correlation_matrix=[dh.GramTarget(target.yhat[sel].contiguous())])
    bad = []
    if not torch.equal(mine, full[sel]):
        bad.append("optimize_feature: max |d| = %g" % (mine.float() - full[sel].float()).abs().max().item())
    # the loss curve summed over the ranks, up to the order of the kernels' atomic adds
    if not all(abs(a - b) <= 1e-5 * abs(a) for a, b in zip(tr_full.losses, tr_mine.losses)):
        bad.append("optimize_feature loss curve %s vs %s" % (tr_mine.losses, tr_full.losses))
    return bad


def _step_case(N, dev):
    from fresco_b200.harness import synth
    ac = torch.from_numpy(np.load(os.path.join(ROOT, "tests", "golden", "ddpm_step.npz"))["alphas_cumprod"])
    pipe = StubPipe(ac, _FrameVAE)
    g = torch.Generator().manual_seed(6)
    eps, x, noise = (torch.randn(n, 4, 32, 32, generator=g).to(dev) for n in (2 * N, N, N))
    flows, occs = synth.smooth_flows(N, 256, 256, dev, seed=7)
    sal = (torch.rand(N, 1, 256, 256, generator=g) > 0.4).float().to(dev)
    return pipe, eps, x, noise, flows, occs, sal


def _step(N, lay, box, dev, graph):
    from fresco_b200 import pipe_FRESCO as pf
    pipe, eps, x, noise, flows, occs, sal = _step_case(N, dev)
    lo, hi = lay.lo, lay.hi
    mine_eps = eps[rows(N, lay, dev)].contiguous()
    bad = []
    for smooth in (False, True) if N > 1 else (False,):         # the warp chain needs two frames
        kw = dict(flows=flows, occs=occs, saliency=sal) if smooth else {}
        full = pf.step(pipe, eps, 700, x, None, guidance_scale=7.5, noise=noise, **kw)
        mine = pf.step(pipe, mine_eps, 700, x[lo:hi].contiguous(), None, guidance_scale=7.5,
                       noise=noise[lo:hi].contiguous(), shard=lay, **kw)
        if not all(torch.equal(a, b[lo:hi]) for a, b in zip(mine, full)):
            bad.append("step smoothing %s: max |d| = %g" % (smooth, (mine[0] - full[0][lo:hi]).abs().max().item()))
    if graph:
        # the per-step exchange and kernels captured once and replayed: all sizes are host ints of the layout
        want = pf.step(pipe, eps, 700, x, None, guidance_scale=7.5, noise=noise)[0][lo:hi]
        s_eps, s_x, s_noise = mine_eps.clone(), x[lo:hi].clone(), noise[lo:hi].clone()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            pf.step(pipe, s_eps, 700, s_x, None, guidance_scale=7.5, noise=s_noise, shard=lay)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        cg = torch.cuda.CUDAGraph()
        with torch.cuda.graph(cg):
            out = pf.step(pipe, s_eps, 700, s_x, None, guidance_scale=7.5, noise=s_noise, shard=lay)[0]
        for _ in range(2):
            cg.replay()
        torch.cuda.synchronize()
        if not torch.equal(out, want):
            bad.append("graph-replayed step: max |d| = %g" % (out - want).abs().max().item())
    return bad


def _idle(N, box, dev):
    """an idle rank: every entry point returns at once, with every collective of torch.distributed failing on use"""
    from fresco_b200 import diffusion_hacked as dh
    from fresco_b200 import flow_utils as fu
    from fresco_b200 import pipe_FRESCO as pf
    bad = []
    pipe, eps, x, noise, flows, occs, sal = _step_case(N, dev)
    with NoCollectives(("all_gather_into_tensor", "all_to_all_single", "all_reduce", "broadcast", "batch_isend_irecv",
                        "new_group", "split_group")):
        none = x[:0]
        if pf.step(pipe, none, 700, none, None, guidance_scale=7.5, flows=flows, occs=occs, saliency=sal,
                   shard=box)[0] is not none:
            bad.append("step")
        if fu.warp_tensor(none, flows, occs, sal, 1, shard=box) is not none:
            bad.append("warp_tensor")
        if dh.optimize_feature(none, flows, occs, [], shard=box) is not none:
            bad.append("optimize_feature")
        out = pf.inference(pipe, None, Ctrl, torch.rand(N, 3, 256, 256, device=dev), torch.randn(2 * N, 5, 8, device=dev),
                           None, [700], num_warmup_steps=0, use_controlnet=False, record_latents=[], shard=box)
        if tuple(out.shape) != (0, 4, 32, 32):
            bad.append("inference returned %s" % (tuple(out.shape),))
    return bad


def _box_worker(rank, world, port, ret, backend, N):
    dev = init(rank, world, port, backend)
    from fresco_b200.dist import Box, shard_layout
    box = Box(world, rank)
    lay = shard_layout(N, box)            # under NCCL every rank of the Box takes part in splitting its groups once
    if lay.idle:
        bad = _idle(N, box, dev) if rank >= 2 * N else ["rank %d idle" % rank]
    else:
        bad = gpu_layer(N, lay, box, dev) + _step(N, lay, box, dev, graph=backend == "nccl")
        if N > 1:
            bad += _optimize(N, lay, box, dev)
    for b in bad:
        print("rank %d of %d (%s), N %d: %s" % (rank, world, backend, N, b), flush=True)
    finish(rank, not bad, ret, dev)


@pytest.mark.parametrize("backend", ["gloo", "nccl"])
@pytest.mark.parametrize("N,world", [(2, 3), (1, 4)])
def test_box_bit_identical(fb, N, world, backend):
    """(2, 3): the unequal-halves layout -- ranks 0 and 1 hold frame 0 and frame 1 of the unconditional half, rank 2
    both frames of the text half.  (1, 4): ranks 0 and 1 hold the two halves of the one frame, ranks 2 and 3 are idle.
    The FRESCO layer (all 8 guidance flag combinations), optimize_feature with the ring halo (N = 2) and a denoise step
    with guidance, with and without background smoothing, equal the one-GPU call bit for bit on every active rank; over
    NCCL a captured step replays to the same bits."""
    run(_box_worker, world, backend, N, gpus=world if backend == "nccl" else 0)
