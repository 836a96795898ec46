"""gloo tests of the sharded per-batch preparation: get_flow_and_interframe_paras (GMFlow pairs split over the ranks),
get_intraframe_paras (the reference pass on this rank's frames), warp_tensor's frame-gather path and inference with
background smoothing.  Same pattern as test_dist_cpu.py: spawned ranks, torch stand-ins for the kernels; every rank
compares its share with the unsharded call on the whole batch."""
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(worker, world, *args, timeout=240):
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    ret = ctx.Queue()
    procs = [ctx.Process(target=worker, args=(r, world, port, ret) + args) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout)
        assert p.exitcode == 0
    assert ret.get(timeout=5) == 1


def _init(rank, world, port):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)


def _finish(rank, ok, ret):
    t = torch.tensor([1 if ok else 0])
    dist.all_reduce(t, op=dist.ReduceOp.MIN)
    if rank == 0:
        ret.put(int(t.item()))
    dist.destroy_process_group()


def _subgroup(rank, world, subgroups):
    """(world, rank, group) of this process: the whole world, or one of two independent groups {0,1} / {2,3}"""
    if not subgroups:
        return world, rank, None
    groups = [dist.new_group([0, 1]), dist.new_group([2, 3])]
    return 2, rank % 2, groups[rank // 2]


def _rows(n, lo, hi, chunks):
    return torch.cat([torch.arange(c * n + lo, c * n + hi) for c in range(chunks)])


# ------------------------------------------------------------------------------------------------ warp_tensor, gather path
def _warp_gather_worker(rank, world, port, ret, subgroups):
    _init(rank, world, port)
    from fresco_b200 import flow_utils as fu
    from oracle import fresco_oracle as O
    from test_cpu_host import _TorchWarpOps
    fu.ops = _TorchWarpOps
    batch = rank // 2 if subgroups else 0                   # each group denoises its own batch
    world, rank, group = _subgroup(rank, world, subgroups)
    N = 4
    flows, occs = O.synth_flows(N, 64, 64, seed=7 + batch, mag=6.0)
    sal = torch.rand(N, 1, 32, 32, generator=torch.Generator().manual_seed(2))
    lo, hi = rank * N // world, (rank + 1) * N // world
    ok = True
    # a decoded image batch (3 channels, image resolution: the dilated-occlusion path) and a 3-channel batch of two CFG
    # chunks at feature resolution; fp32 and fp16 (what the VAE returns)
    for chunks, h in ((1, 64), (2, 16)):
        for dtype in (torch.float32, torch.float16):
            x = torch.rand(chunks * N, 3, h, h, generator=torch.Generator().manual_seed(3 + h + batch)).to(dtype)
            sel = _rows(N, lo, hi, chunks)
            want = O.warp_tensor(x.float(), flows, occs, sal, chunks).to(dtype)
            full = fu.warp_tensor(x, flows, occs, sal, chunks)
            mine = fu.warp_tensor(x[sel].contiguous(), flows, occs, sal, chunks, shard=(world, rank, group))
            ok = ok and mine.dtype == dtype and torch.equal(mine, full[sel])             # the chain sees the same batch
            tol = 1e-5 if dtype == torch.float32 else 1e-2
            ok = ok and (mine.float() - want[sel].float()).abs().max().item() < tol
    _finish(dist.get_rank(), ok, ret)


@pytest.mark.parametrize("world", [2, 4])
def test_sharded_warp_tensor_gather_path_gloo(world):
    """warp_tensor(shard=...) on 3-channel batches, which do not split by channel over the ranks: the frames are
    all-gathered and the chain runs on the whole batch.  Bit-identical to the unsharded call, and equal to the oracle's
    warp_tensor on the full batch.  World 4 leaves one frame per rank."""
    _run(_warp_gather_worker, world, False)


def test_sharded_warp_tensor_gather_path_in_subgroups_gloo():
    """the gather path in two process groups {0,1} and {2,3} of one world, each with its own batch"""
    _run(_warp_gather_worker, 4, True)


# ------------------------------------------------------------------------------------------------ inference + smoothing
class _StubVAE:
    """per-frame, deterministic VAE: every output frame depends on its own input frame only (no reductions across
    channels, so the result does not depend on the batch size on a GPU either)"""

    class config:
        scaling_factor = 0.5

    def encode(self, x):
        class D:
            def __init__(self, v):
                self.latent_dist = self
                self.v = v

            def sample(self):
                return self.v
        p = F.avg_pool2d(x, 8)
        return D(torch.cat([p, 0.5 * (p[:, :1] + p[:, 2:3])], 1) * 2 - 1)

    def decode(self, z):
        class D:
            pass
        d = D()
        img = torch.tanh(z[:, :3] + 0.5 * z[:, 3:])
        d.sample = F.interpolate(img, scale_factor=8, mode="nearest")
        return d


def _inference_smoothing_worker(rank, world, port, ret):
    _init(rank, world, port)
    from fresco_b200 import flow_utils as fu
    from fresco_b200 import pipe_FRESCO as pf
    from oracle import fresco_oracle as O
    from test_cpu_host import _TorchStepOps, _TorchWarpOps
    from test_dist_cpu import _Ctrl, _StubPipe
    pf.ops = _TorchStepOps
    fu.ops = _TorchWarpOps
    ac = torch.from_numpy(np.load(os.path.join(ROOT, "tests", "golden", "ddpm_step.npz"))["alphas_cumprod"])
    N = 4
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
    lo, hi = rank * N // world, (rank + 1) * N // world
    ok = True
    for repeat in (False, True):
        rec_full, rec_sh = [], []
        for propagation in (False, True):
            # schedule steps 14..19: the background-smoothing steps 16 and 17 are loop steps 2 and 3
            kw = dict(num_warmup_steps=14, use_controlnet=False, seed=3, repeat_noise=repeat, bg_smoothing_steps=[16, 17],
                      propagation_mode=propagation, flows=flows, occs=occs, saliency=sal)
            full = pf.inference(pipe(), None, _Ctrl, imgs, pe, None, timesteps, record_latents=rec_full, **kw)
            mine = pf.inference(pipe(), None, _Ctrl, imgs, pe, None, timesteps, record_latents=rec_sh,
                                shard=(world, rank, None), **kw)
            ok = ok and torch.equal(mine, full[lo:hi]) and len(rec_full) == len(rec_sh)
            ok = ok and all(torch.equal(a, b) for a, b in zip(rec_full, rec_sh))
            if not propagation:             # smoothing did change the result: the same run without it differs
                plain = pf.inference(pipe(), None, _Ctrl, imgs, pe, None, timesteps, record_latents=[],
                                     **dict(kw, bg_smoothing_steps=[]))
                ok = ok and not torch.equal(plain, full)
    _finish(rank, ok, ret)


@pytest.mark.parametrize("world", [2, 4])
def test_sharded_inference_with_background_smoothing_gloo(world):
    """pipe_FRESCO.inference frame-sharded with the background-smoothing steps inside the run (per-frame stub VAE,
    saliency map): latents and record_latents of the ranks == the unsharded call, bit for bit, in first-batch and
    propagation mode, with and without repeat_noise.  World 4 leaves one frame per rank."""
    _run(_inference_smoothing_worker, world)


# ------------------------------------------------------------------------------------------------ get_intraframe_paras
class _StandInBackend:
    """the attention stand-in of test_cpu_host (fp32 math, fp16 results) behind ShardedFRESCOAttention's backend API"""

    def attn_fwd(self, q, k, v, heads, q_per_kv, softmax_scale, diag_bias=0.0):
        from test_cpu_host import _TorchOps
        return _TorchOps.attn_fwd(q, k, v, heads, q_per_kv, softmax_scale=softmax_scale, diag_bias=diag_bias)


# stored reference inputs, Gram targets and the guided step's output: the sharded and the unsharded UNet pass differ only
# in the batch size the fp32 CPU convolutions and GEMMs see, so in the last bits (at one rank, exactly 0).  The FRESCO
# processor rounds q / k / v and the attention outputs to fp16, as the kernels do, and a last-bit difference can move
# one of those roundings.  Bound: 1e-4 of the tensor's largest magnitude, a fifth of an fp16 ulp (observed: at most
# 3.1e-5 at world 2).
REL_TOL = 1e-4


def _close(a, b):
    return a.shape == b.shape and (a.float() - b.float()).abs().max().item() <= REL_TOL * max(b.float().abs().max().item(), 1.0)


def _intraframe_worker(rank, world, port, ret):
    _init(rank, world, port)
    from fresco_b200 import diffusion_hacked as dh
    from fresco_b200.dist import ShardedFRESCOAttention
    from fresco_b200.harness.sd15_unet import FakePipe, SD15UNet
    from test_cpu_host import _Sched, _TorchOps
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
    unet.register_forward_pre_hook(lambda m, a: seen.append(a[0].clone()))          # the latents entering the UNet
    N = 4
    g = torch.Generator().manual_seed(5)
    imgs = torch.rand(N, 3, 128, 128, generator=g) * 2 - 1
    pe = torch.randn(2 * N, 7, 24, generator=g)
    t = Sched.timesteps[-1]
    lo, hi = rank * N // world, (rank + 1) * N // world
    sel = _rows(N, lo, hi, 2)

    proc = dh.apply_FRESCO_attn(pipe)
    corr_full = dh.get_intraframe_paras(pipe, imgs, proc, pe, seed=3)
    in_full = seen[-1]
    stored_full = list(proc.controller.stored_attn["decoder_attn"])
    proc.controller.enable_intraattn()
    out_full = pipe.unet(in_full, t, encoder_hidden_states=pe, return_dict=False)[0]

    shard = (world, rank, None)
    proc = dh.apply_FRESCO_attn(pipe, shard=shard)
    proc._sharded = ShardedFRESCOAttention(proc.controller, world, rank, 2, None, backend=_StandInBackend())
    corr = dh.get_intraframe_paras(pipe, imgs, proc, pe, seed=3, shard=shard)
    ctrl = proc.controller
    ok = not ctrl.store and not ctrl.use_intraattn and not ctrl.use_cfattn and not ctrl.use_interattn
    ok = ok and torch.equal(seen[-1], in_full[sel])                                   # same noise, same encoded frames
    stored = ctrl.stored_attn["decoder_attn"]
    ok = ok and len(stored) == len(stored_full) == 6 and all(_close(a, b[sel]) for a, b in zip(stored, stored_full))
    ok = ok and len(corr) == len(corr_full) == 4 and all(_close(a, b[sel]) for a, b in zip(corr, corr_full))
    # the sharded processor runs a spatial-guided step on the stored local references
    ctrl.enable_intraattn()
    out = pipe.unet(seen[-1], t, encoder_hidden_states=pe[sel], return_dict=False)[0]
    ok = ok and _close(out, out_full[sel])
    _finish(rank, ok, ret)


@pytest.mark.parametrize("world", [2, 4])
def test_sharded_get_intraframe_paras_on_harness_unet_gloo(world):
    """get_intraframe_paras(shard=...) on the CPU harness UNet: the latents entering the UNet are bit-identical to this
    rank's frames of the unsharded call; the stored reference inputs and the Gram targets equal the unsharded slices to
    REL_TOL of their magnitude (fp32 round-off of a batch-size-dependent UNet pass); the sharded processor then runs a
    spatial-guided step on them (its reference / hidden-state shapes match) and matches the unsharded step."""
    _run(_intraframe_worker, world)


# ------------------------------------------------------------------------------------------------ get_flow_and_interframe_paras
class _StubFlow(torch.nn.Module):
    """GMFlow's call signature and output layout (forward | backward flows of the pairs); every pair's flow depends on
    that pair's two frames only (elementwise ops and pooling: batch-size independent on a GPU too)"""

    def __init__(self):
        super().__init__()
        self.gain = torch.nn.Parameter(torch.tensor([6.0, -4.0]))

    def _flow(self, a, b):
        grey = lambda x: x[:, 0:1] + x[:, 1:2] + x[:, 2:3]
        d = F.avg_pool2d(grey(b - a) / 192.0, 8)
        s = F.avg_pool2d(grey(a) / 384.0 - 1.0, 8)
        d = F.interpolate(torch.cat([torch.tanh(d + s), torch.tanh(d - s)], 1), size=a.shape[-2:], mode="bilinear")
        return d * self.gain.view(1, 2, 1, 1)

    def forward(self, img0, img1, attn_splits_list=None, corr_radius_list=None, prop_radius_list=None,
                pred_bidir_flow=False):
        assert pred_bidir_flow
        return {"flow_preds": [torch.cat([self._flow(img0, img1), self._flow(img1, img0)]).detach()]}


def _frames(n, h, w, seed):
    """n uint8 HxWx3 frames of one moving, smooth scene"""
    g = torch.Generator().manual_seed(seed)
    base = F.interpolate(torch.rand(1, 3, h // 8 + 4, w // 8 + 4, generator=g), size=(h + 32, w + 32), mode="bicubic")
    out = []
    for i in range(n):
        y, x = 2 * i, 3 * i
        f = base[0, :, y:y + h, x:x + w].clamp(0, 1) * 255
        out.append(f.permute(1, 2, 0).round().to(torch.uint8).numpy())
    return out


def _flow_paras_equal(a, b):
    (fa, oa, ma, pa), (fb, ob, mb, pb) = a, b
    same = lambda x, y: len(x) == len(y) and all(torch.equal(u, v) for u, v in zip(x, y))
    return (same(fa, fb) and same(oa, ob) and same(ma, mb)
            and all(same(pa[k], pb[k]) for k in ("fwd_mappings", "bwd_mappings", "interattn_masks")))


def _flow_worker(rank, world, port, ret):
    _init(rank, world, port)
    from fresco_b200 import diffusion_hacked as dh
    from fresco_b200 import flow_utils as fu
    from test_cpu_host import _TorchWarpOps
    fu.ops = _TorchWarpOps
    N = 4
    imgs = _frames(N, 64, 64, seed=4)
    model = _StubFlow()
    full = dh.get_flow_and_interframe_paras(model, imgs)
    mine = dh.get_flow_and_interframe_paras(model, imgs, shard=(world, rank, None))
    ok = _flow_paras_equal(mine, full)
    ok = ok and 0 < full[1][1].sum().item() < full[1][1].numel()                     # some, not all, pixels occluded
    _finish(rank, ok, ret)


@pytest.mark.parametrize("world", [2, 4])
def test_sharded_get_flow_and_interframe_paras_gloo(world):
    """get_flow_and_interframe_paras(shard=...) with a per-pair stub flow model: each rank runs its own pairs, one
    all-gather assembles the flows; flows, occlusions, K/V masks, mappings and trajectory masks are bit-identical to
    the unsharded call on every rank.  World 4 leaves one pair per rank."""
    _run(_flow_worker, world)
