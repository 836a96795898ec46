"""GPU tests of the sharded per-batch preparation with the real kernels: inference with background smoothing at 512^2
(warp_tensor's frame-gather path around the image-resolution chain and dilation kernels, the fused DDPM step kernels)
and get_flow_and_interframe_paras (flow-warp and mapping kernels on the gathered flows).  The VAE, the UNet and GMFlow
are per-frame stubs; every rank's share must equal the unsharded call bit for bit."""
import os
import socket
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def fb():
    if not torch.cuda.is_available():
        pytest.skip("GPU tests need a CUDA device")
    from fresco_b200 import _lib
    _lib.lib()      # fails loudly if the extension is missing


class _GPUStubUNet(torch.nn.Module):
    """per-frame 'UNet' without reductions: every output frame depends on its own input frame and prompt only"""

    class config:
        in_channels = 4

    dtype = torch.float16

    def forward(self, x, t, encoder_hidden_states=None, **kw):
        return (torch.tanh(x * 0.7 + 0.001 * float(t)) + 0.1 * encoder_hidden_states[:, 0, 0].view(-1, 1, 1, 1),)


class _GPUStubPipe:
    def __init__(self, ac, device):
        from test_cpu_host import _Sched
        from test_dist_batch_cpu import _StubVAE
        self.scheduler = _Sched(ac)
        self.vae = _StubVAE()
        self.unet = _GPUStubUNet()
        self._execution_device = device

    def prepare_latents(self, B, C, H, W, dtype, device, generator, latents=None):
        return torch.randn(B, C, H // 8, W // 8, generator=generator, device=device, dtype=dtype)


def _batch_worker(rank, world, port, ret, backend):
    """``backend`` "nccl": one GPU per rank; "gloo": every rank on GPU 0, the exchanges through host memory"""
    import torch.distributed as dist
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dev = torch.device("cuda", rank if backend == "nccl" else 0)
    torch.cuda.set_device(dev)
    if backend == "nccl":
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    else:
        dist.init_process_group("gloo", rank=rank, world_size=world)
    from fresco_b200 import diffusion_hacked as dh
    from fresco_b200 import pipe_FRESCO as pf
    from fresco_b200.dist import frame_range
    from oracle import fresco_oracle as O
    from test_dist_batch_cpu import _frames, _flow_paras_equal, _StubFlow
    from test_dist_cpu import _Ctrl
    shard = (world, rank, None)
    ok = True
    # inference with background smoothing at 512 x 512: fp16 latents and images, 3-channel frames gathered for the chain
    N, res = 4, 512
    lo, hi = frame_range(N, world, rank)
    ac = torch.from_numpy(np.load(os.path.join(ROOT, "tests", "golden", "ddpm_step.npz"))["alphas_cumprod"])
    g = torch.Generator().manual_seed(1)
    imgs = (torch.rand(N, 3, res, res, generator=g) * 2 - 1).half().to(dev)
    pe = torch.randn(2 * N, 5, 8, generator=g).half().to(dev)
    flows, occs = O.synth_flows(N, res, res, seed=9, mag=12.0)
    flows, occs = [f.to(dev) for f in flows], [o.to(dev) for o in occs]
    sal = (torch.rand(N, 1, res, res, generator=g) > 0.4).float().to(dev)
    timesteps = [950 - 50 * i for i in range(20)]
    for repeat in (False, True):
        rec_full, rec_sh = [], []
        for propagation in (False, True):
            kw = dict(num_warmup_steps=14, use_controlnet=False, seed=3, repeat_noise=repeat, bg_smoothing_steps=[16, 17],
                      propagation_mode=propagation, flows=flows, occs=occs, saliency=sal)
            full = pf.inference(_GPUStubPipe(ac, dev), None, _Ctrl, imgs, pe, None, timesteps, record_latents=rec_full, **kw)
            mine = pf.inference(_GPUStubPipe(ac, dev), None, _Ctrl, imgs, pe, None, timesteps, record_latents=rec_sh,
                                shard=shard, **kw)
            same = bool(torch.equal(mine, full[lo:hi])) and len(rec_full) == len(rec_sh)
            same = same and all(bool(torch.equal(a, b)) for a, b in zip(rec_full, rec_sh))
            if not same:
                print("rank %d: sharded inference differs (repeat_noise=%s, propagation=%s): max |d| = %g"
                      % (rank, repeat, propagation, (mine.float() - full[lo:hi].float()).abs().max().item()), flush=True)
            ok = ok and same
    # per-batch flow parameters at 512 x 512 from a per-pair stub flow model on the GPU
    model = _StubFlow().to(dev)
    frames = _frames(N, res, res, seed=4)
    full = dh.get_flow_and_interframe_paras(model, frames)
    mine = dh.get_flow_and_interframe_paras(model, frames, shard=shard)
    same = _flow_paras_equal(mine, full) and full[1][0].device == dev
    if not same:
        print("rank %d: sharded get_flow_and_interframe_paras differs" % rank, flush=True)
    ok = ok and same
    t = torch.tensor([1 if ok else 0], device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MIN)
    if rank == 0:
        ret.put(int(t.item()))
    dist.destroy_process_group()


def _run(backend):
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    ret = ctx.Queue()
    procs = [ctx.Process(target=_batch_worker, args=(r, 2, port, ret, backend)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(300)
        assert p.exitcode == 0
    assert ret.get(timeout=5) == 1


def test_sharded_batch_preparation_nccl_world2_bit_identical(fb):
    """over NCCL on two GPUs: sharded inference with background smoothing and sharded get_flow_and_interframe_paras ==
    unsharded, bit for bit.  Needs two devices; skipped on a one-GPU box."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    _run("nccl")


def test_sharded_batch_preparation_two_ranks_one_gpu_bit_identical(fb):
    """the same two ranks sharing one GPU, exchanging through gloo: the partition and the real kernels on any box"""
    _run("gloo")
