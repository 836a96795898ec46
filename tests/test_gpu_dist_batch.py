"""GPU tests of the sharded per-batch preparation with the real kernels: inference with background smoothing at 512^2
(warp_tensor's frame-gather path around the image-resolution chain and dilation kernels, the fused DDPM step kernels)
and get_flow_and_interframe_paras (flow-warp and mapping kernels on the gathered flows).  The VAE, the UNet and GMFlow
are per-frame stubs; every rank's share must equal the unsharded call bit for bit."""
import pytest
import torch

from dist_harness import StubFlow, fb, finish, flow_paras_equal, frames, gpu_inference, init, run  # noqa: F401

pytestmark = pytest.mark.gpu


def _batch_worker(rank, world, port, ret, backend):
    dev = init(rank, world, port, backend)
    from fresco_b200 import diffusion_hacked as dh
    from fresco_b200.dist import shard_layout
    N, res = 4, 512
    shard = (world, rank, None)
    bad = gpu_inference(N, shard_layout(N, shard), shard, dev, repeats=(False, True))
    # per-batch flow parameters at 512 x 512 from a per-pair stub flow model on the GPU
    model = StubFlow().to(dev)
    imgs = frames(N, res, res, seed=4)
    full = dh.get_flow_and_interframe_paras(model, imgs)
    mine = dh.get_flow_and_interframe_paras(model, imgs, shard=shard)
    if not (flow_paras_equal(mine, full) and full[1][0].device == dev):
        bad.append("sharded get_flow_and_interframe_paras differs")
    for b in bad:
        print("rank %d: %s" % (rank, b), flush=True)
    finish(rank, not bad, ret, dev)


def test_sharded_batch_preparation_nccl_world2_bit_identical(fb):
    """over NCCL on two GPUs: sharded inference with background smoothing and sharded get_flow_and_interframe_paras ==
    unsharded, bit for bit.  Needs two devices; skipped on a one-GPU box."""
    run(_batch_worker, 2, "nccl", gpus=2)


def test_sharded_batch_preparation_two_ranks_one_gpu_bit_identical(fb):
    """the same two ranks sharing one GPU, exchanging through gloo: the partition and the real kernels on any box"""
    run(_batch_worker, 2, "gloo")
