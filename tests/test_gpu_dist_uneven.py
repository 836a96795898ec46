"""GPU tests of frame-sharded batches whose frame count the rank count does not divide, with the real kernels: every
rank's share must equal the unsharded call bit for bit.  Ranks are processes sharing one GPU over gloo (and one GPU
each over NCCL when the box has enough), or threads in lock step for the ring-halo feature optimisation; plus the
loss-scale entry points of the Gram kernels against the weight entry points."""
import threading

import numpy as np
import pytest
import torch

from dist_harness import fb, finish, gpu_inference, gpu_layer, gpu_warp, init, rows, run  # noqa: F401

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------ attention + warp_tensor
def _layer_worker(rank, world, port, ret, backend, N):
    dev = init(rank, world, port, backend)
    from fresco_b200.dist import shard_layout
    # 1024 trajectories do not split evenly over 3 ranks; the 640 channels re-shard on 2 ranks, gather on 3
    shard = (world, rank, None)
    lay = shard_layout(N, shard)
    bad = gpu_layer(N, lay, shard, dev) + gpu_warp(N, lay, shard, dev)
    for b in bad:
        print("rank %d: %s" % (rank, b), flush=True)
    finish(rank, not bad, ret, dev)


@pytest.mark.parametrize("backend", ["gloo", "nccl"])
@pytest.mark.parametrize("N,world", [(7, 2), (5, 3)])
def test_sharded_layer_uneven_bit_identical(fb, N, world, backend):
    """ShardedFRESCOAttention (all guidance flags) and warp_tensor on uneven frame blocks == unsharded, bit for bit.
    gloo: the ranks share one GPU; nccl: one GPU per rank, skipped on a box with fewer."""
    run(_layer_worker, world, backend, N, gpus=world if backend == "nccl" else 0)


def _inference_worker(rank, world, port, ret, backend, N):
    dev = init(rank, world, port, backend)
    from fresco_b200.dist import shard_layout
    shard = (world, rank, None)
    bad = gpu_inference(N, shard_layout(N, shard), shard, dev, repeats=(True,))
    for b in bad:
        print("rank %d: %s" % (rank, b), flush=True)
    finish(rank, not bad, ret, dev)


@pytest.mark.parametrize("backend", ["gloo", "nccl"])
def test_sharded_inference_uneven_bit_identical(fb, backend):
    """inference with background smoothing at 512^2 on frame blocks of 3 and 2 == unsharded, bit for bit"""
    run(_inference_worker, 2, backend, 5, gpus=2 if backend == "nccl" else 0)


# ------------------------------------------------------------------------------------------------ optimize_feature
@pytest.mark.parametrize("N,C,h,world", [(7, 640, 64, 2), (9, 1280, 32, 2), (15, 1280, 24, 3)])
def test_optimize_feature_ring_halo_uneven_bit_identical(fb, N, C, h, world):
    """optimize_feature (temporal + Gram-L1 terms, Adam, AdaIN) with the ranks as lock-step threads on one GPU: the
    ranks' outputs together are bit-identical to the unsharded call.  (9, 1280, 32) and (15, 1280, 24) are shapes where
    a rank's share of the weight rounded to fp32 gives another Gram loss scale than the unsharded call; the second is
    an even split."""
    from fresco_b200 import diffusion_hacked as dh
    from fresco_b200.dist import shard_layout
    from test_gpu_parity_r2 import _LockstepRing, _layer_case
    flows, occs, cs = _layer_case(N, C, h, seed=31 + h)
    flows = [f.cuda() for f in flows]
    occs = [o.cuda() for o in occs]
    sample = cs.reshape(2 * N, C, h, h).half().cuda()
    g = torch.Generator(device="cuda").manual_seed(5)
    ref = (sample.float() + 0.5 * torch.randn(sample.shape, device="cuda", generator=g)).half()
    target = dh.gram_targets([ref])[0]
    full = dh.optimize_feature(sample, flows, occs, correlation_matrix=[target], iters=6)
    ring = _LockstepRing(world)
    outs, errs = [None] * world, []

    def run(rank):
        ring.lock.acquire()
        try:
            sel = rows(N, shard_layout(N, (world, rank, None)), "cuda")
            tgt = dh.GramTarget(target.yhat[sel].contiguous())
            outs[rank] = (sel, dh.optimize_feature(sample[sel].contiguous(), flows, occs, correlation_matrix=[tgt], iters=6,
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
    for rank, (sel, out) in enumerate(outs):
        assert torch.equal(out, full[sel]), (rank, (out.float() - full[sel].float()).abs().max().item())


# ------------------------------------------------------------------------------------------------ Gram loss-scale entry points
@pytest.mark.parametrize("B,C,h,w", [(14, 1280, 24, 24), (4, 640, 40, 32)])
def test_gram_scaled_entry_points_match_weight_forms(fb, B, C, h, w):
    """fresco_gram_{sign,sign_ref,grad}_scaled with scale = weight / (B L^2) give the tsign and gradient bits of the
    weight entry points, and the same loss up to the order of the kernels' atomic adds"""
    from fresco_b200 import _lib as L
    from fresco_b200 import ops
    lib, P, st = L.lib(), L.ptr, L.stream()
    Lt, weight = h * w, float(np.float32(100.0 * 7 / 15))           # the weight forms take an fp32 weight
    scale = weight / (B * Lt * Lt)
    g = torch.Generator(device="cuda").manual_seed(C + Lt)
    xhat, norms = ops.gram_normalize(torch.randn(B, C, Lt, device="cuda", generator=g))
    yhat, _ = ops.gram_normalize(torch.randn(B, C, Lt, device="cuda", generator=g))
    dense = torch.bmm(yhat.float(), yhat.float().transpose(1, 2)).contiguous()
    runs = {}
    for form in ("weight", "scaled"):
        out = {}
        for name, target in (("sign_ref", yhat), ("sign", dense)):
            tsign = torch.empty(B, Lt, Lt, dtype=torch.float16, device="cuda")
            loss = torch.zeros(1, device="cuda")
            fn = getattr(lib, "fresco_gram_%s%s" % (name, "_scaled" if form == "scaled" else ""))
            L.check(fn(P(xhat), P(target), P(tsign), P(loss), B, Lt, C, scale if form == "scaled" else weight, st), name)
            out[name] = (tsign, loss)
        nbytes = int(lib.fresco_gram_grad_workspace_bytes(B, Lt, C))
        ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
        for v in (2, 1):
            L.set_option("FRESCO_GRAM_V", v)
            try:
                grad = torch.full((B, C, Lt), 0.25, device="cuda")
                if form == "scaled":
                    rc = lib.fresco_gram_grad_scaled(P(out["sign_ref"][0]), P(xhat), P(norms), P(grad), B, Lt, C, scale,
                                                     P(ws), nbytes, st)
                else:
                    rc = lib.fresco_gram_grad(P(out["sign_ref"][0]), P(xhat), P(norms), P(grad), B, Lt, C, weight, P(ws),
                                              nbytes, st)
                L.check(rc, "gram_grad")
            finally:
                L.set_option("FRESCO_GRAM_V", -1)
            out["grad%d" % v] = grad
        runs[form] = out
    a, b = runs["weight"], runs["scaled"]
    for name in ("sign_ref", "sign"):
        assert torch.equal(a[name][0], b[name][0]), name
        la, lb = a[name][1].item(), b[name][1].item()
        assert la > 0 and abs(la - lb) <= 1e-5 * la, (name, la, lb)          # fp32 atomics: the order varies per call
    for v in (2, 1):
        assert torch.equal(a["grad%d" % v], b["grad%d" % v]), v
