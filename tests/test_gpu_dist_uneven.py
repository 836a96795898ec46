"""GPU tests of frame-sharded batches whose frame count the rank count does not divide, with the real kernels: every
rank's share must equal the unsharded call bit for bit.  Ranks are processes sharing one GPU over gloo (and one GPU
each over NCCL when the box has enough), or threads in lock step for the ring-halo feature optimisation; plus the
loss-scale entry points of the Gram kernels against the weight entry points."""
import os
import socket
import sys
import threading

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))


@pytest.fixture(scope="module")
def fb():
    if not torch.cuda.is_available():
        pytest.skip("GPU tests need a CUDA device")
    from fresco_b200 import _lib
    _lib.lib()      # fails loudly if the extension is missing


def _init(rank, world, port, backend):
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
    return dev


def _finish(rank, ok, ret, dev):
    import torch.distributed as dist
    t = torch.tensor([1 if ok else 0], device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MIN)
    if rank == 0:
        ret.put(int(t.item()))
    dist.destroy_process_group()


def _run(worker, world, backend, *args):
    import torch.multiprocessing as mp
    if backend == "nccl" and torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    ret = ctx.Queue()
    procs = [ctx.Process(target=worker, args=(r, world, port, ret, backend) + args) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(600)
        assert p.exitcode == 0
    assert ret.get(timeout=5) == 1


def _rows(n, lo, hi, chunks, dev):
    return torch.cat([torch.arange(c * n + lo, c * n + hi) for c in range(chunks)]).to(dev)


# ------------------------------------------------------------------------------------------------ attention + warp_tensor
def _layer_worker(rank, world, port, ret, backend, N):
    dev = _init(rank, world, port, backend)
    from fresco_b200 import diffusion_hacked as dh
    from fresco_b200 import flow_utils as fu
    from fresco_b200.dist import ShardedFRESCOAttention, frame_range
    from oracle import fresco_oracle as O
    from test_gpu_parity_r2 import _trajectory_case
    lo, hi = frame_range(N, world, rank)
    ok = True
    # level-A FRESCO layer: [2N, 1024, 640], 8 heads (d = 80); 1024 trajectories do not split evenly over 3 ranks
    L, heads, C, chunks = 1024, 8, 640, 2
    g = torch.Generator().manual_seed(N * 7 + L)
    q, k, v, rq, rk = (torch.randn(chunks * N, L, C, generator=g).half().to(dev) for _ in range(5))
    mask = torch.rand(N, L, generator=g) > 0.6
    mask[0] = True
    fwd, tmask = _trajectory_case(N, L, seed=3)
    paras = {"fwd_mappings": [fwd[:, None].to(dev)], "bwd_mappings": [torch.argsort(fwd, 1)[:, None].to(dev)],
             "interattn_masks": [tmask[:, None].to(dev)]}
    sel = _rows(N, lo, hi, chunks, dev)
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
        mine = ShardedFRESCOAttention(ctrl, world, rank, chunks)(q[sel].contiguous(), k[sel].contiguous(), v[sel].contiguous(),
                                                                 heads, ref_q=rq[sel].contiguous(), ref_k=rk[sel].contiguous())
        if not torch.equal(mine, full[sel]):
            print("rank %d: attention flags %d differs: max |d| = %g"
                  % (rank, flags, (mine.float() - full[sel].float()).abs().max().item()), flush=True)
            ok = False
    # warp_tensor: a level-B decoder feature (640 channels: re-shard by channel on 2 ranks, gather on 3) and a decoded
    # 512^2 image batch (3 channels: gather path, dilation and per-step chain kernels)
    flows, occs = O.synth_flows(N, 512, 512, seed=5, mag=12.0)
    flows, occs = [f.to(dev) for f in flows], [o.to(dev) for o in occs]
    sal = torch.rand(N, 1, 512, 512, generator=torch.Generator().manual_seed(2)).to(dev)
    for chunks, shape, dtype in ((2, (640, 64, 64), torch.float16), (1, (3, 512, 512), torch.float32)):
        x = torch.randn((chunks * N,) + shape, generator=torch.Generator().manual_seed(3)).to(dtype).to(dev)
        sel = _rows(N, lo, hi, chunks, dev)
        full = fu.warp_tensor(x, flows, occs, sal, chunks)
        mine = fu.warp_tensor(x[sel].contiguous(), flows, occs, sal, chunks, shard=(world, rank, None))
        if not torch.equal(mine, full[sel]):
            print("rank %d: warp_tensor %s differs" % (rank, (chunks * N,) + shape), flush=True)
            ok = False
    _finish(rank, ok, ret, dev)


@pytest.mark.parametrize("backend", ["gloo", "nccl"])
@pytest.mark.parametrize("N,world", [(7, 2), (5, 3)])
def test_sharded_layer_uneven_bit_identical(fb, N, world, backend):
    """ShardedFRESCOAttention (all guidance flags) and warp_tensor on uneven frame blocks == unsharded, bit for bit.
    gloo: the ranks share one GPU; nccl: one GPU per rank, skipped on a box with fewer."""
    _run(_layer_worker, world, backend, N)


def _inference_worker(rank, world, port, ret, backend, N):
    dev = _init(rank, world, port, backend)
    from fresco_b200 import pipe_FRESCO as pf
    from fresco_b200.dist import frame_range
    from oracle import fresco_oracle as O
    from test_dist_cpu import _Ctrl
    from test_gpu_dist_batch import _GPUStubPipe
    lo, hi = frame_range(N, world, rank)
    res = 512
    ac = torch.from_numpy(np.load(os.path.join(ROOT, "tests", "golden", "ddpm_step.npz"))["alphas_cumprod"])
    g = torch.Generator().manual_seed(1)
    imgs = (torch.rand(N, 3, res, res, generator=g) * 2 - 1).half().to(dev)
    pe = torch.randn(2 * N, 5, 8, generator=g).half().to(dev)
    flows, occs = O.synth_flows(N, res, res, seed=9, mag=12.0)
    flows, occs = [f.to(dev) for f in flows], [o.to(dev) for o in occs]
    sal = (torch.rand(N, 1, res, res, generator=g) > 0.4).float().to(dev)
    timesteps = [950 - 50 * i for i in range(20)]
    ok = True
    rec_full, rec_sh = [], []
    for propagation in (False, True):
        kw = dict(num_warmup_steps=14, use_controlnet=False, seed=3, repeat_noise=True, bg_smoothing_steps=[16, 17],
                  propagation_mode=propagation, flows=flows, occs=occs, saliency=sal)
        full = pf.inference(_GPUStubPipe(ac, dev), None, _Ctrl, imgs, pe, None, timesteps, record_latents=rec_full, **kw)
        mine = pf.inference(_GPUStubPipe(ac, dev), None, _Ctrl, imgs, pe, None, timesteps, record_latents=rec_sh,
                            shard=(world, rank, None), **kw)
        same = bool(torch.equal(mine, full[lo:hi])) and len(rec_full) == len(rec_sh)
        same = same and all(bool(torch.equal(a, b)) for a, b in zip(rec_full, rec_sh))
        if not same:
            print("rank %d: sharded inference differs (propagation=%s)" % (rank, propagation), flush=True)
        ok = ok and same
    _finish(rank, ok, ret, dev)


@pytest.mark.parametrize("backend", ["gloo", "nccl"])
def test_sharded_inference_uneven_bit_identical(fb, backend):
    """inference with background smoothing at 512^2 on frame blocks of 3 and 2 == unsharded, bit for bit"""
    _run(_inference_worker, 2, backend, 5)


# ------------------------------------------------------------------------------------------------ optimize_feature
@pytest.mark.parametrize("N,C,h,world", [(7, 640, 64, 2), (9, 1280, 32, 2), (15, 1280, 24, 3)])
def test_optimize_feature_ring_halo_uneven_bit_identical(fb, N, C, h, world):
    """optimize_feature (temporal + Gram-L1 terms, Adam, AdaIN) with the ranks as lock-step threads on one GPU: the
    ranks' outputs together are bit-identical to the unsharded call.  (9, 1280, 32) and (15, 1280, 24) are shapes where
    a rank's share of the weight rounded to fp32 gives another Gram loss scale than the unsharded call; the second is
    an even split."""
    from fresco_b200 import diffusion_hacked as dh
    from fresco_b200.dist import frame_range
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
            lo, hi = frame_range(N, world, rank)
            sel = _rows(N, lo, hi, 2, "cuda")
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
