"""GPU tests of keyframe batches with fewer frames than ranks, sharded over the two CFG halves (``dist.shard_layout``),
with the real kernels: every rank's rows must equal the unsharded call bit for bit.  The FRESCO layer runs in processes
sharing one GPU over gloo (and one GPU each over NCCL when the box has enough), the ring-halo feature optimisation in
threads in lock step, and one harness-UNet denoise step in processes sharing one GPU (and over NCCL), which matches
to the round-off of the UNet body at another batch size (REL_TOL)."""
import os
import threading

import numpy as np
import pytest
import torch

from dist_harness import ROOT, fb, finish, gpu_layer, gpu_warp, init, rows, run  # noqa: F401

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------ the FRESCO layer
def _layer_worker(rank, world, port, ret, backend, N):
    dev = init(rank, world, port, backend)
    from fresco_b200.dist import shard_layout
    shard = (world, rank, None)
    lay = shard_layout(N, shard)
    bad = ([] if lay.split_halves else ["layout %r" % lay]) + gpu_layer(N, lay, shard, dev) + gpu_warp(N, lay, shard, dev)
    for b in bad:
        print("rank %d: %s" % (rank, b), flush=True)
    finish(rank, not bad, ret, dev)


@pytest.mark.parametrize("backend", ["gloo", "nccl"])
def test_sharded_layer_half_layout_bit_identical(fb, backend):
    """ShardedFRESCOAttention (all guidance flags) and warp_tensor at N = 3 on 4 ranks: rank r holds CFG half r // 2 of
    frames frame_range(3, 2, r % 2); == unsharded, bit for bit.  gloo: the ranks share one GPU; nccl: one GPU each,
    skipped on a box with fewer than 4."""
    run(_layer_worker, 4, backend, 3, gpus=4 if backend == "nccl" else 0)


# ------------------------------------------------------------------------------------------------ optimize_feature
class _HalvesRing:
    """Communicators for `world` ranks emulated by threads of one process on one GPU, in lock step as
    test_gpu_parity_r2's _LockstepRing: the whole shard (loss trace, frame count) and each CFG half's ring."""

    class _Group:
        def __init__(self, ring, size):
            self.ring, self.size = ring, size
            self.barrier = threading.Barrier(size)
            self.slots = [None] * size

    class _Comm:
        def __init__(self, ring, group, index):
            self.ring, self.group, self.index = ring, group, index

        def _sync(self):
            self.ring.lock.release()
            self.group.barrier.wait()
            self.ring.lock.acquire()

        def shift(self, send, recv, direction):
            self.group.slots[self.index] = send
            self._sync()
            recv.copy_(self.group.slots[(self.index - direction) % self.group.size])
            self._sync()

        def all_reduce_sum(self, t):
            self.group.slots[self.index] = t.clone()
            self._sync()
            total = sum(self.group.slots[1:], self.group.slots[0].clone())
            self._sync()
            t.copy_(total)

        def half_comm(self, world, rank):
            per = world // 2
            return _HalvesRing._Comm(self.ring, self.ring.halves[rank // per], rank % per)

    def __init__(self, world):
        self.lock = threading.Lock()
        self.full = self._Group(self, world)
        self.halves = [self._Group(self, world // 2) for _ in range(2)]
        self.barriers = [self.full.barrier] + [h.barrier for h in self.halves]

    def comm(self, rank):
        return self._Comm(self, self.full, rank)


@pytest.mark.parametrize("N,world,C,h", [(3, 4, 640, 64), (5, 8, 1280, 32), (7, 8, 1280, 16)])
def test_optimize_feature_half_layout_bit_identical(fb, N, world, C, h):
    """optimize_feature (temporal + Gram-L1 terms, Adam, AdaIN) in the half layout, the ranks as lock-step threads on
    one GPU: every rank's output equals its rows of the unsharded call bit for bit, and the loss curve summed over the
    ranks matches (up to the order of the kernels' atomic adds)."""
    from fresco_b200 import diffusion_hacked as dh
    from fresco_b200.dist import shard_layout
    from test_gpu_parity_r2 import _layer_case
    flows, occs, cs = _layer_case(N, C, h, seed=31 + h)
    flows = [f.cuda() for f in flows]
    occs = [o.cuda() for o in occs]
    sample = cs.reshape(2 * N, C, h, h).half().cuda()
    g = torch.Generator(device="cuda").manual_seed(5)
    ref = (sample.float() + 0.5 * torch.randn(sample.shape, device="cuda", generator=g)).half()
    target = dh.gram_targets([ref])[0]
    tr_full = dh.OptimizeTrace()
    full = dh.optimize_feature(sample, flows, occs, correlation_matrix=[target], iters=6, trace=tr_full)
    ring = _HalvesRing(world)
    outs, traces, errs = [None] * world, [None] * world, []

    def run(rank):
        ring.lock.acquire()
        try:
            comm = ring.comm(rank)
            lay = shard_layout(N, (world, rank, comm))
            sel = rows(N, lay, "cuda")
            tgt = dh.GramTarget(target.yhat[sel].contiguous())
            tr = dh.OptimizeTrace()
            outs[rank] = (sel, dh.optimize_feature(sample[sel].contiguous(), flows, occs, correlation_matrix=[tgt],
                                                   iters=6, trace=tr, shard=(world, rank, comm)))
            traces[rank] = tr.losses
        except Exception as e:                                  # noqa: BLE001 (reported below; a dead rank must not hang the others)
            errs.append(e)
            for b in ring.barriers:
                b.abort()
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
        assert all(abs(a - b) <= 1e-5 * abs(a) for a, b in zip(tr_full.losses, traces[rank])), (tr_full.losses, traces[rank])


# ------------------------------------------------------------------------------------------------ one denoise step
def _step_worker(rank, world, port, ret, backend, N):
    dev = init(rank, world, port, backend)
    from fresco_b200 import diffusion_hacked as dh
    from fresco_b200 import flow_utils as fu
    from fresco_b200 import pipe_FRESCO as pf
    from fresco_b200.dist import shard_layout
    from fresco_b200.harness import synth
    from fresco_b200.harness.sd15_unet import FakePipe, SD15UNet
    from test_cpu_host import _Sched
    from test_gpu_gram_ragged import _VAE
    H = W = 256
    torch.manual_seed(0)
    pipe = FakePipe(SD15UNet().to(device=dev).eval())
    ac = torch.from_numpy(np.load(os.path.join(ROOT, "tests", "golden", "ddpm_step.npz"))["alphas_cumprod"])
    sched = _Sched(ac)
    sched.timesteps = torch.arange(950, -1, -50)
    pipe.scheduler, pipe.vae, pipe._execution_device = sched, _VAE(), dev
    pipe.prepare_latents = lambda B, C, h, w, dtype, device, generator, latents=None: torch.randn(
        B, C, h // 8, w // 8, generator=generator, dtype=dtype, device=device)
    imgs = synth.frames(N, H, W, dev, seed=H + W)
    pe = 0.5 * torch.randn(2 * N, 77, 768, generator=torch.Generator().manual_seed(4)).to(dev)
    flows, occs = synth.smooth_flows(N, H, W, dev, seed=H * W)
    attn_mask = dh.cross_frame_attn_masks(occs[1])
    fm, bm, im = [], [], []
    for s in (8.0, 16.0):
        f, b, m = fu.get_mapping_ind(flows[1], occs[1], imgs, scale=s)
        fm.append(f), bm.append(b), im.append(m)
    paras = {"fwd_mappings": fm, "bwd_mappings": bm, "interattn_masks": im}
    t = 700
    outs = []
    for shard in (None, (world, rank, None)):
        proc = dh.apply_FRESCO_attn(pipe, shard=shard)
        corr = dh.get_intraframe_paras(pipe, imgs, proc, pe, seed=3, shard=shard)
        # no feature optimisation here: its sign-driven Adam steps turn last-bit differences of the UNet body into
        # differences of the step size (test_optimize_feature_half_layout_bit_identical pins it bit for bit)
        dh.apply_FRESCO_opt(pipe, steps=[], shard=shard)
        proc.controller.enable_controller(interattn_paras=paras, attn_mask=attn_mask)
        outs.append(pf.inference(pipe, None, proc, imgs, pe, None, [t], num_warmup_steps=0, use_controlnet=False, seed=3,
                                 record_latents=[], step_interattn_end=0, shard=shard))
    lay = shard_layout(N, (world, rank, None))
    mine, want = outs[1].float(), outs[0][lay.lo:lay.hi].float()
    same_as_partner = bool(torch.equal(lay.swap(outs[1]), outs[1]))
    err, scale = (mine - want).abs().max().item(), want.abs().max().item()
    print("rank %d: max |sharded - unsharded| = %g of max |x| %g, partner bit-identical %s"
          % (rank, err, scale, same_as_partner), flush=True)
    ok = lay.split_halves and same_as_partner and err <= REL_TOL * scale
    finish(rank, ok, ret, dev)


# The harness UNet body is not batch-invariant on the GPU: cuBLAS / cuDNN pick other algorithms at batch n than at 2N
# (max |d| 1.4e-3 on its output at 256^2, the frame layout at batch 2n as much as the half layout at n), and FRESCO
# attention rounds q / k / v to fp16 after it.  So a whole denoise step matches the unsharded one to round-off, not
# bit for bit; everything after the UNet body (attention layers, the ring-halo optimisation, the guidance and DDPM
# kernels) is pinned bit for bit by the tests above.  Bound: 1e-2 of the latents' magnitude.
REL_TOL = 1e-2


@pytest.mark.parametrize("backend", ["gloo", "nccl"])
@pytest.mark.parametrize("N,world", [(2, 4), (3, 4), (3, 6), (4, 6), (5, 8), (7, 8)])
def test_harness_denoise_step_half_layout_bit_identical(fb, N, world, backend):
    """One denoise step of the harness UNet with every FRESCO flag on (intra-frame targets, cross-frame, spatial- and
    temporal-guided attention, apply_FRESCO_opt on all four decoder layers) in the half layout: the processor builds
    its one-half attention layer, the UNet runs on this rank's half, the partners swap their noise predictions and
    run the guidance and DDPM kernels.  Partners end with bit-identical latents, and every rank's latents equal its
    frames of the unsharded step to REL_TOL (the UNet body's batch-size round-off).
    gloo: the ranks share one GPU (point-to-point transfers staged through host memory); nccl: one GPU each, skipped
    on a box with fewer."""
    run(_step_worker, world, backend, N, gpus=world if backend == "nccl" else 0)
