"""What the multi-rank suites share (not a test module): spawning ranks and collecting their verdicts, this rank's rows
of a batch under a layout, and the stand-ins that let the sharded entry points run without the real networks --
torch backends for the kernels, a per-frame VAE / UNet / flow model, and groups and collectives that fail on use.

A worker is ``worker(rank, world, port, ret, *args)``; it calls ``init`` first and ``finish`` last.  CPU workers run
on gloo; GPU workers pass ``backend`` "gloo" (every rank on GPU 0, the exchanges through host memory) or "nccl" (one
GPU per rank)."""
import math
import os
import socket
import sys

import pytest
import torch
import torch.distributed as dist
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "tests")):
    if _p not in sys.path:
        sys.path.insert(0, _p)


# ------------------------------------------------------------------------------------------------ ranks as processes
def run(worker, world, *args, timeout=600, gpus=0):
    """spawn ``world`` ranks of ``worker`` and assert that every one of them passed; skipped on a box with fewer than
    ``gpus`` GPUs"""
    import torch.multiprocessing as mp
    if gpus and torch.cuda.device_count() < gpus:
        pytest.skip("needs %d GPUs" % gpus)
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


def init(rank, world, port, backend=None):
    """join the process group and return this rank's device: the CPU for ``backend=None`` (gloo), GPU 0 for "gloo",
    GPU ``rank`` for "nccl\""""
    for p in (ROOT, os.path.join(ROOT, "tests")):
        if p not in sys.path:
            sys.path.insert(0, p)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    if backend is None:
        torch.set_num_threads(max(1, (os.cpu_count() or 1) // world))        # the ranks share the host's cores
        dist.init_process_group("gloo", rank=rank, world_size=world)
        return torch.device("cpu")
    dev = torch.device("cuda", rank if backend == "nccl" else 0)
    torch.cuda.set_device(dev)
    if backend == "nccl":
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    else:
        dist.init_process_group("gloo", rank=rank, world_size=world)
    return dev


def finish(rank, ok, ret, dev="cpu"):
    """the AND of every rank's ``ok`` goes to the parent"""
    t = torch.tensor([1 if ok else 0], device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MIN)
    if rank == 0:
        ret.put(int(t.item()))
    dist.destroy_process_group()


@pytest.fixture(scope="module")
def fb():
    if not torch.cuda.is_available():
        pytest.skip("GPU tests need a CUDA device")
    from fresco_b200 import _lib
    _lib.lib()      # fails loudly if the extension is missing


def rows(N, lay, dev=None):
    """this rank's rows of a (chunk, frame)-major batch of both CFG chunks: frames [lo, hi) of each half it holds"""
    out = torch.cat([torch.arange(h * N + lay.lo, h * N + lay.hi) for h in range(*lay.halves)]).long()
    return out if dev is None else out.to(dev)


# ------------------------------------------------------------------------------------------------ kernel stand-ins
class TorchBackend:
    """torch stand-ins with the semantics of the C entry points (fresco_kv_compact_packed, fresco_rows_gather /
    _scatter, fresco_attn_fwd[_kv_strided], fresco_temporal_attn_fwd[_strided])"""

    def kv_compact_packed(self, k, v, idx, kv_out, chunks):
        B, L, C = k.shape
        n_rows = (B // chunks) * L
        n = idx.numel()
        kv_out[:, :n, :C] = k.reshape(chunks, n_rows, C)[:, idx.long()]
        kv_out[:, :n, C:] = v.reshape(chunks, n_rows, C)[:, idx.long()]
        kv_out[:, n:] = float("nan")                       # padding rows must never be read
        return kv_out

    def rows_gather(self, src, idx, dst, dst_col=0):
        dst[:, dst_col:dst_col + src.shape[-1]] = src[idx.long()]
        return dst

    def rows_scatter(self, src, idx, dst):
        dst[idx.long()] = src
        return dst

    def attn_fwd(self, q, k, v, heads, q_per_kv, softmax_scale, diag_bias=0.0):
        B, L, C = q.shape
        d = C // heads
        k = k.repeat_interleave(q_per_kv, 0)
        v = v.repeat_interleave(q_per_kv, 0)
        qh, kh, vh = (t.view(t.shape[0], -1, heads, d).transpose(1, 2) for t in (q, k, v))
        s = qh @ kh.transpose(-1, -2) * softmax_scale
        if diag_bias:
            s = s + torch.eye(L, kh.shape[2]) * diag_bias
        return (torch.softmax(s, -1) @ vh).transpose(1, 2).reshape(B, L, C)

    def attn_fwd_kv_packed(self, q, kv, heads, q_per_kv, softmax_scale):
        C = q.shape[-1]
        return self.attn_fwd(q, kv[..., :C].contiguous(), kv[..., C:].contiguous(), heads, q_per_kv, softmax_scale)

    def temporal_attn_fwd_packed(self, qkv, fwd_map, traj_mask, chunks, heads, scale):
        C = qkv.shape[-1] // 3
        return self.temporal_attn_fwd(qkv[..., :C].contiguous(), qkv[..., C:2 * C].contiguous(), qkv[..., 2 * C:].contiguous(),
                                      fwd_map, traj_mask, chunks, heads, scale)

    def temporal_attn_fwd(self, q, k, v, fwd_map, traj_mask, chunks, heads, scale):
        B, L, C = q.shape
        N = B // chunks
        d = C // heads
        gi = fwd_map[None, :, :, None, None].expand(chunks, N, L, heads, d)
        qt = torch.gather(q.view(chunks, N, L, heads, d), 2, gi)
        kt = torch.gather(k.view(chunks, N, L, heads, d), 2, gi)
        vt = torch.gather(v.view(chunks, N, L, heads, d), 2, gi)
        s = torch.einsum("bfphd,bgphd->bphfg", qt, kt) * scale
        s = s.masked_fill(~traj_mask.bool()[None, :, None], float("-inf"))
        o = torch.einsum("bphfg,bgphd->bfphd", torch.softmax(s, -1), vt)
        out = torch.empty_like(o)
        out.scatter_(2, gi, o)
        return out.reshape(B, L, C)


class StandInBackend:
    """the attention stand-in of test_cpu_host (fp32 math, fp16 results) behind ShardedFRESCOAttention's backend API"""

    def attn_fwd(self, q, k, v, heads, q_per_kv, softmax_scale, diag_bias=0.0):
        from test_cpu_host import _TorchOps
        return _TorchOps.attn_fwd(q, k, v, heads, q_per_kv, softmax_scale=softmax_scale, diag_bias=diag_bias)


class TorchOptBackend:
    """torch stand-ins for the compute steps of optimize_feature (fresco_warp_loss_fwd_bwd[_halo], the Gram-L1 kernels,
    fresco_adam_step, fresco_adain), written from the oracle's formulas.  ``counts`` records the temporal mean's
    element count (chunks * total_frames, times C*h*w) of every temporal evaluation."""

    def __init__(self, O):
        self.O = O
        self.counts = []

    def temporal_prepare(self, flows, occs, h, lo, hi, total):
        ff, bf, fo, bo = self.O._resize_flow_occ(flows, occs, h / flows[0].shape[2])
        return {"ff": ff[lo:hi], "bf": bf[lo:hi], "mf": (1 - fo)[lo:hi], "mb": (1 - bo)[lo:hi]}

    def temporal(self, cs, prep, grad, loss_acc, halo_cs=None, halo_grad=None, total_frames=None):
        O = self.O
        b, n, c, h, w = cs.shape
        total = n if total_frames is None else total_frames
        self.counts.append(b * total)
        rep = lambda t: t.repeat(b, 1, 1, 1)
        ff, bf, mf, mb = rep(prep["ff"]), rep(prep["bf"]), rep(prep["mf"]), rep(prep["mb"])
        if halo_cs is None:
            # the closed ring of this call's frames, averaged over chunks * total frames (the oracle averages over its own)
            loss, g = O.temporal_loss_and_grad(cs, ff, bf, mf, mb)
            loss, g = loss * (n / total), g * (n / total)
        else:
            ext = torch.cat([cs, halo_cs[:, None]], 1)
            c1 = ext[:, :n].reshape(b * n, c, h, w)
            c2 = ext[:, 1:].reshape(b * n, c, h, w)
            r1 = c2 - O.flow_warp(c1, bf)
            r2 = c1 - O.flow_warp(c2, ff)
            k = 2.0 / (b * total * c * h * w)
            loss = ((r1 * mb).abs() + (r2 * mf).abs()).sum() * k
            s1, s2 = torch.sign(r1) * mb * k, torch.sign(r2) * mf * k
            g = (s2 - O.flow_warp_adjoint(s1, bf)).view(b, n, c, h, w).clone()
            g2 = (s1 - O.flow_warp_adjoint(s2, ff)).view(b, n, c, h, w)
            g[:, 1:] += g2[:, :-1]
            halo_grad.copy_(g2[:, -1])
        grad.copy_(g)
        if loss_acc is not None:
            loss_acc += loss

    def spatial(self, cs_bcl, target, weight, grad_bcl, loss_acc):
        B, C, L = cs_bcl.shape
        loss, g = self.O.spatial_loss_and_grad(cs_bcl.reshape(1, B, C, L, 1), target, weight)
        grad_bcl += g.reshape(B, C, L)
        if loss_acc is not None:
            loss_acc += loss

    def adam(self, cs, grad, m, v, it):
        m.mul_(0.9).add_(grad, alpha=0.1)
        v.mul_(0.999).addcmul_(grad, grad, value=0.001)
        cs.sub_((0.2 / (1 - 0.9 ** it)) * m / (v.sqrt() / math.sqrt(1 - 0.999 ** it) + 1e-8))

    def adain(self, cs_bchw, sample):
        return self.O.adain(cs_bchw.to(sample.dtype), sample)


# ------------------------------------------------------------------------------------------------ network stand-ins
class StubVAE:
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


class NoisyVAE(StubVAE):
    """StubVAE whose posterior sample adds noise from the process's global generator, as a diffusers VAE does (and the
    reference leaves unseeded)"""

    def encode(self, x):
        d = super().encode(x)
        d.v = d.v + 0.1 * torch.randn(d.v.shape)
        return d


class StubUNet(torch.nn.Module):
    """per-frame 'UNet': every output frame depends on its own input frame only, like the real UNet body"""

    class config:
        in_channels = 4

    def __init__(self):
        super().__init__()
        self.dtype = torch.float32

    def forward(self, x, t, encoder_hidden_states=None, **kw):
        return (torch.tanh(x * 0.7 + 0.001 * float(t)) + 0.1 * encoder_hidden_states.mean((1, 2))[:, None, None, None],)


class StubPipe:
    def __init__(self, ac, vae=StubVAE):
        from test_cpu_host import _Sched
        self.scheduler = _Sched(ac)
        self.vae = vae()
        self.unet = StubUNet()
        self._execution_device = torch.device("cpu")

    def prepare_latents(self, B, C, H, W, dtype, device, generator, latents=None):
        return torch.randn(B, C, H // 8, W // 8, generator=generator, dtype=dtype)


class Ctrl:
    """the processor argument of inference when no FRESCO attention runs"""

    class controller:
        @staticmethod
        def disable_intraattn():
            pass

        @staticmethod
        def disable_interattn():
            pass


class StubFlow(torch.nn.Module):
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


def frames(n, h, w, seed):
    """n uint8 HxWx3 frames of one moving, smooth scene"""
    g = torch.Generator().manual_seed(seed)
    base = F.interpolate(torch.rand(1, 3, h // 8 + 4, w // 8 + 4, generator=g), size=(h + 32, w + 32), mode="bicubic")
    out = []
    for i in range(n):
        y, x = 2 * i, 3 * i
        f = base[0, :, y:y + h, x:x + w].clamp(0, 1) * 255
        out.append(f.permute(1, 2, 0).round().to(torch.uint8).numpy())
    return out


def flow_paras_equal(a, b):
    (fa, oa, ma, pa), (fb, ob, mb, pb) = a, b
    same = lambda x, y: len(x) == len(y) and all(torch.equal(u, v) for u, v in zip(x, y))
    return (same(fa, fb) and same(oa, ob) and same(ma, mb)
            and all(same(pa[k], pb[k]) for k in ("fwd_mappings", "bwd_mappings", "interattn_masks")))


# ------------------------------------------------------------------------------------------------ groups that fail on use
class NoGroups:
    """stands in for the shard's process group so layouts can be enumerated without creating groups"""

    def __init__(self, tag=()):
        self.tag = tag

    def __eq__(self, other):
        return isinstance(other, NoGroups) and other.tag == self.tag

    def __hash__(self):
        return hash(self.tag)

    def half_comm(self, world, rank):
        return ("half", self.tag, 0 if rank < world - world // 2 else 1)

    def sub_comm(self, active, rank):
        return NoGroups(("active", active))


class Untouchable:
    """an idle rank's process group: fails on any use"""

    def __getattr__(self, name):
        raise AssertionError("an idle rank used its process group (.%s)" % name)


COLLECTIVES = ("all_gather_into_tensor", "all_gather", "all_to_all_single", "all_reduce", "broadcast",
               "batch_isend_irecv", "isend", "irecv", "send", "recv", "barrier", "new_group", "split_group",
               "get_global_rank", "get_backend")


class NoCollectives:
    """replaces every collective and group call of torch.distributed by one that fails"""

    def __init__(self, names=COLLECTIVES):
        self.names = names

    def __enter__(self):
        self.saved = {n: getattr(dist, n) for n in self.names}
        for n in self.names:
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


# ------------------------------------------------------------------------------------------------ GPU workers
class GPUStubUNet(torch.nn.Module):
    """per-frame 'UNet' without reductions: every output frame depends on its own input frame and prompt only"""

    class config:
        in_channels = 4

    dtype = torch.float16

    def forward(self, x, t, encoder_hidden_states=None, **kw):
        return (torch.tanh(x * 0.7 + 0.001 * float(t)) + 0.1 * encoder_hidden_states[:, 0, 0].view(-1, 1, 1, 1),)


class GPUStubPipe:
    def __init__(self, ac, device):
        from test_cpu_host import _Sched
        self.scheduler = _Sched(ac)
        self.vae = StubVAE()
        self.unet = GPUStubUNet()
        self._execution_device = device

    def prepare_latents(self, B, C, H, W, dtype, device, generator, latents=None):
        return torch.randn(B, C, H // 8, W // 8, generator=generator, device=device, dtype=dtype)


def gpu_layer(N, lay, spec, dev):
    """the level-A FRESCO layer ([2N, 1024, 640], 8 heads: d = 80) at all 8 guidance flag combinations with the real
    kernels: this rank's layer == its rows of the one-GPU layer, bit for bit; the processor builds its layer on the
    same ranks.  Returns the checks that failed."""
    from fresco_b200 import diffusion_hacked as dh
    from fresco_b200.dist import ShardedFRESCOAttention
    from test_gpu_parity_r2 import _trajectory_case
    L, heads, C = 1024, 8, 640
    g = torch.Generator().manual_seed(N * 7 + L)
    q, k, v, rq, rk = (torch.randn(2 * N, L, C, generator=g).half().to(dev) for _ in range(5))
    mask = torch.rand(N, L, generator=g) > 0.6
    mask[0] = True
    fwd, tmask = _trajectory_case(N, L, seed=3)
    paras = {"fwd_mappings": [fwd[:, None].to(dev)], "bwd_mappings": [torch.argsort(fwd, 1)[:, None].to(dev)],
             "interattn_masks": [tmask[:, None].to(dev)]}
    chunks = lay.chunks(2)
    proc = dh.FRESCOAttnProcessor2_0(2, dh.AttentionControl(), shard=spec)
    proc.set_batch_frames(N)
    bad = [] if proc._layer_key == (lay.world, lay.rank, lay.group, chunks) else ["processor layer %r" % (proc._layer_key,)]
    sel = rows(N, lay, dev)
    for flags in range(8):
        ctrl = dh.AttentionControl()
        if flags & 2:
            ctrl.stored_attn["decoder_attn"] = [q]
            ctrl.enable_intraattn()
        if flags & 4:
            ctrl.enable_interattn(paras)
        if flags & 1:
            ctrl.enable_cfattn([mask.to(dev)])
        full = ShardedFRESCOAttention(ctrl, 1, 0, 2)(q, k, v, heads, ref_q=rq, ref_k=rk)
        mine = ShardedFRESCOAttention(ctrl, lay.world, lay.rank, chunks, lay.group)(
            q[sel].contiguous(), k[sel].contiguous(), v[sel].contiguous(), heads, ref_q=rq[sel].contiguous(),
            ref_k=rk[sel].contiguous())
        if not torch.equal(mine, full[sel]):
            bad.append("attention flags %d: max |d| = %g" % (flags, (mine.float() - full[sel].float()).abs().max().item()))
    return bad


def gpu_warp(N, lay, spec, dev):
    """warp_tensor with the real kernels: a level-B decoder feature (640 channels: re-shard by channel, or gather when
    they do not split over the ranks) and a decoded 512^2 image batch (3 channels: gather path, dilation and per-step
    chain kernels) == this rank's rows of the one-GPU call, bit for bit"""
    from fresco_b200 import flow_utils as fu
    from oracle import fresco_oracle as O
    flows, occs = O.synth_flows(N, 512, 512, seed=5, mag=12.0)
    flows, occs = [f.to(dev) for f in flows], [o.to(dev) for o in occs]
    sal = torch.rand(N, 1, 512, 512, generator=torch.Generator().manual_seed(2)).to(dev)
    bad = []
    for chunks, shape, dtype in ((2, (640, 64, 64), torch.float16), (1, (3, 512, 512), torch.float32)):
        x = torch.randn((chunks * N,) + shape, generator=torch.Generator().manual_seed(3)).to(dtype).to(dev)
        sel = rows(N, lay, dev) if chunks == 2 else torch.arange(lay.lo, lay.hi, device=dev)
        full = fu.warp_tensor(x, flows, occs, sal, chunks)
        mine = fu.warp_tensor(x[sel].contiguous(), flows, occs, sal, chunks, shard=spec)
        if not torch.equal(mine, full[sel]):
            bad.append("warp_tensor %s differs" % ((chunks * N,) + shape,))
    return bad


def gpu_inference(N, lay, spec, dev, repeats):
    """inference with background smoothing at 512^2 (fp16 latents and images, 3-channel frames gathered for the chain)
    with the real step, warp and dilation kernels, in first-batch and propagation mode: this rank's latents and
    record_latents == the one-GPU call's, bit for bit"""
    import numpy as np
    from fresco_b200 import pipe_FRESCO as pf
    from oracle import fresco_oracle as O
    res = 512
    ac = torch.from_numpy(np.load(os.path.join(ROOT, "tests", "golden", "ddpm_step.npz"))["alphas_cumprod"])
    g = torch.Generator().manual_seed(1)
    imgs = (torch.rand(N, 3, res, res, generator=g) * 2 - 1).half().to(dev)
    pe = torch.randn(2 * N, 5, 8, generator=g).half().to(dev)
    flows, occs = O.synth_flows(N, res, res, seed=9, mag=12.0)
    flows, occs = [f.to(dev) for f in flows], [o.to(dev) for o in occs]
    sal = (torch.rand(N, 1, res, res, generator=g) > 0.4).float().to(dev)
    timesteps = [950 - 50 * i for i in range(20)]
    bad = []
    for repeat in repeats:
        rec_full, rec_sh = [], []
        for propagation in (False, True):
            kw = dict(num_warmup_steps=14, use_controlnet=False, seed=3, repeat_noise=repeat, bg_smoothing_steps=[16, 17],
                      propagation_mode=propagation, flows=flows, occs=occs, saliency=sal)
            full = pf.inference(GPUStubPipe(ac, dev), None, Ctrl, imgs, pe, None, timesteps, record_latents=rec_full, **kw)
            mine = pf.inference(GPUStubPipe(ac, dev), None, Ctrl, imgs, pe, None, timesteps, record_latents=rec_sh,
                                shard=spec, **kw)
            same = bool(torch.equal(mine, full[lay.lo:lay.hi])) and len(rec_full) == len(rec_sh)
            if not (same and all(bool(torch.equal(a, b)) for a, b in zip(rec_full, rec_sh))):
                bad.append("inference differs (repeat_noise=%s, propagation=%s): max |d| = %g"
                           % (repeat, propagation, (mine.float() - full[lay.lo:lay.hi].float()).abs().max().item()))
    return bad
