"""Every way ``dist.shard_layout`` splits a keyframe batch over ranks, and every sharded entry point under each of them.

The pure tests enumerate the partition: ``frame_range``, the layouts of tuples and ``Box``es for G <= 8 and N <= 32
(and the one-rank layout of ``shard=None``), the fp32 Gram loss scale of every rank of every layout, and which ranks
hold the frames propagation mode restores.  The gloo tests run each entry point on the ranks of one layout, with
torch stand-ins for the kernels (``dist_harness``), and compare every rank's rows with the unsharded call on the whole
batch: bit for bit, except optimize_feature and the FRESCO layer against the torch oracle (1e-4: the stand-ins evaluate
in another order) and the harness-UNet pass of get_intraframe_paras (REL_TOL: the CPU UNet runs at another batch
size).  An idle rank of a Box must return empty results without touching its group or any collective."""
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist

from dist_harness import (ROOT, Ctrl, NoCollectives, NoGroups, NoisyVAE, StandInBackend, StubFlow,  # noqa: F401
                          StubPipe, StubVAE, TorchBackend, TorchOptBackend, Untouchable, finish, flow_paras_equal, frames, init,
                          rows, run)


# ------------------------------------------------------------------------------------------------ the partition
def test_frame_range_partition():
    from fresco_b200.dist import block_sizes, frame_range
    assert [frame_range(16, 4, r) for r in range(4)] == [(0, 4), (4, 8), (8, 12), (12, 16)]
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


def _fields(lay):
    return (lay.n_frames, lay.halves, lay.lo, lay.hi, lay.world, lay.rank, lay.group, lay.partner, lay.peers)


def test_shard_layout_of_tuples_enumerated():
    from fresco_b200.dist import frame_range, shard_layout
    for N in range(1, 33):
        one = shard_layout(N, None)                                 # the one-rank layout: everything, no exchange
        assert _fields(one) == _fields(shard_layout(N, (1, 0, None))) == (N, (0, 2), 0, N, 1, 0, None, None, [])
        assert not one.idle and one.ring() is None and one.trace_comm() is None
        assert (one.row_share, one.mean_frames) == (1.0, N)
    for G in range(1, 9):
        for N in range(1, 33):
            if N >= G:
                for r in range(G):
                    lay = shard_layout(N, (G, r, None))
                    assert (lay.lo, lay.hi) == frame_range(N, G, r) and lay.halves == (0, 2)
                    assert (lay.world, lay.rank, lay.group, lay.partner) == (G, r, None, None)
                    assert lay.mean_frames == N
                continue
            if G % 2 or 2 * N < G:
                with pytest.raises(ValueError, match="G <= 2N") as e:
                    shard_layout(N, (G, 0, NoGroups()))
                assert "process group of %d ranks" % N in str(e.value)
                continue
            owned = {}
            lays = [shard_layout(N, (G, r, NoGroups())) for r in range(G)]
            for r, lay in enumerate(lays):
                assert lay.split_halves and lay.halves == (r // (G // 2), r // (G // 2) + 1)
                assert (lay.world, lay.rank) == (G // 2, r % (G // 2))
                assert (lay.lo, lay.hi) == frame_range(N, G // 2, r % (G // 2))
                assert lay.group == ("half", (), lay.half) and lay.mean_frames == 2 * N
                partner = lays[lay.partner]
                assert partner.partner == r and partner.half == 1 - lay.half
                assert (partner.lo, partner.hi) == (lay.lo, lay.hi)                     # partners hold the same frames
                for f in range(lay.lo, lay.hi):
                    assert (lay.half, f) not in owned
                    owned[(lay.half, f)] = r
            assert sorted(owned) == [(h, f) for h in range(2) for f in range(N)]          # every sample exactly once
    with pytest.raises(ValueError, match="both"):
        shard_layout(3, (4, 0, NoGroups())).chunks(1)


def test_shard_layout_of_boxes_enumerated():
    from fresco_b200.dist import Box, frame_range, shard_layout
    for G in range(1, 9):
        for N in range(1, 33):
            lays = [shard_layout(N, Box(G, r, NoGroups())) for r in range(G)]       # never raises
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
                    want = shard_layout(N, (active, r, NoGroups(() if G <= 2 * N else ("active", active))))
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
        shard_layout(4, Box(7, 0, NoGroups())).chunks(1)
    with pytest.raises(ValueError, match="G <= 2N"):                              # the tuple still raises
        shard_layout(4, (7, 0, NoGroups()))


def _level_tokens():
    """L of the four SD decoder levels (latent / 8, / 4, / 2, / 1) for square frames 256..1024 in steps of 64 and for
    640 x 512"""
    sizes = [(r, r) for r in range(256, 1025, 64)] + [(640, 512)]
    return [(w // 8 // f) * (h // 8 // f) for w, h in sizes for f in (8, 4, 2, 1)]


def test_gram_loss_scale_of_every_layout_equals_unsharded():
    """Every rank's fp32 Gram loss scale equals the unsharded one: the unsharded launcher rounds fp32(intra_weight) /
    (2N L^2) once; a rank passes its share of the weight, intra_weight * row_share (optimize_feature), and ops divides
    it by its own batch in double before the one rounding.  Enumerated over the frame layouts (G <= 8, N <= 32), the
    half layouts and the unequal-halves layouts.  Rounding the share to fp32 first (the weight entry points) gives a
    different scale in some frame-layout cases."""
    from fresco_b200.dist import Box, shard_layout
    from fresco_b200.ops import _gram_scale
    f32 = np.float32
    frame = halves = unequal = rounded_share_differs = 0
    lays = []
    for N in range(1, 33):
        lays += [(shard_layout(N, (G, r, None)), "frame") for G in range(1, min(N, 8) + 1) for r in range(G)]
    for G in (2, 4, 6, 8):
        for N in range(G // 2, G):
            lays += [(shard_layout(N, (G, r, NoGroups())), "halves") for r in range(G)]
    for G in (3, 5, 7):
        for N in range((G + 1) // 2, G):
            lays += [(shard_layout(N, Box(G, r, NoGroups())), "unequal") for r in range(G)]
    for intra_weight in (1.0, 10.0, 50.0, 100.0, 200.0):
        for L in _level_tokens():
            for lay, kind in lays:
                N = lay.n_frames
                want = f32(float(f32(intra_weight)) / (2 * N * L * L))
                held = (lay.hi - lay.lo) * (lay.halves[1] - lay.halves[0])
                weight = intra_weight * lay.row_share                             # optimize_feature's share
                assert f32(_gram_scale(weight, held, L)) == want, (intra_weight, L, lay)
                if kind == "frame":
                    rounded_share_differs += f32(float(f32(weight)) / (held * L * L)) != want
                frame += kind == "frame"
                halves += kind == "halves"
                unequal += kind == "unequal"
    assert frame == 5 * len(_level_tokens()) * sum(G * (33 - G) for G in range(1, 9))
    assert halves > 0 and unequal > 0 and rounded_share_differs > 0


def test_box_propagation_frames_held_by_ranks_of_the_first_batch():
    """In propagation mode the ranks holding frame 0 or 1 of a later batch restore them from the first batch's
    record_latents, which only the first batch's active ranks hold.  With a first batch of at least 3 frames (the web
    UI's smallest) on up to 8 ranks, every such rank was active in it."""
    from fresco_b200.dist import Box, shard_layout
    for G in range(1, 9):
        for N0 in range(3, 17):
            active = [not shard_layout(N0, Box(G, r, NoGroups())).idle for r in range(G)]
            for N1 in range(3, 19):
                for r in range(G):
                    lay = shard_layout(N1, Box(G, r, NoGroups()))
                    if not lay.idle and lay.lo < 2:
                        assert active[r], (G, N0, N1, r)


# ------------------------------------------------------------------------------------------------ entry-point workers
# Each takes (N, lay, spec, rank) -- spec the shard argument the caller passes, lay its layout -- and returns the
# checks that failed.  Every rank computes the same unsharded result; one rank of the shard holds it to the oracle,
# every rank holds its own rows to it.

def _first(lay):
    return lay.rank == 0 and lay.halves[0] == 0


def _attention(N, lay, spec, rank):
    """the FRESCO layer at all 8 guidance flag combinations and the no-mask frame-0 broadcast: the rank's layer ==
    the world-1 layer on its rows, bit for bit, and that == the oracle; the processor builds its layer on the same
    ranks"""
    from fresco_b200 import diffusion_hacked as dh
    from fresco_b200.dist import ShardedFRESCOAttention
    from oracle import fresco_oracle as O
    torch.manual_seed(N)
    L, heads, C = 64, 2, 16
    x = torch.randn(2 * N, L, C)
    ref = torch.randn(2 * N, L, C)
    w = [torch.randn(C, C) * 0.3 for _ in range(4)]
    bo = torch.randn(C) * 0.1
    masks = [torch.rand(N, L) > 0.6]
    masks[0][0] = True
    masks[0][-1] = False                                  # a rank may select no row of its own frames
    perm = torch.stack([torch.randperm(L) for _ in range(N)])
    perm[0] = torch.arange(L)
    fm, bm = perm[:, None, :], torch.argsort(perm, dim=1)[:, None, :]
    im = (torch.rand(L, 1, N, N) > 0.3) | torch.eye(N, dtype=torch.bool)[None, None]
    sel = rows(N, lay)
    xl, rl = x[sel], ref[sel]
    proj = lambda t, i: t @ w[i].t()
    chunks = lay.chunks(2)
    proc = dh.FRESCOAttnProcessor2_0(2, dh.AttentionControl(), shard=spec)
    proc.set_batch_frames(N)
    bad = []
    if (proc._layout.halves, proc._layout.lo, proc._layout.hi) != (lay.halves, lay.lo, lay.hi):
        bad.append("processor layout %r" % proc._layout)
    if proc._layer_key != (lay.world, lay.rank, lay.group, chunks):
        bad.append("processor layer on %r" % (proc._layer_key,))
    for flags in range(8):
        cf, intra, inter = bool(flags & 1), bool(flags & 2), bool(flags & 4)
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
            if _first(lay) and not no_mask:
                want = O.fresco_attention(x, w[0], w[1], w[2], w[3], bo, heads, use_cfattn=cf, attn_masks=masks,
                                          use_intraattn=intra, ref_hidden=ref, use_interattn=inter, fwd_mappings=[fm],
                                          bwd_mappings=[bm], interattn_masks=[im])
                if (full @ w[3].t() + bo - want).abs().max().item() >= 1e-4:
                    bad.append("attention flags %d against the oracle" % flags)
    return bad


def _warp(N, lay, spec, rank, seed=0):
    """warp_tensor on decoder features of both CFG chunks (channels that re-shard by channel over the ranks or take
    the gather path), on a 3-channel feature, and on a decoded image batch of one chunk at image resolution (the
    dilated-occlusion path), in fp32 and fp16: the dtype kept, == the unsharded call bit for bit, == the oracle"""
    from fresco_b200 import flow_utils as fu
    from oracle import fresco_oracle as O
    from test_cpu_host import _TorchWarpOps
    fu.ops = _TorchWarpOps
    flows, occs = O.synth_flows(N, 64, 64, seed=5 + N + seed, mag=5.0)
    sal = torch.rand(N, 1, 32, 32, generator=torch.Generator().manual_seed(2))
    bad = []
    for chunks, C, h in ((2, 6, 8), (2, 4, 8), (2, 3, 16), (1, 3, 64)):
        for dtype in (torch.float32, torch.float16):
            g = torch.Generator().manual_seed(3 + h + C + seed)
            x = torch.randn(chunks * N, C, h, h, generator=g).to(dtype)
            sel = rows(N, lay) if chunks == 2 else torch.arange(lay.lo, lay.hi)
            full = fu.warp_tensor(x, flows, occs, sal, chunks)
            mine = fu.warp_tensor(x[sel].contiguous(), flows, occs, sal, chunks, shard=spec)
            if not (mine.dtype == dtype and torch.equal(mine, full[sel])):
                bad.append("warp_tensor chunks %d C %d h %d %s" % (chunks, C, h, dtype))
            tol = 1e-5 if dtype == torch.float32 else 1e-2
            if _first(lay) and (full.float() - O.warp_tensor(x.float(), flows, occs, sal, chunks)).abs().max().item() >= tol:
                bad.append("warp_tensor chunks %d C %d h %d %s against the oracle" % (chunks, C, h, dtype))
    return bad


# (N, seed) data on which the torch stand-ins and the oracle, two fp32 implementations of 6 sign-driven Adam steps,
# part ways with both losses on (SURVEY 9): a few dozen elements flip a sign, max |d| 4e-3 (N = 5) and 8e-3 (N = 4,
# seed 1).  The host loop is held to the oracle on every other data set.
_ORACLE_PARTS_WAYS = {(5, 0), (4, 1)}


def _optimize(N, lay, spec, rank, seed=0):
    """optimize_feature with both losses, each alone: the unsharded call == the oracle, every rank == its rows of the
    unsharded call, the loss curves summed over the ranks agree, and every temporal mean counts the unsharded call's
    2N samples; without flows a tuple counts the batch's frames with one all-reduce and a Box raises"""
    from fresco_b200 import diffusion_hacked as dh
    from fresco_b200.dist import Box
    from oracle import fresco_oracle as O
    chunks, C, h = 2, 6, 8
    flows, occs = O.synth_flows(N, 64, 64, seed=11 + seed, mag=5.0)
    g = torch.Generator().manual_seed(4 + seed)
    base = torch.randn(chunks, 1, C, h, h, generator=g)
    feat = (base + 0.5 * torch.randn(chunks, N, C, h, h, generator=g)).reshape(chunks * N, C, h, h)
    ref = feat + 0.3 * torch.randn(feat.shape, generator=g)
    X = ref.reshape(chunks * N, C, h * h).transpose(1, 2)
    Xh = X / (X ** 2).sum(2, keepdim=True) ** 0.5
    target = torch.bmm(Xh, Xh.transpose(1, 2))
    sel = rows(N, lay)
    be = TorchOptBackend(O)
    bad = []
    for temporal, spatial in ((True, True), (True, False), (False, True)):
        corr, corr_l = ([target], [target[sel]]) if spatial else ([], [])
        tr_full, tr_mine = dh.OptimizeTrace(), dh.OptimizeTrace()
        full = dh.optimize_feature(feat, flows, occs, corr, iters=6, optimize_temporal=temporal, trace=tr_full, backend=be)
        mine = dh.optimize_feature(feat[sel].contiguous(), flows, occs, corr_l, iters=6, optimize_temporal=temporal,
                                   trace=tr_mine, shard=spec, backend=be)
        if _first(lay) and (N, seed) not in _ORACLE_PARTS_WAYS:                 # the host loop itself against the oracle
            want = O.optimize_feature(feat, flows, occs, corr, iters=6, optimize_temporal=temporal)
            if (full - want).abs().max().item() >= 1e-4:
                bad.append("optimize_feature temporal %s spatial %s: unsharded against the oracle" % (temporal, spatial))
        # the stand-ins evaluate the open chain in another order than the ring
        if (mine - full[sel]).abs().max().item() >= 1e-4:
            bad.append("optimize_feature temporal %s spatial %s" % (temporal, spatial))
        if len(tr_full.losses) != 6 or not all(abs(a - b) < 1e-4 * abs(a) for a, b in zip(tr_full.losses, tr_mine.losses)):
            bad.append("optimize_feature loss curve temporal %s spatial %s" % (temporal, spatial))
    if not be.counts or set(be.counts) != {2 * N}:
        bad.append("temporal element counts %s, want %d" % (sorted(set(be.counts)), 2 * N))
    if isinstance(spec, Box):
        with pytest.raises(ValueError, match="flows"):                          # a Box takes N from the flows
            dh.optimize_feature(feat[sel].contiguous(), None, None, [target[sel]], iters=3, shard=spec, backend=be)
    else:
        full = dh.optimize_feature(feat, None, None, [target], iters=3, backend=be)
        mine = dh.optimize_feature(feat[sel].contiguous(), None, None, [target[sel]], iters=3, shard=spec, backend=be)
        if (mine - full[sel]).abs().max().item() >= 1e-4:
            bad.append("optimize_feature without flows")
    return bad


def _step_ops():
    """the torch stand-ins of the step and warp kernels installed; returns the scheduler's alphas_cumprod"""
    from fresco_b200 import flow_utils as fu
    from fresco_b200 import pipe_FRESCO as pf
    from test_cpu_host import _TorchStepOps, _TorchWarpOps
    pf.ops = _TorchStepOps
    fu.ops = _TorchWarpOps
    return torch.from_numpy(np.load(os.path.join(ROOT, "tests", "golden", "ddpm_step.npz"))["alphas_cumprod"])


def _step(N, lay, spec, rank):
    """step with guidance, with and without background smoothing, given the shard and given its layout"""
    from fresco_b200 import pipe_FRESCO as pf
    from fresco_b200.dist import shard_layout
    from oracle import fresco_oracle as O
    pipe = StubPipe(_step_ops())
    g = torch.Generator().manual_seed(6)
    eps = torch.randn(2 * N, 4, 8, 8, generator=g)
    x = torch.randn(N, 4, 8, 8, generator=g)
    noise = torch.randn(N, 4, 8, 8, generator=g)
    flows, occs = O.synth_flows(N, 64, 64, seed=9, mag=6.0)
    sal = (torch.rand(N, 1, 64, 64, generator=g) > 0.4).float()
    lo, hi = lay.lo, lay.hi
    eps_mine = eps[rows(N, lay)]
    bad = []
    for smooth in (False, True):
        kw = dict(flows=flows, occs=occs, saliency=sal) if smooth else {}
        full = pf.step(pipe, eps, 700, x, None, guidance_scale=7.5, noise=noise, **kw)
        for s in ([spec, shard_layout(N, spec)] if smooth else [shard_layout(N, spec)]):
            mine = pf.step(pipe, eps_mine, 700, x[lo:hi].contiguous(), None, guidance_scale=7.5,
                           noise=noise[lo:hi].contiguous(), shard=s, **kw)
            if not all(torch.equal(a, b[lo:hi]) for a, b in zip(mine, full)):
                bad.append("step smoothing %s shard %r" % (smooth, type(s).__name__))
    return bad


def _inference(N, lay, spec, rank):
    """inference with background smoothing, in first-batch and propagation mode, with and without repeat_noise: the
    rank's latents and record_latents == the unsharded call's, bit for bit; without smoothing too, and smoothing does
    change the result.  With the halves split, the two halves' ranks of the same frames agree under a VAE with unseeded
    posterior noise, and a layout that draws it on both halves is caught."""
    from fresco_b200 import pipe_FRESCO as pf
    from fresco_b200.dist import ShardLayout
    from oracle import fresco_oracle as O
    ac = _step_ops()
    g = torch.Generator().manual_seed(1)
    imgs = torch.rand(N, 3, 64, 64, generator=g)
    pe = torch.randn(2 * N, 5, 8, generator=g)
    flows, occs = O.synth_flows(N, 64, 64, seed=9, mag=6.0)
    sal = (torch.rand(N, 1, 64, 64, generator=g) > 0.4).float()
    timesteps = [950 - 50 * i for i in range(20)]
    bad = []
    for repeat in (False, True):
        rec_full, rec_sh = [], []
        for propagation in (False, True):
            # schedule steps 14..19: the background-smoothing steps 16 and 17 are loop steps 2 and 3
            kw = dict(num_warmup_steps=14, use_controlnet=False, seed=3, repeat_noise=repeat, bg_smoothing_steps=[16, 17],
                      propagation_mode=propagation, flows=flows, occs=occs, saliency=sal)
            full = pf.inference(StubPipe(ac), None, Ctrl, imgs, pe, None, timesteps, record_latents=rec_full, **kw)
            mine = pf.inference(StubPipe(ac), None, Ctrl, imgs, pe, None, timesteps, record_latents=rec_sh, shard=spec,
                                **kw)
            if not (torch.equal(mine, full[lay.lo:lay.hi]) and len(rec_full) == len(rec_sh)
                    and all(torch.equal(a, b) for a, b in zip(rec_full, rec_sh))):
                bad.append("inference repeat %s propagation %s" % (repeat, propagation))
            if not (repeat or propagation):
                kw["bg_smoothing_steps"] = []
                plain = pf.inference(StubPipe(ac), None, Ctrl, imgs, pe, None, timesteps, record_latents=[], **kw)
                plain_mine = pf.inference(StubPipe(ac), None, Ctrl, imgs, pe, None, timesteps, record_latents=[],
                                          shard=spec, **kw)
                if not torch.equal(plain_mine, plain[lay.lo:lay.hi]):
                    bad.append("inference without smoothing")
                if torch.equal(plain, full):
                    bad.append("smoothing changed nothing")
    if lay.split_halves:
        kw = dict(num_warmup_steps=14, use_controlnet=False, seed=3, bg_smoothing_steps=[16, 17], flows=flows, occs=occs,
                  saliency=sal)
        torch.manual_seed(100 + rank)
        out = pf.inference(StubPipe(ac, NoisyVAE), None, Ctrl, imgs, pe, None, timesteps, record_latents=[], shard=spec,
                           **kw)
        if not torch.equal(lay.swap(out), out):
            bad.append("the halves differ with a noisy VAE")
        real = ShardLayout.share
        ShardLayout.share = lambda self, make, like, chunks=1: make()
        try:
            out = pf.inference(StubPipe(ac, NoisyVAE), None, Ctrl, imgs, pe, None, timesteps, record_latents=[],
                               shard=spec, **kw)
        finally:
            ShardLayout.share = real
        if torch.equal(lay.swap(out), out):
            bad.append("a VAE sample drawn on both halves went unnoticed")
    return bad


def _flow(N, lay, spec, rank):
    """get_flow_and_interframe_paras with a per-pair stub flow model: flows, occlusions, K/V masks, mappings and
    trajectory masks == the unsharded call's, bit for bit; every pair computed once, on the ranks of half 0"""
    from fresco_b200 import diffusion_hacked as dh
    from fresco_b200 import flow_utils as fu
    from test_cpu_host import _TorchWarpOps
    fu.ops = _TorchWarpOps
    imgs = frames(N, 64, 64, seed=4)
    model = StubFlow()
    calls = []
    model.register_forward_pre_hook(lambda m, a: calls.append(a[0].shape[0]))
    full = dh.get_flow_and_interframe_paras(model, imgs)
    calls.clear()
    mine = dh.get_flow_and_interframe_paras(model, imgs, shard=spec)
    bad = [] if flow_paras_equal(mine, full) else ["get_flow_and_interframe_paras"]
    if not 0 < full[1][1].sum().item() < full[1][1].numel():                     # some, not all, pixels occluded
        bad.append("occlusions all or nothing")
    if calls != ([lay.hi - lay.lo] if lay.halves[0] == 0 else []):
        bad.append("flow model calls %s" % calls)
    return bad


# stored reference inputs, Gram targets and the guided step's output: the sharded and the unsharded UNet pass differ only
# in the batch size the fp32 CPU convolutions and GEMMs see, so in the last bits (at one rank, exactly 0).  The FRESCO
# processor rounds q / k / v and the attention outputs to fp16, as the kernels do, and a last-bit difference can move
# one of those roundings.  Bound: 1e-4 of the tensor's largest magnitude, a fifth of an fp16 ulp (observed: at most
# 3.1e-5 at world 2).
REL_TOL = 1e-4


def _close(a, b):
    return a.shape == b.shape and (a.float() - b.float()).abs().max().item() <= REL_TOL * max(b.float().abs().max().item(), 1.0)


def _intraframe(N, lay, spec, rank):
    """get_intraframe_paras on the CPU harness UNet: the latents entering the UNet are bit-identical to this rank's
    rows of the unsharded call's, the stored reference inputs and the Gram targets equal its slices to REL_TOL, the
    guidance flags are off again, and the sharded processor then runs a spatial-guided step on the stored references
    that matches the unsharded step to REL_TOL"""
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

    pipe.scheduler, pipe.vae, pipe._execution_device = Sched(torch.linspace(0.999, 0.01, 1000)), StubVAE(), torch.device("cpu")
    pipe.prepare_latents = lambda B, C, H, W, dtype, device, generator, latents=None: torch.randn(
        B, C, H // 8, W // 8, generator=generator, dtype=dtype)
    seen = []
    unet.register_forward_pre_hook(lambda m, a: seen.append(a[0].clone()))          # the latents entering the UNet
    g = torch.Generator().manual_seed(5)
    imgs = torch.rand(N, 3, 128, 128, generator=g) * 2 - 1
    pe = torch.randn(2 * N, 7, 24, generator=g)
    t = Sched.timesteps[-1]
    sel = rows(N, lay)

    proc = dh.apply_FRESCO_attn(pipe)
    corr_full = dh.get_intraframe_paras(pipe, imgs, proc, pe, seed=3)
    in_full = seen[-1]
    stored_full = list(proc.controller.stored_attn["decoder_attn"])
    proc.controller.enable_intraattn()
    out_full = pipe.unet(in_full, t, encoder_hidden_states=pe, return_dict=False)[0]

    proc = dh.apply_FRESCO_attn(pipe, shard=spec)
    proc.set_batch_frames(N)
    world, rk, group, chunks = proc._layer_key
    proc._sharded = ShardedFRESCOAttention(proc.controller, world, rk, chunks, group, backend=StandInBackend())
    corr = dh.get_intraframe_paras(pipe, imgs, proc, pe, seed=3, shard=spec)
    ctrl = proc.controller
    bad = []
    if ctrl.store or ctrl.use_intraattn or ctrl.use_cfattn or ctrl.use_interattn:
        bad.append("guidance flags left on")
    if not torch.equal(seen[-1], in_full[sel]):                                      # same noise, same encoded frames
        bad.append("get_intraframe_paras UNet input")
    stored = ctrl.stored_attn["decoder_attn"]
    if not (len(stored) == len(stored_full) == 6 and all(_close(a, b[sel]) for a, b in zip(stored, stored_full))):
        bad.append("get_intraframe_paras stored references")
    if not (len(corr) == len(corr_full) == 4 and all(_close(a, b[sel]) for a, b in zip(corr, corr_full))):
        bad.append("get_intraframe_paras targets")
    ctrl.enable_intraattn()
    out = pipe.unet(seen[-1], t, encoder_hidden_states=pe[sel], return_dict=False)[0]
    if not _close(out, out_full[sel]):
        bad.append("spatial-guided step on the stored references")
    return bad


def _misuse(N, lay, spec, rank):
    """a batch without classifier-free guidance cannot shard over its halves: ValueError on every rank, before any
    collective (the groups exist already: they were created by the calls before)"""
    from fresco_b200 import diffusion_hacked as dh
    from fresco_b200 import pipe_FRESCO as pf
    from oracle import fresco_oracle as O
    pipe = StubPipe(_step_ops())
    flows, occs = O.synth_flows(N, 64, 64, seed=9, mag=6.0)
    n = lay.hi - lay.lo
    calls = {
        "inference": lambda: pf.inference(pipe, None, Ctrl, torch.rand(N, 3, 64, 64), torch.randn(N, 5, 8), None,
                                          [950 - 50 * i for i in range(20)], num_warmup_steps=14, use_controlnet=False,
                                          do_classifier_free_guidance=False, record_latents=[], shard=spec),
        "step": lambda: pf.step(pipe, torch.randn(n, 4, 8, 8), 700, torch.randn(n, 4, 8, 8), None, shard=lay),
        "optimize_feature": lambda: dh.optimize_feature(torch.randn(n, 6, 8, 8), flows, occs, [], iters=2,
                                                        unet_chunk_size=1, shard=spec, backend=TorchOptBackend(O)),
    }
    bad = []
    with NoCollectives():
        for name, call in calls.items():
            try:
                call()
                bad.append("%s without guidance did not raise" % name)
            except ValueError:
                pass
    return bad


def _idle(N, world, rank):
    """every entry point on an idle rank of a Box, its group and every collective failing on use"""
    from fresco_b200 import diffusion_hacked as dh
    from fresco_b200 import flow_utils as fu
    from fresco_b200 import pipe_FRESCO as pf
    from fresco_b200.dist import Box, shard_layout
    from fresco_b200.harness.sd15_unet import FakePipe, SD15UNet
    from oracle import fresco_oracle as O
    box = Box(world, rank, Untouchable())
    ac = _step_ops()
    flows, occs = O.synth_flows(N, 64, 64, seed=9, mag=6.0)
    sal = torch.ones(N, 1, 64, 64)
    pe = torch.randn(2 * N, 5, 8)
    bad = []
    with NoCollectives():
        lay = shard_layout(N, box)
        if not lay.idle:
            return ["rank %d not idle: %r" % (rank, lay)]
        fl, oc, masks, paras = dh.get_flow_and_interframe_paras(StubFlow(), frames(N, 64, 64, seed=4), shard=box)
        if fl[0].shape[0] or oc[0].shape[0] or masks or paras["fwd_mappings"]:
            bad.append("get_flow_and_interframe_paras returned frames")
        unet_pipe = FakePipe(SD15UNet(block_out=(32, 64, 128, 128), heads=8, cross_dim=24))
        unet_pipe.vae, unet_pipe._execution_device = StubVAE(), torch.device("cpu")
        proc = dh.apply_FRESCO_attn(unet_pipe, shard=box)
        if dh.get_intraframe_paras(unet_pipe, torch.rand(N, 3, 64, 64), proc, pe, shard=box) != []:
            bad.append("get_intraframe_paras returned targets")
        dh.apply_FRESCO_opt(unet_pipe, steps=[700], flows=flows, occs=occs, saliency=sal, shard=box)
        none = torch.empty(0, 6, 8, 8)
        if dh.optimize_feature(none, flows, occs, [], shard=box) is not none:
            bad.append("optimize_feature")
        if fu.warp_tensor(none, flows, occs, sal, 2, shard=box) is not none:
            bad.append("warp_tensor")
        pipe = StubPipe(ac)
        x = torch.empty(0, 4, 8, 8)
        if pf.step(pipe, x, 700, x, None, guidance_scale=7.5, flows=flows, occs=occs, saliency=sal, shard=box)[0] is not x:
            bad.append("step")
        rec = []
        out = pf.inference(pipe, None, Ctrl, torch.rand(N, 3, 64, 64), pe, None, [950 - 50 * i for i in range(20)],
                           num_warmup_steps=14, use_controlnet=False, record_latents=rec, flows=flows, occs=occs,
                           saliency=sal, shard=box)
        if tuple(out.shape) != (0, 4, 8, 8) or rec:
            bad.append("inference returned %s" % (tuple(out.shape),))
    return bad


def _layout_worker(rank, world, port, ret, kind, N, parts):
    init(rank, world, port)
    from fresco_b200.dist import Box, shard_layout
    spec = Box(world, rank) if kind == "box" else (world, rank, None)
    if kind == "box" and rank >= 2 * N:
        bad = _idle(N, world, rank)
    else:
        lay = shard_layout(N, spec)
        bad = [b for part in parts for b in globals()[part](N, lay, spec, rank)]
    for b in bad:
        print("rank %d of %d, %s N %d: %s" % (rank, world, kind, N, b), flush=True)
    finish(rank, not bad, ret)


_ALL = ("_attention", "_warp", "_optimize", "_step", "_inference", "_flow", "_intraframe")
_BOX = ("_attention", "_warp", "_optimize", "_step", "_inference", "_flow")
# (shard kind, N, world): the entry points run.  Tuples: the frame layout at even and uneven blocks (one frame per rank
# at (4, 4)) and the half layout (G even, G/2 <= N < G); Boxes: the frame, unequal-halves and idle layouts at worlds 3,
# 5, 7 and the half layout with idle ranks at 8.
LAYOUTS = {
    ("tuple", 4, 2): _ALL,
    ("tuple", 4, 4): ("_warp", "_optimize", "_inference", "_flow", "_intraframe"),
    ("tuple", 5, 2): ("_attention", "_warp", "_inference", "_flow", "_intraframe"),
    ("tuple", 7, 2): ("_attention", "_warp", "_optimize", "_inference", "_flow"),
    ("tuple", 5, 3): ("_inference", "_flow"),
    ("tuple", 7, 3): ("_attention", "_warp", "_inference", "_flow", "_intraframe"),
    ("tuple", 6, 3): ("_optimize",),
    ("tuple", 5, 4): ("_attention",),
    ("tuple", 3, 4): _ALL,
    ("tuple", 2, 4): ("_attention", "_warp", "_optimize"),
    ("tuple", 3, 6): ("_attention", "_flow"),
    ("tuple", 5, 8): ("_attention", "_warp", "_optimize", "_inference", "_flow"),
    ("tuple", 7, 8): ("_attention", "_warp"),
    ("box", 2, 3): _BOX + ("_intraframe", "_misuse"),
    ("box", 3, 3): _BOX,
    ("box", 4, 3): _BOX,
    ("box", 6, 3): _BOX,
    ("box", 2, 5): _BOX,
    ("box", 3, 5): _BOX,
    ("box", 4, 5): _BOX,
    ("box", 6, 5): _BOX,
    ("box", 2, 7): _BOX,
    ("box", 3, 7): _BOX + ("_intraframe",),
    ("box", 4, 7): _BOX + ("_misuse",),
    ("box", 6, 7): _BOX,
    ("box", 3, 8): _BOX,
}


@pytest.mark.parametrize("kind,N,world", list(LAYOUTS), ids=["%s-%d-%d" % k for k in LAYOUTS])
def test_layout_matches_unsharded_gloo(kind, N, world):
    """Every entry point LAYOUTS lists for the shard kind, N and world, each rank on its rows against the unsharded
    call on the whole batch (the workers above say what each checks).  Box ranks beyond 2N are idle and must not touch
    a group or collective; a Box without guidance raises on every rank before any collective."""
    run(_layout_worker, world, kind, N, LAYOUTS[(kind, N, world)], timeout=900)


# ------------------------------------------------------------------------------------------------ shards on sub-groups
def _two_batches_worker(rank, world, port, ret, parts):
    """two sharded batches side by side, on process groups {0,1} and {2,3} of a world of 4, each with its own data:
    the second group does not contain global rank 0, so every peer has to be addressed through the group"""
    init(rank, world, port)
    from fresco_b200.dist import shard_layout
    groups = [dist.new_group([0, 1]), dist.new_group([2, 3])]
    batch = rank // 2
    spec = (2, rank % 2, groups[batch])
    lay = shard_layout(4, spec)
    bad = [b for part in parts for b in globals()[part](4, lay, spec, rank, seed=batch)]
    for b in bad:
        print("rank %d, batch %d: %s" % (rank, batch, b), flush=True)
    finish(rank, not bad, ret)


@pytest.mark.parametrize("parts", [("_optimize",), ("_warp",)], ids=["optimize", "warp"])
def test_two_batches_on_subgroups_gloo(parts):
    run(_two_batches_worker, 4, parts)


def _half_subgroup_worker(rank, world, port, ret, N, G, parts):
    """a shard on the process group of ranks 1..G of the world; ranks 0 and G+1.. take no part after creating it"""
    init(rank, world, port)
    from fresco_b200 import dist as fd
    members = list(range(1, G + 1))
    bad = []
    for attempt in range(2):                     # the second shard group object over the same ranks finds the cache
        group = dist.new_group(members)
        if rank in members:
            spec = (G, rank - 1, group)
            lay = fd.shard_layout(N, spec)
            if not lay.split_halves or lay.partner != 1 + (lay.rank + (1 - lay.half) * (G // 2)):
                bad.append("layout %r" % lay)
            for part in parts if attempt == 0 else ("_attention",):
                bad += globals()[part](N, lay, spec, rank)
    if rank in members and len(fd._HALF_GROUPS) != 1:
        bad.append("%d half groups cached" % len(fd._HALF_GROUPS))
    for b in bad:
        print("rank %d of %d, N %d on a sub-group of %d: %s" % (rank, world, N, G, b), flush=True)
    finish(rank, not bad, ret)


def test_half_layout_on_a_shard_subgroup_gloo():
    """The half layout of a shard on a process sub-group (ranks 1..4 of 6): the half groups are created by the shard's
    ranks alone (ranks 0 and 5 never reach that point), the exchanges and partner transfers address global ranks
    through the group, and a second group object over the same ranks reuses the cached half groups."""
    run(_half_subgroup_worker, 6, 3, 4, ("_attention", "_optimize", "_inference"))
