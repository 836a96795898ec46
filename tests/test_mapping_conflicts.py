"""The pixel mapping's conflict resolution (M1: ``mapping_single_kernel`` in mapping.cu, ``O.single_mapping_ind``) on
inputs built to break it.

The reference walks the sources in ascending order; a source that lands on a target another source already holds
replaces it only when the holder's mse is strictly greater; targets nobody holds receive the sources that hold nothing,
both in ascending order.  The oracle restates that as a lexicographic arg-min of (fp32 mse, source) through ``lexsort``
and the kernel as a 64-bit ``atomicMin`` of (mse bits, source).  ``sequential_mapping`` below is the loop itself,
written out with the mse as ``((a - b) ** 2).mean()`` on CPU fp32 tensors.

CPU: the oracle's closed form equals the loop bit for bit on every family.  GPU (``-m gpu``): the kernel through the
C ABI (outputs prefilled with sentinels) and ``flow_utils.get_mapping_ind`` equal the oracle bit for bit on the same
families at scales 1, 2, 8 and 16, on square and non-square planes.

Families (built on the downsampled grid, every value constant over its s x s block so the downsampling is exact):
identity, shift (integer flows: edge rows unlinked), occluded (every pixel), occ-half (downsampled occlusion exactly
0.5 -- not occluded -- next to the fp32 neighbours of 0.5), collapse (every source onto one target with equal colours:
all mse tie and the smallest source must win), fp32-ties (candidates whose mse ties in fp32 but differs in fp64),
half (y + f exactly on k + 0.5 for even and odd k, and on -0.5, which rounds to -0 and is inside), edge (wy == H and
wx == W exactly, next to H - 1 and W - 1).
"""
import pytest
import torch
import torch.nn.functional as F

from oracle import fresco_oracle as O

FAMILIES = ("identity", "shift", "occluded", "occ-half", "collapse", "fp32-ties", "half", "edge")
SIZES = ((1, 1), (1, 7), (31, 33), (32, 32), (25, 41), (17, 241))     # L = 1, 7, 1023, 1024, 1025, 4097


def _up(x, s):
    """[..., H, W] -> [..., H s, W s], every value repeated over its s x s block."""
    return x.repeat_interleave(s, -2).repeat_interleave(s, -1) if s > 1 else x


def family(name, H, W, s, seed=0):
    """(bwd_flow [1, 2, Hs, Ws], bwd_occ [1, Hs, Ws], imgs [2, 3, Hs, Ws]) fp32 whose downsampled flow (in grid units),
    occlusion and colours are the family's."""
    g = torch.Generator().manual_seed(seed * 7919 + sum(map(ord, name)) + H * 131 + W)
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
    fy, fx = torch.zeros(H, W), torch.zeros(H, W)
    occ = torch.zeros(H, W)
    imgs = torch.rand(2, 3, H, W, generator=g) * 2 - 1
    if name == "identity":
        pass
    elif name == "shift":
        fy.fill_(2.0 if H > 2 else 0.0)
        fx.fill_(-3.0 if W > 3 else -1.0)
    elif name == "occluded":
        occ.fill_(1.0)
    elif name == "occ-half":
        pick = torch.randint(0, 3, (H, W), generator=g)
        half = torch.tensor(0.5)
        occ = torch.where(pick == 0, half, torch.where(pick == 1, torch.nextafter(half, torch.tensor(1.0)),
                                                        torch.nextafter(half, torch.tensor(0.0))))
        fy = torch.randint(-1, 2, (H, W), generator=g).float()
    elif name == "collapse":
        ty, tx = H // 2, W // 3
        fy, fx = ty - ys, tx - xs
        imgs = torch.full((2, 3, H, W), 0.25)
    elif name == "fp32-ties":
        # many sources per target; the source colours differ from the target's (0) by (1, e, 0) with e in {0, 2^-13,
        # 2^-14}: 1 + e^2 is 1 in fp32, so the fp32 mse ties where the fp64 mse does not
        fy = torch.randint(-1, 2, (H, W), generator=g).float()
        fx = torch.randint(-1, 2, (H, W), generator=g).float()
        e = torch.tensor([0.0, 2.0 ** -13, 2.0 ** -14])[torch.randint(0, 3, (H, W), generator=g)]
        imgs = torch.zeros(2, 3, H, W)
        imgs[1, 0] = 1.0
        imgs[1, 1] = e
    elif name == "half":
        # y + f on k + 1/2 (even and odd k) and on -1/2 in both axes, mixed with integer flows
        pick = torch.randint(0, 4, (H, W), generator=g)
        fy = torch.where(pick == 0, torch.tensor(0.5), torch.where(pick == 1, -0.5 - ys, torch.where(
            pick == 2, torch.tensor(-1.5), torch.zeros(H, W))))
        fx = torch.where(pick == 3, torch.tensor(0.5), torch.where(pick == 1, torch.tensor(1.5), -0.5 - xs * (pick == 0)))
    elif name == "edge":
        pick = torch.randint(0, 4, (H, W), generator=g)
        fy = torch.where(pick == 0, H - ys, torch.where(pick == 1, H - 1 - ys, torch.zeros(H, W)))
        fx = torch.where(pick == 2, W - xs, torch.where(pick == 3, W - 1 - xs, torch.zeros(H, W)))
    else:
        raise ValueError(name)
    flow = torch.stack([fx, fy])[None] * s          # (x, y) channels, in full-resolution pixels
    return _up(flow, s).contiguous(), _up(occ[None], s).contiguous(), _up(imgs, s).contiguous()


def _prepared(bwd_flow, bwd_occ, imgs, scale):
    """Downsampled grid, per-source target and validity, and the two frames' colours [2, 3, L] (the reference's
    preparation, flow_utils.py:72-82, as plain torch on the CPU)."""
    down = lambda x: F.interpolate(x, scale_factor=1.0 / scale, mode="bilinear")      # noqa: E731
    fl = down(bwd_flow)[0] / scale
    H, W = fl.shape[1:]
    keep = ~(down(bwd_occ[None]) > 0.5)[0, 0]
    cols = down(imgs).reshape(2, 3, H * W)
    gy = torch.arange(H).reshape(H, 1).expand(H, W)
    gx = torch.arange(W).reshape(1, W).expand(H, W)
    ty, tx = torch.round(gy + fl[1]), torch.round(gx + fl[0])
    ok = (ty >= 0) & (ty < H) & (tx >= 0) & (tx < W) & keep
    return H * W, (ty * W + tx).long().reshape(-1).tolist(), ok.reshape(-1).tolist(), cols


def sequential_mapping(bwd_flow, bwd_occ, imgs, scale):
    """The conflict loop, one source at a time."""
    L, target, ok, cols = _prepared(bwd_flow, bwd_occ, imgs, scale)
    holder = {}
    for src in range(L):
        if not ok[src]:
            continue
        t = target[src]
        if t not in holder:
            holder[t] = src
            continue
        want = cols[0, :, t]
        held = ((cols[1, :, holder[t]] - want) ** 2).mean()
        new = ((cols[1, :, src] - want) ** 2).mean()
        if held > new:                                      # strictly greater: the earlier source keeps a tie
            holder[t] = src
    winners = set(holder.values())
    spare = iter([u for u in range(L) if u not in winners])
    mapping = [holder[t] if t in holder else next(spare) for t in range(L)]
    return torch.tensor(mapping, dtype=torch.int64), torch.tensor([t not in holder for t in range(L)])


def _cases(scales):
    out = []
    for i, fam in enumerate(FAMILIES):
        for j, (H, W) in enumerate(SIZES):
            s = scales[(i + j) % len(scales)]
            out.append(pytest.param(fam, H, W, s, id=f"{fam}-{H}x{W}-s{s}"))
    return out


def _family_has_what_it_is_built_for(fam, d, s):
    L, target, ok, cols = _prepared(*d, s)
    if fam == "occluded":
        assert not any(ok)
    if fam == "collapse":
        assert len({t for t, v in zip(target, ok) if v}) <= 1
    if fam == "fp32-ties" and L > 100:
        c = cols.double()
        found = False
        for t in set(target):
            srcs = [u for u in range(L) if ok[u] and target[u] == t]
            m32 = {float(((cols[1, :, u] - cols[0, :, t]) ** 2).mean()) for u in srcs}
            m64 = {float(((c[1, :, u] - c[0, :, t]) ** 2).mean()) for u in srcs}
            if len(m32) < len(m64):
                found = True
                break
        assert found, "no fp32 tie that fp64 separates"


@pytest.mark.parametrize("fam,H,W,s", _cases((1, 2, 8)))
def test_closed_form_equals_the_sequential_loop(fam, H, W, s):
    d = family(fam, H, W, s)
    _family_has_what_it_is_built_for(fam, d, s)
    mp, unl = O.single_mapping_ind(*d, float(s))
    want_mp, want_unl = sequential_mapping(*d, float(s))
    assert torch.equal(unl, want_unl), f"{(unl != want_unl).sum().item()} unlinked flags differ"
    assert torch.equal(mp, want_mp), f"{(mp != want_mp).sum().item()} mappings differ"
    assert torch.equal(torch.sort(mp).values, torch.arange(H * W)), "not a permutation"


def test_half_family_lands_on_half_pixels():
    """The half family's downsampled y + f and x + f lie exactly on k + 1/2 for even and odd k and on -1/2."""
    H, W, s = 9, 11, 2
    flow, _, _ = family("half", H, W, s)
    fl = F.interpolate(flow, scale_factor=1.0 / s, mode="bilinear")[0] / s
    gy, gx = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    for c in (gy + fl[1], gx + fl[0]):
        frac = c[(c - c.floor()) == 0.5]
        assert (frac == -0.5).any() and (torch.floor(frac) % 2 == 0).any() and (torch.floor(frac) % 2 == 1).any()


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def fb():
    if not torch.cuda.is_available():
        pytest.skip("GPU tests need a CUDA device")
    from fresco_b200 import _lib, flow_utils
    _lib.lib()      # fails loudly if the extension is missing

    class NS:
        pass
    ns = NS()
    ns.lib, ns.c, ns.fu = _lib, _lib.lib(), flow_utils
    return ns


def _gpu_cases():
    out = []
    for i, fam in enumerate(FAMILIES):
        for j, (H, W) in enumerate(SIZES):
            for s in (1, 2, 8, 16):
                if (i + j + s) % 2 == 0 or H * W in (1024, 4097):
                    out.append(pytest.param(fam, H, W, s, id=f"{fam}-{H}x{W}-s{s}"))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("fam,H,W,s", _gpu_cases())
def test_kernel_equals_the_oracle(fb, fam, H, W, s):
    d = family(fam, H, W, s)
    want_mp, want_unl = O.single_mapping_ind(*d, float(s))
    flow, occ, imgs = (t.cuda() for t in d)
    L = H * W
    mapping = torch.full((L + 2,), -7, dtype=torch.int64, device="cuda")
    unlinked = torch.full((L + 2,), 7, dtype=torch.uint8, device="cuda")
    nbytes = int(fb.c.fresco_mapping_workspace_bytes(L))
    ws = torch.full((nbytes,), 0xA5, dtype=torch.uint8, device="cuda")        # the kernel initialises its workspace
    fb.lib.check(fb.c.fresco_mapping_single(flow.data_ptr(), occ.data_ptr(), imgs.data_ptr(), H * s, W * s, s,
                                            mapping[1:].data_ptr(), unlinked[1:].data_ptr(), ws.data_ptr(), nbytes,
                                            fb.lib.stream()), "fresco_mapping_single")
    assert fb.lib.last_kernel() == "mapping_single_kernel"
    mp, unl = mapping.cpu(), unlinked.cpu()
    assert mp[0] == -7 and mp[-1] == -7 and unl[0] == 7 and unl[-1] == 7, "a guard element was written"
    assert torch.equal(unl[1:-1].bool(), want_unl) and torch.equal(unl[1:-1] <= 1, torch.ones(L, dtype=torch.bool))
    assert torch.equal(mp[1:-1], want_mp), f"{(mp[1:-1] != want_mp).sum().item()} mappings differ"


@pytest.mark.gpu
@pytest.mark.parametrize("fam", FAMILIES)
def test_get_mapping_ind_equals_the_oracle(fb, fam):
    """flow_utils.get_mapping_ind over a three-frame chain of the family (scale 8, non-square) equals O.mapping_ind."""
    H, W, s = 17, 24, 8
    parts = [family(fam, H, W, s, seed=k) for k in range(2)]
    flows = torch.cat([p[0] for p in parts])
    occs = torch.cat([p[1] for p in parts])
    imgs = torch.cat([parts[0][2], parts[1][2][1:]])
    want = O.mapping_ind(flows, occs, imgs, float(s))
    got = fb.fu.get_mapping_ind(flows.cuda(), occs.cuda(), imgs.cuda(), float(s))
    for a, b, what in zip(got, want, ("fwd", "bwd", "mask")):
        assert torch.equal(a.cpu(), b), f"{fam}: {what} differs"
