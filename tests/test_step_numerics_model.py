"""The per-step elementwise kernels of hbm_kernels.cu -- adam_kernel, adain_kernel, cfg_pred_x0_kernel,
ddpm_prev_kernel, dilate_kernel -- restated in torch fp32 on the CPU, in each kernel's order of work.

Every product that nvcc may fuse into the following add is evaluated in every contraction mode (``MODES``): Adam's
``m + (g - m) c1``, ``v b2 + g^2 c2``, ``sqrt(v) / sqrt(bc2) + eps`` and ``p - step q``; AdaIN's squared-deviation sums
and its output ``b sigma_s + mu_s``; CFG's ``u + g (t - u)`` and ``s - sqrt(1 - a) e``; the DDPM three-term sum in
each association.  AdaIN's sums run in the kernel's order: 256 per-thread chains, a warp butterfly, the block's second
butterfly over the eight warp sums.

It checks the error model of ``oracle.step_bound`` without a GPU: every mode stays inside the bound on every family,
matches the exact elements and families bit for bit and reports its worst err/tol (so the bound is seen not to be
vacuous); each of ``MUTANTS`` -- a one-line mistake a change to the kernels could make -- leaves the bound or the exact
answer on the family named with it.  torch.optim.Adam, what the reference runs, stays inside the same bound.
"""
import math

import pytest
import torch

from oracle import step_bound as SB

MUTANTS = {
    # name: (kernel, what it does, the family that must catch it)
    "bc2-no-sqrt": ("adam", "divides by bc2 instead of sqrt(bc2)", "steps"),
    "eps-in-sqrt": ("adam", "sqrt(v / bc2 + eps) instead of sqrt(v / bc2) + eps", "tiny-grad"),
    "bc-prev-step": ("adam", "the bias corrections of step - 1", "steps"),
    "biased-var": ("adain", "variance divided by hw instead of hw - 1", "planes"),
    "style-eps": ("adain", "style eps 1e-5: the reference's eps quirk lost", "planes"),
    "no-half-round": ("adain", "content not rounded to fp16 on the half path", "offset"),
    "guidance-reversed": ("cfg", "guidance applied to (u - t)", "schedule"),
    "noise-mod-n": ("ddpm", "noise indexed i % n instead of i % per_frame", "repeat"),
    "zero-pad": ("dilate", "zero padding instead of replicate", "unit"),
    "radius+1": ("dilate", "radius one larger than (k - 1) / 2", "binary"),
    "no-clamp": ("dilate", "the box sum not clamped to [0, 1]", "binary"),
}
MODES = ("none", "fma-a", "fma-b")
DDPM_MODES = ("none", "fma-a", "fma-b", "fma-last")
WORST = {}          # (kernel, family) -> worst err/tol over the modes


def _f(x):
    return torch.tensor(x, dtype=torch.float32)


def _fma(a, b, c):
    """fp32 fma: the product of two fp32 values is exact in fp64, one rounding to fp32 after the add."""
    a, b, c = (t if isinstance(t, torch.Tensor) else _f(t) for t in (a, b, c))
    return (a.double() * b.double() + c.double()).float()


def _note(kernel, fam, r):
    WORST[(kernel, fam)] = max(WORST.get((kernel, fam), 0.0), r)


# ------------------------------------------------------------------------------------------------ Adam
def adam_emulate(d, step, lr, b1, b2, eps, mode="none", mutant=None):
    k = SB.adam_constants(max(step - 1, 1) if mutant == "bc-prev-step" else step, lr, b1, b2, eps)
    c1, b2f, c2, ss, isb, e = (_f(k[n]) for n in ("c1", "b2", "c2", "step_size", "inv_sqrt_bc2", "eps"))
    if mutant == "bc2-no-sqrt":
        isb = _f(SB.f32(1.0 / k["sqrt_bc2"] ** 2))
    p, g, m, v = d["p"], d["g"], d["m"], d["v"]
    dm = g - m
    m1 = m + dm * c1 if mode == "none" else _fma(dm, c1, m)
    gg = g * g
    v1 = {"none": lambda: v * b2f + gg * c2, "fma-a": lambda: _fma(v, b2f, gg * c2),
          "fma-b": lambda: _fma(gg, c2, v * b2f)}[mode]()
    s = torch.sqrt(v1)
    if mutant == "eps-in-sqrt":
        D = torch.sqrt(v1 * isb * isb + e)
    else:
        D = s * isb + e if mode == "none" else _fma(s, isb, e)
    q = m1 / D
    p1 = p - ss * q if mode == "none" else _fma(-ss, q, p)
    return {"p": p1, "m": m1, "v": v1}


@pytest.mark.parametrize("fam", SB.ADAM_FAMILIES)
def test_adam_emulation_within_bound(fam):
    d = SB.adam_family(fam, 4096)
    for cfg in SB.ADAM_CONFIGS[fam]:
        ref = SB.adam_reference_and_bound(d["p"], d["g"], d["m"], d["v"], *cfg)
        for mode in MODES:
            out = adam_emulate(d, *cfg, mode=mode)
            for key in ("p", "m", "v"):
                r = SB.ratio(out[key], *ref[key]).max().item()
                assert r <= 1.0, f"{fam} {cfg} {mode} {key}: err/tol {r:.3g}"
                _note("adam", fam, r)
            ex = d["exact"]
            for key in ("p", "m", "v"):
                assert torch.equal(out[key][ex], d[key][ex]), f"{fam} {mode} {key}: g = m = v = 0 elements changed"


@pytest.mark.parametrize("fam", SB.ADAM_FAMILIES)
def test_torch_adam_within_the_same_bound(fam):
    """torch.optim.Adam (what the reference runs) from the same state, at every step and hyper-parameter set of the
    family, stays inside the bound: it rounds the hyper-parameters to fp32 one by one, as the launcher does."""
    d = SB.adam_family(fam, 4096)
    for step, lr, b1, b2, eps in SB.ADAM_CONFIGS[fam]:
        prm = torch.nn.Parameter(d["p"].clone())
        opt = torch.optim.Adam([prm], lr=lr, betas=(b1, b2), eps=eps)
        opt.state[prm] = {"step": torch.tensor(float(step - 1)), "exp_avg": d["m"].clone(),
                          "exp_avg_sq": d["v"].clone()}
        prm.grad = d["g"].clone()
        opt.step()
        st = opt.state[prm]
        ref = SB.adam_reference_and_bound(d["p"], d["g"], d["m"], d["v"], step, lr, b1, b2, eps)
        for key, got in (("p", prm.data), ("m", st["exp_avg"]), ("v", st["exp_avg_sq"])):
            r = SB.ratio(got, *ref[key]).max().item()
            assert r <= 1.0, f"torch {fam} step {step} {key}: err/tol {r:.3g}"
            _note("torch.optim.Adam", fam, r)


# ------------------------------------------------------------------------------------------------ AdaIN
def _block_sum(x):
    """adain_kernel's block_sum of per-thread chains: x fp32 [P, hw] -> [P] in the kernel's order."""
    P, hw = x.shape
    K = math.ceil(hw / 256)
    t = torch.zeros(P, K * 256)
    t[:, :hw] = x
    t = t.reshape(P, K, 256)
    acc = torch.zeros(P, 256)
    for j in range(K):
        acc = acc + t[:, j]
    return _tree(acc)


def _warp_sum(lanes):
    idx = torch.arange(32)
    for o in (16, 8, 4, 2, 1):
        lanes = lanes + lanes[..., idx ^ o]
    return lanes


def _tree(acc):
    P = acc.shape[0]
    red = _warp_sum(acc.reshape(P, 8, 32))[..., 0]
    t = torch.zeros(P, 32)
    t[:, :8] = red
    return _warp_sum(t)[:, 0]


def _block_sq(dev, mode):
    """sum of dev^2 over per-thread chains, cq += dc * dc rounded or fused."""
    P, hw = dev.shape
    K = math.ceil(hw / 256)
    t = torch.zeros(P, K * 256)
    t[:, :hw] = dev
    t = t.reshape(P, K, 256)
    acc = torch.zeros(P, 256)
    for j in range(K):
        acc = acc + t[:, j] * t[:, j] if mode == "none" else _fma(t[:, j], t[:, j], acc)
    return _tree(acc)


def adain_emulate(content, style, mode="none", mutant=None):
    hw = content.shape[1]
    half = style.dtype == torch.float16
    c = content.half().float() if half and mutant != "no-half-round" else content.float()
    s = style.float()
    out = []
    stats = []
    for x, eps in ((c, _f(SB.CONTENT_EPS)), (s, _f(1e-5 if mutant == "style-eps" else 1.0))):
        mean = _block_sum(x) / _f(float(hw))
        q = _block_sq(x - mean[:, None], mode)
        var = q / _f(float(hw if mutant == "biased-var" else hw - 1))
        stats.append((mean[:, None], torch.sqrt(var + eps)[:, None]))
    (cm, cs), (sm, ss) = stats
    b = (c - cm) / cs
    out = b * ss + sm if mode == "none" else _fma(b, ss.expand_as(b), sm.expand_as(b))
    return out.to(style.dtype)


def _adain_cases():
    return [(fam, hw) for fam in SB.ADAIN_FAMILIES for hw in SB.ADAIN_HW]


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16], ids=["float", "half"])
@pytest.mark.parametrize("fam,hw", _adain_cases())
def test_adain_emulation_within_bound(fam, hw, dtype):
    c, s = SB.adain_family(fam, 6, hw, dtype)
    ref, tol = SB.adain_reference_and_bound(c, s)
    for mode in MODES[:2]:
        out = adain_emulate(c, s, mode)
        r = SB.ratio(out, ref, tol).max().item()
        assert r <= 1.0, f"{fam} hw {hw} {mode}: err/tol {r:.3g}"
        _note("adain", fam, r)


# ------------------------------------------------------------------------------------------------ CFG + DDPM
def cfg_emulate(noise_pred, sample, guidance, alpha, text=True, mode="none", mutant=None):
    n = sample.numel()
    u = noise_pred.reshape(-1)[:n].float()
    s = sample.reshape(-1).float()
    a = _f(alpha)
    sb, isa = torch.sqrt(1 - a), 1 / torch.sqrt(a)
    g = _f(guidance)
    if text:
        t = noise_pred.reshape(-1)[n:].float()
        d = u - t if mutant == "guidance-reversed" else t - u
        e = u + g * d if mode == "none" else _fma(g, d, u)
    else:
        e = u
    y = s - sb * e if mode == "none" else _fma(-sb, e, s)
    return (y * isa).to(sample.dtype).reshape(sample.shape)


def ddpm_emulate(x0, sample, noise, c_x0, c_xt, sigma, repeat, mode="none", mutant=None):
    n, per_frame = sample.numel(), sample[0].numel()
    x, s = x0.reshape(-1).float(), sample.reshape(-1).float()
    z = SB.ddpm_noise(noise, n, per_frame, repeat and mutant != "noise-mod-n").float()
    a, b, c = _f(c_x0), _f(c_xt), _f(sigma)
    if mode == "none":
        out = a * x + b * s + c * z
    elif mode == "fma-a":
        out = _fma(c, z, _fma(a, x, b * s))
    elif mode == "fma-b":
        out = _fma(c, z, _fma(b, s, a * x))
    else:
        out = _fma(c, z, a * x + b * s)
    return out.to(sample.dtype).reshape(sample.shape)


def _check_step(out, ref, tol, dtype):
    tol = SB.out_tol(ref, tol, dtype)
    r = SB.ratio16(out, ref, tol) if dtype == torch.float16 else SB.ratio(out, ref, tol)
    return r.max().item()


def _step_cases(fam, dtype, frames=2, per_frame=300):
    """(t, guidance, text, repeat, operands, coefficients) of a family."""
    ac = SB.sd15_alphas_cumprod()
    out = []
    for i, t in enumerate(SB.TIMESTEPS):
        a, c_x0, c_xt, sigma = SB.step_coefficients(ac, t, t - 20)
        d = SB.step_family(fam, frames, per_frame, dtype, t, seed=i)
        for g in SB.GUIDANCE:
            out.append((t, g, fam != "no-text", fam == "repeat", d, (a, c_x0, c_xt, sigma)))
    return out


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16], ids=["float", "half"])
@pytest.mark.parametrize("fam", SB.STEP_FAMILIES)
def test_cfg_and_ddpm_emulation_within_bound(fam, dtype):
    for t, g, text, repeat, d, (a, c_x0, c_xt, sigma) in _step_cases(fam, dtype):
        n = d["sample"].numel()
        np_ = d["noise_pred"] if text else d["noise_pred"][:d["sample"].shape[0]]
        ref, tol = SB.cfg_reference_and_bound(np_.reshape(-1)[:n], np_.reshape(-1)[n:] if text else None,
                                              d["sample"], g, a)
        for mode in MODES[:2]:
            r = _check_step(cfg_emulate(np_, d["sample"], g, a, text, mode), ref.reshape(d["sample"].shape),
                            tol.reshape(d["sample"].shape), dtype)
            assert r <= 1.0, f"cfg {fam} t {t} g {g} {mode}: err/tol {r:.3g}"
            _note("cfg", fam, r)
        x0 = d["noise_pred"][:d["sample"].shape[0]]           # any finite x0 of the dtype
        for per_frame_repeat in ((True,) if repeat else (False,)):
            ref, tol = SB.ddpm_reference_and_bound(x0, d["sample"], d["noise"], c_x0, c_xt, sigma,
                                                   d["sample"][0].numel(), per_frame_repeat)
            for mode in DDPM_MODES:
                out = ddpm_emulate(x0, d["sample"], d["noise"], c_x0, c_xt, sigma, per_frame_repeat, mode)
                r = _check_step(out, ref, tol, dtype)
                assert r <= 1.0, f"ddpm {fam} t {t} {mode}: err/tol {r:.3g}"
                _note("ddpm", fam, r)


def test_step_coefficients_match_pipe_step():
    """The coefficients the tests use are the ones pipe_FRESCO.step passes to the kernels."""
    from fresco_b200 import pipe_FRESCO as pf
    ac = SB.sd15_alphas_cumprod()

    class Sched:
        alphas_cumprod = ac
        one = torch.tensor(1.0)

        @staticmethod
        def previous_timestep(t):
            return t - 20
    for t in SB.TIMESTEPS:
        assert pf._step_coefficients(Sched, t) == SB.step_coefficients(ac, t, t - 20)
    assert SB.step_coefficients(ac, 0, -20)[3] == pytest.approx(1e-10)
    assert 1 / math.sqrt(SB.step_coefficients(ac, 999, 979)[0]) > 14.5


# ------------------------------------------------------------------------------------------------ dilation
DILATE_CASES = [(3, 4, 4, 13), (2, 1, 17, 5), (2, 19, 1, 5), (3, 16, 16, 1), (2, 24, 20, 13), (4, 9, 13, 3),
                (2, 1, 1, 13)]


def dilate_emulate(x, k, mutant=None):
    P, h, w = x.shape
    r = (k - 1) // 2 + (1 if mutant == "radius+1" else 0)
    acc = torch.zeros(P, h, w)
    ys, xs = torch.arange(h), torch.arange(w)
    for dy in range(-r, r + 1):
        for dx in range(-r, r + 1):
            yy, xx = ys + dy, xs + dx
            v = x[:, yy.clamp(0, h - 1)][:, :, xx.clamp(0, w - 1)]
            if mutant == "zero-pad":
                inside = ((yy >= 0) & (yy < h))[:, None] & ((xx >= 0) & (xx < w))[None]
                v = v * inside
            acc = acc + v
    return acc if mutant == "no-clamp" else acc.clamp(0, 1)


@pytest.mark.parametrize("case", DILATE_CASES, ids=lambda c: "%dx%dx%d-k%d" % c)
@pytest.mark.parametrize("fam", SB.DILATE_FAMILIES)
def test_dilate_emulation_within_bound(fam, case):
    P, h, w, k = case
    x = SB.dilate_family(fam, P, h, w)
    ref, tol = SB.dilate_reference_and_bound(x, k)
    out = dilate_emulate(x, k)
    r = SB.ratio(out, ref, tol).max().item()
    assert r <= 1.0, f"{fam}: err/tol {r:.3g}"
    _note("dilate", fam, r)
    if fam in SB.DILATE_EXACT:
        assert torch.equal(ref.float().double(), ref) and torch.equal(out, ref.float()), f"{fam}: not bit-exact"


def test_dilate_reference_is_the_oracle_on_masks():
    """The clamped-index box sum is oracle.dilate (F.pad replicate + conv2d) wherever the padding fits the plane."""
    from oracle import fresco_oracle as O
    x = SB.dilate_family("binary", 3, 24, 20)
    for k in (1, 5, 13):
        ref, _ = SB.dilate_reference_and_bound(x, k)
        assert torch.equal(O.dilate(x[:, None], k)[:, 0], ref.float())


# ------------------------------------------------------------------------------------------------ mutants
def _mutant_caught(mutant):
    kernel, _, fam = MUTANTS[mutant]
    if kernel == "adam":
        d = SB.adam_family(fam, 4096)
        for cfg in SB.ADAM_CONFIGS[fam]:
            ref = SB.adam_reference_and_bound(d["p"], d["g"], d["m"], d["v"], *cfg)
            out = adam_emulate(d, *cfg, mutant=mutant)
            if any(SB.ratio(out[k], *ref[k]).max().item() > 1 for k in ("p", "m", "v")):
                return True
        return False
    if kernel == "adain":
        for dtype in (torch.float32, torch.float16):
            for hw in SB.ADAIN_HW:
                c, s = SB.adain_family(fam, 6, hw, dtype)
                ref, tol = SB.adain_reference_and_bound(c, s)
                if SB.ratio(adain_emulate(c, s, mutant=mutant), ref, tol).max().item() > 1:
                    return True
        return False
    if kernel in ("cfg", "ddpm"):
        for dtype in (torch.float32, torch.float16):
            for t, g, text, repeat, d, (a, c_x0, c_xt, sigma) in _step_cases(fam, dtype):
                n = d["sample"].numel()
                if kernel == "cfg":
                    ref, tol = SB.cfg_reference_and_bound(d["noise_pred"].reshape(-1)[:n],
                                                          d["noise_pred"].reshape(-1)[n:], d["sample"], g, a)
                    out = cfg_emulate(d["noise_pred"], d["sample"], g, a, True, mutant=mutant)
                    ref, tol = ref.reshape(out.shape), tol.reshape(out.shape)
                else:
                    x0 = d["noise_pred"][:d["sample"].shape[0]]
                    ref, tol = SB.ddpm_reference_and_bound(x0, d["sample"], d["noise"], c_x0, c_xt, sigma,
                                                           d["sample"][0].numel(), True)
                    out = ddpm_emulate(x0, d["sample"], d["noise"], c_x0, c_xt, sigma, True, mutant=mutant)
                if _check_step(out, ref, tol, dtype) > 1:
                    return True
        return False
    for P, h, w, k in DILATE_CASES:
        x = SB.dilate_family(fam, P, h, w)
        ref, tol = SB.dilate_reference_and_bound(x, k)
        out = dilate_emulate(x, k, mutant)
        if SB.ratio(out, ref, tol).max().item() > 1 or (fam in SB.DILATE_EXACT and not torch.equal(out, ref.float())):
            return True
    return False


@pytest.mark.parametrize("mutant", sorted(MUTANTS))
def test_mutant_caught(mutant):
    kernel, what, fam = MUTANTS[mutant]
    assert _mutant_caught(mutant), f"{kernel} mutant {mutant} ({what}) passes the {fam} family"


def test_report_worst_ratios():
    """Prints the largest err/tol of the emulation per kernel and family (-s to see it); each kernel's worst case must
    use a visible share of its bound, or the bound would say nothing."""
    if not WORST:
        pytest.skip("no emulation case ran")
    print("\nworst err/tol of the fp32 emulation per kernel and family")
    for (kn, fam), r in sorted(WORST.items()):
        print(f"  {kn:18s} {fam:12s} {r:.3g}")
    for kn in {k for k, _ in WORST}:
        worst = max(r for (k, _), r in WORST.items() if k == kn)
        assert worst > 1e-3, f"{kn}: the bound is never approached (worst err/tol {worst:.3g})"
