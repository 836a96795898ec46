"""Adam (O4), AdaIN (O5), guidance + DDPM step (S1) and dilation (W2) through the C ABI, against oracle.step_bound.

Every family of the bound runs on both dtypes where the kernel has two, and every call asserts its launch name.
Outputs are prefilled with NaN between NaN guard regions: every element must be written and lie within the bound,
the exact families and elements must match bit for bit, and no guard may change.  Adam works in place, so it runs on
the first n elements of longer buffers whose tails must come back untouched.  Sizes: n in {1, 255, 257, cap - 1, cap,
cap + 1} with cap = 8 x SMs x 256 (the grid-stride loop's first pass, from the device's SM count), Adam at the layer-3
size 16 x 640 x 64 x 64, AdaIN at the plane counts and sizes of the four decoder layers and at 96 x 96 planes.
``pipe_FRESCO.step`` runs end to end at SD-1.5's timesteps 999, 981, 501, 21, 1 and 0 on both dtypes, within the composed
bound of its two kernels.  ``test_report_worst_ratios`` prints the largest err/tol per kernel and family (-s).
"""
import pytest
import torch

from oracle import step_bound as SB

pytestmark = pytest.mark.gpu
RATIOS = {}         # (kernel, family) -> worst err/tol
GUARD = 512


@pytest.fixture(scope="module")
def fb():
    if not torch.cuda.is_available():
        pytest.skip("GPU tests need a CUDA device")
    from fresco_b200 import _lib, ops
    _lib.lib()      # fails loudly if the extension is missing

    class NS:
        pass
    ns = NS()
    ns.lib, ns.ops, ns.c = _lib, ops, _lib.lib()
    ns.cap = 8 * torch.cuda.get_device_properties(0).multi_processor_count * 256
    return ns


def P(t):
    return t.data_ptr()


def _sizes(fb):
    return (1, 255, 257, fb.cap - 1, fb.cap, fb.cap + 1)


def _guarded(n, dtype):
    """(buffer, the n-element output view between two NaN guard regions)."""
    buf = torch.full((n + 2 * GUARD,), float("nan"), dtype=dtype, device="cuda")
    return buf, buf[GUARD:GUARD + n]


def _guards_nan(buf):
    return bool(torch.isnan(buf[:GUARD]).all() and torch.isnan(buf[-GUARD:]).all())


def _record(kernel, fam, out, ref, tol, dtype, what, overflow=False):
    if not overflow:
        assert torch.isfinite(out).all(), f"{what}: {(~torch.isfinite(out)).sum().item()} outputs not written or not finite"
    else:
        assert not torch.isnan(out).any(), f"{what}: {torch.isnan(out).sum().item()} outputs not written"
    tol = SB.out_tol(ref, tol, dtype)
    r = SB.ratio16(out, ref, tol) if dtype == torch.float16 else SB.ratio(out, ref, tol)
    worst = r.max().item()
    if worst > 1:
        i = int(torch.argmax(r.reshape(-1)))
        raise AssertionError(f"{what}: {(r > 1).sum().item()} elements outside the bound, worst err/tol {worst:.3g} at "
                             f"{i}: out {out.reshape(-1)[i].item()!r} ref {ref.reshape(-1)[i].item()!r} "
                             f"tol {tol.reshape(-1)[i].item():.3g}")
    RATIOS[(kernel, fam)] = max(RATIOS.get((kernel, fam), 0.0), worst)
    return worst


# ------------------------------------------------------------------------------------------------ Adam
def _adam(fb, d, n, cfg):
    """fresco_adam_step on the first n elements of the family's (longer) buffers -> their new contents."""
    p, g, m, v = (d[k].clone() for k in ("p", "g", "m", "v"))
    step, lr, b1, b2, eps = cfg
    fb.lib.check(fb.c.fresco_adam_step(P(p), P(g), P(m), P(v), n, step, lr, b1, b2, eps, fb.lib.stream()),
                 "fresco_adam_step")
    assert fb.lib.last_kernel() == "adam_kernel"
    for key, t in (("p", p), ("m", m), ("v", v), ("g", g)):
        assert torch.equal(t[n:], d[key][n:]), f"{key}: the tail past n was written"
    return {"p": p[:n], "m": m[:n], "v": v[:n]}


def _adam_check(d, n, cfg, out, fam, what):
    ref = SB.adam_reference_and_bound(d["p"][:n], d["g"][:n], d["m"][:n], d["v"][:n], *cfg)
    for key in ("p", "m", "v"):
        _record("adam_kernel", fam, out[key], *ref[key], torch.float32, f"{what} {key}")
    ex = d["exact"][:n]
    for key in ("p", "m", "v"):
        assert torch.equal(out[key][ex], d[key][:n][ex]), f"{what} {key}: g = m = v = 0 elements changed"


@pytest.mark.parametrize("fam", SB.ADAM_FAMILIES)
def test_adam_family(fb, fam):
    for i, n in enumerate(_sizes(fb)):
        d = SB.adam_family(fam, n + 300, seed=i, device="cuda")
        for cfg in SB.ADAM_CONFIGS[fam]:
            _adam_check(d, n, cfg, _adam(fb, d, n, cfg), fam, f"adam {fam} n={n} {cfg}")


def test_adam_layer3_size(fb):
    """The layer-3 decoder features of a 16-frame batch at 512 x 512: each thread runs the grid-stride loop ~155 times."""
    n = 16 * 640 * 64 * 64
    d = SB.adam_family("steps", n + 1000, device="cuda")
    for cfg in ((1, 0.2, 0.9, 0.999, 1e-8), (20, 0.2, 0.9, 0.999, 1e-8)):
        _adam_check(d, n, cfg, _adam(fb, d, n, cfg), "layer-3", f"adam layer 3 {cfg}")


@pytest.mark.parametrize("fam", SB.ADAM_FAMILIES)
def test_torch_adam_on_the_gpu_within_the_same_bound(fb, fam):
    """torch.optim.Adam on the GPU (what the reference runs) from the same state stays inside the kernel's bound."""
    d = SB.adam_family(fam, 4096, device="cuda")
    for step, lr, b1, b2, eps in SB.ADAM_CONFIGS[fam]:
        prm = torch.nn.Parameter(d["p"].clone())
        opt = torch.optim.Adam([prm], lr=lr, betas=(b1, b2), eps=eps)
        opt.state[prm] = {"step": torch.tensor(float(step - 1)), "exp_avg": d["m"].clone(),
                          "exp_avg_sq": d["v"].clone()}
        prm.grad = d["g"].clone()
        opt.step()
        ref = SB.adam_reference_and_bound(d["p"], d["g"], d["m"], d["v"], step, lr, b1, b2, eps)
        for key, got in (("p", prm.data), ("m", opt.state[prm]["exp_avg"]), ("v", opt.state[prm]["exp_avg_sq"])):
            _record("torch.optim.Adam", fam, got, *ref[key], torch.float32, f"torch {fam} step {step} {key}")


# ------------------------------------------------------------------------------------------------ AdaIN
def _adain(fb, c, s):
    planes, hw = c.shape
    buf, out = _guarded(planes * hw, s.dtype)
    half = s.dtype == torch.float16
    fb.lib.check(fb.c.fresco_adain(P(c), P(s), P(out), int(half), planes, hw, fb.lib.stream()), "fresco_adain")
    assert fb.lib.last_kernel() == ("adain_kernel<half>" if half else "adain_kernel<float>")
    assert _guards_nan(buf), "a guard element was written"
    return out.reshape(planes, hw)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16], ids=["float", "half"])
@pytest.mark.parametrize("fam", SB.ADAIN_FAMILIES)
def test_adain_family(fb, fam, dtype):
    for hw in SB.ADAIN_HW:
        c, s = SB.adain_family(fam, 24, hw, dtype, device="cuda")
        ref, tol = SB.adain_reference_and_bound(c, s)
        name = "adain_kernel<half>" if dtype == torch.float16 else "adain_kernel<float>"
        _check_adain(name, fam, _adain(fb, c, s), ref, tol, dtype, f"{name} {fam} hw={hw}")


def _check_adain(name, fam, out, ref, tol, dtype, what):
    """adain_reference_and_bound's tol already holds the output rounding."""
    assert torch.isfinite(out).all(), f"{what}: {(~torch.isfinite(out)).sum().item()} outputs not written or not finite"
    r = SB.ratio(out, ref, tol)
    worst = r.max().item()
    assert worst <= 1, f"{what}: {(r > 1).sum().item()} elements outside the bound, worst err/tol {worst:.3g}"
    RATIOS[(name, fam)] = max(RATIOS.get((name, fam), 0.0), worst)


# (planes, hw) of the four decoder layers of a 16-frame batch at 512 x 512, and layer 3 of a 768 x 768 frame
DECODER = ((16 * 1280, 8 * 8), (16 * 1280, 16 * 16), (16 * 1280, 32 * 32), (16 * 640, 64 * 64), (2 * 640, 96 * 96))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16], ids=["float", "half"])
@pytest.mark.parametrize("planes,hw", DECODER)
def test_adain_decoder_layers(fb, planes, hw, dtype):
    c, s = SB.adain_family("planes", planes, hw, dtype, device="cuda")
    ref, tol = SB.adain_reference_and_bound(c, s)
    name = "adain_kernel<half>" if dtype == torch.float16 else "adain_kernel<float>"
    _check_adain(name, "decoder", _adain(fb, c, s), ref, tol, dtype, f"{name} {planes}x{hw}")


# ------------------------------------------------------------------------------------------------ CFG + DDPM
def _cfg(fb, noise_pred, sample, g, a, text):
    n = sample.numel()
    buf, x0 = _guarded(n, sample.dtype)
    half = sample.dtype == torch.float16
    tp = P(noise_pred) + n * sample.element_size() if text else None
    fb.lib.check(fb.c.fresco_cfg_pred_x0(P(noise_pred), tp, P(sample), P(x0), int(half), n, g, a, fb.lib.stream()),
                 "fresco_cfg_pred_x0")
    assert fb.lib.last_kernel() == ("cfg_pred_x0_kernel<half>" if half else "cfg_pred_x0_kernel<float>")
    assert _guards_nan(buf), "a guard element was written"
    return x0.reshape(sample.shape)


def _ddpm(fb, x0, sample, noise, c_x0, c_xt, sigma, per_frame, repeat):
    n = sample.numel()
    buf, prev = _guarded(n, sample.dtype)
    half = sample.dtype == torch.float16
    fb.lib.check(fb.c.fresco_ddpm_prev(P(x0), P(sample), P(noise), P(prev), int(half), n, per_frame, int(repeat),
                                       c_x0, c_xt, sigma, fb.lib.stream()), "fresco_ddpm_prev")
    assert fb.lib.last_kernel() == ("ddpm_prev_kernel<half>" if half else "ddpm_prev_kernel<float>")
    assert _guards_nan(buf), "a guard element was written"
    return prev.reshape(sample.shape)


def _step_shapes(fb, fam):
    """(frames, per_frame) per case; repeat_noise runs with per_frame 1 and per_frame a frame."""
    if fam == "repeat":
        return ((257, 1), (fb.cap + 1, 1), (4, 4 * 64 * 64), (3, 4 * 96 * 96), (5, 4 * 8 * 13))
    return tuple((1, n) for n in _sizes(fb)) + ((16, 4 * 64 * 64),)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16], ids=["float", "half"])
@pytest.mark.parametrize("fam", SB.STEP_FAMILIES)
def test_cfg_and_ddpm_family(fb, fam, dtype):
    ac = SB.sd15_alphas_cumprod()
    shapes = _step_shapes(fb, fam)
    half = dtype == torch.float16
    t16 = "half" if half else "float"
    k = 0
    for i, t in enumerate(SB.TIMESTEPS):
        a, c_x0, c_xt, sigma = SB.step_coefficients(ac, t, t - 20)
        for g in SB.GUIDANCE:
            frames, per_frame = shapes[k % len(shapes)]
            k += 1
            d = SB.step_family(fam, frames, per_frame, dtype, t, seed=k, device="cuda")
            text = fam != "no-text"
            n = d["sample"].numel()
            np_ = d["noise_pred"] if text else d["noise_pred"][:frames].contiguous()
            ref, tol = SB.cfg_reference_and_bound(np_.reshape(-1)[:n], np_.reshape(-1)[n:] if text else None,
                                                  d["sample"], g, a)
            x0 = _cfg(fb, np_, d["sample"], g, a, text)
            over = fam == "overflow" and half
            _record(f"cfg_pred_x0_kernel<{t16}>", fam, x0, ref, tol, dtype, f"cfg {fam} t={t} g={g} n={n}", over)
            # the DDPM operands: the family's own, or for overflow x0 = sample near 65504 so prev crosses it
            x0_in = d["sample"] if fam == "overflow" else d["noise_pred"][:frames].contiguous()
            if over:
                x0_in = (x0_in.float().sign() * 65504.0 * (0.97 + 0.03 * torch.rand(x0_in.shape, device="cuda"))).half()
            repeat = fam == "repeat"
            ref, tol = SB.ddpm_reference_and_bound(x0_in, x0_in if over else d["sample"], d["noise"], c_x0, c_xt,
                                                   sigma, per_frame, repeat)
            prev = _ddpm(fb, x0_in, x0_in if over else d["sample"], d["noise"], c_x0, c_xt, sigma, per_frame, repeat)
            _record(f"ddpm_prev_kernel<{t16}>", fam, prev, ref, tol, dtype, f"ddpm {fam} t={t} n={n}", over)


def test_overflow_family_overflows(fb):
    """The fp16 overflow family really produces infinities at t = 999 (1 / sqrt(a) ~ 14.6)."""
    ac = SB.sd15_alphas_cumprod()
    a = SB.step_coefficients(ac, 999, 979)[0]
    d = SB.step_family("overflow", 1, 4096, torch.float16, 999, device="cuda")
    x0 = _cfg(fb, d["noise_pred"], d["sample"], 7.5, a, True)
    frac = torch.isinf(x0).float().mean().item()
    assert 0.05 < frac < 0.95, frac


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16], ids=["float", "half"])
def test_pipe_step_end_to_end(fb, dtype):
    """pipe_FRESCO.step (guidance fused into the x0 kernel, then the DDPM kernel) on SD-1.5's schedule within the
    composed bound: the x0 bound (with its output rounding) times |c_x0| plus the DDPM bound on the fp64 x0."""
    from fresco_b200 import pipe_FRESCO as pf
    ac = SB.sd15_alphas_cumprod()

    class Sched:
        alphas_cumprod = ac
        one = torch.tensor(1.0)

        @staticmethod
        def previous_timestep(t):
            return t - 20

    class Pipe:
        scheduler = Sched()
    N, shape = 4, (4, 64, 64)
    half = dtype == torch.float16
    for i, t in enumerate(SB.TIMESTEPS):
        for g, repeat in ((7.5, False), (30.0, True), (1.0, i % 2 == 0)):
            d = SB.step_family("schedule", N, 4 * 64 * 64, dtype, t, seed=i, device="cuda")
            raw = d["noise_pred"].reshape(2 * N, *shape)
            sample, noise = d["sample"].reshape(N, *shape), d["noise"].reshape(N, *shape)
            prev, x0 = pf.step(Pipe, raw, t, sample, None, repeat_noise=repeat, guidance_scale=g, noise=noise)
            a, c_x0, c_xt, sigma = SB.step_coefficients(ac, t, t - 20)
            x0_ref, x0_tol = SB.cfg_reference_and_bound(raw[:N], raw[N:], sample, g, a)
            _record("step: x0", "end-to-end", x0, x0_ref, x0_tol, dtype, f"step x0 t={t} g={g}")
            p_ref, p_tol = SB.ddpm_reference_and_bound(x0_ref, sample, noise, c_x0, c_xt, sigma, sample[0].numel(),
                                                       repeat)
            composed = p_tol + abs(c_x0) * SB.out_tol(x0_ref, x0_tol, dtype)
            _record("step: prev", "end-to-end", prev, p_ref, composed, dtype, f"step prev t={t} g={g} rep={repeat}")
            assert fb.lib.last_kernel() == ("ddpm_prev_kernel<half>" if half else "ddpm_prev_kernel<float>")


# ------------------------------------------------------------------------------------------------ dilation
def _dilate_cases(cap):
    return [(3, 4, 4, 13), (2, 1, 17, 5), (2, 19, 1, 5), (3, 16, 16, 1), (1, 1, 1, 13), (5, 96, 96, 13),
            (4, 40, 56, 5), (cap // 4096, 64, 64, 13), (1, 1, cap - 1, 5), (1, 1, cap + 1, 3),
            (cap // 4096 + 1, 64, 64, 5)]


@pytest.mark.parametrize("fam", SB.DILATE_FAMILIES)
def test_dilate_family(fb, fam):
    for P_, h, w, k in _dilate_cases(fb.cap):
        x = SB.dilate_family(fam, P_, h, w, device="cuda")
        buf, out = _guarded(P_ * h * w, torch.float32)
        fb.lib.check(fb.c.fresco_dilate(P(x), P(out), P_, h, w, k, fb.lib.stream()), "fresco_dilate")
        assert fb.lib.last_kernel() == "dilate_kernel"
        assert _guards_nan(buf), "a guard element was written"
        out = out.reshape(P_, h, w)
        ref, tol = SB.dilate_reference_and_bound(x, k)
        _record("dilate_kernel", fam, out, ref, tol, torch.float32, f"dilate {fam} {P_}x{h}x{w} k={k}")
        if fam in SB.DILATE_EXACT:
            assert torch.equal(out, ref.float()), f"dilate {fam} {P_}x{h}x{w} k={k}: not bit-exact"


# ------------------------------------------------------------------------------------------------ refusals
def test_c_entry_points_refuse_without_launching(fb):
    """hw <= 1, an even kernel, in-place dilation and n % per_frame != 0 are refused before any launch."""
    x = torch.zeros(4096, device="cuda")
    y = torch.full_like(x, float("nan"))
    torch.cuda.synchronize()
    before = fb.lib.launch_count()
    s = fb.lib.stream()
    c = fb.c
    calls = ((lambda: c.fresco_adain(P(x), P(x), P(y), 0, 4, 1, s), b"bad shape"),
             (lambda: c.fresco_adain(P(x), P(x), P(y), 1, 4, 0, s), b"bad shape"),
             (lambda: c.fresco_dilate(P(x), P(y), 1, 8, 8, 4, s), b"odd kernel"),
             (lambda: c.fresco_dilate(P(x), P(x), 1, 8, 8, 5, s), b"in-place"),
             (lambda: c.fresco_ddpm_prev(P(x), P(x), P(x), P(y), 0, 100, 30, 1, 1.0, 0.5, 0.1, s), b"per_frame"),
             (lambda: c.fresco_adam_step(P(x), P(x), P(x), P(x), 0, 1, 0.2, 0.9, 0.999, 1e-8, s), b"bad n/step"),
             (lambda: c.fresco_cfg_pred_x0(P(x), P(x), P(x), P(y), 0, 100, 7.5, 0.0, s), b"alpha"))
    for call, msg in calls:
        rc = call()
        assert rc != 0 and msg in c.fresco_last_error(), (rc, c.fresco_last_error())
    torch.cuda.synchronize()
    assert fb.lib.launch_count() == before and torch.isnan(y).all()


def test_report_worst_ratios():
    """Prints the largest err/tol seen per kernel and family (-s to see it)."""
    if not RATIOS:
        pytest.skip("no step-kernel case ran")
    print("\nworst err/tol per kernel and family")
    for (kn, fam), r in sorted(RATIOS.items()):
        print(f"  {kn:28s} {fam:12s} {r:.3g}")
