"""The blending kernels (blend.cu) and the drop-ins of fresco_b200/blend.py against the oracle (oracle/blend_oracle.py)
and the reference's own outputs (tests/golden/blend*.npz).

Outputs are prefilled with 0xFF (uint8) or NaN (fp64) so an element a kernel never writes fails, and each case asserts
the name of the kernel that ran last.  The LUT gathers, the mask chain and the histogram blend are held bit for bit
(the histogram may differ only at counted .5 ties).  The Poisson solution is held elementwise to the exact fp64
solution within oracle.blend_bound.TOL; the uint8 output must equal the oracle's except where the exact solution lies
within TOL of an integer, and those pixels are counted.  ``test_report`` prints the worst err / tol per family (-s).
"""
import os

import numpy as np
import pytest
import torch

from oracle import blend_bound as BB
from oracle import blend_oracle as BO

pytestmark = pytest.mark.gpu
REPORT = {}


@pytest.fixture(scope="module")
def fb():
    if not torch.cuda.is_available():
        pytest.skip("GPU tests need a CUDA device")
    from fresco_b200 import _lib, blend, ops
    _lib.lib()

    class NS:
        pass
    ns = NS()
    ns.L, ns.ops, ns.blend = _lib, ops, blend
    ns.to_lab, ns.to_bgr = blend.luts()
    return ns


@pytest.fixture(scope="module")
def gb(golden):
    return golden("blend")


def case(gb, tag):
    return {k[len(tag) + 1:]: v for k, v in gb.items() if k.startswith(tag + "_")}


def dev(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def ff(shape, dtype=torch.uint8):
    return torch.full(shape, 255 if dtype == torch.uint8 else float("nan"), dtype=dtype, device="cuda")


def test_lut_gathers_equal_cv2_on_every_colour(fb):
    import cv2
    idx = np.arange(1 << 24, dtype=np.uint32)
    every = np.stack([idx >> 16, (idx >> 8) & 255, idx & 255], -1).astype(np.uint8).reshape(4096, 4096, 3)
    for lut, code in ((fb.to_lab, cv2.COLOR_BGR2LAB), (fb.to_bgr, cv2.COLOR_LAB2BGR)):
        out = ff((4096, 4096, 3))
        fb.ops.blend_lut_gather(dev(every), lut, out=out)
        assert fb.L.last_kernel() == "blend_lut_gather_kernel"
        assert np.array_equal(out.cpu().numpy(), cv2.cvtColor(every, code))


def test_mask_chain_bit_exact_on_goldens(fb, gb):
    for tag in gb["cases"]:
        c = case(gb, str(tag))
        out = ff(c["masks"].shape)
        fb.ops.blend_mask_chain(dev(c["dist1"]), dev(c["dist2"]), dev(c["flows"]), out=out)
        assert fb.L.last_kernel() == "blend_mask_step_kernel"
        assert np.array_equal(out.cpu().numpy(), c["masks"]), tag


@pytest.mark.parametrize("h,w", [(64, 96), (33, 17), (1, 40), (29, 1)])
def test_mask_chain_bit_exact_on_tie_flows(fb, h, w):
    """flows on the half-integer grid (rint ties), on quarter steps, far past every border, and random"""
    rng = np.random.default_rng(h * 1000 + w)
    interval = 7
    n = interval - 1
    d1 = rng.random((n, h, w)).astype(np.float32)
    d2 = rng.random((n, h, w)).astype(np.float32)
    flows = (rng.integers(-9, 10, (n, 2, h, w)) / 2.0).astype(np.float32)
    flows[1] = (rng.integers(-20, 21, (2, h, w)) / 4.0)
    flows[2] = rng.normal(0, 3, (2, h, w))
    flows[3, :, ::3] = rng.choice([-1e9, 1e9, -w - 0.5, w + 0.5], flows[3, :, ::3].shape)
    flows = flows.astype(np.float32)
    out = ff((n, h, w))
    fb.ops.blend_mask_chain(dev(d1), dev(d2), dev(flows), out=out)
    assert fb.L.last_kernel() == "blend_mask_step_kernel"
    assert np.array_equal(out.cpu().numpy(), BO.mask_chain(d1, d2, flows, interval))


def test_histogram_matches_oracle(fb, gb):
    ties = 0
    for tag in gb["cases"]:
        c = case(gb, str(tag))
        ws = BO.seq_weights(int(c["interval"]))
        la = np.stack([BO.to_lab(x) for x in c["oa"]])
        lb = np.stack([BO.to_lab(x) for x in c["ob"]])
        weights = dev(np.array([(1 - w1, 1 - w2) for w1, w2 in ws], dtype=np.float64))
        for use_mask in (True, False):
            out = ff(la.shape)
            if use_mask:
                fb.ops.blend_histogram(dev(la), dev(lb), weights, masks=dev(c["masks"]), out=out)
            else:
                le = np.stack([BO.to_lab(x) for x in c["min_error"]])
                fb.ops.blend_histogram(dev(la), dev(lb), weights, lab_min_error=dev(le), out=out)
            assert fb.L.last_kernel() == "blend_hist_apply_kernel"
            got = out.cpu().numpy()
            for k, (w1, w2) in enumerate(ws):
                want, pre = BO.histogram_blend_lab(la[k], lb[k], BO.min_error(la[k], lb[k], c["masks"][k]), 1 - w1,
                                                   1 - w2)
                near = np.abs(np.abs(pre - np.floor(pre)) - 0.5) < 1e-9
                bad = got[k] != want
                assert not (bad & ~near).any(), (tag, k)
                ties += int(bad.sum())
                assert np.array_equal(BO.to_bgr(want), c["hist"][k]) or near.any()
    REPORT["histogram: .5 ties differing"] = ties


def _frames(rng, n, h, w, family):
    blocks = rng.integers(0, 2, (n, 2, (h + 15) // 16, (w + 15) // 16, 3)) * 255
    base = np.repeat(np.repeat(blocks, 16, 2), 16, 3)[:, :, :h, :w].astype(np.int64)
    imgs = np.clip(base + rng.integers(-40, 41, base.shape), 0, 255).astype(np.uint8)
    yy, xx = np.mgrid[:h, :w]
    if family == "zero":
        m = np.zeros((n, h, w))
    elif family == "one":
        m = np.ones((n, h, w))
    elif family == "checker":
        m = np.repeat(((yy + xx) % 2)[None], n, 0)
    else:
        m = np.repeat(np.repeat(rng.integers(0, 2, (n, (h + 6) // 7, (w + 6) // 7)), 7, 1), 7, 2)[:, :h, :w]
    tgt = rng.integers(0, 256, (n, h, w, 3)).astype(np.uint8)
    return tgt, imgs[:, 0], imgs[:, 1], m.astype(np.uint8)


POISSON = [(512, 896, "blocky"), (896, 512, "checker"), (64, 64, "zero"), (64, 64, "one"), (64, 64, "checker"),
           (1, 640, "blocky"), (480, 1, "blocky"), (37, 53, "blocky")]


@pytest.mark.parametrize("h,w,family", POISSON)
def test_poisson_solution_within_bound(fb, h, w, family):
    rng = np.random.default_rng(h + 7 * w)
    n = 2
    tgt, la, lb, m = _frames(rng, n, h, w, family)
    out, sol = ff((n, h, w, 3)), ff((n, 3, h, w), torch.float64)
    fb.ops.blend_poisson(dev(tgt), dev(la), dev(lb), dev(m), (2.5, 0.5, 0.5), out=out, solution=sol)
    assert fb.L.last_kernel() == "blend_poisson_finalize_kernel"
    sol, out = sol.cpu().numpy(), out.cpu().numpy()
    near_count = 0
    for k in range(n):
        exact = BO.poisson_exact(tgt[k], la[k], lb[k], m[k])
        err = np.abs(sol[k] - exact)
        assert np.isfinite(sol[k]).all()
        for c, g in enumerate((2.5, 0.5, 0.5)):
            assert err[c].max() <= BB.TOL, (c, err[c].max())
            key = f"poisson w={g} {family}"
            REPORT[key] = max(REPORT.get(key, 0.0), float(err[c].max() / BB.TOL))
        near = np.moveaxis(np.abs(exact - np.round(exact)) <= BB.TOL, 0, -1)
        bad = out[k] != BO.finalize(exact)
        assert not (bad & ~near).any()
        near_count += int(bad.sum())
    REPORT[f"poisson uint8 differing within TOL of an integer ({h}x{w} {family})"] = near_count


def test_poisson_zero_weight_and_single_pixel(fb):
    rng = np.random.default_rng(5)
    tgt, la, lb, m = _frames(rng, 1, 1, 1, "one")
    out, sol = ff((1, 1, 1, 3)), ff((1, 3, 1, 1), torch.float64)
    fb.ops.blend_poisson(dev(tgt), dev(la), dev(lb), dev(m), (2.5, 0.0, 0.5), out=out, solution=sol)
    assert np.array_equal(out.cpu().numpy(), tgt)          # no edges: u = im exactly
    assert fb.ops.blend_cheby_iterations(64, 64, 0.0) == 0


def test_drop_ins_on_golden_frames(fb, gb):
    c = case(gb, "c")
    k = c["masks"].shape[0] - 1
    w1, w2 = BO.seq_weights(int(c["interval"]))[k]
    got = fb.blend.histogram_blend(c["oa"][k], c["ob"][k], c["min_error"][k], 1 - w1, 1 - w2)
    assert fb.L.last_kernel() == "blend_lut_gather_kernel"
    assert np.array_equal(got, c["hist"][k])
    got = fb.blend.poisson_fusion(c["hist"][k], c["oa"][k], c["ob"][k], c["masks"][k])
    exact = BO.poisson_exact(BO.to_lab(c["hist"][k]), BO.to_lab(c["oa"][k]), BO.to_lab(c["ob"][k]), c["masks"][k])
    near = (np.abs(exact - np.round(exact)) <= BB.TOL).any(0)
    assert not ((got != BO.to_bgr(BO.finalize(exact))).any(-1) & ~near).any()
    assert not ((got != c["final"][k]).any(-1) & ~near & (c["lab"][k] == BO.finalize(exact)).all(-1)).any()


class Sequence:
    """The paths of blender/video_sequence.VideoSequence that process_seq reads and writes (outputs in out_<key>,
    error planes beside them as .bin, flows in tmp/, results in blend/)."""

    def __init__(self, base, keys):
        self.base, self.keys = base, keys
        for d in ["blend", "tmp", "keys0"] + ["out_%d" % k for k in keys]:
            os.makedirs(os.path.join(base, d), exist_ok=True)

    def interval(self, i):
        return self.keys[i + 1] - self.keys[i]

    def get_sequence_beg_id(self, i):
        return self.keys[i]

    def get_key_img(self, i):
        return os.path.join(self.base, "keys0", "%04d.png" % self.keys[i])

    def get_output_sequence(self, i, is_forward=True):
        beg, end = self.keys[i], self.keys[i + 1]
        ids = range(beg, end) if is_forward else range(end, beg, -1)
        return [os.path.join(self.base, "out_%d" % (beg if is_forward else end), "%04d.jpg" % j) for j in ids]

    def get_flow_sequence(self, i):
        return [os.path.join(self.base, "tmp", "flow_f_%04d.npy" % j) for j in range(self.keys[i], self.keys[i + 1] - 1)]

    def get_blending_img(self, i):
        return os.path.join(self.base, "blend", "%04d.jpg" % i)


def test_process_seq_end_to_end(fb, gb, tmp_path, monkeypatch):
    import cv2
    beg, end = int(gb["seq_beg"]), int(gb["seq_end"])
    h, w = gb["seq_key"].shape[:2]
    seq = Sequence(str(tmp_path), [beg, end])
    cv2.imwrite(seq.get_key_img(0), gb["seq_key"])
    for paths, imgs, errs in ((seq.get_output_sequence(0), gb["seq_fwd"], gb["seq_err_fwd"]),
                              (seq.get_output_sequence(0, False), gb["seq_bwd"], gb["seq_err_bwd"])):
        for path, img, err in zip(paths, imgs, errs):
            with open(path, "wb") as f:        # PNG bytes under Ebsynth's .jpg name: lossless, imread reads by content
                f.write(cv2.imencode(".png", img)[1].tobytes())
            with open(path.replace("jpg", "bin"), "wb") as f:
                f.write(np.int64(h * w).tobytes() + err.astype(np.float32).tobytes())
    for path, flow in zip(seq.get_flow_sequence(0), gb["seq_flows"]):
        np.save(path, flow[None])
    written, real = {}, cv2.imwrite

    def imwrite(path, img, *a):
        written[os.path.basename(path)] = img.copy()
        return real(path, img, *a)
    monkeypatch.setattr(cv2, "imwrite", imwrite)
    fb.blend.process_seq(seq, 0)
    assert fb.L.last_kernel() == "blend_lut_gather_kernel"
    n = end - beg - 1
    assert sorted(written) == ["%04d.jpg" % i for i in range(beg, end)]
    assert all(os.path.exists(seq.get_blending_img(i)) for i in range(beg, end))
    want = gb["seq_out"]
    oas = gb["seq_fwd"][1:n + 1]
    obs = np.stack([gb["seq_bwd"][end - beg - 1 - k] for k in range(n)])
    ref = BO.blend_sequence(oas, obs, gb["seq_err_fwd"][1:n + 1], gb["seq_err_bwd"][1:n + 1], gb["seq_flows"],
                            end - beg)
    assert np.array_equal(written["%04d.jpg" % beg], gb["seq_key"])
    differ = 0
    for k in range(n):
        got = written["%04d.jpg" % (beg + k + 1)]
        u = ref["solution"][k]
        near = (np.abs(u - np.round(u)) <= BB.TOL).any(0)
        assert not ((got != ref["final"][k]).any(-1) & ~near).any(), k
        # against the reference's frames, except where its lsqr iterate truncated differently from the exact solution
        lsqr_ok = (want[k + 1] == ref["final"][k]).all(-1)
        assert not ((got != want[k + 1]).any(-1) & ~near & lsqr_ok).any(), k
        differ += int((got != want[k + 1]).any(-1).sum())
    REPORT["process_seq: pixels differing from the reference's frames"] = differ
    with pytest.raises(fb.L.FrescoError):
        fb.blend.process_seq(seq, 0, blend_histogram=False)


def test_ops_refuse_bad_operands_before_launch(fb):
    ops, L = fb.ops, fb.L
    u8 = torch.zeros(2, 8, 8, 3, dtype=torch.uint8, device="cuda")
    m = torch.zeros(2, 8, 8, dtype=torch.uint8, device="cuda")
    d = torch.zeros(2, 8, 8, dtype=torch.float32, device="cuda")
    wts = torch.ones(2, 2, dtype=torch.float64, device="cuda")
    before = L.launch_count()
    bad = [
        lambda: ops.blend_lut_gather(u8.float(), fb.to_lab),
        lambda: ops.blend_lut_gather(u8, fb.to_lab[:100]),
        lambda: ops.blend_lut_gather(u8.cpu(), fb.to_lab),
        lambda: ops.blend_mask_chain(d.double(), d, torch.zeros(2, 2, 8, 8, device="cuda")),
        lambda: ops.blend_mask_chain(d, d, torch.zeros(2, 8, 8, 2, device="cuda")),
        lambda: ops.blend_histogram(u8, u8, wts.float(), masks=m),
        lambda: ops.blend_histogram(u8, u8, wts, masks=m, lab_min_error=u8),
        lambda: ops.blend_histogram(u8, u8[:, :, :4], wts, masks=m),
        lambda: ops.blend_poisson(u8, u8, u8, m.bool()),
        lambda: ops.blend_poisson(u8, u8, u8.transpose(1, 2), m),
        lambda: ops.blend_poisson(u8, u8, u8, m, (2.5, 0.5)),
        lambda: ops.blend_poisson(u8, u8, u8, m, solution=torch.zeros(2, 3, 8, 8, device="cuda")),
    ]
    for f in bad:
        with pytest.raises(L.FrescoError):
            f()
    assert L.launch_count() == before


def test_report():
    for k, v in sorted(REPORT.items()):
        print(f"{k}: {v}")
