"""Generate the ``optimize_ragged`` golden set by running the REAL reference's optimize_feature on CPU at a decoder
layer-0 shape whose token count is not a multiple of 8.

    python tests/golden/make_ragged_golden.py --reference /path/to/FRESCO

The shape is [2N, 1280, 5, 7] with N = 3: layer 0 of a 320 x 448 frame (the web UI's 320 setting at 4:3), 35 tokens.
The sample is fp16, as the UNet hands it to optimize_feature; the flows are given at the 1/8 grid (40 x 56), which
optimize_feature scales by the same rule as full-resolution flows.  Outputs ``optimize_ragged.npz`` (in parts below
1 MB, see make_golden.save_npz) next to this script, consumed by tests/test_oracle_ragged_golden.py.
"""
import numpy as np
import torch

from make_golden import import_reference, save_npz, smooth_flows


def main():
    dh, _, geometry, _, _ = import_reference()
    torch.manual_seed(0)
    N, C, h, w = 3, 1280, 5, 7
    fwd, bwd = smooth_flows(N, 8 * h, 8 * w, seed=11, mag=3.0)
    fo, bocc = geometry.forward_backward_consistency_check(fwd, bwd)
    g = torch.Generator().manual_seed(12)
    base = torch.randn(1, C, h, w, generator=g)
    sample = (base + 0.5 * torch.randn(2 * N, C, h, w, generator=g)).half()
    other = sample.float() + 0.7 * torch.randn(2 * N, C, h, w, generator=g)
    lv = other.reshape(2 * N, C, h * w).transpose(1, 2)
    lv = lv / ((lv ** 2).sum(dim=2, keepdim=True) ** 0.5)
    target = torch.bmm(lv, lv.transpose(-1, -2))
    losses = []
    orig_step = torch.optim.Adam.step

    def rec_step(self, closure=None):
        r = orig_step(self, closure)
        losses.append(float(r))
        return r

    torch.optim.Adam.step = rec_step
    out = {"sample": sample.numpy(), "target": target.numpy(), "fwd": fwd.numpy(), "bwd": bwd.numpy(),
           "fwd_occ": fo.numpy(), "bwd_occ": bocc.numpy()}
    for tag, kw in {"full1": dict(iters=1), "full4": dict(iters=4), "spatial4": dict(iters=4, optimize_temporal=False)}.items():
        losses.clear()
        o = dh.optimize_feature(sample.clone(), [fwd, bwd], [fo, bocc], correlation_matrix=[target], intra_weight=1e2,
                                **kw)
        out[f"{tag}_out"] = o.detach().numpy()
        out[f"{tag}_losses"] = np.array(losses, dtype=np.float64)
    torch.optim.Adam.step = orig_step
    save_npz("optimize_ragged", **out)


if __name__ == "__main__":
    main()
