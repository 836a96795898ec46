"""Pin the CPU oracle's optimize_feature against the real reference at a decoder layer-0 shape with a token count that
is not a multiple of 8: [6, 1280, 5, 7] (35 tokens; layer 0 of a 320 x 448 frame), fp16 sample as the UNet passes it
(tests/golden/make_ragged_golden.py).  CPU only."""
import numpy as np
import torch

from oracle import fresco_oracle as O


def T(a):
    return torch.from_numpy(np.asarray(a))


def test_optimize_feature_ragged_layer0(golden):
    g = golden("optimize_ragged")
    sample, target = T(g["sample"]), T(g["target"])
    assert sample.shape == (6, 1280, 5, 7) and sample.dtype == torch.float16 and (5 * 7) % 8 != 0
    flows = [T(g["fwd"]), T(g["bwd"])]
    occs = [T(g["fwd_occ"]), T(g["bwd_occ"])]
    for tag, kw in {"full1": dict(iters=1), "full4": dict(iters=4),
                    "spatial4": dict(iters=4, optimize_temporal=False)}.items():
        out, trace = O.optimize_feature(sample, flows, occs, correlation_matrix=[target], intra_weight=1e2,
                                        return_trace=True, **kw)
        ref_losses = g[f"{tag}_losses"]
        mine = np.array([t["loss"] for t in trace])
        assert len(mine) == len(ref_losses) and np.allclose(mine, ref_losses, rtol=2e-4), (tag, mine, ref_losses)
        ref = T(g[f"{tag}_out"])
        assert out.dtype == ref.dtype == torch.float16
        diff = (out.float() - ref.float()).abs()
        if kw["iters"] == 1:
            # the fp16 output: at most one fp16 ulp apart (the fp32 values before the cast differ in the last bits)
            assert (diff <= 2.0 ** -9 * ref.float().abs() + 2.0 ** -24).all(), (tag, diff.max().item())
        else:
            assert diff.mean() / ref.float().abs().mean() < 5e-2, tag
