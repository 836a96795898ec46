"""The FMA-pipe exponential of the POLY attention variants (exp2_poly, attn_wgmma.cu), restated in torch on the CPU:
clamp, round-to-nearest by the 1.5 * 2^23 trick, degree-3 minimax on [-0.5, 0.5], exponent patched in with an integer
add.  Its error must stay inside the fp16 rounding of P, and very negative arguments (masked keys) must give ~0."""
import torch


def exp2_poly(t):
    """exp2_poly of attn_wgmma.cu in fp32."""
    t = torch.clamp(t, min=-126.0)
    magic = torch.tensor(12582912.0)
    r = t + magic
    n = r - magic
    f = t - n
    q = torch.tensor(0.05517164617776871) * f + torch.tensor(0.2426111251115799)
    q = q * f + torch.tensor(0.6932609677314758)
    q = q * f + torch.tensor(0.9999280571937561)
    bits = q.view(torch.int32) + (r.view(torch.int32) << 23)
    return bits.view(torch.float32)


def test_polynomial_exp2_error_and_range():
    t = torch.linspace(-100.0, 9.0, 200001)                         # (P is fp16: anything below 2^-25 rounds to zero anyway)
    ref = torch.exp2(t.double())
    rel = ((exp2_poly(t).double() - ref) / ref).abs().max().item()
    assert rel < 1e-4, rel                                          # 7.5e-5 by design: inside the fp16 rounding of P
    edge = exp2_poly(torch.tensor([-1e30, -140.0, -126.0, 0.0, 8.0]))
    assert torch.isfinite(edge).all() and (edge[:3] < 2e-38).all() and abs(edge[3].item() - 1.0) < 1e-4
