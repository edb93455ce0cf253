"""The f16f8 weight gradient on native E5M2 wgmma inside the engine: a tied ensemble large enough not to be launch-bound
(so the plan keeps batch-major copies of the 8-bit planes), a batch_max of 1210 (not a multiple of 16: padded pitch),
ragged batches after a larger one left stale rows, fp32 activations (x's residual plane is used), and the code read back
after the backward call (its residual plane then lives only in the batch-major copy). Checked against the fp64 oracle
on the GPU, with the activity pattern of near-kink coefficients taken from the engine (see test_engine_gpu.py)."""
import math

import pytest
import torch

from oracle import sae_oracle as O

pytestmark = pytest.mark.gpu

M, D, N, BMAX = 4, 512, 4096, 1210
REL = 1e-4


def _relnorm(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp(min=1e-30))


@pytest.mark.parametrize("B", [BMAX, 1037, 5])
def test_native_weight_gradient_ragged(B):
    import sparse_coding_b200 as S
    torch.manual_seed(0)
    models = []
    for a in torch.logspace(math.log10(1e-4), math.log10(1e-2), M).tolist():
        p, b = S.FunctionalTiedSAE.init(D, N, a)
        p["encoder_bias"] = 0.02 * torch.randn(N)
        models.append((p, b))
    ens = S.FunctionalEnsemble([({k: v.clone() for k, v in p.items()}, b) for p, b in models], S.FunctionalTiedSAE,
                               S.adam, {"lr": 1e-3}, device="cuda", arith="f16f8")
    gen = torch.Generator().manual_seed(B)
    ens.forward_batch(torch.randn(BMAX, D, generator=gen).cuda())   # plan with batch_max = BMAX, stale rows behind B
    X = torch.randn(B, D, generator=gen)
    grads, (loss, aux) = ens.grads_batch(X.cuda())
    code = aux["c"].dense()
    Xd = X.double().cuda()
    for i, (p, b) in enumerate(models):
        E, bias, alpha = p["encoder"].double().cuda(), p["encoder_bias"].double().cuda(), float(b["l1_alpha"])
        f0 = O.tied_forward(E, bias, Xd, alpha)
        win = max(1e-5, 1e-4 * float(f0["Z"].pow(2).mean().sqrt()))
        active = torch.where(f0["Z"].abs() < win, code[i] > 0, f0["Z"] > 0)
        f = O.tied_grads(E, bias, Xd, alpha, active=active)
        assert abs(float(loss["loss"][i]) - float(f["loss"])) <= REL * abs(float(f["loss"])), (B, i)
        assert _relnorm(code[i], f["c"]) <= REL, (B, i)
        assert _relnorm(grads["encoder"][i], f["grads"]["encoder"]) <= 2e-4, (B, i)
        assert _relnorm(grads["encoder_bias"][i], f["grads"]["encoder_bias"]) <= 2e-4, (B, i)
