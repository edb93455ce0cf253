"""Generate tests/golden/tied_learned_center.pt by running the REFERENCE's own FunctionalTiedCenteredSAE.loss
(autoencoders/sae_ensemble.py:164-230, HoagyC/sparse_coding @ 69c5ae0) under ``vmap(grad)``, as
FunctionalEnsemble.init_functions drives it (ensemble.py:99-123).

TEST INFRASTRUCTURE. Run in the build container only (needs the reference tree, see make_golden.py):
    python oracle/make_learned_center_golden.py

The file holds one fixture per case, each with the layout of the other fixtures (kind, params including the centre,
buffers, batch, grads, loss_data, c) plus ``init``: the seed and arguments that produce its parameters through the
reference's ``init`` (the centre passed in, every other parameter from the seeded global generator). Cases:
  three_models   three models with non-zero centres, Gaussian data
  mean_offset    sparse-mixture data whose mean lies several times its spread from the origin, zero centres
  f64            fp64 parameters and batch, non-zero centres
  zero_center    zero centres; also records FunctionalTiedSAE's loss_data and gradients on the same encoder, bias and
                 batch (tied_loss_data, tied_grads), which the learned-centre signature must reproduce there
"""
import os

import torch

from make_golden import OUT, import_reference, run_stacked, sparse_mix


def main():
    sae, _, _ = import_reference()
    torch.set_grad_enabled(False)
    cases = {}

    def case(name, M, d, n, B, l1s, seed, data="gauss", dtype=torch.float32, center_scale=0.3, offset=0.0):
        gen = torch.Generator().manual_seed(seed + 1)
        centers = [(center_scale * torch.randn(d, generator=gen)).to(dtype) for _ in l1s]
        torch.manual_seed(seed)
        models = [sae.FunctionalTiedCenteredSAE.init(d, n, l1, center=c.clone(), dtype=dtype) for l1, c in zip(l1s, centers)]
        X = torch.randn(B, d, generator=gen) if data == "gauss" else sparse_mix(B, d, 2 * n, 5, gen)
        if offset:
            mu = torch.randn(d, generator=gen)
            X = X + offset * float(X.std()) * mu / float(mu.abs().mean())
        X = X.to(dtype)
        params, buffers, grads, loss_data, aux = run_stacked(sae.FunctionalTiedCenteredSAE, models, X)
        fx = dict(kind="tied_learned_center", params=params, buffers=buffers, batch=X, grads=grads, loss_data=loss_data,
                  c=aux["c"], init=dict(seed=seed, d=d, n=n, l1=list(l1s), centers=torch.stack(centers), dtype=dtype))
        cases[name] = fx
        return fx, models, X

    case("three_models", 3, 32, 64, 48, [1e-3, 3e-3, 1e-2], 20)
    case("mean_offset", 2, 64, 128, 96, [1e-4, 1e-2], 21, data="mix", center_scale=0.0, offset=4.0)
    case("f64", 2, 32, 64, 40, [1e-3, 1e-2], 22, dtype=torch.float64)
    fx, models, X = case("zero_center", 2, 32, 64, 40, [1e-3, 1e-2], 23, center_scale=0.0)
    tied = []
    for p, b in models:
        tp, tb = sae.FunctionalTiedSAE.init(32, 64, float(b["l1_alpha"]))
        tp = {"encoder": p["encoder"].clone(), "encoder_bias": p["encoder_bias"].clone()}
        tb["bias_decay"] = torch.tensor(0.0)   # reference quirk Q1: FunctionalTiedSAE.init never creates it
        tied.append((tp, tb))
    _, _, tgrads, tloss, _ = run_stacked(sae.FunctionalTiedSAE, tied, X)
    fx["tied_grads"], fx["tied_loss_data"] = tgrads, tloss

    path = os.path.join(OUT, "tied_learned_center.pt")
    torch.save(cases, path)
    print(f"wrote {path}  ({os.path.getsize(path) / 1024:.1f} KiB)")


if __name__ == "__main__":
    main()
