"""Generate tests/golden/positive_tied.pt by running the REFERENCE's own FunctionalPositiveTiedSAE.loss
(autoencoders/mlp_tests.py:68-125, HoagyC/sparse_coding @ 69c5ae0) under ``vmap(grad)``, as
FunctionalEnsemble.init_functions drives it (ensemble.py:99-123).

TEST INFRASTRUCTURE. Run in the build container only (needs the reference tree, see make_golden.py):
    python oracle/make_positive_tied_golden.py

The file holds one fixture per case, each with the layout of the other fixtures (kind, params, buffers, batch, grads,
loss_data, c) plus ``init``: the seed and arguments that produce ``init_params`` through the reference's ``init`` (the
arguments in its own order: activation_size, n_dict_components, l1_alpha, bias_decay, dtype). ``params`` equals
``init_params`` except where a case edits the encoder after init. Cases:
  fresh           seeded init, three models with l1_alpha in {0, 1e-4, 1e-3} and bias_decay in {0, 0.01}, MLP-like data
                  (GELU of Gaussians rounded to fp16: the smallest value is about -0.17, so x + 0.18 stays positive)
  signed_encoder  the encoder after init given negative entries, exact zeros and one row with no positive entry (its
                  clamped row is zero, so it is normalised by the 1e-8 floor; its bias is positive, so its code is not
                  zero and its gradient is dW / 1e-8); a random bias around -1
  f64             fp64 parameters and batch
  ratio1          d = n, the dictionary ratio of the reference's run_positive sweep
``export`` (fresh, model 0) records the reference's to_learned_dict: its TiedSAE's learned dictionary, code and
prediction on the fixture batch.
"""
import os
import sys

import torch

from make_golden import OUT, import_reference, run_stacked


def mlp_like(B, d, gen):
    return torch.nn.functional.gelu(torch.randn(B, d, generator=gen)).half().float()


def main():
    import_reference()
    import autoencoders.mlp_tests as mt   # (on sys.path from import_reference)
    torch.set_grad_enabled(False)
    sig = mt.FunctionalPositiveTiedSAE
    cases = {}

    def case(name, d, n, B, l1s, bds, seed, dtype=torch.float32, edit=None):
        torch.manual_seed(seed)
        models = [sig.init(d, n, l1, bd, dtype=dtype) for l1, bd in zip(l1s, bds)]
        init_params = {k: torch.stack([p[k] for p, _ in models]) for k in models[0][0]}
        gen = torch.Generator().manual_seed(seed + 1)
        if edit is not None:
            models = [edit(p, b, gen) for p, b in models]
        X = mlp_like(B, d, gen).to(dtype)
        params, buffers, grads, loss_data, aux = run_stacked(sig, models, X)
        for i, (p, _) in enumerate(models):   # the reference's loss rebinds params["encoder"] in its own dict only
            assert torch.equal(p["encoder"], params["encoder"][i])
        cases[name] = dict(kind="positive_tied", params=params, buffers=buffers, batch=X, grads=grads,
                           loss_data=loss_data, c=aux["c"], init_params=init_params,
                           init=dict(seed=seed, d=d, n=n, l1=list(l1s), bias_decay=list(bds), dtype=dtype))
        return cases[name]

    def signed(p, b, gen):
        E = p["encoder"].clone()
        n, d = E.shape
        flip = torch.rand(n, d, generator=gen) < 0.3
        E[flip] = -E[flip]                                    # negative entries
        E[torch.rand(n, d, generator=gen) < 0.1] = 0.0        # exact zeros
        E[3] = -E[3].abs()                                    # no positive entry: E+ row = 0
        E[3, ::4] = 0.0
        bias = -1.0 + 0.2 * torch.randn(n, generator=gen)
        bias[3] = 0.5                                         # its code is the bias, so its gradient dW / 1e-8 is not 0
        return {"encoder": E, "encoder_bias": bias}, b

    fx = case("fresh", 32, 64, 48, [0.0, 1e-4, 1e-3], [0.01, 0.0, 0.01], 30)
    case("signed_encoder", 32, 64, 48, [1e-4, 1e-3], [0.01, 0.01], 31, edit=signed)
    case("f64", 32, 64, 40, [1e-4, 1e-3], [0.0, 0.01], 32, dtype=torch.float64)
    case("ratio1", 64, 64, 64, [0.0, 3e-4], [0.01, 0.01], 33)

    p = {k: v[0] for k, v in fx["params"].items()}
    b = {k: v[0] for k, v in fx["buffers"].items()}
    ld = sig.to_learned_dict(p, b)
    fx["export"] = dict(type=f"{type(ld).__module__}.{type(ld).__qualname__}", norm_encoder=ld.norm_encoder,
                        encoder=ld.encoder.clone(), encoder_bias=ld.encoder_bias.clone(),
                        learned_dict=ld.get_learned_dict(), encode=ld.encode(ld.center(fx["batch"])),
                        predict=ld.predict(fx["batch"]))

    path = os.path.join(OUT, "positive_tied.pt")
    torch.save(cases, path)
    print(f"wrote {path}  ({os.path.getsize(path) / 1024:.1f} KiB)")


if __name__ == "__main__":
    sys.exit(main())
