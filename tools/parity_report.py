"""Parity report: the engine (through the C ABI) against the golden vectors recorded from the reference's own loss
functions, one line per fixture and model. Run on a GPU:  python tools/parity_report.py"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import sparse_coding_b200 as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIG = {"tied": S.FunctionalTiedSAE, "untied": S.FunctionalSAE, "masked_tied": S.FunctionalMaskedTiedSAE,
       "masked_untied": S.FunctionalMaskedSAE, "topk": S.TopKEncoder}


def rn(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm().clamp(min=1e-30))


print("# engine vs reference golden vectors (tests/golden/*.pt): relative errors; bar 1e-4 on losses / code / x_hat")
print(f"{'fixture':16s} {'model':>5s} {'loss':>9s} {'l_rec':>9s} {'l_l1':>9s} {'code':>9s} {'nnz ref/eng':>13s}  gradients (norm-relative)")
for name in ["tied_small", "tied_bias", "tied_f64", "tied_centered", "untied_small", "masked_tied", "masked_untied",
             "topk_small", "cfg1"]:
    fx = torch.load(os.path.join(ROOT, "tests", "golden", name + ".pt"), weights_only=False)
    M = next(iter(fx["params"].values())).shape[0]
    models = [({k: v[i].float().clone() for k, v in fx["params"].items()},
               {k: (v[i].float().clone() if v.dtype.is_floating_point else v[i].clone()) for k, v in fx["buffers"].items()})
              for i in range(M)]
    ens = S.FunctionalEnsemble(models, SIG[fx["kind"]], S.adam, {"lr": 1e-3}, device="cuda")
    grads, (loss, aux) = ens.grads_batch(fx["batch"].float().cuda())
    c = aux["c"].dense().cpu()
    for i in range(M):
        rel = lambda k: (abs(float(loss[k][i]) - float(fx["loss_data"][k][i])) / max(abs(float(fx["loss_data"][k][i])), 1e-30)
                         if k in fx["loss_data"] else float("nan"))
        if "c" in fx:
            code = rn(c[i], fx["c"][i])
            nnz = f"{int(fx['c'][i].count_nonzero())}/{int(c[i].count_nonzero())}"
        else:
            code = rn(c[i].double().sum(-1), fx["c_sum"][i])
            nnz = f"{int(fx['c_nnz'][i].sum())}/{int(c[i].count_nonzero())}"
        g = "  ".join(f"{k} {rn(grads[k][i], fx['grads'][k][i]):.1e}" for k in fx["grads"])
        print(f"{name:16s} {i:5d} {rel('loss'):9.1e} {rel('l_reconstruction'):9.1e} {rel('l_l1'):9.1e} {code:9.1e} {nnz:>13s}  {g}")
