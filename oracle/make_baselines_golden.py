"""Generate tests/golden/baselines.pt by running the REFERENCE's own baseline dictionaries (autoencoders/ica.py:18-58
ICAEncoder, learned_dict.py:86-127 IdentityReLU and RandomDict) through its own metrics (standard_metrics.py:305-314
mean_nonzero_activations / fraction_variance_unexplained, :446-454 batched_calc_feature_n_ever_active, :482-511
calc_moments_streaming).

TEST INFRASTRUCTURE. Run in the build container only (needs the reference tree and sklearn):
    python oracle/make_baselines_golden.py

The reference is imported with the stubs of make_metrics_golden.py. Cases:
  * ICA: the reference's ICAEncoder.train (sklearn's StandardScaler and FastICA() in fp64, np.random.seed(fit_seed) before
    the fit) on oracle.ica_oracle.mixed_sources at d = 32 and 64, stored by seed; the fitted arrays are stored as
    float64 tensors. Evaluated on the first N_EVAL rows of the training data, rounded to fp32.
  * RandomDict (torch.manual_seed before construction) and IdentityReLU, each also pickled with torch.save so that loading
    is checked on the real file format; evaluated on gaussian_rows(d, x_seed), which the tests regenerate.
Per case, on N_EVAL rows (not a multiple of the segment): the metrics above with batch_size = SEG, and the FVU or, where the
reference raises (ICA: decode multiplies its fp64 code by the fp32 dictionary), the exception text.

Record selection (interpret.py:82-212 make_feature_activation_dataset, :265-321 interpret), run as make_interp_golden.py
runs it, with its stubs and tiny model, for the d = 32 ICA fit and the n = 48 RandomDict, on N_FRAG fragments of 64 fp16
rows (stored): the first rows of the evaluation data, for ICA moved along four of its sources so that some fragment maxima
are negative. The fixture stores the reference's fp16 maxima table, the fragments its sort_values(...).head(20) selects per
feature, its captured top records and its skipped features."""
import asyncio
import io
import json
import os
import sys
import tempfile

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_metrics_golden import import_reference  # noqa: E402
from ica_oracle import mixed_sources  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "baselines.pt")
N_EVAL, SEG, THRESHOLD = 2500, 1000, 10
N_FRAG = 32                                              # fragments of the record-selection cases
ICA_FITS = [(32, 4000, 11, 3), (64, 6000, 12, 4)]     # (d, rows, data seed, fit seed)


def metrics(sm, ld, x):
    with torch.no_grad():
        out = {"mean_nonzero_activations": sm.mean_nonzero_activations(ld, x).double(),
               "n_ever_active": sm.batched_calc_feature_n_ever_active(ld, x, batch_size=SEG, threshold=THRESHOLD)}
        moments = sm.calc_moments_streaming(ld, x, batch_size=SEG)
        out["moments"] = {k: v.double() for k, v in zip(("times_active", "mean", "var", "skew", "kurtosis", "m4"),
                                                         moments)}
        try:
            out["fvu"] = float(sm.fraction_variance_unexplained(ld, x))
        except Exception as e:     # noqa: BLE001 — the reference's failure is the recorded result
            out["fvu_error"] = f"{type(e).__name__}: {e}"
    return out


def gaussian_rows(d, seed):
    """[N_EVAL, d] fp32 Gaussian rows with a per-column scale and offset, a function of (d, seed) alone."""
    g = torch.Generator().manual_seed(seed)
    scale, offset = 0.5 + torch.rand(d, generator=g), 0.3 * torch.randn(d, generator=g)
    return torch.randn(N_EVAL, d, generator=g) * scale + offset


def record_selection(ld, acts):
    """The reference's record selection for ``ld`` on the fp16 fragments ``acts`` [N_FRAG * L, d] (make_interp_golden.py's
    harness): {"maxes" [N_FRAG, n] fp16, "head" [n, 20], "top": {feature: fragments}, "skipped" [n] bool}."""
    import make_interp_golden as MI
    L, d = MI.L, acts.shape[1]
    n = int(ld.n_feats)
    with tempfile.TemporaryDirectory() as tmp:
        cwd = os.getcwd()
        os.chdir(tmp)
        try:
            with open("secrets.json", "w") as f:
                json.dump({"openai_key": "unused"}, f)
            import interpret as I
            I.load_dataset = lambda *a, **k: [{"text": str(i)} for i in range(N_FRAG + 40)]
            table = torch.cat([acts.float(), torch.zeros(40 * L + 1, d)])
            MI.CAPTURED.clear()
            torch.manual_seed(0)
            np.random.seed(0)
            with torch.no_grad():
                df = I.make_feature_activation_dataset(MI.TinyModel(table), ld, layer=2, layer_loc="residual",
                                                       device="cpu", n_fragments=N_FRAG)
            assert [int(t[0][1:]) // L for t in df["fragment_token_strs"]] == list(range(N_FRAG))
            asyncio.run(I.interpret(df, os.path.join(tmp, "out"), n_feats_to_explain=n))
            maxes = torch.tensor(np.stack([df[f"feature_{f}_max"].to_numpy() for f in range(n)], 1))
            top = {rec.neuron_id.neuron_index: torch.tensor([int(r.tokens[0][1:]) // L
                                                             for r in rec.most_positive_activation_records])
                   for rec in MI.CAPTURED}
            head = torch.stack([torch.tensor(df.sort_values(by=f"feature_{f}_max", ascending=False)
                                             .head(I.TOTAL_EXAMPLES).index.to_numpy()) for f in range(n)])
        finally:
            os.chdir(cwd)
    return {"acts": acts, "maxes": maxes, "head": head, "top": top,
            "skipped": torch.tensor([f not in top for f in range(n)])}


def pickled(obj):
    buf = io.BytesIO()
    torch.save(obj, buf)
    return buf.getvalue()


def main():
    import make_interp_golden as MI
    MI.import_harvest()          # (before the metrics stubs, as make_interp_golden.py orders them)
    MI.stub_neuron_explainer()
    sm, ld, _ = import_reference()
    import autoencoders.ica as ref_ica
    t = lambda a: torch.from_numpy(np.array(a, dtype=np.float64))
    out = {"n_eval": N_EVAL, "segment": SEG, "threshold": THRESHOLD, "n_frag": N_FRAG, "ica": [], "random": [], "identity_relu": []}
    for d, rows, seed, fit_seed in ICA_FITS:
        x, _ = mixed_sources(d, rows, seed)
        np.random.seed(fit_seed)
        ica = ref_ica.ICAEncoder(d)
        ica.train(x.float())
        xe = x[:N_EVAL].float()
        interp = None
        if d == 32:
            # rows moved by -8 sources along features 0, 1 (every fragment) and 2, 3 (the first half): their maxima are
            # negative there, and features 0 and 1 have no fragment with a non-negative maximum
            acts = x[: N_FRAG * 64].clone()
            move = lambda j: -8.0 * torch.from_numpy(ica.scaler.scale_ * ica.ica.mixing_[:, j])
            acts += move(0) + move(1)
            acts[: N_FRAG * 32] += move(2) + move(3)
            interp = record_selection(ica, acts.float().half())
        out["ica"].append({"d": d, "rows": rows, "seed": seed, "fit_seed": fit_seed, "interp": interp,
                           "scaler_mean": t(ica.scaler.mean_), "scaler_var": t(ica.scaler.var_),
                           "scaler_scale": t(ica.scaler.scale_), "components": t(ica.ica.components_),
                           "mixing": t(ica.ica.mixing_), "ica_mean": t(ica.ica.mean_),
                           "code": ica.encode(xe[:64]).double(), "metrics": metrics(sm, ica, xe)})
        print(f"ica d={d}: n_iter {ica.ica.n_iter_}, fvu: {out['ica'][-1]['metrics'].get('fvu_error')}")
    for d, n, seed in ((32, 32, 1), (32, 48, 2)):
        torch.manual_seed(100 + n)
        rd = ld.RandomDict(d, n)
        x = gaussian_rows(d, seed)
        interp = record_selection(rd, x[: N_FRAG * 64].half()) if n == 48 else None
        out["random"].append({"d": d, "n": n, "x_seed": seed, "encoder": rd.encoder.clone(), "pickle": pickled(rd),
                              "metrics": metrics(sm, rd, x), "interp": interp})
    d = 32
    ir = ld.IdentityReLU(d)
    out["identity_relu"].append({"d": d, "x_seed": 3, "pickle": pickled(ir), "metrics": metrics(sm, ir, gaussian_rows(d, 3))})
    try:
        ld.IdentityReLU(d, torch.ones(d))
        out["identity_relu_bias_error"] = None
    except Exception as e:     # noqa: BLE001
        out["identity_relu_bias_error"] = f"{type(e).__name__}: {e}"
    torch.save(out, OUT)
    print("wrote", os.path.normpath(OUT), os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
