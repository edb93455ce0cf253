"""Generate tests/golden/nmf.pt by running the REFERENCE's own NMFEncoder (autoencoders/nmf.py: sklearn's NMF() with its
defaults, fitted in float64 on the CPU) and its exports.

TEST INFRASTRUCTURE. Run in the build container only (needs the reference tree and sklearn):
    python oracle/make_nmf_golden.py

sklearn.decomposition._nmf._update_cdnmf_fast is wrapped to record the violation of every sweep and the factor after
the first four (W, H^T, W, H^T of iterations 1 and 2; of W, its first 64 rows); _fit_coordinate_descent is wrapped to record transform's
iteration count.

Fits (datasets from oracle.nmf_oracle.nmf_rows, stored by seed; fp16 as the reference's chunks are):
  d16, d32     non-negative mixtures, N = 4000 / 8000; their singular values are checked to be well separated
  shift16      a mixture shifted below zero (the shift rule)
  rank12       d = 16 with 4 zero columns: 4 zero singular values, whose components NNDSVDA fills with the average
  sep16        a nearly diagonal mixture on which the fit converges (n_iter_ < max_iter), so the stop rule decides
  d32 again at max_iter = 1 and 3
Per fit: the sweeps above, n_iter_, components_, reconstruction_err_, the codes and transform iteration counts of two
held-out batches of 100 and 257 rows, and the raw rows of to_topk_dict. d16 also stores the pickled reference encoder,
and the TypeError the reference's encode raises after an fp32 fit, as text."""
import io
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_metrics_golden import import_reference  # noqa: E402
from nmf_oracle import nmf_rows  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "nmf.pt")
HELD = (100, 257)
HEAD = 64
CASES = {"d16": dict(d=16, n=4000, seed=1601), "d32": dict(d=32, n=8000, seed=3201),
         "shift16": dict(d=16, n=4000, seed=1602, signed=True), "rank12": dict(d=16, n=4000, seed=1603, rank=12),
         "sep16": dict(d=16, n=4000, seed=1607, separated=True)}


class Recorder:
    def __init__(self, nmf_mod):
        self.mod = nmf_mod
        self.sweeps, self.violations, self.n_iters = [], [], []

    def __enter__(self):
        upd, fcd = self.mod._update_cdnmf_fast, self.mod._fit_coordinate_descent

        def update(W, HHt, XHt, permutation):
            v = upd(W, HHt, XHt, permutation)
            self.violations.append(float(v))
            if len(self.sweeps) < 4:   # W: its first HEAD rows (rows are swept independently); H^T: whole
                self.sweeps.append(torch.from_numpy(np.array(W[:HEAD], dtype=np.float64)))
            return v

        def fit_cd(*a, **k):
            out = fcd(*a, **k)
            self.n_iters.append(int(out[2]))
            return out

        self.orig = (upd, fcd)
        self.mod._update_cdnmf_fast, self.mod._fit_coordinate_descent = update, fit_cd
        return self

    def __exit__(self, *exc):
        self.mod._update_cdnmf_fast, self.mod._fit_coordinate_descent = self.orig


def rows(case):
    c = dict(CASES[case])
    x = nmf_rows(c.pop("d"), c.pop("n") + sum(HELD), c.pop("seed"), **c)
    n = CASES[case]["n"]
    return x[:n], x[n:n + HELD[0]], x[n + HELD[0]:]


def run_fit(NMFEncoder, nmf_mod, case, max_iter=None, pickle=False):
    x, h1, h2 = rows(case)
    d = x.shape[1]
    enc = NMFEncoder(d)
    if max_iter is not None:
        enc.nmf.max_iter = max_iter
    with Recorder(nmf_mod) as rec:
        enc.train(x.clone())
    fit_sweeps = len(rec.violations)
    f = enc.nmf
    entry = {"max_iter": f.max_iter, "n_iter": int(f.n_iter_), "components": torch.from_numpy(f.components_.copy()),
             "err": float(f.reconstruction_err_), "shift": float(enc.shift), "sweeps": rec.sweeps,
             "violations": rec.violations[:fit_sweeps], "topk_rows": enc.to_topk_dict(4).dict.clone()}
    if max_iter is None:
        held = []
        for h in (h1, h2):
            with Recorder(nmf_mod) as r2:
                codes = enc.encode(h.clone())
            held.append({"codes": codes.double(), "n_iter": r2.n_iters[0]})
        entry["held"] = held
    if pickle:
        blob = io.BytesIO()
        torch.save(enc, blob)
        entry["pickle"] = blob.getvalue()
    return entry


def main():
    import_reference()
    from autoencoders.nmf import NMFEncoder  # the reference's (REF is first on sys.path)
    import sklearn
    import sklearn.decomposition._nmf as nmf_mod
    out = {"sklearn": sklearn.__version__, "cases": CASES, "held_rows": HELD, "fits": {}, "stopped": {}}
    for case in CASES:
        x = rows(case)[0].double()
        S = torch.linalg.svdvals(x)
        r = CASES[case].get("rank", x.shape[1])
        gap = float(((S[:r - 1] - S[1:r]) / S[:r - 1]).min())
        assert gap > 1e-3, f"{case}: singular values too close (relative gap {gap:.2e})"
        if r < x.shape[1]:
            assert float(S[r:].max()) == 0.0, case
        entry = run_fit(NMFEncoder, nmf_mod, case, pickle=case == "d16")
        entry["min_rel_gap"] = gap
        out["fits"][case] = entry
    for max_iter in (1, 3):
        out["stopped"][f"d32_it{max_iter}"] = run_fit(NMFEncoder, nmf_mod, "d32", max_iter=max_iter)
    # an fp32 dataset: the reference fits it in fp32, and its encode then raises
    x, h1, _ = rows("d16")
    enc = NMFEncoder(16)
    enc.train(x.float())
    try:
        enc.encode(h1.float())
        out["fp32_failure"] = None
    except Exception as e:   # noqa: BLE001 - recorded, not handled
        out["fp32_failure"] = f"{type(e).__name__}: {e}"
    out["fp32_components_dtype"] = str(enc.nmf.components_.dtype)
    torch.save(out, OUT)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")
    for k, v in out["fits"].items():
        print(k, "n_iter", v["n_iter"], "err", v["err"], "held n_iter", [h["n_iter"] for h in v["held"]],
              "gap", v["min_rel_gap"])
    print("fp32:", out["fp32_failure"])


if __name__ == "__main__":
    main()
