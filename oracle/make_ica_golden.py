"""Generate tests/golden/ica.pt by running the REFERENCE's own ICAEncoder.train (autoencoders/ica.py:18-58: sklearn's
StandardScaler and FastICA() in float64 on the CPU) and its exports.

TEST INFRASTRUCTURE. Run in the build container only (needs the reference tree and sklearn):
    python oracle/make_ica_golden.py

np.random.seed(fit_seed) is set before each fit, so FastICA's w_init is the first normal draw of numpy's global RNG after
it; the fixture stores that w_init. sklearn's _sym_decorrelation is wrapped to record every iterate W_k of the parallel
update, from which the lim of each iteration follows (max_i | |(W_k W_{k-1}^T)_ii| - 1 |).

Fits:
  (a) test/test_ica.py's data: Laplace 1000 x 2 (np.random.seed(0)) and 1000 x 4 (seed 42), stored as they are;
  (b) oracle.ica_oracle.mixed_sources at d = 32 (N = 8000) and d = 64 (N = 16000), stored by seed; their correlation
      eigenvalues are checked to be well separated, since whitening is not unique in a degenerate eigenspace;
  (c) case (b) at max_iter = 1 and 3.
Per fit of (a) and (b): w_init, W after 1 and 3 iterations, the lims, the scaler's and FastICA's fitted arrays, the
first 64 training sources and those of a 64-row held-out block, and (a and d = 32) the pickled reference ICAEncoder;
per fit of (c): the lims, n_iter and the fitted W and components. The reference's to_topk_dict passes raw numpy
components_ to TopKLearnedDict, whose encode then fails (matmul rejects a numpy array); that failure is recorded as
text."""
import io
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_metrics_golden import import_reference  # noqa: E402
from ica_oracle import mixed_sources  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "ica.pt")
HELD = 64


def run_fit(ICAEncoder, fastica_mod, x, held, fit_seed, max_iter=None, pickle=False):
    iterates = []
    orig = fastica_mod._sym_decorrelation

    def recording(W):
        out = orig(W)
        iterates.append(out.copy())
        return out

    fastica_mod._sym_decorrelation = recording
    try:
        np.random.seed(fit_seed)
        w_init = np.random.normal(size=(x.shape[1], x.shape[1]))
        np.random.seed(fit_seed)
        ica = ICAEncoder(x.shape[1])
        if max_iter is not None:
            ica.ica.max_iter = max_iter
        sources = ica.train(x)
    finally:
        fastica_mod._sym_decorrelation = orig
    lims = [float(np.max(np.abs(np.abs(np.einsum("ij,ij->i", b, a)) - 1))) for a, b in zip(iterates, iterates[1:])]
    f, s = ica.ica, ica.scaler
    t = lambda a: torch.from_numpy(np.array(a, dtype=np.float64))
    entry = {"fit_seed": fit_seed, "max_iter": ica.ica.max_iter, "w_init": t(w_init), "lims": lims,
             "W1": t(iterates[1]), "n_iter": int(f.n_iter_),
             "scaler": {"mean": t(s.mean_), "var": t(s.var_), "scale": t(s.scale_), "n": int(s.n_samples_seen_)},
             "ica": {"components": t(f.components_), "mixing": t(f.mixing_), "mean": t(f.mean_),
                     "whitening": t(f.whitening_), "unmixing": t(f._unmixing)},
             "train_sources_head": t(sources[:HELD]), "held_sources": ica.encode(held).double()}
    if len(iterates) > 3:
        entry["W3"] = t(iterates[3])
    if pickle:
        blob = io.BytesIO()
        torch.save(ica, blob)
        entry["pickle"] = blob.getvalue()
    return ica, entry


def main():
    import_reference()
    from autoencoders.ica import ICAEncoder  # the reference's (REF is first on sys.path)
    import sklearn
    import sklearn.decomposition._fastica as fastica_mod
    out = {"sklearn": sklearn.__version__, "held_rows": HELD, "fits": {}, "stopped": {}}

    # (a) test_ica.py's data
    for name, seed, d in (("laplace2", 0, 2), ("laplace4", 42, 4)):
        np.random.seed(seed)
        x = torch.tensor(np.random.laplace(0, 1, (1000 + HELD, d)))
        ica, entry = run_fit(ICAEncoder, fastica_mod, x[:1000], x[1000:], fit_seed=seed + 1, pickle=True)
        entry.update({"x": x[:1000].clone(), "held": x[1000:].clone()})
        out["fits"][name] = entry
        if name == "laplace2":
            try:
                ica.to_topk_dict(1).encode(x[:4].float())
                out["topk_failure"] = None
            except Exception as e:   # noqa: BLE001 - recorded, not handled
                out["topk_failure"] = f"{type(e).__name__}: {e}"

    # (b), (c) mixed sources
    for d, n, seed in ((32, 8000, 3201), (64, 16000, 6401)):
        rows, _ = mixed_sources(d, n + HELD, seed)
        x, held = rows[:n], rows[n:]
        c = torch.corrcoef(x.T)
        lam = torch.linalg.eigvalsh(c)
        gap = float(((lam[1:] - lam[:-1]) / lam[1:]).min())
        assert gap > 1e-3, f"d={d}: correlation eigenvalues too close (relative gap {gap:.2e})"
        _, entry = run_fit(ICAEncoder, fastica_mod, x, held, fit_seed=seed, pickle=d == 32)
        entry.update({"data_seed": seed, "n": n, "d": d, "min_rel_gap": gap})
        out["fits"][f"mixed{d}"] = entry
        for max_iter in (1, 3):   # the same fit stopped early: w_init and the iterates are the entry above's
            _, e = run_fit(ICAEncoder, fastica_mod, x, held, fit_seed=seed, max_iter=max_iter)
            out["stopped"][f"mixed{d}_it{max_iter}"] = {
                "base": f"mixed{d}", "max_iter": max_iter, "lims": e["lims"], "n_iter": e["n_iter"],
                "components": e["ica"]["components"], "unmixing": e["ica"]["unmixing"]}
    torch.save(out, OUT)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
