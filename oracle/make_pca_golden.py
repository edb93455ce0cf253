"""Generate tests/golden/pca.pt by running the REFERENCE's own BatchedPCA (autoencoders/pca.py:41-110) and its exports.

TEST INFRASTRUCTURE. Run in the build container only (needs the reference tree):   python oracle/make_pca_golden.py

The reference is imported with make_metrics_golden.import_reference's stubs. Data: seeded rows with a prescribed, well
separated spectrum around a non-zero mean, fed in 500-row batches with a short tail, as fp32 and as fp64 (the same fp32-representable values; fp64 input
makes the reference's result fp64). Stored: the rows, the reference's mean, cov, eigendecomposition and centring
transform per input dtype, and, of the fp32 fit, the pickled PCAEncoder, Rotation, TopKLearnedDict and TiedSAE exports
(bytes of torch.save) with their encode / predict outputs on a held-out batch."""
import io
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_metrics_golden import import_reference  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "pca.pt")
D, N, BATCH, HELD = 48, 1337, 500, 64


def data(g):
    """[N + HELD, D] fp64 rows: mean + z diag(sqrt(lam)) Q^T, eigenvalues 1.25^-i (gaps of 25 %)."""
    q, _ = torch.linalg.qr(torch.randn(D, D, generator=g, dtype=torch.float64))
    lam = 4.0 * 1.25 ** -torch.arange(D, dtype=torch.float64)
    mu = 3.0 * torch.randn(D, generator=g, dtype=torch.float64)
    z = torch.randn(N + HELD, D, generator=g, dtype=torch.float64)
    return mu + (z * lam.sqrt()) @ q.T, lam


def main():
    import_reference()
    from autoencoders.pca import BatchedPCA  # the reference's (REF is first on sys.path)
    g = torch.Generator().manual_seed(20261016)
    rows, lam = data(g)
    x64, held64 = rows[:N].float().double(), rows[N:]      # fp32-representable rows: both fits see the same values
    out = {"d": D, "batch": BATCH, "lambda": lam, "x": x64.float(), "held": held64.float(), "fits": {}}
    for name, x in (("fp32", x64.float()), ("fp64", x64)):
        pca = BatchedPCA(D, "cpu")
        for i in range(0, N, BATCH):
            pca.train_batch(x[i:i + BATCH])
        vals, vecs = pca.get_pca()
        trans, rot, scale = pca.get_centering_transform()
        out["fits"][name] = {"mean": pca.get_mean().clone(), "cov": pca.cov.clone(), "eigvals": vals, "eigvecs": vecs,
                             "trans": trans.clone(), "rot": rot, "scale": scale, "dict": pca.get_dict()}
        if name != "fp32":
            continue
        held = held64.float()
        exports = {"pca_encoder": pca.to_learned_dict(5), "rotation": pca.to_rotation_dict(12),
                   "topk": pca.to_topk_dict(6), "pve_rotation": pca.to_pve_rotation_dict(10)}
        out["exports"] = {}
        for k, ld in exports.items():
            blob = io.BytesIO()
            torch.save(ld, blob)
            entry = {"pickle": blob.getvalue(), "encode": ld.encode(ld.center(held) if hasattr(ld, "center") else held)}
            if k != "rotation":      # Rotation.predict decodes with matrix rows of a different count: not defined
                entry["predict"] = ld.predict(held)
            out["exports"][k] = entry
    torch.save(out, OUT)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
