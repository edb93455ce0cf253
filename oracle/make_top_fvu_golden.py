"""Generate tests/golden/top_fvu.pt by running the REFERENCE's own fraction_variance_unexplained_top_activating
(standard_metrics.py:316-342) on the reference's own dictionary classes.

TEST INFRASTRUCTURE. Run in the build container only (needs the reference tree and sklearn):
    python oracle/make_top_fvu_golden.py

The reference is imported with the stubs of make_metrics_golden.py. Dictionaries: TiedSAE with identity centring and
with a non-trivial translation, rotation and scale, UntiedSAE, TopKLearnedDict, RandomDict and IdentityReLU, at d = 32
and 64, stored as raw tensors in the layouts oracle/top_fvu_oracle.py reads; and the d = 32 ICAEncoder fit of
make_baselines_golden.py, for which the exception text the reference raises is stored. Each is scored with n_top in
{1, 2, 5} on N_EVAL rows (not a multiple of the engine's segment). The rows' seed is searched until the fp64 mean code
has a gap of at least MIN_GAP (relative to the largest mean) at rank n_top for every n_top: the reference ranks fp32
means and the engine fp64 sums of its own code, so the choice must not hinge on a near tie. The gap is stored."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from make_metrics_golden import import_reference  # noqa: E402
from ica_oracle import mixed_sources  # noqa: E402
from oracle import top_fvu_oracle as TO  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "top_fvu.pt")
N_EVAL = TO.N_EVAL
N_TOPS = (1, 2, 5)
MIN_GAP = 1e-3


def main():
    sm, ld, topk = import_reference()
    import autoencoders.ica as ref_ica
    g = torch.Generator().manual_seed(20261018)
    rn = lambda *s: torch.randn(*s, generator=g)
    dicts = {}
    dicts["tied_identity"] = {"kind": "tied", "encoder": rn(64, 32), "encoder_bias": rn(64) * 0.3 - 0.4}
    dicts["tied_centred"] = {"kind": "tied", "encoder": rn(48, 32), "encoder_bias": rn(48) * 0.3 - 0.4,
                             "center_trans": rn(32) * 0.5, "center_rot": torch.eye(32) + 0.2 * rn(32, 32) / 32 ** 0.5,
                             "center_scale": torch.rand(32, generator=g) * 1.5 + 0.5}
    dicts["untied"] = {"kind": "untied", "encoder": rn(72, 64) * 0.4, "encoder_bias": rn(72) * 0.3 - 0.5,
                       "decoder": rn(72, 64)}
    dicts["topk"] = {"kind": "topk", "dict": topk.TopKEncoder.to_learned_dict({"dict": rn(48, 32)},
                                                                              {"sparsity": torch.tensor(4)}).dict,
                     "sparsity": 4}
    torch.manual_seed(148)
    rd = ld.RandomDict(64, 48)
    dicts["random"] = {"kind": "random", "encoder": rd.encoder.clone(), "encoder_bias": rd.encoder_bias.clone(),
                       "decoder": rd.encoder.clone(), "trans": torch.zeros(64)}
    ir = ld.IdentityReLU(32)
    dicts["identity_relu"] = {"kind": "identity_relu", "encoder": torch.eye(32), "encoder_bias": ir.bias.clone(),
                              "decoder": torch.eye(32), "trans": torch.zeros(32)}

    def make(e):
        if e["kind"] == "tied":
            cen = (e.get("center_trans"), e.get("center_rot"), e.get("center_scale"))
            return ld.TiedSAE(e["encoder"], e["encoder_bias"], centering=cen, norm_encoder=True)
        if e["kind"] == "untied":
            return ld.UntiedSAE(e["encoder"], e["decoder"], e["encoder_bias"])
        if e["kind"] == "topk":
            return topk.TopKLearnedDict(e["dict"], e["sparsity"])
        return rd if e["kind"] == "random" else ir

    f64 = lambda e: {k: (v.double() if torch.is_tensor(v) else v) for k, v in e.items()}
    cases = []
    for name, e in dicts.items():
        d = (e["dict"] if e["kind"] == "topk" else e["encoder"]).shape[1]
        for seed in range(1, 200):
            x = TO.rows(d, seed)
            c = TO.code(f64(e), x.double())
            top_mean = float(c.mean(dim=0).abs().max())
            gaps = [TO.mean_gap(c, k) / top_mean for k in N_TOPS]
            if min(gaps) >= MIN_GAP:
                break
        else:
            raise RuntimeError(f"{name}: no seed gives a gap of {MIN_GAP} at every n_top")
        for k in N_TOPS:
            with torch.no_grad():
                top, rest = sm.fraction_variance_unexplained_top_activating(make(e), x, n_top=k)
                mean = make(e).encode(make(e).center(x)).mean(dim=0)
            ref_top = torch.argsort(mean, descending=True)[:k]
            cases.append({"dict": name, "x_seed": seed, "n_top": k, "fvu_top": float(top), "fvu_rest": float(rest),
                          "top_features": ref_top.clone(), "gap": gaps[N_TOPS.index(k)]})
        print(f"{name}: d {d}, seed {seed}, relative gaps {['%.3g' % v for v in gaps]}")

    # ICAEncoder: the fit of make_baselines_golden.py at d = 32; the reference's decode of its fp64 code raises
    x, _ = mixed_sources(32, 4000, 11)
    np.random.seed(3)
    ica = ref_ica.ICAEncoder(32)
    ica.train(x.float())
    try:
        sm.fraction_variance_unexplained_top_activating(ica, x[:N_EVAL].float(), n_top=2)
        ica_error = None
    except Exception as err:     # noqa: BLE001 — the reference's failure is the recorded result
        ica_error = f"{type(err).__name__}: {err}"
    torch.save({"n_eval": N_EVAL, "n_tops": N_TOPS, "dicts": dicts, "cases": cases, "ica_error": ica_error}, OUT)
    print(f"wrote {len(cases)} cases to {os.path.normpath(OUT)}; ICA: {ica_error}")


if __name__ == "__main__":
    main()
