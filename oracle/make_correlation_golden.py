"""Generate tests/golden/code_correlation.pt from the REFERENCE's own dictionary classes: their ``encode`` of paired
rows, and the fp64 moments and correlation of every pair of those codes (oracle/correlation_oracle.py).

TEST INFRASTRUCTURE. Run in the build container only (needs the reference tree and sklearn):
    python oracle/make_correlation_golden.py

inter_dict_connections.ipynb's covariance cell is not reproduced literally: its running "means" are batch sums, so its
variances, covariances and correlations are not centred moments (SURVEY Q16). What is recorded is what the cell
intends, from the reference's own codes. Side a (width D_A) holds a TiedSAE with a dead feature (its code column is
all zero: zero variance, NaN correlations), an UntiedSAE, a TopKLearnedDict, a RandomDict (drawn after
torch.manual_seed), an IdentityReLU and an ICAEncoder fitted with sklearn; side b (width D_B) encodes the paired rows
x_b = [x_a, extra columns] with a TiedSAE whose rows TIE_COLS are one row of side a's TiedSAE feature 0 (same bias), so
that the best match of that feature is an exact tie, and an UntiedSAE. Each dictionary is stored as raw tensors with
its kind, with its code; each pair (a, b) stores the fp64 outputs but the covariance."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from make_metrics_golden import import_reference  # noqa: E402
from ica_oracle import mixed_sources  # noqa: E402
from oracle import correlation_oracle as CO  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "code_correlation.pt")
N_ROWS = 512
D_A, D_B = 32, 40
DEAD = 3            # side a's TiedSAE feature whose code is all zero
TIE_COLS = (2, 7)   # side b's TiedSAE rows equal to side a's TiedSAE row 0


def main():
    sm, ld, topk = import_reference()
    import autoencoders.ica as ref_ica
    g = torch.Generator().manual_seed(20261020)
    rn = lambda *s: torch.randn(*s, generator=g)
    t64 = lambda a: torch.from_numpy(np.array(a, dtype=np.float64))
    x_a = mixed_sources(D_A, N_ROWS, 21)[0].float()
    x_b = torch.cat([x_a, rn(N_ROWS, D_B - D_A)], 1)
    side_a, side_b = {}, {}

    enc = rn(40, D_A)
    bias = rn(40) * 0.3 - 0.3
    bias[DEAD] = -1e4
    side_a["tied"] = ({"kind": "tied", "encoder": enc, "encoder_bias": bias}, ld.TiedSAE(enc, bias, norm_encoder=True))
    e, dcd, b = rn(40, D_A) * 0.4, rn(40, D_A), rn(40) * 0.3 - 0.2
    side_a["untied"] = ({"kind": "untied", "encoder": e, "decoder": dcd, "encoder_bias": b}, ld.UntiedSAE(e, dcd, b))
    tk = topk.TopKEncoder.to_learned_dict({"dict": rn(40, D_A)}, {"sparsity": torch.tensor(5)})
    side_a["topk"] = ({"kind": "topk", "dict": tk.dict, "sparsity": 5}, tk)
    torch.manual_seed(77)
    rd = ld.RandomDict(D_A, 40)
    side_a["random"] = ({"kind": "random", "encoder": rd.encoder.clone(), "torch_seed": 77}, rd)
    side_a["identity"] = ({"kind": "identity"}, ld.IdentityReLU(D_A))
    np.random.seed(5)
    ica = ref_ica.ICAEncoder(D_A)
    ica.train(x_a)
    side_a["ica"] = ({"kind": "ica", "scaler_mean": t64(ica.scaler.mean_), "scaler_var": t64(ica.scaler.var_),
                      "scaler_scale": t64(ica.scaler.scale_), "components": t64(ica.ica.components_),
                      "mixing": t64(ica.ica.mixing_), "ica_mean": t64(ica.ica.mean_)}, ica)

    enc_b = rn(40, D_B)
    bias_b = rn(40) * 0.3 - 0.3
    for c in TIE_COLS:
        enc_b[c] = torch.cat([enc[0], torch.zeros(D_B - D_A)])
        bias_b[c] = bias[0]
    side_b["tied"] = ({"kind": "tied", "encoder": enc_b, "encoder_bias": bias_b}, ld.TiedSAE(enc_b, bias_b, norm_encoder=True))
    e, dcd, b = rn(40, D_B) * 0.4, rn(40, D_B), rn(40) * 0.3 - 0.2
    side_b["untied"] = ({"kind": "untied", "encoder": e, "decoder": dcd, "encoder_bias": b}, ld.UntiedSAE(e, dcd, b))

    codes = {}
    with torch.no_grad():
        for side, x, dicts in (("a", x_a, side_a), ("b", x_b, side_b)):
            for name, (_, learned) in dicts.items():
                codes[(side, name)] = learned.encode(x).float()
    c = codes[("a", "tied")]
    assert bool((c[:, DEAD] == 0).all())
    assert bool((codes[("b", "tied")][:, TIE_COLS[0]] == codes[("b", "tied")][:, TIE_COLS[1]]).all())
    pairs = {}
    for na in side_a:
        for nb in side_b:
            out = CO.correlation(codes[("a", na)], codes[("b", nb)])
            pairs[(na, nb)] = {k: v for k, v in out.items() if k != "covariance"}
            print(f"{na} x {nb}: NaN {int(torch.isnan(out['correlation']).sum())}, "
                  f"max |corr| {float(out['correlation'].nan_to_num().abs().max()):.3f}")
    tie = pairs[("tied", "tied")]
    assert int(tie["argmax_ab"][0]) == TIE_COLS[0], tie["argmax_ab"][0]
    torch.save({"x_a": x_a, "x_b": x_b, "dead": DEAD, "tie_cols": TIE_COLS,
                "side_a": {k: v[0] for k, v in side_a.items()}, "side_b": {k: v[0] for k, v in side_b.items()},
                "codes": codes, "pairs": pairs}, OUT)
    print("wrote", os.path.normpath(OUT), os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
