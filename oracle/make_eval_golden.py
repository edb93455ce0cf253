"""Generate tests/golden/dict_eval.pt by running the REFERENCE's own dictionary scores (standard_metrics.py:305-314
mean_nonzero_activations / fraction_variance_unexplained, :344-345 r_squared, :446-454
batched_calc_feature_n_ever_active, :482-511 calc_moments_streaming) on the reference's own LearnedDict classes.

TEST INFRASTRUCTURE. Run in the build container only (needs the reference tree):   python oracle/make_eval_golden.py

The reference is imported with the stubs of make_metrics_golden.py. The fixture stores every dictionary as raw tensors
with its kind (the layout oracle/eval_oracle.py reads), the activation sets, and per case the function, its
arguments (names of a dictionary and an activation set, then keyword arguments) and the reference's result."""
import os

import torch

from make_metrics_golden import import_reference

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "dict_eval.pt")


def main():
    sm, ld, topk = import_reference()
    g = torch.Generator().manual_seed(20261016)
    rn = lambda *s: torch.randn(*s, generator=g)
    d = 32
    dicts = {}
    # non-trivial centring: translation, a non-orthogonal rotation, a non-uniform scale
    dicts["tied_centred"] = {"kind": "tied", "encoder": rn(64, d), "encoder_bias": rn(64) * 0.3 - 0.6,
                             "center_trans": rn(d) * 0.5, "center_rot": torch.eye(d) + 0.2 * rn(d, d) / d ** 0.5,
                             "center_scale": torch.rand(d, generator=g) * 1.5 + 0.5}
    b = rn(37) * 0.3 - 0.8
    b[3] = -1e3                                                # a feature that never fires
    dicts["tied_odd"] = {"kind": "tied", "encoder": rn(37, d), "encoder_bias": b}     # n not a multiple of 8
    dicts["untied"] = {"kind": "untied", "encoder": rn(48, d) * 0.4, "encoder_bias": rn(48) * 0.3 - 0.7,
                       "decoder": rn(48, d)}
    dicts["topk"] = {"kind": "topk", "dict": topk.TopKEncoder.to_learned_dict({"dict": rn(48, d)},
                                                                              {"sparsity": torch.tensor(4)}).dict,
                     "sparsity": 4}
    acts = {"x2500": rn(2500, d) * 1.5 + 0.3, "x600": rn(600, d)}    # N not a multiple of 1000, and N < 1000

    def make(name):
        e = dicts[name]
        if e["kind"] == "tied":
            cen = (e.get("center_trans"), e.get("center_rot"), e.get("center_scale"))
            return ld.TiedSAE(e["encoder"], e["encoder_bias"], centering=cen, norm_encoder=True)
        if e["kind"] == "untied":
            return ld.UntiedSAE(e["encoder"], e["decoder"], e["encoder_bias"])
        return topk.TopKLearnedDict(e["dict"], e["sparsity"])

    cases = []

    def case(fn, name, xs, **kw):
        with torch.no_grad():
            out = getattr(sm, fn)(make(name), acts[xs], **kw)
        out = tuple(o.clone() for o in out) if isinstance(out, tuple) else (out.clone() if torch.is_tensor(out) else out)
        cases.append({"fn": fn, "dict": name, "acts": xs, "kwargs": kw, "out": out})

    for name in dicts:
        for xs in acts:
            case("fraction_variance_unexplained", name, xs)
            case("r_squared", name, xs)
            case("mean_nonzero_activations", name, xs)
            case("batched_calc_feature_n_ever_active", name, xs)
            case("calc_moments_streaming", name, xs)
        case("calc_moments_streaming", "tied_odd", "x2500", batch_size=700)
        # threshold equal to a feature's count: that feature is not "ever active" (count > threshold)
        with torch.no_grad():
            counts = (make(name).encode(acts["x2500"]) != 0).sum(0)
        t = int(counts[counts > 0].min())
        case("batched_calc_feature_n_ever_active", name, "x2500", threshold=t)
        case("batched_calc_feature_n_ever_active", name, "x2500", batch_size=333, threshold=t)
    torch.save({"dicts": dicts, "acts": acts, "cases": cases}, OUT)
    print(f"wrote {len(cases)} cases to {os.path.normpath(OUT)}")


if __name__ == "__main__":
    main()
