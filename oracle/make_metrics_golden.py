"""Generate tests/golden/dict_metrics.pt by running the REFERENCE's own dictionary metrics (standard_metrics.py:270-303
mcs_duplicates / mmcs / mcs_to_fixed / mmcs_to_fixed / mmcs_from_list / representedness, :356-362 capacity_per_feature)
on the reference's own LearnedDict classes.

TEST INFRASTRUCTURE. Run in the build container only (needs the reference tree):   python oracle/make_metrics_golden.py

standard_metrics.py imports modules that are not installed here (matplotlib, transformer_lens, torchtyping, the
reference's activation_dataset; torchopt / optree through the autoencoders package). None is used by these functions,
so they are replaced by inert stubs; the arithmetic recorded is the reference's.

The fixture stores every input dictionary as raw tensors with its kind (see oracle/metrics_oracle.py) and, per case,
the function, its arguments (names of stored dictionaries) and the reference's result."""
import os
import sys
import types

import torch

REF = os.environ.get("SCE_REFERENCE", "/root/reference")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "dict_metrics.pt")


def import_reference():
    class _Any(types.ModuleType):
        def __getattr__(self, name):
            if name.startswith("__"):
                raise AttributeError(name)
            return _Any(name)

        def __call__(self, *a, **k):
            return _Any("call")

    for name in ("torchopt", "optree", "matplotlib", "matplotlib.pyplot", "transformer_lens", "activation_dataset"):
        sys.modules.setdefault(name, _Any(name))
    tt = types.ModuleType("torchtyping")

    class _TT:
        def __class_getitem__(cls, item):
            return cls

    tt.TensorType = _TT
    sys.modules.setdefault("torchtyping", tt)
    sys.path.insert(0, REF)
    import standard_metrics as sm  # noqa
    import autoencoders.learned_dict as ld  # noqa
    import autoencoders.topk_encoder as topk  # noqa
    return sm, ld, topk


def main():
    sm, ld, topk = import_reference()
    g = torch.Generator().manual_seed(20261015)
    rn = lambda *s: torch.randn(*s, generator=g)
    d = 48
    dicts = {}     # name -> (kind, raw tensor)
    dicts["tied_a"] = ("tied", rn(200, d))
    dicts["tied_b"] = ("tied", rn(136, d))
    dicts["untied_c"] = ("untied", rn(72, d))
    topk_params = rn(96, d)
    dicts["topk_d"] = ("topk", topk.TopKEncoder.to_learned_dict({"dict": topk_params},
                                                                 {"sparsity": torch.tensor(4)}).dict)
    stack = rn(3, 64, d)                                  # a masked stack: encoder[:dict_size] is what gets exported
    for m, k in enumerate((40, 64, 17)):
        dicts[f"masked_{m}"] = ("tied", stack[m, :k].clone())
    dicts["tiny_a"] = ("tied", rn(8, 8))                  # odd shapes: n, d down to 8
    dicts["tiny_b"] = ("untied", rn(21, 8))
    dicts["odd_a"] = ("tied", rn(13, 40))
    dicts["odd_b"] = ("tied", rn(131, 40))
    dicts["pos"] = ("tied", rn(30, d).abs() + 0.05)       # every cosine between pos and neg is negative
    dicts["neg"] = ("tied", -(rn(45, d).abs() + 0.05))
    zr = rn(24, d)
    zr[5] = 0.0
    dicts["zero_row"] = ("tied", zr)
    dicts["truth"] = ("raw", rn(50, d) * 3.0)             # a ground-truth matrix, used as given
    dicts["truth_odd"] = ("raw", rn(19, 40) * 0.25)

    def make(name):
        kind, w = dicts[name]
        if kind == "tied":
            return ld.TiedSAE(w, torch.zeros(w.shape[0]), norm_encoder=True)
        if kind == "untied":
            return ld.UntiedSAE(torch.zeros_like(w), w, torch.zeros(w.shape[0]))
        if kind == "topk":
            return topk.TopKLearnedDict(w, 4)
        return w

    cases = []

    def case(fn, *args):
        objs = [[make(a) for a in x] if isinstance(x, list) else make(x) for x in args]
        with torch.no_grad():
            out = getattr(sm, fn)(*objs)
        cases.append({"fn": fn, "args": list(args), "out": out.clone()})

    pairs = [("tied_a", "tied_b"), ("tied_b", "tied_a"), ("tied_a", "untied_c"), ("untied_c", "topk_d"),
             ("topk_d", "tied_a"), ("masked_0", "masked_1"), ("masked_2", "masked_1"), ("tiny_a", "tiny_b"),
             ("odd_a", "odd_b"), ("odd_b", "odd_a"), ("pos", "neg"), ("neg", "pos"), ("zero_row", "tied_b")]
    for x, y in pairs:
        case("mcs_duplicates", x, y)
        case("mmcs", x, y)
    for m in ("tied_a", "untied_c", "topk_d", "masked_2", "zero_row"):
        case("mcs_to_fixed", m, "truth")
        case("mmcs_to_fixed", m, "truth")
        case("representedness", "truth", m)
    case("mcs_to_fixed", "odd_b", "truth_odd")
    case("representedness", "truth_odd", "odd_a")
    case("mmcs_from_list", ["tied_a", "tied_b", "untied_c", "topk_d"])
    case("mmcs_from_list", ["masked_0", "masked_1", "masked_2"])
    case("mmcs_from_list", ["odd_a", "odd_b"])
    for m in ("tied_a", "untied_c", "topk_d", "masked_0", "tiny_a", "odd_b", "zero_row"):
        case("capacity_per_feature", m)
    torch.save({"dicts": {k: {"kind": v[0], "w": v[1]} for k, v in dicts.items()}, "cases": cases,
                "topk_params": topk_params, "masked_stack": stack, "masked_sizes": [40, 64, 17]}, OUT)
    print(f"wrote {len(cases)} cases to {os.path.normpath(OUT)}")


if __name__ == "__main__":
    main()
