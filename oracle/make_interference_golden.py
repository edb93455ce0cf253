"""Generate tests/golden/interference.pt by running the REFERENCE's own calc_expected_interference
(big_sweep.py:43-57) on codes of the reference's own dictionary classes.

TEST INFRASTRUCTURE. Run in the build container only (needs the reference tree and sklearn):
    python oracle/make_interference_golden.py

big_sweep.py imports wandb and transformer_lens at module level, so the function definition alone is taken from the
parsed file and executed with torch (as make_resample_golden.py does for WorstIndices). The dictionaries are the
reference's TiedSAE (with a zero-norm row and a feature whose bias keeps its code column all zero), UntiedSAE,
TopKLearnedDict and an ICAEncoder fitted with sklearn. Each case stores the dictionary the reference's sweep would pass
(``get_learned_dict()``, fp32 [n, d]), the code (the reference's ``encode`` of N_ROWS Gaussian rows, fp32 [B, n]) with
crafted rows appended (single active features, all-zero rows; for ICA a signed row whose totals fall below the clamp),
and the reference's result. Rows of the ICA code with an active entry whose fp64 |totals| is below FRAGILE are dropped:
there c / totals is a difference of nearly equal terms, which no fp32 computation reproduces."""
import ast
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from make_golden import REF  # noqa: E402
from make_metrics_golden import import_reference  # noqa: E402
from ica_oracle import mixed_sources  # noqa: E402
from oracle import interference_oracle as IO  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "interference.pt")
N_ROWS = 300
FRAGILE = 1e-3


def import_calc_expected_interference():
    """The reference's calc_expected_interference, executed from its own source."""
    path = os.path.join(REF, "big_sweep.py")
    tree = ast.parse(open(path).read(), filename=path)
    node = next(n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "calc_expected_interference")
    ns = {"torch": torch}
    exec(compile(ast.Module(body=[node], type_ignores=[]), path, "exec"), ns)
    return ns["calc_expected_interference"]


def main():
    calc = import_calc_expected_interference()
    sm, ld, topk = import_reference()
    import autoencoders.ica as ref_ica
    g = torch.Generator().manual_seed(20261019)
    rn = lambda *s: torch.randn(*s, generator=g)
    cases = []

    def add(name, learned, x, extra_rows=(), drop_fragile=False):
        dictionary = learned.get_learned_dict().float()
        code = learned.encode(x).float()
        n = dictionary.shape[0]
        for row in extra_rows:
            code = torch.cat([code, row(dictionary, n)[None]])
        if drop_fragile:
            wn = IO.normalised(dictionary)
            totals = code.double() @ (wn @ wn.T).pow(2).T
            bad = ((code != 0) & (totals.abs() < FRAGILE)).any(1)
            bad[N_ROWS:] = False      # (the crafted rows are kept: their totals are checked below)
            code = code[~bad]
        out = calc(dictionary, code)
        cases.append({"name": name, "dictionary": dictionary, "code": code, "expected": out.float(),
                      "nz_counts": (code != 0).sum(0)})
        print(f"{name}: n {n}, rows {code.shape[0]}, mean L0 {(code != 0).sum(1).float().mean():.1f}, "
              f"|oracle - reference| / |reference| {((IO.expected_interference(dictionary, code) - out.double()).abs().max() / out.abs().max()):.1e}")

    def single(j, v):
        def row(_, n):
            r = torch.zeros(n)
            r[j] = v
            return r
        return row

    zero_row = lambda _, n: torch.zeros(n)
    d = 32
    x = rn(N_ROWS, d)
    enc = rn(64, d)
    enc[5] = 0.0                       # a zero-norm dictionary row (its code is relu(bias))
    bias = rn(64) * 0.3 - 0.4
    bias[5] = 0.2
    bias[9] = -1e4                     # an all-zero code column
    tied = ld.TiedSAE(enc, bias, norm_encoder=True)
    add("tied", tied, x, [single(3, 0.7), single(5, 0.2), zero_row])
    untied = ld.UntiedSAE(rn(72, d) * 0.4, rn(72, d), rn(72) * 0.3 - 0.5)
    add("untied", untied, x, [single(0, 1.5), zero_row])
    tk = topk.TopKEncoder.to_learned_dict({"dict": rn(48, d)}, {"sparsity": torch.tensor(4)})
    add("topk", tk, x, [single(7, 2.0)])
    # ICA: the reference's fit (sklearn, fp64) on mixed sources; its code is signed
    xs = mixed_sources(d, 2000, 11)[0]
    np.random.seed(3)
    ica = ref_ica.ICAEncoder(d)
    ica.train(xs.float())
    wn = IO.normalised(ica.get_learned_dict().float())
    cos2 = (wn @ wn.T).pow(2)
    cos2.fill_diagonal_(0.0)
    i, j = divmod(int(cos2.argmax()), d)
    assert float(cos2[i, j]) > 0.05, float(cos2[i, j])

    def signed(_, n):                  # c_i = 1, c_j = -2 / cos^2(i, j): totals_i = 1 - 2 < 0, clamped to 1e-8
        r = torch.zeros(n)
        r[i], r[j] = 1.0, -2.0 / float(cos2[i, j])
        return r
    add("ica", ica, xs[:N_ROWS].float(), [signed, single(1, -0.8), zero_row], drop_fragile=True)
    c = cases[-1]["code"][-3].double()
    t = c @ (wn @ wn.T).pow(2).T
    assert float(t[i]) < -0.5, float(t[i])
    torch.save({"n_rows": N_ROWS, "fragile": FRAGILE, "signed_feature": i, "cases": cases}, OUT)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
