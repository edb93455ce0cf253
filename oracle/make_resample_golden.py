"""Generate tests/golden/resample.pt: the reference's own worst-row list and its replacement rule on seeded data.

TEST INFRASTRUCTURE. Run in the build container only (needs the reference tree, see make_golden.py):
    python oracle/make_resample_golden.py

``WorstIndices`` (experiments/huge_batch_size.py:120-146) is run from the reference's own source (see
import_worst_indices) and fed per-row losses in batches as
process_reinit feeds it (:209-210). The replacement is inline in process_reinit, so its lines are restated here on the
reference's layout (UntiedSAE.encoder is [d, n], :74): c_totals == 0 (:226-227), get_worst(n_replace) (:231),
``encoder[:, replace_ndxs] = worst_vectors.T * 0.2 / torch.norm(encoder, dim=0).mean()`` (:237-240). Cases:
  worst      losses of 7 batches (the last one short), n_ndxs = 24: the reference's get_worst(24) indices
  replace    a dataset, its per-row losses and c_totals with 5 dead features: the reference-layout encoder before and
             after the replacement (fewer dead features than listed rows, as the reference needs)
Losses are tie-free (get_worst breaks exact ties by the larger index, SURVEY.md Q11).
"""
import ast
import os
import typing

import torch

from make_golden import OUT, REF


def import_worst_indices():
    """The reference's WorstIndices class, executed from its own source. The module cannot be imported whole under
    Python >= 3.11: its config dataclass (:347) has a list default, which dataclasses reject at import time, after
    WorstIndices is defined. So the class definition alone is taken from the parsed file and run with the names it
    uses (typing.List); nothing else of the module runs, so its other imports need no stubs."""
    path = os.path.join(REF, "experiments", "huge_batch_size.py")
    tree = ast.parse(open(path).read(), filename=path)
    node = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == "WorstIndices")
    ns = {"List": typing.List}
    exec(compile(ast.Module(body=[node], type_ignores=[]), path, "exec"), ns)
    return ns["WorstIndices"]


def main():
    WorstIndices = import_worst_indices()
    gen = torch.Generator().manual_seed(5)
    # worst: 7 batches of 16 rows, the last one 9
    losses = torch.randperm(10_000, generator=gen)[:105].double() / 997.0
    wi = WorstIndices(24)
    for r, loss in enumerate(losses.tolist()):
        wi.update(r, loss)
    worst = dict(losses=losses, batch_rows=[16] * 6 + [9], n_ndxs=24, get_worst=torch.tensor(wi.get_worst(24)))
    # replace: d = 16, n = 32, 80 rows
    d, n, N = 16, 32, 32
    data = torch.randn(80, d, generator=gen)
    row_losses = torch.randperm(10_000, generator=gen)[:80].double() / 991.0
    c_totals = torch.rand(n, generator=gen) + 0.1
    c_totals[torch.tensor([2, 7, 8, 19, 31])] = 0.0
    encoder = torch.randn(d, n, generator=gen)            # UntiedSAE.encoder layout [d, n]
    wi = WorstIndices(N)
    for r, loss in enumerate(row_losses.tolist()):
        wi.update(r, loss)
    before = encoder.clone()
    n_replace = int((c_totals == 0).sum().item())
    replace_ndxs = torch.where(c_totals == 0)[0]
    worst_vectors = data[wi.get_worst(n_replace)].to(torch.float32)
    av_encoder_norms = torch.norm(encoder, dim=0).mean()
    encoder[:, replace_ndxs] = worst_vectors.T * 0.2 / av_encoder_norms
    replace = dict(data=data, losses=row_losses, c_totals=c_totals, n_ndxs=N, encoder_before=before,
                   encoder_after=encoder, replace_ndxs=replace_ndxs)
    path = os.path.join(OUT, "resample.pt")
    torch.save({"worst": worst, "replace": replace}, path)
    print(f"wrote {path}  ({os.path.getsize(path) / 1024:.1f} KiB)")


if __name__ == "__main__":
    main()
