"""Top-k selection and the k-sparse kernels on inputs the engine computes exactly, compared with no tolerance.

Each dictionary row holds 4 entries of +-1 (norm 2), so the dictionary-row kernel normalises it to entries of +-1/2 with
all-zero residual planes; the activations are integers in [-R, R]. Every score is then a multiple of 1/2 below 2^10
(at most 11 significant bits), and every product, tensor-core accumulation, fp16 / bf16 plane and fp32 gather sum the
forward pass forms is exact, in f16f8 and in bf16x3. So the code (which columns, which of tied columns, which values),
x^ and the mean count are compared bitwise against a plain fp64 restatement of TopKEncoder.encode with the engine's tie
rule (SURVEY Q8: among equal scores the lowest column is kept). The loss adds fp32 partial sums of r^2 (1e-6 relative);
the dictionary gradient rounds the code-gradient planes (1e-4 relative, against the fp64 gradient on the reference's own
support). Multi-call tests use lr = 0: the step runs every launch (selection, gather, scatter, dW, Adam, re-split,
graph replay where the shape is launch-bound) and leaves the parameters bitwise unchanged, so the inputs stay exact.

Branches of topk_select2_kernel (sce_topk.cuh), n_chunks = ceil(n / 32), full_warps = min(8, n_chunks / 32), and the
case that reaches each:
  whole row, counting ranks (n_chunks < 32)           whole-row-n256
  chunk-maxima path, k up to 32 per full warp          fused-n1040-k32, fused-n2048-k64, fused-n8192-k256
  chunk-maxima path refused by the per-warp limit      whole-row-n1040-k33, whole-row-n2048-k65
  chunk-maxima path refused by n_chunks > 2048         whole-row-n65552-over-2048-chunks
  counting with parts == 1 (exactly 1024 candidates)   count-1024-candidates
  radix select + ordered tie compaction                radix-n2048-all-equal, radix-n8192-periodic, radix-k300-*
  k == n                                               whole-row-n256 (k = 256)
and of the gather kernel (topk_sparse_kernel): its k classes {<= 16, <= 32, <= 64, <= k_max} and 2, 4 or 8 slices of
the activation width, named in the gather-* ids. `classes` in the case table is the number of gather launches a call
makes (0: the dense decode GEMM), which the launch count of every call pins.
"""
import pytest
import torch

import sparse_coding_b200 as S
from oracle import interp_oracle as IO
from oracle import sae_oracle as O
from oracle.plan_paths import gather_classes, launch_bound, launches
from sparse_coding_b200 import metrics as MT

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


# ----------------------------------------------------------------------------------------------------------------
# exact inputs
# ----------------------------------------------------------------------------------------------------------------
def grid_dict(n, d, pattern, gen, nonneg=False, period=5):
    """[n, d] fp32 rows of 4 entries +-1 at distinct columns. ``pattern``: "random" (a random 4-subset per row, moderate
    ties), "periodic" (``period`` random rows repeated: every score appears n / period times in a row), "equal" (one
    row repeated: every score of a row ties)."""
    rows = {"random": n, "periodic": period, "equal": 1}[pattern]
    W = torch.zeros(rows, d)
    cols = torch.rand(rows, d, generator=gen).argsort(dim=-1)[:, :4]
    signs = torch.ones(rows, 4) if nonneg else torch.randint(0, 2, (rows, 4), generator=gen).float() * 2 - 1
    W.scatter_(1, cols, signs)
    return W.repeat((n + rows - 1) // rows, 1)[:n].contiguous()


def grid_batch(B, d, kinds, gen, R=8):
    """[B, d] integer rows, row i of kind ``kinds[i % len(kinds)]``: "rand" (uniform in [-R, R]), "tie" (two non-zero
    entries: few distinct scores, many ties), "zero", "neg" (in [-R, -1])."""
    x = torch.zeros(B, d)
    for i in range(B):
        kind = kinds[i % len(kinds)]
        if kind == "rand":
            x[i] = torch.randint(-R, R + 1, (d,), generator=gen).float()
        elif kind == "tie":
            x[i, torch.randint(0, d, (2,), generator=gen)] = torch.randint(-R, R + 1, (2,), generator=gen).float()
        elif kind == "neg":
            x[i] = torch.randint(-R, 0, (d,), generator=gen).float()
    return x


def ref_topk(W, X, k):
    """fp64 TopKEncoder.encode with the engine's tie rule: scores against the normalised rows, a stable descending sort
    (ties to the lowest column), the first min(k, n), ReLU. Returns (scores, code, selected, x_hat)."""
    Wn = W.double() / W.double().norm(dim=-1, keepdim=True)
    Sc = X.double() @ Wn.T
    idx = torch.sort(Sc, dim=-1, descending=True, stable=True).indices[:, :min(int(k), Sc.shape[-1])]
    sel = torch.zeros_like(Sc, dtype=torch.bool).scatter_(-1, idx, True)
    code = torch.where(sel, Sc, torch.zeros_like(Sc)).clamp(min=0.0)
    return Sc, code, sel, code @ Wn


def sig_bits_at_most(t, bits):
    m, _ = torch.frexp(t)
    return bool((m * 2.0 ** bits == torch.round(m * 2.0 ** bits)).all())


def assert_exact_inputs(Sc, code, x_hat):
    """The precondition of every exact comparison below, checked on the fp64 reference."""
    assert sig_bits_at_most(Sc, 11) and sig_bits_at_most(code, 11)
    q = x_hat * 16
    assert bool((q == torch.round(q)).all()) and bool((x_hat.abs() < 2.0 ** 18).all())


# ----------------------------------------------------------------------------------------------------------------
# one ensemble, compared call by call
# ----------------------------------------------------------------------------------------------------------------
def make_ensemble(W, ks, arith):
    models = [({"dict": W[m].clone()}, {"sparsity": torch.tensor(int(k), dtype=torch.long)}) for m, k in enumerate(ks)]
    return S.FunctionalEnsemble(models, S.TopKEncoder, S.adam, {"lr": 0.0}, device=DEV, arith=arith, no_stacking=True)


class Checker:
    def __init__(self, W, ks, arith, classes, per_model=False):
        self.W = W.to(DEV)                     # [M, n, d]
        self.W0 = self.W.clone()
        self.ks, self.arith, self.classes, self.per_model = list(ks), arith, classes, per_model
        self.ens = make_ensemble(W, ks, arith)
        self.M, self.n, self.d = W.shape

    def refs(self, X):
        out = []
        for m, k in enumerate(self.ks):
            Xm = (X[m] if self.per_model else X).to(DEV).double()
            Sc, code, sel, x_hat = ref_topk(self.W[m], Xm, k)
            assert_exact_inputs(Sc, code, x_hat)
            out.append((Xm, code, sel, x_hat))
        return out

    def common(self, what, loss, aux, refs):
        code = aux["c"].dense()
        assert self.ens.resolved_arith() == self.arith
        for m, (Xm, c, sel, x_hat) in enumerate(refs):
            assert torch.equal(code[m].double(), c), (what, m, int((code[m].double() != c).any(-1).sum()), "rows differ")
            want = float((Xm - x_hat).pow(2).mean())
            assert abs(float(loss["loss"][m]) - want) <= 1e-6 * want + 1e-30, (what, m, float(loss["loss"][m]), want)
            nnz = float((c > 0).sum(-1).double().mean())
            assert abs(float(aux["c"].mean_nnz[m]) - nnz) <= 1e-7 * max(nnz, 1.0), (what, m, float(aux["c"].mean_nnz[m]), nnz)
        xm = self.M if self.per_model else 1
        assert self.ens.gpu_launches_last_call() == launches(what, self.classes, xm, self.arith), what

    def forward(self, X):
        refs = self.refs(X)
        loss, aux, x_hat = self.ens.forward_batch(X.to(DEV), expand_dims=not self.per_model, return_x_hat=True)
        self.common("forward", loss, aux, refs)
        for m, r in enumerate(refs):
            assert torch.equal(x_hat[m].double(), r[3]), ("x_hat", m)

    def grads(self, X):
        refs = self.refs(X)
        g, (loss, aux) = self.ens.grads_batch(X.to(DEV), expand_dims=not self.per_model)
        self.common("grads", loss, aux, refs)
        for m, (Xm, _, sel, _) in enumerate(refs):
            want = O.topk_grads(self.W[m].double(), Xm, self.ks[m], support=sel)["grads"]["dict"]
            err = float((g["dict"][m].double() - want).norm())
            assert err <= 1e-4 * float(want.norm()) + 1e-30, ("dict grad", m, err, float(want.norm()))

    def step(self, X):
        refs = self.refs(X)
        loss, aux = self.ens.step_batch(X.to(DEV), expand_dims=not self.per_model)
        self.common("step", loss, aux, refs)
        assert torch.equal(self.ens.params["dict"], self.W0)            # lr = 0: the dictionary stays on the grid


# ----------------------------------------------------------------------------------------------------------------
# §3: the case table
# ----------------------------------------------------------------------------------------------------------------
ALL = ("rand", "tie", "zero", "neg")
CASES = {
    # id: (d, n, ks, dictionary pattern, batch, row kinds, gather launches)
    "whole-row-n256": (64, 256, [1, 7, 64, 255, 256], "random", 64, ALL, 0),
    "fused-n1040-k32": (64, 1040, [32], "random", 64, ALL, 0),
    "whole-row-n1040-k33": (64, 1040, [33], "random", 64, ALL, 0),
    "fused-n2048-k64": (64, 2048, [64], "random", 64, ALL, 0),
    "whole-row-n2048-k65": (64, 2048, [65], "random", 64, ALL, 0),
    "fused-n8192-k256": (64, 8192, [256], "random", 48, ALL, 0),
    # 257 chunks: the partial one (8 columns) belongs to thread 0, a full warp; "neg" rows score negative everywhere
    "fused-n8200-partial-chunk": (64, 8200, [8, 256], "random-nonneg", 48, ("neg", "rand", "neg", "tie"), 0),
    "count-1024-candidates": (64, 1024, [40], "equal", 32, ALL, 0),
    "radix-n2048-all-equal": (64, 2048, [64, 200], "equal", 32, ALL, 0),
    "radix-n8192-periodic": (64, 8192, [100, 256], "periodic", 32, ALL, 0),
    "radix-k300-n1200": (64, 1200, [300], "random", 48, ALL, 0),
    "radix-k300-mixed-k5": (64, 1200, [300, 5], "random", 48, ALL, 0),
    "whole-row-n65552-over-2048-chunks": (64, 65552, [16, 200], "random", 16, ALL, 2),
    "gather-nonpositive-rows": (64, 6144, [16, 64], "random-nonneg", 48, ("neg", "zero", "rand", "neg"), 2),
    "gather-4-classes-8-slices": (512, 24576, [1, 16, 17, 32, 33, 64, 65, 256], "random", 32, ALL, 4),
    "gather-4-slices": (1024, 6144, [64], "random", 32, ALL, 1),
    "gather-8-slices": (2048, 6144, [16, 64], "random", 32, ALL, 2),
    "gather-odd-width-2-slices": (40, 2304, [3, 17], "random", 64, ALL, 2),
}


def ariths(d, n):
    return ["bf16x3", "f16f8"] if d % 16 == 0 and n % 16 == 0 else ["bf16x3"]


PARAMS = [pytest.param(cid, a, id=f"{cid}-{a}") for cid, c in CASES.items() for a in ariths(c[0], c[1])]


def build_case(cid, arith, seed):
    d, n, ks, pattern, B, kinds, classes = CASES[cid]
    assert gather_classes(d, n, ks) == classes, (cid, gather_classes(d, n, ks))
    gen = torch.Generator().manual_seed(seed)
    nonneg = pattern.endswith("-nonneg")
    W = torch.stack([grid_dict(n, d, pattern.replace("-nonneg", ""), gen, nonneg) for _ in ks])
    return Checker(W, ks, arith, classes), gen, B, kinds


@pytest.mark.parametrize("cid,arith", PARAMS)
def test_case_table(cid, arith):
    chk, gen, B, kinds = build_case(cid, arith, 1)
    d = chk.d
    chk.forward(grid_batch(B, d, kinds, gen))
    chk.grads(grid_batch(B, d, kinds[1:] + kinds[:1], gen))
    chk.step(grid_batch(B, d, kinds[2:] + kinds[:2], gen))
    chk.forward(grid_batch(B // 2 + 1, d, kinds[3:] + kinds[:3], gen))


@pytest.mark.parametrize("arith", ["bf16x3", "f16f8"])
def test_gather_per_model_batches(arith):
    """expand_dims=False: every model reads its own batch (x_model_stride of the gather kernel)."""
    gen = torch.Generator().manual_seed(2)
    d, n, ks = 64, 3072, [8, 32]
    W = torch.stack([grid_dict(n, d, "random", gen) for _ in ks])
    chk = Checker(W, ks, arith, gather_classes(d, n, ks), per_model=True)
    assert chk.classes == 2
    X = lambda B: torch.stack([grid_batch(B, d, ALL[m:] + ALL[:m], gen) for m in range(len(ks))])
    chk.forward(X(64))
    chk.grads(X(64))
    chk.step(X(33))


# ----------------------------------------------------------------------------------------------------------------
# §4: sequences of calls on one plan (anything left over from an earlier call shows up as a mismatch)
# ----------------------------------------------------------------------------------------------------------------
SEQUENCES = {
    # dense decode with lists, launch-bound (graph replay of the step)
    "dense-graph": (64, 2048, [40, 100], 128),
    # gather decode, not launch-bound: every step runs its launches eagerly
    "gather-eager": (1024, 6144, [16, 64], 1024),
}


@pytest.mark.parametrize("arith", ["bf16x3", "f16f8"])
@pytest.mark.parametrize("sid", list(SEQUENCES))
def test_call_sequence(sid, arith):
    d, n, ks, Bmax = SEQUENCES[sid]
    gen = torch.Generator().manual_seed(3)
    W = torch.stack([grid_dict(n, d, "random", gen) for _ in ks])
    chk = Checker(W, ks, arith, gather_classes(d, n, ks))
    assert (chk.classes > 0) == sid.startswith("gather")
    assert launch_bound(len(ks), Bmax, n, d) == sid.endswith("graph")
    sizes = [Bmax, 1, 37, Bmax]
    calls = [chk.step, chk.forward, chk.grads]
    i = 0
    for kind in ALL:
        for B in sizes:
            calls[i % 3](grid_batch(B, d, (kind,), gen))
            i += 1
    # two more steps at one size: the second replays the graph captured by the first (launch-bound plans)
    for kind in ("rand", "tie"):
        chk.step(grid_batch(37, d, (kind, "rand"), gen))


# ----------------------------------------------------------------------------------------------------------------
# §5: changing k after the plan was built; invalid k
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k0,k1", [(16, 20), (16, 300), (64, 8)])
def test_refresh_after_changing_sparsity(k0, k1):
    """refresh() after raising or lowering a model's k (the list capacity and the decode path follow the largest k)
    gives bitwise what a freshly built ensemble gives, and both are the exact reference."""
    gen = torch.Generator().manual_seed(4)
    d, n = 64, 6144
    W = torch.stack([grid_dict(n, d, "random", gen) for _ in range(2)])
    old = Checker(W, [16, k0], "f16f8", gather_classes(d, n, [16, k0]))
    X = grid_batch(64, d, ALL, gen)
    old.forward(X)
    old.step(X)
    old.ens.buffers["sparsity"][1] = k1
    old.ens.refresh()
    old.ks, old.classes = [16, k1], gather_classes(d, n, [16, k1])
    new = Checker(W, [16, k1], "f16f8", old.classes)
    for step, kinds in enumerate((ALL, ("tie", "rand"), ("neg",))):
        X = grid_batch(64 - 13 * step, d, kinds, gen)
        outs = []
        for chk in (old, new):
            chk.forward(X)
            loss, aux, x_hat = chk.ens.forward_batch(X.to(DEV), return_x_hat=True)
            outs.append((loss["loss"], aux["c"].dense(), x_hat))
            chk.grads(X)
            chk.step(X)
        for a, b in zip(*outs):
            assert torch.equal(a, b)


def test_invalid_sparsity_raises():
    gen = torch.Generator().manual_seed(5)
    d, n = 32, 256
    W = grid_dict(n, d, "random", gen)
    X = grid_batch(16, d, ALL, gen).to(DEV)
    for k in (0, -3, n + 1):
        ens = make_ensemble(W[None], [k], "auto")                    # buffers built by hand: TopKEncoder.init refuses
        with pytest.raises(ValueError, match=rf"sparsity must be in \[1, {n}\], got {k}"):
            ens.forward_batch(X)
    ens = make_ensemble(W[None], [8], "auto")
    ens.forward_batch(X)
    ens.buffers["sparsity"][0] = n + 1
    with pytest.raises(ValueError, match="sparsity must be in"):
        ens.refresh()
    with pytest.raises(ValueError, match="sparsity must be in"):     # the rejected k never reaches the engine
        ens.forward_batch(X)
    ld = S.TopKLearnedDict((W / W.norm(dim=-1, keepdim=True)).to(DEV), 0)
    with pytest.raises(ValueError, match="sparsity must be in"):
        MT.evaluate_dicts([ld], X)


# ----------------------------------------------------------------------------------------------------------------
# §6: the forward-only passes (evaluate_dicts, top_activating_fragments) on the same exact data
# ----------------------------------------------------------------------------------------------------------------
def ref_moments(code, segment):
    sums, rows, times = [], [], 0
    for i in range(0, code.shape[0], segment):
        c = code[i:i + segment]
        sums.append(torch.stack([c.sum(0), c.pow(2).sum(0), c.pow(3).sum(0), c.pow(4).sum(0)], dim=-1))
        rows.append(c.shape[0])
        times = times + (c.sum(0) != 0).double()
    means = torch.stack(sums) / torch.tensor(rows, dtype=code.dtype, device=code.device)[:, None, None]
    mean, m2, _, m4 = means.mean(dim=0).unbind(-1)
    return times, mean, m2 - mean ** 2, m4


@pytest.mark.parametrize("arith", ["bf16x3", "f16f8"])
@pytest.mark.parametrize("case", ["tie-heavy", "gather-classes"])
def test_forward_only_passes(case, arith):
    gen = torch.Generator().manual_seed(6)
    if case == "tie-heavy":
        d, n, ks, pattern = 64, 2048, [64, 100], "periodic"
    else:
        d, n, ks, pattern = 256, 6144, [16, 64], "random"
    lds = []
    for k in ks:
        W = grid_dict(n, d, pattern, gen)
        lds.append(S.TopKLearnedDict((W / W.norm(dim=-1, keepdim=True)).to(DEV), k))
    L, segment = 64, 1000
    x = grid_batch(L * 40, d, ALL, gen).to(DEV)
    stats = MT.evaluate_dicts(lds, x, segment=segment, arith=arith)
    frags = MT.top_activating_fragments(lds, x, fragment_len=L, n_top=20, n_random=20, arith=arith)
    for m, (ld, st, fr) in enumerate(zip(lds, stats, frags)):
        Sc, code, _, x_hat = ref_topk(ld.dict, x, ld.sparsity)
        assert_exact_inputs(Sc, code, x_hat)
        assert torch.equal(st["feature_counts"].long().cpu(), (code > 0).sum(0).cpu()), m
        times, mean, var, m4 = ref_moments(code, segment)
        assert torch.equal(st["times_active"].double(), times), m
        for got, want, what in ((st["mean"], mean, "mean"), (st["var"], var, "var"), (st["m4"], m4, "m4")):
            err = float((got.double() - want).abs().max())
            assert err <= 1e-6 * float(want.abs().max()) + 1e-30, (m, what, err)
        fmax, active = IO.fragment_tables(code, L)
        want_tf = IO.select_top(fmax, 20)
        assert torch.equal(fr["top_values"].double(), fmax.T.gather(1, want_tf)), m
        assert torch.equal(fr["top_fragments"], want_tf), m
        assert torch.equal(fr["n_active_fragments"].long(), active.sum(0)), m
