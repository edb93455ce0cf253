"""The forward-only plans of the baseline dictionaries through the ABI (libsce sce_forward_stats, sce_forward_fragments,
sce_read_code on metrics._StatsPlan / _FragmentPlan), against fp64:

  code, x_hat     per 128 x 128 tile with the training-step bars (tile_bounds.BARS[arith]["signed"]). ICAEncoder's plan
                  reads the batch minus its fp32 translation, formed in fp32; the reference here is computed from the same
                  fp32 E and t, and the input scale |x - t| + 2^-24 |x| carries that subtraction's rounding
  moment sums     per feature against oracle/eval_bounds.moment_bound (|c| in the mean-value term: the identity is
                  1-Lipschitz as ReLU is)
  segment counts  exact on the engine's read-back code (c != 0)
  fragment lists  exact on the engine's read-back code: the top lists by (maximum descending, fragment ascending), with
                  negative maxima, lists that fill up with them, and empty entries sorting last
  hygiene         the workspace filled with 0xFF before every call, x followed by NaN rows, guards past every accumulator
  refusal         every training entry point returns SCE_ERR_INVALID on a linear or raw-decoder plan
Shapes: a linear plan at d = 400, n = 1000 (padded, partial chunks and tiles) with calls of B = 4001, 31, 1, and ICA at
d = n = 512 and 2048, each with a translation whose mean is 10^3 times its spread on a quarter of the columns; RandomDict at d = 512 with n = 512 and 4096; a mixed
IdentityReLU + UntiedSAE group."""
import ctypes as C

import numpy as np
import pytest
import torch

from engine_cases import ARITHS, DEV, one_key, untied
from oracle import eval_bounds as EB
from oracle import tile_bounds as T
from sparse_coding_b200 import _lib
from sparse_coding_b200 import metrics as MT
from sparse_coding_b200.ica import FittedFastICA, FittedScaler, ICAEncoder
from sparse_coding_b200.learned_dict import IdentityReLU, RandomDict

pytestmark = pytest.mark.gpu
GUARD = 256
U = 2.0 ** -24


def fake_ica(n, d, seed):
    """An ICAEncoder with n components of width d (not square: the engine does not care) and a large column mean on
    a quarter of the columns."""
    rs = np.random.RandomState(seed)
    mean = rs.normal(size=d) * 0.1
    mean[: d // 4] = 2.0e3 * (1 + rs.uniform(size=d // 4))
    scale = 0.5 + rs.uniform(size=d)
    ica = ICAEncoder(d, n)
    ica.scaler = FittedScaler(mean, scale ** 2, scale, 1000)
    comp = rs.normal(size=(n, d)) / np.sqrt(d)
    ica.ica = FittedFastICA(comp, np.linalg.pinv(comp), 0.01 * rs.normal(size=d), None, None, 0)
    return ica


def rows(B, d, seed, ica=None):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(B, d, generator=g, device=DEV)
    if ica is not None:     # spread ~1 about the fitted mean: mean / spread >= 10^3 on the large columns
        x = x * torch.as_tensor(ica.scaler.scale_, device=DEV).float() + torch.as_tensor(ica.scaler.mean_, device=DEV).float()
    return x


def fp64_inputs(p, ld, k):
    """(E, b, D, t) of model k of plan p as the plan holds them, in fp64 (D normalised unless the decoder is raw)."""
    enc, bias, dec, t = MT._sae_inputs(ld)
    f = lambda a: a.float().to(DEV).double()
    D = f(dec)
    if not _lib.SIGNATURES[p.kind].decoder_raw:
        D = D / D.norm(dim=-1, keepdim=True).clamp(min=1e-8)
    return f(enc), f(bias), D, (f(t) if t is not None else None)


def reference(p, ld, k, x):
    """fp64 code, x_hat and the code's scale for model k on the fp32 rows x."""
    E, b, D, t = fp64_inputs(p, ld, k)
    X = x.double()
    if t is not None:
        Xin = (x - t.float()).double()                # the plan's input, formed in fp32
        Xabs = Xin.abs() + U * X.abs()
    else:
        Xin, Xabs = X, X.abs()
    z = Xin @ E.T + b
    c = z if p.kind == "ica" else z.clamp(min=0.0)
    S_c = T.code_scale(Xabs, E, b)
    return c, c @ D, S_c, S_c @ D.abs()


class Harness:
    def __init__(self, lds, batch_max, arith, case):
        self.lds, self.arith = lds, arith
        self.bars = dict(T.BARS[arith]["signed"], **OWN_BARS.get((case.split("_")[0], arith), {}))
        self.p = MT._StatsPlan(one_key(lds, arith), lds, batch_max, arith, DEV)
        self.lib = _lib.load()
        M, n = self.p.M, self.p.n
        self.sums_buf = torch.randn(M * n * 4 + GUARD, device=DEV, dtype=torch.float64)
        self.counts_buf = torch.randint(-100, 100, (M * n + GUARD,), device=DEV, dtype=torch.int32)
        self.open_buf = torch.zeros(M * n + GUARD, device=DEV, dtype=torch.int32)
        self.worst = T.Worst()

    def call(self, x, seg, phase, tag):
        p, lib = self.p, self.lib
        M, n = p.M, p.n
        B, d = x.shape
        xin = p.batch(x)                               # [B, d], or [M, B, d] rows minus the translation
        xbuf = torch.full((xin.numel() + 64 * d,), float("nan"), device=DEV)
        xbuf[: xin.numel()] = xin.reshape(-1)
        xh = torch.full((M * B * d + GUARD,), -7.25, device=DEV)
        p._pass_ws.fill_(0xFF)
        before = [b.clone() for b in (self.sums_buf, self.counts_buf, self.open_buf)]
        _lib.check(lib.sce_forward_stats(p.plan, xbuf.data_ptr(), B, seg, phase, xh.data_ptr(), p.losses.data_ptr(),
                                         p.nnz.data_ptr(), self.sums_buf.data_ptr(), self.counts_buf.data_ptr(),
                                         self.open_buf.data_ptr(), p.ws_ptr, p.ws_bytes, p.stream), tag)
        assert bool((xh[M * B * d:] == -7.25).all()), (tag, "x_hat guard")
        for buf, b0, k in zip((self.sums_buf, self.counts_buf, self.open_buf), before, (M * n * 4, M * n, M * n)):
            assert torch.equal(buf[k:], b0[k:]), (tag, "accumulator guard")
        code = torch.empty(M, B, n, device=DEV)
        _lib.check(lib.sce_read_code(p.plan, B, code.data_ptr(), p.stream), "sce_read_code")
        x_hat = xh[: M * B * d].view(M, B, d)
        sums, sums0 = self.sums_buf[: M * n * 4].view(M, n, 4), before[0][: M * n * 4].view(M, n, 4)
        for k, ld in enumerate(self.lds):
            size = int(ld.n_feats)
            c, xr, S_c, S_x = reference(p, ld, k, x)
            self.worst.add("code", k, T.tile_ratios(code[k, :, :size], c, S_c))
            self.worst.add("x_hat", k, T.tile_ratios(x_hat[k], xr, S_x))
            bound = EB.moment_bound(c, S_c, self.bars["code"][1], EB.K_TREE)
            ratio = EB.moment_ratios(sums[k, :size], sums0[k, :size], EB.moment_sums(c), bound)
            self.worst.add_scalar("moments", k, float(ratio.max()))
            assert bool(torch.isfinite(sums[k]).all()), tag
            assert torch.equal(sums[k, size:], sums0[k, size:]) if size < n else True, (tag, "padding")
        # segment counts exact on the read-back activity, where it is the mask's (f16f8: a code below ~4e-9 reads back as
        # 0 while the mask has it on; such a feature's count may differ by that excess)
        active = code != 0
        act = torch.zeros(M, n, dtype=torch.int32, device=DEV)
        _lib.check(lib.sce_active_counts(p.plan, B, act.data_ptr(), p.stream), "sce_active_counts")
        excess = act.long() - active.sum(1)
        assert int(excess.min()) >= 0 and (self.arith == "f16f8" or int(excess.max()) == 0), (tag, int(excess.max()))
        exact = excess == 0
        counts0 = before[1][: M * n].view(M, n).long()
        inc, open_ = EB.segment_call(active, seg, phase, before[2][: M * n].view(M, n).long())
        diff = self.counts_buf[: M * n].view(M, n).long() - counts0 - inc
        assert bool((diff[exact] == 0).all()) and bool((diff.abs() <= excess).all()), (tag, "seg_counts")
        if seg > 1:
            assert torch.equal(self.open_buf[: M * n].view(M, n).long()[exact], open_[exact]), (tag, "seg_open")
        if p.kind == "ica":
            assert bool((code < 0).any()), tag
        return code

    def assert_bars(self, tag):
        bars = self.bars
        for name in ("code", "x_hat"):
            print(f"{tag:30s} {self.arith:6s} {name:6s} tile {self.worst.tile[name][0]:.2e} elem {self.worst.elem[name]:.2e} "
                  f"| bars {bars[name][0]:.1e} {bars[name][1]:.1e}")
        print(f"{tag:30s} {self.arith:6s} moments {self.worst.tile['moments'][0]:.3f}")
        for name in ("code", "x_hat"):
            tb, eb = bars[name]
            assert self.worst.tile[name][0] <= tb and self.worst.elem[name] <= eb, (tag, name, self.worst.tile[name])
        assert self.worst.tile["moments"][0] <= 1.0, (tag, self.worst.tile["moments"])

    def close(self):
        self.p.close()


# Bars of their own for the code and x_hat, twice the worst value measured on an H100 SXM (80 GB HBM3, 700 W limit):
#   ica_ragged      bf16x3 code 1.15e-6 / 6.5e-6, x_hat 1.5e-7 / 6.5e-7;  f16f8 code 4.0e-6 / 2.3e-5, x_hat 2.7e-7 / 1.5e-6
#   identity_mixed  bf16x3 code 2.0e-6 / 7.6e-6;  f16f8 code 1.1e-5 / 9.8e-4 (x_hat = code: D = I)
# (ica_512 and ica_2048, at longer K, stay below the ragged case: code tiles at most 3.7e-7 bf16x3, 1.6e-6 f16f8)
# The training-step bars were measured on ReLU codes, where the entries at or below 0 are exactly 0 on both sides; a
# linear code has an error on every entry. The identity's code is one product per entry, with no averaging over d terms,
# and under f16f8 a small |x| meets fp16's coarser relative spacing near 0. The moment bound takes the case's code
# element bar.
# (keyed by the case name's first word: every ica_* case takes the ICA bars)
OWN_BARS = {("ica", "bf16x3"): {"code": (2.3e-6, 1.3e-5), "x_hat": (3.0e-7, 1.3e-6)},
            ("ica", "f16f8"): {"code": (8.0e-6, 4.6e-5), "x_hat": (5.4e-7, 3.1e-6)},
            ("identity", "bf16x3"): {"code": (4.1e-6, 1.6e-5), "x_hat": (4.1e-6, 1.6e-5)},
            ("identity", "f16f8"): {"code": (2.3e-5, 2.0e-3), "x_hat": (2.3e-5, 2.0e-3)}}

CASES = {
    "ica_ragged": (lambda: [fake_ica(1000, 400, 1), fake_ica(1000, 400, 2)], 400, (4001, 31, 1)),
    "ica_512": (lambda: [fake_ica(512, 512, 3)], 512, (4001, 31)),
    "ica_2048": (lambda: [fake_ica(2048, 2048, 4)], 2048, (2048, 1)),
    "random512": (lambda: [RandomDict(512, 512)], 512, (2048, 31)),
    "random4096": (lambda: [RandomDict(512, 4096)], 512, (1000,)),
    "identity_mixed": (lambda: [IdentityReLU(400), untied(400, 400, 9)], 400, (4001, 1)),
}


@pytest.mark.parametrize("arith", ARITHS)
@pytest.mark.parametrize("name", list(CASES))
def test_bounds(name, arith):
    torch.manual_seed(3)
    make, d, sizes = CASES[name]
    lds = make()
    for ld in lds:
        if hasattr(ld, "to_device") and not isinstance(ld, ICAEncoder):
            ld.to_device(DEV)
    h = Harness(lds, max(sizes), arith, name)
    try:
        seen, seg = 0, 37
        for i, B in enumerate(sizes):
            ica = lds[0] if isinstance(lds[0], ICAEncoder) else None
            h.call(rows(B, d, 10 + i, ica), seg, seen % seg, f"{name} call {i} B {B}")
            seen += B
        h.assert_bars(name)
    finally:
        h.close()


@pytest.mark.parametrize("arith", ARITHS)
def test_fragment_lists_exact_on_the_read_back_code(arith):
    d, L, G = 400, 32, 40
    ica = fake_ica(1000, d, 5)
    x = rows(G * L, d, 3, ica)
    # rows moved against the first 20 features' encoder rows: those are negative on every row, their maxima negative
    enc = MT._sae_inputs(ica)[0].to(DEV)
    x = x - 10.0 * enc[:20].sum(0) / enc[:20].pow(2).sum(1).mean()
    p = MT._FragmentPlan(one_key([ica], arith), [ica], G * L, L, 8, 4, 11, True, arith, DEV)
    try:
        p.run(x, 0)
        code = torch.empty(1, G * L, p.n, device=DEV)
        _lib.check(_lib.load().sce_read_code(p.plan, G * L, code.data_ptr(), p.stream), "sce_read_code")
        c = code[0, :, :1000].view(G, L, 1000)
        fm = c.amax(dim=1)                                     # [G, n] on the engine's values
        out = p.results(0, 1000)
        want_o = MT._list_order(fm.T.contiguous(), torch.arange(G, device=DEV).expand(1000, G).contiguous())[:, :8]
        assert torch.equal(out["top_fragments"], want_o)
        assert torch.equal(out["top_values"], fm.T.gather(1, want_o))
        assert bool((out["top_values"] < 0).any()) and bool((fm < 0).all(dim=0).any())
        assert torch.equal(out["top_activations"], c.permute(2, 0, 1).gather(1, want_o[..., None].expand(-1, -1, L)))
        # (f16f8: a code below ~4e-9 reads back as 0 while the activity mask has it)
        excess = out["n_active_fragments"] - (c != 0).any(dim=1).sum(0)
        assert int(excess.min()) >= 0 and (arith == "f16f8" or int(excess.max()) == 0)
    finally:
        p.close()
    # fewer fragments than the list: negative maxima fill it, the empty entries sort last
    p = MT._FragmentPlan(one_key([ica], arith), [ica], 4 * L, L, 6, 0, 0, False, arith, DEV)
    try:
        p.run(x[: 4 * L], 0)
        out = p.results(0, 1000)
        assert torch.equal(out["top_fragments"][:, 4:], torch.full((1000, 2), -1, device=DEV))
        assert bool((out["top_fragments"][:, :4] >= 0).all())
        assert bool((out["top_values"][:20, :4] < 0).all())
    finally:
        p.close()


@pytest.mark.parametrize("kind", ["ica", "random"])
def test_training_entry_points_refuse(kind):
    lib = _lib.load()
    ld = fake_ica(64, 64, 0) if kind == "ica" else RandomDict(64, 64)
    p = MT._StatsPlan(one_key([ld], "bf16x3"), [ld], 128, "bf16x3", DEV)
    try:
        x = torch.zeros(128, 64, device=DEV)
        out = torch.zeros(64, device=DEV)
        host = torch.zeros(128 * 64)
        grads = torch.zeros(64 * 64, device=DEV)
        calls = {
            "sce_step": lambda: lib.sce_step(p.plan, x.data_ptr(), 128, out.data_ptr(), out.data_ptr(), p.stream),
            "sce_step_host": lambda: lib.sce_step_host(p.plan, host.data_ptr(), 128, None, None, p.stream),
            "sce_grads": lambda: lib.sce_grads(p.plan, x.data_ptr(), 128, grads.data_ptr(), out.data_ptr(),
                                               grads.data_ptr(), out.data_ptr(), out.data_ptr(), p.stream),
        }
        ws = torch.zeros(1 << 20, dtype=torch.uint8, device=DEV)
        tr = _lib.SceTrack(err=out.data_ptr(), serial=grads.data_ptr(), rows=grads.data_ptr(), filled=out.data_ptr(),
                           counts=out.data_ptr(), next_serial=0, n_worst=4, workspace=(ws.data_ptr() + 1023) // 1024 * 1024,
                           workspace_bytes=(1 << 20) - 1024)
        calls["sce_step_tracked"] = lambda: lib.sce_step_tracked(p.plan, x.data_ptr(), 128, out.data_ptr(), out.data_ptr(),
                                                                 C.byref(tr), p.stream)
        calls["sce_resample"] = lambda: lib.sce_resample(p.plan, C.byref(tr), C.c_float(0.2), out.data_ptr(),
                                                         out.data_ptr(), out.data_ptr(), p.stream)
        before = torch.cat([x.flatten(), out, grads]).clone()
        for name, f in calls.items():
            assert f() == -1, name      # SCE_ERR_INVALID
            assert b"forward-only" in lib.sce_last_error(), name
        torch.cuda.synchronize()
        assert torch.equal(torch.cat([x.flatten(), out, grads]), before)
        # the forward-only passes run
        _lib.check(lib.sce_forward(p.plan, x.data_ptr(), 128, None, p.losses.data_ptr(), p.nnz.data_ptr(), p.stream),
                   "sce_forward")
    finally:
        p.close()
