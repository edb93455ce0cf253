"""code_correlation on the GPU.

  cross sums   sce_cross_moments per entry against the fp64 sums of the codes the engine holds (sce_read_code after the
               same sce_forward_stats calls), within oracle/correlation_oracle.cross_sum_bound: every kind, both
               arithmetics, mixed groups, n not a multiple of the tile, calls of B = 8192, 4001, 31 and 1, a top-k plan
               with k > 256 (no lists); the workspace filled with 0xFF before each call, guard words past acc, x
               followed by NaN rows
  golden       code_correlation against the fp64 correlation of the reference's own codes
               (tests/golden/code_correlation.pt): 1e-4 absolute where both variances exceed VAR_FLOOR, NaN exactly
               where the golden has it, maxima and argmax, the planted tie to the lower index
  independence two runs bitwise equal; the correlation independent of how the rows are cut into calls within the bound;
               mean / var against fp64
  large        n_a = n_b = 16384 (2 GiB of fp64 accumulator) and one 32768 x 4096 pair"""

import numpy as np
import pytest
import torch

from oracle import correlation_oracle as CO
from sparse_coding_b200 import _lib
from sparse_coding_b200 import metrics as MT
from sparse_coding_b200.ica import FittedFastICA, FittedScaler, ICAEncoder
from sparse_coding_b200.learned_dict import IdentityReLU, RandomDict, TiedSAE, UntiedSAE
from sparse_coding_b200.topk_encoder import TopKLearnedDict

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
GUARD = 64
VAR_FLOOR = 1e-3
ARITHS = ["bf16x3", "f16f8"]


def fake_ica(n, d, seed):
    rs = np.random.RandomState(seed)
    scale = 0.5 + rs.uniform(size=d)
    ica = ICAEncoder(d, n)
    ica.scaler = FittedScaler(rs.normal(size=d) * 0.1, scale ** 2, scale, 1000)
    comp = rs.normal(size=(n, d)) / np.sqrt(d)
    ica.ica = FittedFastICA(comp, np.linalg.pinv(comp), 0.01 * rs.normal(size=d), None, None, 0)
    return ica


def dicts(d, seed):
    """Every kind at width d, with sizes that are not multiples of the 128-column tile."""
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g)
    torch.manual_seed(seed)
    return [TiedSAE(rn(200, d), rn(200) * 0.3 - 0.3), UntiedSAE(rn(136, d) * 0.4, rn(136, d), rn(136) * 0.3 - 0.2),
            TopKLearnedDict(rn(160, d), 8), TopKLearnedDict(rn(512, d), 300), RandomDict(d, 264), IdentityReLU(d),
            fake_ica(48, d, seed)]


def rows_with_nan_tail(B, d, seed):
    """[B, d] rows, a view of a buffer with NaN rows after them."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    buf = torch.full((B + 16, d), float("nan"), device=DEV)
    buf[:B] = torch.randn(B, d, generator=g, device=DEV)
    return buf[:B]


def code_plans(lds, x, arith, batch_max):
    lds, groups, ar = MT._dict_inputs(lds, x, arith, centre=False)
    return [(MT._CodePlan(key, [lds[i] for i in idx], batch_max, ar, DEV), idx) for key, idx in groups.items()], ar


def read_code(p, B):
    out = torch.empty(p.M, B, p.n, device=DEV)
    _lib.check(_lib.load().sce_read_code(p.plan, B, out.data_ptr(), p.stream), "sce_read_code")
    return out


def cross(pa, pb, B, acc):
    lib = _lib.load()
    nbytes = lib.sce_cross_moments_workspace_bytes(pa.plan, pb.plan, B)
    ws, ptr = _lib.workspace(nbytes, DEV, "sce_cross_moments_workspace_bytes")
    ws.fill_(0xFF)
    _lib.check(lib.sce_cross_moments(pa.plan, pb.plan, B, acc.data_ptr(), ptr, nbytes, pa.stream), "sce_cross_moments")


@pytest.mark.parametrize("arith", ARITHS)
def test_cross_sums_every_kind_and_call_size(arith):
    d = 64
    lds_a, lds_b = dicts(d, 1), dicts(d, 2)[:3]
    calls = [8192, 4001, 31, 1]
    with torch.cuda.device(DEV):
        x0 = rows_with_nan_tail(max(calls), d, 0)
        plans_a, _ = code_plans(lds_a, x0, arith, max(calls))
        plans_b, _ = code_plans(lds_b, x0, arith, max(calls))
        try:
            assert len(plans_a) >= 4       # mixed groups: tied, untied + identity, two top-k, random, ica
            for c, B in enumerate(calls):
                x = rows_with_nan_tail(B, d, 10 + c)
                for p, _ in plans_a + plans_b:
                    p.run(x)
                for pa, _ in plans_a:
                    ca = read_code(pa, B)
                    for pb, _ in plans_b + plans_a[:1]:
                        cb = read_code(pb, B)
                        size = pa.M * pb.M * pa.n * pb.n
                        buf = torch.full((size + GUARD,), 7.0, dtype=torch.float64, device=DEV)
                        cross(pa, pb, B, buf)
                        torch.cuda.synchronize()
                        assert bool((buf[size:] == 7.0).all()), "guard words past acc were written"
                        acc = buf[:size].view(pa.M, pb.M, pa.n, pb.n) - 7.0
                        for i in range(pa.M):
                            for j in range(pb.M):
                                want = ca[i].double().T @ cb[j].double()
                                bound = CO.cross_sum_bound(ca[i], cb[j], arith) + 7.0 * 2.0 ** -52
                                err = (acc[i, j] - want).abs()
                                assert bool((err <= bound).all()), (pa.kind, pb.kind, B, i, j, float((err / bound).max()))
        finally:
            for p, _ in plans_a + plans_b:
                p.close()


def rebuild(entry, d):
    k = entry["kind"]
    if k == "tied":
        return TiedSAE(entry["encoder"], entry["encoder_bias"])
    if k == "untied":
        return UntiedSAE(entry["encoder"], entry["decoder"], entry["encoder_bias"])
    if k == "topk":
        return TopKLearnedDict(entry["dict"], entry["sparsity"])
    if k == "random":
        rd = RandomDict(d, entry["encoder"].shape[0])
        rd.encoder = entry["encoder"].clone()
        return rd
    if k == "identity":
        return IdentityReLU(d)
    a = lambda t: t.numpy()
    ica = ICAEncoder(d, entry["components"].shape[0])
    ica.scaler = FittedScaler(a(entry["scaler_mean"]), a(entry["scaler_var"]), a(entry["scaler_scale"]), 512)
    ica.ica = FittedFastICA(a(entry["components"]), a(entry["mixing"]), a(entry["ica_mean"]), None, None, 0)
    return ica


def test_golden_end_to_end(golden):
    # (bf16x3 only: f16f8 needs d and n to be multiples of 16, which side b's width 40 is not; the cross sums above
    # cover f16f8 on every kind)
    arith = "bf16x3"
    g = golden("code_correlation")
    xa, xb = g["x_a"], g["x_b"]
    names_a, names_b = list(g["side_a"]), list(g["side_b"])
    lds_a = [rebuild(g["side_a"][k], xa.shape[1]) for k in names_a]
    lds_b = [rebuild(g["side_b"][k], xb.shape[1]) for k in names_b]
    res = MT.code_correlation(lds_a, xa.to(DEV), lds_b, xb.to(DEV), arith=arith)
    for i, na in enumerate(names_a):
        for j, nb in enumerate(names_b):
            want, got = g["pairs"][(na, nb)], {k: (v.cpu() if torch.is_tensor(v) else v) for k, v in res[i][j].items()}
            what = (na, nb, arith)
            assert got["rows"] == xa.shape[0]
            corr, wc = got["correlation"].double(), want["correlation"]
            assert torch.equal(torch.isnan(corr), torch.isnan(wc)), what
            ok = (want["var_a"] > VAR_FLOOR)[:, None] & (want["var_b"] > VAR_FLOOR)[None, :] & ~torch.isnan(wc)
            assert float((corr - wc)[ok].abs().max()) < 1e-4, what
            for k in ("mean_a", "var_a", "mean_b", "var_b"):
                torch.testing.assert_close(got[k], want[k], rtol=1e-4, atol=1e-5, msg=str(what + (k,)))
            for side in ("ab", "ba"):
                mx, wm = got[f"max_corr_{side}"].double(), want[f"max_corr_{side}"]
                assert torch.equal(torch.isnan(mx), torch.isnan(wm)), what
                assert float((mx - wm).nan_to_num().abs().max()) < 1e-4, what
                # argmax: equal, or a near tie in the golden within the tolerance
                ga, wa = got[f"argmax_{side}"], want[f"argmax_{side}"]
                wcm = wc if side == "ab" else wc.T
                for r in torch.nonzero(ga != wa).flatten().tolist():
                    assert ga[r] >= 0 and float(wm[r] - wcm[r, ga[r]]) < 2e-4, (what, side, r)
    tt = res[names_a.index("tied")][names_b.index("tied")]
    assert int(tt["argmax_ab"][0]) == g["tie_cols"][0]
    assert int(tt["argmax_ab"][g["dead"]]) == -1 and bool(torch.isnan(tt["max_corr_ab"][g["dead"]]))


def test_repeatable_and_independent_of_cuts():
    d = 128
    g = torch.Generator().manual_seed(5)
    a = [TiedSAE(torch.randn(320, d, generator=g), torch.randn(320, generator=g) * 0.3 - 0.2)]
    b = [UntiedSAE(torch.randn(200, d, generator=g), torch.randn(200, d, generator=g), torch.randn(200, generator=g) * 0.2)]
    x = torch.randn(20000, d, generator=g).half()          # CPU fp16, streamed
    r1 = MT.code_correlation(a, x, b)[0][0]
    r2 = MT.code_correlation(a, x, b)[0][0]
    for k, v in r1.items():
        if torch.is_tensor(v):
            assert torch.equal(v.nan_to_num(), r2[k].nan_to_num()), k
    # the same rows cut into different engine calls (a different call length): equal within the bound
    old = MT._EVAL_ROWS
    try:
        MT._EVAL_ROWS = 3000
        r3 = MT.code_correlation(a, x, b)[0][0]
    finally:
        MT._EVAL_ROWS = old
    assert float((r1["correlation"] - r3["correlation"]).nan_to_num().abs().max()) < 1e-5
    # mean / var against fp64 of the codes
    ca = a[0].encode(x.float()).double()
    m, v = CO.moments(ca)
    torch.testing.assert_close(r1["mean_a"].cpu(), m, rtol=1e-5, atol=1e-7)
    torch.testing.assert_close(r1["var_a"].cpu(), v, rtol=1e-4, atol=1e-7)
    # a == b, x_b = None: each feature's co-activation; the diagonal is 1 where defined
    s = MT.code_correlation(a, x, a, full=True)[0][0]
    diag = s["correlation"].diagonal()
    ok = ~torch.isnan(diag)
    assert float((diag[ok] - 1).abs().max()) < 1e-4


@pytest.mark.parametrize("na,nb", [(16384, 16384), (32768, 4096)])
def test_large_dictionaries(na, nb):
    d = 256
    g = torch.Generator().manual_seed(9)
    a = [TiedSAE(torch.randn(na, d, generator=g), torch.randn(na, generator=g) * 0.1 - 1.0)]
    b = [TiedSAE(torch.randn(nb, d, generator=g), torch.randn(nb, generator=g) * 0.1 - 1.0)]
    x = torch.randn(8192 + 100, d, generator=g, device="cpu").to(DEV)
    r = MT.code_correlation(a, x, b, full=False)[0][0]
    assert "correlation" not in r and r["argmax_ab"].shape == (na,) and r["argmax_ba"].shape == (nb,)
    # spot-check a block of rows against fp64 of the reference codes
    ca = a[0].encode(x.cpu())[:, :256].double()
    cb = b[0].encode(x.cpu()).double()
    want = CO.correlation(ca, cb)
    mx = r["max_corr_ab"][:256].cpu().double()
    assert torch.equal(torch.isnan(mx), torch.isnan(want["max_corr_ab"]))
    assert float((mx - want["max_corr_ab"]).nan_to_num().abs().max()) < 1e-3


def test_oversized_accumulator_raises():
    free = torch.cuda.mem_get_info(DEV)[0]
    n = 65536
    d = 64
    a = [TiedSAE(torch.randn(n, d), torch.zeros(n))] * max(1, int(free // (8 * n * n)) + 1)
    with pytest.raises(ValueError, match="bytes"):
        MT.code_correlation(a, torch.randn(16, d, device=DEV), a)
