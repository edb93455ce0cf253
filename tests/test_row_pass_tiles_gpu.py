"""Every output of the row passes per 128 x 128 tile (vectors: per run of 128) and per element against fp64.

sce_second_moments, sce_ica_pass, sce_nmf_project, sce_nmf_grams and sce_nmf_residual are called through the ABI, as
tests/test_nmf_gpu.py does, and each output is measured against its absolute-product scale (oracle/row_pass_bounds.py).
The shapes cover the edges of the sliced row reduction (rows cut into S slices of R rows; test_shapes_cover_every_edge
states them and checks the list against a restatement of mom_slices and gemm_cluster_size): B = 1, 63, 64, 65; a last
slice that is full, one row short or a single row; d = 512 at 64000 rows (33 x 1984, singles) and 65536 rows (32 x 2048,
pairs under bf16x3); 2^21 rows in one call (S = 1024); 4 and 5 column tiles with a partial last one; component counts
8, 16, 208 and 256 (a partial 32-column chunk and a partial tile); k < d; GEMM 1 of the FastICA pass and the NMF
projection in clusters of two and of one at d = 2048, and in pairs under f16f8 at d = n = 8192. Each case runs under
both arithmetics where d and n allow f16f8, with fp16 and fp32 rows and a non-zero shift, and checks in every call:

  - accumulation: every fp64 output starts from random values of its own size, and out - initial is what is measured;
  - the workspace is filled with 0xFF bytes (NaN as floats) before each call; one case per pass runs again on a zeroed
    workspace, and both results must be bitwise equal;
  - the rows x, the matrix (unmix, M, W, H) and the codes are views of larger allocations whose rows past their end hold
    NaN (and f16f8's range flag, which a NaN sets, must stay 0); P's allocation has sentinel rows past B and every fp64
    output a sentinel guard past its end, and both must be unchanged.

Bars (tile ratio, element maximum) per pass, output and arithmetic, set from measurement on an H100 80GB HBM3 (700 W
limit): twice the worst value this file observes at any shape, rounded up, and never below 2^-24, the rounding of the
exact result to fp32, which every bar accepts (tests/test_row_pass_bounds_cpu.py). Every worst value comes from B = 1,
where a tile is a single outer product and nothing averages its rounding; at thousands of rows the same outputs measure
10 to 60 times lower. The leading-plane column is the ratio of a last tile recomputed from the leading operand plane
alone (the negative control below).

  pass     output   arith   worst tile  bar      worst element  bar      leading-plane tile  separated
  moments  gram     bf16x3  4.6e-6      9.2e-6   2.0e-5         4.0e-5   6.0e-5 (d = 8000)  yes
                    f16f8   2.3e-5      4.5e-5   1.3e-4         2.6e-4   7.6e-6 (d = 8000)  no
           col_sum  both    1.5e-8      6.0e-8   5.4e-8         1.1e-7   (fp64 sums of fp32 v; the 2^-24 floor)
  ica      gx       bf16x3  4.6e-7      9.3e-7   2.0e-6         3.9e-6   7.1e-7             no
                    f16f8   1.7e-6      3.4e-6   7.5e-6         1.6e-5   9.0e-8             no
           g_sum    bf16x3  2.1e-7      4.3e-7   1.4e-6         2.8e-6
                    f16f8   7.3e-7      1.5e-6   3.9e-6         7.7e-6
  project  p        bf16x3  9.3e-7      1.9e-6   5.3e-6         1.1e-5   1.2e-4             no (max criterion)
                    f16f8   4.2e-6      8.4e-6   2.4e-5         4.7e-5   1.5e-5             no (max criterion)
           norms    bf16x3  1.7e-7      3.4e-7   7.0e-7         1.5e-6
                    f16f8   8.3e-7      1.7e-6   3.2e-6         6.4e-6
  grams    wtw      bf16x3  2.7e-6      5.4e-6   1.3e-5         2.7e-5
                    f16f8   2.1e-5      4.2e-5   9.4e-5         1.9e-4
           wtv      bf16x3  3.2e-6      6.5e-6   1.4e-5         2.8e-5   1.3e-4             yes
                    f16f8   2.0e-5      4.1e-5   9.5e-5         1.9e-4   1.7e-5             no
  residual (one scalar)     2.4e-11     6.0e-8 (the 2^-24 floor), relative to ||V||^2 + || |W| |H| ||^2

Negative control (test_negative_control_leading_plane_tile): the last, ragged tile of gram (d = 8000), gx, W^T v and P
(d = n = 2000), B = 4001, recomputed from the leading operand plane alone (bf16 under bf16x3, the fp16 plane without
its E5M2 residual under f16f8) and spliced into the engine's output. For the outputs marked separated, the whole-output
criterion of tests/test_pca_gpu.py or test_nmf_gpu.py (a Frobenius ratio of 2e-5) accepts the spliced tensor and the
per-tile check rejects it at that tile. The others are printed, not claimed: under f16f8 and for gx the leading-plane
tile lies within the bar that B = 1 sets (at 4001 rows the fp16 plane alone is as close as a 3-pass single row), and
P's criterion in test_nmf_gpu.py is a maximum over elements, which a single bad tile does not dilute: it rejects the
spliced P itself.
"""
import ctypes as C

import pytest
import torch

from oracle import row_pass_bounds as RB
from oracle import tile_bounds as T
from sparse_coding_b200 import _lib

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
ARITHS = ("bf16x3", "f16f8")
DTYPES = (torch.float16, torch.float32)
ALPHA, ACCUMULATED, BARS = RB.ALPHA, RB.ACCUMULATED, RB.BARS   # (bars: see the module docstring)
GUARD = 8          # NaN rows past the end of every input, sentinel rows / elements past the end of every output
SENTINEL = 7.25
OUTPUTS = {"moments": ("gram", "col_sum"), "ica": ("gx", "g_sum"), "project": ("p", "norms"),
           "grams": ("wtw", "wtv")}
# outputs whose tile bar rejects a leading-plane last tile that the whole-output criterion accepts (the negative
# control asserts only these; the module docstring says why the others are not claimed)
SEPARATED = {"bf16x3": ("gram", "wtv"), "f16f8": ()}

# ---- the cases: (pass, d, n, row counts, arithmetics, input dtypes); n is the component count (unused by moments)
BOTH, BF = ARITHS, ("bf16x3",)
EDGE_B = (1, 63, 64, 65)
SLICE_B = (4096, 4095, 3841)        # at d = 512: 16 slices of 256 rows; the last full, one row short, a single row
BIG = 1 << 21
CASES = {
    "moments": [(128, 0, EDGE_B, BOTH, DTYPES), (512, 0, SLICE_B, BOTH, DTYPES), (512, 0, (64000, 65536), BOTH, DTYPES),
                (64, 0, (BIG,), BF, (torch.float16,)), (400, 0, (3000,), BOTH, DTYPES), (520, 0, (3000,), BF, DTYPES),
                (528, 0, (3000,), BOTH, DTYPES), (2048, 0, (65536,), BF, DTYPES)],
    "ica": [(128, 64, EDGE_B, BOTH, DTYPES), (512, 256, SLICE_B, BOTH, DTYPES), (512, 512, (64000, 65536), BOTH, DTYPES),
            (64, 64, (BIG,), BF, (torch.float16,)), (400, 400, (3000,), BOTH, DTYPES), (520, 520, (3000,), BF, DTYPES),
            (528, 528, (3000,), BOTH, DTYPES), (512, 8, (3000,), BF, DTYPES), (512, 16, (3000,), BOTH, DTYPES),
            (512, 208, (3000,), BOTH, DTYPES), (2048, 2048, (6144,), BF, DTYPES), (2048, 1920, (6144,), BF, DTYPES),
            (8192, 8192, (300,), ("f16f8",), (torch.float16,))],
    "project": [(128, 64, EDGE_B + (3841,), BOTH, DTYPES), (64, 64, (BIG,), BF, (torch.float16,)),
                (400, 400, (3000,), BOTH, DTYPES), (520, 520, (3000,), BF, DTYPES), (528, 528, (3000,), BOTH, DTYPES),
                (512, 8, (3000,), BF, DTYPES), (512, 16, (3000,), BOTH, DTYPES), (512, 208, (3000,), BOTH, DTYPES),
                (512, 256, (3000,), BOTH, DTYPES), (2048, 2048, (3000,), BF, DTYPES),
                (2048, 1920, (3000,), BF, DTYPES), (8192, 8192, (300,), ("f16f8",), (torch.float16,))],
    "grams": [(128, 64, EDGE_B, BOTH, DTYPES), (512, 256, SLICE_B, BOTH, DTYPES), (512, 512, (64000, 65536), BOTH, DTYPES),
              (64, 64, (BIG,), BF, (torch.float16,)), (400, 400, (3000,), BOTH, DTYPES), (520, 520, (3000,), BF, DTYPES),
              (528, 528, (3000,), BOTH, DTYPES), (512, 8, (3000,), BF, DTYPES), (512, 16, (3000,), BOTH, DTYPES),
              (512, 208, (3000,), BOTH, DTYPES), (2048, 2048, (6144,), BF, DTYPES),
              (2048, 1920, (6144,), BF, DTYPES)],
}
# one call per pass also runs on a zeroed workspace: (pass, d, n, B)
ZEROED = {("moments", 512, 0, 3841), ("ica", 512, 256, 3841), ("project", 128, 64, 3841), ("grams", 512, 256, 3841)}
# the residual: (d, k, row counts); fp32 products on the CUDA cores, no arithmetic to choose
RESIDUAL = [(72, 8, (1000, 65)), (72, 24, (1001,)), (72, 72, (64, 127)), (520, 40, (3001,)), (128, 128, (4096,))]


def runs(kind):
    """(d, n, B, arith, dtype) of every call of a pass."""
    for d, n, Bs, ariths, dtypes in CASES[kind]:
        for B in Bs:
            for arith in ariths:
                for dt in dtypes:
                    yield d, n, B, arith, dt


def f16f8_ok(d, n):
    return d % 16 == 0 and n % 16 == 0


def test_shapes_cover_every_edge():
    """The case list holds every edge of the slicing, of the tiles and of the cluster sizes the module docstring names
    (plain Python, before any GPU work)."""
    for kind in CASES:
        calls = list(runs(kind))
        for d, n, B, arith, _ in calls:
            assert arith == "bf16x3" or f16f8_ok(d, n), (kind, d, n, arith)
        Bs = {B for _, _, B, _, _ in calls}
        assert set(EDGE_B) <= Bs and BIG in Bs, kind
        assert any(n and n < d for d, n, *_ in calls) or kind == "moments", kind
        dims = {(d, a) for d, _, _, a, _ in calls}
        assert {(400, "bf16x3"), (400, "f16f8"), (520, "bf16x3"), (528, "bf16x3"), (528, "f16f8")} <= dims, kind
        assert (-(-400 // 128), 400 % 128 != 0, -(-520 // 128) % 2, -(-528 // 128) % 2) == (4, True, 1, 1)
        if kind != "moments":
            ns = {(n, a) for d, n, _, a, _ in calls if d == 512}
            assert {(8, "bf16x3"), (16, "bf16x3"), (16, "f16f8"), (208, "f16f8"), (256, "f16f8")} <= ns, kind
        cl = [(d, n, B, a, RB.pass_clusters(kind, d, n, B, a)) for d, n, B, a, _ in calls]
        if kind == "project":
            assert {c["gemm1"] for d, n, B, a, c in cl if d == 2048 and a == "bf16x3"} == {1, 2}
            assert any(c["gemm1"] == 2 and d == n == 8192 and a == "f16f8" for d, n, B, a, c in cl)
            continue
        S_R = {(d, B): RB.mom_slices(d, B) for d, _, B, _, _ in calls}
        # the last slice full, one row short, a single row (S > 1 each)
        assert any(S > 1 and B == S * R for (d, B), (S, R) in S_R.items()), kind
        assert any(S > 1 and B == S * R - 1 for (d, B), (S, R) in S_R.items()), kind
        assert any(S > 1 and B == (S - 1) * R + 1 for (d, B), (S, R) in S_R.items()), kind
        assert S_R[(512, 64000)] == (33, 1984) and S_R[(512, 65536)] == (32, 2048) and S_R[(64, BIG)] == (1024, 2048)
        wide = "wtv" if kind == "grams" else "sliced"
        pairs = {d for d, n, B, a, c in cl if c[wide] == 2}
        assert {512, 2048} <= pairs and pairs <= {512, 2048}, (kind, pairs)
        assert all(c[wide] == 1 for d, n, B, a, c in cl if d == 520 or a == "f16f8" or (d, B) == (512, 64000))
        if kind == "ica":
            assert {c["gemm1"] for d, n, B, a, c in cl if d == 2048 and a == "bf16x3"} == {1, 2}
            assert any(c["gemm1"] == 2 and d == n == 8192 and a == "f16f8" for d, n, B, a, c in cl)
    for kind, d, n, B in ZEROED:
        assert any((d, n, B) == r[:3] for r in runs(kind)), (kind, d, n, B)
    ks = {k for _, k, _ in RESIDUAL}
    assert {8, 24, 40} <= ks and any(k < d for d, k, _ in RESIDUAL) and any(d == 72 for d, _, _ in RESIDUAL)
    assert any(B % 64 for *_, Bs in RESIDUAL for B in Bs)


# ---- buffers with guards
def stream():
    return C.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)


def guarded_rows(t):
    """A copy of t [R, C] in an allocation of R + GUARD rows, NaN past R: (view, allocation)."""
    full = torch.full((t.shape[0] + GUARD, t.shape[1]), float("nan"), dtype=t.dtype, device=DEV)
    full[:t.shape[0]] = t
    return full[:t.shape[0]], full


def guarded_out(init):
    """An fp64 output holding `init`, with GUARD sentinel elements past its end: (view, allocation)."""
    full = torch.full((init.numel() + 2 * GUARD,), SENTINEL, dtype=torch.float64, device=DEV)
    full[:init.numel()] = init.flatten()
    return full[:init.numel()].view(init.shape), full


def check_guards(full, n_valid, what):
    assert bool((full[n_valid:] == SENTINEL).all()), f"{what}: written past its end"


def workspace(nbytes, fill):
    ws, ptr = _lib.workspace(nbytes, DEV, "workspace query")
    ws.fill_(fill)
    return ws, ptr, ws.numel() - 1024


# ---- operands
def operands(kind, d, n, B, dtype, seed):
    """x [B, d] (dtype), shift [d] (non-zero) and the pass's matrix: unmix [n, d], M [n, d] or W [B, n]."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    mu = 3.0 * torch.randn(d, generator=g, device=DEV)
    x = (torch.randn(B, d, generator=g, device=DEV) + mu).to(dtype)
    shift = (mu + 0.1 * torch.randn(d, generator=g, device=DEV)).contiguous()
    if kind == "moments":
        mat = None
    elif kind in ("ica", "project"):
        mat = torch.randn(n, d, generator=g, device=DEV) / d ** 0.5
    else:
        mat = torch.rand(B, n, generator=g, device=DEV) * (torch.rand(B, n, generator=g, device=DEV) < 0.3)
    return x, shift, mat


def call(kind, x, shift, mat, n, arith, inits, fill=0xFF):
    """One call of the pass on guarded copies of its inputs and outputs. Returns ({output: value}, where the fp64 outputs
    are out - initial) and checks the guards and the range flag."""
    lib = _lib.load()
    B, d = x.shape
    half = int(x.dtype == torch.float16)
    xv, xf = guarded_rows(x)
    mv, mf = guarded_rows(mat) if mat is not None else (None, None)
    flag = torch.zeros(1, dtype=torch.int32, device=DEV)
    outs = {k: guarded_out(v) for k, v in inits.items()}
    ptr = lambda k: outs[k][0].data_ptr()
    ar = _lib.arith_code(arith)
    if kind == "moments":
        ws, wp, wb = workspace(lib.sce_second_moments_workspace_bytes(d, B), fill)
        rc = lib.sce_second_moments(xv.data_ptr(), half, B, d, shift.data_ptr(), ar, ptr("col_sum"), ptr("gram"),
                                    flag.data_ptr(), wp, wb, stream())
    elif kind == "ica":
        ws, wp, wb = workspace(lib.sce_ica_pass_workspace_bytes(d, n, B), fill)
        rc = lib.sce_ica_pass(xv.data_ptr(), half, B, d, shift.data_ptr(), mv.data_ptr(), n, C.c_float(ALPHA), ar,
                              ptr("g_sum"), ptr("gx"), flag.data_ptr(), wp, wb, stream())
    elif kind == "project":
        pf = torch.full((B + GUARD, n), SENTINEL, dtype=torch.float32, device=DEV)
        ws, wp, wb = workspace(lib.sce_nmf_project_workspace_bytes(d, n, B), fill)
        rc = lib.sce_nmf_project(xv.data_ptr(), half, B, d, shift.data_ptr(), mv.data_ptr(), n, ar, pf.data_ptr(),
                                 ptr("norms"), flag.data_ptr(), wp, wb, stream())
    else:
        ws, wp, wb = workspace(lib.sce_nmf_grams_workspace_bytes(d, n, B), fill)
        rc = lib.sce_nmf_grams(xv.data_ptr(), half, B, d, shift.data_ptr(), mv.data_ptr(), n, ar, ptr("wtw"),
                               ptr("wtv"), flag.data_ptr(), wp, wb, stream())
    _lib.check(rc, f"row pass {kind}")
    torch.cuda.synchronize()
    assert int(flag.item()) == 0, "range flag set: a NaN past the inputs' end was read"
    got = {}
    for k, (view, full) in outs.items():
        check_guards(full, view.numel(), k)
        got[k] = view - inits[k]
    if kind == "project":
        assert bool((pf[B:] == SENTINEL).all()), "P written past row B"
        got["p"] = pf[:B].clone()
    del ws
    return got


def initial(want):
    """Random non-zero starting values of each accumulated output, of the size of its reference."""
    g = torch.Generator(device=DEV).manual_seed(want[0].numel())
    size = float(want[1].abs().mean()) + 1.0
    return size * (torch.rand(want[0].shape, generator=g, device=DEV, dtype=torch.float64) + 0.5)


def report(tag, kind, d, n, B, arith, r):
    S, R = RB.mom_slices(d, B) if kind != "project" else (1, -(-B // 64) * 64)
    cl = RB.pass_clusters(kind, d, n, B, arith)
    for k, v in r.items():
        tb, eb = BARS[kind][k][arith]
        print(f"{tag:42s} S x R = {S:4d} x {R:4d} clusters {cl} | {k:7s} worst tile {v['worst'][0]:.2e} at "
              f"{v['worst'][1]} element {v['elem']:.2e} | bars {tb:.1e} {eb:.1e}")


def run(kind, d, n, B, arith, dtype, zeroed=False):
    x, shift, mat = operands(kind, d, n, B, dtype, seed=d * 7919 + n * 31 + B)
    ref = RB.reference(kind, x, shift, mat, ALPHA)
    inits = {k: initial(ref[k]) for k in OUTPUTS[kind] if k in ACCUMULATED}
    got = call(kind, x, shift, mat, n, arith, inits)
    if zeroed:
        again = call(kind, x, shift, mat, n, arith, inits, fill=0)
        for k in got:
            assert torch.equal(got[k], again[k]), f"{k}: a zeroed workspace changes the result"
    tag = f"{kind} d={d} n={n} B={B} {arith} {str(dtype)[6:]}"
    r = {k: T.tile_ratios(got[k], *ref[k]) for k in OUTPUTS[kind]}
    report(tag, kind, d, n, B, arith, r)
    return tag, r


def check(kind, arith, tag, r):
    for k, v in r.items():
        tb, eb = BARS[kind][k][arith]
        assert v["worst"][0] <= tb, (tag, k, "tile", v["worst"], tb)
        assert v["elem"] <= eb, (tag, k, "element", v["elem"], eb)


@pytest.mark.parametrize("kind,case", [pytest.param(k, i, id=f"{k}-d{c[0]}-n{c[1]}-B{c[2][0]}")
                                       for k in CASES for i, c in enumerate(CASES[k])])
def test_every_tile_against_fp64(kind, case):
    d, n, Bs, ariths, dtypes = CASES[kind][case]
    for B in Bs:
        for arith in ariths:
            for dt in dtypes:
                tag, r = run(kind, d, n, B, arith, dt, zeroed=(kind, d, n, B) in ZEROED and arith == ariths[0]
                             and dt == dtypes[0])
                check(kind, arith, tag, r)
                del r
                torch.cuda.empty_cache()


def residual_call(x, shift, W, H, init, fill=0xFF):
    lib = _lib.load()
    B, d = x.shape
    k = W.shape[1]
    xv, _ = guarded_rows(x)
    wv, _ = guarded_rows(W)
    hv, _ = guarded_rows(H)
    out, full = guarded_out(torch.full((1,), init, dtype=torch.float64, device=DEV))
    ws, wp, wb = workspace(lib.sce_nmf_residual_workspace_bytes(d, B), fill)
    _lib.check(lib.sce_nmf_residual(xv.data_ptr(), int(x.dtype == torch.float16), B, d, shift.data_ptr(), wv.data_ptr(),
                                    k, hv.data_ptr(), out.data_ptr(), wp, wb, stream()), "sce_nmf_residual")
    torch.cuda.synchronize()
    check_guards(full, 1, "residual")
    return float(out) - init


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("shape", RESIDUAL, ids=lambda s: f"d{s[0]}_k{s[1]}")
def test_residual_against_fp64(shape, dtype):
    """||V - W H||^2 against fp64, relative to ||V||^2 + || |W| |H| ||^2, accumulated into a non-zero start."""
    d, k, Bs = shape
    for B in Bs:
        g = torch.Generator(device=DEV).manual_seed(d + k + B)
        H = torch.rand(k, d, generator=g, device=DEV) * (torch.rand(k, d, generator=g, device=DEV) < 0.3)
        W = torch.rand(B, k, generator=g, device=DEV) * (torch.rand(B, k, generator=g, device=DEV) < 0.3)
        shift = 0.25 * torch.ones(d, device=DEV) + 0.01 * torch.randn(d, generator=g, device=DEV)
        x = (W @ H + shift + 1e-2 * torch.randn(B, d, generator=g, device=DEV)).to(dtype)
        want, scale = RB.nmf_residual(RB.shifted(x, shift, clamp=True), W, H)
        init = 0.5 * want + 1.0
        got = residual_call(x, shift, W, H, init)
        again = residual_call(x, shift, W, H, init, fill=0)
        e = abs(got - want) / scale
        print(f"residual d={d} k={k} B={B} {str(dtype)[6:]}: {e:.2e} of ||V||^2 + |||W||H|||^2 "
              f"(residual {want / scale:.1e} of it) | bar {BARS['residual']:.1e}")
        assert got == again
        assert e <= BARS["residual"], (d, k, B, e)


# ---- negative control
def lead(t, arith):
    """The values of t's leading operand plane: bf16 (bf16x3) or the fp16 plane alone (f16f8)."""
    t = t.float()
    return (t.bfloat16() if arith == "bf16x3" else t.half()).double()


# (pass, output, d = n): the last tile of each is ragged (80 x 80 at d = 2000; 64 x 64 of 63 x 63 tiles at d = 8000,
# enough tiles that the Gram's Frobenius criterion dilutes one of them below its bar)
CONTROLS = (("moments", "gram", 8000), ("ica", "gx", 2000), ("grams", "wtv", 2000), ("project", "p", 2000))


@pytest.mark.parametrize("arith", ARITHS)
def test_negative_control_leading_plane_tile(arith):
    B = 4001                    # P: 32 x 16 tiles, the last one 33 x 80
    out = {}
    for kind, name, d in CONTROLS:
        n = d
        x, shift, mat = operands(kind, d, n, B, torch.float32, seed=4242)
        ref = RB.reference(kind, x, shift, mat, ALPHA)
        inits = {k: torch.zeros_like(ref[k][0]) for k in OUTPUTS[kind] if k in ACCUMULATED}
        got = call(kind, x, shift, mat, n, arith, inits)[name]
        want, scale = ref[name]
        del ref
        R, Cc = want.shape
        r0, c0 = (R - 1) // 128 * 128, (Cc - 1) // 128 * 128
        V = RB.shifted(x, shift, clamp=kind in ("project", "grams"))
        if kind == "moments":
            tile = lead(V[:, r0:], arith).T @ lead(V[:, c0:], arith)
        elif kind == "ica":
            t = torch.tanh(ALPHA * (V @ mat.double().T))
            tile = lead(t[:, r0:], arith).T @ lead(V[:, c0:], arith)
        elif kind == "grams":
            tile = lead(mat[:, r0:], arith).T @ lead(V[:, c0:], arith)
        else:
            tile = lead(V[r0:], arith) @ lead(mat[c0:], arith).T
        spliced = got.double().clone()
        spliced[r0:, c0:] = tile
        if name == "p":     # test_nmf_gpu.py: max error over max |P|
            whole = float((spliced - want).abs().max() / want.abs().max())
            bar = 2e-5 if arith == "bf16x3" else 1.5e-4
        else:               # test_pca_gpu.py (2e-5), test_ica_gpu.py (1.5e-4), test_nmf_gpu.py (2e-5): Frobenius
            whole = float((spliced - want).norm() / want.norm())
            bar = 1.5e-4 if name == "gx" else 2e-5
        r = T.tile_ratios(spliced, want, scale)
        r3 = T.tile_ratios(got, want, scale)
        at = (0, (R - 1) // 128, (Cc - 1) // 128)
        tb = BARS[kind][name][arith][0]
        print(f"negative control {arith:6s} {name:4s} d={d}: whole-output {whole:.2e} (bar {bar:.1e}); spliced tile "
              f"{float(r['ratio'][at]):.2e}, 3-pass worst {r3['worst'][0]:.2e}, tile bar {tb:.1e}")
        out[name] = (whole, bar, r["worst"], at, tb)
        del got, want, scale, spliced, r, r3, V
        torch.cuda.empty_cache()
    for name in SEPARATED[arith]:
        whole, bar, worst, at, tb = out[name]
        assert whole <= bar, (name, whole, bar)                     # the whole-output criterion misses the tile ...
        assert worst[0] > tb and worst[1] == at, (name, worst, at, tb)   # ... the per-tile check does not
