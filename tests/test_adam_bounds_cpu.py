"""The per-element Adam bars of oracle/adam_bounds.py: they accept an fp32 emulation of the engine's adam_apply
(sparse_coding_b200/csrc/sce_kernels.cuh) under every choice of FMA contraction the compiler may make, over adversarial
inputs, and reject each planted defect of the step. Also shows that at step 1 from zero moments the emulation is
exactly the closed form tests/test_adam_step_gpu.py asserts: m' = fp32((1 - b1) g), v' = fp32(fp32((1 - b2) g) g)."""
import numpy as np
import pytest
import torch

from oracle import adam_bounds as A
from sparse_coding_b200.optim import AdamConfig

f32 = np.float32
DEFAULT = AdamConfig()
OTHER = AdamConfig(lr=3e-3, b1=0.8, b2=0.99, eps=1e-6)
ORDERS = ["none", "first", "second"]     # no contraction; the first or the second product of each sum fused


def fma32(a, b, c):
    """fp32 fma(a, b, c), correctly rounded: a b is exact in fp64, the sum is rounded to odd in fp64 (TwoSum error
    decides the direction), and 53 >= 24 + 2 bits make the final rounding to fp32 the correct one."""
    a, b, c = (np.asarray(x, dtype=f32).astype(np.float64) for x in (a, b, c))
    p = a * b
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)
    even = (s.view(np.int64) & 1) == 0
    s = np.where((err != 0) & even, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)
    return s.astype(f32)


def bias_corrections(h, t):
    """hyper_for: 1 - b^t in fp64 from the fp32 betas, rounded once to fp32."""
    return f32(1.0 - float(f32(h.b1)) ** t), f32(1.0 - float(f32(h.b2)) ** t)


def adam_apply32(p, g, m, v, h, t, order="none", defect=None):
    """adam_apply in fp32 (numpy), the FMA contraction given by ``order``; ``defect`` plants one of DEFECTS."""
    p, g, m, v = (np.asarray(x, dtype=f32) for x in (p, g, m, v))
    lr, b1, b2, eps, eps_root = (f32(getattr(h, k)) for k in ("lr", "b1", "b2", "eps", "eps_root"))
    t = t + {"t+1": 1, "t-1": -1}.get(defect, 0)
    bc1, bc2 = bias_corrections(h, t)
    if defect == "bc swapped":
        bc1, bc2 = bc2, bc1
    if defect == "eps_root dropped":
        eps_root = f32(0)
    bv = b1 if defect == "b1 in v" else b2
    one = f32(1)
    if order == "first":
        m2 = fma32(b1, m, (one - b1) * g)
        v2 = fma32(bv, v, ((one - bv) * g) * g)
    elif order == "second":
        m2 = fma32(one - b1, g, b1 * m)
        v2 = fma32((one - bv) * g, g, bv * v)
    else:
        m2 = b1 * m + (one - b1) * g
        v2 = bv * v + ((one - bv) * g) * g
    mu, nu = (m, v) if defect == "old moments" else (m2, v2)
    mh = mu / bc1
    vh = nu / bc2
    if defect == "eps in sqrt":
        den = np.sqrt(vh + eps_root + eps)
    else:
        den = np.sqrt(vh + eps_root) + eps
    q = mh / den
    p2 = fma32(-lr, q, p) if order != "none" else p - lr * q
    return p2, m2, v2


def ratios(p, g, m, v, h, t, out):
    ref = A.reference(*(torch.from_numpy(np.asarray(x, dtype=f32)) for x in (p, g, m, v)), t, h)
    return {k: A.ratios(torch.from_numpy(o), ref[k], ref["bar_" + k]) for k, o in zip(("p", "m", "v"), out)}


def inputs(kind, n=20000, seed=0):
    """(p, g, m, v) of one adversarial kind, fp32."""
    r = np.random.default_rng(seed)
    p = r.normal(0, 0.05, n)
    g = r.normal(0, 1e-3, n) * np.exp(r.normal(0, 1, n))
    m = r.normal(0, 1e-4, n)
    v = np.abs(r.normal(0, 1e-6, n))
    if kind == "zero_grad":
        g = np.zeros(n)
    elif kind == "tiny_grad":                    # |g| << eps
        g, m, v = g * 1e-9, m * 1e-9, v * 1e-18
    elif kind == "large_grad":
        g, m, v = g * 1e6, m * 1e6, v * 1e12
    elif kind == "cancelling":                   # m of the opposite sign: b1 m + (1 - b1) g close to 0
        b1 = float(f32(0.9))
        m = -(1 - b1) / b1 * g * (1 + r.normal(0, 1e-6, n))
    elif kind == "subnormal_v":                  # v and (1 - b2) g^2 below 2^-126
        g, m, v = g * 1e-18, m * 1e-18, np.abs(r.normal(0, 1e-39, n))
    elif kind == "zero_moments":
        m, v = np.zeros(n), np.zeros(n)
    elif kind == "small_v":                      # v / bc2 comparable to eps
        g, m, v = g * 1e-2, m * 1e-2, v * 1e-4
    return tuple(x.astype(f32) for x in (p, g, m, v))


KINDS = ["generic", "zero_grad", "tiny_grad", "large_grad", "cancelling", "subnormal_v", "zero_moments", "small_v"]


@pytest.mark.parametrize("t", [1, 2, 50, 1000])
@pytest.mark.parametrize("hyper", ["default", "other", "large_eps_root"])
@pytest.mark.parametrize("kind", KINDS)
def test_bars_accept_the_fp32_step(kind, hyper, t):
    """Every FMA contraction of the fp32 step is within every bar, on every kind of input."""
    h = {"default": DEFAULT, "other": OTHER, "large_eps_root": AdamConfig(eps_root=1.0)}[hyper]
    x = inputs(kind)
    for order in ORDERS:
        r = ratios(*x, h, t, adam_apply32(*x, h, t, order))
        for k, v in r.items():
            assert float(v.max()) <= 1.0, (kind, hyper, t, order, k, float(v.max()))


def test_bars_are_tight_enough_to_matter():
    """The fp32 step uses a visible share of each bar on generic inputs (the bars are not vacuous)."""
    x = inputs("generic")
    r = ratios(*x, DEFAULT, 3, adam_apply32(*x, DEFAULT, 3, "none"))
    for k, v in r.items():
        assert float(v.max()) >= 0.05, (k, float(v.max()))


DEFECTS = {
    # defect: (output whose bar rejects it, step number, hyper-parameters, inputs)
    "t+1": ("p", 3, DEFAULT, "generic"),
    "t-1": ("p", 3, DEFAULT, "generic"),
    "bc swapped": ("p", 3, DEFAULT, "generic"),
    "eps in sqrt": ("p", 3, DEFAULT, "small_v"),          # visible where v / bc2 is not far above eps
    "eps_root dropped": ("p", 3, AdamConfig(eps_root=1e-6), "generic"),
    "b1 in v": ("v", 3, DEFAULT, "generic"),
    "old moments": ("p", 3, DEFAULT, "generic"),
}


@pytest.mark.parametrize("defect", list(DEFECTS))
def test_bars_reject_planted_defects(defect):
    """Most elements of the output the defect corrupts fail their bar, under every contraction."""
    out, t, h, kind = DEFECTS[defect]
    x = inputs(kind, seed=1)
    for order in ORDERS:
        r = ratios(*x, h, t, adam_apply32(*x, h, t, order, defect))[out]
        assert float((r > 1).double().mean()) > 0.5, (defect, order, float((r > 1).double().mean()))


def test_bars_reject_a_gradient_eight_ulps_off():
    """At step 1 from zero moments, a gradient 8 ulps off fails the m' bar at every element."""
    p, g, m, v = inputs("zero_moments", seed=2)
    g_off = g.copy()
    for _ in range(8):
        g_off = np.nextafter(g_off, np.full_like(g_off, np.inf))
    for order in ORDERS:
        r = ratios(p, g, m, v, DEFAULT, 1, adam_apply32(p, g_off, m, v, DEFAULT, 1, order))["m"]
        assert bool((r > 1).all()), (order, float(r.min()))


@pytest.mark.parametrize("hyper", ["default", "other"])
def test_step_one_closed_form(hyper):
    """From zero moments, every contraction gives m' = fp32((1 - b1) g) and v' = fp32(fp32((1 - b2) g) g) exactly:
    the identity the GPU test uses to show that the step applied the gradient grads_batch reports."""
    h = DEFAULT if hyper == "default" else OTHER
    for kind in ("generic", "large_grad", "tiny_grad", "zero_moments"):
        p, g, _, _ = inputs(kind, seed=3)
        z = np.zeros_like(g)
        b1, b2 = f32(h.b1), f32(h.b2)
        for t in (1, 2, 50):
            for order in ORDERS:
                _, m2, v2 = adam_apply32(p, g, z, z, h, t, order)
                assert np.array_equal(m2, (f32(1) - b1) * g), (kind, t, order)
                assert np.array_equal(v2, ((f32(1) - b2) * g) * g), (kind, t, order)


def test_fma32_is_correctly_rounded():
    """The emulated fma against an exact rational computation, at inputs chosen to make double rounding likely."""
    from fractions import Fraction
    r = np.random.default_rng(4)
    a = r.normal(0, 1, 400).astype(f32)
    b = r.normal(0, 1, 400).astype(f32)
    # c cancels most of a b, so the exact sum's low bits decide the rounding
    c = (-(a.astype(np.float64) * b)).astype(f32) + (r.normal(0, 1e-7, 400)).astype(f32)
    got = fma32(a, b, c)
    for i in range(400):
        exact = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        lo = f32(float(exact))
        cands = [lo, np.nextafter(lo, f32(np.inf)), np.nextafter(lo, f32(-np.inf))]
        best = min(cands, key=lambda y: (abs(Fraction(float(y)) - exact), int(np.float32(y).view(np.int32)) & 1))
        assert got[i] == best, (i, got[i], best)
