"""CPU emulation A/B of operand arithmetics (oracle/arith_emulation.py): the two the engine implements and the
block-scaled 4-bit cross-term candidate of DESIGN.md section 9.1, on a tied-SAE step (forward, x_hat, pattern-pinned
weight gradient) against fp64.   python tools/arith_ab.py"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from oracle import arith_emulation as A


def rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm())


def problem(d, n, B, seed, kind):
    g = torch.Generator().manual_seed(seed)
    if kind == "mixture":                      # the bench's distribution: sparse mixture of unit features + noise
        feats = torch.randn(1024, d, generator=g)
        feats /= feats.norm(dim=1, keepdim=True)
        codes = (torch.rand(B, 1024, generator=g) < 0.01).float() * torch.rand(B, 1024, generator=g)
        x = codes @ feats + 0.05 * torch.randn(B, d, generator=g)
    else:
        x = torch.randn(B, d, generator=g)
        if kind == "outliers":
            x[:, :4] *= 200.0
    E = torch.randn(n, d, generator=g)
    W = E / E.norm(dim=1, keepdim=True)
    return x, W, 0.02 * torch.randn(n, generator=g)


def fp64_step(x, W, bias, alpha):
    B, d = x.shape
    xd, Wd = x.double(), W.double()
    z = xd @ Wd.T + bias.double()
    act = z > 0
    c = z.clamp(min=0)
    xh = c @ Wd
    r = xh - xd
    dz = (r @ Wd.T * (2 / (B * d)) + alpha / B) * act
    return z, act, xh, dz.T @ xd + c.T @ (r * (2 / (B * d)))


ARITHS = [
    ("bf16x3 (implemented)", A.mm_bf16x3, "3", "4"),
    ("f16f8  (implemented, default)", A.mm_f16f8, "2", "4"),
    ("f16 + MXFP4 cross terms, OCP scale (saturating)", A.make_mm_f16mx4(True), "1.5", "3.06"),
    ("f16 + MXFP4 cross terms, scale rounded up", A.make_mm_f16mx4(False), "1.5", "3.06"),
    ("fp16 plane only (no cross terms)", lambda a, b: a.half().double() @ b.half().double(), "1", "2"),
]
print("# CPU emulation (fp64 accumulation) of one tied-SAE step: relative errors against fp64; d = 256, n = 1024, B = 512,")
print("# ReLU pattern pinned to the fp64 one for the gradient. Bar of the north star: 1e-4 on x_hat and the loss.")
print(f"{'arithmetic':52s} {'passes':>6s} {'B/elem':>6s}  " + "  ".join(f"{k:>30s}" for k in ("Gaussian", "x200 outlier dimensions", "sparse mixture (bench)")))
print(f"{'':52s} {'':>6s} {'':>6s}  " + "  ".join(f"{'z':>9s} {'x_hat':>9s} {'dW':>9s} " for _ in range(3)))
for name, mm, passes, byt in ARITHS:
    cells = []
    for kind in ("gauss", "outliers", "mixture"):
        x, W, bias = problem(256, 1024, 512, 0, kind)
        z64, act, xh64, dW64 = fp64_step(x, W, bias, 1e-2)
        z, xh, dW = A.tied_step_emulated(mm, x, W, bias, 1e-2, pin_active=act)
        cells.append(f"{rel(z, z64):9.1e} {rel(xh, xh64):9.1e} {rel(dW, dW64):9.1e} ")
    print(f"{name:52s} {passes:>6s} {byt:>6s}  " + "  ".join(cells))
print("""
# Reading: MXFP4 cross terms keep x_hat at 4-5e-5 — inside the 1e-4 bar but with 2x instead of 5x margin. The gain would
# be fewer operand bytes per element (4 -> 3.06); it needs a GPU with block-scaled FP4 MMA, which sm_90 does not have.""")
