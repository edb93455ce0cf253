"""TEST INFRASTRUCTURE ONLY (like everything under oracle/): a CPU emulation of the engine's two operand arithmetics
(include/sce.h `sce_arith`, DESIGN.md section 2), exact in everything but the tensor core's fp32 accumulation order —
products are accumulated in fp64 here. It pins the ERROR MODEL of the arithmetics without a GPU: what the planes can
represent, which partial products are formed, what is dropped.

  f16f8 : x ~= h + l,  h = fp16(x);  planes: h (fp16), h8 = e5m2(x), l8 = e5m2((x - h) * 2^11)
          a @ b ~= h_a @ h_b + (l8_a @ h8_b + h8_a @ l8_b) * 2^-11        (sce_ptx.cuh "fp16 + fp8 arithmetic")
  bf16x3: x ~= hi + lo, hi = bf16(x), lo = bf16(x - hi)
          a @ b ~= hi_a @ hi_b + lo_a @ hi_b + hi_a @ lo_b                 (sce_gemm.cuh)
"""
import torch

LO_SHIFT = 11            # kLoShift in sparse_coding_b200/csrc/sce_ptx.cuh
_S = float(1 << LO_SHIFT)


def planes_f16f8(a: torch.Tensor):
    """(h, h8, l8) as fp32 tensors holding exactly the values the device planes hold."""
    a = a.float()
    h = a.half().float()
    h8 = a.to(torch.float8_e5m2).float()
    l8 = ((a - h) * _S).to(torch.float8_e5m2).float()
    return h, h8, l8


def mm_f16f8(a: torch.Tensor, b: torch.Tensor, skip_a_residual: bool = False) -> torch.Tensor:
    """a [m,k] @ b [k,n] in the f16f8 arithmetic (fp64 accumulation). ``skip_a_residual`` drops the l8_a @ h8_b term,
    as the device does when a's residual plane is flagged all-zero."""
    ah, a8, al = planes_f16f8(a)
    bh, b8, bl = planes_f16f8(b)
    cross = a8.double() @ bl.double()
    if not skip_a_residual:
        cross = cross + al.double() @ b8.double()
    return ah.double() @ bh.double() + cross / _S


def mm_bf16x3(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    a, b = a.float(), b.float()
    ah = a.bfloat16().float()
    al = (a - ah).bfloat16().float()
    bh = b.bfloat16().float()
    bl = (b - bh).bfloat16().float()
    return ah.double() @ bh.double() + al.double() @ bh.double() + ah.double() @ bl.double()


def tied_step_emulated(mm, x, W, bias, alpha, pin_active=None):
    """Forward + backward GEMMs of the tied SAE in the given arithmetic, in the scaling the engine uses for f16f8 (the
    backward pass runs on the residual r, outputs are multiplied by 2/(B d)). W: unit-norm rows [n,d]. Returns
    (z, x_hat, dW); ``pin_active`` (bool [B,n]) pins the ReLU pattern."""
    B, d = x.shape
    z = mm(x, W.T.contiguous()).float() + bias
    active = (z > 0) if pin_active is None else pin_active
    c = (z * active).float()
    x_hat = mm(c, W).float()
    r = x_hat - x
    dz = ((mm(r, W.T.contiguous()).float() + alpha * d / 2) * active).float()
    dW = (mm(dz.T.contiguous(), x) + mm(c.T.contiguous(), r)) * (2.0 / (B * d))
    return z, x_hat, dW


# ----------------------------------------------------------------------------------------------------------------
# Candidate (NOT implemented on the device; DESIGN.md section 9.1): cross terms on block-scaled 4-bit planes
# (block-scaled FP4 MMA, which sm_90 does not have: E2M1 elements, one E8M0 scale per 32 elements along K, K = 64 per instruction at four times the
# kind::f16 rate): 1 + 2 * 1/4 = 1.5 pass-equivalents and 2 + 0.5 + 0.5 (+ scales) ~= 3.06 bytes per operand element.
# ----------------------------------------------------------------------------------------------------------------
_E2M1 = torch.tensor([0.0, 0.5, 1.0, 1.5, 2.0, 3.0, 4.0, 6.0])


def mxfp4(t: torch.Tensor, block: int = 32, saturate: bool = True) -> torch.Tensor:
    """Values of `t` after MXFP4 quantisation along the LAST dim (blocks of `block`; zero-padded): shared power-of-two
    scale 2^(floor(log2(amax)) - 2) as in the OCP MX spec (elements in (6, 8) * scale then saturate to 6), or with
    ``saturate=False`` the next scale up (nothing saturates, one bit less for the rest of the block)."""
    t = t.double()
    k = t.shape[-1]
    pad = (-k) % block
    if pad:
        t = torch.nn.functional.pad(t, (0, pad))
    b = t.reshape(*t.shape[:-1], -1, block)
    amax = b.abs().amax(dim=-1, keepdim=True).clamp(min=1e-300)
    e = torch.floor(torch.log2(amax)) - 2.0
    if not saturate:
        e = torch.where(amax / torch.exp2(e) > 6.0, e + 1.0, e)
    q = (b / torch.exp2(e)).clamp(-6.0, 6.0)
    grid = _E2M1.double()
    idx = (q.abs().unsqueeze(-1) - grid).abs().argmin(dim=-1)          # nearest grid point (ties: the lower index)
    out = torch.sign(q) * grid[idx] * torch.exp2(e)
    return out.reshape(*t.shape[:-1], -1)[..., :k]


def make_mm_f16mx4(saturate: bool = True):
    def mm(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
        """a [m,k] @ b [k,n]: fp16 x fp16 dominant term + two cross terms whose four planes are MXFP4 along k."""
        a, b = a.float(), b.float()
        ah, bh = a.half().float(), b.half().float()
        al, bl = (a - ah), (b - bh)                                        # block scaling needs no 2^11 shift
        q = lambda t: mxfp4(t, saturate=saturate)
        bt, blt = b.T.contiguous(), bl.T.contiguous()                      # blocks run along k for both operands
        cross = q(al) @ q(bt).T + q(a) @ q(blt).T
        return ah.double() @ bh.double() + cross
    return mm
