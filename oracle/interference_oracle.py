"""fp64 restatement of the reference's calc_expected_interference (big_sweep.py:43-57). Its ``batch`` argument is the
CODE [B, n], not the activations. Every dictionary row is divided by max(||row||, 1e-8), whatever the dictionary's own
decode normalises; cap = c / max(totals, 1e-8), so a signed code whose totals fall to or below zero takes the clamp; the
non-zero count is floored at 1 (SURVEY Q15).

Device-agnostic: runs on the CPU against tests/golden/interference.pt and on the GPU at scale, where the code is taken
in slices of rows so that the [B, n] intermediates stay small."""
import torch

CLAMP = 1e-8


def normalised(dictionary):
    w = dictionary.double()
    return w / w.norm(dim=-1).clamp(min=CLAMP)[:, None]


def sums(dictionary, code, rows=8192, margin=0.0):
    """(cap_sums [n] fp64, nz_counts [n] int64, fragile [n] bool) of ``code`` [B, n] with ``dictionary`` [n, d].
    ``fragile`` marks the features with some row where c != 0 and |totals| <= ``margin``: there totals is a difference of
    nearly equal terms (signed codes), so c / max(totals, 1e-8) has no useful fp32 accuracy."""
    wn = normalised(dictionary).to(code.device)
    cos2 = (wn @ wn.T).pow(2)
    n = wn.shape[0]
    cap = torch.zeros(n, dtype=torch.float64, device=code.device)
    nz = torch.zeros(n, dtype=torch.int64, device=code.device)
    fragile = torch.zeros(n, dtype=torch.bool, device=code.device)
    for s in range(0, code.shape[0], rows):
        c = code[s:s + rows].double()
        totals = c @ cos2.T                     # totals[b, i] = sum_j cos^2(i, j) c[b, j]
        cap += (c / totals.clamp(min=CLAMP)).sum(0)
        active = c != 0
        nz += active.sum(0)
        fragile |= (active & (totals.abs() <= margin)).any(0)
    return cap, nz, fragile


def expected_interference(dictionary, code):
    """[n] fp64: the reference's nonzero_capacity."""
    cap, nz, _ = sums(dictionary, code)
    return cap / nz.clamp(min=1).double()
