"""Shared by the expected-interference tests: the golden fixture's cases and the workspace size libsce documents."""
import torch

from oracle import interference_oracle as IO

KINDS = ("tied", "untied", "topk", "ica")


def cases(golden):
    """{name: case} of tests/golden/interference.pt: dictionary [n, d], code [B, n], the reference's result, counts."""
    return {c["name"]: c for c in golden("interference")["cases"]}


def workspace_bytes(M, n, d, B):
    """The size include/sce.h gives: the normalised dictionary [M][n][ceil(d / 32) 32] and the partials
    [M][ceil(B / 32)][2][n], fp32, each carved at a 1024-byte boundary."""
    up = lambda v: -(-v // 1024) * 1024
    return up(up(4 * M * n * (-(-d // 32) * 32)) + 4 * M * (-(-B // 32)) * 2 * n)


def oracle_of_codes(dictionary, codes, margin=0.0):
    """fp64 (cap_sums, nz_counts, fragile) of the list of codes [B_i, n] with one dictionary, summed over the list."""
    cap = nz = fragile = None
    for c in codes:
        a, b, f = IO.sums(dictionary, c, margin=margin)
        cap, nz, fragile = (a, b, f) if cap is None else (cap + a, nz + b, fragile | f)
    return cap, nz, fragile


def rel_err(a, b):
    """max over entries of |a - b| / max(|b|, 1e-30) (fp64)."""
    a, b = a.double(), b.double().to(a.device)
    return float(((a - b).abs() / b.abs().clamp(min=1e-30)).max())
