"""fp64 restatement of the reference's record selection for reading what features mean (interpret.py:82-212
make_feature_activation_dataset encodes each fragment of 64 rows, with no ``center()``, and keeps its per-feature
maximum; :265-321 interpret takes per feature the 20 fragments with the largest maximum and 20 random fragments whose
maximum is non-zero, and skips the feature when fewer than 20 such fragments exist), with the engine's determinism:
ties in the top list go to the lower fragment index, and the random draw is the order of a counter-based priority
(splitmix64 of seed, feature and fragment), which has the distribution of the reference's fresh permutation per
feature. Device-agnostic: runs on the CPU against tests/golden/interp.pt and on the GPU at scale.

A dictionary is the dict of fp64 tensors of oracle/eval_oracle.py."""
import torch

from oracle import eval_oracle as E

_MASK64 = (1 << 64) - 1


def _s64(c):
    """An unsigned 64-bit constant as the int64 with the same bits."""
    return c - (1 << 64) if c >= 1 << 63 else c


def _srl(z, s):
    """Logical right shift of int64 bit patterns."""
    return (z >> s) & ((1 << (64 - s)) - 1)


def splitmix64(z: torch.Tensor) -> torch.Tensor:
    """splitmix64 on int64 tensors holding uint64 bit patterns (torch's int64 products wrap modulo 2^64)."""
    z = z + _s64(0x9E3779B97F4A7C15)
    z = (z ^ _srl(z, 30)) * _s64(0xBF58476D1CE4E5B9)
    z = (z ^ _srl(z, 27)) * _s64(0x94D049BB133111EB)
    return z ^ _srl(z, 31)


def priority(seed: int, features: torch.Tensor, fragments: torch.Tensor) -> torch.Tensor:
    """[G, n] int64: splitmix64(splitmix64(splitmix64(seed) ^ feature) ^ fragment) >> 1 for fragments [G] x features [n]."""
    s = splitmix64(torch.tensor(_s64(int(seed) & _MASK64), dtype=torch.int64, device=features.device))
    h = splitmix64(s ^ features.long())
    return _srl(splitmix64(h[None, :] ^ fragments.long()[:, None]), 1)


def fragment_tables(code: torch.Tensor, L: int):
    """code [N, n] -> (maxima [G, n], active [G, n] bool) over fragments of L rows."""
    G = code.shape[0] // L
    c = code[: G * L].reshape(G, L, -1)
    return c.amax(1), (c > 0).any(1)


def select_top(fmax: torch.Tensor, n_top: int) -> torch.Tensor:
    """[n, n_top] fragments by (maximum descending, fragment ascending); -1 past the last fragment."""
    order = torch.sort(fmax.T, dim=-1, descending=True, stable=True).indices[:, :n_top]
    pad = n_top - order.shape[1]
    return torch.nn.functional.pad(order, (0, pad), value=-1) if pad > 0 else order


def select_random(active: torch.Tensor, n_random: int, seed: int) -> torch.Tensor:
    """[n, n_random] active fragments in draw order (priority descending, fragment ascending); -1 where unfilled."""
    G, n = active.shape
    p = priority(seed, torch.arange(n, device=active.device), torch.arange(G, device=active.device))
    p = torch.where(active, p, torch.full_like(p, -1)).T                      # inactive: below every priority
    order = torch.sort(p, dim=-1, descending=True, stable=True).indices[:, :n_random]
    ok = torch.gather(active.T, 1, order)
    out = torch.where(ok, order, torch.full_like(order, -1))
    pad = n_random - out.shape[1]
    return torch.nn.functional.pad(out, (0, pad), value=-1) if pad > 0 else out


def select(m, x: torch.Tensor, L: int = 64, n_top: int = 20, n_random: int = 20, seed: int = 0, rows: int = 8192):
    """The records of dictionary ``m`` on activations ``x`` [N, d] (raw rows, no centring): dict with ``code`` [N, n],
    ``fmax`` / ``active`` [G, n], ``top_fragments`` [n, n_top], ``random_fragments`` [n, n_random],
    ``n_active_fragments`` [n] and ``skipped`` [n]."""
    x = x.double()
    code = torch.cat([E.encode(m, x[i:i + rows]) for i in range(0, x.shape[0], rows)])
    fmax, active = fragment_tables(code, L)
    n_act = active.sum(0)
    return {"code": code, "fmax": fmax, "active": active, "top_fragments": select_top(fmax, n_top),
            "random_fragments": select_random(active, n_random, seed), "n_active_fragments": n_act,
            "skipped": n_act < n_random}


def fragment_values(code: torch.Tensor, frags: torch.Tensor, L: int) -> torch.Tensor:
    """[n, k] fragments -> [n, k, L] per-token values of each feature on them (0 where the fragment is -1)."""
    n, k = frags.shape
    t = torch.arange(L, device=code.device)
    r = (frags.clamp(min=0)[..., None] * L + t).reshape(n, -1)                  # [n, k L] rows
    v = torch.gather(code.T, 1, r).reshape(n, k, L)
    return torch.where(frags[..., None] >= 0, v, torch.zeros((), dtype=v.dtype, device=v.device))
