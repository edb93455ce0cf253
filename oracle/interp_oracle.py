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


# ----------------------------------------------------------------------------------------------------------------------
# one engine call (sce_forward_fragments' fragment_merge_kernel) and the per-element bounds of its values
# ----------------------------------------------------------------------------------------------------------------------
def list_order(key: torch.Tensor, frag: torch.Tensor) -> torch.Tensor:
    """[n, k] -> [n, k] per row, the permutation that sorts (key descending, fragment ascending) with the empty entries
    (fragment < 0) last. The key of an empty entry is never compared: it may be anything, NaN included."""
    empty = frag < 0
    key = torch.where(empty, torch.zeros_like(key), key)
    o = torch.sort(torch.where(empty, torch.iinfo(torch.int64).max, frag), dim=-1, stable=True).indices
    o = o.gather(-1, torch.sort(key.gather(-1, o), dim=-1, descending=True, stable=True).indices)
    return o.gather(-1, torch.sort(empty.gather(-1, o).to(torch.int8), dim=-1, stable=True).indices)


def _keep(key, frag, rows, cand_key, cand_frag, frag0, code, L, cap):
    """The ``cap`` highest of a list (key, frag, rows: [n, cap], [n, cap], [n, cap, L] or None) and the candidates
    (cand_key, cand_frag: [n, G], fragment -1 where not a candidate; their rows are those of ``code``), in list order."""
    if cap == 0:
        return key, frag, rows
    allk, allf = torch.cat([key, cand_key.to(key.dtype)], 1), torch.cat([frag, cand_frag], 1)
    idx = list_order(allk, allf)[:, :cap]
    f = allf.gather(1, idx)
    empty = f < 0
    k = torch.where(empty, torch.zeros_like(allk[:, :cap]), allk.gather(1, idx))
    f = torch.where(empty, torch.full_like(f, -1), f)
    r = None
    if rows is not None:
        old = idx < cap
        kept = rows.gather(1, idx.clamp(max=cap - 1)[..., None].expand(-1, -1, L))
        new = fragment_values(code, torch.where(old | empty, torch.full_like(f, -1), f - frag0), L).to(rows.dtype)
        r = torch.where(empty[..., None], torch.zeros_like(kept), torch.where(old[..., None], kept, new))
    return k, f, r


def merge_call(top, rnd, fmax: torch.Tensor, active: torch.Tensor, frag0: int, seed: int, code: torch.Tensor = None,
               L: int = None):
    """One sce_forward_fragments call on the caller's lists: what fragment_merge_kernel leaves in them.

    ``top`` = (values [n, n_top], fragments [n, n_top], rows [n, n_top, L] or None) and ``rnd`` = (keys [n, n_random],
    fragments, rows) as the caller holds them, an entry with fragment < 0 empty whatever its key and rows; ``fmax`` /
    ``active`` [G, n]: the call's fragment maxima and activity (fragment_tables), its fragment g being frag0 + g; ``code``
    [G L, n]: the call's code, where rows are wanted. Returns (top, rnd) in the same form, as sets: each list in list
    order, its empty entries last with key 0, fragment -1 and zero rows. A list of length 0 passes through.

    The top list keeps the n_top highest (maximum, fragment) over its entries and every fragment of the call; the random
    list the n_random highest (priority, fragment) over its entries and the call's active fragments."""
    G, n = fmax.shape
    frags = frag0 + torch.arange(G, device=fmax.device)
    cand = frags[:, None].expand(G, n).T                                         # [n, G]
    out_top = _keep(*top, fmax.T, cand, frag0, code, L, top[1].shape[1])
    p = priority(seed, torch.arange(n, device=fmax.device), frags).T
    out_rnd = _keep(*rnd, p, torch.where(active.T, cand, torch.full_like(cand, -1)), frag0, code, L, rnd[1].shape[1])
    return out_top, out_rnd


def empty_lists(n: int, k: int, L: int = None, key_dtype=torch.float64, row_dtype=torch.float64, device=None):
    """n lists of length k with every entry empty, as merge_call takes them (rows only when L is given)."""
    rows = torch.zeros(n, k, L, dtype=row_dtype, device=device) if L else None
    return (torch.zeros(n, k, dtype=key_dtype, device=device), torch.full((n, k), -1, dtype=torch.int64, device=device),
            rows)


def value_bounds(S: torch.Tensor, e: float, L: int):
    """Per-element bounds of the engine's code values and fragment maxima from the code's element bar ``e``
    (tile_bounds.BARS / TOPK_BARS) and its scale S [N, n] (tile_bounds.code_scale; top-k: on the pinned support). The
    engine's code is relu of its fp32 pre-activation, and relu is 1-Lipschitz, so |c' - c| <= e S per element (the
    argument of oracle/eval_bounds.py); a maximum moves by at most the largest bound of its fragment's elements:
    |max_t c'_t - max_t c_t| <= max_t e S_t. Returns (code bound [N, n], fragment-maximum bound [G, n])."""
    b = e * S.double().abs()
    return b, b.reshape(S.shape[0] // L, L, -1).amax(1)


def top_ratios(values: torch.Tensor, frags: torch.Tensor, fmax: torch.Tensor, fbound: torch.Tensor):
    """The engine's top lists ([n, n_top] values and fragments, numbered as the rows of ``fmax``; -1 empty) against the
    fp64 fragment maxima ``fmax`` [G, n] and their bounds ``fbound`` (value_bounds). Returns per entry, [n, n_top]:
      value   |value - fmax[frag]| / fbound[frag]
      set     for a fragment the fp64 top list does not hold: (m_k - fmax[frag]) / (fbound[frag] + fbound[k-th]), m_k
              the fp64 n_top-th maximum, so it may stand in for the k-th only within both bounds (0 otherwise)
    Ratios above 1 fail; a NaN value is an infinite ratio."""
    n_top = frags.shape[1]
    ref = select_top(fmax, n_top)
    on = frags >= 0
    f = frags.clamp(min=0)
    want, fb = fmax.T.gather(1, f), fbound.T.gather(1, f)
    err = (values.double() - want).abs()
    err = torch.where(torch.isnan(err), torch.full_like(err, float("inf")), err)
    value = torch.where(on & (err > 0), err / fb, torch.zeros_like(err))
    kth = ref[:, -1:].clamp(min=0)
    m_k, fb_k = fmax.T.gather(1, kth), fbound.T.gather(1, kth)
    extra = on & ~(frags[..., None] == ref[:, None, :]).any(-1)
    gap = (m_k - want).clamp(min=0.0)
    return {"value": value, "set": torch.where(extra & (gap > 0), gap / (fb + fb_k), torch.zeros_like(gap))}
